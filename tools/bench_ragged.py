#!/usr/bin/env python
"""Ragged session calls: frames/s of the hops actually advanced when every session of a pool advances by its own number
of hops per call (pnb_process_sessions_ragged_device_f32).  One JSON line.

  python tools/bench_ragged.py [--streams S] [--frames F] [--steps K] [--warmup W] [--nn tensor|fp32]

Defaults: 16 384 slots and as many sessions, every session listed in every call, calls of F = 10 hops, tensor engine.
Configurations, alternated over three runs of K calls each, frames/s from device events:
  plain       pnb_process_sessions_device_f32 of F hops
  ragged_all  ragged calls with every hop count at F (the same launches as plain)
  jitter      hop counts uniform in {F-2, F-1, F}
  one_pct_1   1 % of the sessions at 1 hop, the rest at F
  split       what (jitter) costs without ragged calls: an (F-2)-hop call of everyone, then one pool call of one hop for
              the sessions with at least F-1 hops and one for those with F (the pool parks whoever a call does not list)
The fix-up launch's time per call comes from pnb_profile_timeline in a separate profiled run of (jitter) and (one_pct_1).
The card's name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench import make_step_inputs  # noqa: E402
from bench_churn import card_info  # noqa: E402

KINDS = ["plain", "ragged_all", "jitter", "one_pct_1", "split"]


def run(args):
    import torch
    from percepnet_b200 import api
    from percepnet_b200.weights import synth_model
    if not torch.cuda.is_available():
        print(json.dumps({"error": "no CUDA device: ragged calls have no CPU fallback"}))
        return 2
    S, F, K, W = args.streams, args.frames, max(args.steps, 20), max(args.warmup, 3)
    device = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    card = card_info(0)
    flags = api.NN_FP32 if args.nn == "fp32" else api.NN_TENSOR
    pool = api.Engine(S, F, synth_model(0), flags)
    pool.reserve_sessions(S)
    n_buf = 3
    bufs = make_step_inputs(S, F, n_buf, 0, device)
    outs = [torch.empty_like(b) for b in bufs]
    stream = torch.cuda.current_stream()
    st = stream.cuda_stream
    evs = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    rng = np.random.RandomState(20261016)
    ids = np.arange(S, dtype=np.int32)
    full = np.full(S, F, np.int32)
    jitter = [rng.randint(F - 2, F + 1, size=S).astype(np.int32) for _ in range(8)]
    one_pct = []
    for _ in range(8):
        h = full.copy()
        h[rng.choice(S, S // 100, replace=False)] = 1
        one_pct.append(h)
    hops_of = {"plain": [full], "ragged_all": [full], "jitter": jitter, "one_pct_1": one_pct, "split": jitter}

    def call(kind, i):
        """One tick of `kind`; returns the hops it advanced."""
        b = i % n_buf
        pin, pout, stride = bufs[b].data_ptr(), outs[b].data_ptr(), bufs[b].stride(0)
        h = hops_of[kind][i % len(hops_of[kind])]
        if kind == "plain":
            pool.process_sessions_device(ids, pin, stride, pout, stride, F, 0, st)
        elif kind == "split":
            pool.process_sessions_device(ids, pin, stride, pout, stride, F - 2, 0, st)
            for k in (F - 1, F):
                sel = ids[h >= k]
                if len(sel):
                    pool.process_sessions_device(sel, pin, stride, pout, stride, 1, 0, st)
        else:
            pool.process_sessions_device(ids, pin, stride, pout, stride, 0, 0, st, hops=h)
        return int(h.sum())

    res = {k: [] for k in KINDS}
    i = 0
    for k in KINDS:                                            # warm every configuration
        for _ in range(W):
            call(k, i)
            i += 1
    pool.flush(st)
    torch.cuda.synchronize()
    for _ in range(3):
        for k in KINDS:
            for _ in range(2):                                 # settle into this pattern
                call(k, i)
                i += 1
            pool.flush(st)
            evs[0].record(stream)
            hops = 0
            for _ in range(K):
                hops += call(k, i)
                i += 1
            pool.flush(st)
            evs[1].record(stream)
            torch.cuda.synchronize()
            res[k].append(hops / (evs[0].elapsed_time(evs[1]) * 1e-3))
    pool.check(st)
    # the fix-up's time: the slide-class launch right after each call's synthesis (a history slide, when there is one,
    # follows the fix-up)
    fixup = {}
    for k in ("jitter", "one_pct_1"):
        pool.profile(True)
        for _ in range(K):
            call(k, i)
            i += 1
        tl = pool.profile_timeline(cap=1 << 16)
        pool.profile(False)
        ms = [t1 - t0 for (c0, _, _), (c, t0, t1) in zip(tl, tl[1:]) if c0 == "synthesis_kernel" and c == "slide_history_kernel"]
        fixup[k] = {"ms_per_call": float(np.median(ms)) if ms else None, "calls": len(ms)}
    pool.check(st)
    base = float(np.median(res["plain"]))
    out = {k: {"fps": float(np.median(v)), "fps_runs": [round(x) for x in v], "vs_plain": float(np.median(v)) / base}
           for k, v in res.items()}
    print(json.dumps({
        "metric": "ragged_session_frames_per_sec", "value": out["jitter"]["fps"], "unit": "frames/s", "n_gpus": 1,
        "steps": K, "warmup": W, "higher_is_better": True, "data": "synthetic",
        "config": {"slots": S, "sessions": S, "frames_per_call": F, "nn": args.nn, "runs": 3},
        "card": card, "results": out, "fixup": fixup,
        "note": ("frames/s of the hops actually advanced (sum of hops / s) of back-to-back session calls without g/r, every "
                 "session listed in every call; median of three alternated runs; fixup: median device time of the "
                 "ragged call's fix-up launch from pnb_profile_timeline")}))
    pool.close()
    return 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=16384)
    ap.add_argument("--frames", type=int, default=10, help="hops per call (10 = a 100 ms serving cadence)")
    ap.add_argument("--steps", type=int, default=20, help="calls per timed run (at least 20)")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--nn", default="tensor", choices=["tensor", "fp32"])
    return run(ap.parse_args())


if __name__ == "__main__":
    sys.exit(main())
