#!/usr/bin/env python
"""Session pool under churn: frames/s of the advanced sessions when every call lists a subset of the pool's sessions
(pnb_process_sessions_device_f32) and a fraction of the listed sessions is replaced by parked ones between calls.  One
JSON line.

  python tools/bench_sessions.py [--streams S] [--sessions N] [--frames F] [--steps K] [--warmup W] [--nn tensor|fp32]
                                 [--churn 0,0.01,0.1]

Defaults: 16 384 slots, 20 000 sessions, calls of 10 hops, churn 0, 1 % and 10 %.  The baseline is plain
pnb_submit_device_f32 calls of all 16 384 slots on a second engine of the same shape (an engine in session mode refuses
the slot-level calls).  Configurations are alternated over three runs; frames/s from device events.  Moves per call from
pnb_session_stats; state bytes per second computed from the shapes (tools/bench_churn.py).  The card's name and power
limit are read in the same run.
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
from bench_churn import STATE_BLOB, STATE_GRU, STATE_GRU_F16, STATE_HIST, STATE_SIGNAL, STATE_TERMS, card_info  # noqa: E402


def move_bytes(nn_mode):
    """(park, unpark, relocation) bytes per session: engine side read + blob written; blob read + engine side written
    (the fp16 GRU terms too on tensor engines); engine side read and written raw."""
    if nn_mode == "tensor":
        eng = STATE_SIGNAL + STATE_GRU + STATE_TERMS
        return eng + STATE_BLOB, STATE_BLOB + eng + STATE_GRU_F16, 2 * (eng + STATE_GRU_F16)
    eng = STATE_SIGNAL + STATE_GRU + STATE_HIST
    return eng + STATE_BLOB, STATE_BLOB + eng, 2 * eng


def run(args):
    import torch
    from percepnet_b200 import api
    from percepnet_b200.weights import synth_model
    if not torch.cuda.is_available():
        print(json.dumps({"error": "no CUDA device: the session pool has no CPU fallback"}))
        return 2
    S, N, F, K, W = args.streams, args.sessions, args.frames, max(args.steps, 20), max(args.warmup, 3)
    device = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    card = card_info(0)
    nn_mode = "fp32" if args.nn == "fp32" else "tensor"
    flags = api.NN_FP32 if nn_mode == "fp32" else api.NN_TENSOR
    model = synth_model(0)
    plain = api.Engine(S, F, model, flags)
    pool = api.Engine(S, F, model, flags)
    pool.reserve_sessions(N)
    n_buf = 3
    bufs = make_step_inputs(S, F, n_buf, 0, device)
    outs = [torch.empty_like(b) for b in bufs]
    stream = torch.cuda.current_stream()
    st = stream.cuda_stream
    evs = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    rng = np.random.RandomState(20261015)
    listed = rng.permutation(N)[:S].astype(np.int32)

    def next_list(f):
        """Replace a fraction f of the listed sessions by parked ones (at the same list rows)."""
        nonlocal listed
        m = int(round(f * S))
        if m:
            parked = np.setdiff1d(np.arange(N, dtype=np.int32), listed, assume_unique=True)
            rows = rng.choice(S, m, replace=False)
            listed = listed.copy()
            listed[rows] = rng.choice(parked, m, replace=False)
        return listed

    def call(kind, i):
        b = i % n_buf
        if kind == "plain":
            plain.submit_device(bufs[b].data_ptr(), bufs[b].stride(0), outs[b].data_ptr(), outs[b].stride(0), F, stream=st)
        else:
            pool.process_sessions_device(next_list(kind), bufs[b].data_ptr(), bufs[b].stride(0), outs[b].data_ptr(),
                                         outs[b].stride(0), F, 0, st)

    fracs = [float(f) for f in args.churn.split(",") if f.strip()]
    kinds = ["plain"] + fracs
    res = {k: {"fps": [], "moves": []} for k in kinds}
    i = 0
    for k in kinds:                                            # warm every configuration
        for _ in range(W):
            call(k, i)
            i += 1
    for e in (plain, pool):
        e.flush(st)
    torch.cuda.synchronize()
    for _ in range(3):
        for k in kinds:
            for _ in range(2):                                 # settle into this pattern
                call(k, i)
                i += 1
            before = pool.session_stats()
            (plain if k == "plain" else pool).flush(st)
            evs[0].record(stream)
            for _ in range(K):
                call(k, i)
                i += 1
            (plain if k == "plain" else pool).flush(st)
            evs[1].record(stream)
            torch.cuda.synchronize()
            after = pool.session_stats()
            res[k]["fps"].append(S * F * K / (evs[0].elapsed_time(evs[1]) * 1e-3))
            res[k]["moves"].append({m: (after[m] - before[m]) / K for m in after})
    plain.check(st)
    pool.check(st)
    b_park, b_unpark, b_reloc = move_bytes(nn_mode)
    base = float(np.median(res["plain"]["fps"]))
    out = {"plain": {"fps": base, "fps_runs": [round(x) for x in res["plain"]["fps"]]}}
    for f in fracs:
        r = res[f]
        fps = float(np.median(r["fps"]))
        mv = {m: float(np.mean([x[m] for x in r["moves"]])) for m in ("parks", "unparks", "relocations")}
        calls_per_s = fps / (S * F)
        bps = calls_per_s * (mv["parks"] * b_park + mv["unparks"] * b_unpark + mv["relocations"] * b_reloc)
        out[f"{f:g}"] = {"fps": fps, "fps_runs": [round(x) for x in r["fps"]], "vs_plain": fps / base,
                         "moves_per_call": mv, "state_gb_per_s": bps / 1e9}
    print(json.dumps({
        "metric": "session_pool_frames_per_sec", "value": out[f"{fracs[0]:g}"]["fps"], "unit": "frames/s", "n_gpus": 1,
        "steps": K, "warmup": W, "higher_is_better": True, "data": "synthetic",
        "config": {"slots": S, "sessions": N, "frames_per_call": F, "nn": nn_mode, "runs": 3,
                   "bytes_per_move": {"park": b_park, "unpark": b_unpark, "relocation": b_reloc}},
        "card": card, "results": out,
        "note": ("frames/s of the advanced sessions (slots x hops / s) of back-to-back pnb_process_sessions_device_f32 calls "
                 "without g/r; between calls a fraction of the listed sessions is replaced by parked ones; plain: "
                 "pnb_submit_device_f32 of all slots on a second engine of the same shape; median of three alternated runs")}))
    plain.close()
    pool.close()
    return 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=16384)
    ap.add_argument("--sessions", type=int, default=20000)
    ap.add_argument("--frames", type=int, default=10, help="hops per call (10 = a 100 ms serving cadence)")
    ap.add_argument("--steps", type=int, default=20, help="calls per timed run (at least 20)")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--nn", default="tensor", choices=["tensor", "fp32"])
    ap.add_argument("--churn", default="0,0.01,0.1", help="fractions of the listed sessions replaced between calls")
    return run(ap.parse_args())


if __name__ == "__main__":
    sys.exit(main())
