#!/usr/bin/env python
"""Cost of the split call on a session pool: pnb_analyze_sessions_device_f32 + pnb_compute_rnn_sessions_device +
pnb_synthesize_sessions_device_f32 against the fused pnb_process_sessions_device_f32 call on the same lists, under
churn, and a ragged leg against pnb_process_sessions_ragged_device_f32.  One JSON line.

  python tools/bench_split_sessions.py [--streams S] [--sessions N] [--frames F] [--steps K] [--warmup W]
                                       [--churn 0,0.01,0.1] [--ragged 8,9,10]

Defaults: one tensor engine of 16 384 slots and 20 000 sessions, calls of 10 hops, churn 0, 1 % and 10 % of the listed
sessions replaced by parked ones between calls (tools/bench_sessions.py), and a ragged leg at churn 0 whose hop counts
are drawn from {8, 9, 10} (one session at 10 in every call).  Fused and split legs run on the same engine and alternate
within each of three runs; frames/s (slots x call hops / s) from device events, median of the three.  The card's name,
power limit and SM clocks are read in the same run.
"""
from __future__ import annotations

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import make_step_inputs  # noqa: E402


def card_info(index=0):
    """Name, power limit and SM clocks (current and maximum, MHz) of the card, from nvidia-smi in the same run."""
    try:
        out = subprocess.run(["nvidia-smi", f"--id={index}",
                              "--query-gpu=name,power.limit,enforced.power.limit,clocks.sm,clocks.max.sm",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=20).stdout
        f = [x.strip() for x in out.strip().splitlines()[0].split(",")]
        return {"name": f[0], "power_limit_w": float(f[1]), "enforced_power_limit_w": float(f[2]),
                "sm_clock_mhz": float(f[3]), "sm_clock_max_mhz": float(f[4])}
    except Exception as ex:
        return {"name": None, "power_limit_w": None, "error": type(ex).__name__}


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
    pool = api.Engine(S, F, synth_model(0), api.NN_TENSOR)
    pool.reserve_sessions(N)
    n_buf = 3
    bufs = make_step_inputs(S, F, n_buf, 0, device)
    outs = [torch.empty_like(b) for b in bufs]
    feat = torch.empty((S, F, 70), dtype=torch.float32, device=device)
    gr = torch.empty((S, F, 68), dtype=torch.float32, device=device)
    stream = torch.cuda.current_stream()
    st = stream.cuda_stream
    evs = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    rng = np.random.RandomState(20261017)
    listed = rng.permutation(N)[:S].astype(np.int32)
    ragged_hops = np.array([int(h) for h in args.ragged.split(",")], np.int32)
    T = F * 480

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

    def hops_of(kind):
        if kind[0] != "ragged":
            return None
        h = rng.choice(ragged_hops, size=S).astype(np.int32)
        h[rng.randint(S)] = F
        return h

    def call(kind, i):
        """kind: (churn fraction or "ragged", "fused" | "split")."""
        b = i % n_buf
        ids = next_list(0.0 if kind[0] == "ragged" else kind[0])
        hops = hops_of(kind)
        x, y = bufs[b], outs[b]
        if kind[1] == "fused":
            pool.process_sessions_device(ids, x.data_ptr(), T, y.data_ptr(), T, F, 0, st, hops=hops)
        else:
            pool.analyze_sessions_device(ids, x.data_ptr(), T, F, feat.data_ptr(), F * 70, stream=st, hops=hops)
            pool.compute_rnn_sessions_device(ids, api.RNN_FEATURES, feat.data_ptr(), F * 70, F, gr.data_ptr(), F * 68,
                                             stream=st, hops=hops)
            pool.synthesize_sessions_device(ids, gr.data_ptr(), F * 68, F, y.data_ptr(), T, stream=st)

    fracs = [float(f) for f in args.churn.split(",") if f.strip()]
    kinds = [(f, leg) for f in fracs + ["ragged"] for leg in ("fused", "split")]
    res = {k: {"fps": [], "moves": []} for k in kinds}
    i = 0
    for k in kinds:                                            # warm every configuration
        for _ in range(W):
            call(k, i)
            i += 1
    pool.flush(st)
    torch.cuda.synchronize()
    for _ in range(3):
        for k in kinds:
            for _ in range(2):                                 # settle into this pattern
                call(k, i)
                i += 1
            before = pool.session_stats()
            pool.flush(st)
            evs[0].record(stream)
            for _ in range(K):
                call(k, i)
                i += 1
            pool.flush(st)
            evs[1].record(stream)
            torch.cuda.synchronize()
            after = pool.session_stats()
            res[k]["fps"].append(S * F * K / (evs[0].elapsed_time(evs[1]) * 1e-3))
            res[k]["moves"].append({m: (after[m] - before[m]) / K for m in after})
    pool.check(st)
    out = {}
    for f in fracs + ["ragged"]:
        name = "ragged" if f == "ragged" else f"churn_{f:g}"
        fused, split = (float(np.median(res[(f, leg)]["fps"])) for leg in ("fused", "split"))
        out[name] = {"fused_fps": fused, "split_fps": split, "split_vs_fused": split / fused,
                     "fused_fps_runs": [round(x) for x in res[(f, "fused")]["fps"]],
                     "split_fps_runs": [round(x) for x in res[(f, "split")]["fps"]],
                     "moves_per_call": {m: float(np.mean([x[m] for x in res[(f, "split")]["moves"]]))
                                        for m in ("parks", "unparks", "relocations")}}
    print(json.dumps({
        "metric": "session_split_vs_fused", "value": out[f"churn_{fracs[0]:g}"]["split_vs_fused"], "unit": "ratio",
        "n_gpus": 1, "steps": K, "warmup": W, "higher_is_better": True, "data": "synthetic",
        "config": {"slots": S, "sessions": N, "frames_per_call": F, "nn": "tensor", "runs": 3,
                   "ragged_hops": ragged_hops.tolist()},
        "card": card, "results": out,
        "note": ("frames/s (slots x call hops / s) of back-to-back device calls without g/r out of the fused call: fused = "
                 "pnb_process_sessions_device_f32 (ragged leg: _ragged_), split = pnb_analyze_sessions_device_f32 + "
                 "pnb_compute_rnn_sessions_device + pnb_synthesize_sessions_device_f32 on the same lists and engine; "
                 "median of three alternated runs")}))
    pool.close()
    return 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=16384)
    ap.add_argument("--sessions", type=int, default=20000)
    ap.add_argument("--frames", type=int, default=10, help="hops per call (10 = a 100 ms serving cadence)")
    ap.add_argument("--steps", type=int, default=20, help="calls per timed run (at least 20)")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--churn", default="0,0.01,0.1", help="fractions of the listed sessions replaced between calls")
    ap.add_argument("--ragged", default="8,9,10", help="hop counts the ragged leg draws from (max = --frames)")
    return run(ap.parse_args())


if __name__ == "__main__":
    sys.exit(main())
