#!/usr/bin/env python
"""Session churn in a running engine: stream states moved per second by pnb_export_states + pnb_import_states,
serving throughput while slots are reset or moved between calls, and serving throughput at partial occupancy (the
engine's active range, pnb_set_active_streams).  One JSON line, in the style of bench.py's paths.

  python tools/bench_churn.py [--streams S] [--frames F] [--steps K] [--warmup W] [--nn tensor|fp32] [--churn 0.01]
                              [--active 0.25,0.5,0.75,1.0]

Defaults: 16 384 streams on the tensor path, calls of 10 hops (a 100 ms serving cadence), 1 % of the slots churned
before every call, occupancy sweep over a quarter, half, three quarters and all of the slots.  The card's name and power limit are read in the same run.  The inputs, clock sampling and peak
figures are bench.py's own (imported, not changed).
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
from bench import ClockSampler, make_step_inputs, measured_peaks  # noqa: E402


# Bytes one stream's state operation moves, from the shapes of StreamState (percepnet_b200/csrc/pnb_state.h) and of the
# engine buffers it is gathered from / scattered into (pnb_state.cu: state_segs, tc_state_segs).
STATE_BLOB = 63_804                                      # pnb_state_size()
STATE_SIGNAL = (5280 + 480 + 1 + 1 + 5 * 800 + 5 * 34) * 4  # history, overlap-add, pitch continuity, five spectrum slots
STATE_GRU = (4 * 512 + 128) * 4                          # fp32 GRU states
STATE_HIST = (4 * 128 + 2 * 512) * 4                     # fp32 conv histories (fp32 engines)
STATE_TERMS = 3 * (4 * 128 + 2 * 512) * 2                # their three bf16 term planes (tensor engines)
STATE_GRU_F16 = (4 * 512 + 128) * 2 * 2                  # fp16 hi / lo GRU terms (tensor engines, written on import)


def churn_bytes(nn_mode):
    """(export, import) bytes per stream: engine reads + blob writes, blob reads (+ the check kernel's) + engine writes"""
    if nn_mode == "tensor":
        eng = STATE_SIGNAL + STATE_GRU + STATE_TERMS
        export = eng + STATE_BLOB
        imp = (8 + 4 + STATE_SIGNAL + STATE_GRU + STATE_TERMS) + (8 + STATE_GRU) + eng + STATE_GRU_F16
    else:
        eng = STATE_SIGNAL + STATE_GRU + STATE_HIST
        export = eng + STATE_BLOB
        imp = (8 + eng) + 8 + eng
    return export, imp


def card_info(index=0):
    """Name and power limit of the card, read in the same run (nvidia-smi query; None when unavailable)."""
    try:
        out = subprocess.run(["nvidia-smi", f"--id={index}", "--query-gpu=name,power.limit,enforced.power.limit",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=20).stdout
        f = [x.strip() for x in out.strip().splitlines()[0].split(",")]
        return {"name": f[0], "power_limit_w": float(f[1]), "enforced_power_limit_w": float(f[2])}
    except Exception as ex:
        return {"name": None, "power_limit_w": None, "error": type(ex).__name__}


def run_churn(args):
    """Session churn in a running engine (pnb_reset_streams / pnb_export_states / pnb_import_states).
    value: stream states moved per second -- one state moved = exported and imported once -- for all S streams per
    repetition, device events, repeated for at least half a second.  serving: frames/s of back-to-back submitted calls
    with no churn, with `--churn` of the slots reset before every call, and with that fraction exported and imported
    (moved to other slots) before every call; the three alternate in one process."""
    import torch
    from percepnet_b200 import api
    from percepnet_b200.weights import synth_model
    if not torch.cuda.is_available():
        print(json.dumps({"error": "no CUDA device: the state kernels have no CPU fallback"}))
        return 2
    S, F, K, W = args.streams, args.frames, max(args.steps, 20), max(args.warmup, 3)
    device = torch.device("cuda", 0)
    torch.cuda.set_device(0)
    card = card_info(0)
    nn_mode = "fp32" if args.nn == "fp32" else "tensor"
    flags = api.NN_FP32 if nn_mode == "fp32" else api.NN_TENSOR
    eng = api.Engine(S, F, synth_model(0), flags)
    n_buf = 3
    bufs = make_step_inputs(S, F, n_buf, 0, device)
    outs = [torch.empty_like(b) for b in bufs]
    stream = torch.cuda.current_stream()
    st = stream.cuda_stream
    nb = eng.state_size

    def call(i):
        b = i % n_buf
        eng.submit_device(bufs[b].data_ptr(), bufs[b].stride(0), outs[b].data_ptr(), outs[b].stride(0), F, stream=st)
    for i in range(W):
        call(i)
    eng.flush(st)
    torch.cuda.synchronize()

    # ---- state throughput: export + import of all S streams
    every = np.arange(S)
    blobs = torch.empty((S, nb), dtype=torch.uint8, device=device)
    evs = [torch.cuda.Event(enable_timing=True) for _ in range(3)]

    def move_all():
        eng.export_states(every, blobs.data_ptr(), nb, stream=st)
        eng.import_states(every, blobs.data_ptr(), nb, stream=st)
    move_all()
    torch.cuda.synchronize()
    evs[0].record(stream)
    move_all()
    evs[1].record(stream)
    torch.cuda.synchronize()
    reps = max(3, int(np.ceil(0.5 / max(1e-6, evs[0].elapsed_time(evs[1]) * 1e-3))))
    sampler = ClockSampler(0)
    sampler.start()
    exp_ms = imp_ms = 0.0
    for _ in range(reps):                                  # export and import timed apart, back to back on one stream
        evs[0].record(stream)
        eng.export_states(every, blobs.data_ptr(), nb, stream=st)
        evs[1].record(stream)
        eng.import_states(every, blobs.data_ptr(), nb, stream=st)
        evs[2].record(stream)
        torch.cuda.synchronize()
        exp_ms += evs[0].elapsed_time(evs[1])
        imp_ms += evs[1].elapsed_time(evs[2])
    clocks = sampler.stop()
    eng.check(st)
    value = S * reps / ((exp_ms + imp_ms) * 1e-3)
    b_exp, b_imp = churn_bytes(nn_mode)
    peaks = measured_peaks()
    gbs = (b_exp + b_imp) * S * reps / ((exp_ms + imp_ms) * 1e-3) / 1e9
    roof = {"bound": "hbm", "kernel": "state_move_kernel (+ state_check_kernel on import)", "achieved": gbs,
            "peak": peaks["hbm_gbs"], "unit": "GB/s", "frac": gbs / peaks["hbm_gbs"], "peak_source": peaks["source"],
            "bytes_per_stream": {"export": b_exp, "import": b_imp, "blob": STATE_BLOB},
            "export_gbs": b_exp * S * reps / (exp_ms * 1e-3) / 1e9, "import_gbs": b_imp * S * reps / (imp_ms * 1e-3) / 1e9}

    # ---- serving: back-to-back submitted calls with and without churn, alternated
    rng = np.random.RandomState(20261015)
    n_churn = max(1, int(round(args.churn * S)))
    small = torch.empty((n_churn, nb), dtype=torch.uint8, device=device)

    def before(kind):
        if kind == "reset":
            eng.reset_streams(rng.choice(S, n_churn, replace=False), stream=st)
        elif kind == "move":
            src = rng.choice(S, n_churn, replace=False)
            eng.export_states(src, small.data_ptr(), nb, stream=st)
            eng.import_states(rng.permutation(src), small.data_ptr(), nb, stream=st)

    kinds = ("none", "reset", "move")
    fps = {k: [] for k in kinds}
    i = W
    for _ in range(3):
        for kind in kinds:
            for _ in range(2):                             # settle the schedule into this pattern
                before(kind)
                call(i)
                i += 1
            eng.flush(st)
            evs[0].record(stream)
            for _ in range(K):
                before(kind)
                call(i)
                i += 1
            eng.flush(st)
            evs[1].record(stream)
            torch.cuda.synchronize()
            fps[kind].append(S * F * K / (evs[0].elapsed_time(evs[1]) * 1e-3))
    eng.check(st)

    # ---- occupancy: calls advance only the first n = fraction x S slots; fractions alternated over three runs
    fracs = [float(f) for f in args.active.split(",") if f.strip()]
    occ = {f: {"n": max(1, min(S, int(round(f * S)))), "fps": [], "ms": []} for f in fracs}
    for _ in range(3):
        for f in fracs:
            n = occ[f]["n"]
            eng.set_active(n, stream=st)                   # a grow resets the entering slots (not timed)
            for _ in range(2):
                call(i)
                i += 1
            eng.flush(st)
            evs[0].record(stream)
            for _ in range(K):
                call(i)
                i += 1
            eng.flush(st)
            evs[1].record(stream)
            torch.cuda.synchronize()
            ms = evs[0].elapsed_time(evs[1])
            occ[f]["fps"].append(n * F * K / (ms * 1e-3))
            occ[f]["ms"].append(ms / K)
    for f in fracs:                                        # per-class kernel time of one profiled call
        eng.set_active(occ[f]["n"], stream=st)
        call(i)
        i += 1
        eng.flush(st)
        torch.cuda.synchronize()
        eng.profile(True)
        call(i)
        i += 1
        eng.flush(st)
        occ[f]["kernel_ms"] = {k: round(v[0], 4) for k, v in eng.profile_read().items()}
        eng.profile(False)
    eng.check(st)
    eng.close()
    full_ms = float(np.median(occ[max(fracs)]["ms"]))
    occupancy = {"runs_per_fraction": 3, "calls_per_run": K, "note": (
        "frames/s of live streams (n x hops / s) and ms per call of back-to-back pnb_submit_device_f32 calls after "
        "pnb_set_active_streams(n); fractions alternated in one process, median of three runs; kernel_ms: per-class "
        "device time of one profiled call (pnb_profile_read); ms_vs_largest: ms per call relative to the largest fraction")}
    for f in fracs:
        o = occ[f]
        ms = float(np.median(o["ms"]))
        occupancy[f"{f:g}"] = {"active": o["n"], "fps": float(np.median(o["fps"])), "fps_runs": [round(x) for x in o["fps"]],
                               "ms_per_call": ms, "ms_vs_largest": ms / full_ms, "kernel_ms": o["kernel_ms"]}
    serving = {k: {"value": float(np.median(v)), "runs": [round(x) for x in v]} for k, v in fps.items()}
    serving["calls_per_run"] = K
    serving["churn"] = args.churn
    serving["slots_per_call"] = n_churn
    serving["note"] = ("frames/s of back-to-back pnb_submit_device_f32 calls; reset: pnb_reset_streams of the slots before "
                       "every call; move: pnb_export_states + pnb_import_states of the slots (to a permutation of them) "
                       "before every call; slots drawn by a seeded RNG; median of three alternated runs")
    print(json.dumps({
        "metric": "stream_states_moved_per_sec", "value": value, "unit": "states/s", "n_gpus": 1, "steps": reps,
        "warmup": W, "higher_is_better": True, "dtype": "bytes (fp32 / bf16 / fp16 state as stored)", "data": "synthetic",
        "config": {"workload": f"export + import of all {S} streams per repetition ({nn_mode} engine, {F}-hop calls)",
                   "streams": S, "frames_per_call": F, "nn": nn_mode,
                   "repetitions": reps, "export_ms": exp_ms / reps, "import_ms": imp_ms / reps},
        "card": card, "clocks": clocks, "roofline": roof, "serving": serving, "occupancy": occupancy}))
    return 0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", type=int, default=16384)
    ap.add_argument("--frames", type=int, default=10, help="hops per call (10 = a 100 ms serving cadence)")
    ap.add_argument("--steps", type=int, default=20, help="calls per timed serving run (at least 20)")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--nn", default="tensor", choices=["tensor", "fp32"])
    ap.add_argument("--churn", type=float, default=0.01, help="fraction of the slots reset / moved before every call")
    ap.add_argument("--active", default="0.25,0.5,0.75,1.0", help="occupancy sweep: fractions of the slots the calls advance")
    return run_churn(ap.parse_args())


if __name__ == "__main__":
    sys.exit(main())
