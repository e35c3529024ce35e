#!/usr/bin/env python
"""Cost of the split call (pnb_analyze_device_* / pnb_synthesize_device_*) against the fused pnb_process_device_* call
of the same shape, on device buffers, on one tensor engine.

    python tools/bench_split.py [--streams 16384] [--frames 100] [--calls 3] [--warmup 1] [--runs 3] [--out FILE]

Three legs, each `calls` calls per timed run, the legs alternating within every run (`runs` runs, median reported):
  process        pnb_process_device_f32
  split          pnb_analyze_device_f32 + pnb_synthesize_device_f32 (g/r fixed at 0.5: the signal path alone)
  split+network  pnb_analyze_device_f32 + pnb_compute_rnn_device + pnb_synthesize_device_f32 (the fused call's work
                 plus the four layout moves between the caller's rows and the per-call buffers)
A run is timed with CUDA events on the launching stream.  One profiled call of each leg then gives every launch's
device time in launch order (pnb_profile_timeline), so the layout moves (class stage_in_kernel) can be read off
directly.  Prints one JSON object per leg (and writes them to --out), with the card name and power limit read in the
same run.  Needs a GPU; there is no CPU path.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from percepnet_b200 import api  # noqa: E402
from percepnet_b200.synth import synth_pcm  # noqa: E402
from percepnet_b200.weights import synth_model  # noqa: E402


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        power = q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return name, power


def main():
    import torch
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--streams", type=int, default=16384)
    ap.add_argument("--frames", type=int, default=100)
    ap.add_argument("--calls", type=int, default=3, help="calls per leg per timed run")
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", help="also write the JSON lines to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_split: no CUDA device")
    S, F, T = a.streams, a.frames, a.frames * 480
    name, power = card()
    base = torch.from_numpy(synth_pcm(64, F, seed=20261017)).cuda()
    x = (base[torch.arange(S, device="cuda") % 64] * (0.25 + torch.rand(S, 1, device="cuda"))).contiguous()
    del base
    y = torch.empty_like(x)
    feat = torch.empty((S, F, 70), dtype=torch.float32, device="cuda")
    gr = torch.full((S, F, 68), 0.5, dtype=torch.float32, device="cuda")
    eng = api.Engine(S, F, synth_model(0), api.NN_TENSOR)

    def process():
        eng.process_device(x.data_ptr(), T, y.data_ptr(), T, F)

    def split():
        eng.analyze_device(x.data_ptr(), T, F, feat.data_ptr(), F * 70)
        eng.synthesize_device(gr.data_ptr(), F * 68, F, y.data_ptr(), T)

    def split_network():
        eng.analyze_device(x.data_ptr(), T, F, feat.data_ptr(), F * 70)
        eng.compute_rnn_device(api.RNN_FEATURES, feat.data_ptr(), F * 70, F, gr.data_ptr(), F * 68)
        eng.synthesize_device(gr.data_ptr(), F * 68, F, y.data_ptr(), T)

    legs = {"process": process, "split": split, "split+network": split_network}
    for leg in legs.values():
        for _ in range(a.warmup):
            leg()
    eng.check()
    gr.fill_(0.5)
    times = {k: [] for k in legs}
    st = torch.cuda.current_stream()
    for _ in range(a.runs):
        for k, leg in legs.items():
            if k == "split":
                gr.fill_(0.5)   # split+network overwrote it with the network's g/r
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record(st)
            for _ in range(a.calls):
                leg()
            eng.flush()
            t1.record(st)
            t1.synchronize()
            times[k].append(t0.elapsed_time(t1) / a.calls)
    eng.check()
    ms = {k: float(np.median(v)) for k, v in times.items()}
    moved = S * F * (70 + 68) * 4 * 2   # bytes the split call's two moves (features out, g/r in) read and write
    lines = []
    for k, leg in legs.items():
        eng.profile(True)
        leg()
        tl = eng.profile_timeline()
        eng.profile(False)
        moves = [t1 - t0 for cls, t0, t1 in tl if cls == "stage_in_kernel"]
        r = {"tool": "bench_split", "leg": k, "engine": "tensor", "streams": S, "frames_per_call": F,
             "calls_per_run": a.calls, "runs_ms_per_call": [round(t, 3) for t in times[k]], "ms_per_call": round(ms[k], 3),
             "vs_process": round(ms[k] / ms["process"], 4),
             "profiled_launches_ms": [(cls, round(t1 - t0, 3)) for cls, t0, t1 in tl],
             "stage_in_class_ms": round(sum(moves), 3), "gpu": name, "power_limit": power}
        if k != "process":
            r["split_move_bytes"] = moved
        lines.append(json.dumps(r))
        print(lines[-1], flush=True)
    eng.check()
    eng.close()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
