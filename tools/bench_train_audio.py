#!/usr/bin/env python
"""Cost of the training-data generator's ideal-gain audio: a records-only engine (PNB_TRAIN_DATA, pnb_train_records_device)
next to an audio engine (PNB_TRAIN_DATA | PNB_TRAIN_AUDIO, pnb_train_audio_device) on the same device-resident int16
pairs.

    python tools/bench_train_audio.py [--pairs 8192] [--frames 64] [--calls 20] [--warmup 3] [--runs 3] [--out FILE]

The default shape is gen_features' batch of 8 192 pairs (16 384 analysed streams) in calls of its default 64 frames.
The pairs are 64 synthetic speech / speech-plus-noise pairs, each row one of them shifted by its own number of frames.
Each engine gets `warmup` calls, then `runs` timed runs of `calls` calls each, alternating between the engines; a run
is timed with CUDA events on the launching stream and the median run is reported.  A separate profiled call of each
gives the per-kernel-class split (pnb_profile_read).  The device memory an engine takes is the drop in
cudaMemGetInfo's free bytes across its pnb_create.  Prints one JSON object per engine (and writes them to --out), with
the card name and power limit read in the same run.  Needs a GPU; there is no CPU path.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from percepnet_b200 import api  # noqa: E402
from percepnet_b200.synth import synth_pairs  # noqa: E402


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


def pair_rows(N, F, seed=20261017):
    """(speech, noisy) [N, F*480] int16 on the device."""
    import torch
    c, n = synth_pairs(64, F, seed=seed)
    rng = np.random.RandomState(seed)
    rows, shift = np.arange(N) % 64, rng.randint(0, F, N) * 480
    c = np.stack([np.roll(c[r], s) for r, s in zip(rows, shift)])
    n = np.stack([np.roll(n[r], s) for r, s in zip(rows, shift)])
    return torch.from_numpy(c).cuda(), torch.from_numpy(n).cuda()


def split(prof):
    return {k: round(v[0], 3) for k, v in sorted(prof.items())}


def main():
    import torch
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--pairs", type=int, default=8192)
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--calls", type=int, default=20, help="calls per timed run")
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", help="also write the JSON lines to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_train_audio: no CUDA device")
    N, F = a.pairs, a.frames
    name, power = card()
    speech, noisy = pair_rows(N, F)
    rec = torch.empty((N, F, 138), dtype=torch.float32, device="cuda")
    audio = torch.empty((N, F * 480), dtype=torch.int16, device="cuda")
    torch.cuda.synchronize()
    engines, mem = {}, {}
    for mode, flags in (("records", api.TRAIN_DATA), ("audio", api.TRAIN_DATA | api.TRAIN_AUDIO)):
        free0 = torch.cuda.mem_get_info()[0]
        engines[mode] = api.Engine(2 * N, F, None, flags)
        mem[mode] = free0 - torch.cuda.mem_get_info()[0]

    def call(mode):
        eng = engines[mode]
        if mode == "audio":
            eng.train_audio_device(speech.data_ptr(), F * 480, noisy.data_ptr(), F * 480, F, rec.data_ptr(), F * 138,
                                   audio.data_ptr(), F * 480)
        else:
            eng.train_records_device(speech.data_ptr(), F * 480, noisy.data_ptr(), F * 480, F, rec.data_ptr(), F * 138)

    for mode, eng in engines.items():
        for _ in range(a.warmup):
            call(mode)
        eng.check()
    times = {m: [] for m in engines}
    st = torch.cuda.current_stream()
    for _ in range(a.runs):
        for mode, eng in engines.items():
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record(st)
            for _ in range(a.calls):
                call(mode)
            eng.flush()
            t1.record(st)
            t1.synchronize()
            times[mode].append(t0.elapsed_time(t1) / a.calls)
    lines = []
    for mode, eng in engines.items():
        eng.check()
        eng.profile(True)
        call(mode)
        prof = eng.profile_read()
        eng.profile(False)
        ms = float(np.median(times[mode]))
        r = {"tool": "bench_train_audio", "engine": mode, "pairs": N, "streams": 2 * N, "frames_per_call": F,
             "calls_per_run": a.calls, "runs_ms_per_call": [round(t, 3) for t in times[mode]], "ms_per_call": round(ms, 3),
             "pair_frames_per_s": N * F / (ms / 1e3), "call_split_ms": split(prof),
             "engine_device_bytes": int(mem[mode]), "gpu": name, "power_limit": power}
        lines.append(json.dumps(r))
        print(lines[-1], flush=True)
    for eng in engines.values():
        eng.close()
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")


if __name__ == "__main__":
    main()
