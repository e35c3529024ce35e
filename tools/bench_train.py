#!/usr/bin/env python
"""Steps per second of the GPU trainer (pnb_train_grad_device + pnb_train_adam) against the same training step in
torch on the same GPU (tests/train_oracle.py's restatement of rnn_train.PercepNet, cuDNN GRUs, torch.optim.Adam), in
float32 with TF32 allowed (cuDNN's default) and with TF32 off.

    python tools/bench_train.py [--shapes 10x500,32x500,128x2000] [--steps 3] [--runs 3] [--out FILE]

Shapes are windows x frames: 10 x 500 is train()'s batch of 500-frame sequences, 128 x 2000 the --train_length_size
default.  Records are random (features at a moderate scale, labels uniform in [0, 1]) and stay on the device.  Every
variant gets one warm-up step, then `runs` timed runs of `steps` steps each, alternating between the variants; a run
is timed with CUDA events and the median and the spread (max / min) over the runs are reported.  FLOP per step is
3 x 2 x the network's MACs per frame x frames (forward, and a backward twice its size).  One extra profiled step
(torch.profiler, CUDA activities) of the trainer splits its time by kernel into forward contractions, recurrence,
BPTT, backward contractions, weight gradients, Adam and the rest.  The card name and power limit are read in the same
run.  Prints one JSON object.  Needs a GPU; there is no CPU path.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from percepnet_b200 import api  # noqa: E402
from percepnet_b200.weights import MACS_PER_FRAME, pack_state_dict, synth_state_dict  # noqa: E402


def card():
    import torch
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        power = q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return torch.cuda.get_device_name(0), power


def records(B, T, seed=7):
    import torch
    g = torch.Generator(device="cuda").manual_seed(seed)
    r = torch.rand((B, T, 138), generator=g, device="cuda")
    r[..., :68] *= 0.05
    return r.contiguous()


class Ours:
    name = "gpu_trainer"

    def __init__(self, sd, rec):
        import torch
        self.B, self.T = rec.shape[0], rec.shape[1]
        self.eng = api.Engine(self.B, self.T, pack_state_dict(sd), api.TRAIN_NETWORK)
        self.rec = rec
        self.sums = torch.empty((self.B, 4), dtype=torch.float64, device="cuda")
        self.k = 0

    def step(self, stream):
        self.k += 1
        self.eng.train_grad_device(self.rec.data_ptr(), self.T * 138, self.T, None, self.sums.data_ptr(), stream)
        self.eng.train_adam(1e-4, self.k, stream)

    def close(self):
        self.eng.close()


class Torch:
    def __init__(self, sd, rec, tf32):
        import torch
        import train_oracle as O
        self.name = "torch_cudnn_tf32" if tf32 else "torch_cudnn_fp32"
        self.tf32 = tf32
        self.m = O.model(sd, torch.float32, "cuda")
        self.opt = torch.optim.Adam(self.m.parameters(), lr=1e-4)
        x = rec[..., :70].clone()
        x[..., :68] *= 30
        self.x, self.y, self.O = x, rec[..., 70:].contiguous(), O

    def step(self, stream):
        import torch
        torch.backends.cuda.matmul.allow_tf32 = self.tf32
        torch.backends.cudnn.allow_tf32 = self.tf32
        with torch.cuda.stream(torch.cuda.ExternalStream(stream)):
            self.opt.zero_grad(set_to_none=True)
            self.O.loss(self.m(self.x), self.y).backward()
            self.opt.step()

    def close(self):
        pass


PHASES = (("recurrence", ("gru_fwd_rec",)), ("bptt", ("gru_bwd_rec",)), ("weight_gradients", ("<true, false>", "train_parts")),
          ("backward_contractions", ("<false, true>",)), ("forward_contractions", ("<false, false>",)),
          ("adam", ("train_adam",)))


def phase_split(v, stream):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        v.step(stream)
        torch.cuda.synchronize()
    out = {p: 0.0 for p, _ in PHASES}
    out["other"] = 0.0
    for ev in prof.key_averages():
        t = ev.device_time_total / 1000.0 if hasattr(ev, "device_time_total") else ev.cuda_time_total / 1000.0
        if t <= 0:
            continue
        for p, keys in PHASES:
            if any(k in ev.key for k in keys):
                out[p] += t
                break
        else:
            out["other"] += t
    return {k: round(x, 3) for k, x in out.items()}


def main():
    import torch
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--shapes", default="10x500,32x500,128x2000")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out")
    a = ap.parse_args()
    name, power = card()
    result = {"card": name, "power_limit": power, "steps_per_run": a.steps, "runs": a.runs, "shapes": []}
    sd = synth_state_dict(0)
    stream = torch.cuda.Stream()
    for shp in a.shapes.split(","):
        B, T = (int(s) for s in shp.split("x"))
        rec = records(B, T)
        variants = [Ours(sd, rec), Torch(sd, rec, True), Torch(sd, rec, False)]
        for v in variants:
            v.step(stream.cuda_stream)
        torch.cuda.synchronize()
        ms = {v.name: [] for v in variants}
        for _ in range(a.runs):
            for v in variants:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                for _ in range(a.steps):
                    v.step(stream.cuda_stream)
                e1.record(stream)
                e1.synchronize()
                ms[v.name].append(e0.elapsed_time(e1) / a.steps)
        flop = 6.0 * MACS_PER_FRAME * B * T
        row = {"windows": B, "frames": T, "flop_per_step": flop}
        for v in variants:
            med = float(np.median(ms[v.name]))
            row[v.name] = {"ms_per_step": round(med, 3), "steps_per_s": round(1000 / med, 3),
                           "frames_per_s": round(B * T * 1000 / med, 1), "tflops": round(flop / med / 1e9, 2),
                           "spread": round(max(ms[v.name]) / min(ms[v.name]), 3)}
        row["phase_ms"] = phase_split(variants[0], stream.cuda_stream)
        for v in variants:
            v.close()
        del variants
        torch.cuda.empty_cache()
        result["shapes"].append(row)
        print(json.dumps(row), flush=True)
    print(json.dumps(result))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
