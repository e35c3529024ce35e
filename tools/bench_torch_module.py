#!/usr/bin/env python
"""One training step with torch_module.PercepNet -- zero_grad, forward, CustomLoss in torch, backward,
torch.optim.Adam.step -- against the two baselines of tools/bench_train.py on the same GPU: the trainer's closed loop
(pnb_train_grad_device + pnb_train_adam) and train_oracle's model on cuDNN with TF32 allowed and with TF32 off.

    python tools/bench_torch_module.py [--shapes 10x500,32x500,128x2000] [--steps 3] [--runs 3] [--out FILE]

The module's step differs from the trainer's by the packing of the parameters into the blob (a 32 MB gather per
forward), the scatter of the blob gradient back to the parameters, torch's loss and its autograd, and torch's Adam on
30 tensors instead of one kernel.  The gather and the scatter are also timed on their own (20 of each, CUDA events).
Records, warm-up and timing are bench_train.py's: random records at a moderate scale on the device, one warm-up step
per variant, then `runs` runs of `steps` steps alternating between the variants, each timed with CUDA events; the
median and the spread (max / min) are reported, with the card's name and power limit read in the same run.  Prints
one JSON object.  Needs a GPU; there is no CPU path.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, os.path.join(ROOT, "tools"))
from bench_train import Ours, Torch, card, records  # noqa: E402
from percepnet_b200 import torch_module as tm  # noqa: E402
from percepnet_b200.weights import synth_state_dict  # noqa: E402


class Module:
    name = "torch_module"

    def __init__(self, sd, rec):
        import torch
        import train_oracle as O
        self.m = tm.PercepNet()
        self.m.load_state_dict({k: torch.from_numpy(np.asarray(v, np.float32)) for k, v in sd.items()})
        self.m.cuda()
        self.opt = torch.optim.Adam(self.m.parameters(), lr=1e-4)
        x = rec[..., :70].clone()
        x[..., :68] *= 30
        self.x, self.y, self.O = x, rec[..., 70:].contiguous(), O

    def step(self, stream):
        import torch
        with torch.cuda.stream(torch.cuda.ExternalStream(stream)):
            self.opt.zero_grad(set_to_none=True)
            self.O.loss(self.m(self.x), self.y).backward()
            self.opt.step()

    def engine_bytes(self):
        return sum(t.eng.device_bytes for t in self.m._trainers.values())

    def close(self):
        self.m.close()


def permutation_ms(mod, stream, n=20):
    """ms per gather (parameters -> blob) and per scatter (blob gradient -> parameters) of the module's index."""
    import torch
    idx = mod.m._index_on(mod.x.device)
    params = [p.detach() for p in mod.m.parameters()]
    out = {}
    with torch.cuda.stream(stream):
        flat = torch.cat([p.reshape(-1) for p in params])
        blob = tm.to_blob(flat, idx)
        for name, f in (("gather_ms", lambda: tm.to_blob(torch.cat([p.reshape(-1) for p in params]), idx)),
                        ("scatter_ms", lambda: tm.from_blob(blob, idx))):
            f()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for _ in range(n):
                f()
            e1.record(stream)
            e1.synchronize()
            out[name] = round(e0.elapsed_time(e1) / n, 3)
    return out


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
        variants = [Module(sd, rec), Ours(sd, rec), Torch(sd, rec, True), Torch(sd, rec, False)]
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
        row = {"windows": B, "frames": T}
        for v in variants:
            med = float(np.median(ms[v.name]))
            row[v.name] = {"ms_per_step": round(med, 3), "steps_per_s": round(1000 / med, 3),
                           "spread": round(max(ms[v.name]) / min(ms[v.name]), 3)}
        row["module_over_trainer_ms"] = round(row["torch_module"]["ms_per_step"] - row["gpu_trainer"]["ms_per_step"], 3)
        row["module_engine_bytes"] = variants[0].engine_bytes()
        row.update(permutation_ms(variants[0], stream))
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
