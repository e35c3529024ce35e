#!/usr/bin/env python
"""A truncated-BPTT training step with torch_module.PercepNet against the plain step on the same GPU.

    python tools/bench_torch_state.py [--shapes 10x500,32x500,128x2000] [--steps 3] [--runs 3] [--out FILE]

Variants, each zero_grad, forward, CustomLoss in torch, backward, torch.optim.Adam.step:
  plain       m(x): every window from zero state (tools/bench_torch_module.py's step)
  tbptt       out, s = m(x, s, return_state=True), then s = s.detach(): the state scattered in and gathered out
              (two launches of B x 3712 floats)
  state_grad  the same with the incoming state requiring a gradient: also dL/d(state in), one more recurrence step per
              GRU and the six history contractions
Records, warm-up and timing are bench_train.py's: random records at a moderate scale on the device, one warm-up step per
variant, then `runs` runs of `steps` steps alternating between the variants, each timed with CUDA events; the median and
the spread (max / min) are reported, with the card's name and power limit read in the same run.  Prints one JSON
object.  Needs a GPU; there is no CPU path.
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
from bench_torch_module import Module  # noqa: E402
from bench_train import card, records  # noqa: E402
from percepnet_b200 import torch_module as tm  # noqa: E402
from percepnet_b200.weights import synth_state_dict  # noqa: E402


class Stateful(Module):
    """Module's step carrying the state from one step to the next."""

    def __init__(self, sd, rec, state_grad):
        import torch
        super().__init__(sd, rec)
        self.name = "state_grad" if state_grad else "tbptt"
        self.state_grad = state_grad
        self.s = torch.zeros((rec.shape[0], tm.STATE_FLOATS), device=rec.device)

    def step(self, stream):
        import torch
        with torch.cuda.stream(torch.cuda.ExternalStream(stream)):
            self.opt.zero_grad(set_to_none=True)
            s = self.s.requires_grad_(True) if self.state_grad else self.s
            out, s_out = self.m(self.x, s, return_state=True)
            self.O.loss(out, self.y).backward()
            self.opt.step()
            self.s = s_out.detach()


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
        variants = [Module(sd, rec), Stateful(sd, rec, False), Stateful(sd, rec, True)]
        variants[0].name = "plain"
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
            row[v.name] = {"ms_per_step": round(med, 3), "spread": round(max(ms[v.name]) / min(ms[v.name]), 3)}
        for v in ("tbptt", "state_grad"):
            row[f"{v}_over_plain_ms"] = round(row[v]["ms_per_step"] - row["plain"]["ms_per_step"], 3)
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
