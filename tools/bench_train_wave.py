#!/usr/bin/env python
"""The waveform-training step of python -m percepnet_b200.train_wave: steps/s and hops/s, and where a step's device
time goes.

    python tools/bench_train_wave.py [--shapes 10x500,32x500] [--steps 10] [--warmup 3] [--out FILE]

For each shape B x W (B rows, windows of W hops) the CLI's step runs on synthetic pairs of 1 200 hops (three windows of
500 per track, the lag flushed), rows carrying their signal and network state from window to window and starting new
tracks as the schedule gives them: host input assembly (train_wave.step_inputs, timed on the host clock), the copy to
the device, analysis and operand export, PercepNet forward, synthesis and loss, backward, Adam, and reading the loss
back as the CLI's log does.  CUDA events split each step's device time:
  signal + loss   analysis and export (analysis_ms), synthesis and the masked L1 (synthesis_loss_ms), and in the
                  backward the loss's and the synthesis's gradient (signal_backward_ms, up to the hook on g/r)
  percepnet       the module's forward and its backward (from the hook on g/r to the end of backward)
  adam            torch.optim.Adam.step
Steps/s is the host clock over `steps` steps that end in a device synchronise, after `warmup` steps.  Prints one JSON
object per shape and one for the run, with the card's name and power limit read in the same run.  Needs a GPU.
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from percepnet_b200 import train_wave as TW  # noqa: E402

HOPS = 1200


def card():
    """(name, power limit) of cuda:0 from nvidia-smi, read in this run."""
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power = (q.stdout.strip().split(", ") + ["?", "?"])[:2]
    return name, power


def shape(B, W, steps, warmup):
    import torch
    from percepnet_b200.synth import synth_pairs
    from percepnet_b200.torch_module import STATE_FLOATS, PercepNet
    from percepnet_b200.torch_signal import SignalPath
    from percepnet_b200.weights import synth_state_dict
    n_pairs = B + 3
    clean, noisy = synth_pairs(n_pairs, HOPS, seed=960)
    data = [(clean[k], noisy[k]) for k in range(n_pairs)]
    hops = [HOPS] * n_pairs
    dev = torch.device("cuda", 0)
    net = PercepNet()
    net.load_state_dict({k: torch.from_numpy(v) for k, v in synth_state_dict(0).items()})
    net = net.to(dev)
    opt = torch.optim.Adam(net.parameters(), lr=1e-4)
    sp = SignalPath(B, W, device=dev)
    state = torch.zeros((B, STATE_FLOATS), device=dev)
    cur = TW.first_cursor(n_pairs, B, 0)
    parts = {"signal_loss_ms": [], "analysis_ms": [], "synthesis_loss_ms": [], "signal_backward_ms": [],
             "percepnet_ms": [], "adam_ms": [], "host_inputs_ms": []}

    def step():
        nonlocal cur, state
        new = [b for b in range(B) if cur.offset[b] == 0]
        if new:
            sp.reset(new)
            state[new] = 0
        t0 = time.perf_counter()
        x, tgt, lo, hi = TW.step_inputs(data, cur, W)
        t1 = time.perf_counter()
        count = int((hi - lo).sum())
        xt, tt = torch.from_numpy(x).to(dev).float(), torch.from_numpy(tgt).to(dev).float()
        lo_t, hi_t = torch.from_numpy(lo).to(dev), torch.from_numpy(hi).to(dev)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(7)]
        ev[0].record()
        features, ops = sp.analyze(xt)
        ev[1].record()
        gr, state_out = net(features, state, return_state=True)
        ev[2].record()
        loss = TW.masked_l1(sp.synthesize(gr, ops), tt, lo_t, hi_t, count)
        ev[3].record()
        gr.register_hook(lambda g: ev[4].record())
        opt.zero_grad()
        loss.backward()
        ev[5].record()
        opt.step()
        ev[6].record()
        state = state_out.detach()
        loss.item()      # the CLI logs every step's loss, which waits for the step
        cur = TW.next_cursor(cur, hops, W, 0)
        return ev, (t1 - t0) * 1e3

    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    evs = []
    t0 = time.perf_counter()
    for _ in range(steps):
        ev, host_ms = step()
        evs.append(ev)
        parts["host_inputs_ms"].append(host_ms)
    torch.cuda.synchronize()
    wall = time.perf_counter() - t0
    for ev in evs:
        t = lambda i, j: ev[i].elapsed_time(ev[j])  # noqa: E731
        parts["signal_loss_ms"].append(t(0, 1) + t(2, 3) + t(3, 4))
        parts["analysis_ms"].append(t(0, 1))
        parts["synthesis_loss_ms"].append(t(2, 3))
        parts["signal_backward_ms"].append(t(3, 4))
        parts["percepnet_ms"].append(t(1, 2) + t(4, 5))
        parts["adam_ms"].append(t(5, 6))
    row = {"rows": B, "window": W, "steps": steps, "step_ms": round(wall / steps * 1e3, 2),
           "steps_per_s": round(steps / wall, 3), "hops_per_s": round(steps * B * W / wall, 1)}
    for k, v in parts.items():
        row[k] = round(float(np.median(v)), 3)
    row["signal_loss_share"] = round(row["signal_loss_ms"] / row["step_ms"], 4)
    sp.close()
    net.close()
    del net, opt, state
    torch.cuda.empty_cache()
    return row


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--shapes", default="10x500,32x500")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out")
    a = ap.parse_args()
    name, power = card()
    result = {"card": name, "power_limit": power, "shapes": []}
    for shp in a.shapes.split(","):
        B, W = (int(s) for s in shp.split("x"))
        row = shape(B, W, a.steps, a.warmup)
        result["shapes"].append(row)
        print(json.dumps(row), flush=True)
    print(json.dumps(result))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
