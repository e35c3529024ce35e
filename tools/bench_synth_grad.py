#!/usr/bin/env python
"""The synthesis's gradient on the GPU: the operand export, the synthesis and the backward, beside a PercepNet
forward + backward at the same shapes.

    python tools/bench_synth_grad.py [--shapes 10x500,32x500,128x2000,16384x100] [--reps 10] [--out FILE]

For each shape B x T (B rows of T hops) on a PNB_SIGNAL_ONLY engine with int16-scale synthetic PCM:
  export      pnb_synthesis_operands_device of the pending synthesis
  synthesis   pnb_synthesize_device_f32 (g/r stage + synthesis_kernel [+ history move]): the engine's profile gives
              synthesis_kernel alone
  backward    pnb_synthesis_backward_device
  percepnet   torch_module.PercepNet forward + backward with dL/d(out), up to 128 x 2000 hops (the trainer keeps about
              70 KB per hop: 16384 x 100 would take 115 GB)
Each is warmed up, then timed with CUDA events over `reps` repetitions (export and backward back to back; the
synthesis with a fresh analysis before each, timed alone).  The bytes each kernel must move are counted from the shapes.
Prints one JSON object per shape and one for the run, with the card's name and power limit read in the same run.
Needs a GPU; there is no CPU path.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from percepnet_b200 import api  # noqa: E402
from percepnet_b200.synth import synth_pcm  # noqa: E402

FRAME, OPS = 480, api.SYNTH_OPS_FLOATS


def card():
    """(name, power limit) of cuda:0 from nvidia-smi, read in this run."""
    q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                       capture_output=True, text=True)
    name, power = (q.stdout.strip().split(", ") + ["?", "?"])[:2]
    return name, power


def timed(fn, reps, before=None):
    """Median and spread of fn's device time over reps calls (CUDA events around each call; before() runs untimed)."""
    import torch
    ms = []
    for _ in range(reps):
        if before:
            before()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        ms.append(e0.elapsed_time(e1))
    return round(float(np.median(ms)), 4), round(max(ms) / min(ms), 3)


def shape(B, T, reps):
    import torch
    base = torch.from_numpy(synth_pcm(min(B, 64), T, seed=700, scale=32768.0)).cuda()
    x = base.repeat((B + base.shape[0] - 1) // base.shape[0], 1)[:B].contiguous()
    eng = api.Engine(B, T, None, api.SIGNAL_ONLY)
    st = torch.cuda.current_stream().cuda_stream
    feat = torch.empty((B, T, 70), device="cuda")
    ops = torch.empty((B, T * OPS), device="cuda")
    gr = torch.rand((B, T, 68), device="cuda")
    out = torch.empty((B, T * FRAME), device="cuda")
    dout = torch.randn((B, T * FRAME), device="cuda")
    dgr = torch.empty((B, T, 68), device="cuda")
    analyze = lambda: eng.analyze_device(x.data_ptr(), T * FRAME, T, feat.data_ptr(), T * 70, st)  # noqa: E731
    export = lambda: eng.synthesis_operands_device(ops.data_ptr(), T * OPS, st)  # noqa: E731
    synth = lambda: eng.synthesize_device(gr.data_ptr(), T * 68, T, out.data_ptr(), T * FRAME, st)  # noqa: E731
    backward = lambda: api.synthesis_backward_device(ops.data_ptr(), T * OPS, gr.data_ptr(), T * 68, B, T, False,  # noqa: E731
                                                     dout.data_ptr(), T * FRAME, dgr.data_ptr(), T * 68, st)
    analyze()
    export()
    synth()
    backward()
    torch.cuda.synchronize()
    row = {"rows": B, "frames": T}
    analyze()
    row["export_ms"], row["export_spread"] = timed(export, reps)
    synth()
    row["backward_ms"], row["backward_spread"] = timed(backward, reps)
    row["synthesize_ms"], row["synthesize_spread"] = timed(synth, reps, before=analyze)
    eng.profile(True)
    for _ in range(reps):
        analyze()
        synth()
    prof = eng.profile_read()
    eng.profile(False)
    ms, n = prof["synthesis_kernel"]
    row["synthesis_kernel_ms"] = round(ms / n, 4)
    hops = B * T
    row["export_bytes"] = hops * (1600 * 4 + 34 * 4 + 1 + OPS * 4)
    row["backward_bytes"] = hops * (OPS * 4 + (FRAME + 2 * 68) * 4)
    row["backward_GBps"] = round(row["backward_bytes"] / row["backward_ms"] / 1e6, 1)
    row["backward_over_synthesis_kernel"] = round(row["backward_ms"] / row["synthesis_kernel_ms"], 2)
    eng.close()
    del x, base, ops, out, dout, dgr, feat, gr
    from percepnet_b200.torch_module import PercepNet
    if B * T <= 128 * 2000:
        torch.manual_seed(701)
        net = PercepNet().cuda()
        xf = torch.rand((B, T, 70), device="cuda")
        d = torch.randn((B, T, 68), device="cuda")

        def step():
            net.zero_grad(set_to_none=True)
            net(xf).backward(d)

        step()
        torch.cuda.synchronize()
        row["percepnet_fwd_bwd_ms"], row["percepnet_spread"] = timed(step, max(3, reps // 3))
        net.close()
        del net, xf, d
    torch.cuda.empty_cache()
    return row


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--shapes", default="10x500,32x500,128x2000,16384x100")
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out")
    a = ap.parse_args()
    name, power = card()
    result = {"card": name, "power_limit": power, "reps": a.reps, "shapes": []}
    for shp in a.shapes.split(","):
        B, T = (int(s) for s in shp.split("x"))
        row = shape(B, T, a.reps)
        result["shapes"].append(row)
        print(json.dumps(row), flush=True)
    print(json.dumps(result))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
