#!/usr/bin/env python
"""Gradient accumulation and data-parallel training steps of the GPU trainer.

    python tools/bench_train_dp.py [--windows 64] [--frames 2000] [--splits 1,2,4] [--steps 3] [--runs 3]
                                   [--worlds 1,2,4,8] [--out FILE]

One GPU: the step time (gradient calls, pnb_train_accumulate after each, pnb_train_finish, pnb_train_adam) of
windows x frames as one call and cut into 2 and 4 micro-batches (an engine of windows / k streams each), records on
the device, timed with CUDA events over `runs` runs of `steps` steps, alternating the splits; median and spread
(max / min).  Then pnb_train_accumulate and pnb_train_finish alone (CUDA events around each, 20 times, median) with
the bytes each moves: the accumulate reads the gradient (4 N) and reads and writes the accumulator (16 N); the finish
reads the accumulator and writes the gradient and the zeroed accumulator (20 N), and its non-finite check reads the
gradient again (4 N).

Exchange: the accumulator's export, all-reduce (SUM) and import between two ranks, as percepnet_b200.train runs it:
over gloo on host copies with both ranks on device 0, and over NCCL on device buffers when two devices are visible
(else not measured).  Median of 10 after 2 warm-ups.

Several GPUs: steps per second of W ranks (NCCL, one device each, windows x frames per rank, one micro-batch) for
each W in --worlds with W devices visible; the others are reported as not measured, never estimated.  The card name
and power limit are read in the same run.  Prints one JSON object.  Needs a GPU; there is no CPU path.
"""
import argparse
import json
import os
import socket
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from percepnet_b200 import api  # noqa: E402
from percepnet_b200.weights import N_PARAMS, pack_state_dict, synth_state_dict  # noqa: E402


def card():
    import torch
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30)
        power = q.stdout.strip() or "unknown"
    except (OSError, subprocess.SubprocessError):
        power = "unknown"
    return torch.cuda.get_device_name(0), power


def records(B, T, device, seed=7):
    import torch
    g = torch.Generator(device=f"cuda:{device}").manual_seed(seed)
    r = torch.rand((B, T, 138), generator=g, device=f"cuda:{device}")
    r[..., :68] *= 0.05
    return r.contiguous()


class Stepper:
    """One training step of `rec` ([B, T, 138] on the device) as k micro-batches of B / k windows."""

    def __init__(self, sd, rec, k, device=0):
        import torch
        self.B, self.T = rec.shape[0], rec.shape[1]
        self.k, self.n = k, self.B // k
        self.eng = api.Engine(self.n, self.T, pack_state_dict(sd), api.TRAIN_NETWORK, device=device)
        self.rec = rec
        self.sums = torch.empty((self.n, 4), dtype=torch.float64, device=rec.device)
        self.step = 0

    def grads(self, stream):
        row = self.T * 138
        for j in range(self.k):
            ptr = self.rec.data_ptr() + j * self.n * row * 4
            self.eng.train_grad_device(ptr, row, self.T, None, self.sums.data_ptr(), stream)
            self.eng.train_accumulate(stream)

    def finish(self, stream):
        self.eng.train_finish(stream)
        self.step += 1
        self.eng.train_adam(1e-4, self.step, stream)

    def close(self):
        self.eng.close()


def one_gpu(sd, B, T, splits, steps, runs):
    import torch
    rec = records(B, T, 0)
    st = {k: Stepper(sd, rec, k) for k in splits}
    s = torch.cuda.Stream()
    for x in st.values():   # warm-up
        x.grads(s.cuda_stream)
        x.finish(s.cuda_stream)
    s.synchronize()
    times = {k: [] for k in splits}
    for _ in range(runs):
        for k, x in st.items():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(s)
            for _ in range(steps):
                x.grads(s.cuda_stream)
                x.finish(s.cuda_stream)
            b.record(s)
            b.synchronize()
            times[k].append(a.elapsed_time(b) / steps)
    for x in st.values():
        x.close()
    del rec
    torch.cuda.empty_cache()
    out = {}
    for k, t in times.items():
        med = float(np.median(t))
        out[f"{k}x{B // k}"] = {"step_ms": med, "spread": max(t) / min(t), "frames_per_s": B * T / med * 1e3,
                                "vs_one_call": med / float(np.median(times[splits[0]]))}
    return out


def kernels_alone(sd):
    import torch
    rec = records(2, 10, 0)
    x = Stepper(sd, rec, 1)
    s = torch.cuda.Stream()
    ta, tf = [], []
    for it in range(22):
        x.eng.train_grad_device(rec.data_ptr(), 10 * 138, 10, None, x.sums.data_ptr(), s.cuda_stream)
        e = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        e[0].record(s)
        x.eng.train_accumulate(s.cuda_stream)
        e[1].record(s)
        x.eng.train_finish(s.cuda_stream)
        e[2].record(s)
        e[2].synchronize()
        if it >= 2:
            ta.append(e[0].elapsed_time(e[1]))
            tf.append(e[1].elapsed_time(e[2]))
    x.close()
    a_ms, f_ms = float(np.median(ta)), float(np.median(tf))
    a_bytes, f_bytes = 20 * N_PARAMS, 24 * N_PARAMS
    return {"accumulate": {"ms": a_ms, "bytes": a_bytes, "GB_per_s": a_bytes / a_ms / 1e6},
            "finish_and_check": {"ms": f_ms, "bytes": f_bytes, "GB_per_s": f_bytes / f_ms / 1e6}}


def _port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _rank(rank, world, port, mode, shared, B, T, steps, out_dir):
    """One rank of a spawned group: mode "exchange" times the accumulator's exchange, "step" W-rank training steps."""
    os.environ.update(WORLD_SIZE=str(world), RANK=str(rank), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1",
                      MASTER_PORT=str(port))
    if shared:
        os.environ["CUDA_VISIBLE_DEVICES"] = "0"
    import torch
    from percepnet_b200.train import Ranks
    ranks = Ranks(0)
    dev = ranks.device
    sd = synth_state_dict(0)
    x = Stepper(sd, records(B, T, dev, seed=7 + rank), 1, device=dev)
    s = torch.cuda.Stream(device=dev)
    times = []
    if mode == "exchange":
        x.grads(s.cuda_stream)
        s.synchronize()
        for it in range(12):
            torch.distributed.barrier()
            t0 = time.perf_counter()
            ranks.sum_accumulators(x.eng)
            x.eng.wait()
            if it >= 2:
                times.append((time.perf_counter() - t0) * 1e3)
    else:
        for it in range(2 + steps):
            torch.distributed.barrier()
            t0 = time.perf_counter()
            x.grads(s.cuda_stream)
            s.synchronize()
            ranks.sum_accumulators(x.eng)
            x.finish(s.cuda_stream)
            s.synchronize()
            if it >= 2:
                times.append((time.perf_counter() - t0) * 1e3)
    x.close()
    if rank == 0:
        with open(os.path.join(out_dir, "r.json"), "w") as f:
            json.dump({"backend": ranks.backend, "ms": times}, f)
    ranks.close()


def spawned(world, mode, shared, B, T, steps):
    import torch.multiprocessing as mp
    with tempfile.TemporaryDirectory() as d:
        mp.spawn(_rank, args=(world, _port(), mode, shared, B, T, steps, d), nprocs=world, join=True)
        with open(os.path.join(d, "r.json")) as f:
            return json.load(f)


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--windows", type=int, default=64)
    ap.add_argument("--frames", type=int, default=2000)
    ap.add_argument("--splits", default="1,2,4")
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--worlds", default="1,2,4,8")
    ap.add_argument("--out")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("needs a CUDA device")
    name, power = card()
    n_dev = torch.cuda.device_count()
    sd = synth_state_dict(0)
    B, T = a.windows, a.frames
    splits = [int(k) for k in a.splits.split(",")]
    res = {"card": name, "power_limit": power, "devices": n_dev, "shape": f"{B}x{T}"}
    res["one_gpu"] = one_gpu(sd, B, T, splits, a.steps, a.runs)
    res["kernels"] = kernels_alone(sd)
    ex = {}
    g = spawned(2, "exchange", True, 2, 10, 0)
    ex["gloo_2_ranks_one_device"] = {"backend": g["backend"], "ms": float(np.median(g["ms"]))}
    if n_dev >= 2:
        nc = spawned(2, "exchange", False, 2, 10, 0)
        ex["nccl_2_ranks_two_devices"] = {"backend": nc["backend"], "ms": float(np.median(nc["ms"]))}
    else:
        ex["nccl_2_ranks_two_devices"] = f"not measured: {n_dev} device visible"
    res["exchange"] = ex
    scaling = {}
    for W in (int(w) for w in a.worlds.split(",")):
        if W == 1:
            one = res["one_gpu"][f"1x{B}"]["step_ms"]
            scaling["1"] = {"steps_per_s": 1e3 / one, "source": "one_gpu 1 x windows"}
        elif W <= n_dev:
            r = spawned(W, "step", False, B, T, a.steps)
            med = float(np.median(r["ms"]))
            scaling[str(W)] = {"backend": r["backend"], "step_ms": med, "steps_per_s": 1e3 / med,
                               "frames_per_s": W * B * T / med * 1e3}
        else:
            scaling[str(W)] = f"not measured: {n_dev} device(s) visible"
    res["ranks"] = scaling
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
