#!/usr/bin/env python
"""The rnnoise shim with and without pooling (PNB_SHIM_POOL): T threads x H handles, each thread feeding its handles one
10 ms frame at a time through the blocking rnnoise_process_frame, the way a server with one handle per participant
would.  One JSON line.

  python tools/bench_shim_pool.py [--threads 1,4,16,64] [--handles 2] [--frames 300] [--warmup 50] [--nn fp32|tensor]
                                  [--slots 0]

The threads are native (a small C++ driver compiled into a temporary directory and linked to librnnoise_b200.so), so
the numbers are the shim's, not Python's.  For every T the unpooled run (one engine per handle) and the pooled run
(one shared engine, --slots slots, 0 = T x H) alternate.  Reported per run:
  frames_per_s          frames completed over the wall time of the timed frames, all threads together
  p50_us / p99_us       per-frame latency of rnnoise_process_frame as its caller sees it
  device_mib            device memory taken by the handles (cudaMemGetInfo before create and after the warm-up)
  calls_per_frame       pooled only: session calls issued per frame advanced (pnb_shim_pool_stats)
  parks_per_call        pooled only: sessions parked per call
The card's name and power limit are read in the same run.
"""
from __future__ import annotations

import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
LIBDIR = os.path.join(ROOT, "percepnet_b200")

DRIVER = r"""
#include <stdio.h>
#include <string.h>
#include <atomic>
#include <chrono>
#include <thread>
#include <vector>
struct DenoiseState;
struct RNNModel;
DenoiseState *rnnoise_create(RNNModel *model);
void rnnoise_destroy(DenoiseState *st);
float rnnoise_process_frame(DenoiseState *st, float *out, const float *in, FILE *f_feature);

extern "C" {
int drv_create(void *model, int n, void **out) {
  for (int i = 0; i < n; i++) {
    out[i] = rnnoise_create((RNNModel *)model);
    if (!out[i]) return -1;
  }
  return 0;
}
void drv_destroy(void **h, int n) {
  for (int i = 0; i < n; i++) rnnoise_destroy((DenoiseState *)h[i]);
}
// T threads, thread t owns handles [t*H, (t+1)*H); handle i reads signal i % n_sig ([n_sig][n_frames*480]) from frame f0.
// lat_us: [T*H*n_frames] per-call latency.  Returns the wall seconds from the common start to the last finish.
double drv_run(void **h, int T, int H, int f0, int n_frames, const float *sig, int n_sig, int sig_frames, float *lat_us) {
  std::atomic<int> ready(0);
  std::atomic<bool> go(false);
  std::vector<std::thread> th;
  for (int t = 0; t < T; t++)
    th.emplace_back([=, &ready, &go]() {
      std::vector<float> buf(480);
      ready++;
      while (!go.load()) std::this_thread::yield();
      for (int f = 0; f < n_frames; f++)
        for (int j = 0; j < H; j++) {
          const int i = t * H + j, fr = (f0 + f) % sig_frames;
          memcpy(buf.data(), sig + ((size_t)(i % n_sig) * sig_frames + fr) * 480, 480 * sizeof(float));
          auto a = std::chrono::steady_clock::now();
          rnnoise_process_frame((DenoiseState *)h[i], buf.data(), buf.data(), NULL);
          auto b = std::chrono::steady_clock::now();
          lat_us[((size_t)t * H + j) * n_frames + f] = std::chrono::duration<float, std::micro>(b - a).count();
        }
    });
  while (ready.load() < T) std::this_thread::yield();
  auto s = std::chrono::steady_clock::now();
  go = true;
  for (auto &x : th) x.join();
  return std::chrono::duration<double>(std::chrono::steady_clock::now() - s).count();
}
}
"""


def build_driver(tmp):
    src, so = os.path.join(tmp, "drv.cpp"), os.path.join(tmp, "libdrv.so")
    with open(src, "w") as f:
        f.write(DRIVER)
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.run([cxx, "-O2", "-std=c++11", "-pthread", "-fPIC", "-shared", "-o", so, src, "-L" + LIBDIR, "-lrnnoise_b200",
                    "-Wl,-rpath," + LIBDIR], check=True)
    L = C.CDLL(so)
    L.drv_create.argtypes = [C.c_void_p, C.c_int, C.c_void_p]
    L.drv_destroy.argtypes = [C.c_void_p, C.c_int]
    L.drv_run.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_void_p]
    L.drv_run.restype = C.c_double
    return L


def sm_clocks(index=0):
    """Current and maximum SM clock in MHz (nvidia-smi query; None when unavailable)."""
    try:
        out = subprocess.run(["nvidia-smi", f"--id={index}", "--query-gpu=clocks.sm,clocks.max.sm",
                              "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=20).stdout
        f = [x.strip() for x in out.strip().splitlines()[0].split(",")]
        return {"sm_clock_mhz": float(f[0]), "max_sm_clock_mhz": float(f[1])}
    except Exception as ex:
        return {"sm_clock_mhz": None, "error": type(ex).__name__}


def pool_stats(shim):
    a = (C.c_longlong * 6)()
    shim.pnb_shim_pool_stats(a)
    return [int(v) for v in a]


def one_run(drv, shim, model_ptr, sig, T, H, frames, warmup, nn, slots):
    import torch
    os.environ["PNB_SHIM_NN"] = nn
    if slots:
        os.environ["PNB_SHIM_POOL"] = str(slots)
    else:
        os.environ.pop("PNB_SHIM_POOL", None)
    n = T * H
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info(0)[0]
    hs = (C.c_void_p * n)()
    try:
        if drv.drv_create(model_ptr, n, hs) != 0:
            raise RuntimeError("rnnoise_create returned NULL")
        n_sig, sig_frames = sig.shape[0], sig.shape[1] // 480
        lat = np.zeros(n * max(frames, warmup), np.float32)
        drv.drv_run(hs, T, H, 0, warmup, sig.ctypes.data, n_sig, sig_frames, lat.ctypes.data)
        free1 = torch.cuda.mem_get_info(0)[0]
        s0 = pool_stats(shim)
        lat = np.zeros(n * frames, np.float32)
        wall = drv.drv_run(hs, T, H, warmup, frames, sig.ctypes.data, n_sig, sig_frames, lat.ctypes.data)
        s1 = pool_stats(shim)
    finally:
        drv.drv_destroy(hs, n)
        os.environ.pop("PNB_SHIM_POOL", None)
    r = {"frames_per_s": round(n * frames / wall, 1), "p50_us": round(float(np.percentile(lat, 50)), 1),
         "p99_us": round(float(np.percentile(lat, 99)), 1), "device_mib": round((free0 - free1) / 2**20, 1)}
    if slots:
        calls, adv, parks = s1[1] - s0[1], s1[2] - s0[2], s1[4] - s0[4]
        r.update({"slots": slots, "calls_per_frame": round(calls / max(adv, 1), 4),
                  "parks_per_call": round(parks / max(calls, 1), 3), "largest_batch": s1[3]})
    return r


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--threads", default="1,4,16,64")
    p.add_argument("--handles", type=int, default=2)
    p.add_argument("--frames", type=int, default=300)
    p.add_argument("--warmup", type=int, default=50)
    p.add_argument("--nn", default="fp32", choices=("fp32", "tensor"))
    p.add_argument("--slots", type=int, default=0)
    args = p.parse_args()
    import torch
    if not torch.cuda.is_available():
        print(json.dumps({"error": "no CUDA device: the shim has no CPU path"}))
        return 2
    torch.cuda.set_device(0)
    torch.zeros(1, device="cuda")                    # the context exists before the first memory reading
    from bench_churn import card_info
    from percepnet_b200 import build
    from percepnet_b200.synth import synth_pcm
    from percepnet_b200.weights import synth_model
    build.build()
    card = card_info(0)
    model = synth_model(0)
    model_ptr = C.addressof(model.as_c_model())
    sig = np.ascontiguousarray(synth_pcm(16, 400, seed=11))
    shim = C.CDLL(os.path.join(LIBDIR, "librnnoise_b200.so"))
    shim.pnb_shim_pool_stats.argtypes = [C.c_void_p]
    res = {}
    with tempfile.TemporaryDirectory() as tmp:
        drv = build_driver(tmp)
        for T in (int(t) for t in args.threads.split(",")):
            n = T * args.handles
            res[f"T{T}"] = {
                "handles": n,
                "unpooled": one_run(drv, shim, model_ptr, sig, T, args.handles, args.frames, args.warmup, args.nn, 0),
                "pooled": one_run(drv, shim, model_ptr, sig, T, args.handles, args.frames, args.warmup, args.nn,
                                  args.slots or min(n, 4096)),
            }
    card.update(sm_clocks(0))                        # read right after the load, while the clock reflects it
    print(json.dumps({"bench": "shim_pool", "nn": args.nn, "handles_per_thread": args.handles, "frames": args.frames,
                      "card": card, "runs": res}))
    return 0


if __name__ == "__main__":
    sys.exit(main())
