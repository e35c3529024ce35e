#!/usr/bin/env python
"""Throughput of the network-only call (pnb_compute_rnn_device) on device-resident features, next to the network's
share of a full PCM call of the same shape, on the tensor engine and on the fp32 engine; then the scoring leg.

    python tools/bench_compute_rnn.py [--streams 16384] [--frames 100] [--calls 5] [--warmup 2] [--runs 3] [--out FILE]

The features are what the DSP makes: one PCM call of synthetic speech-plus-noise on the engine, read back through
PNB_TAP_FEATURES and kept on the device as [streams, frames, 70].  Each engine then gets `warmup` feature calls, and
`runs` timed runs of `calls` feature calls each, alternating between the engines; a run is timed with CUDA events on
the launching stream and the median run is reported.  A separate profiled feature call and a profiled PCM call give
the per-kernel-class split (pnb_profile_read).  Prints one JSON object per engine (and writes them to --out).  The card
name and power limit are read in the same run.  Needs a GPU; there is no CPU path.

The scoring leg runs PNB_NETWORK_ONLY engines on records made from the same features (labels drawn uniformly in
[0, 1]).  Device form: pnb_score_records_device without g/r against pnb_compute_rnn_device on the same records, ms
per call, timed like the feature calls.  Host form: what eval_records did before it scored on the device
(pnb_compute_rnn_host, then eval_records.loss_sums of every row in numpy) against pnb_score_records_host, records per
second end to end (host clock around blocking calls), `runs` alternating runs of one call each.  It also reports
pnb_engine_bytes of a PCM engine and of a network-only engine of the shape, per network path.  Every host-form call
starts from a reset engine, so both forms score the same predictions and "max_rel_sums_vs_numpy" compares their sums.
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

NETWORK_CLASSES = {"tensor": ("tc_gemm_kernel", "tc_aux_kernel"),
                   "fp32": ("fc_f32_kernel", "gemm_f32_kernel", "f32_carry_kernel")}


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


def pcm_rows(S, F, seed=20261016):
    """[S, F*480] float32 on the device: 64 synthetic streams, each row one of them at its own level."""
    import torch
    base = torch.from_numpy(synth_pcm(64, F, seed=seed)).cuda()
    g = torch.Generator().manual_seed(seed)
    level = (0.25 + torch.rand(S, 1, generator=g)).cuda()
    return (base[torch.arange(S, device="cuda") % 64] * level).contiguous()


def split(prof):
    return {k: round(v[0], 3) for k, v in sorted(prof.items())}


def main():
    import torch
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--streams", type=int, default=16384)
    ap.add_argument("--frames", type=int, default=100)
    ap.add_argument("--calls", type=int, default=5, help="feature calls per timed run")
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--out", help="also write the JSON lines to this file")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_compute_rnn: no CUDA device")
    S, F = a.streams, a.frames
    name, power = card()
    model = synth_model(0)
    engines, feats, gr, res = {}, None, None, {}
    x = pcm_rows(S, F)
    y = torch.empty_like(x)
    for mode, flags in (("tensor", api.NN_TENSOR), ("fp32", api.NN_FP32)):
        eng = api.Engine(S, F, model, flags)
        eng.process_device(x.data_ptr(), F * 480, y.data_ptr(), F * 480, F)       # warm-up PCM call
        eng.profile(True)
        eng.process_device(x.data_ptr(), F * 480, y.data_ptr(), F * 480, F)       # profiled PCM call
        prof = eng.profile_read()
        eng.profile(False)
        eng.check()
        if feats is None:
            feats = torch.from_numpy(np.ascontiguousarray(eng.read_tap("features", F).transpose(1, 0, 2))).cuda()
            gr = torch.empty((S, F, 68), dtype=torch.float32, device="cuda")
        res[mode] = {"pcm_engine_bytes": eng.device_bytes, "pcm_call_split_ms": split(prof),
                     "pcm_call_network_ms": round(sum(prof[k][0] for k in NETWORK_CLASSES[mode] if k in prof), 3),
                     "pcm_call_ms": round(sum(v[0] for v in prof.values()), 3)}
        engines[mode] = eng
    del x, y
    torch.cuda.empty_cache()

    def call(eng):
        eng.compute_rnn_device(api.RNN_FEATURES, feats.data_ptr(), F * 70, F, gr.data_ptr(), F * 68)

    for mode, eng in engines.items():
        for _ in range(a.warmup):
            call(eng)
        eng.check()
    times = {m: [] for m in engines}
    st = torch.cuda.current_stream()
    for _ in range(a.runs):
        for mode, eng in engines.items():
            t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t0.record(st)
            for _ in range(a.calls):
                call(eng)
            eng.flush()
            t1.record(st)
            t1.synchronize()
            times[mode].append(t0.elapsed_time(t1) / a.calls)
    lines = []
    for mode, eng in engines.items():
        eng.check()
        eng.profile(True)
        call(eng)
        prof = eng.profile_read()
        eng.profile(False)
        ms = float(np.median(times[mode]))
        r = {"tool": "bench_compute_rnn", "engine": mode, "streams": S, "frames_per_call": F, "calls_per_run": a.calls,
             "runs_ms_per_call": [round(t, 3) for t in times[mode]], "ms_per_call": round(ms, 3),
             "frames_per_s": S * F / (ms / 1e3), "feature_call_split_ms": split(prof),
             "feature_call_network_ms": round(sum(prof[k][0] for k in NETWORK_CLASSES[mode] if k in prof), 3),
             **res[mode], "gpu": name, "power_limit": power}
        lines.append(json.dumps(r))
        print(lines[-1], flush=True)
        eng.close()
    del gr
    torch.cuda.empty_cache()
    lines += score_leg(a, S, F, model, feats, name, power)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write("\n".join(lines) + "\n")


def score_leg(a, S, F, model, feats, name, power):
    """The scoring leg (see the module docstring); returns its JSON lines."""
    import time

    import torch
    from percepnet_b200.eval_records import loss_sums
    g = torch.Generator(device="cuda").manual_seed(20261017)
    rec = torch.empty((S, F, 138), dtype=torch.float32, device="cuda")
    rec[..., :68] = feats[..., :68] / 30
    rec[..., 68:70] = feats[..., 68:70]
    rec[..., 70:] = torch.rand((S, F, 68), generator=g, device="cuda")
    d_gr = torch.empty((S, F, 68), dtype=torch.float32, device="cuda")
    d_sums = torch.empty((S, 4), dtype=torch.float64, device="cuda")
    rec_h = rec.cpu().numpy()
    st = torch.cuda.current_stream()
    lines = []
    for mode, flags in (("tensor", api.NN_TENSOR), ("fp32", api.NN_FP32)):
        eng = api.Engine(S, F, model, flags | api.NETWORK_ONLY)
        legs = {"compute": lambda: eng.compute_rnn_device(api.RNN_RECORDS, rec.data_ptr(), F * 138, F, d_gr.data_ptr(),
                                                          F * 68),
                "score": lambda: eng.score_records_device(rec.data_ptr(), F * 138, F, None, d_sums.data_ptr())}
        for leg in legs.values():
            for _ in range(a.warmup):
                leg()
        eng.check()
        dev = {k: [] for k in legs}
        for _ in range(a.runs):
            for k, leg in legs.items():
                t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0.record(st)
                for _ in range(a.calls):
                    leg()
                eng.flush()
                t1.record(st)
                t1.synchronize()
                dev[k].append(t0.elapsed_time(t1) / a.calls)
        eng.check()

        def old_path():   # eval_records before device-side scoring: g/r to the host, the loss in numpy per row
            gr = eng.compute_rnn(rec_h)
            return np.stack([loss_sums(gr[i], rec_h[i]) for i in range(S)])

        host = {"compute_rnn_host+loss_sums": old_path, "score_records_host": lambda: eng.score_records(rec_h)[0]}
        hs = {k: [] for k in host}
        out = {}
        for _ in range(a.runs):
            for k, f in host.items():
                eng.reset()   # both forms score the same fresh streams
                t = time.perf_counter()
                out[k] = f()
                hs[k].append(time.perf_counter() - t)
        want, got = out["compute_rnn_host+loss_sums"], out["score_records_host"]
        rel = float(np.max(np.abs(got - want) / np.maximum(np.abs(want), 1e-300)))
        dms = {k: float(np.median(v)) for k, v in dev.items()}
        r = {"tool": "bench_compute_rnn", "leg": "score", "engine": mode, "streams": S, "frames_per_call": F,
             "device_runs_ms_per_call": {k: [round(t, 3) for t in v] for k, v in dev.items()},
             "compute_rnn_device_ms": round(dms["compute"], 3), "score_records_device_ms": round(dms["score"], 3),
             "score_over_compute": round(dms["score"] / dms["compute"], 4),
             "host_runs_s": {k: [round(t, 3) for t in v] for k, v in hs.items()},
             "host_records_per_s": {k: S * F / float(np.median(v)) for k, v in hs.items()},
             "host_speedup": round(float(np.median(hs["compute_rnn_host+loss_sums"]) / np.median(hs["score_records_host"])), 3),
             "max_rel_sums_vs_numpy": rel, "network_only_engine_bytes": eng.device_bytes,
             "gpu": name, "power_limit": power}
        eng.close()
        pcm = api.Engine(S, F, model, flags)
        r["pcm_engine_bytes"] = pcm.device_bytes
        pcm.close()
        r["bytes_saved"] = r["pcm_engine_bytes"] - r["network_only_engine_bytes"]
        lines.append(json.dumps(r))
        print(lines[-1], flush=True)
    return lines


if __name__ == "__main__":
    main()
