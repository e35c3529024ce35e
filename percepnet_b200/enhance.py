"""Batch enhancement CLI: the GPU counterpart of the reference's ``percepNet_run`` binary
(/root/reference/src/main.cpp), for one file with the reference's argv or for a list of files as one batch.

  python -m percepnet_b200.enhance --weights model.pnbw <in.pcm> <out.pcm>
  python -m percepnet_b200.enhance --weights model.pnbw --list jobs.txt [--batch 4096] [--chunk 100] [--nn tensor]
  python -m percepnet_b200.enhance --gains gains.f32 <in.pcm> <out.pcm>

File format and framing are main.cpp's (:30-39): raw int16 mono 48 kHz in; frames of 480 samples are read until
the first short read (a trailing partial frame is dropped); every processed frame except the first is written, so
the output holds (n_frames - 1) * 480 samples, converted with C truncation of x * 32768.  ``--gr <file>`` also
stores the per-frame g[34], r[34] the reference dumps to feature_test.raw (denoise.cpp:533-534).

Weights come from a binary weight file (percepnet_b200.weights.PackedModel.save_blob; INTEGRATION.md 3) -- the
reference binary has them compiled in.  ``--seed N`` uses the synthetic random-init model instead (tests, benches).
All files of a list run as independent streams of one engine.  Within a batch the files are sorted longest first, and
each call advances only the files that still have frames (the engine's active range), so the padding behind a file
that has ended is not processed.

``--gains <file>`` resynthesises <in.pcm> with the caller's per-frame g, r instead of running the network, on a
signal-only engine (no --weights needed): the file is what ``--gr`` writes and the reference writes to
feature_test.raw, [n_frames][68] float32 (34 g then 34 r), one row per processed frame, the first included.  In list
mode a job line may carry a third path, its gains file; jobs without one run the network.  A gains file that does not
hold exactly n_frames x 68 floats is an error, reported before any engine is created.
There is no CPU path: without the CUDA library / a GPU this exits with an error.
"""
from __future__ import annotations

import argparse
import sys

import numpy as np

FRAME = 480


def run_jobs(jobs, model, nn: str = "tensor", batch: int = 4096, chunk: int = 100, device: int = 0, gr_paths=None,
             gains=None) -> None:
    """jobs: list of (in_path, out_path); gr_paths: optional list of paths (or None) for the g/r dump of each job.
    gains: None, or one [n_frames, 68] float32 array per job (read_gains): each input is resynthesised with its own g/r
    on a signal-only engine (analyze, then synthesize) instead of running the network; model is then unused."""
    from . import api
    flags = api.SIGNAL_ONLY if gains is not None else api.NN_TENSOR if nn == "tensor" else api.NN_FP32
    order = sorted(range(len(jobs)), key=lambda k: -_n_frames(jobs[k][0]))       # similar lengths share a batch
    for b0 in range(0, len(order), batch):
        group = order[b0:b0 + batch]
        nfr = [_n_frames(jobs[k][0]) for k in group]
        S, Fmax = len(group), max(nfr)
        if Fmax == 0:
            for k in group:
                open(jobs[k][1], "wb").close()
            continue
        x = np.zeros((S, Fmax * FRAME), np.int16)
        for row, k in enumerate(group):
            x[row, :nfr[row] * FRAME] = np.fromfile(jobs[k][0], dtype="<i2", count=nfr[row] * FRAME)
        eng = api.Engine(S, min(chunk, Fmax), None if gains is not None else model, flags, device=device)
        want_gr = gr_paths is not None and any(gr_paths[k] for k in group)
        out = np.zeros_like(x)
        gr = np.zeros((Fmax, S, 68), np.float32) if want_gr else None              # [F, S, 68]
        for t0 in range(0, Fmax, chunk):
            t1 = min(Fmax, t0 + chunk)
            n = sum(1 for f in nfr if f > t0)   # rows [0, n): the files (longest first) that still have frames
            if n != eng.active:
                eng.set_active(n)               # only shrinks: the files that left have ended
            xin = np.ascontiguousarray(x[:n, t0 * FRAME:t1 * FRAME])
            if gains is not None:
                gin = np.zeros((n, t1 - t0, 68), np.float32)   # zero behind a file's end: that output is not written
                for row in range(n):
                    g = gains[group[row]][t0:t1]
                    gin[row, :len(g)] = g
                eng.analyze(xin)
                out[:n, t0 * FRAME:t1 * FRAME] = eng.synthesize(gin, int16=True)
                continue
            o, g = eng.process(xin, want_gr=want_gr)
            out[:n, t0 * FRAME:t1 * FRAME] = o
            if want_gr:
                gr[t0:t1, :n] = g
        eng.close()
        for row, k in enumerate(group):
            n = nfr[row]
            out[row, FRAME:n * FRAME].astype("<i2").tofile(jobs[k][1])            # first frame dropped, main.cpp:37-38
            if want_gr and gr_paths[k]:
                gr[:n, row].astype("<f4").tofile(gr_paths[k])


def _n_frames(path: str) -> int:
    import os
    return os.path.getsize(path) // (2 * FRAME)


def read_gains(gains_path: str, pcm_path: str) -> np.ndarray:
    """The g/r of a gains file for the frames of pcm_path: [n_frames, 68] float32.  Raises ValueError unless the file
    holds exactly n_frames x 68 floats."""
    import os
    n, size = _n_frames(pcm_path), os.path.getsize(gains_path)
    if size != n * 68 * 4:
        raise ValueError(f"{gains_path}: {size} bytes, but {pcm_path} has {n} frames: a gains file holds n_frames x 68 "
                         f"float32 = {n * 68 * 4} bytes")
    return np.fromfile(gains_path, dtype="<f4").reshape(n, 68)


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("args", nargs="*", help="<in.pcm> <out.pcm>")
    ap.add_argument("--list", help="text file, one '<in.pcm> <out.pcm> [<gains.f32>]' job per line")
    ap.add_argument("--weights", help="binary weight file (PackedModel.save_blob)")
    ap.add_argument("--seed", type=int, help="use the synthetic random-init model with this seed instead of --weights")
    ap.add_argument("--nn", default="tensor", choices=["tensor", "fp32"])
    ap.add_argument("--gr", help="single-file mode: also write the per-frame g, r (feature_test.raw of the reference)")
    ap.add_argument("--gains", help="single-file mode: resynthesise with these per-frame g, r ([n_frames][68] float32) "
                                    "instead of running the network")
    ap.add_argument("--batch", type=int, default=4096, help="files per GPU batch")
    ap.add_argument("--chunk", type=int, default=100, help="frames per GPU call")
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args(argv)
    if a.gains and (a.list or a.gr):
        sys.stderr.write("--gains is for single-file mode and replaces the network: not with --list or --gr\n")
        return 1
    if a.list:
        lines = [line.split() for line in open(a.list) if line.split()]
        jobs = [tuple(p[:2]) for p in lines]
        gain_paths = [p[2] if len(p) > 2 else None for p in lines]
        grp = None
    elif len(a.args) == 2:
        jobs = [(a.args[0], a.args[1])]
        gain_paths = [a.gains]
        grp = [a.gr]
    else:
        sys.stderr.write("usage: percepnet_b200.enhance <in.pcm> <out.pcm>   (or --list jobs.txt)\n")
        return 1
    try:
        gains = {k: read_gains(gp, jobs[k][0]) for k, gp in enumerate(gain_paths) if gp}
    except ValueError as ex:
        sys.stderr.write(f"{ex}\n")
        return 2
    net = [k for k in range(len(jobs)) if k not in gains]
    if net:
        from . import api
        from .weights import synth_model
        if a.weights:
            model = api.BlobModel(a.weights)
        elif a.seed is not None:
            model = synth_model(a.seed)
        else:
            sys.stderr.write("give --weights <file.pnbw> (or --seed N for the synthetic model)\n")
            return 1
        run_jobs([jobs[k] for k in net], model, a.nn, a.batch, a.chunk, a.device, grp and [grp[k] for k in net])
    if gains:
        ks = sorted(gains)
        run_jobs([jobs[k] for k in ks], None, batch=a.batch, chunk=a.chunk, device=a.device, gains=[gains[k] for k in ks])
    return 0


if __name__ == "__main__":
    sys.exit(main())
