"""Training-data generator CLI: the GPU counterpart of the reference's ``percepNet`` binary built with TRAINING=1
(/root/reference/src/denoise.cpp:600-787, ``train()``; driven by /root/reference/utils/run.sh:95-117).

  python -m percepnet_b200.gen_features <speech.pcm> <noisy.pcm> <count> <output.f32>      # the reference's argv
  python -m percepnet_b200.gen_features --list jobs.txt [--batch 4096] [--chunk 64]         # one job per line
  ... [--test-audio]                                                                       # plus train()'s TEST audio

Each job reads two raw int16 48 kHz files and writes ``count`` records of 138 float32
(Ey_lookahead[34] Ephaty[34] T pitchcorr g[34] r[34], denoise.cpp:761-773) -- the file ``rnn_train.py:44-53`` and
``utils/bin2h5.py`` consume.  Jobs of a list run as one batch of pairs per GPU call (pnb_train_records_host).
Like train(), a file shorter than ``count`` frames is re-read from its start (denoise.cpp:676-679, 687-690).
With ``--test-audio`` each job also writes ``<output>.test_input.pcm`` and ``<output>.test_output.pcm``, ``count`` x 480
int16 each: what train() writes to test_input.pcm / test_output.pcm in its working directory (denoise.cpp:722-728,
742-759), the noisy input as read and the noisy input resynthesised with its own labels, named per job so that the
jobs of a list do not overwrite each other (pnb_train_audio_host).
There is no CPU path: without the CUDA library / a GPU this exits with an error.
"""
from __future__ import annotations

import argparse
import sys

import numpy as np

FRAME = 480


def read_cyclic_frames(path: str, count: int) -> np.ndarray:
    """The sample sequence train() sees for one input file: whole 480-sample frames in file order, starting over
    at the first frame whenever a read hits the end of the file (a trailing partial frame is never used)."""
    raw = np.fromfile(path, dtype="<i2")
    nf = raw.size // FRAME
    if nf == 0:
        raise ValueError(f"{path}: shorter than one frame of {FRAME} samples")
    frames = raw[:nf * FRAME].reshape(nf, FRAME)
    if count <= nf:
        return np.ascontiguousarray(frames[:count]).reshape(-1)
    return frames[np.arange(count) % nf].reshape(-1)


def run_jobs(jobs, batch: int = 4096, chunk: int = 64, device: int = 0, test_audio: bool = False) -> None:
    """jobs: list of (speech_path, noisy_path, count, output_path); test_audio: also write each job's
    <output>.test_input.pcm and <output>.test_output.pcm."""
    from . import api
    jobs = sorted(jobs, key=lambda j: -j[2])                   # similar lengths share a batch
    for b0 in range(0, len(jobs), batch):
        group = jobs[b0:b0 + batch]
        N, Fmax = len(group), group[0][2]
        speech = np.zeros((N, Fmax * FRAME), np.int16)
        noisy = np.zeros((N, Fmax * FRAME), np.int16)
        for k, (sp, no, cnt, _) in enumerate(group):
            speech[k, :cnt * FRAME] = read_cyclic_frames(sp, cnt)
            noisy[k, :cnt * FRAME] = read_cyclic_frames(no, cnt)
        flags = api.TRAIN_DATA | (api.TRAIN_AUDIO if test_audio else 0)
        eng = api.Engine(2 * N, min(chunk, Fmax), None, flags, device=device)
        parts, audio = [], []
        for t0 in range(0, Fmax, chunk):
            t1 = min(Fmax, t0 + chunk)
            sp, no = speech[:, t0 * FRAME:t1 * FRAME], noisy[:, t0 * FRAME:t1 * FRAME]
            if test_audio:
                r, a = eng.train_audio(sp, no)
                audio.append(a)
            else:
                r = eng.train_records(sp, no)
            parts.append(r)
        eng.close()
        rec = np.concatenate(parts, axis=1)
        audio = np.concatenate(audio, axis=1) if test_audio else None
        for k, (_, _, cnt, out) in enumerate(group):
            rec[k, :cnt].astype("<f4").tofile(out)
            if test_audio:
                noisy[k, :cnt * FRAME].astype("<i2").tofile(out + ".test_input.pcm")
                audio[k, :cnt * FRAME].astype("<i2").tofile(out + ".test_output.pcm")


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("args", nargs="*", help="<speech> <noisy> <count> <output>")
    ap.add_argument("--list", help="text file, one '<speech> <noisy> <count> <output>' job per line")
    ap.add_argument("--batch", type=int, default=4096, help="pairs per GPU batch")
    ap.add_argument("--chunk", type=int, default=64, help="frames per GPU call")
    ap.add_argument("--device", type=int, default=0)
    ap.add_argument("--test-audio", action="store_true",
                    help="also write <output>.test_input.pcm and <output>.test_output.pcm, as train() writes its TEST audio")
    a = ap.parse_args(argv)
    if a.list:
        jobs = []
        for line in open(a.list):
            f = line.split()
            if f:
                jobs.append((f[0], f[1], int(f[2]), f[3]))
    elif len(a.args) == 4:
        jobs = [(a.args[0], a.args[1], int(a.args[2]), a.args[3])]
    else:
        sys.stderr.write(f"usage: {sys.argv[0]} <speech> <noisy> <count> <output>\n")   # denoise.cpp:637
        return 1
    run_jobs(jobs, a.batch, a.chunk, a.device, a.test_audio)
    return 0


if __name__ == "__main__":
    sys.exit(main())
