#!/usr/bin/env python
"""Writes tests/golden/train_audio.npz from the REAL reference: the test_input.pcm / test_output.pcm its own train()
(src/denoise.cpp:722-728, 742-759) writes for the pairs of tests/golden/train.npz, which it reads as committed and
leaves untouched.  Run where the reference library is built (oracle/_ref/libpercepnet_ref.so, oracle/Makefile):

    python tests/golden/make_train_audio_golden.py
"""
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle.ffi import Reference, build  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))


def main():
    build()
    R = Reference()
    g = np.load(os.path.join(OUT, "train.npz"))
    tin, tout = [], []
    with tempfile.TemporaryDirectory() as d:
        for k in range(g["speech"].shape[0]):
            n = g["speech"].shape[1] // 480
            fc, fn, fo = (os.path.join(d, f"{nm}{k}") for nm in ("c", "n", "o"))
            g["speech"][k].tofile(fc)
            g["noisy"][k].tofile(fn)
            assert R.train_files(fc, fn, n, fo) == 0           # train() writes its TEST audio beside the output file
            rec = np.fromfile(fo, np.float32).reshape(n, 138)
            assert np.array_equal(rec.view(np.int32), g["records"][k].view(np.int32))
            tin.append(np.fromfile(os.path.join(d, "test_input.pcm"), np.int16))
            tout.append(np.fromfile(os.path.join(d, "test_output.pcm"), np.int16))
    np.savez_compressed(os.path.join(OUT, "train_audio.npz"), test_input=np.stack(tin), test_output=np.stack(tout))
    print("train_audio.npz", os.path.getsize(os.path.join(OUT, "train_audio.npz")))


if __name__ == "__main__":
    main()
