#!/usr/bin/env python
"""Writes tests/golden/synthesis_digests.json from the REAL reference: for each fixed-gain model whose g and r are
exactly 0 or 1 (tests/synthesis_oracle.py, EXACT_PATTERNS), the digest of what the reference's float C API
(rnnoise_process_frame) and its CLI's int16 conversions (src/main.cpp:30-39) make of the full-scale square waves of
wrap_pcm16().  tests/test_oracle_synthesis.py compares the oracle with these where the reference is not built.  Run
where the reference library is built (oracle/_ref/libpercepnet_ref.so, oracle/Makefile):

    python tests/golden/make_synthesis_golden.py
"""
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle.ffi import Reference, build  # noqa: E402
from synthesis_oracle import EXACT_PATTERNS, pattern_model, wrap_pcm16  # noqa: E402
from util import digest  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "synthesis_digests.json")


def main():
    build()
    R = Reference()
    x16 = wrap_pcm16()
    table = {}
    for name in EXACT_PATTERNS:
        model = pattern_model(name)
        R.set_model(model)
        ys, o16s = [], []
        for s in range(x16.shape[0]):
            h = R.create()
            y, _ = R.process_stream(h, x16[s].astype(np.float32) / np.float32(32768))
            R.destroy(h)
            ys.append(y)
            o16s.append(R.run_pcm16(x16[s])[0])
        table[name] = digest(np.stack(ys), np.stack(o16s))
    with open(OUT, "w") as f:
        json.dump(table, f, indent=0, sort_keys=True)
        f.write("\n")
    print(OUT, table)


if __name__ == "__main__":
    main()
