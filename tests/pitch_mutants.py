"""Comparison mutants of the pitch stage, and the pitch stage of any build of the oracle.

The GPU's pitch_stage (percepnet_b200/csrc/pnb_dsp.cu) restates pitch_search and remove_doubling (pitch.cpp:283-386,
423-527) lane-parallel and must reproduce their decisions bit for bit, as oracle/pn_oracle.c does sequentially.  Each
mutant below is one textual change to pn_oracle.c that flips a strict/non-strict comparison or drops a clamp; the
comment names the line of pitch_stage that makes the same decision.  An input on which a mutant's pitch outputs
differ from the original's is an input on which the corresponding mistake in the kernel would be seen.  The edge
corpus (tests/golden/make_pitch_edges.py, pitch_edges.npz) is built so that it tells every one of them apart.
"""
import os
import re
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")

# name -> (text in pn_oracle.c, replacement, the decision it changes; pnb_dsp.cu's equivalent)
MUTANTS = {
    "A_xcorr_ge0": ("if (xcorr[i] > 0) {", "if (xcorr[i] >= 0) {",
                    "zero correlations become candidates; best2_rounds(S, valid && xv > 0.f, ...)"),
    "C_second_tie": ("if (num * den1 > num1 * syy) {", "if (num * den1 >= num1 * syy) {",
                     "ties of num*den against the second best; best2_rounds' pass test"),
    "E_fine_clamp": ("xc[i] = -1 > s ? -1 : s;", "xc[i] = s;",
                     "the -1 floor of the fine xcorr read by the interpolation and returned as corr; "
                     "W.xc[fl] = (-1.f > sacc) ? -1.f : sacc"),
    "G_search_off_tie": ("if ((c - a) > .7f * (b - a)) off = 1;", "if ((c - a) >= .7f * (b - a)) off = 1;",
                         "ties of the sub-lag offset of pitch_search; (cc - a) > .7f * (b - a)"),
    "G_doubling_off_tie": ("if ((xc[2] - xc[0]) > .7f * (xc[1] - xc[0])) off = 1;",
                           "if ((xc[2] - xc[0]) >= .7f * (xc[1] - xc[0])) off = 1;",
                           "ties of the sub-lag offset of remove_doubling; (x2 - x0) > .7f * (x1 - x0)"),
    "O_T1_le90": ("if (T1 < 3 * minp) thresh", "if (T1 <= 3 * minp) thresh",
                  "the 0.4 / 0.85 threshold at T1 = 90; if (T1 < 90)"),
    "Q_k2_ge": ("if (k == 2) T1b = (T1 + T0 > maxp) ? T0 : T0 + T1;",
                "if (k == 2) T1b = (T1 + T0 >= maxp) ? T0 : T0 + T1;",
                "the second lag of k = 2 at T0 = 256; (T1 + T0 > 384) (both places)"),
    "U_syy_floor": ("syy = 1 > syy ? 1 : syy;", "",
                    "the floor of 1 under the running energy; max_nan(syy + d, 1.f) in energy_chain"),
}


def oracle_cflags():
    """The compiler and flags oracle/Makefile builds libpn_oracle.so with."""
    mk = open(os.path.join(ORACLE_DIR, "Makefile")).read()
    m = re.search(r"^libpn_oracle\.so:.*\n\t\$\(CC\) (.*) -o \$@ pn_oracle\.c (.*)$", mk, re.M)
    assert m, "oracle/Makefile: libpn_oracle.so recipe not found"
    return m.group(1).split(), m.group(2).split()


def mutant_source(name):
    src = open(os.path.join(ORACLE_DIR, "pn_oracle.c")).read()
    old, new, _ = MUTANTS[name]
    assert src.count(old) == 1, f"{name}: the mutated text must occur exactly once in pn_oracle.c"
    return src.replace(old, new)


def build_mutant(name, out_dir):
    """Compile pn_oracle.c with mutant `name` applied (None: unchanged) into out_dir; returns the library's path."""
    src = open(os.path.join(ORACLE_DIR, "pn_oracle.c")).read() if name is None else mutant_source(name)
    tag = name or "original"
    c = os.path.join(out_dir, f"pn_oracle_{tag}.c")
    so = os.path.join(out_dir, f"libpn_oracle_{tag}.so")
    with open(c, "w") as f:
        f.write(src)
    flags, libs = oracle_cflags()
    # -I oracle/: pn_oracle.h and, relative to it, ../include/
    subprocess.run(["gcc"] + flags + ["-w", "-I", ORACLE_DIR, "-o", so, c] + libs, check=True)
    return so


def build_all(out_dir):
    """{None: original, name: mutant} -> library path, compiled in parallel."""
    from concurrent.futures import ThreadPoolExecutor
    names = [None] + list(MUTANTS)
    with ThreadPoolExecutor(max_workers=min(8, os.cpu_count() or 1)) as ex:
        paths = list(ex.map(lambda n: build_mutant(n, out_dir), names))
    return dict(zip(names, paths))


def pitch_outputs(lib, bufs, prev_period, prev_gain):
    """pitch_downsample -> pitch_search -> remove_doubling (denoise.cpp:404-414) of every row with `lib` (an
    oracle.ffi.Oracle or Reference): (lag int32, corr float32, T int32, gain float32), each [n]."""
    n = bufs.shape[0]
    lag, T = np.empty(n, np.int32), np.empty(n, np.int32)
    corr, gain = np.empty(n, np.float32), np.empty(n, np.float32)
    for k in range(n):
        lp = lib.pitch_downsample(bufs[k])
        r = lib.pitch_search(lp)
        lag[k], corr[k] = r[0], r[1]
        T[k], gain[k] = lib.remove_doubling(lp, 768 - int(lag[k]), int(prev_period[k]), float(prev_gain[k]))
    return lag, corr, T, gain


def differs(a, b):
    """[n] bool: rows whose (lag, corr, T, gain) differ; floats compare by bits, -0 == +0."""
    from util import bits
    out = np.zeros(a[0].shape[0], bool)
    for x, y in zip(a, b):
        if x.dtype.kind == "f":
            out |= (bits(x) != bits(y)) & ~((x == 0) & (y == 0))
        else:
            out |= x != y
    return out
