#!/usr/bin/env python
"""Writes tests/golden/pitch_edges.npz: 1728-sample pitch buffers, each with a (prev_period, prev_gain), that put the
comparisons and clamps of the pitch stage on the path of an output, and the reference's lag / corr / T / gain for each.

The buffers come from a seeded, deterministic search over families of inputs built for one boundary each:

  quiet     harmonic mixtures and noise at 1e-26 .. 1e-2, some with a silent gap: num = (xcorr * 1e-12)^2
            underflows to 0 so candidates tie, zero correlations sit next to positive ones, and correlations that
            are a few subnormal steps wide tie in the sub-lag offsets
  t1_90     periods around 2 * T0 with T0 = 180, 270, 360 and a mixture of the fundamental and its k-th harmonic:
            T1 = 90 with g1 near the 0.4 / 0.85 threshold
  t0_256    period 512 (T0 = 256) with a strong second harmonic, with and without a previous period near 256: the
            k = 2 candidate, whose second lag T0 + T1 = 384 sits on the maxperiod comparison
  burst     an int16-scale burst, silence, then (mostly) a quiet periodic tail: the running energy of
            find_best_pitch drifts below 1 and the floor decides, and the fine xcorr next to the peak falls below -1
            where the -1 floor moves the sub-lag offset

A candidate is kept only if it tells some mutant of tests/pitch_mutants.py from the original oracle (every mutant is
one comparison or clamp of pn_oracle.c, and the GPU kernels must reproduce pn_oracle.c's decisions bit for bit).
Up to KEEP rows are kept per mutant, chosen greedily so that rows killing several mutants come first.  The script
refuses to write a corpus that leaves a mutant alive.  The stored outputs are the reference's own
(oracle/_ref/libpercepnet_ref.so), and where the reference is built the oracle must agree with them row by row.

    python tests/golden/make_pitch_edges.py
"""
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import pitch_mutants as pm  # noqa: E402
from oracle.ffi import Oracle, Reference, build  # noqa: E402

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "pitch_edges.npz")
N = 1728
KEEP = 3            # rows kept per mutant
BATCH = 256         # candidates per family per round
MAX_ROUNDS = 60


def _harmonics(rng, period, amps, t):
    x = np.zeros_like(t)
    for h, a in enumerate(amps, 1):
        x += a * np.sin(2 * np.pi * h * t / period + rng.rand() * 6.283)
    return x


def fam_quiet(rng):
    t = np.arange(N, dtype=np.float64)
    period = 182 + 586 * rng.rand()
    x = _harmonics(rng, period, rng.rand(8) / np.arange(1, 9), t)
    noise = rng.rand()
    x = x / (np.abs(x).max() + 1e-30) * (1 - noise) + noise * 0.3 * rng.randn(N)
    if rng.rand() < 0.3:
        g0 = rng.randint(0, N - 480)
        x[g0:g0 + rng.randint(100, 480)] = 0
    x *= 10.0 ** rng.uniform(-26, -2)
    return x, _prev(rng)


def fam_t1_90(rng):
    k = rng.randint(2, 5)
    T0 = {2: (179, 180), 3: (269, 271), 4: (358, 361)}[k]
    period = 2 * rng.uniform(T0[0] - 0.5, T0[1] + 0.5)
    t = np.arange(N, dtype=np.float64)
    amps = 0.2 * rng.rand(8)
    amps[0] = rng.rand()
    amps[k - 1] = 1.0
    x = _harmonics(rng, period, amps, t) + 0.05 * rng.rand() * rng.randn(N)
    x *= 10.0 ** rng.uniform(-2, 4.3) / (np.abs(x).max() + 1e-30)
    if rng.rand() < 0.5:
        return x, (int(rng.randint(176, 186)), float(rng.rand()))
    return x, _prev(rng)


def fam_t0_256(rng):
    period = rng.uniform(511.0, 514.0)
    t = np.arange(N, dtype=np.float64)
    amps = 0.3 * rng.rand(8)
    amps[0] = rng.rand()
    amps[1] = rng.uniform(0.3, 1.0)
    x = _harmonics(rng, period, amps, t) + 0.1 * rng.rand() * rng.randn(N)
    x *= 10.0 ** rng.uniform(-2, 4.3) / (np.abs(x).max() + 1e-30)
    if rng.rand() < 0.6:
        return x, (int(rng.randint(250, 263)), float(rng.rand()))
    return x, _prev(rng)


def fam_burst(rng):
    x = np.zeros(N)
    L = rng.randint(40, 560)
    x[:L] = np.clip(rng.randn(L) * rng.uniform(1e2, 3e4), -32767, 32767)     # within int16 range
    if rng.rand() < 0.8:
        s = rng.randint(L + 1, 1400)
        t = np.arange(N - s, dtype=np.float64)
        x[s:] = _harmonics(rng, 182 + 586 * rng.rand(), rng.rand(4), t) * 10.0 ** rng.uniform(-4, 1)
    return x, _prev(rng)


def _prev(rng):
    if rng.rand() < 0.4:
        return 0, 0.0
    return int(rng.randint(60, 769)), float(rng.rand())


FAMILIES = {"quiet": fam_quiet, "t1_90": fam_t1_90, "t0_256": fam_t0_256, "burst": fam_burst}


def search(libs, seed=2026):
    """Seeded search until every mutant is killed by KEEP rows: [(buf, prev_period, prev_gain, killed set, family)]."""
    names = list(pm.MUTANTS)
    kills = {n: [] for n in names}
    rows = []
    for r in range(MAX_ROUNDS):
        for fi, (fam, gen) in enumerate(FAMILIES.items()):
            rng = np.random.RandomState(seed + 1000 * r + fi)
            cand = [gen(rng) for _ in range(BATCH)]
            bufs = np.stack([c[0] for c in cand]).astype(np.float32)
            pp = np.array([c[1][0] for c in cand], np.int32)
            pg = np.array([c[1][1] for c in cand], np.float32)
            base = pm.pitch_outputs(libs[None], bufs, pp, pg)
            killed = np.zeros((BATCH, len(names)), bool)
            for j, n in enumerate(names):
                killed[:, j] = pm.differs(base, pm.pitch_outputs(libs[n], bufs, pp, pg))
            for i in np.nonzero(killed.any(1))[0]:
                ks = {names[j] for j in np.nonzero(killed[i])[0]}
                rows.append((bufs[i], int(pp[i]), float(pg[i]), ks, fam))
                for n in ks:
                    kills[n].append(len(rows) - 1)
        count = {n: len(v) for n, v in kills.items()}
        print(f"round {r}: rows killing each mutant {count}", flush=True)
        if min(count.values()) >= KEEP:
            break
    return rows


def select(rows):
    """Greedy: repeatedly take the row that kills the most mutants still short of KEEP rows."""
    need = {n: KEEP for n in pm.MUTANTS}
    chosen = []
    while any(v > 0 for v in need.values()):
        best, gain = None, 0
        for i, r in enumerate(rows):
            if i in chosen:
                continue
            g = sum(1 for n in r[3] if need[n] > 0)
            if g > gain:
                best, gain = i, g
        if best is None:
            break
        chosen.append(best)
        for n in rows[best][3]:
            need[n] -= 1
    return [rows[i] for i in chosen]


def main():
    build()
    if not Reference.available():
        sys.exit("the reference library (oracle/_ref/libpercepnet_ref.so) is not built: the corpus stores its outputs")
    with tempfile.TemporaryDirectory() as d:
        libs = {k: Oracle(v) for k, v in pm.build_all(d).items()}
        rows = select(search(libs))
        alive = [n for n in pm.MUTANTS if not any(n in r[3] for r in rows)]
        if alive:
            sys.exit(f"refusing to write {OUT}: no row kills {alive}")
        bufs = np.stack([r[0] for r in rows]).astype(np.float32)
        pp = np.array([r[1] for r in rows], np.int32)
        pg = np.array([r[2] for r in rows], np.float32)
        ref = pm.pitch_outputs(Reference(), bufs, pp, pg)
        assert not pm.differs(ref, pm.pitch_outputs(libs[None], bufs, pp, pg)).any(), "the oracle disagrees with the reference"
        # re-check kills from the stored arrays, so the file is exactly what the test will see
        for n in pm.MUTANTS:
            assert pm.differs(ref, pm.pitch_outputs(libs[n], bufs, pp, pg)).any(), n
    np.savez_compressed(OUT, buf=bufs, prev_period=pp, prev_gain=pg, lag=ref[0], corr=ref[1], T=ref[2], gain=ref[3],
                        family=np.array([r[4] for r in rows]))
    for i, r in enumerate(rows):
        print(f"row {i:2d} {r[4]:8s} kills {' '.join(sorted(r[3]))}")
    for n in pm.MUTANTS:
        print(f"{n:20s} killed by {sum(n in r[3] for r in rows)} of {len(rows)} rows")
    print(f"wrote {OUT}: {len(rows)} rows")


if __name__ == "__main__":
    main()
