"""Pins the CPU restatement of the synthesis (tests/synthesis_oracle.py) before anything is compared with it: composed
from the oracle's own per-hop taps it reproduces oracle.process_stream's output and Xout spectrum BIT FOR BIT, and with
the CLI's conversion (cli_short) the int16 output of src/main.cpp, wrapped samples included.  For the fixed-gain models
whose g and r are exactly 0 or 1 the oracle's end-to-end output is the compiled reference's: live where oracle/_ref is
built, otherwise through tests/golden/synthesis_digests.json (tests/golden/make_synthesis_golden.py).  CPU only."""
import json
import os

import numpy as np
import pytest

from conftest import GOLDEN
from synthesis_oracle import (EXACT_PATTERNS, FRAME, GAIN_PATTERNS, cli_short, gained_spectrum, pattern_gains,
                              pattern_model, post_filter, sine_libm, sine_rounded, synthesize, wrap_pcm16)
from test_gpu_parity import _inputs
from util import bits, digest, same_bits

DIGESTS = os.path.join(GOLDEN, "synthesis_digests.json")
CALLS = (8, 7, 9)          # the GPU test's call split (tests/test_gpu_synthesis.py)
PNO_POSTFILTER = 1


@pytest.fixture(scope="module")
def models(model0):
    m = {name: pattern_model(name) for name in GAIN_PATTERNS}
    m["model0"] = model0
    return m


@pytest.fixture(scope="module")
def ref_or_digests():
    """(the compiled reference or None, the stored digests)."""
    from oracle import ffi
    ffi.build()
    with open(DIGESTS) as f:
        table = json.load(f)
    return (ffi.Reference() if ffi.Reference.available() else None), table


@pytest.mark.parametrize("scale", [1.0, 32768.0], ids=["unit", "int16scale"])
@pytest.mark.parametrize("flags", [0, PNO_POSTFILTER], ids=["plain", "postfilter"])
@pytest.mark.parametrize("name", ["model0"] + list(GAIN_PATTERNS))
def test_composition_is_process_frame(oracle, models, name, flags, scale):
    """Each hop composed from the oracle's taps (X, P, silence, the gains as applied, r) with a carried overlap-add
    memory equals the oracle's own output and gained spectrum, across calls split as on the GPU."""
    x = _inputs(scale, sum(CALLS), n_synth=2)
    hw, _ = oracle.tables()
    silent = voiced = 0
    for s in range(x.shape[0]):
        h = oracle.create(models[name])
        mem = np.zeros(FRAME, np.float32)
        t0 = 0
        for n in CALLS:
            out, _, taps = oracle.process_stream(h, x[s, t0 * FRAME:(t0 + n) * FRAME], flags=flags, taps=True)
            for k, tp in enumerate(taps):
                X, P, g, r = tp.np("X")[:800], tp.np("P")[:800], tp.np("g_used"), tp.np("r")
                tag = (s, t0 + k)
                assert same_bits(gained_spectrum(oracle, X, P, tp.silence, g, r), tp.np("Xout")), tag
                assert same_bits(synthesize(oracle, X, P, tp.silence, g, r, mem, hw), out[k * FRAME:(k + 1) * FRAME]), tag
                if flags & PNO_POSTFILTER:
                    assert same_bits(post_filter(tp.np("g"), tp.np("Ex"), sine_libm), g), tag
                silent += tp.silence
                voiced += not tp.silence
            t0 += n
        oracle.destroy(h)
    assert silent > 0 and voiced > 0, (silent, voiced)      # both branches of the comb mix ran


def test_sines_one_ulp_apart():
    """The post-filter's one step the device does not reproduce: the C library's sinf against the rounded double sine,
    on the arguments (float)(M_PI/2 * g) of g in [0, 1].  They differ by one ulp at most, on a few percent of the
    arguments."""
    g = np.random.RandomState(5).rand(20000).astype(np.float32)
    x = (np.pi / 2 * g.astype(np.float64)).astype(np.float32)
    d = np.abs(bits(sine_libm(x)).astype(np.int64) - bits(sine_rounded(x)).astype(np.int64))
    print(f"sinf vs rounded double sine: {np.mean(d != 0):.2%} of {d.size} arguments one ulp apart")
    assert d.max() <= 1


def test_cli_short_wraps_like_x86():
    """main.cpp:36 built with g++ -O3 on x86-64 converts these so."""
    y = np.array([1.0, 1.05, -1.05, 1.9999, 70000.0, np.nan, -1.0, 0.99999, -0.3, 0.3], np.float32)
    want = np.array([-32768, -31130, 31130, -4, 0, 0, -32768, 32767, -9830, 9830], np.int16)
    assert np.array_equal(cli_short(y), want)
    assert cli_short(y).dtype == np.int16


@pytest.mark.parametrize("name", EXACT_PATTERNS)
def test_fixed_gains_end_to_end(oracle, ref_or_digests, name):
    """Full-scale square waves through a fixed-gain model: g and r are exactly the pattern's, the composition with them
    and the CLI's conversion is run_pcm16's int16 output (wrapped where the overshoot passes |1|: pass, comb), and the
    float and int16 outputs are the compiled reference's."""
    model = pattern_model(name)
    g_want, r_want = pattern_gains(name)
    hw, _ = oracle.tables()
    x16 = wrap_pcm16()
    ys, o16s, wrapped = [], [], 0
    for s in range(x16.shape[0]):
        xf = x16[s].astype(np.float32) / np.float32(32768)     # main.cpp:34 (exact: a power of two)
        h = oracle.create(model)
        y, gr, taps = oracle.process_stream(h, xf, taps=True)
        oracle.destroy(h)
        assert same_bits(gr, np.tile(np.concatenate([g_want, r_want]), (len(taps), 1)))
        mem = np.zeros(FRAME, np.float32)
        comp = np.concatenate([synthesize(oracle, tp.np("X")[:800], tp.np("P")[:800], tp.silence, g_want, r_want, mem, hw)
                               for tp in taps])
        assert same_bits(comp, y)
        o16, _ = oracle.run_pcm16(model, x16[s])
        assert np.array_equal(cli_short(comp)[FRAME:], o16)
        wrapped += int(np.sum(np.abs(y[FRAME:]) >= 1.0))
        assert sum(1 for tp in taps if not tp.silence) > len(taps) // 2
        ys.append(y)
        o16s.append(o16)
    if name in ("pass", "comb"):
        assert wrapped > 0, "the overshoot must take some samples past full scale"
    if name == "mute":
        assert not np.any(np.stack(ys)) and not np.any(np.stack(o16s))
    print(f"{name}: {wrapped} samples wrapped")
    ref, table = ref_or_digests
    if ref is not None:
        ref.set_model(model)
        for s in range(x16.shape[0]):
            h = ref.create()
            y_ref, _ = ref.process_stream(h, x16[s].astype(np.float32) / np.float32(32768))
            ref.destroy(h)
            assert same_bits(ys[s], y_ref), (name, s)
            assert np.array_equal(o16s[s], ref.run_pcm16(x16[s])[0]), (name, s)
    assert digest(np.stack(ys), np.stack(o16s)) == table[name], name
