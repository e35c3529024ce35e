"""The synthesis kernel (synthesis_kernel, percepnet_b200/csrc/pnb_dsp.cu: pitch_filter, interp_band_gain, the gain
apply, the optional post-filter, the Hermitian extension, the inverse FFT-960, the window, overlap-add and the int16
conversion) against the CPU restatement (tests/synthesis_oracle.py, pinned to the reference by
tests/test_oracle_synthesis.py) at the kernel's OWN inputs: the X, P, silence and gain taps and the g/r it read, taken
back from the device after every call, so no network error is mixed in.

Bars: every output sample BIT-IDENTICAL to the composition, in float and through the CLI's int16 conversion (wrapped
samples included).  The post-filtered gains: bit-identical to the restatement with the device's sine (the double sine
rounded to float); the reference calls the C library's sinf, which is one ulp away on about 1.3 % of the arguments, so
against oracle.post_filter no band more than 4 ulp away (the fraction of identical frames is printed).  With the fixed-gain models
(g, r exactly 0 or 1 on both network paths) the whole enhancement path is bit-identical to the oracle end to end, and
the int16 wire format to the CLI's output."""
import numpy as np
import pytest

from synthesis_oracle import (EXACT_PATTERNS, FRAME, cli_short, pattern_gains, pattern_model, post_filter, sine_rounded,
                              synthesize, wrap_pcm16)
from test_gpu_parity import _inputs
from util import bits, random_mixtures, same_bits

pytestmark = pytest.mark.gpu

S = 37                     # not a multiple of the kernel's 4 streams per block, and more than one block
FMAX, CALLS = 9, (8, 7, 9)  # the overlap-add memory crosses two call boundaries
F = sum(CALLS)
# one ulp of the sine moves gw by at most one, e1 and through q the common factor G by about one more, and G * gw
# rounds once: 4 ulp leaves room for both roundings of the chain (3 measured on an H100 80GB HBM3 at 700 W)
PF_MAX_ULP = 4


@pytest.fixture(scope="module")
def api():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device")
    from percepnet_b200 import api
    api.load_library()
    return api


@pytest.fixture(scope="module")
def models(model0):
    return {"model0": model0, "ramp": pattern_model("ramp"), "stripes": pattern_model("stripes")}


@pytest.fixture(scope="module")
def hw(oracle):
    return oracle.tables()[0]


def _engine_flags(api, name):
    return {"fp32": api.NN_FP32, "tensor": api.NN_TENSOR, "fp32_postfilter": api.NN_FP32 | api.POSTFILTER,
            "tensor_postfilter": api.NN_TENSOR | api.POSTFILTER}[name]


def _batch(loud):
    """[37, F*480] float32: the parity inputs at unit scale (12 streams) and at `loud` (12), and 13 random mixtures whose
    exact-silence gaps toggle the silence flag inside a stream."""
    x = np.concatenate([_inputs(1.0, F), _inputs(loud, F), random_mixtures(13, F, seed=3737)]).astype(np.float32)
    assert x.shape == (S, F * FRAME)
    return x


def _compose(oracle, hw, taps, g, r, mem):
    """The restatement of one call at the kernel's inputs: taps = (X [n,S,800], P [n,S,800], silence [n,S]), g the
    gains as applied and r, [n,S,34] each; mem [S,480] carried across calls.  Returns [S, n*480] float32."""
    X, P, sil = taps
    n = X.shape[0]
    out = np.empty((S, n * FRAME), np.float32)
    for s in range(S):
        for k in range(n):
            out[s, k * FRAME:(k + 1) * FRAME] = synthesize(oracle, X[k, s], P[k, s], sil[k, s], g[k, s], r[k, s], mem[s], hw)
    return out


def _read_taps(eng, n):
    return eng.read_tap("X", n), eng.read_tap("P", n), eng.read_tap("pitch", n)[..., 2]


def _assert_same(got, want, what):
    """Bit-identical floats (or equal integers), with where it first differs when not."""
    if got.dtype == np.int16:
        bad = got != want
    else:
        bad = ~((bits(got) == bits(want)) | ((got == 0) & (want == 0)))
    if bad.any():
        s, i = np.argwhere(bad)[0]
        d = np.abs(got.astype(np.float64) - want.astype(np.float64))
        pytest.fail(f"{what}: {int(bad.sum())} samples differ, first at stream {s} hop {i // FRAME} sample {i % FRAME} "
                    f"({got[s, i]!r} vs {want[s, i]!r}), max |diff| {d.max():.3g}")


@pytest.mark.parametrize("model_name", ["model0", "ramp", "stripes"])
@pytest.mark.parametrize("engine", ["fp32", "tensor", "fp32_postfilter", "tensor_postfilter"])
def test_own_inputs_bit_exact(api, oracle, models, hw, engine, model_name):
    """Every sample of every stream equals the composition at the kernel's own inputs, call after call."""
    flags = _engine_flags(api, engine)
    # the tensor path keeps model0's network inside the domain of the reference's tansig_approx only up to a few hundred
    # times the CLI's scale (test_gpu_tensor_path); the fixed-gain models' all-zero layers are safe at any scale
    loud = 256.0 if (flags & api.NN_TENSOR and model_name == "model0") else 32768.0
    x = _batch(loud)
    eng = api.Engine(S, FMAX, models[model_name], flags | api.KEEP_TAPS)
    mem = np.zeros((S, FRAME), np.float32)
    silent = voiced = 0
    t0 = 0
    for n in CALLS:
        out, gr = eng.process(x[:, t0 * FRAME:(t0 + n) * FRAME], want_gr=True)
        taps = _read_taps(eng, n)
        g_used = eng.read_tap("g_used", n)
        if not flags & api.POSTFILTER:
            assert same_bits(g_used, gr[..., :34])
        want = _compose(oracle, hw, taps, g_used, gr[..., 34:], mem)
        _assert_same(out, want, f"{engine} {model_name} hops {t0}..{t0 + n - 1}")
        silent += int(np.sum(taps[2] != 0))
        voiced += int(np.sum(taps[2] == 0))
        t0 += n
    eng.close()
    print(f"{engine} {model_name}: {S} streams x {F} hops bit-identical ({silent} silent, {voiced} non-silent frames)")
    assert silent > 0 and voiced > 0


def test_device_buffers_and_int16_wire(api, oracle, models, hw):
    """The same bits through pnb_process_device_f32 (torch buffers, g/r written to device memory) and through
    pnb_submit_host_i16 / pnb_wait: the int16 output is cli_short of the composition, wrapped samples included (the
    int16 leg runs the pass-through model, whose overshoot on clipped input passes full scale)."""
    import torch
    from percepnet_b200.synth import to_int16
    model = models["ramp"]
    x = _batch(32768.0)
    eng = api.Engine(S, FMAX, model, api.NN_FP32 | api.KEEP_TAPS)
    mem = np.zeros((S, FRAME), np.float32)
    t0 = 0
    for n in CALLS:
        d_in = torch.from_numpy(np.ascontiguousarray(x[:, t0 * FRAME:(t0 + n) * FRAME])).cuda()
        d_out = torch.full_like(d_in, 7.0)
        d_gr = torch.empty((n, S, 68), dtype=torch.float32, device="cuda")
        torch.cuda.synchronize()
        eng.process_device(d_in.data_ptr(), d_in.stride(0), d_out.data_ptr(), d_out.stride(0), n, d_gr=d_gr.data_ptr())
        torch.cuda.synchronize()
        gr = d_gr.cpu().numpy()
        want = _compose(oracle, hw, _read_taps(eng, n), eng.read_tap("g_used", n), gr[..., 34:], mem)
        _assert_same(d_out.cpu().numpy(), want, f"process_device hops {t0}..{t0 + n - 1}")
        t0 += n
    eng.close()

    # int16 on the wire: unit-scale inputs, the same inputs 1.25 times louder (clipped to full scale: the synthesis
    # overshoots and the conversion wraps), random mixtures
    u = _inputs(1.0, F)
    x16 = np.concatenate([to_int16(u), to_int16(u * np.float32(1.25)), to_int16(random_mixtures(13, F, seed=3737))])
    eng = api.Engine(S, FMAX, pattern_model("pass"), api.NN_FP32 | api.KEEP_TAPS)
    mem = np.zeros((S, FRAME), np.float32)
    wrapped = 0
    t0 = 0
    for n in CALLS:
        xin = np.ascontiguousarray(x16[:, t0 * FRAME:(t0 + n) * FRAME])
        out16 = np.full_like(xin, 77)
        eng.submit(xin, out16)
        eng.wait()
        gr = eng.read_tap("gr", n)
        y = _compose(oracle, hw, _read_taps(eng, n), eng.read_tap("g_used", n), gr[..., 34:], mem)
        _assert_same(out16, cli_short(y), f"submit int16 hops {t0}..{t0 + n - 1}")
        wrapped += int(np.sum(np.abs(y) >= 1.0))
        t0 += n
    eng.close()
    print(f"int16 wire: {wrapped} wrapped samples")
    assert wrapped > 0


@pytest.mark.parametrize("engine", ["fp32_postfilter", "tensor_postfilter"])
def test_postfilter_at_own_inputs(api, oracle, models, engine):
    """The post-filtered gains (g_used tap) from the device's own g and Ex taps: bit-identical to the restatement with
    the device's sine on every frame, and within PF_MAX_ULP of oracle.post_filter (the reference's sinf)."""
    flags = _engine_flags(api, engine)
    frames = same = 0
    hist = np.zeros(PF_MAX_ULP + 2, np.int64)        # bands by ulp distance from the oracle; the last bin: beyond
    for model_name in ("model0", "ramp"):
        loud = 256.0 if (flags & api.NN_TENSOR and model_name == "model0") else 32768.0
        x = _batch(loud)
        eng = api.Engine(S, FMAX, models[model_name], flags | api.KEEP_TAPS)
        t0 = 0
        for n in CALLS:
            _, gr = eng.process(x[:, t0 * FRAME:(t0 + n) * FRAME], want_gr=True)
            g_used, ex = eng.read_tap("g_used", n), eng.read_tap("Ex", n)
            for k in range(n):
                for s in range(S):
                    got, g, e = g_used[k, s], gr[k, s, :34], ex[k, s]
                    assert same_bits(got, post_filter(g, e, sine_rounded)), (model_name, t0 + k, s)
                    want = oracle.post_filter(g, e)
                    ulp = np.abs(bits(got).astype(np.int64) - bits(want).astype(np.int64))
                    ulp[(got == 0) & (want == 0)] = 0
                    hist += np.bincount(np.minimum(ulp, PF_MAX_ULP + 1), minlength=hist.size)
                    same += int(not ulp.any())
                    frames += 1
            t0 += n
        eng.close()
    print(f"{engine}: post-filtered gains bit-identical to the reference's on {same / frames:.2%} of {frames} frames; "
          f"bands by ulp distance 0..{PF_MAX_ULP}: {hist[:-1].tolist()}, beyond: {hist[-1]}")
    assert hist[-1] == 0


_ORACLE_OUT = {}


def _e2e_inputs():
    return np.concatenate([_inputs(1.0, 12, n_synth=2), _inputs(32768.0, 12, n_synth=2)]).astype(np.float32)


@pytest.mark.parametrize("path", ["fp32", "tensor"])
@pytest.mark.parametrize("name", EXACT_PATTERNS)
def test_fixed_gains_end_to_end(api, oracle, name, path):
    """With g, r exactly 0 or 1 the engine's float output is oracle.process_stream's bit for bit, and its int16 wire
    output (first hop dropped) is the CLI's (oracle.run_pcm16) sample for sample, wrapped samples included."""
    model = pattern_model(name)
    flags = api.NN_TENSOR if path == "tensor" else api.NN_FP32
    g, r = pattern_gains(name)
    x = _e2e_inputs()
    if name not in _ORACLE_OUT:
        _ORACLE_OUT[name] = oracle.process_streams(model, x)
    eng = api.Engine(x.shape[0], 12, model, flags)
    out, gr = eng.process(x, want_gr=True)
    eng.close()
    assert same_bits(gr, np.broadcast_to(np.concatenate([g, r]), gr.shape)), "g/r are not exactly the pattern's"
    _assert_same(out, _ORACLE_OUT[name], f"{path} {name} float")
    if name == "mute":
        assert not np.any(out)
    if name not in ("pass", "comb"):
        return
    x16 = wrap_pcm16()
    n = x16.shape[1] // FRAME
    eng = api.Engine(x16.shape[0], n, model, flags)
    o16, _ = eng.process(x16)
    eng.close()
    want = np.stack([oracle.run_pcm16(model, x16[s])[0] for s in range(x16.shape[0])])
    _assert_same(o16[:, FRAME:], want, f"{path} {name} int16")
    # the samples whose float value passed full scale, where the conversion wrapped
    xf = x16.astype(np.float32) / np.float32(32768)
    wrapped = 0
    for s in range(x16.shape[0]):
        h = oracle.create(model)
        y, _, _ = oracle.process_stream(h, xf[s])
        oracle.destroy(h)
        wrapped += int(np.sum(np.abs(y[FRAME:]) >= 1.0))
    print(f"{path} {name}: int16 output identical to the CLI's, {wrapped} wrapped samples")
    assert wrapped > 0
