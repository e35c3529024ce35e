"""The synthesis half of rnnoise_process_frame (src/denoise.cpp:536-544 after compute_rnn) on the CPU, composed from
the oracle's stage functions (oracle/pn_oracle.c): the restatement the GPU's synthesis kernel is checked against at its
own inputs, and the int16 conversions of the CLI (src/main.cpp:36) and of train() (src/denoise.cpp:755-758).

    if (!silence) pitch_filter(X, P, ..., g, r);             :536-538
    interp_band_gain(gf, g);  X *= gf;                       :539-544
    frame_synthesis(st, out, X);                             :352-359 (inverse transform :306-324, window, overlap-add)

Every float operation is one IEEE single-precision operation on the same operands as the reference's, so the result is
the reference's bit for bit (tests/test_oracle_synthesis.py pins it to oracle.process_stream and to the reference).

Also the envelope post-filter with a choice of sine (the reference's sinf or the device's rounded double sine), and the
fixed-gain models: networks whose output layers compute sigmoid_approx(bias) whatever the features are, so that
g and r are known exactly on every network path and the enhancement path can be compared end to end bit for bit.
"""
import math

import numpy as np

FRAME, WIN, NFREQ, NBANDS = 480, 960, 481, 34


def _spectrum(v):
    """962 interleaved floats (481 bins) from a spectrum tap: the device keeps bins 0..399 (800 floats); from bin 400 up
    every gain is zero (DESIGN.md section 2), so zero padding changes at most the sign of zeros."""
    a = np.zeros(2 * NFREQ, np.float32)
    v = np.asarray(v, np.float32).ravel()
    a[:v.size] = v
    return a


def gained_spectrum(oracle, X, P, silence, g, r):
    """The spectrum frame_synthesis transforms: X comb-mixed with P unless the frame is silent, then times the per-bin
    gains interpolated from g (the gains as applied: with the post-filter, the filtered ones)."""
    Y = _spectrum(X)
    if not silence:
        Y = oracle.pitch_filter(Y, _spectrum(P), np.asarray(r, np.float32))
    gf = oracle.interp_band_gain(np.asarray(g, np.float32))
    Y[0::2] *= gf
    Y[1::2] *= gf
    return Y


def frame_synthesis(oracle, Y, mem, hw):
    """denoise.cpp:306-324 (inverse_transform) and :352-359: out [480] float32; mem is updated in place."""
    a = np.zeros(2 * WIN, np.float32)
    a[:2 * NFREQ] = Y
    k = WIN - np.arange(NFREQ, WIN)                       # x[i] = conj(x[960 - i]) for i in [481, 960)
    a[2 * NFREQ::2] = a[2 * k]
    a[2 * NFREQ + 1::2] = -a[2 * k + 1]
    b = oracle.fft960(a)[0::2]                            # real parts
    x = np.empty(WIN, np.float32)
    x[0] = np.float32(WIN) * b[0]
    x[1:] = np.float32(WIN) * b[WIN - np.arange(1, WIN)]
    x[:FRAME] *= hw                                       # apply_window, :282-289
    x[WIN - 1 - np.arange(FRAME)] *= hw
    out = x[:FRAME] + mem
    mem[:] = x[FRAME:]
    return out


def synthesize(oracle, X, P, silence, g, r, mem, hw):
    """One hop of rnnoise_process_frame after compute_rnn: out [480] float32; mem ([480] float32, the overlap-add
    memory, zero for a fresh stream) is updated in place.  hw: the half window, oracle.tables()[0]."""
    return frame_synthesis(oracle, gained_spectrum(oracle, X, P, silence, g, r), mem, hw)


def sine_libm(x):
    """sinf of the C library, as the reference's post_filtering calls it (denoise.cpp:227): float32 array."""
    global _sinf
    if _sinf is None:
        import ctypes
        import ctypes.util
        _sinf = ctypes.CDLL(ctypes.util.find_library("m")).sinf
        _sinf.restype, _sinf.argtypes = ctypes.c_float, [ctypes.c_float]
    return np.array([_sinf(float(v)) for v in np.asarray(x, np.float32).ravel()], np.float32)


_sinf = None


def sine_rounded(x):
    """The device's sine (synthesis_kernel, train_labels_kernel): the double sine of the float argument, rounded to
    float.  glibc's sinf is not correctly rounded: about 1.3 % of the arguments in [0, pi/2] come out one ulp away."""
    return np.array([math.sin(float(v)) for v in np.asarray(x, np.float32).ravel()]).astype(np.float32)


def post_filter(g, Ey, sine):
    """The envelope post-filter, denoise.cpp:216-250 (beta = 0.02), one IEEE single-precision operation per step as
    oracle.post_filter, with the sine of (float)(M_PI/2 * g) taken from `sine` (sine_libm: the reference's;
    sine_rounded: the device's).  Returns the filtered g [34] float32."""
    g = np.asarray(g, np.float32)
    Ey = np.asarray(Ey, np.float32)
    gw = g * sine((np.pi / 2 * g.astype(np.float64)).astype(np.float32))
    e0 = e1 = np.float32(0)
    for i in range(NBANDS):
        e0 = np.float32(e0 + g[i] * Ey[i])
    for i in range(NBANDS):
        e1 = np.float32(e1 + gw[i] * Ey[i])
    beta, one = np.float32(0.02), np.float32(1)
    q = e0 / (e1 + np.float32(1e-6))
    G = np.sqrt(((one + beta) * q) / (one + beta * (q * q)))
    return (G * gw).astype(np.float32)


def to_short(v):
    """(short)fmax(-32768, fmin(32767, v)) with v promoted to double, as in train() (NaN gives 32767)."""
    return np.trunc(np.fmax(-32768.0, np.fmin(32767.0, np.asarray(v, np.float64)))).astype(np.int16)


def cli_short(y):
    """src/main.cpp:36, `tmp[i] = x[i]*32768` into a short, as g++ compiles it on x86-64: the product rounded to float,
    truncated to int32 by cvttss2si (out of range or NaN: INT_MIN), the low 16 bits kept.  So the output wraps:
    1.0 -> -32768, 1.05 -> -31130, -1.05 -> 31130, 1.9999 -> -4, 70000 -> 0, NaN -> 0.

    The device's (short)(int)(y*32768.f) agrees wherever |y| < 65536.  Beyond, its conversion saturates instead
    (+huge -> INT_MAX -> -1 where x86 gives 0); an int16-in / int16-out call cannot get there, so that is not tested."""
    p = np.asarray(y, np.float32) * np.float32(32768)
    with np.errstate(invalid="ignore"):
        ok = (p >= -2.0 ** 31) & (p < 2.0 ** 31)          # False for NaN
    i = np.where(ok, np.trunc(np.where(ok, p, 0)).astype(np.int64), -2 ** 31)
    return (i & 0xFFFF).astype(np.uint16).view(np.int16)


# --------------------------------------------------------------------------------------------- fixed-gain models
def fixed_gain_model(g_bias, r_bias):
    """A PackedModel with the shapes of synth_model(0) whose every weight and bias is zero except the 34 fc_gb and the
    34 fc_rb biases: every layer before them outputs exactly 0 (and conv2 stays far from the tensor path's domain
    limit), so the network's g and r are sigmoid_approx(g_bias) and sigmoid_approx(r_bias) on every path, for any
    input.  A bias of +-40 gives exactly 1.0 / 0.0 (tansig_approx(+-20) is the table's last entry, 1.0, with dy = 0)."""
    from percepnet_b200.weights import LAYERS, PackedModel
    z = lambda *shape: np.zeros(shape, np.float32)   # noqa: E731
    arrays = {}
    for spec in LAYERS:
        name, kind = spec[0], spec[1]
        if kind == "dense":
            arrays[name + "_weights"], arrays[name + "_bias"] = z(spec[2], spec[3]), z(spec[3])
        elif kind == "conv":
            arrays[name + "_weights"], arrays[name + "_bias"] = z(spec[3], spec[2], spec[4]), z(spec[4])
        else:
            m, h = spec[2], spec[3]
            arrays[name + "_weights"], arrays[name + "_recurrent_weights"] = z(m, 3 * h), z(h, 3 * h)
            arrays[name + "_bias"] = z(6 * h)
    arrays["fc_gb_bias"] = np.ascontiguousarray(g_bias, np.float32).reshape(NBANDS)
    arrays["fc_rb_bias"] = np.ascontiguousarray(r_bias, np.float32).reshape(NBANDS)
    return PackedModel(arrays)


_ON, _OFF = 40.0, -40.0
_ALT = np.arange(NBANDS) % 2 == 0

# name -> (g bias, r bias).  pass: g = 1, r = 0; comb: g = 1, r = 1; mute: g = 0; stripes: g 1/0 and r 0/1 alternating
# across neighbouring bands (the steepest interpolation at every band border); ramp: intermediate g and r.
GAIN_PATTERNS = {
    "pass": (np.full(NBANDS, _ON), np.full(NBANDS, _OFF)),
    "comb": (np.full(NBANDS, _ON), np.full(NBANDS, _ON)),
    "mute": (np.full(NBANDS, _OFF), np.full(NBANDS, _OFF)),
    "stripes": (np.where(_ALT, _ON, _OFF), np.where(_ALT, _OFF, _ON)),
    "ramp": (np.linspace(-5.9, 5.9, NBANDS), np.linspace(5.3, -5.7, NBANDS)),
}
# the patterns whose g and r are exactly 0 or 1 on every network path (the tensor path's sigmoid uses fmaf, so the
# intermediate values of `ramp` may differ from the oracle's in the last bit)
EXACT_PATTERNS = ("pass", "comb", "mute", "stripes")


def pattern_model(name):
    return fixed_gain_model(*GAIN_PATTERNS[name])


def pattern_gains(name):
    """The exact g, r of an EXACT_PATTERNS model: [34] float32 each."""
    g, r = GAIN_PATTERNS[name]
    return (np.asarray(g) > 0).astype(np.float32), (np.asarray(r) > 0).astype(np.float32)


def wrap_pcm16(n_frames=16):
    """[2, n_frames*480] int16: full-scale square waves (150 Hz, and 450 Hz with a phase offset).  The synthesis cuts
    everything above bin 400 (20 kHz), so the pass-through's Gibbs overshoot takes |y| above 1 and the CLI's
    conversion wraps."""
    t = np.arange(n_frames * FRAME) / 48000.0
    a = np.where(np.sin(2 * np.pi * 150.0 * t) >= 0, 32767, -32768)
    b = np.where(np.sin(2 * np.pi * 450.0 * t + 1.0) >= 0, 32767, -32768)
    return np.stack([a, b]).astype(np.int16)
