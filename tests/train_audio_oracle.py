"""train() with its TEST block (src/denoise.cpp:722-728, 742-759) on in-memory int16 "files", on the CPU, composed from
the oracle's stage functions (oracle/pn_oracle.c) -- the reference the GPU's training-data audio is checked against.

For every frame train() writes the noisy frame to test_input.pcm, then resynthesises it with the frame's own labels
and writes the result to test_output.pcm:

    post_filtering(g, Ey);                                   :743   (the g of the record, pn_oracle_train_records)
    if (!silence) pitch_filter(Y, Phat, ..., g, r);          :744-746
    interp_band_gain(gf, g);  Y *= gf;                       :747-752
    frame_synthesis(st, out, Y);                             :754   (inverse transform, window, overlap-add)
    out_short = (short)fmax(-32768, fmin(32767, out));       :755-758

Y, Phat and silence are the noisy stream's analysis (compute_frame_features, :734), which the oracle's per-frame taps
expose.  Every float operation below is one IEEE single-precision operation on the same operands as the reference's,
so the result is the reference's bit for bit (tests/test_oracle_train_audio.py pins it to the reference's own files).
"""
import numpy as np

FRAME, WIN, NFREQ = 480, 960, 481


def noisy_analysis(oracle, noisy16):
    """Per frame of the noisy stream: (Y [481] complex64 as 962 interleaved floats, Phat likewise, silence)."""
    from percepnet_b200.weights import synth_model
    model = synth_model(0)            # the taps' analysis does not depend on the network that runs after it
    h = oracle.create(model)
    _, _, taps = oracle.process_stream(h, np.asarray(noisy16, np.float32), taps=True)   # NORM_RATIO 1
    oracle.destroy(h)
    return [(t.np("X"), t.np("P"), int(t.silence)) for t in taps]


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


def to_short(v):
    """(short)fmax(-32768, fmin(32767, v)) with v promoted to double, as in train() (NaN gives 32767)."""
    return np.trunc(np.fmax(-32768.0, np.fmin(32767.0, np.asarray(v, np.float64)))).astype(np.int16)


def train_audio(oracle, speech16, noisy16):
    """[count*480] int16 each -> (records [count, 138] float32, test_input [count*480] int16, test_output [count*480]
    int16), what train() writes to <output>, test_input.pcm and test_output.pcm."""
    speech16 = np.ascontiguousarray(speech16, np.int16)
    noisy16 = np.ascontiguousarray(noisy16, np.int16)
    rec = oracle.train_records(speech16, noisy16)
    hw, _ = oracle.tables()
    mem = np.zeros(FRAME, np.float32)                     # the synthesis memory of train()'s `st`
    out = np.empty(noisy16.size, np.int16)
    for t, (Y, P, silence) in enumerate(noisy_analysis(oracle, noisy16)):
        g, r = rec[t, 70:104], rec[t, 104:138]
        if not silence:
            Y = oracle.pitch_filter(Y, P, r)
        gf = oracle.interp_band_gain(g)
        Y = Y.copy()
        Y[0::2] *= gf
        Y[1::2] *= gf
        out[t * FRAME:(t + 1) * FRAME] = to_short(frame_synthesis(oracle, Y, mem, hw))
    return rec, to_short(noisy16), out
