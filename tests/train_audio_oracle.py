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
expose.  The synthesis steps are those of the enhancement path (tests/synthesis_oracle.py); every float operation is one
IEEE single-precision operation on the same operands as the reference's, so the result is the reference's bit for bit
(tests/test_oracle_train_audio.py pins it to the reference's own files).
"""
import numpy as np

from synthesis_oracle import FRAME, synthesize, to_short


def noisy_analysis(oracle, noisy16):
    """Per frame of the noisy stream: (Y [481] complex64 as 962 interleaved floats, Phat likewise, silence)."""
    from percepnet_b200.weights import synth_model
    model = synth_model(0)            # the taps' analysis does not depend on the network that runs after it
    h = oracle.create(model)
    _, _, taps = oracle.process_stream(h, np.asarray(noisy16, np.float32), taps=True)   # NORM_RATIO 1
    oracle.destroy(h)
    return [(t.np("X"), t.np("P"), int(t.silence)) for t in taps]


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
        out[t * FRAME:(t + 1) * FRAME] = to_short(synthesize(oracle, Y, P, silence, rec[t, 70:104], rec[t, 104:138],
                                                             mem, hw))
    return rec, to_short(noisy16), out
