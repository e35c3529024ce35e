"""The training-data generator's ideal-gain audio on the GPU (flag PNB_TRAIN_AUDIO, pnb_train_audio_*): every noisy
file resynthesised with its own labels, as the reference's train() writes test_output.pcm (src/denoise.cpp:742-759),
against the CPU restatement (tests/train_audio_oracle.py, pinned to the reference) and against what the reference itself wrote
(tests/golden/train_audio.npz).

Bars: records exactly as a PNB_TRAIN_DATA engine writes them.  At the synthesis kernel's own inputs -- the labels
the device wrote and its analysis taps of the noisy rows -- the audio is bit-identical to the restatement
(tests/synthesis_oracle.py), clamped samples included: the device's synthesis is the reference's operation for
operation.  Against the oracle's own records and the reference's files the audio is within 1 LSB: about 0.6 % of g
labels differ by an ulp through the post-filter's sinf (the device rounds a double sine), so a sample may truncate to the
neighbouring integer.  At least 99 % of the samples must be identical there (measured on an H100 80GB HBM3 at 700 W:
100 % against the oracle and against the reference, every sample of these inputs).
"""
import os

import numpy as np
import pytest

from conftest import GOLDEN
from synthesis_oracle import FRAME, synthesize, to_short
from train_audio_oracle import train_audio
from util import same_bits

pytestmark = pytest.mark.gpu

SAME_FLOOR = 0.99


@pytest.fixture(scope="module")
def api():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device")
    from percepnet_b200 import api
    api.load_library()
    return api


def _audio_close(got, want, what):
    assert got.shape == want.shape and got.dtype == np.int16
    d = np.abs(got.astype(np.int32) - want.astype(np.int32))
    same = float(np.mean(d == 0))
    print(f"{what}: {same:.2%} of {got.size} samples identical, max |diff| {d.max()} LSB")
    assert d.max() <= 1, (what, d.max())
    assert same >= SAME_FLOOR, (what, same)


def _pairs():
    """Speech-like pairs at several SNRs plus a silent noisy file and a noisy file with a silent stretch."""
    from percepnet_b200.synth import synth_pairs
    F = 36
    clean, noisy = synth_pairs(5, F, seed=515)
    gap = noisy[1:2].copy()
    gap[:, 10 * 480:20 * 480] = 0
    clean = np.concatenate([clean, clean[:1], clean[1:2]])
    noisy = np.concatenate([noisy, np.zeros_like(noisy[:1]), gap])
    return clean, noisy, F


def test_audio_matches_reference_golden(api):
    g = np.load(os.path.join(GOLDEN, "train.npz"))
    a = np.load(os.path.join(GOLDEN, "train_audio.npz"))
    speech, noisy = g["speech"], g["noisy"]
    N, F = speech.shape[0], speech.shape[1] // 480
    eng = api.Engine(2 * N, F, None, api.TRAIN_DATA | api.TRAIN_AUDIO | api.KEEP_TAPS)
    rec, audio = eng.train_audio(speech, noisy)
    silent = eng.read_tap("pitch", F)[:, :N, 2]
    eng.close()
    assert np.mean(silent) < 0.25, "most frames must be non-silent so that pitch_filter runs"
    assert np.array_equal(a["test_input"], noisy)
    _audio_close(audio, a["test_output"], "reference test_output.pcm")
    plain = api.Engine(2 * N, F, None, api.TRAIN_DATA)
    assert same_bits(rec, plain.train_records(speech, noisy))
    plain.close()


def test_audio_matches_oracle_and_records_unchanged(api, oracle):
    clean, noisy, F = _pairs()
    N = clean.shape[0]
    eng = api.Engine(2 * N, F, None, api.TRAIN_DATA | api.TRAIN_AUDIO | api.KEEP_TAPS)
    rec, audio = eng.train_audio(clean, noisy)
    silent = eng.read_tap("pitch", F)[:, :5, 2]
    eng.close()
    assert np.mean(silent) < 0.25, "most frames of the speech-like pairs must be non-silent"
    want = [train_audio(oracle, clean[k], noisy[k]) for k in range(N)]
    assert all(np.array_equal(w[1], noisy[k]) for k, w in enumerate(want))
    _audio_close(audio, np.stack([w[2] for w in want]), "oracle test_output")
    assert not np.any(audio[5]), "a silent noisy file resynthesises to silence"
    # the records are bit-identical to those of an engine without the flag
    plain = api.Engine(2 * N, F, None, api.TRAIN_DATA)
    assert same_bits(rec, plain.train_records(clean, noisy))
    plain.close()


def _clamping_pair(n_frames):
    """A pair loud enough that the resynthesis leaves the int16 range (as tests/test_oracle_train_audio.py builds it)."""
    t = np.arange(n_frames * FRAME) / 48000.0
    sq = np.sign(np.sin(2 * np.pi * 150 * t)) + 0.6 * np.sign(np.sin(2 * np.pi * 450 * t + 1))
    return np.clip(np.rint(sq * 32767), -32768, 32767).astype(np.int16)


def test_audio_at_own_inputs_bit_exact(api, oracle):
    """The audio equals the synthesis composed from each record's g/r and the noisy rows' X, P and silence taps,
    followed by train()'s clamp, sample for sample, on the pairs above plus one that clamps at both ends."""
    clean, noisy, F = _pairs()
    loud = _clamping_pair(F)
    clean, noisy = np.concatenate([clean, loud[None]]), np.concatenate([noisy, loud[None]])
    N = clean.shape[0]
    eng = api.Engine(2 * N, F, None, api.TRAIN_DATA | api.TRAIN_AUDIO | api.KEEP_TAPS)
    rec, audio = eng.train_audio(clean, noisy)
    X, P, sil = eng.read_tap("X", F), eng.read_tap("P", F), eng.read_tap("pitch", F)[..., 2]
    eng.close()
    hw, _ = oracle.tables()
    for p in range(N):                                          # the noisy file of pair p is row p
        mem = np.zeros(FRAME, np.float32)
        want = np.concatenate([to_short(synthesize(oracle, X[t, p], P[t, p], sil[t, p], rec[p, t, 70:104],
                                                   rec[p, t, 104:138], mem, hw)) for t in range(F)])
        d = np.nonzero(audio[p] != want)[0]
        assert d.size == 0, (p, d.size, d[0], int(audio[p, d[0]]), int(want[d[0]]))
    assert np.any(audio[N - 1] == 32767) and np.any(audio[N - 1] == -32768)
    assert np.mean(sil[:, :5]) < 0.25 and np.all(sil[:, 5])        # the comb branch and the silent branch both ran


def test_call_grouping_reset_and_device_entry(api):
    """Audio and records do not depend on how frames are grouped into calls, and are the same again after a reset and
    through the device entry point."""
    import torch
    clean, noisy, F = _pairs()
    N = clean.shape[0]
    eng = api.Engine(2 * N, F, None, api.TRAIN_DATA | api.TRAIN_AUDIO)
    rec, audio = eng.train_audio(clean, noisy)
    for rounds in range(2):
        eng.reset()
        parts, t0 = [], 0
        for n in (1, 16, 7, 12):
            parts.append(eng.train_audio(clean[:, t0 * 480:(t0 + n) * 480], noisy[:, t0 * 480:(t0 + n) * 480]))
            t0 += n
        assert t0 == F
        assert same_bits(np.concatenate([p[0] for p in parts], axis=1), rec)
        assert np.array_equal(np.concatenate([p[1] for p in parts], axis=1), audio)
    eng.reset()
    d_c, d_n = torch.from_numpy(clean).cuda(), torch.from_numpy(noisy).cuda()
    d_rec = torch.full((N, F, 138), -7.0, dtype=torch.float32, device="cuda")
    d_audio = torch.full((N, F * 480 + 32), 77, dtype=torch.int16, device="cuda")   # a row stride wider than the call
    torch.cuda.synchronize()
    eng.train_audio_device(d_c.data_ptr(), F * 480, d_n.data_ptr(), F * 480, F, d_rec.data_ptr(), F * 138,
                           d_audio.data_ptr(), F * 480 + 32, 0)
    assert eng.L.pnb_wait(eng.h) == 0
    torch.cuda.synchronize()
    assert same_bits(d_rec.cpu().numpy(), rec)
    got = d_audio.cpu().numpy()
    assert np.array_equal(got[:, :F * 480], audio) and np.all(got[:, F * 480:] == 77)
    eng.close()


def test_state_migration(api):
    """Both streams of three pairs, exported mid-file and imported into an audio engine of another pair count, continue
    the records and the audio bit for bit (the overlap-add memory travels in the blob's synth piece)."""
    clean, noisy, F = _pairs()
    N, h = clean.shape[0], 20
    eng = api.Engine(2 * N, F, None, api.TRAIN_DATA | api.TRAIN_AUDIO)
    rec, audio = eng.train_audio(clean, noisy)
    eng.reset()
    eng.train_audio(clean[:, :h * 480], noisy[:, :h * 480])
    pairs = [0, 3, 6]
    blobs = eng.export_states(pairs + [N + p for p in pairs], None)
    eng.close()
    M = 4                                                       # pairs p -> slots 3, 1, 0 of the new engine
    dst = [3, 1, 0]
    e2 = api.Engine(2 * M, F, None, api.TRAIN_DATA | api.TRAIN_AUDIO)
    e2.import_states(dst + [M + q for q in dst], blobs)
    c2 = np.zeros((M, (F - h) * 480), np.int16)
    n2 = np.zeros_like(c2)
    for p, q in zip(pairs, dst):
        c2[q], n2[q] = clean[p, h * 480:], noisy[p, h * 480:]
    r2, a2 = e2.train_audio(c2, n2)
    e2.close()
    for p, q in zip(pairs, dst):
        assert same_bits(r2[q], rec[p, h:])
        assert np.array_equal(a2[q], audio[p, h * 480:])


def test_refusals_and_launch_counts(api):
    N, F = 2, 4
    with pytest.raises(api.PnbError):
        api.Engine(2 * N, F, None, api.TRAIN_AUDIO)                       # without PNB_TRAIN_DATA
    with pytest.raises(api.PnbError):
        api.Engine(2 * N, F, None, api.TRAIN_AUDIO | api.KEEP_TAPS)
    from percepnet_b200.weights import synth_model
    with pytest.raises(api.PnbError):
        api.Engine(2 * N, F, synth_model(0), api.NN_FP32 | api.TRAIN_AUDIO)  # an enhancement engine
    z = np.zeros((N, F * 480), np.int16)
    rec = np.empty((N, F, 138), np.float32)
    au = np.empty((N, F * 480), np.int16)
    audio_eng = api.Engine(2 * N, F, None, api.TRAIN_DATA | api.TRAIN_AUDIO)
    plain = api.Engine(2 * N, F, None, api.TRAIN_DATA)
    A, P = audio_eng.L, plain.L
    # the records entry points on an audio engine (its audio would have gaps), the audio ones on a plain engine
    with pytest.raises(api.PnbError):
        audio_eng.train_records(z, z)
    assert A.pnb_submit_train_records(audio_eng.h, z.ctypes.data, F * 480, z.ctypes.data, F * 480, F, rec.ctypes.data, F * 138) != 0
    assert A.pnb_train_records_device(audio_eng.h, 1, F * 480, 1, F * 480, F, 1, F * 138, None) != 0
    with pytest.raises(api.PnbError):
        plain.train_audio(z, z)
    assert P.pnb_train_audio_device(plain.h, 1, F * 480, 1, F * 480, F, 1, F * 138, 1, F * 480, None) != 0
    # short audio stride, NULL pointers, too many frames
    h = audio_eng.h
    args = [z.ctypes.data, F * 480, z.ctypes.data, F * 480, F, rec.ctypes.data, F * 138]
    assert A.pnb_train_audio_host(h, *args, au.ctypes.data, F * 480 - 1) != 0
    assert b"audio_stride" in A.pnb_last_error()
    assert A.pnb_train_audio_host(h, *args, None, F * 480) != 0
    assert A.pnb_train_audio_host(h, None, *args[1:], au.ctypes.data, F * 480) != 0
    assert A.pnb_train_audio_host(h, *args[:5], None, F * 138, au.ctypes.data, F * 480) != 0
    assert A.pnb_train_audio_host(None, *args, au.ctypes.data, F * 480) != 0
    assert A.pnb_train_audio_device(h, 1, F * 480, 1, F * 480, F, 1, F * 138, None, F * 480, None) != 0
    with pytest.raises(api.PnbError):
        audio_eng.train_audio(np.zeros((N, (F + 1) * 480), np.int16), np.zeros((N, (F + 1) * 480), np.int16))
    assert audio_eng.launches == 0 and plain.launches == 0                # nothing was enqueued by a refused call
    # launches: one more per call on the audio engine, which pnb_launches_per_call reports
    assert audio_eng.launches_per_call(F) == plain.launches_per_call(F) + 1
    for n in (F, 1, 3):
        a0, p0 = audio_eng.launches, plain.launches
        audio_eng.train_audio(z[:, :n * 480], z[:, :n * 480])
        plain.train_records(z[:, :n * 480], z[:, :n * 480])
        assert (audio_eng.launches - a0) - (plain.launches - p0) == 1
        assert audio_eng.launches_per_call(n) - plain.launches_per_call(n) == 1
    audio_eng.close()
    plain.close()


def test_cli_test_audio(api, tmp_path):
    """gen_features --test-audio, with the reference's argv and with a job list: per-job test audio files byte-equal to
    the Engine's output, records as without the option."""
    from percepnet_b200 import gen_features
    clean, noisy, F = _pairs()
    jobs = []
    for k in range(3):
        fc, fn, fo = (str(tmp_path / f"{nm}{k}") for nm in ("c", "n", "o"))
        clean[k].tofile(fc)
        noisy[k].tofile(fn)
        jobs.append((fc, fn, F - 5 * k, fo))
    eng = api.Engine(6, F, None, api.TRAIN_DATA | api.TRAIN_AUDIO)
    rec, audio = eng.train_audio(clean[:3], noisy[:3])
    eng.close()
    assert gen_features.main([jobs[0][0], jobs[0][1], str(F), jobs[0][3], "--test-audio"]) == 0
    assert np.fromfile(jobs[0][3] + ".test_output.pcm", np.int16).tobytes() == audio[0].tobytes()
    assert np.fromfile(jobs[0][3] + ".test_input.pcm", np.int16).tobytes() == noisy[0].tobytes()
    lst = tmp_path / "jobs.txt"
    lst.write_text("".join(f"{a} {b} {c} {d}\n" for a, b, c, d in jobs))
    assert gen_features.main(["--list", str(lst), "--chunk", "16", "--test-audio"]) == 0
    for k, (_, _, n, fo) in enumerate(jobs):
        assert open(fo + ".test_output.pcm", "rb").read() == audio[k, :n * 480].astype("<i2").tobytes()
        assert open(fo + ".test_input.pcm", "rb").read() == noisy[k, :n * 480].astype("<i2").tobytes()
        assert same_bits(np.fromfile(fo, np.float32).reshape(n, 138), rec[k, :n])
    os.remove(jobs[0][3] + ".test_output.pcm")
    assert gen_features.main([jobs[0][0], jobs[0][1], str(F), jobs[0][3]]) == 0     # without the option: no audio files
    assert not os.path.exists(jobs[0][3] + ".test_output.pcm")
