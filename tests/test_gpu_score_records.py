"""Scoring on the GPU: PNB_NETWORK_ONLY engines (the network without the signal path's buffers) and the device-side
CustomLoss of pnb_score_records_* (Engine.score_records), on the fp32 engine, the tensor engine and the tensor engine
with PNB_CONV_WIDE; and eval_records, which runs both.

A network-only engine computes what a PCM engine's pnb_compute_rnn_* computes, bit for bit, and its state blobs move
both ways between the two.  The loss sums are eval_records.loss_sums of the same call's predictions, to float64
rounding, and the same bits whatever else shares the call.
"""
import os

import numpy as np
import pytest

from util import crowd, same_bits

pytestmark = pytest.mark.gpu

MODES = ["fp32", "tensor", "tensor_wide"]
SIGNAL_BYTES = 39736   # offsetof(StreamState, fc_hist): the blob's signal part; the network part follows


@pytest.fixture(scope="module")
def api():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device")
    from percepnet_b200 import api
    api.load_library()
    return api


@pytest.fixture(scope="module")
def records(api):
    """[12, 36, 138] float32: train() records of synthetic pairs (inside the tensor path's domain), with labels drawn
    uniformly in [0, 1] and some set to exactly 0 and 1."""
    from percepnet_b200.synth import synth_pairs
    N, F = 12, 36
    clean, noisy = synth_pairs(N, F, seed=610)
    clean, noisy = (clean // 64).astype(np.int16), (noisy // 64).astype(np.int16)
    te = api.Engine(2 * N, F, None, api.TRAIN_DATA)
    rec = te.train_records(clean, noisy)
    te.close()
    rng = np.random.RandomState(611)
    rec[:, :, 70:] = rng.rand(N, F, 68).astype(np.float32)
    rec[:, ::5, 70:80] = 0.0
    rec[:, ::7, 110:120] = 1.0
    rec[:, 3::4, 75:77] = 1.0
    rec[:, 2::6, 130] = 0.0
    return rec


def _flags(api, mode):
    return {"fp32": api.NN_FP32, "tensor": api.NN_TENSOR, "tensor_wide": api.NN_TENSOR | api.CONV_WIDE}[mode]


def _features(rec):
    return np.ascontiguousarray(np.concatenate([rec[..., :68] * np.float32(30), rec[..., 68:70]], axis=-1))


def _host_sums(pred, rec, frames):
    from percepnet_b200.eval_records import loss_sums
    return np.stack([loss_sums(pred[i, :f], rec[i, :f]) for i, f in enumerate(frames)])


def _check_sums(got, want):
    """rtol 1e-12, counts exact, NaN exactly where the host has NaN."""
    assert got.shape == want.shape
    assert np.array_equal(got[:, 3], want[:, 3])
    assert np.array_equal(np.isnan(got), np.isnan(want))
    ok = ~np.isnan(want)
    assert np.allclose(got[ok], want[ok], rtol=1e-12, atol=0), np.abs(got[ok] - want[ok]).max()


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("fmt", ["features", "records"])
def test_network_only_same_bits_as_pcm_engine(api, model0, records, mode, fmt):
    """compute_rnn g/r and network state of a network-only engine equal a PCM engine's, over three chunked calls on an
    active range below n_streams."""
    flags = _flags(api, mode)
    x = records[:7] if fmt == "records" else _features(records[:7])
    out = {}
    for kind in ("pcm", "net"):
        eng = api.Engine(10, 16, model0, flags | (api.NETWORK_ONLY if kind == "net" else 0))
        eng.set_active(7)
        parts = [eng.compute_rnn(np.ascontiguousarray(x[:, a:b])) for a, b in ((0, 16), (16, 21), (21, 36))]
        nn = {k: v[:7] for k, v in eng.read_nn_state().items()}
        eng.check()
        out[kind] = (np.concatenate(parts, axis=1), nn)
        eng.close()
    assert same_bits(out["net"][0], out["pcm"][0])
    assert all(same_bits(out["net"][1][k], out["pcm"][1][k]) for k in out["pcm"][1])


def _signal_bytes(S, F, keep_taps):
    """Bytes of the buffers a network-only engine does not allocate (pnb_create's sizes)."""
    line_calls = 1 if F >= 128 else min(128 // F, 8)
    pcm = S * (5280 + line_calls * F * 480) * 4
    n = pcm + S * 480 * 4 + S * 4 + S * 4                       # d_pcm, d_synth, d_last_period, d_last_gain
    n += (F + 5) * S * 400 * 8 + (F + 5) * S * 34 * 4            # d_zring, d_ering
    n += F * S * 400 * 8 + F * S * 34 * 4 + F * S                # d_P, d_Ex, d_sil
    if keep_taps:
        n += F * S * 16 + F * S * 8 + F * S * 34 * 4             # pitch taps, g as applied
    return n


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("shape", [(6, 10, False), (5, 200, False), (3, 7, True)], ids=["short", "long", "taps"])
def test_device_bytes_saving(api, model0, mode, shape):
    S, F, taps = shape
    flags = _flags(api, mode) | (api.KEEP_TAPS if taps else 0)
    pcm = api.Engine(S, F, model0, flags)
    net = api.Engine(S, F, model0, flags | api.NETWORK_ONLY)
    assert pcm.device_bytes - net.device_bytes == _signal_bytes(S, F, taps)
    assert net.device_bytes > 0
    pcm.close()
    net.close()


@pytest.mark.parametrize("mode", MODES)
def test_refusals(api, model0, mode):
    """The PCM, submit, train, session and signal-tap calls of a network-only engine return PNB_ERR_ARG and launch
    nothing; invalid flag combinations are refused at create."""
    import torch
    flags = _flags(api, mode)
    S, F = 4, 6
    for bad in (api.TRAIN_DATA, api.TRAIN_AUDIO, api.TRAIN_DATA | api.TRAIN_AUDIO, api.POSTFILTER):
        with pytest.raises(api.PnbError, match=r"\(-1\)"):
            api.Engine(S, F, model0 if not bad & api.TRAIN_DATA else None, (flags if not bad & api.TRAIN_DATA else 0)
                       | bad | api.NETWORK_ONLY)
    eng = api.Engine(S, F, model0, flags | api.NETWORK_ONLY | api.KEEP_TAPS)
    L, h = eng.L, eng.h
    eng.compute_rnn(np.zeros((S, F, 70), np.float32))
    before = eng.launches
    x = np.zeros((S, F * 480), np.float32)
    x16 = np.zeros((S, F * 480), np.int16)
    rec = np.zeros((S, F, 138), np.float32)
    d_x = torch.zeros((S, F * 480), device="cuda")
    d_x16 = torch.zeros((S, F * 480), dtype=torch.int16, device="cuda")
    xp, dxp, d16 = x.ctypes.data, d_x.data_ptr(), d_x16.data_ptr()
    calls = [
        L.pnb_process_host_f32(h, xp, F * 480, xp, F * 480, F, None),
        L.pnb_process_host_i16(h, x16.ctypes.data, F * 480, x16.ctypes.data, F * 480, F, None),
        L.pnb_process_device_f32(h, dxp, F * 480, dxp, F * 480, F, None, None),
        L.pnb_process_device_i16(h, d16, F * 480, d16, F * 480, F, None, None),
        L.pnb_submit_host_f32(h, xp, F * 480, xp, F * 480, F),
        L.pnb_submit_host_i16(h, x16.ctypes.data, F * 480, x16.ctypes.data, F * 480, F),
        L.pnb_submit_device_f32(h, dxp, F * 480, dxp, F * 480, F, None),
        L.pnb_submit_device_i16(h, d16, F * 480, d16, F * 480, F, None),
        L.pnb_train_records_host(h, x16.ctypes.data, F * 480, x16.ctypes.data, F * 480, F, rec.ctypes.data, F * 138),
        L.pnb_submit_train_records(h, x16.ctypes.data, F * 480, x16.ctypes.data, F * 480, F, rec.ctypes.data, F * 138),
        L.pnb_train_records_device(h, d16, F * 480, d16, F * 480, F, dxp, F * 138, None),
        L.pnb_train_audio_host(h, x16.ctypes.data, F * 480, x16.ctypes.data, F * 480, F, rec.ctypes.data, F * 138,
                               x16.ctypes.data, F * 480),
    ]
    for k, rc in enumerate(calls):
        assert rc == -1, k
    assert b"PNB_NETWORK_ONLY" in L.pnb_last_error()
    assert L.pnb_sessions_reserve(h, 8) == -1 and b"PNB_NETWORK_ONLY" in L.pnb_last_error()
    with pytest.raises(api.PnbError, match="PNB_NETWORK_ONLY"):
        eng.process_sessions([0], x[:1])
    for tap in ("pitch", "pitchf", "X", "P", "Ex", "g_used"):
        with pytest.raises(api.PnbError, match=r"\(-1\)"):
            eng.read_tap(tap, F)
    assert eng.launches == before
    eng.read_tap("features", F)
    eng.read_tap("gr", F)
    eng.read_nn_state()
    # an accepted call: launches_per_call is one compute_rnn call
    per = eng.launches_per_call(F)
    eng.compute_rnn(rec)
    assert eng.launches == before + per
    eng.check()
    eng.close()


def _blobs(eng, n):
    import torch
    b = eng.export_states(list(range(n)), None)
    torch.cuda.synchronize()
    return b


@pytest.mark.parametrize("mode", MODES)
def test_state_moves_between_pcm_and_network_only(api, model0, records, mode):
    """A blob exported mid-stream moves either way and the stream continues with the same g/r bits; a network-only
    export has a zero signal part; reset and set_active rows equal a fresh engine's."""
    flags = _flags(api, mode)
    n, F = 5, 12
    rec = records[:n]
    x = crowd(n, F, seed=620) / np.float32(64)
    # PCM engine -> network-only engine, after a PCM call and a network call
    pcm = api.Engine(n, F, model0, flags)
    pcm.process(x)
    pcm.compute_rnn(np.ascontiguousarray(rec[:, :F]))
    blob = _blobs(pcm, n)
    assert blob.cpu().numpy()[:, 8:SIGNAL_BYTES].any()
    want = pcm.compute_rnn(np.ascontiguousarray(rec[:, F:2 * F]))
    net = api.Engine(n, F, model0, flags | api.NETWORK_ONLY)
    net.import_states(list(range(n)), blob)
    got = net.compute_rnn(np.ascontiguousarray(rec[:, F:2 * F]))
    assert same_bits(got, want)
    # network-only -> PCM: the network part carries, the signal part is zero
    nb = _blobs(net, n)
    nbh = nb.cpu().numpy()
    assert not nbh[:, 8:SIGNAL_BYTES].any()
    want = net.compute_rnn(np.ascontiguousarray(rec[:, 2 * F:3 * F]))
    pcm2 = api.Engine(n, F, model0, flags)
    pcm2.import_states(list(range(n)), nb)
    got = pcm2.compute_rnn(np.ascontiguousarray(rec[:, 2 * F:3 * F]))
    assert same_bits(got, want)
    net.check()
    pcm2.check()
    # reset rows and rows entering the active range start fresh
    fresh = api.Engine(n, F, model0, flags | api.NETWORK_ONLY)
    f_gr = fresh.compute_rnn(np.ascontiguousarray(rec[:, :F]))
    net.reset_streams([1, 3])
    net.set_active(2)
    net.set_active(n)                                # rows 2..4 enter fresh
    gr = net.compute_rnn(np.ascontiguousarray(rec[:, :F]))
    assert same_bits(gr[1:], f_gr[1:])
    net.reset()
    assert same_bits(net.compute_rnn(np.ascontiguousarray(rec[:, :F])), f_gr)
    for e in (pcm, net, pcm2, fresh):
        e.close()


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("kind", ["pcm", "net"])
def test_loss_against_the_host_reference(api, model0, records, mode, kind):
    """Per-row sums of a device-form call with wide strides equal loss_sums of the same call's predictions (frames 0, 1,
    F and in between; labels at 0 and 1; r > 1 gives NaN where the host gives NaN); its g/r are compute_rnn's bits;
    launches: compute_rnn's without g/r, one more with."""
    import torch
    flags = _flags(api, mode) | (api.NETWORK_ONLY if kind == "net" else 0)
    N, F = 8, 36
    rec = records[:N].copy()
    rec[3, 2, 120] = 1.5                              # counted: row 3's dr sum is NaN
    rec[4, 30, 110] = 1.25                            # after row 4's frames: not counted
    frames = [0, 1, F, 5, 17, F, 35, 2]
    rs, gs = F * 138 + 50, F * 68 + 9
    d_rec = torch.zeros((N, rs), device="cuda")
    d_rec[:, :F * 138] = torch.from_numpy(rec.reshape(N, -1)).cuda()
    d_gr = torch.full((N, gs), -3.0, device="cuda")
    d_sums = torch.full((N, 4), -1.0, dtype=torch.float64, device="cuda")
    eng = api.Engine(N, F, model0, flags)
    n0 = eng.launches
    eng.score_records_device(d_rec.data_ptr(), rs, F, frames, d_sums.data_ptr(), d_gr.data_ptr(), gs)
    eng.check()
    ref = api.Engine(N, F, model0, flags)
    per = ref.launches
    want_gr = ref.compute_rnn(rec)
    per = ref.launches - per
    ref.close()
    assert eng.launches - n0 == per + 1
    gr = d_gr.cpu().numpy()
    assert (gr[:, F * 68:] == -3.0).all()
    pred = gr[:, :F * 68].reshape(N, F, 68)
    assert same_bits(pred, want_gr)
    sums = d_sums.cpu().numpy()
    want = _host_sums(pred, rec, frames)
    assert np.isnan(want[3, 2]) and not np.isnan(want[4]).any()
    _check_sums(sums, want)
    assert (sums[0] == 0).all()
    # without g/r: compute_rnn's launches, the same sums; the host form too
    eng.reset()
    n0 = eng.launches
    eng.score_records_device(d_rec.data_ptr(), rs, F, frames, d_sums.data_ptr())
    eng.check()
    assert eng.launches - n0 == per
    assert np.array_equal(d_sums.cpu().numpy(), sums, equal_nan=True)
    eng.reset()
    hs, hg = eng.score_records(rec, frames, want_gr=True)
    assert np.array_equal(hs, sums, equal_nan=True) and same_bits(hg, pred)
    eng.reset()
    hs, hg = eng.score_records(rec)
    assert hg is None
    _check_sums(hs, _host_sums(pred, rec, [F] * N))
    eng.close()


@pytest.mark.parametrize("mode", MODES)
def test_sums_are_the_same_bits_whatever_shares_the_call(api, model0, records, mode):
    """Two runs, a row scored alone and inside a larger batch on an active range, PCM and network-only engines, chunked
    and whole: the same sums bit for bit."""
    flags = _flags(api, mode)
    rec = records[:9]
    frames = [36, 20, 1, 36, 33, 0, 36, 7, 36]

    def run(fl, rows, S, chunks):
        eng = api.Engine(S, max(b - a for a, b in chunks), model0, fl)
        eng.set_active(len(rows))
        x = rec[rows]
        total = np.zeros((len(rows), 4))
        for a, b in chunks:
            fr = np.clip(np.asarray(frames)[rows] - a, 0, b - a)
            s, _ = eng.score_records(np.ascontiguousarray(x[:, a:b]), fr)
            total += s
        eng.close()
        return total

    whole = [(0, 36)]
    base = run(flags | api.NETWORK_ONLY, list(range(9)), 9, whole)
    assert np.array_equal(run(flags | api.NETWORK_ONLY, list(range(9)), 9, whole), base, equal_nan=True)
    assert np.array_equal(run(flags, list(range(9)), 12, whole), base, equal_nan=True)
    for r in (0, 4, 8):
        assert np.array_equal(run(flags | api.NETWORK_ONLY, [r], 1, whole)[0], base[r], equal_nan=True)
    assert np.array_equal(run(flags | api.NETWORK_ONLY, [6, 4, 0], 5, whole), base[[6, 4, 0]], equal_nan=True)
    chunked = run(flags | api.NETWORK_ONLY, list(range(9)), 9, [(0, 10), (10, 20), (20, 36)])
    assert np.array_equal(chunked[:, 3], base[:, 3])
    assert np.allclose(chunked, base, rtol=1e-12, atol=0)


def test_score_refusals(api, model0, records):
    import torch
    S, F = 4, 8
    eng = api.Engine(S, F, model0, api.NN_FP32 | api.NETWORK_ONLY)
    L, h = eng.L, eng.h
    rec = np.ascontiguousarray(records[:S, :F])
    sums = np.zeros((S, 4))
    gr = np.zeros((S, F, 68), np.float32)
    fr = np.array([F, 0, 3, F], np.int32)
    rp, sp, gp, fp = rec.ctypes.data, sums.ctypes.data, gr.ctypes.data, fr.ctypes.data
    before = eng.launches
    bad_hi, bad_lo = np.array([F, F + 1, 0, 0], np.int32), np.array([0, 0, -1, 0], np.int32)
    refused = [
        (None, rp, F * 138, F, fp, sp, gp, F * 68),
        (h, None, F * 138, F, fp, sp, gp, F * 68),
        (h, rp, F * 138, F, fp, None, gp, F * 68),
        (h, rp, F * 138, F, fp, None, None, 0),
        (h, rp, F * 138 - 1, F, fp, sp, None, 0),
        (h, rp, F * 70, F, fp, sp, None, 0),
        (h, rp, F * 138, F, fp, sp, gp, F * 68 - 1),
        (h, rp, F * 138, F, bad_hi.ctypes.data, sp, None, 0),
        (h, rp, F * 138, F, bad_lo.ctypes.data, sp, None, 0),
        (h, rp, F * 138, 0, None, sp, None, 0),
        (h, rp, F * 138, F + 1, None, sp, None, 0),
    ]
    for args in refused:
        assert L.pnb_score_records_host(*args) == -1, args
    assert eng.launches == before
    assert L.pnb_score_records_host(h, rp, F * 138, F, fp, sp, None, 0) == 0
    eng.close()
    # refused on training-data engines and in session mode
    te = api.Engine(4, F, None, api.TRAIN_DATA)
    assert te.L.pnb_score_records_host(te.h, rp, F * 138, F, None, sp, None, 0) == -1
    te.close()
    pe = api.Engine(S, F, model0, api.NN_FP32)
    pe.reserve_sessions(8)
    assert pe.L.pnb_score_records_host(pe.h, rp, F * 138, F, None, sp, None, 0) == -1
    d_rec = torch.from_numpy(rec).cuda()
    d_sums = torch.zeros((S, 4), dtype=torch.float64, device="cuda")
    assert pe.L.pnb_score_records_device(pe.h, d_rec.data_ptr(), F * 138, F, None, d_sums.data_ptr(), None, 0, None) == -1
    pe.close()


def test_tensor_score_reports_records_past_the_domain(api, model0):
    """Records whose features drive conv2 past 8.5e7: PNB_ERR_DOMAIN from the host form and from pnb_wait after the
    device form, as compute_rnn."""
    import torch
    S, F = 3, 5
    rec = np.full((S, F, 138), 1e9, np.float32)
    rec[:, :, 68:70] = 1.0
    rec[:, :, 70:] = 0.5
    for flags in (api.NN_TENSOR, api.NN_TENSOR | api.CONV_WIDE):
        eng = api.Engine(S, F, model0, flags | api.NETWORK_ONLY)
        with pytest.raises(api.PnbError, match="-5"):
            eng.score_records(rec)
        eng.reset()
        d_rec = torch.from_numpy(rec).cuda()
        d_sums = torch.zeros((S, 4), dtype=torch.float64, device="cuda")
        eng.score_records_device(d_rec.data_ptr(), F * 138, F, None, d_sums.data_ptr())
        assert eng.L.pnb_wait(eng.h) == -5
        eng.close()


def _table(printed):
    """{first column: (frames, g2, g4, r2, total)} of an eval_records table."""
    rows = {}
    for line in printed.strip().splitlines()[1:]:
        w = line.split()
        rows[w[0]] = (int(w[1]), *map(float, w[2:6]))
    return rows


@pytest.mark.parametrize("mode", MODES)
def test_eval_records_end_to_end(api, model0, mode, tmp_path, capsys):
    """gen_features files through eval_records.main: the printed terms are loss_sums of the --pred-dir predictions (at
    the print precision); --window L with L the longest file prints what no window prints; a file scored with
    --window w equals its w-frame pieces scored as separate files."""
    from percepnet_b200 import eval_records as E
    from percepnet_b200 import gen_features
    from percepnet_b200.synth import synth_pairs
    counts = [26, 11, 19]
    clean, noisy = synth_pairs(3, max(counts), seed=630)
    clean, noisy = (clean // 64).astype(np.int16), (noisy // 64).astype(np.int16)
    jobs, files = [], []
    for k, cnt in enumerate(counts):
        fc, fn, fo = (str(tmp_path / f"{nm}{k}") for nm in ("c", "n", "rec"))
        clean[k, :cnt * 480].tofile(fc)
        noisy[k, :cnt * 480].tofile(fn)
        jobs.append(f"{fc} {fn} {cnt} {fo}\n")
        files.append(fo)
    (tmp_path / "jobs.txt").write_text("".join(jobs))
    assert gen_features.main(["--list", str(tmp_path / "jobs.txt"), "--chunk", "16"]) == 0
    blob = str(tmp_path / "m.pnbw")
    model0.save_blob(blob)
    extra = {"fp32": [], "tensor": ["--tensor"], "tensor_wide": ["--tensor", "--conv-wide"]}[mode]
    base = ["--model", blob, "--chunk", "8", *extra]

    def run(*args):
        assert E.main([*base, *args]) == 0
        return _table(capsys.readouterr().out)

    pd = tmp_path / "pred"
    t = run("--pred-dir", str(pd), *files)
    total = np.zeros(4)
    for f, cnt in zip(files, counts):
        pred = np.fromfile(str(pd / (os.path.basename(f) + ".pred.f32")), np.float32).reshape(cnt, 68)
        s = E.loss_sums(pred, E.read_records(f))
        total += s
        w = E.loss_terms(s)
        assert t[f][0] == cnt
        assert np.allclose(t[f][1:], [w["g2"], w["g4"], w["r2"], w["total"]], rtol=1e-6, atol=0), f
    w = E.loss_terms(total)
    assert np.allclose(t["overall"][1:], [w["g2"], w["g4"], w["r2"], w["total"]], rtol=1e-6, atol=0)
    assert t == run("--batch", "2", *files)
    assert t == run("--window", str(max(counts)), *files)
    # --window 5 equals the 5-frame pieces as files of their own
    rec0 = E.read_records(files[0])
    pieces = []
    for a in range(0, counts[0], 5):
        p = str(tmp_path / f"piece{a}")
        rec0[a:a + 5].tofile(p)
        pieces.append(p)
    win = run("--window", "5", files[0])
    sep = run(*pieces)
    assert win[files[0]] == win["overall"] and win["overall"][1:] == sep["overall"][1:]
    assert win["overall"][0] == sep["overall"][0] == counts[0]
    assert win[files[0]][1:] != t[files[0]][1:]       # fresh windows are a different loss
