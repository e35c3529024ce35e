"""The network alone (pnb_compute_rnn_*, Engine.compute_rnn): the batched compute_rnn on caller-supplied features or
training records, on the fp32 engine, the tensor engine and the tensor engine with PNB_CONV_WIDE.

Its results are those of the PCM path bit for bit: a fresh engine fed the features a PCM call analysed (or the records
the training-data generator wrote for the same noisy signal) ends with the same g/r and the same network state.
"""
import os

import numpy as np
import pytest

from util import crowd, device_first_hop_major, same_bits

pytestmark = pytest.mark.gpu

DOMAIN = 8.5e7
GR_RTOL = 1e-4
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


def _flags(api, mode):
    return {"fp32": api.NN_FP32, "tensor": api.NN_TENSOR, "tensor_wide": api.NN_TENSOR | api.CONV_WIDE}[mode]


def _pcm_run(api, model, flags, x, S=None, active=None):
    """One PCM call on a PNB_KEEP_TAPS engine: (features [n, F, 70], g/r [n, F, 68], network state rows [0, n))."""
    F = x.shape[1] // 480
    eng = api.Engine(S or x.shape[0], F, model, flags | api.KEEP_TAPS)
    if active:
        eng.set_active(active)
    n = eng.active
    _, gr = eng.process(x, want_gr=True)
    feats = eng.read_tap("features", F)[:, :n]
    nn = {k: v[:n] for k, v in eng.read_nn_state().items()}
    eng.close()
    return np.ascontiguousarray(feats.transpose(1, 0, 2)), np.ascontiguousarray(gr.transpose(1, 0, 2)), nn


def _rnn_run(api, model, flags, feats, S=None, active=None, calls=None):
    """A fresh engine fed `feats` ([n, F, 70|138]) through compute_rnn in calls of `calls` hops: (g/r, network state)."""
    n, F = feats.shape[0], feats.shape[1]
    calls = calls or [F]
    eng = api.Engine(S or n, max(calls), model, flags)
    if active:
        eng.set_active(active)
    parts, t0 = [], 0
    for c in calls:
        parts.append(eng.compute_rnn(np.ascontiguousarray(feats[:, t0:t0 + c])))
        t0 += c
    assert t0 == F
    nn = {k: v[:n] for k, v in eng.read_nn_state().items()}
    eng.close()
    return np.concatenate(parts, axis=1), nn


def _same_state(a, b):
    return all(same_bits(a[k], b[k]) for k in a)


def _device_run(api, eng, x):
    """compute_rnn_device on torch tensors: (g/r [n, F, 68] as computed, pnb_wait's return code)."""
    import torch
    n, F, W = x.shape
    d_in = torch.from_numpy(np.ascontiguousarray(x, np.float32)).cuda()
    d_gr = torch.full((n, F, 68), -7.0, dtype=torch.float32, device="cuda")
    torch.cuda.synchronize()
    eng.compute_rnn_device(api.RNN_FEATURES if W == 70 else api.RNN_RECORDS, d_in.data_ptr(), F * W, F, d_gr.data_ptr(),
                           F * 68)
    rc = eng.L.pnb_wait(eng.h)
    out = d_gr.cpu().numpy()
    return out, rc


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("streams", ["3", "129", "first_hop_major", "200_of_300"])
def test_same_bits_as_the_pcm_path(api, model0, mode, streams):
    """A fresh engine fed the features of a PCM call gives that call's g/r and network state, bit for bit; the sizes run
    the tensor chain in both unit orders, and on an active range."""
    flags = _flags(api, mode)
    F = 8
    S, active = {"3": (3, None), "129": (129, None), "first_hop_major": (device_first_hop_major(), None),
                 "200_of_300": (300, 200)}[streams]
    n = active or S
    x = crowd(n, F, seed=310 + n)
    feats, gr, nn = _pcm_run(api, model0, flags, x, S, active)
    got, nn2 = _rnn_run(api, model0, flags, feats, S, active)
    assert same_bits(got, gr)
    assert _same_state(nn2, nn)


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("div", [1, 64], ids=["full_scale", "quiet"])
def test_records_end_to_end(api, model0, mode, div):
    """Records of pnb_train_records_* through compute_rnn (records format, scaled x30 on the device) give the g/r of a
    PCM engine fed the noisy signal as int16-valued floats (NORM_RATIO 1, denoise.cpp:41), bit for bit; a tensor engine
    that reports PNB_ERR_DOMAIN on one reports it on the other."""
    from percepnet_b200.synth import synth_pairs
    flags = _flags(api, mode)
    N, F = 6, 24
    clean, noisy = synth_pairs(N, F, seed=321)
    clean, noisy = (clean // div).astype(np.int16), (noisy // div).astype(np.int16)
    te = api.Engine(2 * N, F, None, api.TRAIN_DATA)
    rec = te.train_records(clean, noisy)
    te.close()
    results = []
    for run in ("pcm", "records"):
        try:
            if run == "pcm":
                eng = api.Engine(N, F, model0, flags)
                _, gr = eng.process(noisy.astype(np.float32), want_gr=True)
                results.append(np.ascontiguousarray(gr.transpose(1, 0, 2)))
            else:
                eng = api.Engine(N, F, model0, flags)
                results.append(eng.compute_rnn(rec))
        except api.PnbError as ex:
            assert "(-5)" in str(ex), ex
            results.append("domain")
        eng.close()
    if isinstance(results[0], str) or isinstance(results[1], str):
        assert results[0] == results[1] == "domain"
        assert mode != "fp32"
    else:
        assert same_bits(results[1], results[0])


@pytest.mark.parametrize("mode", MODES)
def test_grouping_of_hops_into_calls(api, model0, mode):
    """40 hops as one call, as 33 + 7 (across the fp32 network's 32-hop chunk) and as 40 one-hop calls: same bits."""
    flags = _flags(api, mode)
    S, F = 37, 40
    feats, _, _ = _pcm_run(api, model0, flags, crowd(S, F, seed=330))
    one, nn1 = _rnn_run(api, model0, flags, feats)
    for calls in ([33, 7], [1] * 40):
        got, nn = _rnn_run(api, model0, flags, feats, calls=calls)
        assert same_bits(got, one), calls[:2]
        assert _same_state(nn, nn1), calls[:2]


@pytest.mark.parametrize("mode", MODES)
def test_garbage_rows_leave_their_neighbours_alone(api, model0, mode):
    """NaN, Inf and 1e30 features in some rows leave every other row's g/r bit-identical (the tensor engine may report
    PNB_ERR_DOMAIN for them; the other rows are still computed)."""
    flags = _flags(api, mode)
    S, F = 9, 12
    feats, _, _ = _pcm_run(api, model0, flags, crowd(S, F, seed=340))
    bad = feats.copy()
    bad[1, 3:, 5] = np.nan
    bad[4, 6, :] = np.inf
    bad[7, 2:, 68] = 1e30
    eng = api.Engine(S, F, model0, flags)
    clean, rc0 = _device_run(api, eng, feats)
    assert rc0 == 0
    eng.reset()
    dirty, _ = _device_run(api, eng, bad)
    eng.close()
    keep = [0, 2, 3, 5, 6, 8]
    assert same_bits(dirty[keep], clean[keep])


@pytest.mark.parametrize("mode", MODES)
def test_feature_call_between_pcm_calls(api, model0, mode):
    """PCM call, feature call, export: the signal part of the blob is that of the export before the feature call, its
    network part that of an engine that got the PCM call's features and then the same feature call; a PCM call follows."""
    import torch
    flags = _flags(api, mode)
    S, F = 5, 6
    x = crowd(S, 3 * F, seed=350)
    fx, _, _ = _pcm_run(api, model0, flags, crowd(S, F, seed=351))   # the features of the feature call
    idx = list(range(S))
    eng = api.Engine(S, F, model0, flags | api.KEEP_TAPS)
    eng.process(x[:, :F * 480])
    f1 = np.ascontiguousarray(eng.read_tap("features", F).transpose(1, 0, 2))
    before = eng.export_states(idx, None)
    eng.compute_rnn(fx)
    after = eng.export_states(idx, None)
    torch.cuda.synchronize()
    before, after = before.cpu().numpy(), after.cpu().numpy()
    assert np.array_equal(after[:, :SIGNAL_BYTES], before[:, :SIGNAL_BYTES])
    other = api.Engine(S, F, model0, flags)
    other.compute_rnn(f1)
    other.compute_rnn(fx)
    want = other.export_states(idx, None)
    torch.cuda.synchronize()
    assert np.array_equal(after[:, SIGNAL_BYTES:], want.cpu().numpy()[:, SIGNAL_BYTES:])
    other.close()
    out, gr = eng.process(x[:, F * 480:2 * F * 480], want_gr=True)
    eng.check()
    assert np.isfinite(out).all() and np.isfinite(gr).all()
    eng.close()


@pytest.mark.parametrize("mode", ["fp32", "tensor_wide"])
@pytest.mark.parametrize("dist", ["uniform", "loguniform"])
def test_features_the_dsp_never_makes(api, oracle, model0, mode, dist):
    """Uniform features and log-uniform ones up to 1e3: g/r within 1e-4 relative of the double-precision network."""
    flags = _flags(api, mode)
    S, F = 8, 10
    rng = np.random.RandomState(360)
    if dist == "uniform":
        feats = rng.rand(S, F, 70).astype(np.float32)
    else:
        feats = (10.0 ** rng.uniform(-4, 3, (S, F, 70))).astype(np.float32)
    truth, mp = np.empty((S, F, 68)), np.empty(S)
    for s in range(S):
        g, r, m = oracle.rnn_f64(model0, feats[s])
        truth[s, :, :34], truth[s, :, 34:], mp[s] = g, r, m.max()
    print(f"{dist}: max |pre-activation| {mp.max():.3g}")
    assert (mp < DOMAIN).all()
    eng = api.Engine(S, F, model0, flags)
    got = eng.compute_rnn(feats)
    eng.close()
    rel = (np.abs(got - truth) / np.maximum(np.abs(truth), 1e-6)).max()
    print(f"{mode} {dist}: max relative distance to float64 {rel:.3e}")
    assert rel < GR_RTOL


def test_tensor_engine_reports_features_past_the_domain(api, oracle, model0):
    """Features that drive conv2 past 8.5e7: the tensor engine returns PNB_ERR_DOMAIN (pnb_wait after the device form,
    the host form itself) instead of plausible numbers; the fp32 engine computes what the reference computes."""
    S, F = 4, 6
    feats = np.full((S, F, 70), 1e10, np.float32)
    feats[:, :, 68:] = 1.0
    _, _, m = oracle.rnn_f64(model0, feats[0])
    assert m.max() >= DOMAIN
    for flags in (api.NN_TENSOR, api.NN_TENSOR | api.CONV_WIDE):
        eng = api.Engine(S, F, model0, flags)
        _, rc = _device_run(api, eng, feats)
        assert rc == -5, eng.L.pnb_last_error()
        eng.reset()
        with pytest.raises(api.PnbError, match="-5"):
            eng.compute_rnn(feats)
        eng.close()
    eng = api.Engine(S, F, model0, api.NN_FP32)
    eng.compute_rnn(feats)
    eng.check()
    eng.close()


@pytest.mark.parametrize("mode", MODES)
def test_refusals(api, model0, mode):
    """Every refused call returns its code and launches nothing; an accepted call adds the network's launches + 2."""
    import torch
    flags = _flags(api, mode)
    S, F = 4, 8
    eng = api.Engine(S, F, model0, flags)
    L, h = eng.L, eng.h
    x = np.zeros((S, F, 138), np.float32)
    gr = np.zeros((S, F, 68), np.float32)
    d_x = torch.zeros((S, F, 138), device="cuda")
    d_gr = torch.zeros((S, F, 68), device="cuda")
    xp, gp, dxp, dgp = x.ctypes.data, gr.ctypes.data, d_x.data_ptr(), d_gr.data_ptr()
    before = eng.launches
    refused = [
        (None, 0, xp, 70 * F, F, gp, 68 * F),          # engine NULL
        (h, 0, None, 70 * F, F, gp, 68 * F),           # input NULL
        (h, 0, xp, 70 * F, F, None, 68 * F),           # output NULL
        (h, 2, xp, 138 * F, F, gp, 68 * F),            # format
        (h, -1, xp, 138 * F, F, gp, 68 * F),
        (h, 0, xp, 70 * F, 0, gp, 68 * F),             # n_frames outside [1, max_frames]
        (h, 0, xp, 70 * F, F + 1, gp, 68 * F),
        (h, 0, xp, 70 * F - 1, F, gp, 68 * F),         # short strides
        (h, 1, xp, 70 * F, F, gp, 68 * F),             # records need 138 per hop
        (h, 0, xp, 70 * F, F, gp, 68 * F - 1),
    ]
    for args in refused:
        assert L.pnb_compute_rnn_host(*args) == -1, args
        d = tuple(dxp if a == xp else dgp if a == gp else a for a in args)
        assert L.pnb_compute_rnn_device(*d, None) == -1, args
    assert eng.launches == before
    # accepted, both forms: the network's launches (a PCM call's without stage_in, analysis and synthesis) + 2
    per = eng.launches_per_call(F) - 3 + 2
    assert L.pnb_compute_rnn_host(h, 0, xp, 138 * F, F, gp, 68 * F) == 0
    assert eng.launches == before + per
    assert L.pnb_compute_rnn_device(h, 1, dxp, 138 * F, F, dgp, 68 * F, None) == 0
    assert L.pnb_wait(h) == 0
    assert eng.launches == before + 2 * per
    # session mode: refused like the other slot calls
    eng.reserve_sessions(8)
    n0 = eng.launches
    assert L.pnb_compute_rnn_host(h, 0, xp, 70 * F, F, gp, 68 * F) == -1
    assert b"session" in L.pnb_last_error()
    assert eng.launches == n0
    eng.close()
    # a training-data engine
    te = api.Engine(4, F, None, api.TRAIN_DATA)
    assert te.L.pnb_compute_rnn_host(te.h, 0, xp, 70 * F, F, gp, 68 * F) == -1
    assert te.L.pnb_compute_rnn_device(te.h, 0, dxp, 70 * F, F, dgp, 68 * F, None) == -1
    assert te.launches == 0
    te.close()


@pytest.mark.parametrize("mode", MODES)
def test_eval_records_cli(api, model0, mode, tmp_path, capsys):
    """gen_features on synthetic pairs, then eval_records with --pred-dir: the predictions are Engine.compute_rnn of the
    same records, and a file scored alone equals the same file inside a batch with longer files."""
    from percepnet_b200 import eval_records, gen_features
    from percepnet_b200.synth import synth_pairs
    flags = _flags(api, mode)
    counts = [30, 17, 9]
    clean, noisy = synth_pairs(3, max(counts), seed=370)
    clean, noisy = (clean // 64).astype(np.int16), (noisy // 64).astype(np.int16)   # inside the tensor path's domain
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
    (tmp_path / "files.txt").write_text("".join(f + "\n" for f in files))
    extra = {"fp32": [], "tensor": ["--tensor"], "tensor_wide": ["--tensor", "--conv-wide"]}[mode]
    pd = tmp_path / "pred"
    assert eval_records.main(["--model", blob, "--list", str(tmp_path / "files.txt"), "--chunk", "8",
                              "--pred-dir", str(pd), *extra]) == 0
    printed = capsys.readouterr().out
    assert "overall" in printed
    for f, cnt in zip(files, counts):
        rec = eval_records.read_records(f)
        assert rec.shape == (cnt, 138)
        pred = np.fromfile(str(pd / (os.path.basename(f) + ".pred.f32")), np.float32).reshape(cnt, 68)
        eng = api.Engine(1, cnt, model0, flags)
        want = eng.compute_rnn(rec[None])[0]
        eng.close()
        assert same_bits(pred, want), f
    pd2 = tmp_path / "alone"
    assert eval_records.main(["--model", blob, files[2], "--pred-dir", str(pd2), *extra]) == 0
    alone = np.fromfile(str(pd2 / (os.path.basename(files[2]) + ".pred.f32")), np.float32)
    inside = np.fromfile(str(pd / (os.path.basename(files[2]) + ".pred.f32")), np.float32)
    assert same_bits(alone, inside)
