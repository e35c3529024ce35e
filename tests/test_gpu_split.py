"""The signal path without the network (pnb_analyze_* / pnb_synthesize_*, Engine.analyze / Engine.synthesize) and the
engines without a network (PNB_SIGNAL_ONLY).

A split call -- analyze, the caller's g/r, synthesize -- is the fused pnb_process_* call cut where the network sits:
with the network's own g/r in between it gives the fused call's output, taps and state bit for bit, and with the
compiled reference's g/r (tests/golden/e2e.npz) the reference's output bit for bit, with no network error mixed in.
"""
import os

import numpy as np
import pytest

from conftest import GOLDEN
from synthesis_oracle import FRAME, synthesize
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


def _flags(api, mode):
    return {"fp32": api.NN_FP32, "tensor": api.NN_TENSOR, "tensor_wide": api.NN_TENSOR | api.CONV_WIDE}[mode]


def _blobs(eng, n):
    import torch
    b = eng.export_states(list(range(n)), None)
    torch.cuda.synchronize()
    return b.cpu().numpy()


def _split(api, eng, x, where, int16):
    """analyze -> compute_rnn -> synthesize through the host forms, or through the device forms on torch buffers
    chained with no reshaping: (out [n, F*480], g/r [n, F, 68], features [n, F, 70], launches of the analysis, launches
    of the synthesis)."""
    import torch
    n, T = x.shape
    F = T // FRAME
    n0 = eng.launches
    if where == "host":
        feat = eng.analyze(x)
        n1 = eng.launches
        gr = eng.compute_rnn(feat)
        n2 = eng.launches
        out = eng.synthesize(gr, int16=int16)
        return out, gr, feat, n1 - n0, eng.launches - n2
    d_in = torch.from_numpy(np.ascontiguousarray(x)).cuda()
    d_feat = torch.full((n, F, 70), -7.0, device="cuda")
    d_gr = torch.full((n, F, 68), -7.0, device="cuda")
    d_out = torch.empty_like(d_in)
    torch.cuda.synchronize()
    eng.analyze_device(d_in.data_ptr(), T, F, d_feat.data_ptr(), F * 70, int16=int16)
    n1 = eng.launches
    eng.compute_rnn_device(api.RNN_FEATURES, d_feat.data_ptr(), F * 70, F, d_gr.data_ptr(), F * 68)
    n2 = eng.launches
    eng.synthesize_device(d_gr.data_ptr(), F * 68, F, d_out.data_ptr(), T, int16=int16)
    eng.check()
    return d_out.cpu().numpy(), d_gr.cpu().numpy(), d_feat.cpu().numpy(), n1 - n0, eng.launches - n2


def _fused_device(eng, x, int16):
    import torch
    n, T = x.shape
    F = T // FRAME
    d_in = torch.from_numpy(np.ascontiguousarray(x)).cuda()
    d_out = torch.empty_like(d_in)
    d_gr = torch.empty((F, n, 68), device="cuda")
    torch.cuda.synchronize()
    eng.process_device(d_in.data_ptr(), T, d_out.data_ptr(), T, F, d_gr=d_gr.data_ptr(), int16=int16)
    eng.check()
    return d_out.cpu().numpy(), d_gr.cpu().numpy()


@pytest.mark.parametrize("post", [False, True], ids=["plain", "postfilter"])
@pytest.mark.parametrize("mode", MODES)
def test_split_call_is_the_fused_call(api, model0, mode, post):
    """analyze -> compute_rnn(features) -> synthesize(g/r) against a twin engine's pnb_process_* on the same input, on
    an active range below n_streams, in calls of unequal length through every host and device form (f32 and int16):
    output, g/r, the features, g_used and network-state taps and the exported blobs are bit-identical after every call
    pair, and so are the outputs of the pnb_process_* calls that follow on both engines."""
    from percepnet_b200.synth import to_int16
    flags = _flags(api, mode) | api.KEEP_TAPS | (api.POSTFILTER if post else 0)
    S, n, FMAX = 7, 5, 9
    calls = [(9, "host", False), (4, "host", True), (7, "device", False), (3, "device", True)]
    total = sum(c[0] for c in calls)
    x = crowd(n, total + 6, seed=400)
    x16 = to_int16(x)
    fused, split = (api.Engine(S, FMAX, model0, flags) for _ in range(2))
    for e in (fused, split):
        e.set_active(n)
    t0 = 0
    for F, where, i16 in calls:
        xin = np.ascontiguousarray((x16 if i16 else x)[:, t0 * FRAME:(t0 + F) * FRAME])
        tag = f"hops {t0}..{t0 + F - 1} {where} {'int16' if i16 else 'f32'}"
        want, want_gr = fused.process(xin, want_gr=True) if where == "host" else _fused_device(fused, xin, i16)
        got, gr, feat, _, _ = _split(api, split, xin, where, i16)
        assert got.dtype == want.dtype, tag
        assert (np.array_equal(got, want) if i16 else same_bits(got, want)), tag
        assert same_bits(gr, want_gr.transpose(1, 0, 2)), tag
        assert same_bits(feat, fused.read_tap("features", F)[:, :n].transpose(1, 0, 2)), tag
        for tap in ("features", "g_used"):
            assert same_bits(split.read_tap(tap, F)[:, :n], fused.read_tap(tap, F)[:, :n]), (tag, tap)
        a, b = fused.read_nn_state(), split.read_nn_state()
        assert all(same_bits(a[k][:n], b[k][:n]) for k in a), tag
        assert np.array_equal(_blobs(split, n), _blobs(fused, n)), tag
        t0 += F
    want, _ = fused.process(np.ascontiguousarray(x[:, t0 * FRAME:]))
    got, _ = split.process(np.ascontiguousarray(x[:, t0 * FRAME:]))
    assert same_bits(got, want)
    fused.close()
    split.close()


@pytest.mark.parametrize("mode", ["fp32", "tensor"])
def test_split_call_slides_where_the_fused_call_does(api, model0, mode):
    """Ten 2-hop split calls at max_frames 2 against a twin engine's pnb_process_* calls, through every host and device
    form (f32 and int16), on an active range below n_streams.  The history line holds eight such calls, so the eighth
    moves it back to the start of the rows.  After every pair the output, g/r, features and exported blobs are
    bit-identical; the analysis issues three launches and the synthesis two plus the history move, which is whatever
    the fused call issued beyond launches_per_call."""
    from percepnet_b200.synth import to_int16
    S, n, F, calls = 5, 4, 2, 10
    x = crowd(n, (calls + 1) * F, seed=450)
    x16 = to_int16(x)
    fused, split = (api.Engine(S, F, model0, _flags(api, mode) | api.KEEP_TAPS) for _ in range(2))
    for e in (fused, split):
        e.set_active(n)
    per_call = fused.launches_per_call(F)
    slides = []
    for k in range(calls):
        where, i16 = ("host", "device")[k % 2], (k // 2) % 2 == 1
        xin = np.ascontiguousarray((x16 if i16 else x)[:, k * F * FRAME:(k + 1) * F * FRAME])
        tag = f"call {k} {where} {'int16' if i16 else 'f32'}"
        n0 = fused.launches
        want, want_gr = fused.process(xin, want_gr=True) if where == "host" else _fused_device(fused, xin, i16)
        slide = fused.launches - n0 - per_call
        got, gr, feat, n_analysis, n_synthesis = _split(api, split, xin, where, i16)
        assert (np.array_equal(got, want) if i16 else same_bits(got, want)), tag
        assert same_bits(gr, want_gr.transpose(1, 0, 2)), tag
        assert same_bits(feat, fused.read_tap("features", F)[:, :n].transpose(1, 0, 2)), tag
        assert np.array_equal(_blobs(split, n), _blobs(fused, n)), tag
        assert (n_analysis, n_synthesis) == (3, 2 + slide), tag
        if slide:
            slides.append(k)
    assert slides == [7]
    rest = np.ascontiguousarray(x[:, calls * F * FRAME:])
    assert same_bits(split.process(rest)[0], fused.process(rest)[0])
    fused.close()
    split.close()


@pytest.mark.parametrize("mode", ["fp32", "tensor"])
def test_signal_only_and_network_only_engines(api, model0, mode):
    """A PNB_SIGNAL_ONLY engine's analyze / synthesize with a PNB_NETWORK_ONLY engine's compute_rnn in between is one
    PCM engine's process, bit for bit; the signal-only blob is the PCM blob in its signal part and zero behind it, and
    a PCM blob imported into a fresh signal-only engine continues the signal path bit for bit."""
    flags = _flags(api, mode)
    S, F = 6, 8
    x = crowd(S, 4 * F, seed=410)
    pcm = api.Engine(S, F, model0, flags)
    sig = api.Engine(S, F, None, api.SIGNAL_ONLY)
    net = api.Engine(S, F, model0, flags | api.NETWORK_ONLY)
    assert sig.device_bytes < pcm.device_bytes
    assert sig.launches_per_call(F) == 5

    def step(sig_eng, k):
        xin = np.ascontiguousarray(x[:, k * F * FRAME:(k + 1) * F * FRAME])
        want, _ = pcm.process(xin)
        got = sig_eng.synthesize(net.compute_rnn(sig_eng.analyze(xin)))
        assert same_bits(got, want), k

    step(sig, 0)
    step(sig, 1)
    pb, sb = _blobs(pcm, S), _blobs(sig, S)
    assert np.array_equal(sb[:, :SIGNAL_BYTES], pb[:, :SIGNAL_BYTES])
    assert not sb[:, SIGNAL_BYTES:].any()
    import torch
    fresh = api.Engine(S, F, None, api.SIGNAL_ONLY)
    fresh.import_states(list(range(S)), torch.from_numpy(pb).cuda())
    step(fresh, 2)
    step(fresh, 3)
    for e in (pcm, sig, net, fresh):
        e.close()


def _oracle_features(oracle, model, x):
    h = oracle.create(model)
    _, _, taps = oracle.process_stream(h, x, True, taps=True)
    oracle.destroy(h)
    return np.stack([t.np("features") for t in taps])


def test_reference_gains_reproduce_the_reference(api, oracle, model0):
    """The compiled reference's own g/r (tests/golden/e2e.npz) through analyze / synthesize, no network in between: the
    CLI's int16 output with the first hop dropped, and the float output at unit and at int16 scale, exactly; the
    analysed features are the oracle's bit for bit.  The int16 analysis feeds the f32 synthesis too (the halves mix)."""
    g = np.load(os.path.join(GOLDEN, "e2e.npz"))
    x16 = g["x16"]
    F = x16.size // FRAME
    eng = api.Engine(1, F, None, api.SIGNAL_ONLY)
    eng.analyze(x16[None])
    out16 = eng.synthesize(g["cli_gr"][None], int16=True)
    assert np.array_equal(out16[0, FRAME:], g["cli_out16"])
    eng.reset()
    eng.analyze(x16[None])
    assert same_bits(eng.synthesize(g["gr_unit"][None]), g["out_unit"][None])
    for name, x in (("unit", x16.astype(np.float32) * np.float32(1 / 32768.0)), ("int16", x16.astype(np.float32))):
        eng.reset()
        feat = eng.analyze(x[None])
        assert same_bits(feat[0], _oracle_features(oracle, model0, x)), name
        out = eng.synthesize(g[f"gr_{name}"][None])
        assert same_bits(out[0], g[f"out_{name}"]), name
    eng.close()


def test_caller_gains_the_network_never_makes(api, oracle):
    """Random finite g/r and edge values (0, 1, subnormals, above 1, negative) against the synthesis restatement at the
    analysis taps, bit-identical; rows of NaN / Inf g/r complete with PNB_OK and leave their neighbours' bits alone."""
    S, F = 8, 6
    hw = oracle.tables()[0]
    x = crowd(S, 2 * F, seed=420) * np.float32(2000.0)
    rng = np.random.RandomState(421)
    edges = np.array([0.0, 1.0, 1e-40, -1e-42, 1.5, 7.0, 100.0, -0.5, -3.0, 0.25], np.float32)
    eng = api.Engine(S, F, None, api.SIGNAL_ONLY | api.KEEP_TAPS)
    mem = np.zeros((S, FRAME), np.float32)
    silent = 0
    for k in range(2):
        xin = np.ascontiguousarray(x[:, k * F * FRAME:(k + 1) * F * FRAME])
        gr = rng.rand(S, F, 68).astype(np.float32)
        gr[S // 2:] = rng.choice(edges, (S - S // 2, F, 68))
        eng.analyze(xin)
        out = eng.synthesize(gr)
        X, P, sil = eng.read_tap("X", F), eng.read_tap("P", F), eng.read_tap("pitch", F)[..., 2]
        assert same_bits(eng.read_tap("g_used", F), gr.transpose(1, 0, 2)[..., :34])
        for s in range(S):
            for t in range(F):
                want = synthesize(oracle, X[t, s], P[t, s], sil[t, s], gr[s, t, :34], gr[s, t, 34:], mem[s], hw)
                assert same_bits(out[s, t * FRAME:(t + 1) * FRAME], want), (k, s, t)
        silent += int(np.sum(sil != 0))
    eng.close()
    assert silent < 2 * F * S   # the comb filter (r) ran on some frames

    x1 = np.ascontiguousarray(x[:, :F * FRAME])
    gr = rng.rand(S, F, 68).astype(np.float32)
    bad = gr.copy()
    bad[1, 2:, 3] = np.nan
    bad[4, :, 40] = np.inf
    bad[6, 3, :34] = -np.inf
    outs = []
    for g in (gr, bad):
        eng = api.Engine(S, F, None, api.SIGNAL_ONLY)
        eng.analyze(x1)
        outs.append(eng.synthesize(g))
        eng.check()
        eng.close()
    keep = [0, 2, 3, 5, 7]
    assert same_bits(outs[1][keep], outs[0][keep])


def test_torch_interop(api):
    """analyze_device into a torch tensor, a torch op on torch's current (non-default) stream, synthesize_device on that
    stream: the features and the output of the host forms given the same g/r."""
    import torch
    S, F = 5, 7
    x = crowd(S, F, seed=430)
    dev = api.Engine(S, F, None, api.SIGNAL_ONLY)
    host = api.Engine(S, F, None, api.SIGNAL_ONLY)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        st = torch.cuda.current_stream().cuda_stream
        d_in = torch.from_numpy(x).cuda()
        d_feat = torch.empty((S, F, 70), device="cuda")
        dev.analyze_device(d_in.data_ptr(), F * FRAME, F, d_feat.data_ptr(), F * 70, stream=st)
        d_gr = torch.sigmoid(d_feat[..., :68] * 0.1).contiguous()
        d_out = torch.empty_like(d_in)
        dev.synthesize_device(d_gr.data_ptr(), F * 68, F, d_out.data_ptr(), F * FRAME, stream=st)
        feat, gr, out = d_feat.cpu().numpy(), d_gr.cpu().numpy(), d_out.cpu().numpy()
    side.synchronize()
    assert same_bits(feat, host.analyze(x))
    assert same_bits(out, host.synthesize(gr))
    dev.close()
    host.close()


def test_refusals_and_accounting(api, model0):
    """Every refusal returns PNB_ERR_ARG, launches nothing and leaves later results unchanged; pnb_reset cancels a
    pending synthesis; an analysis issues three launches and a synthesis two; the engine kinds that cannot split refuse."""
    import torch
    L = api.load_library()
    S, F = 4, 6
    x = crowd(S, 3 * F, seed=440)
    x1 = np.ascontiguousarray(x[:, :F * FRAME])
    x16 = np.zeros((S, F * FRAME), np.int16)
    feat = np.zeros((S, F, 70), np.float32)
    gr = np.full((S, F, 68), 0.5, np.float32)
    out = np.zeros((S, F * FRAME), np.float32)
    blob = np.zeros(L.pnb_state_size(), np.uint8)
    d_x, d_feat, d_gr = torch.from_numpy(x1).cuda(), torch.zeros((S, F, 70), device="cuda"), torch.zeros((S, F, 68), device="cuda")
    d_out, d_blobs = torch.zeros_like(d_x), torch.zeros((S, L.pnb_state_size()), dtype=torch.uint8, device="cuda")
    idx = np.arange(S, dtype=np.int32)
    xp, fp, gp, op = x1.ctypes.data, feat.ctypes.data, gr.ctypes.data, out.ctypes.data

    eng, twin = api.Engine(S, F, model0), api.Engine(S, F, model0)
    h = eng.h
    n0 = eng.launches
    # nothing pending, bad arguments
    assert L.pnb_synthesize_host_f32(h, gp, 68 * F, F, op, F * FRAME) == -1
    assert b"pnb_analyze_" in L.pnb_last_error()
    assert L.pnb_synthesize_device_f32(h, d_gr.data_ptr(), 68 * F, F, d_out.data_ptr(), F * FRAME, None) == -1
    for args in [(None, xp, F * FRAME, F, fp, 70 * F), (h, None, F * FRAME, F, fp, 70 * F), (h, xp, F * FRAME, F, None, 70 * F),
                 (h, xp, F * FRAME - 1, F, fp, 70 * F), (h, xp, F * FRAME, F, fp, 70 * F - 1), (h, xp, F * FRAME, 0, fp, 70 * F),
                 (h, xp, F * FRAME, F + 1, fp, 70 * (F + 1))]:
        assert L.pnb_analyze_host_f32(*args) == -1, args
    assert eng.launches == n0

    assert L.pnb_analyze_host_f32(h, xp, F * FRAME, F, fp, 70 * F) == 0
    assert eng.launches == n0 + 3
    twin.analyze(x1)
    n1 = eng.launches
    # pending: every other call and state operation is refused before anything is enqueued
    refused = {
        "analyze_host_f32": lambda: L.pnb_analyze_host_f32(h, xp, F * FRAME, F, fp, 70 * F),
        "analyze_host_i16": lambda: L.pnb_analyze_host_i16(h, x16.ctypes.data, F * FRAME, F, fp, 70 * F),
        "analyze_device_f32": lambda: L.pnb_analyze_device_f32(h, d_x.data_ptr(), F * FRAME, F, d_feat.data_ptr(), 70 * F, None),
        "synthesize_other_frames": lambda: L.pnb_synthesize_host_f32(h, gp, 68 * F, F - 1, op, F * FRAME),
        "process_host_f32": lambda: L.pnb_process_host_f32(h, xp, F * FRAME, op, F * FRAME, F, None),
        "submit_host_f32": lambda: L.pnb_submit_host_f32(h, xp, F * FRAME, op, F * FRAME, F),
        "process_device_f32": lambda: L.pnb_process_device_f32(h, d_x.data_ptr(), F * FRAME, d_out.data_ptr(), F * FRAME, F, None, None),
        "submit_device_f32": lambda: L.pnb_submit_device_f32(h, d_x.data_ptr(), F * FRAME, d_out.data_ptr(), F * FRAME, F, None),
        "set_active_streams": lambda: L.pnb_set_active_streams(h, S - 1, None),
        "reset_streams": lambda: L.pnb_reset_streams(h, idx.ctypes.data, S, None),
        "export_states": lambda: L.pnb_export_states(h, idx.ctypes.data, S, d_blobs.data_ptr(), d_blobs.stride(0), None),
        "import_states": lambda: L.pnb_import_states(h, idx.ctypes.data, S, d_blobs.data_ptr(), d_blobs.stride(0), None),
        "get_state": lambda: L.pnb_get_state(h, 0, blob.ctypes.data, blob.size),
        "set_state": lambda: L.pnb_set_state(h, 0, blob.ctypes.data, blob.size),
        "sessions_reserve": lambda: L.pnb_sessions_reserve(h, 8),
    }
    for name, call in refused.items():
        assert call() == -1, name
        assert eng.launches == n1, name
    assert eng.active == S
    # allowed while pending
    assert L.pnb_wait(h) == 0 and L.pnb_check(h, None) == 0 and L.pnb_flush(h, None) == 0
    eng.read_tap("features", F)
    assert L.pnb_synthesize_host_f32(h, gp, 68 * F, F, op, F * FRAME) == 0
    assert eng.launches == n1 + 2
    assert same_bits(out, twin.synthesize(gr))
    nxt = np.ascontiguousarray(x[:, F * FRAME:2 * F * FRAME])
    assert same_bits(eng.process(nxt)[0], twin.process(nxt)[0])
    # pnb_reset cancels the pending synthesis
    eng.analyze(x1)
    eng.reset()
    assert L.pnb_synthesize_host_f32(h, gp, 68 * F, F, op, F * FRAME) == -1
    eng.process(x1)
    # session mode
    eng.reserve_sessions(8)
    assert L.pnb_analyze_host_f32(h, xp, F * FRAME, F, fp, 70 * F) == -1
    assert b"session" in L.pnb_last_error()
    eng.close()
    twin.close()

    # engines that cannot split
    for flags, model in ((api.NETWORK_ONLY, model0), (api.TRAIN_DATA, None)):
        e = api.Engine(S, F, model, flags)
        assert L.pnb_analyze_host_f32(e.h, xp, F * FRAME, F, fp, 70 * F) == -1, flags
        assert e.launches == 0
        e.close()
    # a signal-only engine: the split calls only; no network flags, no network taps, no session pool
    for bad in (api.NN_TENSOR, api.NN_TENSOR | api.CONV_WIDE, api.TRAIN_DATA, api.TRAIN_DATA | api.TRAIN_AUDIO, api.NETWORK_ONLY):
        with pytest.raises(api.PnbError, match="SIGNAL_ONLY"):
            api.Engine(S, F, None, api.SIGNAL_ONLY | bad)
    sig = api.Engine(S, F, None, api.SIGNAL_ONLY | api.POSTFILTER | api.KEEP_TAPS)
    sh = sig.h
    rec = np.zeros((S, F, 138), np.float32)
    sums = np.zeros((S, 4), np.float64)
    for name, call in {
        "process_host_f32": lambda: L.pnb_process_host_f32(sh, xp, F * FRAME, op, F * FRAME, F, None),
        "submit_host_f32": lambda: L.pnb_submit_host_f32(sh, xp, F * FRAME, op, F * FRAME, F),
        "process_device_f32": lambda: L.pnb_process_device_f32(sh, d_x.data_ptr(), F * FRAME, d_out.data_ptr(), F * FRAME, F, None, None),
        "compute_rnn_host": lambda: L.pnb_compute_rnn_host(sh, 0, fp, 70 * F, F, gp, 68 * F),
        "score_records_host": lambda: L.pnb_score_records_host(sh, rec.ctypes.data, 138 * F, F, None, sums.ctypes.data, None, 0),
        "train_records_host": lambda: L.pnb_train_records_host(sh, x16.ctypes.data, F * FRAME, x16.ctypes.data, F * FRAME, F, rec.ctypes.data, 138 * F),
        "sessions_reserve": lambda: L.pnb_sessions_reserve(sh, 8),
    }.items():
        assert call() == -1, name
    assert sig.launches == 0
    with pytest.raises(api.PnbError, match="network state"):
        sig.read_nn_state()
    sig.analyze(x1)
    sig.synthesize(gr)
    assert sig.launches == sig.launches_per_call(F) == 5
    sig.close()


def test_enhance_gains_cli(api, tmp_path):
    """enhance --gains on the e2e input with the reference's g/r reproduces the reference CLI's output exactly, in
    single-file mode and in list mode, where a shorter file in the same batch gets the first hops of that output."""
    from percepnet_b200 import enhance
    g = np.load(os.path.join(GOLDEN, "e2e.npz"))
    x16, cli_gr, want = g["x16"], g["cli_gr"], g["cli_out16"]
    pin, gains, out = (str(tmp_path / n) for n in ("in.pcm", "gains.f32", "out.pcm"))
    x16.astype("<i2").tofile(pin)
    cli_gr.astype("<f4").tofile(gains)
    assert enhance.main(["--gains", gains, pin, out]) == 0
    assert np.array_equal(np.fromfile(out, "<i2"), want)
    short_in, short_gains = str(tmp_path / "short.pcm"), str(tmp_path / "short.f32")
    x16[:30 * FRAME].astype("<i2").tofile(short_in)
    cli_gr[:30].astype("<f4").tofile(short_gains)
    (tmp_path / "jobs.txt").write_text(f"{pin} {tmp_path / 'a.pcm'} {gains}\n{short_in} {tmp_path / 'b.pcm'} {short_gains}\n")
    assert enhance.main(["--list", str(tmp_path / "jobs.txt"), "--chunk", "16"]) == 0
    assert np.array_equal(np.fromfile(str(tmp_path / "a.pcm"), "<i2"), want)
    assert np.array_equal(np.fromfile(str(tmp_path / "b.pcm"), "<i2"), want[:29 * FRAME])
