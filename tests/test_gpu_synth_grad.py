"""The synthesis's gradient on the GPU (include/pnb_synth_grad.h, percepnet_b200/torch_signal.py).

The exported operands are the synthesis's own: the float32 synthesis restated on them (tests/synthesis_oracle.py) with
the engine's overlap-add memory reproduces the engine's output bit for bit over consecutive calls.  The backward is
checked against the float64 restatement's autograd (tests/synth_grad_oracle.py) at the same operands and g/r, the torch
path against the engine calls it makes, the lag against the header's, and a waveform loss end to end.
"""
import numpy as np
import pytest

import synth_grad_oracle as SG
from synthesis_oracle import FRAME, post_filter, sine_rounded, synthesize
from util import same_bits

pytestmark = pytest.mark.gpu

OPS = SG.OPS
SYNTH_OFFSET = 21128   # offsetof(StreamState, synth): the overlap-add memory in a pnb_get_state blob
GRAD_BAR = 1e-6        # worst |dgr - dgr64| on a row over that row's largest float64 component


@pytest.fixture(scope="module")
def api():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device")
    from percepnet_b200 import api
    api.load_library()
    return api


@pytest.fixture(scope="module")
def tab(oracle):
    return SG.Tables(oracle)


def _pcm(n, T, seed):
    """Rows of synthetic speech plus noise: int16-scale floats (the pitch filter runs), a unit-scale row (every hop
    silent) and a row that switches from unit to int16 scale halfway (both)."""
    from percepnet_b200.synth import synth_pcm
    x = synth_pcm(n, T, seed=seed, scale=32768.0)
    if n > 2:
        x[2] /= 32768.0
    if n > 3:
        x[3, :T // 2 * FRAME] /= 32768.0
    return np.ascontiguousarray(x)


def _export(eng, n, F, stride):
    import torch
    ops = torch.full((n, stride), float("nan"), device="cuda")
    eng.synthesis_operands_device(ops.data_ptr(), stride)
    eng.check()
    return ops


@pytest.mark.parametrize("post", [False, True], ids=["plain", "postfilter"])
@pytest.mark.parametrize("mode", ["fp32", "tensor", "signal"])
def test_operands_are_the_synthesis_own(api, oracle, model0, mode, post):
    """Three consecutive calls of 4, 3 and 6 hops (the first five hops of each read ring slots of the call before):
    the restated float32 synthesis on the exported operands, from the overlap-add memory in the engine's state blob,
    gives the engine's output bit for bit; the silence flags are PNB_TAP_PITCH[2]; the padding is 0."""
    S, Fmax, calls = 4, 6, (4, 3, 6)
    flags = {"fp32": api.NN_FP32, "tensor": api.NN_TENSOR, "signal": api.SIGNAL_ONLY}[mode] | api.KEEP_TAPS
    flags |= api.POSTFILTER if post else 0
    eng = api.Engine(S, Fmax, None if mode == "signal" else model0, flags)
    x = _pcm(S, sum(calls), seed=610)
    rng = np.random.RandomState(611)
    hw, _ = oracle.tables()
    t0, silent = 0, 0
    for F in calls:
        mems = [np.frombuffer(eng.get_state(s), np.float32, FRAME, SYNTH_OFFSET).copy() for s in range(S)]
        eng.analyze(np.ascontiguousarray(x[:, t0 * FRAME:(t0 + F) * FRAME]))
        ops = _export(eng, S, F, F * OPS).cpu().numpy().reshape(S, F, OPS)
        pitch = eng.read_tap("pitch", F)
        gr = rng.rand(S, F, 68).astype(np.float32)
        gr[0, 0] = 1.0
        gr[1, -1, :34] = 0.0
        out = eng.synthesize(gr)
        assert np.array_equal(ops[..., 1634], (pitch[:, :, 2].T != 0).astype(np.float32))
        assert np.all(ops[..., 1635] == 0)
        silent += int(ops[..., 1634].sum())
        for s in range(S):
            mem = mems[s]
            for t in range(F):
                o = ops[s, t]
                g = post_filter(gr[s, t, :34], o[1600:1634], sine_rounded) if post else gr[s, t, :34]
                want = synthesize(oracle, o[:800], o[800:1600], bool(o[1634]), g, gr[s, t, 34:], mem, hw)
                assert same_bits(want, out[s, (t * FRAME):(t + 1) * FRAME]), (F, s, t)
        t0 += F
    assert 0 < silent < S * sum(calls)
    eng.close()


def _backward(api, ops, ops_stride, gr, dout, post, pads=(0, 0, 0)):
    """pnb_synthesis_backward_device of host g/r and dL/d(out) on the device operands, every row at a padded stride;
    returns dgr [n, F, 68] and the padding of its rows (which must stay as filled)."""
    import torch
    n, F = gr.shape[:2]
    gs, ds, dgs = F * 68 + pads[0], F * FRAME + pads[1], F * 68 + pads[2]
    d_gr = torch.zeros((n, gs), device="cuda")
    d_gr[:, :F * 68] = torch.from_numpy(gr.reshape(n, -1)).cuda()
    d_dout = torch.zeros((n, ds), device="cuda")
    d_dout[:, :F * FRAME] = torch.from_numpy(dout.reshape(n, -1)).cuda()
    d_dgr = torch.full((n, dgs), -7.0, device="cuda")
    api.synthesis_backward_device(ops.data_ptr(), ops_stride, d_gr.data_ptr(), gs, n, F, post, d_dout.data_ptr(), ds,
                                  d_dgr.data_ptr(), dgs)
    torch.cuda.synchronize()
    h = d_dgr.cpu().numpy()
    return h[:, :F * 68].reshape(n, F, 68), h[:, F * 68:]


@pytest.mark.parametrize("post", [False, True], ids=["plain", "postfilter"])
def test_gradient_against_float64(api, tab, post):
    """dL/d(g, r) against the float64 restatement's autograd at the same operands and g/r: four active rows of a
    five-row engine (int16-scale speech plus noise, a unit-scale row that is silent throughout, a row that is both),
    calls of max and of one hop, random g/r and g/r at 0 and 1, an all-zero-g hop, padded strides for every array.
    Silent hops get dr exactly 0; under the post-filter the all-zero-g hop gets dg exactly 0."""
    S, n, Fmax = 5, 4, 12
    eng = api.Engine(S, Fmax, None, api.SIGNAL_ONLY | (api.POSTFILTER if post else 0))
    eng.set_active(n)
    x = _pcm(n, Fmax + 1, seed=620)
    rng = np.random.RandomState(621)
    worst, t0 = 0.0, 0
    for F in (Fmax, 1):
        eng.analyze(np.ascontiguousarray(x[:, t0 * FRAME:(t0 + F) * FRAME]))
        ops_stride = F * OPS + 7
        d_ops = _export(eng, n, F, ops_stride)
        gr = rng.rand(n, F, 68).astype(np.float32)
        gr[0, -1, :34] = 0.0                      # every g zero
        gr[1, -1] = 1.0
        gr[3, 0] = 0.0
        eng.synthesize(gr)
        dout = (rng.randn(n, F * FRAME) * 100).astype(np.float32)
        dgr, pad = _backward(api, d_ops, ops_stride, gr, dout, post, pads=(5, 3, 9))
        assert np.all(pad == -7.0)
        ops = d_ops[:, :F * OPS].cpu().numpy().reshape(n, F, OPS)
        ref = SG.grad(tab, ops.astype(np.float64), gr.astype(np.float64), dout.astype(np.float64), post).numpy()
        sil = ops[..., 1634] != 0
        assert np.all(dgr[..., 34:][sil] == 0)
        if F == Fmax:
            assert sil[2].all() and not sil[0].all() and sil[3].any() and not sil[3].all(), sil
        if post:
            assert np.all(dgr[0, -1, :34] == 0)
        for i in range(n):
            if not np.any(ref[i]):      # one zero-g hop under the post-filter: no gain, so no gradient at all
                assert np.all(dgr[i] == 0), (F, i)
                continue
            err = np.abs(dgr[i] - ref[i]).max() / np.abs(ref[i]).max()
            worst = max(worst, err)
            assert err < GRAD_BAR, (F, i, err)
        t0 += F
    print(f"post={post}: worst row error {worst:.2e}")
    eng.close()


def test_signal_path_autograd(api):
    """SignalPath against a twin signal-only engine driven through Engine.analyze_device / synthesize_device on the
    same PCM and g/r: features and output bit for bit; torch.autograd.grad through synthesize is the direct backward
    call bit for bit, and unchanged when taken after the next window's analyze; under autocast g/r are cast to float32."""
    import torch
    from percepnet_b200.torch_signal import OPS_FLOATS, SignalPath
    B, T = 3, 10
    sp = SignalPath(B, T, postfilter=True, device="cuda")
    twin = api.Engine(B, T, None, api.SIGNAL_ONLY | api.POSTFILTER)
    x = torch.from_numpy(_pcm(B, 3 * T, seed=630)).cuda()
    gen = torch.Generator(device="cuda").manual_seed(631)
    held = None
    for w in range(3):
        xw = x[:, w * T * FRAME:(w + 1) * T * FRAME]
        feat, ops = sp.analyze(xw)
        xc = xw.contiguous()
        tf = torch.empty((B, T, 70), device="cuda")
        twin.analyze_device(xc.data_ptr(), T * FRAME, T, tf.data_ptr(), T * 70)
        torch.cuda.synchronize()
        assert torch.equal(feat, tf)
        if held is not None:      # the last window's gradient after this window's analyze
            out0, gr0, dout0, g0 = held
            (again,) = torch.autograd.grad(out0, gr0, dout0)
            assert torch.equal(again, g0)
        gr = torch.rand((B, T, 68), device="cuda", generator=gen)
        if w == 2:
            with torch.autocast("cuda", dtype=torch.bfloat16):
                grh = gr.to(torch.bfloat16).requires_grad_(True)
                out = sp.synthesize(grh, ops)
            gr_used, leaf = grh.float(), grh
        else:
            leaf = gr.requires_grad_(True)
            out = sp.synthesize(leaf, ops)
            gr_used = gr
        gu = gr_used.detach().contiguous()
        to = torch.empty((B, T * FRAME), device="cuda")
        twin.synthesize_device(gu.data_ptr(), T * 68, T, to.data_ptr(), T * FRAME)
        torch.cuda.synchronize()
        assert out.dtype == torch.float32 and torch.equal(out, to), w
        dout = torch.randn((B, T * FRAME), device="cuda", generator=gen)
        (g1,) = torch.autograd.grad(out, leaf, dout, retain_graph=True)
        direct = torch.empty((B, T, 68), device="cuda")
        api.synthesis_backward_device(ops.data_ptr(), T * OPS_FLOATS, gu.data_ptr(), T * 68, B, T, True,
                                      dout.data_ptr(), T * FRAME, direct.data_ptr(), T * 68)
        torch.cuda.synchronize()
        assert torch.equal(g1.float(), direct.to(g1.dtype).float()), w
        held = (out, leaf, dout, g1)
    sp.close()
    twin.close()


def test_lag_is_the_headers(api):
    """With g = 1 and r = 0 the output is the input delayed by PNB_LATENCY_FRAMES hops, 2880 samples, on a
    band-limited input (bins from 400 up never reach the output); one hop more or less does not fit."""
    import torch
    from percepnet_b200.torch_signal import LATENCY_SAMPLES, SignalPath
    T = 24
    rng = np.random.RandomState(640)
    spec = np.fft.rfft(rng.randn(2, T * FRAME), axis=1)
    spec[:, np.fft.rfftfreq(T * FRAME, 1 / 48000.0) > 15000.0] = 0
    x = (np.fft.irfft(spec, T * FRAME, axis=1) * 3000).astype(np.float32)
    sp = SignalPath(2, T)
    _, ops = sp.analyze(torch.from_numpy(x).cuda())
    gr = torch.zeros((2, T, 68), device="cuda")
    gr[..., :34] = 1.0
    out = sp.synthesize(gr, ops).cpu().numpy()
    scale = np.abs(x).max()
    for lag in (LATENCY_SAMPLES - FRAME, LATENCY_SAMPLES, LATENCY_SAMPLES + FRAME):
        err = np.abs(out[:, lag + FRAME:] - x[:, FRAME:x.shape[1] - lag]).max() / scale
        print(f"lag {lag}: max error / max |x| = {err:.2e}")
        assert (err < 1e-5) == (lag == LATENCY_SAMPLES == 2880), (lag, err)
    sp.close()


def test_waveform_loss_trains_percepnet(api):
    """PercepNet between the analysis and the synthesis, an L1 loss on the output against the clean signal delayed by
    the lag, on fixed-seed synthetic pairs: every parameter gets a finite gradient, and Adam steps lower the loss."""
    import torch
    from percepnet_b200.synth import synth_pairs
    from percepnet_b200.torch_module import PercepNet
    from percepnet_b200.torch_signal import LATENCY_SAMPLES as LAG, SignalPath
    torch.manual_seed(650)
    B, T = 4, 40
    clean, noisy = synth_pairs(B, T, seed=651)
    noisy = torch.from_numpy(noisy.astype(np.float32)).cuda()      # int16-scale floats
    clean = torch.from_numpy(clean.astype(np.float32)).cuda()
    net = PercepNet().cuda()
    sp = SignalPath(B, T, device="cuda")
    opt = torch.optim.Adam(net.parameters(), lr=1e-3)
    losses = []
    for step in range(12):
        sp.reset()
        feat, ops = sp.analyze(noisy)
        out = sp.synthesize(net(feat), ops)
        loss = (out[:, LAG:] - clean[:, :-LAG]).abs().mean() / 1000.0
        opt.zero_grad()
        loss.backward()
        if step == 0:
            for name, p in net.named_parameters():
                assert p.grad is not None and torch.isfinite(p.grad).all(), name
            assert any(p.grad.abs().max() > 0 for p in net.parameters())
        opt.step()
        losses.append(float(loss.detach()))
    print("losses:", " ".join(f"{v:.4f}" for v in losses))
    assert losses[-1] < losses[0]
    sp.close()
    net.close()


def test_refusals_and_accounting(api, model0):
    """Every refusal returns PNB_ERR_ARG before anything is enqueued; the export issues one counted launch and leaves
    the synthesis pending and its output unchanged."""
    import torch
    L = api.load_library()
    S, F = 3, 4
    x = _pcm(S, 2 * F, seed=660)
    x1 = np.ascontiguousarray(x[:, :F * FRAME])
    gr = np.full((S, F, 68), 0.5, np.float32)
    ops = torch.zeros((S, F * OPS), device="cuda")
    op = ops.data_ptr()
    eng, twin = api.Engine(S, F, None, api.SIGNAL_ONLY), api.Engine(S, F, None, api.SIGNAL_ONLY)
    h = eng.h
    n0 = eng.launches
    assert L.pnb_synthesis_operands_device(h, op, F * OPS, None) == -1       # nothing pending
    assert b"pnb_analyze_" in L.pnb_last_error()
    eng.analyze(x1)
    twin.analyze(x1)
    n1 = eng.launches
    assert n1 == n0 + 3
    for args in [(None, op, F * OPS, None), (h, None, F * OPS, None), (h, op, F * OPS - 1, None)]:
        assert L.pnb_synthesis_operands_device(*args) == -1, args
    assert eng.launches == n1
    assert L.pnb_synthesis_operands_device(h, op, F * OPS, None) == 0
    assert eng.launches == n1 + 1
    assert L.pnb_synthesis_operands_device(h, op, F * OPS + 3, None) == 0   # still pending: again
    assert eng.launches == n1 + 2
    assert same_bits(eng.synthesize(gr), twin.synthesize(gr))
    assert L.pnb_synthesis_operands_device(h, op, F * OPS, None) == -1       # the synthesis took it
    eng.close()
    twin.close()

    # a PCM engine in session mode, with a session split pending
    ses = api.Engine(S, F, model0)
    ses.reserve_sessions(8)
    ses.analyze_sessions([0, 1, 2], x1)
    assert L.pnb_synthesis_operands_device(ses.h, op, F * OPS, None) == -1
    assert b"session" in L.pnb_last_error()
    ses.close()
    # the engines without a synthesis
    for flags, model in ((api.NETWORK_ONLY, model0), (api.TRAIN_NETWORK, model0), (api.TRAIN_DATA, None)):
        e = api.Engine(2 * S if flags == api.TRAIN_DATA else S, F, model, flags)
        assert L.pnb_synthesis_operands_device(e.h, op, F * OPS, None) == -1, flags
        assert e.launches == 0
        e.close()

    # the backward, which needs no engine
    d_gr = torch.full((S, F * 68), 0.5, device="cuda")
    d_dout = torch.ones((S, F * FRAME), device="cuda")
    d_dgr = torch.full((S, F * 68), -7.0, device="cuda")
    good = [op, F * OPS, d_gr.data_ptr(), F * 68, S, F, 0, d_dout.data_ptr(), F * FRAME, d_dgr.data_ptr(), F * 68, None]
    bad = {0: None, 2: None, 7: None, 9: None, 1: F * OPS - 1, 3: F * 68 - 1, 8: F * FRAME - 1, 10: F * 68 - 1,
           4: 0, 5: 0, 6: 2}
    for k, v in bad.items():
        args = list(good)
        args[k] = v
        assert L.pnb_synthesis_backward_device(*args) == -1, k
    args = list(good)
    args[6] = -1
    assert L.pnb_synthesis_backward_device(*args) == -1
    torch.cuda.synchronize()
    assert torch.all(d_dgr == -7.0)
    assert L.pnb_synthesis_backward_device(*good) == 0
    torch.cuda.synchronize()
    assert torch.isfinite(d_dgr).all()
