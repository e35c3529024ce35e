"""torch_module.PercepNet on the GPU: the bits of the trainer's forward and backward halves against pnb_train_grad_*
and ATen, gradients of torch losses against float64 autograd of the torch restatement (train_oracle) at the module's
own weights, stream order and determinism, the recompute of a forward whose engine moved on, launch counts, refusals,
non-finite gradients, and rnn_train.py's training step closing the loop.  The halves' bits depend on the call alone
(active rows of a larger engine, padded strides, NULL weights or gradient), their seed is ATen's at saturated outputs and
non-finite or subnormal dL/d(out), and the module gives the plain step's bits for autocast, strided views, expanded or
partial dL/d(out), no dL/dx and frozen parameters."""

import numpy as np
import pytest
import torch

from percepnet_b200 import api, torch_module as tm
from percepnet_b200.eval_records import loss_terms
from percepnet_b200.weights import N_PARAMS, pack_state_dict, synth_state_dict
import train_oracle as O
from test_gpu_train import LOWER, generator_records, moderate_records, trainer, windows

pytestmark = pytest.mark.gpu


def module(sd):
    m = tm.PercepNet()
    m.load_state_dict({k: torch.from_numpy(np.asarray(v, np.float32)) for k, v in sd.items()})
    return m.cuda()


def feats(rec):
    return torch.from_numpy(O.features(rec)).cuda()


def custom_loss(out, y):
    return O.loss(out, y)


def arbitrary_loss(seed):
    """A random weighting of out plus a squared error against random targets (fixed per seed, any dtype)."""
    def f(out, y):
        g = torch.Generator().manual_seed(seed)
        w = torch.rand(out.shape, generator=g, dtype=torch.float64).to(out)
        tgt = torch.rand(out.shape, generator=g, dtype=torch.float64).to(out)
        return (out * w).mean() + ((out - tgt) ** 2).mean()
    return f


def step(m, x, y, loss_fn, want_dx=True):
    """zero_grad, forward, loss, backward: (out, loss, {name: grad} of the parameters that require it, dx).  x keeps
    its dtype and strides."""
    m.zero_grad(set_to_none=True)
    x = x.detach().requires_grad_(want_dx)
    out = m(x)
    L = loss_fn(out, y)
    L.backward()
    return out.detach(), float(L.detach()), \
        {k: p.grad.detach().clone() for k, p in m.named_parameters() if p.requires_grad}, \
        (x.grad.detach().clone() if want_dx else None)


def float64_truth(sd, x, y, loss_fn):
    ref = O.model(sd, torch.float64, "cuda")
    x64 = x.double().clone().requires_grad_(True)
    out = ref(x64)
    L = loss_fn(out, y.double())
    L.backward()
    return out.detach(), float(L.detach()), {k: p.grad.detach() for k, p in ref.named_parameters()}, x64.grad.detach()


def errors(g, g64):
    d = g.double() - g64
    return (float(d.norm() / max(float(g64.norm()), 1e-300)), float(d.abs().max() / max(float(g64.abs().max()), 1e-300)))


def check(sd, rec, loss_fn, label, lower=True):
    """Output within 1e-5 and every parameter gradient and dL/dx within |g - g64| / |g64| <= 1e-4 and
    max|g - g64| <= 1e-3 max|g64|; with lower=False the 24 tensors above fc, conv1 and conv2 only, the rest printed."""
    m = module(sd)
    x, y = feats(rec), torch.from_numpy(np.ascontiguousarray(rec[..., 70:])).cuda()
    out, L, g, dx = step(m, x, y, loss_fn)
    out64, L64, g64, dx64 = float64_truth(sd, x, y, loss_fn)
    m.close()
    dout = float((out.double() - out64).abs().max())
    err = {k: errors(g[k], g64[k]) for k in g64}
    err["dL/dx"] = errors(dx, dx64)
    held = [k for k in err if lower or not (k.startswith(LOWER) or k == "dL/dx")]
    print(f"\n{label}: max|out - out64| {dout:.2e}, loss {L:.9e} float64 {L64:.9e}")
    for k in sorted(held, key=lambda k: -err[k][0])[:3]:
        print(f"  {k}: |g - g64| / |g64| = {err[k][0]:.2e}, max|g - g64| / max|g64| = {err[k][1]:.2e}")
    for k in sorted(set(err) - set(held)):
        print(f"  {k} (not held): |g - g64| / |g64| = {err[k][0]:.2e}")
    assert dout <= 1e-5 or not lower
    assert all(torch.isfinite(v).all() for v in g.values())
    bad = {k: err[k] for k in held if not (err[k][0] <= 1e-4 and err[k][1] <= 1e-3)}
    assert not bad, sorted((k, f"{e[0]:.1e}", f"{e[1]:.1e}") for k, e in bad.items())


def test_halves_are_train_grads_bits():
    """After pnb_train_forward_device the fc, conv1 and conv2 taps equal those after pnb_train_grad_* on the same
    windows bit for bit, and after pnb_train_backward_device the output pre-activations' gradient equals ATen's
    sigmoid_backward of the caller's dL/d(out) at the output bit for bit."""
    sd = synth_state_dict(1)
    B, T = 3, 40
    rec = moderate_records(B, T, 200)
    eng = trainer(sd, B, T)
    eng.train_grad(rec)
    want = {k: eng.read_tap(k, T, B) for k in ("train_fc", "train_c1", "train_c2pre")}
    x = feats(rec)
    out = torch.empty((B, T, 68), dtype=torch.float32, device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    eng.train_forward_device(x.data_ptr(), T * 70, T, 0, out.data_ptr(), T * 68, s)
    for k, w in want.items():
        assert np.array_equal(eng.read_tap(k, T, B).view(np.int32), w.view(np.int32)), k
    dout = torch.randn((B, T, 68), generator=torch.Generator().manual_seed(201)).cuda()
    eng.train_backward_device(dout.data_ptr(), T * 68, 0, 0, 0, s)
    got = eng.read_tap("train_dpre", T, B)
    sb = torch.ops.aten.sigmoid_backward(dout.transpose(0, 1), out.transpose(0, 1)).cpu().numpy()
    assert np.array_equal(got.view(np.int32), np.ascontiguousarray(sb).view(np.int32))
    eng.close()


SENTINEL = 0x7FA5A5A5   # a NaN bit pattern that no kernel writes: what a store must leave alone keeps it
FWD_TAPS = ("train_fc", "train_c1", "train_c2pre")


def padded(a, stride, pad=(float("nan"),)):
    """a [n, T, w] as rows of `stride` floats, the padding cycling through `pad`."""
    n = a.shape[0]
    flat = a.reshape(n, -1)
    p = torch.tensor(pad, dtype=torch.float32).repeat(stride - flat.shape[1])[:stride - flat.shape[1]]
    return torch.cat([flat, p.to(a.device).expand(n, -1)], 1).contiguous()


def sentinel(rows, stride):
    return torch.full((rows, stride), SENTINEL, dtype=torch.int32, device="cuda").view(torch.float32)


def _tbits(a):
    return a.contiguous().view(torch.int32)


def test_halves_bits_depend_on_the_call_alone():
    """A 10 x 40 forward and backward on the active 10 rows of a 16 x 48 engine created with other weights, after
    forward / backward pairs on all 16 rows and on 10 rows of 48 hops, through padded strides (x padded with NaN and
    1e30, dL/d(out) with NaN) and the caller's blob: out, the fc / c1 / c2pre and dpre taps, dL/dx and d_grad (also the
    exported gradient) are the bits of the same call with exact strides on a fresh 10 x 40 engine of the blob's
    weights, whose weights the engine then holds.  The padding and rows 10..15 of out and dL/dx keep their sentinel.  A
    forward with d_weights NULL after it, and a backward with d_grad NULL, give the same bits again."""
    sd = synth_state_dict(1)
    B, T, S, Fm = 10, 40, 16, 48
    blob = torch.from_numpy(pack_state_dict(sd).flat()).cuda()
    x = feats(moderate_records(B, T, 280))
    dout = torch.randn((B, T, 68), generator=torch.Generator().manual_seed(281)).cuda()

    base = trainer(sd, B, T)
    out0, dx0 = torch.empty((B, T, 68), device="cuda"), torch.empty((B, T, 70), device="cuda")
    g0 = torch.empty(N_PARAMS, device="cuda")
    base.train_forward_device(x.data_ptr(), T * 70, T, 0, out0.data_ptr(), T * 68)
    taps0 = {k: base.read_tap(k, T, B) for k in FWD_TAPS}
    base.train_backward_device(dout.data_ptr(), T * 68, dx0.data_ptr(), T * 70, g0.data_ptr())
    taps0["train_dpre"] = base.read_tap("train_dpre", T, B)
    base.wait()
    base.close()

    eng = trainer(synth_state_dict(3), S, Fm)
    for n in (S, B):                                 # rows and hops past the call's hold other values
        eng.set_active(n)
        xr = feats(moderate_records(n, Fm, 282 + n))
        o, d = torch.empty((n, Fm, 68), device="cuda"), torch.empty((n, Fm, 70), device="cuda")
        do = torch.rand((n, Fm, 68), device="cuda")
        eng.train_forward_device(xr.data_ptr(), Fm * 70, Fm, 0, o.data_ptr(), Fm * 68)
        eng.train_backward_device(do.data_ptr(), Fm * 68, d.data_ptr(), Fm * 70)
        eng.wait()
    xs, os_, ds, dxs = T * 70 + 5, T * 68 + 3, T * 68 + 7, T * 70 + 9
    xp = padded(x, xs, (float("nan"), 1e30))
    dp = padded(dout, ds)

    def call(weights, want_grad):
        out, dx = sentinel(S, os_), sentinel(S, dxs)
        grad = sentinel(1, N_PARAMS)[0]
        eng.train_forward_device(xp.data_ptr(), xs, T, weights, out.data_ptr(), os_)
        taps = {k: eng.read_tap(k, T, B) for k in FWD_TAPS}
        eng.train_backward_device(dp.data_ptr(), ds, dx.data_ptr(), dxs, grad.data_ptr() if want_grad else 0)
        taps["train_dpre"] = eng.read_tap("train_dpre", T, B)
        eng.wait()
        return out, dx, grad, taps

    for label, weights, want_grad in (("blob", blob.data_ptr(), True), ("d_weights NULL, d_grad NULL", 0, False)):
        out, dx, grad, taps = call(weights, want_grad)
        assert _bits(out[:B, :T * 68].reshape(B, T, 68), out0), (label, "out")
        assert _bits(dx[:B, :T * 70].reshape(B, T, 70), dx0), (label, "dx")
        for k, w in taps0.items():
            assert np.array_equal(taps[k].view(np.int32), w.view(np.int32)), (label, k)
        held = torch.from_numpy(eng.train_export("gradient")).cuda()
        assert _bits(held, g0), (label, "held gradient")
        if want_grad:
            assert _bits(grad, g0), (label, "d_grad")
        else:
            assert bool((_tbits(grad) == SENTINEL).all()), (label, "d_grad NULL")
        for name, a, w in (("out", out, T * 68), ("dx", dx, T * 70)):
            assert bool((_tbits(a[:, w:]) == SENTINEL).all()), (label, name, "padding")
            assert bool((_tbits(a[B:]) == SENTINEL).all()), (label, name, "rows past the active range")
        assert np.array_equal(eng.train_export("weights").view(np.int32), blob.cpu().numpy().view(np.int32)), label
    eng.close()


def test_seed_at_saturated_outputs_and_edge_gradients():
    """dL/d(out) of +-inf, NaN, +-0, +-FLT_TRUE_MIN, 1e-40 and +-3e38 (and 1) at every band, on outputs of exactly 1
    and below 1e-12 (biases of +-30 on bands of both output layers): the seed is ATen's sigmoid_backward bit for bit,
    the NaN of inf x 0 included."""
    sd = synth_state_dict(0, 4.0)
    for k in ("fc_gb.0.bias", "fc_rb.0.bias"):
        sd[k] = sd[k].copy()
        sd[k][:4], sd[k][4:8] = 30.0, -30.0
    B, T = 3, 40
    eng = trainer(sd, B, T)
    x = feats(moderate_records(B, T, 290))
    out = torch.empty((B, T, 68), device="cuda")
    eng.train_forward_device(x.data_ptr(), T * 70, T, 0, out.data_ptr(), T * 68)
    tiny = float(np.finfo(np.float32).smallest_subnormal)
    edges = torch.tensor([float("inf"), -float("inf"), float("nan"), 0.0, -0.0, tiny, -tiny, 1e-40, 3e38, -3e38, 1.0])
    # 11 values along the flat index: 68 hops' worth of bands step it by 68 = 2 (mod 11), so every band meets each
    dout = edges[torch.arange(B * T * 68) % len(edges)].reshape(B, T, 68).cuda()
    eng.train_backward_device(dout.data_ptr(), T * 68)
    got = eng.read_tap("train_dpre", T, B)
    eng.close()
    want = torch.ops.aten.sigmoid_backward(dout, out).transpose(0, 1).cpu().numpy()
    o = out.cpu().numpy()
    print(f"\n{int((o == 1).sum())} outputs exactly 1, {int((o <= 1e-12).sum())} at or below 1e-12, "
          f"{int((o == 0).sum())} exactly 0; {int(np.isnan(want).sum())} NaN seeds")
    assert (o == 1).any() and (o <= 1e-12).any()
    inf_at_one = np.isinf(dout.transpose(0, 1).cpu().numpy()) & (o.transpose(1, 0, 2) == 1)
    assert inf_at_one.any() and np.isnan(want[inf_at_one]).all()
    assert np.array_equal(got.view(np.int32), np.ascontiguousarray(want).view(np.int32))


@pytest.mark.parametrize("B,T", [(3, 40), (8, 500)], ids=["3x40", "8x500"])
@pytest.mark.parametrize("loss", ["custom", "arbitrary"])
def test_against_float64_moderate(B, T, loss):
    """Moderate records (no layer saturates): all 30 parameter gradients and dL/dx held to the bar."""
    rec = moderate_records(B, T, 210 + B)
    check(synth_state_dict(1), rec, custom_loss if loss == "custom" else arbitrary_loss(B), f"{B}x{T} {loss} loss")


@pytest.mark.parametrize("B,T", [(3, 40), (8, 500)], ids=["3x40", "8x500"])
def test_against_float64_generator_records(B, T):
    """Generator records at int16 scale, as test_gpu_train.test_gradients_against_float64: the 24 tensors above fc,
    conv1 and conv2 are held, those three and dL/dx printed."""
    rec = windows(B, T, 220 + B)
    check(synth_state_dict(0), rec, arbitrary_loss(B), f"{B}x{T} generator records", lower=False)


def _bits(a, b):
    return torch.equal(a.contiguous().view(torch.int32), b.contiguous().view(torch.int32))


def _same_step(a, b, label):
    assert _bits(a[0], b[0]), (label, "out")
    for k in a[2]:
        assert _bits(a[2][k], b[2][k]), (label, k)
    assert _bits(a[3], b[3]), (label, "dx")


def test_stream_order_and_determinism():
    sd = synth_state_dict(1)
    m = module(sd)
    rec1, rec2 = moderate_records(4, 50, 230), moderate_records(4, 50, 231)
    x1, x2 = feats(rec1), feats(rec2)
    y1, y2 = (torch.from_numpy(np.ascontiguousarray(r[..., 70:])).cuda() for r in (rec1, rec2))
    first = step(m, x1, y1, custom_loss)
    _same_step(first, step(m, x1, y1, custom_loss), "second identical step")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        other = step(m, x1, y1, custom_loss)
    torch.cuda.current_stream().wait_stream(s)
    _same_step(first, other, "non-default stream")
    # two graphs before one backward, and one graph backwards twice: the engine's pending forward is another's
    second = step(m, x2, y2, custom_loss)
    m.zero_grad(set_to_none=True)
    a, b = x1.clone().requires_grad_(True), x2.clone().requires_grad_(True)
    (custom_loss(m(a), y1) + custom_loss(m(b), y2)).backward()
    for k, p in m.named_parameters():
        assert _bits(p.grad, first[2][k] + second[2][k]), ("l1 + l2", k)
    assert _bits(a.grad, first[3]) and _bits(b.grad, second[3])
    m.zero_grad(set_to_none=True)
    a = x1.clone().requires_grad_(True)
    L = custom_loss(m(a), y1)
    L.backward(retain_graph=True)
    L.backward()
    for k, p in m.named_parameters():
        assert _bits(p.grad, first[2][k] + first[2][k]), ("retain_graph", k)
    assert _bits(a.grad, first[3] + first[3])
    m.close()


def test_growing_and_shrinking_shapes():
    """One module through batches and lengths that grow and shrink equals a fresh module at each shape."""
    sd = synth_state_dict(1)
    m = module(sd)
    for i, (B, T) in enumerate([(2, 30), (5, 60), (3, 20), (5, 60), (6, 10)]):
        rec = moderate_records(B, T, 240 + i)
        x, y = feats(rec), torch.from_numpy(np.ascontiguousarray(rec[..., 70:])).cuda()
        got = step(m, x, y, custom_loss)
        fresh = module(sd)
        _same_step(got, step(fresh, x, y, custom_loss), f"{B}x{T}")
        fresh.close()
    m.close()


def test_module_edges_give_the_plain_steps_bits():
    """fp16 and bf16 x under autocast (x.grad the plain dL/dx in that dtype), x as a strided slice and as a transposed
    view, out.sum() (dL/d(out) expanded, stride 0) against an explicit weighting by ones, a loss of the g half only
    against a weighting with zeros on r, x without requires_grad (100 launches in the backward, not 102) and a frozen fc
    (the other 28 gradients): each gives the bits of the same step on float32 contiguous x."""
    sd = synth_state_dict(1)
    m = module(sd)
    B, T = 4, 30
    rec = moderate_records(B, T, 300)
    x, y = feats(rec), torch.from_numpy(np.ascontiguousarray(rec[..., 70:])).cuda()
    plain = step(m, x, y, custom_loss)
    for dt in (torch.float16, torch.bfloat16):
        xl = x.to(dt)
        want = step(m, xl.float(), y, custom_loss)
        with torch.autocast("cuda", dtype=dt):
            got = step(m, xl, y, custom_loss)
        assert got[3].dtype == dt, dt
        _same_step(got, want[:3] + (want[3].to(dt),), str(dt))
    wide = torch.full((B, 2 * T, 70), float("nan"), device="cuda")
    wide[:, ::2] = x
    for label, xv in (("[:, ::2] slice", wide[:, ::2]), ("transposed view", x.transpose(0, 1).contiguous().transpose(0, 1))):
        assert not xv.is_contiguous() and torch.equal(xv, x)
        _same_step(step(m, xv, y, custom_loss), plain, label)
    _same_step(step(m, x, y, lambda o, y: o.sum()), step(m, x, y, lambda o, y: (o * torch.ones_like(o)).sum()),
               "out.sum()")
    w = torch.rand((B, T, 68), generator=torch.Generator().manual_seed(301)).cuda()
    wz = w.clone()
    wz[..., 34:] = 0
    _same_step(step(m, x, y, lambda o, y: (o[..., :34] * w[..., :34]).sum()), step(m, x, y, lambda o, y: (o * wz).sum()),
               "g half only")
    tr = m._trainers[x.device]
    m.zero_grad(set_to_none=True)
    L = custom_loss(m(x), y)
    n0 = tr.eng.launches
    L.backward()
    assert tr.eng.launches - n0 == 100
    for k, p in m.named_parameters():
        assert _bits(p.grad, plain[2][k]), ("x without requires_grad", k)
    m.fc.requires_grad_(False)
    got = step(m, x, y, custom_loss)
    m.fc.requires_grad_(True)
    assert sorted(got[2]) == sorted(k for k in plain[2] if not k.startswith("fc.")) and len(got[2]) == 28
    _same_step(got, plain, "fc frozen")
    m.close()


def test_row_limit():
    """B x T above 65535 x 64 rows raises ValueError before any engine exists (x an expanded zero-stride tensor, no
    memory); pnb_create of a PNB_TRAIN_NETWORK engine one row above refuses it with PNB_ERR_ARG.  One stream of
    4 194 241 hops: what the engine allocates before that check per stream (network state, the f32 chain's rings)
    is then one stream's, and only the per-row feature and g/r buffers (2.3 GB) remain."""
    m = module(synth_state_dict(0))
    for shape in ((tm.MAX_ROWS + 1, 1, 70), (1, tm.MAX_ROWS + 1, 70), (2049, 2048, 70)):
        with pytest.raises(ValueError, match="65535 x 64"):
            m(torch.zeros((1, 1, 1), device="cuda").expand(*shape))
    assert not m._trainers
    with pytest.raises(api.PnbError, match=r"\(-1\): PNB_TRAIN_NETWORK: n_streams x max_frames_per_call above 65535 x 64"):
        api.Engine(1, tm.MAX_ROWS + 1, pack_state_dict(synth_state_dict(0)), api.TRAIN_NETWORK)


def test_launch_counts():
    """Each new call issues a fixed number of launches whatever T; pnb_train_grad_* still issues 118."""
    sd = synth_state_dict(0)
    counts = []
    for T in (40, 500):
        eng = trainer(sd, 2, T)
        rec = moderate_records(2, T, 250)
        x = feats(rec)
        out = torch.empty((2, T, 68), device="cuda")
        dx = torch.empty((2, T, 70), device="cuda")
        n0 = eng.launches
        eng.train_grad(rec)
        n1 = eng.launches
        eng.train_forward_device(x.data_ptr(), T * 70, T, 0, out.data_ptr(), T * 68)
        n2 = eng.launches
        eng.train_backward_device(out.data_ptr(), T * 68)
        n3 = eng.launches
        eng.train_forward_device(x.data_ptr(), T * 70, T, 0, out.data_ptr(), T * 68)
        n4 = eng.launches
        eng.train_backward_device(out.data_ptr(), T * 68, dx.data_ptr(), T * 70)
        eng.wait()
        counts.append((n1 - n0, n2 - n1, n3 - n2, eng.launches - n4, eng.launches_per_call(T)))
        eng.close()
    print(f"\nlaunches (train_grad, forward, backward, backward with dx, per call): {counts}")
    assert counts[0] == counts[1] == (118, 17, 100, 102, 118)


def test_refusals():
    L = api.load_library()
    pm = pack_state_dict(synth_state_dict(0))
    B, T = 2, 10
    x = torch.zeros((B, T, 70), device="cuda")
    out = torch.zeros((B, T, 68), device="cuda")
    dx = torch.zeros((B, T, 70), device="cuda")
    other = api.Engine(B, T, pm, api.NETWORK_ONLY)
    with pytest.raises(api.PnbError, match="PNB_TRAIN_NETWORK"):
        other.train_forward_device(x.data_ptr(), T * 70, T, 0, out.data_ptr(), T * 68)
    with pytest.raises(api.PnbError, match="PNB_TRAIN_NETWORK"):
        other.train_backward_device(out.data_ptr(), T * 68)
    other.close()
    eng = api.Engine(B, T, pm, api.TRAIN_NETWORK)
    n0 = eng.launches
    fwd = lambda: eng.train_forward_device(x.data_ptr(), T * 70, T, 0, out.data_ptr(), T * 68)
    bwd = lambda: eng.train_backward_device(out.data_ptr(), T * 68, dx.data_ptr(), T * 70)
    with pytest.raises(api.PnbError, match="no pnb_train_forward_device"):
        bwd()
    for n_frames in (0, T + 1):
        assert L.pnb_train_forward_device(eng.h, x.data_ptr(), T * 70, n_frames, None, out.data_ptr(), T * 68, None) == -1
    assert L.pnb_train_forward_device(eng.h, None, T * 70, T, None, out.data_ptr(), T * 68, None) == -1
    assert L.pnb_train_forward_device(eng.h, x.data_ptr(), T * 70, T, None, None, T * 68, None) == -1
    assert L.pnb_train_forward_device(eng.h, x.data_ptr(), T * 70 - 1, T, None, out.data_ptr(), T * 68, None) == -1
    assert L.pnb_train_forward_device(eng.h, x.data_ptr(), T * 70, T, None, out.data_ptr(), T * 68 - 1, None) == -1
    assert eng.launches == n0
    fwd()
    n1 = eng.launches
    assert L.pnb_train_backward_device(eng.h, None, T * 68, None, 0, None, None) == -1
    assert L.pnb_train_backward_device(eng.h, out.data_ptr(), T * 68 - 1, None, 0, None, None) == -1
    assert L.pnb_train_backward_device(eng.h, out.data_ptr(), T * 68, dx.data_ptr(), T * 70 - 1, None, None) == -1
    assert eng.launches == n1
    bwd()
    n2 = eng.launches
    with pytest.raises(api.PnbError, match="no pnb_train_forward_device"):
        bwd()                                        # one backward per forward
    fwd()
    eng.train_grad(np.zeros((B, T, 138), np.float32))
    n3 = eng.launches
    with pytest.raises(api.PnbError, match="no pnb_train_forward_device"):
        bwd()                                        # a gradient call ends the wait
    fwd()
    eng.set_active(1)
    n4 = eng.launches
    with pytest.raises(api.PnbError, match="no pnb_train_forward_device"):
        bwd()                                        # so does a new active range
    eng.set_active(2)
    fwd()
    eng.reset()
    n5 = eng.launches
    with pytest.raises(api.PnbError, match="no pnb_train_forward_device"):
        bwd()                                        # and pnb_reset
    assert (eng.launches, n2 - n1, n3 - n2, n4 - n3) == (n5, 102, 17 + 118, 17)
    eng.wait()
    eng.close()

    # an Adam step and an import of the weights rewrite the weights the pending forward's backward would take: both
    # end the wait, and the refused backward changes nothing (the next step is a twin's that saw no refusal)
    sd = synth_state_dict(0)
    x = feats(moderate_records(B, T, 310))
    dout = torch.rand((B, T, 68), generator=torch.Generator().manual_seed(311)).cuda()
    w2 = pack_state_dict(synth_state_dict(2)).flat()
    for label, change in (("train_adam", lambda e: e.train_adam(1e-3, 1)),
                          ("train_import of the weights", lambda e: e.train_import("weights", w2))):
        eng, twin = trainer(sd, B, T), trainer(sd, B, T)
        runs = {}
        for e in (eng, twin):
            e.train_forward_device(x.data_ptr(), T * 70, T, 0, out.data_ptr(), T * 68)
            e.train_backward_device(dout.data_ptr(), T * 68)
        n0 = eng.launches
        eng.train_forward_device(x.data_ptr(), T * 70, T, 0, out.data_ptr(), T * 68)
        n1 = eng.launches
        change(eng)
        n2 = eng.launches
        with pytest.raises(api.PnbError, match="no pnb_train_forward_device.*pnb_train_adam"):
            eng.train_backward_device(dout.data_ptr(), T * 68, dx.data_ptr(), T * 70)
        assert (n1 - n0, eng.launches) == (17, n2), label
        change(twin)
        for name, e in (("refused", eng), ("twin", twin)):
            o, d = torch.empty_like(out), torch.empty_like(dx)
            g = torch.empty(N_PARAMS, device="cuda")
            e.train_forward_device(x.data_ptr(), T * 70, T, 0, o.data_ptr(), T * 68)
            e.train_backward_device(dout.data_ptr(), T * 68, d.data_ptr(), T * 70, g.data_ptr())
            e.wait()
            runs[name] = (o, d, g, e.train_export("weights"))
            e.close()
        for k in range(3):
            assert _bits(runs["refused"][k], runs["twin"][k]), (label, k)
        assert np.array_equal(runs["refused"][3].view(np.int32), runs["twin"][3].view(np.int32)), label
    # an import of m keeps the wait: the parameters are unchanged
    eng = trainer(sd, B, T)
    eng.train_forward_device(x.data_ptr(), T * 70, T, 0, out.data_ptr(), T * 68)
    eng.train_import("m", np.zeros(N_PARAMS, np.float32))
    eng.train_backward_device(dout.data_ptr(), T * 68, dx.data_ptr(), T * 70)
    eng.wait()
    eng.close()


def test_nonfinite_gradient_passes_through():
    """A NaN in dL/d(out) reaches .grad without raising, the engine keeps working (no domain bit), and pnb_train_adam
    on that held gradient is skipped; the next finite step applies."""
    sd = synth_state_dict(1)
    m = module(sd)
    rec = moderate_records(2, 20, 260)
    x, y = feats(rec), torch.from_numpy(np.ascontiguousarray(rec[..., 70:])).cuda()
    nan_at = torch.zeros((2, 20, 68), device="cuda")
    nan_at[0, 5, 3] = float("nan")
    _, _, g, dx = step(m, x, y, lambda out, y: custom_loss(out, y) + (out * nan_at).sum())
    assert any(torch.isnan(v).any() for v in g.values()) and torch.isnan(dx).any()
    tr = m._trainers[x.device]
    tr.eng.check()                                   # no PNB_ERR_DOMAIN
    w = tr.eng.train_export("weights")
    tr.eng.train_adam(1e-3, 1)
    tr.eng.wait()
    assert np.array_equal(tr.eng.train_export("weights").view(np.int32), w.view(np.int32))
    _, _, g, _ = step(m, x, y, custom_loss)
    assert all(torch.isfinite(v).all() for v in g.values())
    tr.eng.train_adam(1e-3, 1)
    tr.eng.check()
    assert not np.array_equal(tr.eng.train_export("weights"), w)
    m.close()


def test_closing_the_loop():
    """rnn_train.py's step body -- zero_grad, model(x), CustomLoss, backward, torch.optim.Adam.step at lr 1e-3 -- for 200
    steps on 8 x 100 quiet generator windows lowers the loss; pack_state_dict of the module's state_dict loads in a
    network-only engine, whose score matches the module's exact-activation loss within 1e-3."""
    rec = generator_records(8, 100, 108, quiet=64).cpu().numpy()
    x, y = feats(rec), torch.from_numpy(np.ascontiguousarray(rec[..., 70:])).cuda()
    m = module(synth_state_dict(2))
    opt = torch.optim.Adam(m.parameters(), lr=1e-3)
    losses = []
    for _ in range(200):
        opt.zero_grad()
        L = custom_loss(m(x), y)
        L.backward()
        opt.step()
        losses.append(float(L.detach()))
    first, last = np.mean(losses[:20]), np.mean(losses[-20:])
    print(f"\nloss: first 20 steps {first:.6f}, last 20 {last:.6f}")
    assert np.all(np.isfinite(losses)) and last < first
    with torch.no_grad():
        exact = float(custom_loss(m(x).double(), y.double()))
    m.close()
    pm = pack_state_dict({k: v.detach().cpu().numpy() for k, v in m.state_dict().items()})
    eng = api.Engine(8, 100, pm, api.NETWORK_ONLY)
    sums, _ = eng.score_records(rec)
    eng.close()
    deployed = loss_terms(sums.sum(0))["total"]
    print(f"deployed (tansig) loss {deployed:.9f}, module (exact) loss {exact:.9f}, rel {abs(deployed - exact) / exact:.2e}")
    assert abs(deployed - exact) <= 1e-3 * exact
