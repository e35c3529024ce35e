"""torch_module.PercepNet on the GPU: the bits of the trainer's forward and backward halves against pnb_train_grad_*
and ATen, gradients of torch losses against float64 autograd of the torch restatement (train_oracle) at the module's
own weights, stream order and determinism, the recompute of a forward whose engine moved on, launch counts, refusals,
non-finite gradients, and rnn_train.py's training step closing the loop."""

import numpy as np
import pytest
import torch

from percepnet_b200 import api, torch_module as tm
from percepnet_b200.eval_records import loss_terms
from percepnet_b200.weights import pack_state_dict, synth_state_dict
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
    """zero_grad, forward, loss, backward: (out, loss, {name: grad}, dx)."""
    m.zero_grad(set_to_none=True)
    x = x.clone().requires_grad_(want_dx)
    out = m(x)
    L = loss_fn(out, y)
    L.backward()
    return out.detach(), float(L.detach()), {k: p.grad.detach().clone() for k, p in m.named_parameters()}, \
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
