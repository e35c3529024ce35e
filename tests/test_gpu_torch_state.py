"""Network state in and out of torch_module.PercepNet and the trainer's forward and backward on the GPU: zero state is
the call without state bit for bit, chained windows are the whole window bit for bit, per-window lengths are each window
run alone, gradients through two chained calls (dL/d(state) included) against float64 autograd of the restatement with
state (train_state_oracle), the recompute of a stateful forward, and the launch count of every option and the refusals
of the state calls."""

import numpy as np
import pytest
import torch

from percepnet_b200 import api, torch_module as tm
from percepnet_b200.weights import N_PARAMS, synth_state_dict
import train_oracle as O
import train_state_oracle as SO
from test_gpu_train import LOWER, moderate_records, trainer, windows
from test_gpu_torch_module import _bits, arbitrary_loss, custom_loss, errors, feats, module

pytestmark = pytest.mark.gpu
S = tm.STATE_FLOATS


def labels(rec):
    return torch.from_numpy(np.ascontiguousarray(rec[..., 70:])).cuda()


def grads_of(m):
    return {k: p.grad.detach().clone() for k, p in m.named_parameters()}


def test_zero_state_is_todays_call():
    """m(x, state=zeros), m(x, return_state=True) and both give m(x)'s out, parameter gradients and dL/dx bit for bit;
    the raw state calls with every option NULL give the plain calls' bits, and the plain calls still issue 17, 100
    and 102 launches."""
    sd = synth_state_dict(1)
    B, T = 3, 40
    rec = moderate_records(B, T, 400)
    x, y = feats(rec), labels(rec)
    m = module(sd)

    def run(**kw):
        m.zero_grad(set_to_none=True)
        xx = x.clone().requires_grad_(True)
        res = m(xx, **kw)
        out = res[0] if isinstance(res, tuple) else res
        custom_loss(out, y).backward()
        return out.detach(), grads_of(m), xx.grad.detach().clone()

    plain = run()
    for label, with_state, ret in (("state=zeros", True, False), ("return_state", False, True), ("both", True, True)):
        zeros = torch.zeros((B, S), device="cuda", requires_grad=True)
        got = run(**({"state": zeros} if with_state else {}), return_state=ret)
        assert _bits(got[0], plain[0]), (label, "out")
        assert _bits(got[2], plain[2]), (label, "dx")
        for k in plain[1]:
            assert _bits(got[1][k], plain[1][k]), (label, k)
        if with_state:
            assert zeros.grad is not None and bool(torch.isfinite(zeros.grad).all()), label
    m.close()

    eng = trainer(sd, B, T)
    dout = torch.randn((B, T, 68), generator=torch.Generator().manual_seed(401)).cuda()
    res = {}
    for label in ("plain", "state, NULLs"):
        out, dx, g = torch.empty((B, T, 68), device="cuda"), torch.empty((B, T, 70), device="cuda"), torch.empty(N_PARAMS, device="cuda")
        n0 = eng.launches
        if label == "plain":
            eng.train_forward_device(x.data_ptr(), T * 70, T, 0, out.data_ptr(), T * 68)
            n1 = eng.launches
            eng.train_backward_device(dout.data_ptr(), T * 68, 0, 0, 0)
            n2 = eng.launches
            eng.train_forward_device(x.data_ptr(), T * 70, T, 0, out.data_ptr(), T * 68)
            eng.train_backward_device(dout.data_ptr(), T * 68, dx.data_ptr(), T * 70, g.data_ptr())
        else:
            eng.train_forward_state_device(x.data_ptr(), T * 70, T, d_out=out.data_ptr(), out_stride=T * 68)
            n1 = eng.launches
            eng.train_backward_state_device(dout.data_ptr(), T * 68)
            n2 = eng.launches
            eng.train_forward_state_device(x.data_ptr(), T * 70, T, d_out=out.data_ptr(), out_stride=T * 68)
            eng.train_backward_state_device(dout.data_ptr(), T * 68, d_dx=dx.data_ptr(), dx_stride=T * 70,
                                            d_grad=g.data_ptr())
        eng.wait()
        res[label] = (out, dx, g, (n1 - n0, n2 - n1, eng.launches - n2))
    eng.close()
    for k in range(3):
        assert _bits(res["plain"][k], res["state, NULLs"][k]), k
    assert res["plain"][3] == res["state, NULLs"][3] == (17, 100, 17 + 102)


@pytest.mark.parametrize("B,T,cuts", [(3, 40, (1, 3, 4, 17)), (8, 500, (250,))], ids=["3x40", "8x500"])
def test_chunks_are_the_whole_window(B, T, cuts):
    """Chained chunks, each from the state out of the one before, give the outputs and the final state of one forward
    over the whole window bit for bit, from zero state and from a random state."""
    rec = moderate_records(B, T, 410 + B)
    x = feats(rec)
    m = module(synth_state_dict(1))
    for s0 in (None, SO.random_state(B, 411).cuda()):
        with torch.no_grad():
            whole, s_whole = m(x, s0, return_state=True)
            outs, s = [], s0
            for a, b in zip((0,) + cuts, cuts + (T,)):
                o, s = m(x[:, a:b], s, return_state=True)
                outs.append(o)
        label = "zero state" if s0 is None else "random state"
        assert _bits(torch.cat(outs, 1), whole), (label, "out")
        assert _bits(s, s_whole), (label, "state out")
    m.close()


def test_lengths():
    """Windows of lengths 40, 1, 17 and 3 in a 40-hop call, padded with NaN, from a random state: each window's rows
    below its length and its state out are that window run alone over its hops bit for bit, its later rows are zeros,
    and NaN in dL/d(out) past its end reaches no gradient: every gradient is the one with zeros there, bit for bit, and
    dL/dx past the end is zero."""
    B, T, lens = 4, 40, [40, 1, 17, 3]
    rec = moderate_records(B, T, 420)
    x = feats(rec)
    xp = x.clone()
    past = torch.zeros((B, T), dtype=torch.bool)
    for b, L in enumerate(lens):
        past[b, L:] = True
    past = past.cuda()
    xp[past] = float("nan")
    s0 = SO.random_state(B, 421).cuda()
    m = module(synth_state_dict(1))
    g = torch.Generator().manual_seed(422)
    w, ws = torch.rand((B, T, 68), generator=g).cuda(), torch.rand((B, S), generator=g).cuda()
    wn = w.clone()
    wn[past] = float("nan")

    def run(dout):
        m.zero_grad(set_to_none=True)
        xx, ss = xp.clone().requires_grad_(True), s0.clone().requires_grad_(True)
        out, s_out = m(xx, ss, lengths=lens, return_state=True)
        torch.autograd.backward([out, s_out], [dout, ws])
        return out.detach(), s_out.detach(), grads_of(m), xx.grad.detach().clone(), ss.grad.detach().clone()

    out, s_out, gp, dx, ds = run(wn)
    for b, L in enumerate(lens):
        with torch.no_grad():
            ob, sb = m(x[b:b + 1, :L], s0[b:b + 1], return_state=True)
        assert _bits(out[b, :L], ob[0]) and _bits(s_out[b], sb[0]), (b, L)
        assert bool((out[b, L:].view(torch.int32) == 0).all()), (b, L)
    zero = run(torch.where(past[..., None], torch.zeros_like(w), w))
    assert all(bool(torch.isfinite(v).all()) for v in gp.values()) and bool(torch.isfinite(ds).all())
    for k in gp:
        assert _bits(gp[k], zero[2][k]), k
    assert _bits(dx, zero[3]) and _bits(ds, zero[4])
    assert bool((dx[past] == 0).all()) and bool(torch.isfinite(dx).all())
    m.close()


def state_loss(kind, B):
    """(loss of (out, state_out, y), whether it weights state_out): CustomLoss of out, or an arbitrary loss of out plus
    a random weighting of the final state."""
    if kind == "custom":
        return (lambda out, s, y: custom_loss(out, y)), False
    f = arbitrary_loss(B)
    ws = torch.rand((B, S), generator=torch.Generator().manual_seed(431), dtype=torch.float64)

    def loss(out, s, y):
        return f(out, y) + (s * ws.to(s)).mean()
    return loss, True


def check_chain(sd, rec, kind, label, lower=True):
    """Two chained calls (hops [0, T/2) and [T/2, T)) from a random state that requires a gradient, the state not
    detached between them, against float64 autograd of the restatement over all T hops: out within 1e-5, every parameter
    gradient, dL/dx and dL/d(state) within |g - g64| / |g64| <= 1e-4 and max|g - g64| <= 1e-3 max|g64|.  With
    lower=False fc, conv1, conv2, dL/dx and the gradient at the state's conv histories are printed, not held."""
    B, T = rec.shape[:2]
    T1 = T // 2
    x, y = feats(rec), labels(rec)
    s0 = SO.random_state(B, 430).cuda()
    loss, weights_state = state_loss(kind, B)
    m = module(sd)
    xx, ss = x.clone().requires_grad_(True), s0.clone().requires_grad_(True)
    o1, s1 = m(xx[:, :T1], ss, return_state=True)
    o2, s2 = m(xx[:, T1:], s1, return_state=True)
    out = torch.cat([o1, o2], 1)
    loss(out, s2, y).backward()
    g = grads_of(m)
    m.close()
    ref = O.model(sd, torch.float64, "cuda")
    x64, s64 = x.double().requires_grad_(True), s0.double().requires_grad_(True)
    out64, s_out64 = SO.forward(ref, x64, s64)
    loss(out64, s_out64, y.double()).backward()
    dout = float((out.detach().double() - out64.detach()).abs().max())
    # relative: on generator records the fc history holds int16-scale values
    dstate = float((s2.detach().double() - s_out64.detach()).abs().max() / s_out64.detach().abs().max())
    err = {k: errors(g[k], p.grad) for k, p in ref.named_parameters()}
    err["dL/dx"] = errors(xx.grad, x64.grad)
    err["dL/d(state) GRUs"] = errors(ss.grad[:, 1536:], s64.grad[:, 1536:])
    err["dL/d(state) histories"] = errors(ss.grad[:, :1536], s64.grad[:, :1536])
    held = [k for k in err if lower or not (k.startswith(LOWER) or k in ("dL/dx", "dL/d(state) histories"))]
    print(f"\n{label}: max|out - out64| {dout:.2e}, max|state - state64| / max|state64| {dstate:.2e}, "
          f"loss weights state: {weights_state}")
    for k in sorted(held, key=lambda k: -err[k][0])[:4]:
        print(f"  {k}: |g - g64| / |g64| = {err[k][0]:.2e}, max|g - g64| / max|g64| = {err[k][1]:.2e}")
    for k in sorted(set(err) - set(held)):
        print(f"  {k} (not held): |g - g64| / |g64| = {err[k][0]:.2e}")
    assert (dout <= 1e-5 and dstate <= 1e-5) or not lower
    assert all(bool(torch.isfinite(v).all()) for v in g.values()) and bool(torch.isfinite(ss.grad).all())
    bad = {k: err[k] for k in held if not (err[k][0] <= 1e-4 and err[k][1] <= 1e-3)}
    assert not bad, sorted((k, f"{e[0]:.1e}", f"{e[1]:.1e}") for k, e in bad.items())


@pytest.mark.parametrize("B,T,kind", [(3, 40, "custom"), (3, 40, "arbitrary"), (8, 500, "arbitrary")],
                         ids=["3x40-custom", "3x40-arbitrary", "8x500-arbitrary"])
def test_chain_against_float64_moderate(B, T, kind):
    check_chain(synth_state_dict(1), moderate_records(B, T, 440 + B), kind, f"{B}x{T} {kind} loss, moderate records")


@pytest.mark.parametrize("B,T", [(3, 40), (8, 500)], ids=["3x40", "8x500"])
def test_chain_against_float64_generator_records(B, T):
    check_chain(synth_state_dict(0), windows(B, T, 450 + B), "arbitrary", f"{B}x{T} generator records", lower=False)


def test_recompute_of_a_stateful_forward():
    """A stateful forward with lengths, another stateful forward, then the first one's backward: the first one's
    gradients (parameters, dL/dx, dL/d(state)) are those of a lone forward and backward bit for bit."""
    B, T, lens = 3, 30, [30, 7, 2]
    rec = moderate_records(B, T, 460)
    x, x2 = feats(rec), feats(moderate_records(B, T, 461))
    s0, s2 = SO.random_state(B, 462).cuda(), SO.random_state(B, 463).cuda()
    loss, _ = state_loss("arbitrary", B)
    y = labels(rec)
    m = module(synth_state_dict(1))

    def first():
        m.zero_grad(set_to_none=True)
        xx, ss = x.clone().requires_grad_(True), s0.clone().requires_grad_(True)
        out, s = m(xx, ss, lengths=lens, return_state=True)
        return xx, ss, loss(out, s, y)

    xx, ss, L = first()
    L.backward()
    lone = (grads_of(m), xx.grad.clone(), ss.grad.clone())
    xx, ss, L = first()
    with torch.no_grad():
        m(x2, s2, lengths=[5, 30, 1], return_state=True)
    L.backward()
    for k, v in lone[0].items():
        assert _bits(m.get_parameter(k).grad, v), k
    assert _bits(xx.grad, lone[1]) and _bits(ss.grad, lone[2])
    m.close()


def test_launch_counts_and_refusals():
    """Every combination of the forward's state in, lengths and state out, and of the backward's dL/dx, dL/d(state out)
    and dL/d(state in), issues its documented count at two lengths.  Short state strides, lengths outside [1, n_frames]
    and a lengths array of the wrong size are refused before anything is enqueued, and the engine then gives a fresh
    engine's bits.  The module refuses a state on another device."""
    sd = synth_state_dict(0)
    B = 3
    for T in (10, 40):
        eng = trainer(sd, B, T)
        x = feats(moderate_records(B, T, 470))
        st_in, st_out = SO.random_state(B, 471).cuda(), torch.empty((B, S), device="cuda")
        out, dout = torch.empty((B, T, 68), device="cuda"), torch.rand((B, T, 68), device="cuda")
        dx, dsi, dso = torch.empty((B, T, 70), device="cuda"), torch.empty((B, S), device="cuda"), torch.rand((B, S), device="cuda")
        lens = [T, 1, T // 2]
        for si in (0, 1):
            for ln in (0, 1):
                for so in (0, 1):
                    n0 = eng.launches
                    eng.train_forward_state_device(x.data_ptr(), T * 70, T, lens if ln else None, 0,
                                                   st_in.data_ptr() if si else 0, S, out.data_ptr(), T * 68,
                                                   st_out.data_ptr() if so else 0, S)
                    assert eng.launches - n0 == 17 + si + 2 * ln + so, (T, si, ln, so)
                    eng.train_backward_state_device(dout.data_ptr(), T * 68)
        for ddx in (0, 1):
            for dso_ in (0, 1):
                for dsi_ in (0, 1):
                    eng.train_forward_state_device(x.data_ptr(), T * 70, T, lens, 0, st_in.data_ptr(), S,
                                                   out.data_ptr(), T * 68)
                    n0 = eng.launches
                    eng.train_backward_state_device(dout.data_ptr(), T * 68, dso.data_ptr() if dso_ else 0, S,
                                                    dx.data_ptr() if ddx else 0, T * 70, dsi.data_ptr() if dsi_ else 0,
                                                    S)
                    assert eng.launches - n0 == 100 + 2 * ddx + dso_ + 6 * dsi_, (T, ddx, dso_, dsi_)
        eng.wait()
        eng.close()

    T = 10
    L = api.load_library()
    x = feats(moderate_records(B, T, 472))
    st_in = SO.random_state(B, 473).cuda()
    dout, dso = torch.rand((B, T, 68), device="cuda"), torch.rand((B, S), device="cuda")

    def call(eng):
        o, so, d, dsi = (torch.empty((B, T, 68), device="cuda"), torch.empty((B, S), device="cuda"),
                         torch.empty((B, T, 70), device="cuda"), torch.empty((B, S), device="cuda"))
        gr = torch.empty(N_PARAMS, device="cuda")
        eng.train_forward_state_device(x.data_ptr(), T * 70, T, [T, 3, 1], 0, st_in.data_ptr(), S, o.data_ptr(), T * 68,
                                       so.data_ptr(), S)
        eng.train_backward_state_device(dout.data_ptr(), T * 68, dso.data_ptr(), S, d.data_ptr(), T * 70,
                                        dsi.data_ptr(), S, gr.data_ptr())
        eng.wait()
        return o, so, d, dsi, gr

    fresh = trainer(sd, B, T)
    want = call(fresh)
    fresh.close()
    eng = trainer(sd, B, T)
    n0 = eng.launches
    ok_lens = np.array([T, 3, 1], np.int32)
    fwd = L.pnb_train_forward_state_device
    for lens in ([0, 3, 1], [T + 1, 3, 1], [T, -1, 1]):
        a = np.array(lens, np.int32)
        assert fwd(eng.h, x.data_ptr(), T * 70, T, a.ctypes.data, None, st_in.data_ptr(), S, dout.data_ptr(), T * 68,
                   None, 0, None) == -1, lens
        assert b"lengths[" in L.pnb_last_error()
    assert fwd(eng.h, x.data_ptr(), T * 70, T, ok_lens.ctypes.data, None, st_in.data_ptr(), S - 1, dout.data_ptr(),
               T * 68, None, 0, None) == -1
    assert b"state_in_stride" in L.pnb_last_error()
    assert fwd(eng.h, x.data_ptr(), T * 70, T, None, None, None, 0, dout.data_ptr(), T * 68, dso.data_ptr(), S - 1,
               None) == -1
    assert b"state_out_stride" in L.pnb_last_error()
    with pytest.raises(api.PnbError, match="lengths needs one entry per active row"):
        eng.train_forward_state_device(x.data_ptr(), T * 70, T, [T, 3], d_out=dout.data_ptr(), out_stride=T * 68)
    assert eng.launches == n0
    o = torch.empty((B, T, 68), device="cuda")
    eng.train_forward_state_device(x.data_ptr(), T * 70, T, None, 0, 0, S, o.data_ptr(), T * 68)
    n1 = eng.launches
    bwd = L.pnb_train_backward_state_device
    assert bwd(eng.h, dout.data_ptr(), T * 68, dso.data_ptr(), S - 1, None, 0, None, 0, None, None) == -1
    assert b"dstate_out_stride" in L.pnb_last_error()
    assert bwd(eng.h, dout.data_ptr(), T * 68, None, 0, None, 0, dso.data_ptr(), S - 1, None, None) == -1
    assert b"dstate_in_stride" in L.pnb_last_error()
    assert eng.launches == n1
    got = call(eng)
    eng.close()
    for k in range(5):
        assert _bits(got[k], want[k]), k

    m = module(sd)
    with pytest.raises(ValueError, match="x's device"):
        m(x, st_in.cpu())
    m.close()
