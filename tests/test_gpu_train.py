"""The trainer on the GPU (PNB_TRAIN_NETWORK): gradients against float64 autograd of the torch restatement
(train_oracle), saturated outputs, padding, determinism, the launch count, Adam against torch.optim.Adam, non-finite
gradients, a closed training loop, and the refusals."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from percepnet_b200 import api
from percepnet_b200.eval_records import loss_terms
from percepnet_b200.synth import synth_pairs
from percepnet_b200.weights import PackedModel, pack_state_dict, synth_state_dict, unpack_state_dict
import train_oracle as O

pytestmark = pytest.mark.gpu


def generator_records(n_pairs, F, seed, quiet=1):
    """Records of a PNB_TRAIN_DATA engine, handed over on the device (pnb_train_records_device); quiet > 1 divides the
    int16 audio first (band energies / quiet^2)."""
    c16, n16 = synth_pairs(n_pairs, F, seed=seed)
    c16, n16 = (c16 // quiet).astype(np.int16), (n16 // quiet).astype(np.int16)
    eng = api.Engine(2 * n_pairs, F, None, api.TRAIN_DATA)
    ds, dn = torch.from_numpy(c16).cuda(), torch.from_numpy(n16).cuda()
    rec = torch.empty((n_pairs, F, 138), dtype=torch.float32, device="cuda")
    eng.train_records_device(ds.data_ptr(), F * 480, dn.data_ptr(), F * 480, F, rec.data_ptr(), F * 138)
    eng.wait()
    eng.close()
    return rec


def trainer(sd, B, T):
    return api.Engine(B, T, pack_state_dict(sd), api.TRAIN_NETWORK)


def grads_of(eng):
    return unpack_state_dict(PackedModel.from_flat(eng.train_export("gradient")))


def windows(B, T, seed, quiet=1):
    return np.ascontiguousarray(generator_records(B, T, seed, quiet).cpu().numpy())


CASES = [(3, 40, (40, 23, 40)), (8, 500, None)]


LOWER = ("fc.", "conv1.", "conv2.")


def moderate_records(B, T, seed):
    """Records whose network input is of order one (band energies x 30 up to 1.5, pitch fields in [0, 1]), labels uniform
    in [0, 1]: no layer saturates."""
    rng = np.random.RandomState(seed)
    rec = rng.rand(B, T, 138).astype(np.float32)
    rec[..., :68] *= np.float32(0.05)
    return rec


def check_against_float64(sd, rec, frames, label, lower=True):
    """Every one of the 30 parameter tensors (lower=False: all but fc, conv1 and conv2, whose errors are printed) within
    |g - g64| / |g64| <= 1e-4 and max|g - g64| <= 1e-3 max|g64|, and the loss within 1e-6 of float64."""
    B, T = rec.shape[:2]
    eng = trainer(sd, B, T)
    sums = eng.train_grad(rec, frames)
    g = grads_of(eng)
    eng.close()
    L64, g64 = O.grads(sd, rec, frames, torch.float64, "cuda")
    loss = loss_terms(sums.sum(0))["total"]
    print(f"\n{label}: loss {loss:.9e} float64 {L64:.9e} rel {abs(loss - L64) / L64:.2e}")
    assert abs(loss - L64) <= 1e-6 * abs(L64)
    err = {}
    for k, w in g64.items():
        assert np.all(np.isfinite(g[k])), k
        d = np.asarray(g[k], np.float64) - w
        err[k] = (np.linalg.norm(d) / max(np.linalg.norm(w), 1e-300), np.abs(d).max() / max(np.abs(w).max(), 1e-300))
    for k in sorted(err, key=lambda k: -err[k][0])[:3]:
        print(f"  {k}: |g - g64| / |g64| = {err[k][0]:.2e}, max|g - g64| / max|g64| = {err[k][1]:.2e}")
    for k in sorted(err):
        if k.startswith(LOWER) and not lower:
            print(f"  {k}: |g - g64| / |g64| = {err[k][0]:.2e} (|g64| = {np.linalg.norm(g64[k]):.2e})")
    bad = {k: e for k, e in err.items() if not (e[0] <= 1e-4 and e[1] <= 1e-3) and (lower or not k.startswith(LOWER))}
    assert not bad, sorted((k, f"{e[0]:.1e}", f"{e[1]:.1e}") for k, e in bad.items())
    return g, g64


@pytest.mark.parametrize("B,T,frames", CASES, ids=["3x40", "8x500"])
@pytest.mark.parametrize("seed,gain", [(0, 1.0), (1, 1.0), (0, 4.0)], ids=["seed0", "seed1", "gain4"])
def test_gradients_against_float64(B, T, frames, seed, gain):
    """Generator records at the generator's own scale: the network input reaches 1e8 (band energies of int16-scale
    audio x 30), the fc and conv1 outputs 1e6 and more, and conv2's pre-activations are differences of such terms, whose
    fp32 rounding alone moves tanh'(pre) wherever pre is of order one.  The gradients of fc, conv1 and conv2 depend on
    exactly those units, so no fp32 forward pass gets them to the bar; their errors are printed.  The other 24 tensors
    are held to it."""
    rec = windows(B, T, 100 + B)
    if B == 3:
        rec[:2] = np.load(os.path.join(GOLDEN, "train.npz"))["records"][:, :T]
    check_against_float64(synth_state_dict(seed, gain), rec, frames, f"{B}x{T} seed {seed} gain {gain}", lower=False)


@pytest.mark.parametrize("B,T,frames", CASES, ids=["3x40", "8x500"])
def test_gradients_against_float64_unsaturated(B, T, frames):
    """Records of moderate scale: conv2 stays out of saturation, and all 30 tensors are held to the bar."""
    rec = moderate_records(B, T, 110 + B)
    sd = synth_state_dict(1)
    m = O.model(sd)
    with torch.no_grad():
        y = m.fc(torch.from_numpy(O.features(rec))).permute(0, 2, 1)
        pre = m.conv2[0](m.conv1(y)[:, :, :-4])[:, :, :-2]
    sat = float((torch.tanh(pre).abs() == 1).float().mean())
    print(f"\nconv2 outputs at +-1 in fp32: {sat:.2%}")
    assert sat < 0.01
    check_against_float64(sd, rec, frames, f"{B}x{T} quiet")


def test_saturated_outputs_are_finite():
    """Bands whose fc_rb pre-activation is 30 give r = 1 exactly in fp32, where torch's float32 autograd of
    CustomLoss multiplies an infinite d/dr by a zero sigmoid derivative: NaN.  The trainer's gradient is finite there
    and within the bar of float64's."""
    sd = synth_state_dict(0, 4.0)
    sd["fc_rb.0.bias"] = sd["fc_rb.0.bias"].copy()
    sd["fc_rb.0.bias"][:4] = 30.0
    rec = moderate_records(3, 40, 103)
    _, g32 = O.grads(sd, rec, None, torch.float32, "cuda")
    assert any(np.isnan(v).any() for v in g32.values()), "no NaN in torch's float32 autograd: the outputs do not saturate"
    check_against_float64(sd, rec, None, "saturated r")


def test_padding_determinism_and_entries():
    sd = synth_state_dict(1)
    rec = windows(3, 40, 104)
    frames = [40, 23, 31]
    eng = trainer(sd, 3, 40)
    a = eng.train_grad(rec, frames)
    ga = eng.train_export("gradient")
    junk = rec.copy()
    junk[1, 23:] = np.nan
    junk[2, 31:] = 1e30
    b = eng.train_grad(junk, frames)
    assert np.array_equal(a.view(np.int64), b.view(np.int64))
    assert np.array_equal(ga.view(np.int32), eng.train_export("gradient").view(np.int32))
    # device entry, on two different streams
    d_rec = torch.from_numpy(rec).cuda()
    for s in (torch.cuda.Stream(), torch.cuda.Stream()):
        d_sums = torch.empty((3, 4), dtype=torch.float64, device="cuda")
        eng.train_grad_device(d_rec.data_ptr(), 40 * 138, 40, frames, d_sums.data_ptr(), s.cuda_stream)
        eng.check(s.cuda_stream)
        assert np.array_equal(d_sums.cpu().numpy().view(np.int64), a.view(np.int64))
        assert np.array_equal(eng.train_export("gradient").view(np.int32), ga.view(np.int32))
    eng.close()


def test_launch_count_does_not_grow_with_T():
    sd = synth_state_dict(0)
    counts = []
    for T in (40, 500):
        eng = trainer(sd, 2, T)
        n0 = eng.launches
        eng.train_grad(windows(2, T, 105))
        counts.append((eng.launches_per_call(T), eng.launches - n0))
        eng.close()
    assert counts[0] == counts[1] and counts[0][0] == counts[0][1], counts


def test_adam_against_torch():
    """Three pnb_train_adam steps against torch.optim.Adam stepping float32 CPU parameters whose .grad is the engine's
    exported gradient.  Each step starts both from torch's state (pnb_train_import), so each is compared on its own.
    The moments are bit-identical.  The weights are bit-identical to torch's formula evaluated with the correctly rounded
    square root of v, and equal torch's own weights wherever torch's CPU sqrt of v is correctly rounded: torch's CPU sqrt
    (MKL's vectorised sqrt) is not everywhere, the GPU's is (DESIGN.md section 1 gives the measured counts)."""
    sd = synth_state_dict(0)
    rec = windows(4, 30, 106, quiet=16)
    eng = trainer(sd, 4, 30)
    lr = 1e-3
    p = torch.from_numpy(eng.train_export("weights").copy()).requires_grad_(True)
    opt = torch.optim.Adam([p], lr=lr)
    for step in range(1, 4):
        eng.train_grad(rec)
        p_old = p.detach().numpy().copy()
        st = opt.state[p]
        if step > 1:
            for name, key in (("weights", None), ("m", "exp_avg"), ("v", "exp_avg_sq")):
                eng.train_import(name, p_old if key is None else st[key].numpy())
        p.grad = torch.from_numpy(eng.train_export("gradient"))
        opt.step()
        eng.train_adam(lr, step)
        eng.wait()
        st = opt.state[p]
        for name, key in (("m", "exp_avg"), ("v", "exp_avg_sq")):
            assert np.array_equal(eng.train_export(name).view(np.int32), st[key].numpy().view(np.int32)), (step, name)
        mine, theirs = eng.train_export("weights"), p.detach().numpy()
        v, m = st["exp_avg_sq"].numpy(), st["exp_avg"].numpy()
        f32 = np.float32
        den = ((np.sqrt(v) / f32((1 - 0.999 ** step) ** 0.5)).astype(f32) + f32(1e-8)).astype(f32)
        ieee = (p_old + ((f32(-(lr / (1 - 0.9 ** step))) * m).astype(f32) / den).astype(f32)).astype(f32)
        rounded = torch.sqrt(st["exp_avg_sq"]).numpy() == np.sqrt(v)
        print(f"\nstep {step}: {np.count_nonzero(mine != theirs)} of {mine.size} weights differ from torch's; torch's sqrt "
              f"is not correctly rounded at {np.count_nonzero(~rounded)}; {np.count_nonzero(mine != ieee)} differ from "
              f"torch's formula with a correctly rounded sqrt, {np.count_nonzero((mine != theirs) & rounded)} from torch "
              f"where its sqrt is")
        assert np.array_equal(mine.view(np.int32), ieee.view(np.int32))
        assert not np.any((mine != theirs) & rounded)
    eng.close()


def test_nonfinite_gradient_skips_the_step():
    """NaN inside a valid frame: the host gradient call reports PNB_ERR_DOMAIN, the next Adam step leaves weights, m and
    v as they were, the report sticks until pnb_reset, which keeps them; the next clean step applies."""
    sd = synth_state_dict(0)
    rec = windows(2, 20, 107, quiet=16)
    eng = trainer(sd, 2, 20)
    eng.train_grad(rec)
    eng.train_adam(1e-3, 1)
    w, m, v = (eng.train_export(k) for k in ("weights", "m", "v"))
    bad = rec.copy()
    bad[0, 5, 3] = np.nan
    with pytest.raises(api.PnbError, match=r"\(-5\)"):
        eng.train_grad(bad)
    eng.train_adam(1e-3, 2)
    with pytest.raises(api.PnbError, match=r"\(-5\)"):
        eng.wait()
    for k, a in (("weights", w), ("m", m), ("v", v)):
        assert np.array_equal(eng.train_export(k).view(np.int32), a.view(np.int32)), k
    eng.reset()
    for k, a in (("weights", w), ("m", m), ("v", v)):
        assert np.array_equal(eng.train_export(k).view(np.int32), a.view(np.int32)), k
    eng.train_grad(rec)
    eng.train_adam(1e-3, 2)
    eng.wait()
    assert not np.array_equal(eng.train_export("weights"), w)
    eng.close()


def test_closing_the_loop(tmp_path):
    """200 Adam steps at lr 1e-3 on 8 x 100 generator windows lower the loss; the trained weights score the same on the
    training engine and on a fresh network-only engine from the exported blob, within 1e-3 of the trainer's own
    exact-activation loss, and load in a tensor-path engine.  The audio is quiet (/ 64) so that the deployed arithmetic
    stays where the reference's tansig_approx is defined (|x| < 8.5e7): at the generator's own scale the band energies
    x 30 reach 3e8 at the network input already."""
    rec = generator_records(8, 100, 108, quiet=64).cpu().numpy()
    eng = trainer(synth_state_dict(2), 8, 100)
    losses = []
    for step in range(1, 201):
        losses.append(loss_terms(eng.train_grad(rec).sum(0))["total"])
        eng.train_adam(1e-3, step)
    eng.wait()
    first, last = np.mean(losses[:20]), np.mean(losses[-20:])
    print(f"\nloss: first 20 steps {first:.6f}, last 20 {last:.6f}")
    assert last < first
    exact = loss_terms(eng.train_grad(rec).sum(0))["total"]
    s_train, _ = eng.score_records(rec)
    blob = str(tmp_path / "trained.pnbw")
    PackedModel.from_flat(eng.train_export("weights")).save_blob(blob)
    eng.close()
    bm = api.BlobModel(blob)
    fresh = api.Engine(8, 100, bm, api.NETWORK_ONLY)
    s_fresh, _ = fresh.score_records(rec)
    fresh.close()
    assert np.array_equal(s_train.view(np.int64), s_fresh.view(np.int64))
    deployed = loss_terms(s_fresh.sum(0))["total"]
    print(f"deployed (tansig) loss {deployed:.9f}, trainer (exact) loss {exact:.9f}, rel {abs(deployed - exact) / exact:.2e}")
    assert abs(deployed - exact) <= 1e-3 * exact
    tc = api.Engine(8, 100, bm, api.NN_TENSOR | api.NETWORK_ONLY)
    s_tc, _ = tc.score_records(rec)
    tc.close()
    bm.free()
    assert np.all(np.isfinite(s_tc))


def test_refusals():
    L = api.load_library()
    pm = pack_state_dict(synth_state_dict(0))
    h = C.c_void_p()
    for bad in (api.NN_TENSOR, api.CONV_WIDE | api.NN_TENSOR, api.TRAIN_DATA, api.TRAIN_DATA | api.TRAIN_AUDIO,
                api.POSTFILTER, api.SIGNAL_ONLY):
        assert L.pnb_create(C.byref(h), 2, 10, C.addressof(pm.as_c_model()), api.TRAIN_NETWORK | bad, 0) == -1
    rec = np.zeros((2, 10, 138), np.float32)
    other = api.Engine(2, 10, pm, api.NETWORK_ONLY)
    with pytest.raises(api.PnbError, match="PNB_TRAIN_NETWORK"):
        other.train_grad(rec)
    with pytest.raises(api.PnbError, match="PNB_TRAIN_NETWORK"):
        other.train_adam(1e-3, 1)
    with pytest.raises(api.PnbError, match="PNB_TRAIN_NETWORK"):
        other.train_export("weights")
    other.close()
    eng = api.Engine(2, 10, pm, api.TRAIN_NETWORK)
    n0 = eng.launches
    sums = np.empty((2, 4), np.float64)
    for frames in ([0, 10], [11, 10], [-1, 3]):
        with pytest.raises(api.PnbError, match="frames"):
            eng.train_grad(rec, frames)
    with pytest.raises(api.PnbError, match="n_frames"):
        eng.train_grad(np.zeros((2, 11, 138), np.float32))
    assert L.pnb_train_grad_host(eng.h, None, 1380, 10, None, sums.ctypes.data) == -1
    assert L.pnb_train_grad_host(eng.h, rec.ctypes.data, 1379, 10, None, sums.ctypes.data) == -1
    assert L.pnb_train_grad_host(eng.h, rec.ctypes.data, 1380, 10, None, None) == -1
    for lr in (float("nan"), float("inf"), -1e-3):
        with pytest.raises(api.PnbError, match="lr"):
            eng.train_adam(lr, 1)
    w = eng.train_export("weights")
    with pytest.raises(api.PnbError, match="bytes"):
        eng.train_import("weights", w[:-1])
    with pytest.raises(api.PnbError, match="gradient"):
        eng.train_import("gradient", w)
    assert eng.launches == n0
    eng.close()
