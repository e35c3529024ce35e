"""The trainer's fc, conv1 and conv2 on the generator's own records, checked at the trainer's own forward values.

On int16-scale records conv2's pre-activations are differences of products of order 1e6, so any fp32 forward pass moves
tanh'(pre) by percents, and float64 autograd of the records (test_gpu_train.py) cannot hold the gradients of fc, conv1
and conv2 to a bar.  Here the two questions are taken apart:
* the forward: each of the three layers against float64 at its own fp32 inputs (the staged records for fc, the tapped
  fc output for conv1, the tapped conv1 output for conv2), element by element, within the rounding bound of an fp32
  FMA chain;
* the backward: all 30 gradient tensors against float64 autograd at the trainer's own forward values
  (train_oracle.grads_at, through the PNB_TAP_TRAIN_* taps), with the bars of test_gpu_train.py.
The same for the forward and backward halves (pnb_train_forward_device / pnb_train_backward_device), seeded with a
torch loss's dL/d(out) at their own fp32 output: their output against float64 at the own values, and dL/dx held to the
gradients' bars too.
What remains is the accuracy of the trainer's own arithmetic, which is what a defect in its kernels would move."""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as Fn

from conftest import GOLDEN
from percepnet_b200 import api
from percepnet_b200.eval_records import loss_terms
from percepnet_b200.weights import N_PARAMS, PackedModel, pack_state_dict, synth_state_dict, unpack_state_dict
from test_gpu_torch_module import arbitrary_loss
from test_gpu_train import grads_of, ragged_frames, trainer, windows
import train_oracle as O

pytestmark = pytest.mark.gpu

U = 2.0 ** -24                   # fp32 unit roundoff (round to nearest)
FLT_MIN = float(np.finfo(np.float32).tiny)
DEVICE = "cuda"                  # of the float64 references
TAPS = ("train_fc", "train_c1", "train_c2pre")
# fp32 FMA chains of K products from zero, then the bias: K + 1 roundings, each within U of a value <= A + |b|
K = {"fc": 70, "conv1": 5 * 128, "conv2": 3 * 512}


def run_trainer(sd, rec, frames):
    """One gradient call: (loss, gradients by name, the fc / conv1 / conv2-pre taps [T][B][w])."""
    B, T = rec.shape[:2]
    eng = trainer(sd, B, T)
    sums = eng.train_grad(rec, frames)
    g = grads_of(eng)
    taps = [eng.read_tap(name, T, B) for name in TAPS]
    eng.close()
    return loss_terms(sums.sum(0))["total"], g, taps


def run_halves(sd, rec, engine):
    """One forward and one backward of the halves on the first B rows of an engine of shape `engine` (active B), x the
    records' features, dL/d(out) arbitrary_loss's at the fp32 out: (out, dout, gradients and dL/dx by name, taps)."""
    B, T = rec.shape[:2]
    eng = trainer(sd, *engine)
    if engine[0] != B:
        eng.set_active(B)
    x = torch.from_numpy(O.features(rec)).cuda()
    out = torch.empty((B, T, 68), device="cuda")
    eng.train_forward_device(x.data_ptr(), T * 70, T, 0, out.data_ptr(), T * 68)
    taps = [eng.read_tap(name, T, B) for name in TAPS]
    o = out.clone().requires_grad_(True)
    arbitrary_loss(B)(o, None).backward()
    dout = o.grad.detach().contiguous()
    dx = torch.empty((B, T, 70), device="cuda")
    grad = torch.empty(N_PARAMS, device="cuda")
    eng.train_backward_device(dout.data_ptr(), T * 68, dx.data_ptr(), T * 70, grad.data_ptr())
    eng.wait()
    g = unpack_state_dict(PackedModel.from_flat(grad.cpu().numpy()))
    g["dL/dx"] = dx.cpu().numpy()
    eng.close()
    return out.cpu().numpy(), dout.cpu().numpy().astype(np.float64), g, taps


def staged_input(rec, frames):
    """The trainer's network input {30 rec[0..67], rec[68], rec[69]} in fp32, zero past each window's end: [B][T][70]."""
    x = O.features(rec)
    if frames is not None:
        for b, f in enumerate(frames):
            x[b, f:] = 0
    return x


def forward_errors(sd, rec, frames, taps, chunk=16):
    """Each layer's fp32 output against float64 at its own fp32 inputs, on every hop (those past a window's end too):
    (worst |err| / bound, p99.9 of |err| / sum|w||x|) per layer, bound = (K + 2) 2^-24 (sum|w||x| + |b|)."""
    fc32, c1_32, c2p32 = taps
    dev = dict(device=DEVICE, dtype=torch.float64)
    w = {k: torch.tensor(sd[f"{k}.0.weight"], **dev) for k in K}
    b = {k: torch.tensor(sd[f"{k}.0.bias"], **dev) for k in K}
    x = staged_input(rec, frames)
    worst = {k: 0.0 for k in K}
    rel = {k: [] for k in K}
    for c0 in range(0, rec.shape[0], chunk):
        part = slice(c0, min(rec.shape[0], c0 + chunk))
        tap = lambda a: torch.from_numpy(np.ascontiguousarray(a[:, part].transpose(1, 2, 0))).to(**dev)  # [b][w][T]
        xin = torch.from_numpy(x[part]).to(**dev)
        fc_t, c1_t, c2p_t = tap(fc32), tap(c1_32), tap(c2p32)
        layers = {  # (own fp32 output, float64 pre-activation, sum |w||x|) as [b][w][T]
            "fc": (fc_t, Fn.linear(xin, w["fc"], b["fc"]).transpose(1, 2),
                   Fn.linear(xin.abs(), w["fc"].abs()).transpose(1, 2)),
            "conv1": (c1_t, Fn.conv1d(fc_t, w["conv1"], b["conv1"], padding=4)[..., :-4],
                      Fn.conv1d(fc_t.abs(), w["conv1"].abs(), padding=4)[..., :-4]),
            "conv2": (c2p_t, Fn.conv1d(c1_t, w["conv2"], b["conv2"], padding=2)[..., :-2],
                      Fn.conv1d(c1_t.abs(), w["conv2"].abs(), padding=2)[..., :-2]),
        }
        for k, (own, pre, A) in layers.items():
            want = pre if k == "conv2" else pre.clamp_min(0)      # fc and conv1 are tapped after their ReLU
            err = (own - want).abs()
            bound = (K[k] + 2) * U * (A + b[k].abs()[None, :, None])
            worst[k] = max(worst[k], float((err / bound).max()))
            nz = A > 0
            rel[k].append((err[nz] / A[nz]).float().cpu().numpy())
    return {k: (worst[k], float(np.quantile(np.concatenate(rel[k]), 0.999))) for k in K}


def kernel_dtanh(c2p32):
    """kEpiDTanh's factor as the kernel evaluates it, in fp32: 4 e / ((1 + e)(1 + e)), e = expf(-2 |a|)."""
    a = np.abs(np.asarray(c2p32, np.float32))
    with np.errstate(under="ignore"):
        e = np.exp(np.float32(-2) * a)
        return (np.float32(4) * e / ((np.float32(1) + e) * (np.float32(1) + e))).astype(np.float64)


def gradient_errors(g, g64):
    err = {}
    for k, w in g64.items():
        assert np.all(np.isfinite(g[k])), k
        d = np.asarray(g[k], np.float64) - w
        err[k] = (np.linalg.norm(d) / max(np.linalg.norm(w), 1e-300), np.abs(d).max() / max(np.abs(w).max(), 1e-300))
    return err


def misses(err):
    return sorted(k for k, e in err.items() if not (e[0] <= 1e-4 and e[1] <= 1e-3))


def check_at_own_inputs(sd, rec, frames, label, chunk=16, halves=None):
    """The forward bound on fc, conv1 and conv2, and the gradients' bars at the own forward values, of a gradient call
    (halves None) or of the forward and backward halves on the first B rows of an engine of shape `halves` (frames
    None), whose out is also held within 1e-5 of float64's at the own values and whose dL/dx is held like a gradient."""
    B, T = rec.shape[:2]
    if halves is None:
        loss, g, taps = run_trainer(sd, rec, frames)
        seed = {}
    else:
        out, dout, g, taps = run_halves(sd, rec, halves)
        seed = dict(dout=dout, want_dx=True)
    print(f"\n{label}:")
    fwd = forward_errors(sd, rec, frames, taps, chunk)
    for k, (worst, p999) in fwd.items():
        print(f"  forward {k:5s} (K = {K[k]:4d}): p99.9 |err| / sum|w||x| = {p999:.2e}, worst |err| / bound = {worst:.3f}")
    assert all(worst <= 1 for worst, _ in fwd.values()), fwd

    c2p32 = taps[2]
    if frames is not None:
        counted = np.arange(T)[:, None] < np.asarray(frames)[None, :]
    else:
        counted = np.ones((T, B), bool)
    lo = np.abs(c2p32[counted]).min(0)        # the smallest |c2p| of each unit over the counted hops
    print(f"  smallest |c2p| per unit over counted hops: min {lo.min():.3g}, median {np.median(lo):.3g}, "
          f"max {lo.max():.3g}; {np.count_nonzero(lo > 43.7)} of 512 units above 43.7 (fp32 tanh' subnormal there)")

    def reference(**kw):
        L64, g64, out64, dx64 = O.grads_at(sd, rec, frames, *taps, chunk=chunk, device=DEVICE, **seed, **kw)
        if dx64 is not None:
            g64["dL/dx"] = dx64
        return L64, g64, out64

    L64, g64, out64 = reference()
    if halves is None:
        print(f"  loss {loss:.9e}, float64 at own inputs {L64:.9e}, rel {abs(loss - L64) / abs(L64):.2e}")
        assert abs(loss - L64) <= 1e-6 * abs(L64)
    else:
        d = float(np.abs(out - out64).max())
        print(f"  max|out - out64| at own inputs {d:.2e}")
        assert d <= 1e-5
    err = gradient_errors(g, g64)
    for k in sorted(err, key=lambda k: -err[k][0])[:3]:
        print(f"  {k}: |g - g64| / |g64| = {err[k][0]:.2e}, max|g - g64| / max|g64| = {err[k][1]:.2e}")
    if "dL/dx" in err:
        print(f"  dL/dx: |g - g64| / |g64| = {err['dL/dx'][0]:.2e}, max|g - g64| / max|g64| = {err['dL/dx'][1]:.2e}")
    zero = sorted(k for k in g64 if not np.any(g64[k]))
    if zero:
        print(f"  float64's gradient is exactly zero for {zero}; the trainer's max |g| there "
              f"{max(np.abs(g[k]).max() for k in zero):.1e}")
    bad = misses(err)
    if bad:
        # fp32 cannot hold a tanh' below FLT_MIN (|a| > 43.7: expf(-2|a|) is subnormal, and zero beyond 51.9).  Where
        # float64's factor is below FLT_MIN, the kernel's own fp32 factor is taken as one more own input; a tensor that
        # then meets the bar missed it for that reason alone.
        a = np.abs(c2p32.astype(np.float64))
        e = np.exp(-2 * a)
        exact = 4 * e / ((1 + e) * (1 + e))
        tiny = exact < FLT_MIN
        print(f"  {bad} miss the bar; {np.count_nonzero(tiny)} of {tiny.size} tanh' factors below FLT_MIN: "
              f"the kernel's fp32 factor taken there")
        assert tiny.any(), f"{label}: {bad} miss the bar at own inputs"
        _, g64, _ = reference(dtanh=np.where(tiny, kernel_dtanh(c2p32), exact))
        err = gradient_errors(g, g64)
        for k in bad:
            print(f"  {k} with own factors below FLT_MIN: |g - g64| / |g64| = {err[k][0]:.2e}, "
                  f"max|g - g64| / max|g64| = {err[k][1]:.2e}")
        still = misses(err)
        assert not still, sorted((k, f"{err[k][0]:.1e}", f"{err[k][1]:.1e}") for k in still)


_records = {}


def records(B, T, seed):
    if (B, T, seed) not in _records:
        _records[(B, T, seed)] = windows(B, T, seed)
    return _records[(B, T, seed)]


@pytest.mark.parametrize("seed,gain", [(0, 1.0), (1, 1.0), (0, 4.0), (1, 4.0)],
                         ids=["seed0", "seed1", "seed0-gain4", "seed1-gain4"])
def test_own_inputs_3x40(seed, gain):
    """3 x 40, window 1 ending at hop 23, windows 0 and 1 the two tests/golden/train.npz windows."""
    rec = records(3, 40, 203).copy()
    rec[:2] = np.load(os.path.join(GOLDEN, "train.npz"))["records"][:, :40]
    check_at_own_inputs(synth_state_dict(seed, gain), rec, [40, 23, 40], f"3x40 seed {seed} gain {gain}")


@pytest.mark.parametrize("B,T,gain", [(10, 500, 1.0), (10, 500, 4.0), (128, 2000, 1.0)],
                         ids=["10x500", "10x500-gain4", "128x2000"])
def test_own_inputs_at_training_shapes(B, T, gain):
    """The CLI's batch (10 x 500, ragged windows) at gains 1 and 4, and 128 x 2000 full windows: the longest
    weight-gradient sums, over rows whose x reaches 3e8 and fc / conv1 outputs 1e6."""
    rec = records(B, T, 210 + B)
    frames = ragged_frames(B, T, 220 + B) if T == 500 else None
    check_at_own_inputs(synth_state_dict(0, gain), rec, frames, f"{B}x{T} seed 0 gain {gain}")


@pytest.mark.parametrize("gain", [1.0, 4.0], ids=["gain1", "gain4"])
def test_halves_own_inputs_3x40(gain):
    """The halves on 3 x 40: the two tests/golden/train.npz windows and one generator window."""
    rec = records(3, 40, 203).copy()
    rec[:2] = np.load(os.path.join(GOLDEN, "train.npz"))["records"][:, :40]
    check_at_own_inputs(synth_state_dict(0, gain), rec, None, f"halves 3x40 gain {gain}", halves=(3, 40))


@pytest.mark.parametrize("B,T,engine", [(10, 500, (16, 600)), (32, 500, (32, 500))], ids=["10x500-of-16x600", "32x500"])
def test_halves_own_inputs_at_training_shapes(B, T, engine):
    """The halves on the CLI's batch as the active 10 rows of a 16 x 600 engine in a 500-hop call, and on 32 x 500.
    128 x 2000 is left to test_own_inputs_at_training_shapes: its long weight-gradient sums are backward_half's, which
    the halves share with the gradient call; the halves' own kernels (stage, seed, dL/dx, stores) are per row."""
    check_at_own_inputs(synth_state_dict(0), records(B, T, 210 + B), None, f"halves {B}x{T} on {engine[0]}x{engine[1]}",
                        halves=engine)


def test_train_taps_follow_the_last_gradient_call():
    """The taps are [F][n][w] of the last gradient call on the active rows (a 3-row, 10-hop call on a 4 x 12 engine),
    the values grads_at pins (fc within the bound above of the records' own fc), unchanged by Adam, accumulate and
    finish; and refused on any other engine, before the first gradient call, and into a buffer one byte short."""
    L = api.load_library()
    sd = synth_state_dict(0)
    pm = pack_state_dict(sd)
    for flags in (api.NETWORK_ONLY | api.KEEP_TAPS, api.NN_FP32 | api.KEEP_TAPS):
        other = api.Engine(2, 10, pm, flags)
        for name in TAPS:
            with pytest.raises(api.PnbError, match="PNB_TRAIN_NETWORK"):
                other.read_tap(name, 10, 2)
        other.close()
    eng = trainer(sd, 4, 12)
    for name in TAPS:
        with pytest.raises(api.PnbError, match="pnb_train_grad"):
            eng.read_tap(name, 10, 3)
    eng.set_active(3)
    rec = records(3, 10, 230)
    frames = [10, 4, 7]
    eng.train_grad(rec, frames)
    taps = [eng.read_tap(name, 10, 3) for name in TAPS]
    for name, t in zip(TAPS, taps):
        buf = np.empty(t.nbytes - 1, np.uint8)
        assert L.pnb_read_tap(eng.h, api.TAPS[name][0], buf.ctypes.data, buf.nbytes) == -1
        assert f"needs {t.nbytes} bytes" in L.pnb_last_error().decode()
    eng.train_accumulate()
    eng.train_finish()
    eng.train_adam(1e-3, 1)
    eng.wait()
    for name, t in zip(TAPS, taps):
        assert np.array_equal(eng.read_tap(name, 10, 3).view(np.int32), t.view(np.int32)), name
    eng.close()
    x = staged_input(rec, frames)
    fc64 = np.maximum(x.astype(np.float64) @ sd["fc.0.weight"].T.astype(np.float64) + sd["fc.0.bias"], 0)
    A = np.abs(x.astype(np.float64)) @ np.abs(sd["fc.0.weight"].T.astype(np.float64)) + np.abs(sd["fc.0.bias"])
    assert np.all(np.abs(taps[0].transpose(1, 0, 2) - fc64) <= (K["fc"] + 2) * U * A)
    assert np.any(taps[0] > 0) and np.any(taps[1] > 0) and np.all(np.isfinite(taps[2]))
