"""The trainer's truth on the CPU: the torch restatement of rnn_train.py (train_oracle) against the reference's own
classes, the closed-form loss gradient against autograd, the layout round trips of the exported vectors, and the Adam
restatement against torch.optim.Adam."""
import importlib.util
import os
import sys
import types

import numpy as np
import pytest
import torch

from conftest import REFERENCE_TREE
from percepnet_b200.weights import N_PARAMS, PackedModel, pack_state_dict, synth_state_dict, unpack_state_dict
import train_oracle as O


def bits_equal(a, b):
    a, b = np.atleast_1d(np.asarray(a)), np.atleast_1d(np.asarray(b))
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def records(B, T, seed):
    rng = np.random.RandomState(seed)
    rec = rng.rand(B, T, 138).astype(np.float32)
    rec[..., :68] *= np.float32(0.05)
    return rec


def load_reference():
    path = os.path.join(REFERENCE_TREE, "rnn_train.py")
    if not os.path.exists(path):
        pytest.skip("the reference tree is absent")
    stubs = {}
    for name in ("h5py", "tensorboardX", "matplotlib", "matplotlib.pyplot"):
        if name not in sys.modules:
            mod = types.ModuleType(name)
            mod.SummaryWriter = object
            mod.switch_backend = lambda *a, **k: None
            stubs[name] = mod
    sys.modules.update(stubs)
    try:
        spec = importlib.util.spec_from_file_location("ref_rnn_train", path)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
    finally:
        for name in stubs:
            sys.modules.pop(name, None)
    return mod


def test_oracle_is_rnn_train():
    """Outputs, CustomLoss and every autograd gradient of the restatement equal the reference's PercepNet and CustomLoss
    bit for bit in float32, on the same synth_state_dict weights."""
    ref = load_reference()
    sd = synth_state_dict(0)
    rec = records(2, 24, 5)
    x = torch.from_numpy(O.features(rec))
    y = torch.from_numpy(np.ascontiguousarray(rec[..., 70:]))
    mine, theirs = O.model(sd), ref.PercepNet()
    theirs.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()})
    o1, o2 = mine(x), theirs(x)
    l1, l2 = O.loss(o1, y), ref.CustomLoss()(o2, y)
    l1.backward()
    l2.backward()
    assert bits_equal(o1.detach().numpy(), o2.detach().numpy())
    assert bits_equal(l1.detach().numpy(), l2.detach().numpy())
    g2 = dict(theirs.named_parameters())
    for k, p in mine.named_parameters():
        assert bits_equal(p.grad.numpy(), g2[k].grad.numpy()), k


def test_closed_form_loss_gradient():
    """dloss_dpre equals float64 autograd of CustomLoss at the sigmoid inputs wherever autograd is finite, and is finite
    (the limit) where a prediction is exactly 0 or 1."""
    rng = np.random.RandomState(3)
    a = torch.tensor(rng.randn(4, 7, 68) * 6, dtype=torch.float64, requires_grad=True)
    y = torch.tensor(rng.rand(4, 7, 68), dtype=torch.float64)
    p = torch.sigmoid(a)
    O.loss(p, y).backward()
    want = a.grad.numpy()
    got = O.dloss_dpre(p.detach().numpy(), y.numpy(), 4 * 7 * 34)
    assert np.all(np.isfinite(want))
    np.testing.assert_allclose(got, want, rtol=1e-12, atol=1e-300)
    edge = np.zeros((1, 1, 68))
    edge[..., 1::2] = 1.0
    d = O.dloss_dpre(edge, np.full((1, 1, 68), 0.5), 34)
    assert np.all(np.isfinite(d)) and np.all(d == 0)


def test_grads_at_own_values_is_grads():
    """grads_at fed float64's own forward values (fc and conv1 outputs, conv2's pre-activation) is grads, loss and all
    30 tensors within 1e-12, with the taps cut into chunks of windows like the records; and so is it seeded with
    dL/d(out) of that loss instead, with dL/dx and out those of plain float64 autograd of the model within 1e-12."""
    sd = synth_state_dict(0)
    rec = records(3, 24, 7)
    frames = [24, 13, 24]
    L, g = O.grads(sd, rec, frames)
    fc, c1, c2p = O.forward_taps(sd, rec, frames)
    assert fc.shape == (24, 3, 128) and c1.shape == (24, 3, 512) and c2p.shape == (24, 3, 512)
    La, ga, _, dxa = O.grads_at(sd, rec, frames, fc, c1, c2p, chunk=2)
    assert abs(La - L) <= 1e-12 * abs(L) and dxa is None
    for k in g:
        assert np.linalg.norm(ga[k] - g[k]) <= 1e-12 * np.linalg.norm(g[k]), k

    m = O.model(sd, torch.float64)
    x, y, fr = O._inputs(rec, np.asarray(frames), slice(0, 3), frames, torch.float64, "cpu")
    x.requires_grad_(True)
    out = m(x)
    dout, = torch.autograd.grad(O.loss(out, y, fr), out, retain_graph=True)
    O.loss(out, y, fr).backward()
    Ld, gd, outd, dxd = O.grads_at(sd, rec, frames, fc, c1, c2p, chunk=2, dout=dout.numpy(), want_dx=True)
    assert Ld is None and outd.shape == (3, 24, 68) and dxd.shape == (3, 24, 70)
    for k in g:
        assert np.linalg.norm(gd[k] - g[k]) <= 1e-12 * np.linalg.norm(g[k]), k
    dx = x.grad.numpy()
    assert np.linalg.norm(dxd - dx) <= 1e-12 * np.linalg.norm(dx)
    want = out.detach().numpy()
    assert np.abs(outd - want).max() <= 1e-12 * np.abs(want).max()


def test_grads_at_takes_tanh_prime_at_the_given_preactivation():
    """Two conv2 pre-activations that differ at one unit j of one hop only, both deep in saturation (tanh = 1 exactly in
    float64, tanh' of 1.7e-17 and 4.6e-17): every value of the network is the same, only tanh' at that unit moves.  So the
    24 tensors above conv2 are bit-identical, conv2's bias gradient moves at unit j alone, and conv2's weight gradient in
    row j alone, by that move times the conv1 outputs the unit sees (hops t - 2 .. t of its window)."""
    sd = synth_state_dict(0)
    rec = records(2, 24, 8)
    fc, c1, c2p = O.forward_taps(sd, rec)
    j, t, b = 37, 9, 1
    a = c2p.copy()
    a[:, :, j] = 20.0
    p = a.copy()
    p[t, b, j] = 19.5
    assert np.tanh(20.0) == 1.0 and np.tanh(19.5) == 1.0
    _, ga, _, _ = O.grads_at(sd, rec, None, fc, c1, a)
    _, gp, _, _ = O.grads_at(sd, rec, None, fc, c1, p)
    for k in ga:
        if not k.startswith(("fc.", "conv1.", "conv2.")):
            assert bits_equal(ga[k], gp[k]), k
    moved = np.flatnonzero(ga["conv2.0.bias"] != gp["conv2.0.bias"])
    assert moved.tolist() == [j]
    delta = gp["conv2.0.bias"][j] - ga["conv2.0.bias"][j]
    assert delta != 0
    dw = gp["conv2.0.weight"] - ga["conv2.0.weight"]       # [out 512][in 512][tap 3]: tap k sees hop t - 2 + k
    assert not np.any(np.delete(dw, j, axis=0))
    want = delta * np.stack([c1[t - 2 + k, b] for k in range(3)], -1)
    np.testing.assert_allclose(dw[j], want, rtol=1e-9, atol=1e-9 * np.abs(want).max())


def test_layout_round_trips():
    sd = synth_state_dict(1, gain=2.0)
    back = unpack_state_dict(pack_state_dict(sd))
    assert sorted(back) == sorted(sd)
    for k in sd:
        assert bits_equal(back[k], sd[k]), k
    pm = pack_state_dict(sd)
    v = pm.flat()
    assert v.size == N_PARAMS and v.dtype == np.float32
    again = PackedModel.from_flat(v)
    assert sorted(again.arrays) == sorted(pm.arrays)
    for k in pm.arrays:
        assert bits_equal(again.arrays[k], pm.arrays[k]), k
    with pytest.raises(ValueError):
        PackedModel.from_flat(v[:-1])


def test_adam_restatement_is_torch():
    """Five steps of adam_step against torch.optim.Adam (defaults, CPU float32), each from torch's state: the moments
    bit for bit, the weights bit for bit wherever torch's CPU sqrt of v is the correctly rounded square root (MKL's
    vectorised sqrt is not everywhere; adam_step and the GPU use the correctly rounded one)."""
    rng = np.random.RandomState(9)
    p0 = (rng.randn(10007) * 0.1).astype(np.float32)
    t = torch.from_numpy(p0.copy()).requires_grad_(True)
    opt = torch.optim.Adam([t], lr=1e-3)
    p, m, v = p0.copy(), np.zeros_like(p0), np.zeros_like(p0)
    for step in range(1, 6):
        g = (rng.randn(p0.size) * 10.0 ** rng.uniform(-6, 0)).astype(np.float32)
        t.grad = torch.from_numpy(g.copy())
        opt.step()
        p, m, v = O.adam_step(p, g, m, v, 1e-3, step)
        st = opt.state[t]
        rounded = torch.sqrt(st["exp_avg_sq"]).numpy() == np.sqrt(v)
        assert not np.any((t.detach().numpy() != p) & rounded), step
        assert bits_equal(st["exp_avg"].numpy(), m) and bits_equal(st["exp_avg_sq"].numpy(), v), step
        p = t.detach().numpy().copy()


# ---- the training CLI's host side (percepnet_b200.train)

def write_records(path, frames, seed):
    rec = records(1, frames, seed)[0]
    rec.astype("<f4").tofile(path)
    return rec


def test_windows_of_cuts_files_into_windows(tmp_path):
    """Each file is cut into --window-frame windows in file order; a file's last window is shorter, zero-padded, and
    counts only its own frames."""
    from percepnet_b200.train import windows_of
    a = write_records(tmp_path / "a.f32", 7, 20)
    b = write_records(tmp_path / "b.f32", 3, 21)
    c = write_records(tmp_path / "c.f32", 6, 22)
    x, frames = windows_of([str(tmp_path / n) for n in ("a.f32", "b.f32", "c.f32")], 3)
    assert x.shape == (6, 3, 138) and x.dtype == np.float32
    assert frames.dtype == np.int32 and frames.tolist() == [3, 3, 1, 3, 3, 3]
    for i, w in enumerate([a[0:3], a[3:6], a[6:7], b[0:3], c[0:3], c[3:6]]):
        assert bits_equal(x[i, :len(w)], w), i
    assert not np.any(x[2, 1:])


def test_batches_are_seeded_full_and_reshuffled():
    """Full batches only (the remainder of an epoch is dropped), each epoch a permutation of its own, the same for the
    same seed."""
    from percepnet_b200.train import batches
    it = batches(11, 3, 5)
    first = [next(it) for _ in range(9)]
    assert [e for e, _ in first] == [0, 0, 0, 1, 1, 1, 2, 2, 2]
    for e in range(3):
        got = np.concatenate([idx for ep, idx in first if ep == e])
        assert all(len(idx) == 3 for ep, idx in first if ep == e)
        assert len(set(got.tolist())) == 9 and got.min() >= 0 and got.max() < 11
        assert got.tolist() == np.random.default_rng([5, e]).permutation(11)[:9].tolist()
    assert first[0][1].tolist() != first[3][1].tolist() or first[1][1].tolist() != first[4][1].tolist()
    again = batches(11, 3, 5)
    assert all(np.array_equal(next(again)[1], idx) for _, idx in first)
    other = batches(11, 3, 6)
    assert any(not np.array_equal(next(other)[1], idx) for _, idx in first)


@pytest.mark.parametrize("extra", [["--window", "0"], ["--batch", "0"], ["--steps", "-1"], ["--lr", "nan"],
                                   ["--lr", "-1e-4"], ["--lr", "inf"], ["--dev-list", "dev.txt"]],
                         ids=["window0", "batch0", "steps-1", "lr_nan", "lr_negative", "lr_inf", "dev_without_every"])
def test_parse_args_refusals(extra, capsys):
    from percepnet_b200.train import parse_args
    base = ["--list", "l.txt", "--steps", "1", "--out", "o.pnbw"]
    a = parse_args(base)
    assert (a.window, a.batch, a.lr, a.seed) == (500, 10, 1e-4, 0)
    with pytest.raises(SystemExit) as ex:
        parse_args(base + extra)
    assert ex.value.code == 2
    assert "error" in capsys.readouterr().err


def test_fewer_windows_than_the_batch(tmp_path, capsys):
    """Two files of 5 and 3 frames at --window 4 are three windows: --batch 4 returns 2 before any engine exists."""
    from percepnet_b200 import train
    for name, n in (("a.f32", 5), ("b.f32", 3)):
        write_records(tmp_path / name, n, 23)
    lst = tmp_path / "list.txt"
    lst.write_text(f"{tmp_path / 'a.f32'}\n\n{tmp_path / 'b.f32'}\n")
    out = tmp_path / "o.pnbw"
    assert train.main(["--list", str(lst), "--window", "4", "--batch", "4", "--steps", "1", "--out", str(out)]) == 2
    assert "3 windows, fewer than --batch 4" in capsys.readouterr().err
    assert not out.exists()
