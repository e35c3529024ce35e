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
