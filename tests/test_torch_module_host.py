"""torch_module.PercepNet on the CPU: the permutation between its parameters and the PNBW blob is weights.py's layout
bit for bit, its parameters are rnn_train.PercepNet's, and there is no CPU path."""
import numpy as np
import pytest
import torch

from percepnet_b200 import torch_module as tm
from percepnet_b200.weights import N_PARAMS, pack_state_dict, unpack_state_dict, synth_state_dict
import train_oracle as O


def _flat(sd, names):
    return torch.cat([torch.from_numpy(np.ascontiguousarray(sd[k], np.float32)).reshape(-1) for k in names])


@pytest.mark.parametrize("seed,gain", [(0, 1.0), (3, 4.0)])
def test_blob_index_is_pack_state_dict(seed, gain):
    """to_blob of random parameters equals pack_state_dict(sd).flat() bit for bit, and from_blob of that blob gives
    back unpack_state_dict's tensors bit for bit."""
    m = tm.PercepNet()
    names = [k for k, _ in m.named_parameters()]
    sd = synth_state_dict(seed, gain)
    blob = tm.to_blob(_flat(sd, names), m._index)
    want = pack_state_dict(sd).flat()
    assert blob.shape == (N_PARAMS,)
    assert np.array_equal(blob.numpy().view(np.int32), want.view(np.int32))
    back = tm.from_blob(torch.from_numpy(want), m._index)
    un = unpack_state_dict(pack_state_dict(sd))
    at = 0
    for k, p in m.named_parameters():
        got = back[at:at + p.numel()].view(p.shape).numpy()
        assert np.array_equal(got.view(np.int32), un[k].view(np.int32)), k
        at += p.numel()
    assert at == N_PARAMS


def test_parameters_are_rnn_train_percepnet():
    """The module's state_dict has train_oracle.Net's keys (the in-repo restatement of rnn_train.PercepNet), in order,
    with its shapes, and a state dict goes through load_state_dict / state_dict unchanged."""
    m, ref = tm.PercepNet(), O.Net()
    assert [(k, tuple(v.shape)) for k, v in m.state_dict().items()] == \
        [(k, tuple(v.shape)) for k, v in ref.state_dict().items()]
    sd = {k: torch.from_numpy(v) for k, v in synth_state_dict(5).items()}
    m.load_state_dict(sd)
    out = m.state_dict()
    assert set(out) == set(sd)
    for k, v in sd.items():
        assert torch.equal(out[k].view(torch.int32), v.view(torch.int32)), k


def test_cpu_input_raises():
    m = tm.PercepNet()
    with pytest.raises(RuntimeError, match="CUDA"):
        m(torch.zeros(2, 3, 70))
