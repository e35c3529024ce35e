"""Network state in and out of the trainer, on the CPU: include/pnb_train_state.h against its Python signature table and
the library's exports, the header as C99 and C++11, the state layout against StreamState's network part, the float64
restatement with state against train_oracle.Net, and the module's refusals of bad state and lengths."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from conftest import ROOT
from percepnet_b200 import torch_module as tm
from percepnet_b200.weights import synth_state_dict
import train_oracle as O
import train_state_oracle as SO
from test_api_mirror_train_device import KINDS, _prototypes

INC = os.path.join(ROOT, "include")


@pytest.fixture(scope="module")
def api():
    from percepnet_b200 import api, build
    build.build()
    return api


def test_library_types_match_every_prototype(api):
    protos = _prototypes("pnb_train_state.h")
    assert set(protos) == {"pnb_train_forward_state_device", "pnb_train_backward_state_device"} == \
        set(api.TRAIN_STATE_EXPORTS)
    for other in ("percepnet_b200.h", "pnb_train_device.h"):
        assert not set(protos) & set(_prototypes(other)), other
    assert not set(protos) & (set(api.EXPORTS) | set(api.TRAIN_DEVICE_EXPORTS))
    L = api.load_library()
    for name, (ret, params) in protos.items():
        f = getattr(L, name)
        assert ret == "int" and f.restype is C.c_int, name
        assert len(f.argtypes) == len(params), (name, params, f.argtypes)
        for k, (p, t) in enumerate(zip(params, f.argtypes)):
            assert (t is C.c_void_p) if p == "*" else t in KINDS[p], (name, k, p, t)


@pytest.mark.parametrize("first", ["pnb_train_state.h", "percepnet_b200.h"])
def test_header_is_plain_c(tmp_path, first):
    src = tmp_path / "hdr.c"
    src.write_text(f'#include "{first}"\n'
                   "int main(void) { int (*f)(pnb_engine *, const float *, size_t, const float *, size_t, float *, size_t, "
                   "float *, size_t, float *, void *) = pnb_train_backward_state_device; (void)f; "
                   "(void)pnb_train_forward_state_device; (void)pnb_train_forward_device; "
                   "return PNB_TRAIN_STATE_FLOATS; }\n")
    cc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.run([cc, "-std=c99", "-pedantic", "-Wall", "-Werror", "-fsyntax-only", "-I", INC, str(src)], check=True)
    subprocess.run([cxx, "-std=c++11", "-Wall", "-Werror", "-fsyntax-only", "-x", "c++", "-I", INC, str(src)], check=True)


def test_layout_is_stream_states_network_part(api):
    """STATE_FLOATS is the header's value and spans StreamState's fc_hist .. h; each slice starts at its field's offset
    (pnb_state.h's static_assert) and the GRU states follow h's order (four of 512, then 128)."""
    hdr = open(os.path.join(INC, "pnb_train_state.h")).read()
    assert int(re.search(r"#define PNB_TRAIN_STATE_FLOATS (\d+)", hdr).group(1)) == tm.STATE_FLOATS == api.TRAIN_STATE_FLOATS
    st = open(os.path.join(ROOT, "percepnet_b200", "csrc", "pnb_state.h")).read()
    off = {k: int(v) for k, v in re.findall(r"offsetof\(StreamState, (\w+)\) == (\d+)", st)}
    assert tm.STATE_FLOATS * 4 == off["has_terms"] - off["fc_hist"] == 54584 - 39736
    L = tm.STATE_LAYOUT
    assert L["fc_hist"].start * 4 + off["fc_hist"] == off["fc_hist"]
    assert L["c1_hist"].start * 4 + off["fc_hist"] == off["c1_hist"]
    assert L["gru1"].start * 4 + off["fc_hist"] == off["h"]
    sizes = [(k, s.stop - s.start) for k, s in L.items()]
    assert sizes == [("fc_hist", 512), ("c1_hist", 1024), ("gru1", 512), ("gru2", 512), ("gru3", 512),
                     ("gru_gb", 512), ("gru_rb", 128)]
    assert all(a.stop == b.start for a, b in zip(list(L.values()), list(L.values())[1:]))
    assert list(L.values())[-1].stop == tm.STATE_FLOATS


def test_restatement_from_zero_state_is_net_and_chains():
    """The float64 restatement from zero state is Net.forward; from a random state, two chained calls give one whole
    call's outputs and state out."""
    m = O.model(synth_state_dict(1), torch.float64)
    rng = np.random.RandomState(5)
    x = torch.from_numpy(rng.rand(2, 9, 70) * 0.5)
    with torch.no_grad():
        out, _ = SO.forward(m, x)
        assert torch.allclose(out, m(x), rtol=1e-12, atol=1e-14)
        s0 = SO.random_state(2, 6, torch.float64)
        whole, s_whole = SO.forward(m, x, s0)
        for cut in (1, 3, 4, 7):
            a, sa = SO.forward(m, x[:, :cut], s0)
            b, sb = SO.forward(m, x[:, cut:], sa)
            assert torch.allclose(torch.cat([a, b], 1), whole, rtol=1e-12, atol=1e-14), cut
            assert torch.allclose(sb, s_whole, rtol=1e-12, atol=1e-14), cut


def test_module_refuses_bad_state_and_lengths():
    m = tm.PercepNet()
    x = torch.zeros(2, 5, 70)
    ok = torch.zeros(2, tm.STATE_FLOATS)
    for bad in (torch.zeros(3, tm.STATE_FLOATS), torch.zeros(2, tm.STATE_FLOATS - 1), torch.zeros(2, 1, tm.STATE_FLOATS)):
        with pytest.raises(ValueError, match="state must be"):
            m(x, bad)
    with pytest.raises(TypeError, match="state must be float32"):
        m(x, ok.double())
    with pytest.raises(ValueError, match="x's device"):
        m(x, torch.zeros(2, tm.STATE_FLOATS, device="meta"))
    for bad in ([5], [1, 2, 3], [[1, 2]], torch.tensor([3])):
        with pytest.raises(ValueError, match="one entry per window"):
            m(x, lengths=bad)
    for bad in ([0, 5], [1, 6], torch.tensor([-1, 2])):
        with pytest.raises(ValueError, match=r"in \[1, 5\]"):
            m(x, ok, lengths=bad)
    with pytest.raises(TypeError, match="integers"):
        m(x, lengths=[1.0, 2.0])
    with pytest.raises(ValueError, match="CPU"):
        m(x, lengths=torch.tensor([1, 2], device="meta"))
    # well-formed state and lengths get as far as the CPU input's refusal
    for kw in ({"state": ok}, {"lengths": torch.tensor([5, 1])}, {"lengths": (2, 3), "return_state": True}):
        with pytest.raises(RuntimeError, match="CUDA"):
            m(x, **kw)
