"""The synthesis's gradient on the CPU: the float64 restatement (tests/synth_grad_oracle.py) against the float32
synthesis that is bit-exact to the reference (tests/synthesis_oracle.py) on operands the oracle's analysis makes, its
autograd against central differences, include/pnb_synth_grad.h against its Python signature table and the library's
exports, and SignalPath's refusals."""
import ctypes as C
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from conftest import ROOT
from percepnet_b200 import torch_signal as ts
from percepnet_b200.synth import synth_pairs
import synth_grad_oracle as SG
from synthesis_oracle import FRAME, post_filter, sine_rounded, synthesize
from test_api_mirror_train_device import KINDS, _prototypes

INC = os.path.join(ROOT, "include")


@pytest.fixture(scope="module")
def api():
    from percepnet_b200 import api, build
    build.build()
    return api


@pytest.fixture(scope="module")
def tab(oracle):
    return SG.Tables(oracle)


def oracle_ops(oracle, model, pcm):
    """[n, T*480] PCM at the C API's scale -> ops [n, T, 1636] float32 as the engine exports them, from the oracle's
    per-hop taps of a fresh stream per row (X and P bins 0..399, Ex, the silence flag)."""
    n, T = pcm.shape[0], pcm.shape[1] // FRAME
    ops = np.zeros((n, T, SG.OPS), np.float32)
    for i in range(n):
        h = oracle.create(model)
        _, _, taps = oracle.process_stream(h, pcm[i].astype(np.float32), taps=True)
        oracle.destroy(h)
        for t, tp in enumerate(taps):
            ops[i, t, :800] = tp.np("X")[:800]
            ops[i, t, 800:1600] = tp.np("P")[:800]
            ops[i, t, 1600:1634] = tp.np("Ex")
            ops[i, t, 1634] = 1.0 if tp.silence else 0.0
    return ops


def pair_ops(oracle, model, n, T, seed):
    """Operands of int16-scale synthetic noisy speech (synth_pairs), with the middle third of row 0 zeroed so that
    both silent and voiced hops occur."""
    _, noisy = synth_pairs(n, T, seed=seed)
    x = noisy.astype(np.float32)
    x[0, T // 3 * FRAME:2 * T // 3 * FRAME] = 0
    return oracle_ops(oracle, model, x)


def random_gr(rng, n, T):
    gr = rng.rand(n, T, 68).astype(np.float32)
    gr[:, 1, :] = 1.0
    gr[:, 2, :34] = 0.0
    return gr


@pytest.mark.parametrize("post", [False, True], ids=["plain", "postfilter"])
def test_restatement_is_the_synthesis(oracle, model0, tab, post):
    """The float64 restatement of a call of T hops equals the float32 synthesis hop by hop, overlap-add memory carried,
    within float32 rounding: silent and voiced hops, g/r random and at 0 and 1."""
    n, T = 2, 24
    ops = pair_ops(oracle, model0, n, T, seed=501)
    sil = ops[..., 1634]
    assert sil.any() and not sil.all(), sil
    gr = random_gr(np.random.RandomState(7), n, T)
    hw, _ = oracle.tables()
    mem0 = np.random.RandomState(8).randn(n, FRAME).astype(np.float32) * 100
    out64, mem64 = SG.synthesize(tab, torch.from_numpy(ops.astype(np.float64)), torch.from_numpy(gr.astype(np.float64)),
                                 post, torch.from_numpy(mem0.astype(np.float64)))
    for i in range(n):
        mem = mem0[i].copy()
        want = []
        for t in range(T):
            g, r = gr[i, t, :34], gr[i, t, 34:]
            if post:
                g = post_filter(g, ops[i, t, 1600:1634], sine_rounded)
            want.append(synthesize(oracle, ops[i, t, :800], ops[i, t, 800:1600], bool(sil[i, t]), g, r, mem, hw))
        want = np.concatenate(want).astype(np.float64)
        got = out64[i].numpy()
        scale = np.abs(want).max()
        err = np.abs(got - want).max() / scale
        print(f"row {i} post={post}: max |out64 - out32| / max |out| = {err:.2e}")
        assert err < 2e-6, (i, err)
        assert np.abs(mem64[i].numpy() - mem).max() / scale < 2e-6


@pytest.mark.parametrize("post", [False, True], ids=["plain", "postfilter"])
def test_restatement_gradient_is_central_differences(oracle, model0, tab, post):
    """Autograd of the restatement against float64 central differences of L = sum(out * dout), every component of
    g/r of a three-hop call, a silent hop included."""
    ops = pair_ops(oracle, model0, 1, 18, seed=502)[:, 5:8]
    ops[0, 1, 1634] = 1.0
    rng = np.random.RandomState(9)
    gr = rng.rand(1, 3, 68) * 0.8 + 0.1
    dout = rng.randn(1, 3 * FRAME)
    o = torch.from_numpy(ops.astype(np.float64))
    d = torch.from_numpy(dout)
    grad = SG.grad(tab, o, gr, dout, post).numpy()

    def loss(v):
        out, _ = SG.synthesize(tab, o, torch.from_numpy(v), post)
        return float((out * d).sum())

    h = 1e-6
    fd = np.zeros_like(gr)
    for idx in np.ndindex(gr.shape):
        a, b = gr.copy(), gr.copy()
        a[idx] += h
        b[idx] -= h
        fd[idx] = (loss(a) - loss(b)) / (2 * h)
    err = np.abs(grad - fd).max() / np.abs(fd).max()
    print(f"post={post}: max |autograd - central differences| / max = {err:.2e}")
    assert err < 1e-6
    assert np.all(grad[0, 1, 34:] == 0)                       # the silent hop's r takes no gradient


def test_post_filter_gradient_vanishes_at_zero_gains(tab):
    """Every g zero under the post-filter: the filtered gains and their gradient are exactly 0, not inf * 0."""
    g = torch.zeros(1, 34, dtype=torch.float64, requires_grad=True)
    Ey = torch.rand(1, 34, dtype=torch.float64) * 1e4
    gu = SG.post_filter(g, Ey)
    (d,) = torch.autograd.grad(gu.sum(), g)
    assert torch.all(gu == 0) and torch.all(d == 0)


def test_library_types_match_every_prototype(api):
    protos = _prototypes("pnb_synth_grad.h")
    assert set(protos) == {"pnb_synthesis_operands_device", "pnb_synthesis_backward_device"} == \
        set(api.SYNTH_GRAD_EXPORTS)
    for other in ("percepnet_b200.h", "pnb_train_device.h", "pnb_train_state.h"):
        assert not set(protos) & set(_prototypes(other)), other
    assert not set(protos) & (set(api.EXPORTS) | set(api.TRAIN_DEVICE_EXPORTS) | set(api.TRAIN_STATE_EXPORTS))
    L = api.load_library()
    kinds = {**KINDS, "long long": (C.c_longlong,)}
    for name, (ret, params) in protos.items():
        f = getattr(L, name)
        assert ret == "int" and f.restype is C.c_int, name
        assert len(f.argtypes) == len(params), (name, params, f.argtypes)
        for k, (p, t) in enumerate(zip(params, f.argtypes)):
            assert (t is C.c_void_p) if p == "*" else t in kinds[p], (name, k, p, t)
    hdr = open(os.path.join(INC, "pnb_synth_grad.h")).read()
    assert int(re.search(r"#define PNB_SYNTH_OPS_FLOATS (\d+)", hdr).group(1)) == api.SYNTH_OPS_FLOATS == \
        ts.OPS_FLOATS == SG.OPS
    top = open(os.path.join(INC, "percepnet_b200.h")).read()
    assert int(re.search(r"#define PNB_LATENCY_FRAMES (\d+)", top).group(1)) == ts.LATENCY_FRAMES


@pytest.mark.parametrize("first", ["pnb_synth_grad.h", "percepnet_b200.h"])
def test_header_is_plain_c(tmp_path, first):
    src = tmp_path / "hdr.c"
    src.write_text(f'#include "{first}"\n'
                   "int main(void) { int (*f)(const float *, size_t, const float *, size_t, long long, int, int, "
                   "const float *, size_t, float *, size_t, void *) = pnb_synthesis_backward_device; (void)f; "
                   "(void)pnb_synthesis_operands_device; (void)pnb_train_forward_state_device; "
                   "return PNB_SYNTH_OPS_FLOATS; }\n")
    cc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.run([cc, "-std=c99", "-pedantic", "-Wall", "-Werror", "-fsyntax-only", "-I", INC, str(src)], check=True)
    subprocess.run([cxx, "-std=c++11", "-Wall", "-Werror", "-fsyntax-only", "-x", "c++", "-I", INC, str(src)], check=True)


def test_signal_path_refusals():
    """Refused before any engine exists: wrong shapes and dtypes, B or T above the path's, a synthesis with no analysis
    pending or with other operands; well-formed CPU tensors get as far as the CPU input's refusal."""
    with pytest.raises(ValueError, match=">= 1"):
        ts.SignalPath(0, 10)
    with pytest.raises(RuntimeError, match="CUDA device"):
        ts.SignalPath(2, 10, device="cpu")
    sp = ts.SignalPath(2, 10)
    for bad in (torch.zeros(2, 4 * FRAME + 1), torch.zeros(2, 3, FRAME), torch.zeros(0, FRAME), torch.zeros(2, 0)):
        with pytest.raises(ValueError, match=r"\[B, T\*480\]"):
            sp.analyze(bad)
    for dt in (torch.float64, torch.int32, torch.float16):
        with pytest.raises(TypeError, match="float32 or int16"):
            sp.analyze(torch.zeros(2, FRAME, dtype=dt))
    for bad in (torch.zeros(3, FRAME), torch.zeros(2, 11 * FRAME)):
        with pytest.raises(ValueError, match="above the path's 2 rows x 10 hops"):
            sp.analyze(bad)
    ops = torch.zeros(2, 4, ts.OPS_FLOATS)
    for bad in (torch.zeros(2, 4, 67), torch.zeros(2, 4), torch.zeros(2, 0, 68)):
        with pytest.raises(ValueError, match=r"\[B, T, 68\]"):
            sp.synthesize(bad, ops)
    with pytest.raises(TypeError, match="gr must be float32"):
        sp.synthesize(torch.zeros(2, 4, 68, dtype=torch.float64), ops)
    with pytest.raises(ValueError, match="pending analysis"):
        sp.synthesize(torch.zeros(2, 4, 68), ops)
    for dt in (torch.float32, torch.int16):
        with pytest.raises(RuntimeError, match="CUDA tensor"):
            sp.analyze(torch.zeros(2, 4 * FRAME, dtype=dt))
    sp._pending = ops                                # as an analysis would leave it
    with pytest.raises(ValueError, match=r"= \[2, 4, 68\] as the pending analysis"):
        sp.synthesize(torch.zeros(1, 4, 68), ops)
    with pytest.raises(RuntimeError, match="CUDA tensor"):
        sp.synthesize(torch.zeros(2, 4, 68), ops)
