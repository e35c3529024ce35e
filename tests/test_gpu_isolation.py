"""Serving properties of the batched engine that the single-stream reference has by construction: a stream's
output depends on nothing but its own samples -- not on the batch size, its row index, the other rows' content
(even NaN/Inf), nor on how the hops are grouped into calls.  The tensor path's GRU chain walks its units in
anti-diagonal order for few active streams and in hop-major order from util.first_hop_major streams on (the order every
large batch runs); the unit order must not change a single bit either."""
import numpy as np
import pytest

from util import crowd, device_first_hop_major, same_bits

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def api():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device")
    from percepnet_b200 import api
    api.load_library()
    return api


@pytest.mark.parametrize("nn", ["fp32", "tensor"])
def test_stream_is_independent_of_batch_and_neighbours(api, model0, nn):
    from percepnet_b200.synth import synth_pcm
    flags = api.NN_FP32 if nn == "fp32" else api.NN_TENSOR
    F = 14
    probe = synth_pcm(3, F, seed=777)                       # the streams we follow
    # (a) alone in a small batch
    e = api.Engine(3, F, model0, flags)
    out_a, gr_a = e.process(probe, want_gr=True)
    e.close()
    # (b) scattered through a batch of 261 (crosses two 128-row tiles of the tensor path) among other signals
    S = 261
    others = synth_pcm(S, F, seed=4000)
    rows = [5, 130, 260]
    x = others.copy()
    x[rows] = probe
    e = api.Engine(S, F, model0, flags)
    out_b, gr_b = e.process(x, want_gr=True)
    # (c) same batch, but the neighbours are poisoned with NaN / Inf / full-scale garbage from hop 3 on
    y = x.copy()
    bad = [r for r in range(S) if r not in rows]
    y[bad[0::3], 3 * 480 + 7] = np.nan
    y[bad[1::3], 4 * 480:] = np.inf
    y[bad[2::3], 3 * 480:] = 1e30
    e.reset()
    out_c, gr_c = e.process(y, want_gr=True)
    e.close()
    assert same_bits(out_b[rows], out_a) and same_bits(gr_b[:, rows], gr_a)
    assert same_bits(out_c[rows], out_a) and same_bits(gr_c[:, rows], gr_a)
    assert np.isfinite(out_c[rows]).all()


@pytest.mark.parametrize("nn,streams", [("fp32", 9), ("tensor", 9), ("fp32", "hop-major"), ("tensor", "hop-major")],
                         ids=["fp32", "tensor", "fp32-hop-major", "tensor-hop-major"])
def test_call_granularity_does_not_change_the_output(api, model0, nn, streams):
    """9 streams (anti-diagonal chain order) and util.first_hop_major streams (hop-major order, 127 padding rows in the
    last row tile): calls of 1, 9, 2, 8 and 3 hops equal one call of 23 bit for bit."""
    from percepnet_b200.synth import synth_pcm
    flags = api.NN_FP32 if nn == "fp32" else api.NN_TENSOR
    F = 23
    S = 9 if streams == 9 else device_first_hop_major()
    x = synth_pcm(9, F, seed=31) if S == 9 else crowd(S, F, seed=31)
    e = api.Engine(S, F, model0, flags)
    whole, gr_whole = e.process(x, want_gr=True)
    e.close()
    e = api.Engine(S, 9, model0, flags)                      # 9 = one group of 8 hops + 1: exercises the hop-group pre-pass
    outs, grs, t0 = [], [], 0
    for n in (1, 9, 2, 8, 3):
        o, g = e.process(x[:, t0 * 480:(t0 + n) * 480], want_gr=True)
        outs.append(o); grs.append(g); t0 += n
    e.close()
    assert t0 == F
    assert same_bits(np.concatenate(outs, axis=1), whole)
    assert same_bits(np.concatenate(grs, axis=0), gr_whole)


CALLS = (1, 2, 5, 23)                                         # hops per call


def _probes(oracle, model, mode, F):
    """unit scale (default engine): synth_pcm, the edge signals and random mixtures; PNB_CONV_WIDE: the same families at
    int16 scale, those whose float64 pre-activations stay inside the tanh domain (test_gpu_layer_bounds.families)."""
    if mode == "wide":
        from test_gpu_layer_bounds import families
        return np.stack([v for v, tag in families(oracle, model, F) if tag == "int16"])
    from percepnet_b200.synth import synth_pcm
    from util import edge_signals, random_mixtures
    return np.concatenate([synth_pcm(3, F, seed=777), np.stack(list(edge_signals(F).values())),
                           random_mixtures(4, F, seed=777)]).astype(np.float32)


def _run_calls(e, x, actives=None):
    """CALLS on engine e; actives[c]: the active range set before call c (None: leave it).  Returns the outputs and g/r
    of all S rows over all hops (rows beyond a call's active range are NaN)."""
    S = x.shape[0]
    out = np.full(x.shape, np.nan, np.float32)
    gr = np.full((sum(CALLS), S, 68), np.nan, np.float32)
    t0 = 0
    for c, n in enumerate(CALLS):
        if actives is not None:
            e.set_active(actives[c])
        k = e.active
        o, g = e.process(np.ascontiguousarray(x[:k, t0 * 480:(t0 + n) * 480]), want_gr=True)
        out[:k, t0 * 480:(t0 + n) * 480] = o
        gr[t0:t0 + n, :k] = g
        t0 += n
    e.check()
    return out, gr


def _first_difference(out, gr, rows, out_t, gr_t, P):
    """(row, probe, first differing hop) of every probe row whose outputs or g/r differ from its twin row's"""
    bad = []
    for k, r in enumerate(rows):
        p = k % P
        if same_bits(out[r], out_t[p]) and same_bits(gr[:, r], gr_t[:, p]):
            continue
        hop = next(t for t in range(gr.shape[0]) if not (same_bits(out[r, t * 480:(t + 1) * 480], out_t[p, t * 480:(t + 1) * 480])
                                                          and same_bits(gr[t, r], gr_t[t, p])))
        bad.append((r, p, hop))
    return bad


@pytest.mark.parametrize("mode", ["tensor", "wide"])
def test_unit_order_does_not_change_the_bits(api, oracle, model0, mode):
    """Probe streams at rows 0, 127, 128, h - 1, h and the last row of a 2h + 200-slot engine (h = first_hop_major: the
    chain runs hop-major) among other signals, in calls of 1, 2, 5 and 23 hops, against the probes alone in an engine of
    their own (anti-diagonal order): same outputs and g/r, bit for bit.  Then the same engine alternates its active range
    between h - 1 and h before every call, so the order flips call by call while the probes (rows < h - 1) carry their
    state across; they still match the twin bit for bit."""
    flags = api.NN_TENSOR | (api.CONV_WIDE if mode == "wide" else 0)
    h = device_first_hop_major()
    F, S = sum(CALLS), 2 * h + 200
    probes = _probes(oracle, model0, mode, F)
    P = len(probes)
    assert P >= 6, P
    tw = api.Engine(P, max(CALLS), model0, flags)
    try:
        out_t, gr_t = _run_calls(tw, probes)
    finally:
        tw.close()
    assert np.abs(out_t).max() > 0
    x = crowd(S, F, seed=55)
    e = api.Engine(S, max(CALLS), model0, flags)
    try:
        # probe k % P at rows[k]: the six rows above first, then neighbours of tile and order boundaries
        rows = [0, 127, 128, h - 1, h, S - 1, 1, 129, 255, 256, h - 2, h + 1, 2 * h - 1, 2 * h, S - 2, S - 129]
        x[rows] = probes[np.arange(len(rows)) % P]
        out, gr = _run_calls(e, x)
        bad = _first_difference(out, gr, rows, out_t, gr_t, P)
        assert not bad, f"hop-major engine: (row, probe, first differing hop) {bad}"
        # the order flips between calls: anti-diagonal at h - 1 active streams, hop-major at h
        e.reset()
        rows = [0, 1, 127, 128, 129, 255, 256, 1023, 1024, h - 5, h - 4, h - 3, h - 2]
        x[rows] = probes[np.arange(len(rows)) % P]
        out, gr = _run_calls(e, x, actives=[h - 1, h, h - 1, h])
        bad = _first_difference(out, gr, rows, out_t, gr_t, P)
        assert not bad, f"order switching between calls: (row, probe, first differing hop) {bad}"
    finally:
        e.close()
