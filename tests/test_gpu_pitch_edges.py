"""The GPU pitch stage (pitch_stage<> in pnb_dsp.cu) on the edge corpus of tests/golden/make_pitch_edges.py: inputs
that sit on its comparisons and clamps (candidate ties, the -1 floor of the fine xcorr, sub-lag offset ties, T1 = 90,
T0 = 256, the energy floor).  Every row carries the reference's own outputs; integer results must be equal and float
results bit-identical.

* pitch_only_kernel through pnb_pitch_only_device (padded rows, a unit count that is not a multiple of the block's 8
  warps) and through pnb_pitch_only_host;
* the corpus replicated to 65 536 units, the size bench.py --path xcorr measures (BASELINE.json config 5);
* analysis_kernel, with every corpus buffer laid out as the pitch buffer of one hop of a stream, plus quiet random
  mixtures: every DSP tap bit-identical to oracle.process_stream, across ragged chunks of hops.
"""
import os

import numpy as np
import pytest

from conftest import GOLDEN
from util import random_mixtures, same_bits

pytestmark = pytest.mark.gpu

FRAME = 480
HOP_AT = 8                   # the hop whose pitch buffer is the corpus row
OFF_AT = HOP_AT * FRAME - 3648  # pitch buffer of hop t = input samples [480 t - 3648, 480 t - 1920) (hist[1632:3360))
N_HOPS = 10


@pytest.fixture(scope="module")
def api():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device")
    from percepnet_b200 import api
    api.load_library()
    return api


@pytest.fixture(scope="module")
def corpus():
    return dict(np.load(os.path.join(GOLDEN, "pitch_edges.npz")))


def _check(c, idx, lag, T, corr, gain):
    """outputs of units `idx` of the corpus against the stored reference values"""
    bad = np.nonzero((lag != c["lag"][idx]) | (T != c["T"][idx]))[0]
    assert bad.size == 0, f"lag / T differ at units {bad[:10]} (rows {idx[bad[:10]]})"
    assert same_bits(corr, c["corr"][idx]), np.nonzero(corr != c["corr"][idx])[0][:10]
    assert same_bits(gain, c["gain"][idx]), np.nonzero(gain != c["gain"][idx])[0][:10]


def _device_run(api, bufs, pT, pg, stride):
    import torch
    n = bufs.shape[0]
    d_buf = torch.zeros((n, stride), dtype=torch.float32, device="cuda")
    d_buf[:, :1728] = torch.from_numpy(bufs).cuda()
    d_pT, d_pg = torch.from_numpy(pT).cuda(), torch.from_numpy(pg).cuda()
    d_T = torch.empty(n, dtype=torch.int32, device="cuda")
    d_lag = torch.empty(n, dtype=torch.int32, device="cuda")
    d_corr = torch.empty(n, dtype=torch.float32, device="cuda")
    d_gain = torch.empty(n, dtype=torch.float32, device="cuda")
    api.pitch_only_device(d_buf.data_ptr(), stride, n, d_T.data_ptr(), d_corr.data_ptr(), d_gain.data_ptr(),
                          d_lag.data_ptr(), d_pT.data_ptr(), d_pg.data_ptr())
    torch.cuda.synchronize()
    return d_lag.cpu().numpy(), d_T.cpu().numpy(), d_corr.cpu().numpy(), d_gain.cpu().numpy()


def test_pitch_only_device_edges(api, corpus):
    n = corpus["buf"].shape[0]
    idx = np.arange(n + (3 - n) % 8) % n              # a count that leaves 3 warps of the last block busy
    assert idx.size % 8 == 3 and idx.size >= n
    lag, T, corr, gain = _device_run(api, corpus["buf"][idx], corpus["prev_period"][idx], corpus["prev_gain"][idx],
                                     stride=1728 + 40)
    _check(corpus, idx, lag, T, corr, gain)


def test_pitch_only_host_edges(api, corpus):
    T, corr, gain, lag = api.pitch_only(corpus["buf"], corpus["prev_period"], corpus["prev_gain"])
    _check(corpus, np.arange(corpus["buf"].shape[0]), lag, T, corr, gain)


def test_pitch_only_edges_replicated_65536(api, corpus):
    """BASELINE.json config 5's 65 536 units: each a replica of a corpus row, each bit-identical to its base row"""
    n = corpus["buf"].shape[0]
    U = 65536
    idx = np.random.RandomState(5).permutation(U) % n   # replicas of one row spread over every block and warp slot
    lag, T, corr, gain = _device_run(api, corpus["buf"][idx], corpus["prev_period"][idx], corpus["prev_gain"][idx],
                                     stride=1728)
    _check(corpus, idx, lag, T, corr, gain)


def _edge_streams(corpus):
    """one stream per corpus row: silence, the row as the pitch buffer of hop HOP_AT, silence"""
    n = corpus["buf"].shape[0]
    x = np.zeros((n, N_HOPS * FRAME), np.float32)
    x[:, OFF_AT:OFF_AT + 1728] = corpus["buf"]
    return x


def test_analysis_kernel_edges_taps(api, oracle, model0, corpus):
    edge = _edge_streams(corpus)
    quiet = random_mixtures(16, N_HOPS, seed=404)
    x = np.concatenate([edge, quiet * np.float32(1e-3), quiet * np.float32(1e-6)]).astype(np.float32)
    S, ne = x.shape[0], edge.shape[0]
    taps = []
    for s in range(S):
        h = oracle.create(model0)
        taps.append(oracle.process_stream(h, x[s], True, taps=True)[2])
        oracle.destroy(h)
    # the layout puts each row where the oracle's own pitch buffer is: lag and corr depend on nothing else
    assert [taps[s][HOP_AT].pitch_search for s in range(ne)] == corpus["lag"].tolist()
    assert same_bits([taps[s][HOP_AT].pitch_corr for s in range(ne)], corpus["corr"])
    Fmax = 4
    eng = api.Engine(S, Fmax, model0, api.NN_FP32 | api.KEEP_TAPS)
    t0 = 0
    while t0 < N_HOPS:                   # ragged chunking: 4, 4, 2 hops -> state carried across calls
        n = min(Fmax, N_HOPS - t0)
        eng.process(x[:, t0 * FRAME:(t0 + n) * FRAME])
        got = {k: eng.read_tap(k, n) for k in ("pitch", "pitchf", "features", "X", "P", "Ex")}
        for s in range(S):
            for k in range(n):
                tp = taps[s][t0 + k]
                tag = f"stream {s} hop {t0 + k}"
                assert got["pitch"][k, s, 0] == tp.pitch_search, tag
                assert got["pitch"][k, s, 1] == tp.pitch_index, tag
                assert got["pitch"][k, s, 2] == tp.silence, tag
                assert same_bits(got["pitchf"][k, s], [tp.pitch_corr, tp.pitch_gain]), tag
                assert same_bits(got["features"][k, s], tp.np("features")), tag
                assert same_bits(got["X"][k, s], tp.np("X")[:800]), tag
                assert same_bits(got["P"][k, s], tp.np("P")[:800]), tag
                assert same_bits(got["Ex"][k, s], tp.np("Ex")), tag
        t0 += n
    eng.close()
