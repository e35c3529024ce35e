"""The conv layers run two neighbouring hops per tile (conv_pair_kernel): a hop is the first or the second of a pair, or
alone when a call has an odd number of hops, depending on how the hops are grouped into calls.  Its bits must not
depend on which.  These cases cover the three-term mode (PNB_CONV_WIDE, at int16 scale) and ragged calls whose short
rows stop on the first hop of a pair; test_gpu_isolation and test_gpu_ragged cover the default mode."""
import numpy as np
import pytest

from util import crowd, device_first_hop_major, same_bits

pytestmark = pytest.mark.gpu

HOP = 480


@pytest.fixture(scope="module")
def api():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device")
    from percepnet_b200 import api
    api.load_library()
    return api


@pytest.mark.parametrize("streams", [9, "hop-major"])
def test_wide_call_granularity_does_not_change_the_output(api, model0, streams):
    """9 streams and util.first_hop_major streams (127 padding rows in the last row tile) on a PNB_CONV_WIDE engine:
    calls of 1, 9, 2, 8 and 3 hops (lone hops and pairs at every parity) equal one call of 23 bit for bit."""
    from percepnet_b200.synth import synth_pcm
    flags = api.NN_TENSOR | api.CONV_WIDE
    F = 23
    S = 9 if streams == 9 else device_first_hop_major()
    x = synth_pcm(9, F, seed=31, scale=32768.0) if S == 9 else crowd(S, F, seed=31) * np.float32(32768.0)
    e = api.Engine(S, F, model0, flags)
    whole, gr_whole = e.process(x, want_gr=True)
    e.check()
    e.close()
    e = api.Engine(S, 9, model0, flags)
    outs, grs, t0 = [], [], 0
    for n in (1, 9, 2, 8, 3):
        o, g = e.process(np.ascontiguousarray(x[:, t0 * HOP:(t0 + n) * HOP]), want_gr=True)
        outs.append(o); grs.append(g); t0 += n
    e.check()
    e.close()
    assert t0 == F
    assert np.abs(whole).max() > 1.0
    assert same_bits(np.concatenate(outs, axis=1), whole)
    assert same_bits(np.concatenate(grs, axis=0), gr_whole)


def test_wide_ragged_rows_stop_on_the_first_hop_of_a_pair(api, model0):
    """A ragged call of 6 hops on a PNB_CONV_WIDE session pool of util.first_hop_major sessions (the last row tile
    partial): rows run 1, 3, 5 or 6 hops, so most stop on the first hop of a pair, whose second hop is computed but
    frozen.  A second call of 3 hops continues every row from its own last hop.  Outputs and g/r of both calls equal a
    plain engine that runs each row's hops back to back, and the frozen hops come back as zeros."""
    flags = api.NN_TENSOR | api.CONV_WIDE
    S = device_first_hop_major()
    F, F2 = 6, 3
    rng = np.random.RandomState(7)
    hops = rng.choice([1, 3, 5, 6], size=S).astype(np.int32)
    hops[0] = F
    x = crowd(S, F + F2, seed=41) * np.float32(32768.0)
    t = api.Engine(S, F + F2, model0, flags)
    whole, gr_whole = t.process(x, want_gr=True)
    t.check()
    t.close()

    e = api.Engine(S, F, model0, flags)
    e.reserve_sessions(S)
    ids = np.arange(S, dtype=np.int32)
    xin = np.full((S, F * HOP), np.nan, np.float32)          # input beyond a row's own hops is never read
    for r, h in enumerate(hops):
        xin[r, :h * HOP] = x[r, :h * HOP]
    out1, gr1 = e.process_sessions(ids, xin, want_gr=True, hops=hops)
    xin2 = np.stack([x[r, h * HOP:(h + F2) * HOP] for r, h in enumerate(hops)])
    out2, gr2 = e.process_sessions(ids, xin2, want_gr=True)
    e.check()
    e.close()
    for r, h in enumerate(hops):
        assert same_bits(out1[r, :h * HOP], whole[r, :h * HOP]), r
        assert not out1[r, h * HOP:].any(), r
        assert same_bits(gr1[:h, r], gr_whole[:h, r]), r
        assert not gr1[h:, r].any(), r
        assert same_bits(out2[r], whole[r, h * HOP:(h + F2) * HOP]), r
        assert same_bits(gr2[:, r], gr_whole[h:h + F2, r]), r
