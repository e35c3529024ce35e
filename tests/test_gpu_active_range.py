"""Active range (pnb_set_active_streams): a call advances slots [0, n) only.  Every active row must equal, bit for bit,
the same row of a twin engine that advances all slots and resets the slots that enter the range; compaction by export /
import keeps live sessions exact; refused arguments leave the engine usable."""
import ctypes

import numpy as np
import pytest

from test_gpu_lifecycle import _engine, _ops_stream, _signal
from test_gpu_parity import api  # noqa: F401

pytestmark = pytest.mark.gpu

HOP = 480
FM = 16
# (id, network mode, streams, overlap); 1000 is not a multiple of the 128-row tile.  overlap: the state operations (the
# resets of a grow included) go to a non-blocking stream of their own, beside the streams the calls run on.
CONFIGS = [("fp32-1000", "fp32", 1000, False), ("fp32-2048", "fp32", 2048, False), ("tensor-1000", "tensor", 1000, False),
           ("tensor-2048", "tensor", 2048, False), ("tensor-1000-overlap", "tensor", 1000, True)]
IDS = [c[0] for c in CONFIGS]


def _schedule(S):
    """(active count, hops) per call: shrink, hold, shrink to one, grow to all, shrink; F in {1, 3, 16}."""
    return list(zip([S, 617, 617, 129, 1, S, 300], [3, 16, 1, 3, 16, 1, 16]))


def _inputs(S, hops, seed):
    x = np.concatenate([_signal(S, 1, seed + k)[:, :8 * HOP] for k in range((hops + 7) // 8)], axis=1)
    return np.ascontiguousarray(x[:, :hops * HOP])


def _to_i16(x):
    return np.clip(np.rint(x * 16384.0), -32768, 32767).astype(np.int16)


def _resize(a, b, n_old, n, stream=0):
    """a goes to n active slots; its full-range twin b resets the slots that enter."""
    a.set_active(n, stream)
    if n > n_old:
        b.reset_streams(np.arange(n_old, n), stream)


def _twins(api, model0, cfg):
    _, mode, S, _ = cfg
    return _engine(api, model0, S, mode, Fm=FM), _engine(api, model0, S, mode, Fm=FM)


@pytest.mark.parametrize("dtype", ["f32", "i16"])
@pytest.mark.parametrize("cfg", CONFIGS, ids=IDS)
def test_host_calls_match_full_range_twin(api, model0, cfg, dtype):
    S = cfg[2]
    sched = _schedule(S)
    x = _inputs(S, sum(f for _, f in sched), 11)
    if dtype == "i16":
        x = _to_i16(x)
    a, b = _twins(api, model0, cfg)
    ops = _ops_stream(cfg)
    n_old, t = S, 0
    for n, F in sched:
        _resize(a, b, n_old, n, ops)
        assert a.active == n and b.active == S
        xc = np.ascontiguousarray(x[:, t * HOP:(t + F) * HOP])
        out_a, gr_a = a.process(xc[:n], want_gr=True)
        out_b, gr_b = b.process(xc, want_gr=True)
        assert out_a.shape == (n, F * HOP) and gr_a.shape == (F, n, 68)
        assert np.array_equal(out_a, out_b[:n]), (n, F)
        assert np.array_equal(gr_a.view(np.int32), gr_b[:, :n].view(np.int32)), (n, F)
        n_old, t = n, t + F
    assert np.abs(out_a.astype(np.float32)).max() > 0
    for e in (a, b):
        e.check()
        e.close()


@pytest.mark.parametrize("cfg", CONFIGS, ids=IDS)
def test_device_calls_match_full_range_twin(api, model0, cfg):
    import torch
    S = cfg[2]
    sched = _schedule(S)
    x = torch.from_numpy(_inputs(S, sum(f for _, f in sched), 12)).cuda()
    a, b = _twins(api, model0, cfg)
    st = torch.cuda.current_stream().cuda_stream
    ops = _ops_stream(cfg, st)
    n_old, t = S, 0
    for n, F in sched:
        _resize(a, b, n_old, n, ops)
        xa = x[:n, t * HOP:(t + F) * HOP].contiguous()
        xb = x[:, t * HOP:(t + F) * HOP].contiguous()
        oa, ob = torch.empty_like(xa), torch.empty_like(xb)
        ga = torch.empty((F, n, 68), device="cuda")
        gb = torch.empty((F, S, 68), device="cuda")
        a.process_device(xa.data_ptr(), F * HOP, oa.data_ptr(), F * HOP, F, ga.data_ptr(), st)
        b.process_device(xb.data_ptr(), F * HOP, ob.data_ptr(), F * HOP, F, gb.data_ptr(), st)
        torch.cuda.synchronize()
        assert torch.equal(oa.view(torch.int32), ob[:n].view(torch.int32)), (n, F)
        assert torch.equal(ga.view(torch.int32), gb[:, :n].contiguous().view(torch.int32)), (n, F)
        n_old, t = n, t + F
    for e in (a, b):
        e.check(st)
        e.close()


@pytest.mark.parametrize("cfg", CONFIGS, ids=IDS)
def test_submitted_calls_with_mixed_ranges_match_twin(api, model0, cfg):
    """Submitted calls of different n in flight together (one flush per three calls); i16 I/O."""
    import torch
    S = cfg[2]
    sched = _schedule(S)
    x = torch.from_numpy(_to_i16(_inputs(S, sum(f for _, f in sched), 13))).cuda()
    a, b = _twins(api, model0, cfg)
    st = torch.cuda.current_stream().cuda_stream
    ops = _ops_stream(cfg, st)
    pending = []
    n_old, t = S, 0
    for k, (n, F) in enumerate(sched):
        _resize(a, b, n_old, n, ops)
        xa = x[:n, t * HOP:(t + F) * HOP].contiguous()
        xb = x[:, t * HOP:(t + F) * HOP].contiguous()
        oa, ob = torch.empty_like(xa), torch.empty_like(xb)
        a.submit_device(xa.data_ptr(), F * HOP, oa.data_ptr(), F * HOP, F, st, int16=True)
        b.submit_device(xb.data_ptr(), F * HOP, ob.data_ptr(), F * HOP, F, st, int16=True)
        pending.append((n, F, xa, xb, oa, ob))
        if k % 3 == 2 or k == len(sched) - 1:
            a.flush(st)
            b.flush(st)
            torch.cuda.synchronize()
            for n_, F_, _, _, oa_, ob_ in pending:
                assert torch.equal(oa_, ob_[:n_]), (n_, F_)
            pending = []
        n_old, t = n, t + F
    for e in (a, b):
        e.check(st)
        e.close()


@pytest.mark.parametrize("cfg", CONFIGS, ids=IDS)
def test_compaction_keeps_live_streams_exact(api, model0, cfg):
    """Sessions end at random slots; the last live slot moves into the hole (export n-1, import at k, shrink).  The twin
    does the same moves but keeps advancing every slot."""
    import torch
    S = cfg[2]
    F = 3
    rounds = 4
    x = _inputs(S, F * (rounds + 1), 14)
    a, b = _twins(api, model0, cfg)
    rng = np.random.RandomState(3)
    st = _ops_stream(cfg, torch.cuda.current_stream().cuda_stream)
    blob = torch.empty((1, a.state_size), dtype=torch.uint8, device="cuda")
    n = S
    for r in range(rounds + 1):
        xc = np.ascontiguousarray(x[:, r * F * HOP:(r + 1) * F * HOP])
        out_a, gr_a = a.process(xc[:n], want_gr=True)
        out_b, gr_b = b.process(xc, want_gr=True)
        assert np.array_equal(out_a, out_b[:n]) and np.array_equal(gr_a.view(np.int32), gr_b[:, :n].view(np.int32)), (r, n)
        if r == rounds:
            break
        for k in sorted(rng.choice(n, size=3, replace=False), reverse=True):  # three sessions end
            if k != n - 1:
                for e in (a, b):
                    e.export_states([n - 1], blob.data_ptr(), a.state_size, st)
                    e.import_states([int(k)], blob, stream=st)
            n -= 1
            a.set_active(n, st)
        torch.cuda.synchronize()
        assert a.active == n
    for e in (a, b):
        e.check()
        e.close()


@pytest.mark.parametrize("mode", ["fp32", "tensor"])
def test_refused_arguments_leave_engine_usable(api, model0, mode):
    import torch
    S, n = 270, 200
    e = _engine(api, model0, S, mode, Fm=8)   # 8 hops: output hop t carries input hop t-6
    L, h = e.L, e.h
    assert L.pnb_active_streams(h) == S
    for bad in (0, -1, S + 1):
        assert L.pnb_set_active_streams(h, bad, None) == -1  # PNB_ERR_ARG
    assert e.active == S
    e.set_active(n)
    blob = torch.zeros((1, e.state_size), dtype=torch.uint8, device="cuda")
    good = e.export_states([n - 1], None)
    torch.cuda.synchronize()
    for s in (n, S - 1):
        idx = np.array([s], np.int32)
        assert L.pnb_reset_streams(h, idx.ctypes.data, 1, None) == -1
        assert L.pnb_export_states(h, idx.ctypes.data, 1, blob.data_ptr(), e.state_size, None) == -1
        assert L.pnb_import_states(h, idx.ctypes.data, 1, good.data_ptr(), e.state_size, None) == -1
        buf = ctypes.create_string_buffer(e.state_size)
        assert L.pnb_get_state(h, s, buf, len(buf)) == -1
        assert L.pnb_set_state(h, s, e.get_state(0), e.state_size) == -1
    assert e.active == n
    x = _inputs(S, 8, 15)
    out, _ = e.process(x[:n])
    assert out.shape == (n, 8 * HOP) and np.abs(out).max() > 0
    e.check()
    e.reset()
    assert e.active == S and L.pnb_active_streams(h) == S
    out, _ = e.process(x)
    assert out.shape == (S, 8 * HOP)
    e.check()
    e.close()

    t = api.Engine(270, 4, None, api.TRAIN_DATA)
    assert t.L.pnb_set_active_streams(t.h, 100, None) == -1
    assert t.active == 270
    t.close()
