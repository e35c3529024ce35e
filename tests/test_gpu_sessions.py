"""Session pool (pnb_sessions_reserve / pnb_process_sessions_*): calls advance any listed subset of sessions, the others
keep their state.  Every session must match, bit for bit, a row of a plain twin engine that runs only that session's
participating hops back to back (outputs are causal and independent of batch neighbours and of how hops are grouped into
calls).  A session reset mid-run is a fresh twin row from that hop on."""
import ctypes

import numpy as np
import pytest

from test_gpu_lifecycle import _engine, _signal
from test_gpu_parity import api  # noqa: F401

pytestmark = pytest.mark.gpu

HOP = 480
FM = 16
SIZES = [1, 127, 128, 129, 256]


def _to_i16(x):
    return np.clip(np.rint(x * 16384.0), -32768, 32767).astype(np.int16)


def _schedule(seed, n_calls=40, S=256, N=700):
    """[(ids, F, resets before the call)]: list sizes 1 / 127 / 128 / 129 / 256 in random order, F in {1, 3, 16};
    sessions 600.. appear only in the second half, so most sessions skip many calls and some first appear late."""
    rng = np.random.RandomState(seed)
    sizes = (SIZES * (n_calls // len(SIZES) + 1))[:n_calls]
    rng.shuffle(sizes)
    out = []
    for c, k in enumerate(sizes):
        pool = 600 if c < n_calls // 2 else N
        ids = rng.choice(pool, size=min(k, S), replace=False).astype(np.int32)
        resets = rng.choice(N, size=4, replace=False) if c in (11, 27) else np.empty(0, np.int64)
        out.append((ids, int(rng.choice([1, 3, 16])), resets))
    return out


class Twin:
    """Where each (session, epoch) lives in the twin: one row per epoch (a reset starts a new row), hops back to back."""

    def __init__(self, N, sched):
        self.row = list(range(N))
        self.pos = [0] * N
        self.calls = []
        nxt = N
        for ids, F, resets in sched:
            for s in resets:
                self.row[s] = nxt
                nxt += 1
                self.pos.append(0)
            rows = [self.row[s] for s in ids]
            self.calls.append([(r, self.pos[r]) for r in rows])
            for r in rows:
                self.pos[r] += F
        self.R, self.H = nxt, max(self.pos)

    def inputs(self, seed, dtype):
        x = _signal(self.R, (self.H + 7) // 8, seed)[:, :self.H * HOP].copy()
        for r, n in enumerate(self.pos):
            x[r, n * HOP:] = 0.0
        return _to_i16(x) if dtype == "i16" else np.ascontiguousarray(x)


def _twin_run(api, model0, mode, x):
    t = _engine(api, model0, x.shape[0], mode, Fm=FM)
    out, gr = t.process_stream_chunks(x, want_gr=True)
    t.check()
    t.close()
    return out, gr


def _gather(x, place, F):
    return np.ascontiguousarray(np.stack([x[r, p * HOP:(p + F) * HOP] for r, p in place]))


@pytest.mark.parametrize("dtype", ["f32", "i16"])
@pytest.mark.parametrize("mode", ["fp32", "tensor"])
def test_pool_matches_twin(api, model0, mode, dtype):
    """256 slots, 700 sessions, 40 calls; host and device entry points, d_gr null and set, device calls and resets
    alternating between two non-default CUDA streams, nothing synchronised until the end."""
    import torch
    S, N = 256, 700
    sched = _schedule(7 if mode == "fp32" else 8)
    tw = Twin(N, sched)
    x = tw.inputs(21, dtype)
    out_t, gr_t = _twin_run(api, model0, mode, x)
    e = _engine(api, model0, S, mode, Fm=FM)
    e.reserve_sessions(N)
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    pending = []
    for c, ((ids, F, resets), place) in enumerate(zip(sched, tw.calls)):
        xin = _gather(x, place, F)
        sx = streams[c & 1]
        if len(resets):
            e.reset_sessions(resets, stream=sx.cuda_stream)
        if c % 3 == 0:                                        # blocking host form
            out, gr = e.process_sessions(ids, xin, want_gr=(c % 2 == 0))
            pending.append((place, F, out, gr))
            continue
        with torch.cuda.stream(sx):
            d_in = torch.from_numpy(xin).to("cuda", non_blocking=False)
            d_out = torch.empty_like(d_in)
            d_gr = torch.empty((F, len(ids), 68), device="cuda") if c % 2 else None
            e.process_sessions_device(ids, d_in.data_ptr(), F * HOP, d_out.data_ptr(), F * HOP, F,
                                      d_gr.data_ptr() if d_gr is not None else 0, sx.cuda_stream, int16=(dtype == "i16"))
        pending.append((place, F, d_out, d_gr, d_in))
    torch.cuda.synchronize()
    e.check()
    for c, p in enumerate(pending):
        place, F, out, gr = p[:4]
        if not isinstance(out, np.ndarray):
            out = out.cpu().numpy()
            gr = None if gr is None else gr.cpu().numpy()
        v = np.int16 if dtype == "i16" else np.int32
        assert np.array_equal(out.view(v), _gather(out_t, place, F).view(v)), c
        if gr is not None:
            want_gr = np.stack([gr_t[p0:p0 + F, r] for r, p0 in place], axis=1)
            assert np.array_equal(gr.view(np.int32), want_gr.view(np.int32)), c
    assert np.abs(out_t.astype(np.float32)).max() > 0
    st = e.session_stats()
    assert st["unparks"] >= len({int(s) for ids, _, _ in sched for s in ids}) and st["parks"] > 0 and st["relocations"] > 0
    e.close()


def test_move_counts_on_gpu(api, model0):
    """Through pnb_session_stats, the minimal counts of the planner."""
    e = _engine(api, model0, 16, "tensor", Fm=2)
    e.reserve_sessions(48)
    x = _signal(16, 1, 3)[:, :2 * HOP]

    def step(ids):
        before = e.session_stats()
        e.process_sessions(np.asarray(ids, np.int32), np.ascontiguousarray(x[:len(ids)]))
        after = e.session_stats()
        return [after[k] - before[k] for k in ("parks", "unparks", "relocations")]

    base = list(range(10, 22))
    assert step(base) == [0, 12, 0]
    assert step(base[::-1]) == [0, 0, 0]
    assert step(list(np.random.RandomState(1).permutation(base))) == [0, 0, 0]
    assert step(base[:-1]) == [1, 0, 0]                       # the last slot's session leaves
    assert step(base[:-1] + [40]) == [0, 1, 0]
    cur = base[:-1] + [40]
    d = step(cur[:4] + cur[8:])                               # k 12 -> 8: four leave, four relocate
    assert d == [4, 0, 4]
    e.check()
    e.close()


def _continue(e, ids, x, pooled=True):
    if pooled:
        return e.process_sessions(np.asarray(ids, np.int32), x, want_gr=True)
    return e.process(x, want_gr=True)


def test_blobs_move_between_pooled_and_plain_engines(api, model0):
    """Export from a pooled tensor engine of 256 slots (resident and parked sessions), import into a pooled engine of 130
    slots and, through pnb_set_state, into a plain engine: all three continue bit for bit.  An fp32-mode blob imported
    into a tensor pool is accepted and continues like pnb_set_state of the same blob."""
    import torch
    a = _engine(api, model0, 256, "tensor", Fm=8)
    a.reserve_sessions(700)
    x = _signal(700, 3, 5)
    a.process_sessions(np.arange(0, 200, dtype=np.int32), np.ascontiguousarray(x[0:200, :8 * HOP]))
    a.process_sessions(np.arange(100, 300, dtype=np.int32), np.ascontiguousarray(x[100:300, :8 * HOP]))
    moved = np.array([150, 299, 5, 60], np.int32)            # two resident, two parked
    blobs = a.export_sessions(moved, None)
    torch.cuda.synchronize()
    b = _engine(api, model0, 130, "tensor", Fm=8)
    b.reserve_sessions(300)
    b_ids = np.array([7, 250, 0, 129], np.int32)
    b.process_sessions(np.arange(30, 160, dtype=np.int32), np.ascontiguousarray(x[:130, :8 * HOP]))  # occupy slots
    b.import_sessions(b_ids, blobs)
    c = _engine(api, model0, 4, "tensor", Fm=8)
    host = blobs.cpu().numpy()
    for i in range(4):
        c.set_state(i, host[i].tobytes())
    xn = np.ascontiguousarray(x[:4, 16 * HOP:24 * HOP])
    oa, ga = _continue(a, moved, xn)
    ob, gb = _continue(b, b_ids, xn)
    oc, gc = _continue(c, None, xn, pooled=False)
    assert np.array_equal(oa.view(np.int32), oc.view(np.int32)) and np.array_equal(ob.view(np.int32), oc.view(np.int32))
    assert np.array_equal(ga.view(np.int32), gc.view(np.int32)) and np.array_equal(gb.view(np.int32), gc.view(np.int32))
    for e in (a, b, c):
        e.check()

    f = _engine(api, model0, 8, "fp32", Fm=8)
    f.reserve_sessions(16)
    f.process_sessions(np.array([3, 4], np.int32), np.ascontiguousarray(x[:2, :8 * HOP]))
    fb = f.export_sessions([4], None)
    torch.cuda.synchronize()
    b.import_sessions([9], fb)
    b.wait()                                                  # accepted: no rejection reported
    c.set_state(0, fb.cpu().numpy()[0].tobytes())
    ob, gb = _continue(b, [9, 7], np.ascontiguousarray(xn[:2]))
    oc, gc = _continue(c, None, xn, pooled=False)
    assert np.array_equal(ob[0].view(np.int32), oc[0].view(np.int32)) and np.array_equal(gb[:, 0].view(np.int32), gc[:, 0].view(np.int32))
    for e in (b, c, f):
        e.check()
        e.close()
    a.close()


def test_rejected_blob_leaves_session_fresh(api, model0):
    """A bad magic or a GRU value above 1.0001 is rejected: the session is fresh, and PNB_ERR_ARG is reported once,
    naming the lowest rejected session id."""
    import torch
    e = _engine(api, model0, 16, "tensor", Fm=4)
    e.reserve_sessions(64)
    x = _signal(16, 1, 9)
    e.process_sessions(np.arange(8, dtype=np.int32), np.ascontiguousarray(x[:8, :4 * HOP]))
    good = e.export_sessions([0, 1, 2], None)
    torch.cuda.synchronize()
    bad = good.clone()
    bad[0, :4] = 0                                            # magic
    gru = np.frombuffer(bad[2].cpu().numpy().tobytes(), np.uint8).copy()
    gru[45880:45884] = np.frombuffer(np.float32(1.01).tobytes(), np.uint8)  # StreamState.h[0]
    bad[2] = torch.from_numpy(gru).cuda()
    e.import_sessions([40, 3, 12], bad)                       # 40 and 12 rejected, 3 accepted
    rc = e.L.pnb_wait(e.h)
    assert rc == -1 and b"session 12" in e.L.pnb_last_error()
    assert e.L.pnb_wait(e.h) == 0                             # reported once
    fresh = _engine(api, model0, 2, "tensor", Fm=4)
    fresh.set_state(1, good.cpu().numpy()[1].tobytes())
    xn = np.ascontiguousarray(x[8:10, :4 * HOP])
    o, g = e.process_sessions(np.array([12, 3], np.int32), xn, want_gr=True)
    of, gf = fresh.process(xn, want_gr=True)
    assert np.array_equal(o.view(np.int32), of.view(np.int32)) and np.array_equal(g.view(np.int32), gf.view(np.int32))
    e.check()
    for t in (e, fresh):
        t.close()


@pytest.mark.parametrize("mode", ["fp32", "tensor"])
def test_reset_and_refusals(api, model0, mode):
    """pnb_reset in session mode makes every session fresh; every refused argument and every slot-level call returns
    PNB_ERR_ARG and leaves the pool as it was."""
    import torch
    S, N = 130, 300
    e = _engine(api, model0, S, mode, Fm=4)
    L, h = e.L, e.h
    ids = np.array([5, 299, 0, 131], np.int32)
    x = _signal(4, 2, 4)
    x1, x2 = np.ascontiguousarray(x[:, :4 * HOP]), np.ascontiguousarray(x[:, 4 * HOP:8 * HOP])
    out = np.empty_like(x2)
    assert L.pnb_process_sessions_host_f32(h, ids.ctypes.data, 4, x1.ctypes.data, 4 * HOP, out.ctypes.data, 4 * HOP, 4,
                                           None) == -1  # before pnb_sessions_reserve
    e.reserve_sessions(N)
    o1, _ = e.process_sessions(ids, x1)
    o2, _ = e.process_sessions(ids[::-1], x2[::-1])
    e.reset()
    assert np.array_equal(e.process_sessions(ids, x1)[0].view(np.int32), o1.view(np.int32))
    before = e.session_stats()
    d = torch.zeros((4, 4 * HOP), device="cuda")
    blob = torch.zeros((1, e.state_size), dtype=torch.uint8, device="cuda")

    def host(i, n=4, inp=x2, F=4, stride=4 * HOP):
        return L.pnb_process_sessions_host_f32(h, i.ctypes.data, n, inp.ctypes.data, stride, out.ctypes.data, 4 * HOP, F, None)
    for bad in (np.array([5, 299, 0, 5], np.int32), np.array([5, 300, 0, 1], np.int32), np.array([5, -1, 0, 1], np.int32)):
        assert host(bad) == -1
    assert host(ids, n=0) == -1 and host(ids, n=S + 1) == -1
    assert host(ids, F=0) == -1 and host(ids, F=5) == -1 and host(ids, stride=4 * HOP - 1) == -1
    assert L.pnb_process_sessions_host_f32(h, None, 4, x2.ctypes.data, 4 * HOP, out.ctypes.data, 4 * HOP, 4, None) == -1
    assert L.pnb_process_sessions_device_f32(h, ids.ctypes.data, 4, None, 4 * HOP, d.data_ptr(), 4 * HOP, 4, None, None) == -1
    assert L.pnb_export_sessions(h, ids.ctypes.data, 1, blob.data_ptr(), e.state_size - 4, None) == -1
    assert L.pnb_import_sessions(h, ids.ctypes.data, 1, None, e.state_size, None) == -1
    assert L.pnb_reset_sessions(h, np.array([N], np.int32).ctypes.data, 1, None) == -1
    # slot-level calls in session mode
    one = np.array([0], np.int32)
    assert L.pnb_process_host_f32(h, x2.ctypes.data, 4 * HOP, out.ctypes.data, 4 * HOP, 4, None) == -1
    assert L.pnb_submit_host_f32(h, x2.ctypes.data, 4 * HOP, out.ctypes.data, 4 * HOP, 4) == -1
    assert L.pnb_process_device_f32(h, d.data_ptr(), 4 * HOP, d.data_ptr(), 4 * HOP, 4, None, None) == -1
    assert L.pnb_submit_device_f32(h, d.data_ptr(), 4 * HOP, d.data_ptr(), 4 * HOP, 4, None) == -1
    assert L.pnb_set_active_streams(h, 4, None) == -1
    assert L.pnb_reset_streams(h, one.ctypes.data, 1, None) == -1
    assert L.pnb_export_states(h, one.ctypes.data, 1, blob.data_ptr(), e.state_size, None) == -1
    assert L.pnb_import_states(h, one.ctypes.data, 1, blob.data_ptr(), e.state_size, None) == -1
    buf = ctypes.create_string_buffer(e.state_size)
    assert L.pnb_get_state(h, 0, buf, len(buf)) == -1 and L.pnb_set_state(h, 0, buf, len(buf)) == -1
    assert e.session_stats() == before
    # the next valid call continues like the run without reset
    assert np.array_equal(e.process_sessions(ids[::-1], x2[::-1])[0].view(np.int32), o2.view(np.int32))
    e.check()
    e.close()
    t = api.Engine(270, 4, None, api.TRAIN_DATA)
    assert t.L.pnb_sessions_reserve(t.h, 10) == -1
    t.close()


@pytest.mark.parametrize("mode", ["fp32", "tensor"])
def test_session_state_launches(api, model0, mode):
    """pnb_launch_count grows by each session operation's own launches: one for a reset, a blob check and the blob
    rewrite for an import, and for an export one per kind of session listed (resident ones from their slots, parked
    ones from their parking blobs); none for n = 0."""
    import torch
    e = _engine(api, model0, 16, mode, Fm=4)
    e.reserve_sessions(64)
    x = _signal(16, 1, 9)
    e.process_sessions(np.arange(8, dtype=np.int32), np.ascontiguousarray(x[:8, :4 * HOP]))   # 0..7 resident
    blobs = e.export_sessions([0, 1], None)
    ops = [("export resident", lambda: e.export_sessions([2, 5, 3], None), 1),
           ("export parked", lambda: e.export_sessions([40, 20], None), 1),
           ("export mixed", lambda: e.export_sessions([41, 4, 21], None), 2),
           ("reset", lambda: e.reset_sessions([6, 30]), 1),
           ("import", lambda: e.import_sessions([7, 31], blobs), 2),
           ("reset n 0", lambda: e.reset_sessions([]), 0),
           ("export n 0", lambda: e.export_sessions([], None), 0),
           ("import n 0", lambda: e.import_sessions([], 0), 0)]
    for name, op, want in ops:
        n = e.launches
        op()
        assert e.launches - n == want, name
    torch.cuda.synchronize()
    e.check()
    e.close()
