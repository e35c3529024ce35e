"""Ragged session calls (pnb_process_sessions_ragged_*): each listed session advances by its own number of hops in one
call of F = max(hops) hops.  Every session must match, bit for bit, a row of a plain twin engine that runs only that
session's hops back to back -- its outputs, its g/r and, at the end, its exported state.  The hops a session does not
run in a call come back as zeros, and its input beyond its own hops is never read."""
import numpy as np
import pytest

from test_gpu_lifecycle import _engine, _signal
from test_gpu_parity import api  # noqa: F401
from test_gpu_sessions import SIZES, _to_i16

pytestmark = pytest.mark.gpu

HOP = 480
FM = 16
KEEP, LINE_CALLS = 5280, 8   # history samples carried between calls; calls between two history slides (pnb_common.cuh)


def _schedule(seed, n_calls=40, N=700):
    """[(ids, hops, resets before the call)]: list sizes 1 / 127 / 128 / 129 / 256 in random order, F in {1, 3, 16};
    hop counts random in [1, F], all at F, or one at F and the rest at 1.  Sessions 600.. appear only in the second half."""
    rng = np.random.RandomState(seed)
    sizes = (SIZES * (n_calls // len(SIZES) + 1))[:n_calls]
    rng.shuffle(sizes)
    out = []
    for c, k in enumerate(sizes):
        pool = 600 if c < n_calls // 2 else N
        ids = rng.choice(pool, size=k, replace=False).astype(np.int32)
        F = int(rng.choice([1, 3, 16]))
        kind = c % 4
        if kind == 2:
            hops = np.full(k, F, np.int32)
        elif kind == 3:
            hops = np.ones(k, np.int32)
        else:
            hops = rng.randint(1, F + 1, size=k).astype(np.int32)
        hops[rng.randint(k)] = F
        resets = rng.choice(N, size=4, replace=False) if c in (11, 27) else np.empty(0, np.int64)
        out.append((ids, hops, resets))
    return out


class Twin:
    """Where each (session, epoch) lives in the twin: one row per epoch (a reset starts a new row), hops back to back."""

    def __init__(self, N, sched):
        self.row = list(range(N))
        self.pos = [0] * N
        self.calls = []
        nxt = N
        for ids, hops, resets in sched:
            for s in resets:
                self.row[s] = nxt
                nxt += 1
                self.pos.append(0)
            rows = [self.row[s] for s in ids]
            self.calls.append([(r, self.pos[r], int(h)) for r, h in zip(rows, hops)])
            for r, h in zip(rows, hops):
                self.pos[r] += int(h)
        self.R, self.H = nxt, max(self.pos)

    def inputs(self, seed, dtype):
        x = _signal(self.R, (self.H + 7) // 8, seed)[:, :self.H * HOP].copy()
        for r, n in enumerate(self.pos):
            x[r, n * HOP:] = 0.0
        return _to_i16(x) if dtype == "i16" else np.ascontiguousarray(x)

    def run(self, api, model, mode, x, Fm):
        """The twin's outputs and g/r over all hops, and every row's exported state after its own last hop."""
        t = _engine(api, model, self.R, mode, Fm=Fm)
        blobs = np.zeros((self.R, t.state_size), np.uint8)
        pos = np.asarray(self.pos)

        def export(b):
            rows = np.flatnonzero(pos == b)
            if len(rows):
                blobs[rows] = t.export_states(rows, None).cpu().numpy()
        export(0)
        outs, grs, t0 = [], [], 0
        for b in sorted(set(self.pos) - {0}):
            while t0 < b:
                t1 = min(b, t0 + Fm)
                o, g = t.process(np.ascontiguousarray(x[:, t0 * HOP:t1 * HOP]), want_gr=True)
                outs.append(o)
                grs.append(g)
                t0 = t1
            export(b)
        t.check()
        t.close()
        return np.concatenate(outs, axis=1), np.concatenate(grs, axis=0), blobs


def _ragged_inputs(x, place, F, dtype, rng):
    """Row i: the session's hops, then NaN (int16: random junk) up to F hops."""
    if dtype == "i16":
        xin = rng.randint(-32768, 32767, size=(len(place), F * HOP)).astype(np.int16)
    else:
        xin = np.full((len(place), F * HOP), np.nan, np.float32)
    for i, (r, p, h) in enumerate(place):
        xin[i, :h * HOP] = x[r, p * HOP:(p + h) * HOP]
    return xin


def _check_call(c, out, gr, place, F, out_t, gr_t, dtype):
    v = np.int16 if dtype == "i16" else np.int32
    for i, (r, p, h) in enumerate(place):
        assert np.array_equal(out[i, :h * HOP].view(v), out_t[r, p * HOP:(p + h) * HOP].view(v)), (c, i)
        assert not out[i, h * HOP:].any(), (c, i)
        if gr is not None:
            assert np.array_equal(gr[:h, i].view(np.int32), gr_t[p:p + h, r].view(np.int32)), (c, i)
            assert not gr[h:, i].any(), (c, i)


def _run_pool(api, model, mode, dtype, S, N, Fm, sched, seed):
    """The schedule on a pool of S slots and N sessions, host and device forms, d_gr null and set, device calls and resets
    alternating between two CUDA streams, nothing synchronised until the end.  Checks every call against the twin, the
    launches of every call, and every session's exported state.  Returns the number of history slides crossed."""
    import torch
    tw = Twin(N, sched)
    x = tw.inputs(seed, dtype)
    out_t, gr_t, blobs_t = tw.run(api, model, mode, x, Fm)
    e = _engine(api, model, S, mode, Fm=Fm)
    e.reserve_sessions(N)
    rng = np.random.RandomState(seed)
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    pcm_stride = KEEP + min(128 // Fm, LINE_CALLS) * Fm * HOP
    line_off, slides = 0, 0
    pending = []
    for c, ((ids, hops, resets), place) in enumerate(zip(sched, tw.calls)):
        F = int(hops.max())
        xin = _ragged_inputs(x, place, F, dtype, rng)
        sx = streams[c & 1]
        if len(resets):
            e.reset_sessions(resets, stream=sx.cuda_stream)
        before, stats = e.launches, e.session_stats()
        if c % 3 == 0:                                        # blocking host form
            want = c % 2 == 0
            out, gr = e.process_sessions(ids, xin, want_gr=want, hops=hops)
            pending.append((place, F, out, gr))
        else:
            with torch.cuda.stream(sx):
                d_in = torch.from_numpy(xin).to("cuda")
                d_out = torch.full_like(d_in, 12345) if dtype == "i16" else torch.full_like(d_in, float("nan"))
                want = c % 2 == 1
                d_gr = torch.full((F, len(ids), 68), float("nan"), device="cuda") if want else None
                e.process_sessions_device(ids, d_in.data_ptr(), F * HOP, d_out.data_ptr(), F * HOP, 0,
                                          d_gr.data_ptr() if want else 0, sx.cuda_stream, int16=(dtype == "i16"), hops=hops)
            pending.append((place, F, d_out, d_gr, d_in))
        # launches: a plain call of F hops, the state launch when anything moved, the g/r gather, the fix-up when a
        # session stopped early, the history slide when the line is used up
        line_off += F * HOP
        slide = line_off + KEEP + Fm * HOP > pcm_stride
        if slide:
            line_off, slides = 0, slides + 1
        moved = e.session_stats() != stats
        want_launches = e.launches_per_call(F) + moved + want + bool((hops < F).any()) + slide
        assert e.launches - before == want_launches, c
    torch.cuda.synchronize()
    e.check()
    for c, p in enumerate(pending):
        place, F, out, gr = p[:4]
        if not isinstance(out, np.ndarray):
            out = out.cpu().numpy()
            gr = None if gr is None else gr.cpu().numpy()
        _check_call(c, out, gr, place, F, out_t, gr_t, dtype)
    assert np.abs(out_t.astype(np.float32)).max() > 0
    blobs = e.export_sessions(np.arange(N), None).cpu().numpy()
    for s in range(N):
        assert np.array_equal(blobs[s], blobs_t[tw.row[s]]), s
    e.check()
    e.close()
    return slides


@pytest.mark.parametrize("dtype", ["f32", "i16"])
@pytest.mark.parametrize("mode", ["fp32", "tensor"])
def test_ragged_pool_matches_twin(api, model0, mode, dtype):
    """256 slots, 700 sessions, 40 calls of per-session hop counts; outputs, g/r and final states equal the twin's."""
    slides = _run_pool(api, model0, mode, dtype, 256, 700, FM, _schedule(17 if mode == "fp32" else 18), 31)
    assert slides >= 1


def _schedule_hop_major(seed, h, S, N, n_calls=10):
    """Like _schedule, with list sizes h - 1 / h / S (h = first_hop_major: the chain's anti-diagonal order, then
    hop-major) so consecutive calls change order, F in {1, 4, 9}, resets before call 5."""
    rng = np.random.RandomState(seed)
    sizes = [h - 1, h, S] * (n_calls // 3 + 1)
    rng.shuffle(sizes)
    out = []
    for c, k in enumerate(sizes[:n_calls]):
        ids = rng.choice(N, size=k, replace=False).astype(np.int32)
        F = int(rng.choice([1, 4, 9]))
        kind = c % 4
        if kind == 2:
            hops = np.full(k, F, np.int32)
        elif kind == 3:
            hops = np.ones(k, np.int32)
        else:
            hops = rng.randint(1, F + 1, size=k).astype(np.int32)
        hops[rng.randint(k)] = F
        resets = rng.choice(N, size=4, replace=False) if c == 5 else np.empty(0, np.int64)
        out.append((ids, hops, resets))
    return out


def test_ragged_pool_matches_twin_hop_major(api, model0):
    """A tensor pool of first_hop_major + 255 slots and 300 more sessions: list sizes on both sides of the chain's
    switch to hop-major order, so frozen rows (hops beyond a session's count store nothing) and session moves run in
    both orders and calls change order.  Outputs, g/r and final states equal the twin's."""
    from util import device_first_hop_major
    h = device_first_hop_major()
    S = h + 255
    N = S + 300
    _run_pool(api, model0, "tensor", "f32", S, N, 9, _schedule_hop_major(19, h, S, N), 37)


def test_fp32_chunks(api, model0):
    """An fp32 pool with max_frames = 40: hop counts 1, 31, 32, 33 and 40 straddle the 32-hop chunk of the fp32 network."""
    rng = np.random.RandomState(5)
    sched = []
    for c in range(6):
        ids = rng.choice(12, size=int(rng.choice([5, 8])), replace=False).astype(np.int32)
        hops = rng.choice([1, 31, 32, 33, 40], size=len(ids)).astype(np.int32)
        hops[0] = [40, 33, 32, 31, 40, 33][c]
        sched.append((ids, hops, np.empty(0, np.int64)))
    _run_pool(api, model0, "fp32", "f32", 8, 12, 40, sched, 9)


@pytest.mark.parametrize("mode", ["fp32", "tensor"])
def test_uniform_hops_are_the_plain_session_call(api, model0, mode):
    """A ragged call whose hops are all equal issues the launches of pnb_process_sessions_* and gives the same bits."""
    import torch
    a, b = _engine(api, model0, 130, mode, Fm=8), _engine(api, model0, 130, mode, Fm=8)
    for e in (a, b):
        e.reserve_sessions(300)
    rng = np.random.RandomState(3)
    x = _signal(130, 1, 6)
    for c in range(6):
        k, F = int(rng.choice([1, 64, 129, 130])), int(rng.choice([1, 5, 8]))
        ids = rng.choice(300, size=k, replace=False).astype(np.int32)
        xin = np.ascontiguousarray(x[:k, :F * HOP])
        la, lb = a.launches, b.launches
        if c % 2:
            oa, ga = a.process_sessions(ids, xin, want_gr=True, hops=np.full(k, F, np.int32))
            ob, gb = b.process_sessions(ids, xin, want_gr=True)
        else:
            d_in = torch.from_numpy(xin).cuda()
            outs = [torch.empty_like(d_in) for _ in range(2)]
            grs = [torch.empty((F, k, 68), device="cuda") for _ in range(2)]
            a.process_sessions_device(ids, d_in.data_ptr(), F * HOP, outs[0].data_ptr(), F * HOP, F, grs[0].data_ptr(),
                                      hops=np.full(k, F, np.int32))
            b.process_sessions_device(ids, d_in.data_ptr(), F * HOP, outs[1].data_ptr(), F * HOP, F, grs[1].data_ptr())
            torch.cuda.synchronize()
            (oa, ob), (ga, gb) = [o.cpu().numpy() for o in outs], [g.cpu().numpy() for g in grs]
        assert a.launches - la == b.launches - lb, c
        assert np.array_equal(oa.view(np.int32), ob.view(np.int32)) and np.array_equal(ga.view(np.int32), gb.view(np.int32)), c
    for e in (a, b):
        e.check()
        e.close()


def test_domain_flag_is_masked_for_frozen_hops(api, model0):
    """The conv2 epilogue raises PNB_ERR_DOMAIN only for hops a session runs.  A session's conv1 history is set to
    hist[0] = 0, hist[1] = alpha sign(W2[0:512, col]): its hop 1 reads hist[1] through conv2's tap 0 at >= 1.5 x 8.5e7,
    its hop 0 reads it through tap 1, inside the domain for every column.  Run for 1 hop in a 2-hop call it raises
    nothing; run for 2 hops it raises."""
    import torch
    from percepnet_b200.synth import synth_pcm
    from test_gpu_layer_bounds import BLOB, DOMAIN
    a = model0.arrays
    W2 = a["conv2_weights"].reshape(1536, 512).astype(np.float64)
    b2 = a["conv2_bias"].astype(np.float64)
    col = int(np.argmax(np.abs(W2[:512]).sum(0)))
    # what a hop's own conv1 output (|.| < 100 for a unit-scale signal) and the bias can add, in float64
    slack = np.abs(b2).max() + np.abs(W2[512:]).sum(0).max() * 100.0
    alpha = (1.5 * DOMAIN + slack) / np.abs(W2[:512, col]).sum()
    sg = np.sign(W2[:512, col])
    assert alpha * np.abs(W2[:512, col]).sum() - slack >= 1.5 * DOMAIN                         # hop 1, tap 0
    assert (np.abs(b2 + alpha * sg @ W2[512:1024]) + np.abs(W2[1024:]).sum(0) * 100.0).max() < 0.5 * DOMAIN  # hop 0
    x = synth_pcm(2, 2, seed=4)

    def run(h_session, h_neighbour):
        e = _engine(api, model0, 4, "tensor", Fm=2)
        try:
            e.reserve_sessions(8)
            raw = e.export_sessions([5], None).cpu().numpy()
            v = raw.view(BLOB).reshape(-1)
            v["c1_hist"][0, 0] = 0.0
            v["c1_hist"][0, 1] = (alpha * sg).astype(np.float32)
            v["has_terms"][0] = 0
            e.import_sessions([5], torch.from_numpy(raw).cuda())
            hops = np.array([h_session, h_neighbour], np.int32)
            e.process_sessions(np.array([5, 2], np.int32), np.ascontiguousarray(x[:, :int(hops.max()) * HOP]), hops=hops)
            e.check()
            return "ok"
        except api.PnbError as err:
            return str(err)
        finally:
            e.close()

    assert run(1, 2) == "ok"
    for hs, hn in ((2, 2), (2, 1)):
        verdict = run(hs, hn)
        assert "-5" in verdict, verdict


@pytest.mark.parametrize("mode", ["fp32", "tensor"])
def test_refusals(api, model0, mode):
    """hops NULL, a hop of 0 or above max_frames, a stride below max(hops) x 480 and a call before pnb_sessions_reserve
    return PNB_ERR_ARG, change nothing, and the next valid call continues like a pool that never saw them."""
    S, N = 8, 16
    e, t = _engine(api, model0, S, mode, Fm=4), _engine(api, model0, S, mode, Fm=4)
    L, h = e.L, e.h
    ids = np.array([3, 11, 0], np.int32)
    hops = np.array([4, 2, 1], np.int32)
    x = _signal(3, 2, 8)
    x1, x2 = np.ascontiguousarray(x[:, :4 * HOP]), np.ascontiguousarray(x[:, 4 * HOP:8 * HOP])
    out = np.empty_like(x1)

    def host(i=ids, hp=hops, stride=4 * HOP, n=3):
        return L.pnb_process_sessions_ragged_host_f32(h, i.ctypes.data, None if hp is None else hp.ctypes.data, n,
                                                      x2.ctypes.data, stride, out.ctypes.data, 4 * HOP, None)
    assert host() == -1                                       # before pnb_sessions_reserve
    for p in (e, t):
        p.reserve_sessions(N)
        p.process_sessions(ids, x1, hops=hops)
    before = e.session_stats()
    assert host(hp=None) == -1
    assert host(hp=np.array([4, 0, 1], np.int32)) == -1
    assert host(hp=np.array([4, 5, 1], np.int32)) == -1
    assert host(stride=4 * HOP - 1) == -1
    assert host(i=np.array([3, 3, 0], np.int32)) == -1
    assert host(n=0) == -1
    assert L.pnb_process_sessions_ragged_device_f32(h, ids.ctypes.data, hops.ctypes.data, 3, None, 4 * HOP, None, 4 * HOP,
                                                    None, None) == -1
    assert e.session_stats() == before
    o, g = e.process_sessions(ids, x2, want_gr=True, hops=hops[::-1].copy())
    ot, gt = t.process_sessions(ids, x2, want_gr=True, hops=hops[::-1].copy())
    assert np.array_equal(o.view(np.int32), ot.view(np.int32)) and np.array_equal(g.view(np.int32), gt.view(np.int32))
    for p in (e, t):
        p.check()
        p.close()
