"""Split and network calls on a session pool (pnb_analyze_sessions_*, pnb_synthesize_sessions_*,
pnb_compute_rnn_sessions_*): analyze -> the network's g/r -> synthesize on a list of sessions is the fused
pnb_process_sessions_* (or _ragged_*) call bit for bit -- output, g/r, features, residency counts and every session's
blob -- with sessions joining, parking, returning, relocating and listed in another order.  Network calls on sessions
alone match one plain engine per session, and every refusal launches nothing."""
import numpy as np
import pytest

from test_gpu_lifecycle import _engine
from test_gpu_parity import api  # noqa: F401
from test_gpu_sessions import _to_i16
from util import crowd, same_bits

pytestmark = pytest.mark.gpu

HOP = 480
KEEP, LINE_CALLS = 5280, 8   # history samples carried between calls; calls between two history slides (pnb_common.cuh)
SIGNAL_BYTES = 39736         # offsetof(StreamState, fc_hist): the blob's signal part
S, N, FM = 13, 40, 4
F_SEQ = [4, 3, 4, 2, 4, 4, 3, 4, 4, 3]   # 35 hops: the history slides once, after the call that crosses 28 hops


def _flags(api, mode):
    return {"fp32": api.NN_FP32, "tensor": api.NN_TENSOR, "tensor_wide": api.NN_TENSOR | api.CONV_WIDE}[mode]


def _lists(seed):
    """Ten session lists on 13 slots and 40 sessions: sessions join, sit calls out (parked) and return, residents of
    slots >= k relocate when the list shrinks, and the same set comes back in another order."""
    rng = np.random.RandomState(seed)
    c6 = rng.choice(N, 13, replace=False)
    c8 = rng.choice(N, 13, replace=False)
    lists = [np.arange(10), np.arange(13), np.r_[5:13, 20:25], np.r_[0, 1, 2, 12, 11, 10, 9, 8],
             np.r_[9, 0, 12, 2, 8, 1, 11, 10], np.r_[8, 9, 20, 21], c6, rng.choice(N, 7, replace=False), c8, c8[::-1]]
    return [np.ascontiguousarray(ids, np.int32) for ids in lists]


def _hops(ids, F, c, rng, ragged):
    """None, or one of three patterns by call: 1 hop or F (F = max_frames on some calls), one short session, all F."""
    if not ragged:
        return None
    k = len(ids)
    kind = c % 3
    if kind == 0:
        h = rng.choice([1, F], size=k).astype(np.int32)
    elif kind == 1:
        h = np.full(k, F, np.int32)
        if F > 1:
            h[rng.randint(k)] = rng.randint(1, F)
    else:
        h = np.full(k, F, np.int32)
    h[rng.randint(k)] = F
    return h


class Plan:
    """The slot of each listed session (pnb_session_plan.h): a listed resident of a slot < k stays; every other listed
    session takes the lowest free slot < k, in list order; after the call the residents are exactly the list."""

    def __init__(self):
        self.where = np.full(N, -1)

    def slots(self, ids):
        k = len(ids)
        row = np.full(k, -1)
        for i, s in enumerate(ids):
            if 0 <= self.where[s] < k:
                row[self.where[s]] = i
        p = 0
        for i, s in enumerate(ids):
            if 0 <= self.where[s] < k:
                continue
            while row[p] >= 0:
                p += 1
            row[p] = i
        self.where[:] = -1
        self.where[ids[row]] = np.arange(k)
        return self.where[ids].copy()


def _inputs(x, pos, ids, hops, F, i16, rng):
    """Row i: the session's next hops, then NaN (int16: junk) up to F hops."""
    h = np.full(len(ids), F) if hops is None else hops
    xin = np.full((len(ids), F * HOP), np.nan, np.float32)
    for i, s in enumerate(ids):
        xin[i, :h[i] * HOP] = x[s, pos[s] * HOP:(pos[s] + h[i]) * HOP]
    if i16:
        junk = rng.randint(-32768, 32767, size=xin.shape).astype(np.int16)
        return np.where(np.isnan(xin), junk, _to_i16(np.nan_to_num(xin)))
    return xin


def _dev(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _host(t):
    import torch
    if isinstance(t, np.ndarray):
        return t
    torch.cuda.synchronize()
    return t.cpu().numpy()


def _fused(A, ids, xin, hops, F, device):
    if not device:
        return A.process_sessions(ids, xin, want_gr=True, hops=hops)
    import torch
    d_in = _dev(xin)
    d_out = torch.empty_like(d_in)
    d_gr = torch.empty((F, len(ids), 68), device="cuda")
    torch.cuda.synchronize()
    A.process_sessions_device(ids, d_in.data_ptr(), F * HOP, d_out.data_ptr(), F * HOP, F, d_gr.data_ptr(),
                              int16=xin.dtype == np.int16, hops=hops)
    return _host(d_out), _host(d_gr)


def _split(api, B, ids, xin, hops, F, forms, streams, caller_gr=None):
    """B's analyze -> compute_rnn (or the caller's g/r) -> synthesize, each half in its host or device form.  The device
    buffers are made first; device halves then go to alternating torch streams with nothing between them but the
    engine's own ordering.  Returns (out, g/r [n, F, 68], features [n, F, 70], the launches of each half)."""
    import torch
    n, i16 = len(ids), xin.dtype == np.int16
    d_in = _dev(xin)
    d_feat = torch.full((n, F, 70), -7.0, device="cuda")
    d_gr = _dev(caller_gr) if caller_gr is not None else torch.full((n, F, 68), -7.0, device="cuda")
    d_out = torch.full((n, F * HOP), 12345 if i16 else float("nan"), device="cuda", dtype=torch.int16 if i16 else torch.float32)
    torch.cuda.synchronize()
    counts, feat, gr, out = [], None, caller_gr, None
    l0 = B.launches
    if forms[0] == "host":
        feat = B.analyze_sessions(ids, xin, hops=hops)
        d_feat.copy_(torch.from_numpy(feat))
        torch.cuda.synchronize()
    else:
        B.analyze_sessions_device(ids, d_in.data_ptr(), F * HOP, F, d_feat.data_ptr(), F * 70,
                                  stream=streams[0].cuda_stream, int16=i16, hops=hops)
    counts.append(B.launches - l0)
    l0 = B.launches
    if caller_gr is None and forms[1] == "host":
        feat = _host(d_feat) if feat is None else feat
        gr = B.compute_rnn_sessions(ids, feat, hops=hops)
        d_gr.copy_(torch.from_numpy(gr))
        torch.cuda.synchronize()
    elif caller_gr is None:
        B.compute_rnn_sessions_device(ids, api.RNN_FEATURES, d_feat.data_ptr(), F * 70, F, d_gr.data_ptr(), F * 68,
                                      stream=streams[1].cuda_stream, hops=hops)
    counts.append(B.launches - l0)
    l0 = B.launches
    if forms[2] == "host":
        gr = _host(d_gr) if gr is None else gr
        out = B.synthesize_sessions(ids, gr, int16=i16)
    else:
        B.synthesize_sessions_device(ids, d_gr.data_ptr(), F * 68, F, d_out.data_ptr(), F * HOP,
                                     stream=streams[0].cuda_stream, int16=i16)
    counts.append(B.launches - l0)
    torch.cuda.synchronize()
    return (_host(d_out) if out is None else out, _host(d_gr) if gr is None else gr,
            _host(d_feat) if feat is None else feat, counts)


FORMS = [("host", "host", "host"), ("device", "device", "device"), ("host", "device", "host"), ("device", "host", "device")]
CASES = [("fp32", False), ("tensor", False), ("tensor_wide", False), ("tensor", True)]


def _run(api, model, mode, post, ragged, seed, caller_gr=False):
    import torch
    flags = _flags(api, mode) | (api.POSTFILTER if post else 0)
    A, B = _engine(api, model, S, mode, Fm=FM, flags=flags), _engine(api, model, S, mode, Fm=FM, flags=flags)
    for e in (A, B):
        e.reserve_sessions(N)
    x = crowd(N, sum(F_SEQ) + 1, seed=seed)
    pos = np.zeros(N, np.int64)
    rng = np.random.RandomState(seed)
    plan = Plan()
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    pcm_stride = KEEP + min(128 // FM, LINE_CALLS) * FM * HOP
    line_off, slides, shorts = 0, 0, 0
    for c, (ids, F) in enumerate(zip(_lists(seed), F_SEQ)):
        hops = _hops(ids, F, c, rng, ragged)
        h = np.full(len(ids), F) if hops is None else hops
        xin = _inputs(x, pos, ids, hops, F, c % 2 == 1, rng)
        tag = (c, list(ids), None if hops is None else list(hops))
        la, st = A.launches, A.session_stats()
        want, want_gr = _fused(A, ids, xin, hops, F, device=c % 4 in (1, 3))
        fused_launches = A.launches - la
        tap = A.read_tap("features", F)[:, plan.slots(ids)].transpose(1, 0, 2)
        got, gr, feat, counts = _split(api, B, ids, xin, hops, F, FORMS[c % 4], streams,
                                       caller_gr=want_gr.transpose(1, 0, 2).copy() if caller_gr else None)
        moved = A.session_stats() != st
        short = bool((h < F).any())
        line_off += F * HOP
        slide = line_off + KEEP + FM * HOP > pcm_stride
        if slide:
            line_off, slides = 0, slides + 1
        shorts += short
        assert B.session_stats() == A.session_stats(), tag
        assert (np.array_equal(got, want) if got.dtype == np.int16 else same_bits(got, want)), tag
        assert same_bits(gr, want_gr.transpose(1, 0, 2)), tag
        for i in range(len(ids)):
            assert same_bits(feat[i, :h[i]], tap[i, :h[i]]), (tag, i)
            assert not feat[i, h[i]:].any() and not gr[i, h[i]:].any(), (tag, i)
        # the launches the header documents
        net = A.launches_per_call(F) - 3
        assert fused_launches == 3 + net + moved + 1 + short + slide, tag
        want_counts = [moved + 3, 0 if caller_gr else 2 + net, 2 + short + slide]
        assert counts == want_counts, (tag, counts, want_counts)
        pos[ids] += h
    for e in (A, B):
        e.check()
    stats = A.session_stats()
    assert slides == 1 and stats["relocations"] > 0 and stats["parks"] > 0 and stats["unparks"] > 0, (slides, stats)
    assert shorts > 0 if ragged else shorts == 0
    a = A.export_sessions(np.arange(N), None).cpu().numpy()
    b = B.export_sessions(np.arange(N), None).cpu().numpy()
    torch.cuda.synchronize()
    if caller_gr:
        assert np.array_equal(a[:, :SIGNAL_BYTES], b[:, :SIGNAL_BYTES])
    else:
        assert np.array_equal(a, b)
    for e in (A, B):
        e.close()


@pytest.mark.parametrize("ragged", [False, True], ids=["plain", "ragged"])
@pytest.mark.parametrize("mode,post", CASES, ids=[m + ("-postfilter" if p else "") for m, p in CASES])
def test_split_sessions_are_the_fused_call(api, model0, mode, post, ragged):
    """13 slots, 40 sessions, ten calls: pnb_process_sessions_* (ragged: _ragged_*, with 1-or-max, one-short and all-equal
    hop patterns) on A, analyze -> compute_rnn -> synthesize on the same lists on B, host and device halves mixed, f32 and
    int16.  Output, g/r, features (A's tap through the slot of each session), residency counts and every launch count
    match after each call; every session's blob matches at the end."""
    _run(api, model0, mode, post, ragged, seed=500 + 7 * CASES.index((mode, post)) + ragged)


@pytest.mark.parametrize("ragged", [False, True], ids=["plain", "ragged"])
def test_caller_gains_between_the_halves(api, model0, ragged):
    """B runs analyze -> synthesize with A's g/r and no network call: the same output, and the signal part of every
    session's blob, as A's fused calls."""
    _run(api, model0, "tensor", False, ragged, seed=540 + ragged, caller_gr=True)


@pytest.mark.parametrize("mode", ["fp32", "tensor"])
def test_network_calls_on_sessions(api, model0, mode):
    """pnb_compute_rnn_sessions_* alone, with parks, ragged calls and both formats: every session's g/r equals a
    1-stream engine's fed only the calls that list it, and the sessions' signal state stays fresh."""
    import torch
    Sn, Nn, Fm = 5, 9, 4
    e = _engine(api, model0, Sn, mode, Fm=Fm)
    e.reserve_sessions(Nn)
    plain = [_engine(api, model0, 1, mode, Fm=Fm) for _ in range(Nn)]
    rng = np.random.RandomState(3)
    for c in range(8):
        k = int(rng.randint(2, Sn + 1))
        ids = rng.choice(Nn, k, replace=False).astype(np.int32)
        F = int(rng.randint(1, Fm + 1))
        hops = None
        if c % 2:
            hops = rng.randint(1, F + 1, size=k).astype(np.int32)
            hops[rng.randint(k)] = F
        h = np.full(k, F) if hops is None else hops
        W = 70 if c % 3 else 138
        x = (rng.randn(k, F, W) * 0.5).astype(np.float32) if W == 70 else rng.rand(k, F, W).astype(np.float32)
        before, st = e.launches, e.session_stats()
        if c % 4 < 2:
            gr = e.compute_rnn_sessions(ids, x, hops=hops)
        else:
            d_x, d_gr = _dev(x), torch.zeros((k, F, 68), device="cuda")
            torch.cuda.synchronize()
            e.compute_rnn_sessions_device(ids, api.RNN_FEATURES if W == 70 else api.RNN_RECORDS, d_x.data_ptr(), F * W, F,
                                          d_gr.data_ptr(), F * 68, hops=hops)
            gr = _host(d_gr)
        moved = e.session_stats() != st
        assert e.launches - before == moved + 2 + e.launches_per_call(F) - 3, c
        for i, s in enumerate(ids):
            want = plain[s].compute_rnn(np.ascontiguousarray(x[i:i + 1, :h[i]]))
            assert same_bits(gr[i, :h[i]], want[0]), (c, i)
            assert not gr[i, h[i]:].any(), (c, i)
    e.check()
    assert e.session_stats()["parks"] > 0
    blobs = e.export_sessions(np.arange(Nn), None).cpu().numpy()
    assert not blobs[:, 8:SIGNAL_BYTES].any()
    for p in [e] + plain:
        p.close()


def test_refusals_and_reset(api, model0):
    """Every refused call and state operation returns PNB_ERR_ARG with pnb_launch_count and the residency counts
    unchanged; the accepted split afterwards matches a twin's ragged session call; pnb_reset cancels a pending split and
    keeps session mode."""
    import torch
    L = api.load_library()
    Sr, Nr, F = 4, 10, 3
    e, t = _engine(api, model0, Sr, "tensor", Fm=F), _engine(api, model0, Sr, "tensor", Fm=F)
    h = e.h
    ids = np.array([3, 7, 1], np.int32)
    hops = np.array([3, 1, 2], np.int32)
    x = crowd(3, 2 * F, seed=550)
    x1, x2 = np.ascontiguousarray(x[:, :F * HOP]), np.ascontiguousarray(x[:, F * HOP:])
    feat = np.zeros((3, F, 70), np.float32)
    gr = np.full((3, F, 68), 0.5, np.float32)
    out = np.zeros((3, F * HOP), np.float32)
    blobs = torch.zeros((Nr, L.pnb_state_size()), dtype=torch.uint8, device="cuda")
    xp, fp, gp, op = x1.ctypes.data, feat.ctypes.data, gr.ctypes.data, out.ctypes.data

    keep = []   # the int arrays handed to the library stay alive for the whole test

    def p(a):
        if a is None:
            return None
        keep.append(np.ascontiguousarray(a, np.int32))
        return keep[-1].ctypes.data

    def analyze(i=ids, hp=hops, n=3, nf=F, x_=xp, xs=F * HOP, f=fp, fs=70 * F):
        return L.pnb_analyze_sessions_host_f32(h, p(i), p(hp), n, x_, xs, nf, f, fs)

    def network(i=ids, hp=hops, n=3, nf=F, fmt=0, fs=70 * F, g=gp, gs=68 * F):
        return L.pnb_compute_rnn_sessions_host(h, p(i), p(hp), n, fmt, fp, fs, nf, g, gs)

    def synth(i=ids, n=3, nf=F, g=gp, gs=68 * F, o=op, os_=F * HOP):
        return L.pnb_synthesize_sessions_host_f32(h, p(i), n, g, gs, nf, o, os_)

    # not in session mode; engines without a session pool
    for call in (analyze, network, synth):
        assert call() == -1 and b"pnb_sessions_reserve" in L.pnb_last_error()
    assert e.launches == 0
    for flags, model in ((api.SIGNAL_ONLY, None), (api.NN_TENSOR | api.NETWORK_ONLY, model0)):
        o = api.Engine(Sr, F, model, flags)
        assert L.pnb_sessions_reserve(o.h, Nr) == -1
        assert L.pnb_analyze_sessions_host_f32(o.h, p(ids), None, 3, xp, F * HOP, F, fp, 70 * F) == -1
        assert L.pnb_compute_rnn_sessions_host(o.h, p(ids), None, 3, 0, fp, 70 * F, F, gp, 68 * F) == -1
        assert o.launches == 0
        o.close()
    for q in (e, t):
        q.reserve_sessions(Nr)
    n0, st0 = e.launches, e.session_stats()
    # nothing pending: bad arguments
    bad = {
        "synth_nothing_pending": lambda: synth(),
        "hops_zero": lambda: analyze(hp=[3, 0, 2]),
        "hops_above_max": lambda: analyze(hp=[4, 1, 2], nf=4),
        "frames_not_max_hops": lambda: analyze(nf=2, xs=2 * HOP, fs=140),
        "frames_not_max_hops_network": lambda: network(hp=[2, 1, 2]),
        "ids_null": lambda: L.pnb_analyze_sessions_host_f32(h, None, None, 3, xp, F * HOP, F, fp, 70 * F),
        "in_null": lambda: analyze(x_=None),
        "feat_null": lambda: analyze(f=None),
        "in_stride": lambda: analyze(xs=F * HOP - 1),
        "feat_stride": lambda: analyze(fs=70 * F - 1),
        "id_twice": lambda: analyze(i=[3, 3, 1]),
        "id_range": lambda: analyze(i=[3, Nr, 1]),
        "n_zero": lambda: analyze(n=0),
        "n_above_slots": lambda: analyze(i=[0, 1, 2, 3, 4], hp=None, n=5),
        "network_format": lambda: network(fmt=2),
        "network_gr_stride": lambda: network(gs=68 * F - 1),
        "network_gr_null": lambda: network(g=None),
        "slot_analyze": lambda: L.pnb_analyze_host_f32(h, xp, F * HOP, F, fp, 70 * F),
        "slot_compute_rnn": lambda: L.pnb_compute_rnn_host(h, 0, fp, 70 * F, F, gp, 68 * F),
    }
    for name, call in bad.items():
        assert call() == -1, name
        assert e.launches == n0 and e.session_stats() == st0, name
    # a split pending
    assert analyze() == 0
    n1 = e.launches
    d_blob = blobs.data_ptr()
    pending = {
        "process_sessions": lambda: L.pnb_process_sessions_host_f32(h, p(ids), 3, xp, F * HOP, op, F * HOP, F, None),
        "process_sessions_ragged": lambda: L.pnb_process_sessions_ragged_host_f32(h, p(ids), p(hops), 3, xp, F * HOP, op,
                                                                                  F * HOP, None),
        "analyze_again": lambda: analyze(),
        "analyze_other": lambda: analyze(i=[0, 2, 4]),
        "reset_sessions": lambda: L.pnb_reset_sessions(h, p([5]), 1, None),
        "export_sessions": lambda: L.pnb_export_sessions(h, p([3]), 1, d_blob, blobs.stride(0), None),
        "import_sessions": lambda: L.pnb_import_sessions(h, p([5]), 1, d_blob, blobs.stride(0), None),
        "sessions_reserve": lambda: L.pnb_sessions_reserve(h, 2 * Nr),
        "network_other_order": lambda: network(i=[7, 3, 1], hp=[1, 3, 2]),
        "network_other_ids": lambda: network(i=[3, 7, 2]),
        "network_other_hops": lambda: network(hp=[3, 2, 2]),
        "network_no_hops": lambda: network(hp=None),
        "network_fewer": lambda: network(i=[3, 7], hp=[3, 1], n=2),
        "synth_other_n": lambda: synth(i=[3, 7], n=2),
        "synth_other_id": lambda: synth(i=[3, 7, 2]),
        "synth_other_order": lambda: synth(i=[1, 7, 3]),
        "synth_other_frames": lambda: synth(nf=2, gs=136, os_=2 * HOP),
        "slot_synthesize": lambda: L.pnb_synthesize_host_f32(h, gp, 68 * F, F, op, F * HOP),
    }
    for name, call in pending.items():
        assert call() == -1, name
        assert e.launches == n1, name
    # the accepted split: the twin's ragged session call
    assert network() == 0 and synth() == 0
    want, _ = t.process_sessions(ids, x1, hops=hops)
    assert same_bits(out, want)
    got = e.process_sessions(ids, x2, hops=hops)[0]
    assert same_bits(got, t.process_sessions(ids, x2, hops=hops)[0])
    # pnb_reset cancels the pending split and keeps session mode
    assert analyze() == 0
    e.reset()
    assert synth() == -1
    e.process_sessions(ids, x1, hops=hops)
    assert analyze() == 0 and synth() == 0
    for q in (e, t):
        q.check()
        q.close()
