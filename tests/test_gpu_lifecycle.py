"""Stream slots recycled inside a running engine: pnb_reset_streams / pnb_export_states / pnb_import_states.  A reset slot
is a fresh stream, an exported and imported stream continues bit for bit, the operations keep stream order with the
calls around them, and bad blobs or arguments touch no other stream."""
import numpy as np
import pytest

from test_gpu_parity import GR_RTOL, _inputs, api  # noqa: F401

pytestmark = pytest.mark.gpu

F = 8
# (id, network mode, streams, overlap); 270 is not a multiple of the 256-row tile pair.  overlap: the state operations go
# to a non-blocking stream of their own, which nothing but the engine orders with the streams its calls run on.
CONFIGS = [("fp32-270", "fp32", 270, False), ("tensor-270", "tensor", 270, False),
           ("tensor-2048-overlap", "tensor", 2048, True)]
HOP = 480


def _ops_stream(cfg, default=0):
    """The stream a config issues its state operations on."""
    import torch
    return torch.cuda.Stream().cuda_stream if cfg[3] else default


def _flags(api, mode):
    return api.NN_FP32 if mode == "fp32" else api.NN_TENSOR


def _engine(api, model, S, mode, Fm=F, flags=None):
    return api.Engine(S, Fm, model, _flags(api, mode) if flags is None else flags)


def _signal(S, n_calls, seed):
    """[S, n_calls*F*480] float32: rows differ from each other (seeded signals at per-row levels)."""
    base = _inputs(1.0, n_calls * F, n_synth=6)
    rng = np.random.RandomState(seed)
    rows = rng.randint(0, base.shape[0], S)
    level = (0.25 + rng.rand(S)).astype(np.float32)
    shift = rng.randint(0, 5, S) * HOP
    x = np.stack([np.roll(base[r], s) for r, s in zip(rows, shift)]) * level[:, None]
    return np.ascontiguousarray(x.astype(np.float32))


def _call(x, k):
    return np.ascontiguousarray(x[:, k * F * HOP:(k + 1) * F * HOP])


def _blob_rows(api, e, idx, stream=0):
    import torch
    t = e.export_states(idx, None, stream=stream)
    torch.cuda.synchronize()
    return t.cpu().numpy()


# ---------------------------------------------------------------------------------------------- 1
@pytest.mark.parametrize("cfg", CONFIGS, ids=[c[0] for c in CONFIGS])
def test_batched_export_matches_single_stream_export(api, model0, cfg):
    _, mode, S, _ = cfg
    x = _signal(S, 2, 1)
    e = _engine(api, model0, S, mode)
    e.process(_call(x, 0))
    e.process(_call(x, 1))
    idx = [0, 1, 137, S - 1]
    got = _blob_rows(api, e, idx, _ops_stream(cfg))
    assert got.shape == (4, e.state_size)
    for i, s in enumerate(idx):
        assert got[i].tobytes() == e.get_state(s), s
    e.check()
    e.close()


def test_batched_export_matches_single_stream_export_traindata(api):
    from percepnet_b200.synth import synth_pairs
    c16, n16 = synth_pairs(135, 2 * F, seed=5)
    e = api.Engine(270, F, None, api.TRAIN_DATA)
    e.train_records(c16[:, :F * HOP], n16[:, :F * HOP])
    e.train_records(c16[:, F * HOP:], n16[:, F * HOP:])
    idx = [0, 1, 137, 269]
    got = _blob_rows(api, e, idx)
    for i, s in enumerate(idx):
        assert got[i].tobytes() == e.get_state(s), s
    assert np.abs(got[:, 8:8 + 5280 * 4]).max() > 0
    e.close()


# ---------------------------------------------------------------------------------------------- 2
@pytest.mark.parametrize("cfg", CONFIGS, ids=[c[0] for c in CONFIGS])
def test_reset_stream_equals_fresh_stream(api, model0, cfg):
    _, mode, S, _ = cfg
    x = _signal(S, 4, 2)
    z = _signal(S, 2, 3)
    R = [0, 5, S - 1]
    y = x.copy()
    y[R, 2 * F * HOP:] = z[R]                      # from the third call on, the reset slots carry a new session
    a = _engine(api, model0, S, mode)              # reset after two calls
    b = _engine(api, model0, S, mode)              # no reset
    c = _engine(api, model0, S, mode)              # fresh engine fed the new sessions
    for k in range(2):
        a.process(_call(y, k))
        b.process(_call(x, k))
    a.reset_streams(R, stream=_ops_stream(cfg))    # the next host call runs on the engine's own stream
    for k in (2, 3):
        out_a, gr_a = a.process(_call(y, k), want_gr=True)
        out_b, gr_b = b.process(_call(x, k), want_gr=True)
        out_c, gr_c = c.process(_call(z, k - 2), want_gr=True)
        others = np.setdiff1d(np.arange(S), R)
        assert np.array_equal(out_a[R], out_c[R]) and np.array_equal(gr_a[:, R], gr_c[:, R]), k
        assert np.array_equal(out_a[others], out_b[others]) and np.array_equal(gr_a[:, others], gr_b[:, others]), k
    assert np.abs(out_a[R]).max() > 0
    for e in (a, b, c):
        e.check()
        e.close()


# ---------------------------------------------------------------------------------------------- 3
PAIRS = [("fp32-fp32", "fp32", "fp32", 300), ("tensor-tensor", "tensor", "tensor", 2048),
         ("fp32-tensor", "fp32", "tensor", 2048)]


@pytest.mark.parametrize("pair", PAIRS, ids=[p[0] for p in PAIRS])
def test_import_moves_streams_exactly(api, model0, pair):
    import torch
    _, mode_a, mode_b, S_b = pair
    S_a = 270
    x = _signal(S_a, 3, 4)
    other = _signal(S_b, 1, 5) * np.float32(0.5)
    a = _engine(api, model0, S_a, mode_a)
    for k in range(2):
        a.process(_call(x, k))
    src, dst = [3, 100, S_a - 1], [S_b - 1, 0, 7]
    blobs = a.export_states(src, None)
    want, want_gr = a.process(_call(x, 2), want_gr=True)
    b = _engine(api, model0, S_b, mode_b, Fm=10)  # other batch size, max_frames, hop count
    b.process(np.ascontiguousarray(other))
    b.import_states(dst, blobs)
    y = np.zeros((S_b, F * HOP), np.float32)
    y[dst] = _call(x, 2)[src]
    got, got_gr = b.process(y, want_gr=True)
    torch.cuda.synchronize()
    w, wg, g, gg = want[src], want_gr[:, src], got[dst], got_gr[:, dst]
    if mode_a == mode_b:
        assert np.array_equal(w, g) and np.array_equal(wg, gg)
    else:  # the bounds of test_stream_migrates_between_network_modes
        rel = np.abs(gg - wg) / np.maximum(np.abs(wg), 1e-6)
        assert rel.max() < GR_RTOL
        assert np.abs(np.trunc(w.astype(np.float64) * 32768) - np.trunc(g.astype(np.float64) * 32768)).max() <= 1
    assert np.abs(w).max() > 0
    a.check()
    b.check()
    a.close()
    b.close()


def test_device_blob_and_host_blob_interchange(api, model0):
    """A blob exported on the device is a pnb_set_state blob, and a pnb_get_state blob imports on the device."""
    import torch
    x = _signal(270, 2, 6)
    a = _engine(api, model0, 270, "tensor")
    a.process(_call(x, 0))
    dev = a.export_states([11], None)[0].cpu().numpy().tobytes()
    host = a.get_state(12)
    b = _engine(api, model0, 64, "tensor")
    b.set_state(3, dev)
    t = torch.from_numpy(np.frombuffer(host, np.uint8).copy()).cuda()[None]
    b.import_states([4], t)
    got = _blob_rows(api, b, [3, 4])
    assert got[0].tobytes() == dev and got[1].tobytes() == host
    b.check()
    a.close()
    b.close()


# ---------------------------------------------------------------------------------------------- 4
ORDER_CONFIGS = [("fp32-270", "fp32", 270, False), ("tensor-2048-overlap", "tensor", 2048, True)]


def _order_sequence(api, e, x, st, submitted, ops_st=None):
    """calls interleaved with reset / export / import; returns (outputs, exported blobs) as device tensors"""
    import torch
    S = e.n_streams
    xd = torch.from_numpy(x).cuda()
    yd = torch.zeros_like(xd)
    nb = e.state_size
    blobs = torch.zeros((3, 3, nb), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()

    def call(k):
        a, b = xd[:, k * F * HOP:], yd[:, k * F * HOP:]
        f = e.submit_device if submitted else e.process_device
        f(a.data_ptr(), xd.stride(0), b.data_ptr(), yd.stride(0), F, stream=st)
        if not submitted:
            torch.cuda.synchronize()

    def op(fn, *args):
        fn(*args, stream=st if ops_st is None else ops_st)
        if not submitted:
            torch.cuda.synchronize()
    call(0)
    op(e.reset_streams, [2, 9, S - 1])
    call(1)
    op(e.export_states, [1, 2, 3], blobs[0].data_ptr(), nb)
    op(e.import_states, [S - 2, 4], blobs[0].data_ptr(), nb)      # slots 1 and 2 continue in slots S-2 and 4
    call(2)
    op(e.export_states, [4, S - 2, 6], blobs[1].data_ptr(), nb)
    op(e.reset_streams, [6])
    call(3)
    op(e.export_states, [6, 0, S - 1], blobs[2].data_ptr(), nb)
    if submitted:
        e.flush(st)
    torch.cuda.synchronize()
    e.check()
    return yd.cpu().numpy(), blobs.cpu().numpy()


@pytest.mark.parametrize("cfg", ORDER_CONFIGS, ids=[c[0] for c in ORDER_CONFIGS])
def test_state_operations_keep_stream_order(api, model0, cfg):
    import torch
    _, mode, S, _ = cfg
    x = _signal(S, 4, 7)
    ref_e = _engine(api, model0, S, mode)
    ref = _order_sequence(api, ref_e, x, torch.cuda.current_stream().cuda_stream, submitted=False)
    ref_e.close()
    e = _engine(api, model0, S, mode)
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        got = _order_sequence(api, e, x, side.cuda_stream, submitted=True, ops_st=_ops_stream(cfg, None))
    e.close()
    assert np.array_equal(ref[0], got[0])
    assert np.array_equal(ref[1], got[1])
    assert np.abs(ref[0]).max() > 0


# ---------------------------------------------------------------------------------------------- 5
@pytest.mark.parametrize("cfg", CONFIGS, ids=[c[0] for c in CONFIGS])
def test_bad_blobs_are_rejected(api, model0, cfg):
    import torch
    _, mode, S, _ = cfg
    ops = _ops_stream(cfg)
    x = _signal(S, 2, 8)
    e = _engine(api, model0, S, mode)
    e.process(_call(x, 0))
    e.process(_call(x, 1))
    fresh_e = _engine(api, model0, 16, mode)
    fresh = _blob_rows(api, fresh_e, [0])[0]
    fresh_e.close()
    good = e.export_states([1, 2, 3], None, stream=ops)
    torch.cuda.synchronize()
    bad = good.clone()
    bad[0, 0] ^= 0xFF                                                   # magic
    h0 = 45880                                                          # offsetof(StreamState, h)
    bad[1, h0:h0 + 4] = torch.from_numpy(np.frombuffer(np.float32(2.0).tobytes(), np.uint8).copy()).cuda()
    before = _blob_rows(api, e, np.arange(S), ops)
    dst = [12, 10, 11]
    e.import_states(dst, bad, stream=ops)
    with pytest.raises(api.PnbError, match=r"stream 10\b" if mode == "tensor" else r"stream 12\b"):
        e.check()
    e.check()                                                           # reported once
    after = _blob_rows(api, e, np.arange(S), ops)
    assert after[12].tobytes() == fresh.tobytes()                       # bad magic: left fresh
    if mode == "tensor":
        assert after[10].tobytes() == fresh.tobytes()                   # GRU value 2.0: left fresh
    else:                                                               # fp32 engines have no GRU bound
        assert after[10].tobytes() == bad[1].cpu().numpy().tobytes()
    assert after[11].tobytes() == good[2].cpu().numpy().tobytes()
    rest = np.setdiff1d(np.arange(S), dst)
    assert np.array_equal(before[rest], after[rest])
    e.close()


def test_rejection_names_lowest_slot(api, model0):
    import torch
    e = _engine(api, model0, 270, "tensor")
    b = torch.zeros((2, e.state_size), dtype=torch.uint8, device="cuda")
    e.import_states([200, 30], b)
    with pytest.raises(api.PnbError, match=r"stream 30\b"):
        e.wait()
    e.wait()
    e.close()


# ---------------------------------------------------------------------------------------------- 6
@pytest.mark.parametrize("cfg", CONFIGS[:2], ids=[c[0] for c in CONFIGS[:2]])
def test_bad_arguments_are_refused(api, model0, cfg):
    import torch
    _, mode, S, _ = cfg
    x = _signal(S, 2, 9)
    e = _engine(api, model0, S, mode)
    ref = _engine(api, model0, S, mode)
    out0 = e.process(_call(x, 0))[0]
    assert np.array_equal(out0, ref.process(_call(x, 0))[0])
    blobs = e.export_states([0, 1], None)
    torch.cuda.synchronize()
    nb = e.state_size
    bad = [lambda: e.reset_streams([3, 3]),                                 # duplicate
           lambda: e.reset_streams([S]),                                    # out of range
           lambda: e.reset_streams([-1]),
           lambda: e.export_states([0, 4, 0], None),                        # duplicate
           lambda: e.export_states([0, 1], blobs.data_ptr(), nb - 4),       # short stride
           lambda: e.import_states([5, 6], blobs.data_ptr(), nb - 1),
           lambda: e.import_states([S + 7], blobs.data_ptr(), nb),
           lambda: e.export_states([0], 0),                                 # NULL
           lambda: e.import_states([0], 0)]
    for f in bad:
        with pytest.raises(api.PnbError):
            f()
    assert e.L.pnb_reset_streams(e.h, None, 2, None) == -1                 # NULL slot array: PNB_ERR_ARG
    e.reset_streams([])                                                     # n = 0: a no-op
    torch.cuda.synchronize()
    out1, gr1 = e.process(_call(x, 1), want_gr=True)
    want1, wgr1 = ref.process(_call(x, 1), want_gr=True)
    assert np.array_equal(out1, want1) and np.array_equal(gr1, wgr1)
    e.check()
    e.close()
    ref.close()


# ---------------------------------------------------------------------------------------------- 7
@pytest.mark.parametrize("mode", ["fp32", "tensor"])
def test_state_operation_launches(api, model0, mode):
    """pnb_launch_count grows by each state operation's own launches: one move for a reset, an export, pnb_get_state and
    a grown active range; a blob check and a move for an import and pnb_set_state; none for n = 0 or a shrunk range."""
    import torch
    S = 16
    e = _engine(api, model0, S, mode)
    e.process(_call(_signal(S, 1, 9), 0))
    blobs = e.export_states([1, 2], None)
    blob = e.get_state(3)
    ops = [("reset", lambda: e.reset_streams([0, 5]), 1),
           ("export", lambda: e.export_states([4, 6], blobs.data_ptr()), 1),
           ("import", lambda: e.import_states([7, 8], blobs), 2),
           ("get_state", lambda: e.get_state(9), 1),
           ("set_state", lambda: e.set_state(10, blob), 2),
           ("shrink", lambda: e.set_active(12), 0),
           ("grow", lambda: e.set_active(S), 1),
           ("reset n 0", lambda: e.reset_streams([]), 0),
           ("export n 0", lambda: e.export_states([], blobs.data_ptr()), 0),
           ("import n 0", lambda: e.import_states([], 0), 0)]
    for name, op, want in ops:
        n = e.launches
        op()
        assert e.launches - n == want, name
    torch.cuda.synchronize()
    e.check()
    e.close()
