"""Call ordering across CUDA streams.  The calls and state operations of one engine run in the order they are issued,
whichever streams they are issued on; pnb_flush makes another stream wait for all of them, pnb_wait the host.  Every
result must be bit-identical to the same calls issued on one stream."""
import numpy as np
import pytest

from test_gpu_lifecycle import F, HOP, _signal
from test_gpu_parity import _inputs, api  # noqa: F401

pytestmark = pytest.mark.gpu

MODES = ["fp32", "tensor"]
S = 270                       # not a multiple of the 128-row tile
STALL = 50_000_000            # GPU clock cycles (~30 ms): work queued behind a stall has not run when the host looks


def _flags(api, mode):
    return api.NN_FP32 if mode == "fp32" else api.NN_TENSOR


def _stall(stream):
    """Holds `stream` back, so that anything not ordered behind it runs first and shows up as a wrong result."""
    import torch
    with torch.cuda.stream(stream):
        torch.cuda._sleep(STALL)


def _plain(api, model, mode, x, lens):
    """The reference: blocking host calls of the given hop counts, one after the other."""
    e = api.Engine(x.shape[0], max(lens), model, _flags(api, mode))
    outs, t = [], 0
    for n in lens:
        outs.append(e.process(np.ascontiguousarray(x[:, t * HOP:(t + n) * HOP]))[0])
        t += n
    e.close()
    return np.concatenate(outs, axis=1)


@pytest.mark.parametrize("dtype", ["f32", "i16"])
@pytest.mark.parametrize("mode", MODES)
def test_submitted_calls_match_plain_calls(api, model0, mode, dtype):
    """pnb_submit_host_* / pnb_wait and pnb_submit_device_* / pnb_flush, with calls of different lengths and a plain
    call in the middle of submitted ones, give the bits of blocking calls."""
    import torch
    from percepnet_b200.synth import to_int16
    lens = [22, 22, 22, 5, 22, 17, 22, 22]                 # hops per call
    x = np.ascontiguousarray(np.tile(_inputs(1.0, sum(lens), n_synth=6), (20, 1))[:S])
    if dtype == "i16":
        x = to_int16(x)
    ref = _plain(api, model0, mode, x, lens)

    eng = api.Engine(S, max(lens), model0, _flags(api, mode))
    ins, outs, t = [], [], 0
    for n in lens:
        ins.append(np.ascontiguousarray(x[:, t * HOP:(t + n) * HOP]))
        outs.append(np.empty_like(ins[-1]))
        eng.submit(ins[-1], outs[-1])
        t += n
    eng.wait()
    eng.close()
    assert np.array_equal(ref, np.concatenate(outs, axis=1))

    eng = api.Engine(S, max(lens), model0, _flags(api, mode))
    xd = torch.from_numpy(x).cuda()
    yd = torch.zeros_like(xd)
    st = torch.cuda.current_stream().cuda_stream
    t = 0
    for i, n in enumerate(lens):
        a, b = xd[:, t * HOP:], yd[:, t * HOP:]
        if i == 4:                                         # a plain call in the middle of submitted ones
            eng.process_device(a.data_ptr(), xd.stride(0), b.data_ptr(), yd.stride(0), n, stream=st, int16=dtype == "i16")
        else:
            eng.submit_device(a.data_ptr(), xd.stride(0), b.data_ptr(), yd.stride(0), n, stream=st, int16=dtype == "i16")
        t += n
    eng.flush(st)
    torch.cuda.synchronize()
    eng.check()
    got = yd.cpu().numpy()
    eng.close()
    assert np.array_equal(ref, got)
    assert np.abs(ref.astype(np.float32)).max() > 0


@pytest.mark.parametrize("mode", MODES)
def test_flush_orders_another_stream(api, model0, mode):
    """Calls submitted on stream A, pnb_flush(e, B), then the output read through B alone."""
    import torch
    x = _signal(S, 2, 21)
    ref = _plain(api, model0, mode, x, [F, F])
    e = api.Engine(S, F, model0, _flags(api, mode))
    xd = torch.from_numpy(x).cuda()
    yd = torch.zeros_like(xd)
    A, B = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    _stall(A)
    for k in range(2):
        e.submit_device(xd[:, k * F * HOP:].data_ptr(), xd.stride(0), yd[:, k * F * HOP:].data_ptr(), yd.stride(0), F,
                        stream=A.cuda_stream)
    e.flush(B.cuda_stream)
    with torch.cuda.stream(B):
        got = yd.cpu().numpy()                             # a copy on B, and a wait for B only
    torch.cuda.synchronize()
    e.check()
    e.close()
    assert np.array_equal(ref, got)


@pytest.mark.parametrize("mode", MODES)
def test_wait_covers_calls_on_any_stream(api, model0, mode):
    """Calls submitted on stream A, then pnb_wait with no flush: the output is complete when it returns."""
    import torch
    x = _signal(S, 2, 22)
    ref = _plain(api, model0, mode, x, [F, F])
    e = api.Engine(S, F, model0, _flags(api, mode))
    xd = torch.from_numpy(x).cuda()
    yd = torch.zeros_like(xd)
    A, C = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    _stall(A)
    for k in range(2):
        e.submit_device(xd[:, k * F * HOP:].data_ptr(), xd.stride(0), yd[:, k * F * HOP:].data_ptr(), yd.stride(0), F,
                        stream=A.cuda_stream)
    e.wait()
    with torch.cuda.stream(C):                             # a stream that never waited for A
        got = yd.cpu().numpy()
    torch.cuda.synchronize()
    e.close()
    assert np.array_equal(ref, got)


def _alternating(api, e, x, streams, state_stream):
    """Five calls and four state operations; call k is issued on streams[k % len(streams)], the state operations on
    state_stream, each behind a stall of its stream.  Returns (outputs, exported blobs)."""
    import torch
    xd = torch.from_numpy(x).cuda()
    yd = torch.zeros_like(xd)
    nb = e.state_size
    blobs = torch.zeros((2, 3, nb), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    calls = iter(range(5))

    def call():
        k = next(calls)
        st = streams[k % len(streams)]
        _stall(st)
        e.process_device(xd[:, k * F * HOP:].data_ptr(), xd.stride(0), yd[:, k * F * HOP:].data_ptr(), yd.stride(0), F,
                         stream=st.cuda_stream)

    def op(fn, *args):
        _stall(state_stream)
        fn(*args, stream=state_stream.cuda_stream)
    call()
    call()                                                 # directly behind a call on the other stream
    op(e.reset_streams, [2, 9, S - 1])
    call()
    op(e.export_states, [1, 2, 3], blobs[0].data_ptr(), nb)
    op(e.import_states, [S - 2, 4], blobs[0].data_ptr(), nb)  # slots 1 and 2 continue in slots S-2 and 4
    call()
    call()
    op(e.export_states, [4, S - 2, 0], blobs[1].data_ptr(), nb)
    torch.cuda.synchronize()
    e.check()
    return yd.cpu().numpy(), blobs.cpu().numpy()


@pytest.mark.parametrize("mode", MODES)
def test_calls_alternating_streams_keep_issue_order(api, model0, mode):
    """Calls alternating between streams A and B, with reset / export / import on a third stream between them, give the
    bits of the same sequence on one stream."""
    import torch
    x = _signal(S, 5, 23)
    one = torch.cuda.Stream()
    ref_e = api.Engine(S, F, model0, _flags(api, mode))
    ref = _alternating(api, ref_e, x, [one], one)
    ref_e.close()
    e = api.Engine(S, F, model0, _flags(api, mode))
    got = _alternating(api, e, x, [torch.cuda.Stream(), torch.cuda.Stream()], torch.cuda.Stream())
    e.close()
    assert np.array_equal(ref[0], got[0])
    assert np.array_equal(ref[1], got[1])
    assert np.abs(ref[0]).max() > 0
