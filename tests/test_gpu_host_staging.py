"""Host-buffer calls share the engine's device staging.  Blocking and pipelined calls of either wire format, mixed on
one engine, give the bits of blocking calls of the same types on a twin engine; so do the training-record calls.  The
refusals of every call entry point are in test_gpu_refusals.py."""
import numpy as np
import pytest

from test_gpu_lifecycle import HOP, _signal
from test_gpu_parity import api  # noqa: F401

pytestmark = pytest.mark.gpu

MODES = ["fp32", "tensor"]
S = 270                       # not a multiple of the 128-row tile
ACTIVE = 201                  # rows after the shrink in the middle of the mixed sequence
FMAX = 8
# (call, wire format, hops): the mixed sequence; "shrink" sets the active range to ACTIVE
STEPS = [("process", "f32", 8), ("submit", "i16", 8), ("submit", "i16", 5), ("shrink", None, 0), ("submit", "i16", 8),
         ("process", "i16", 3), ("submit", "f32", 8), ("submit", "f32", 6), ("wait", None, 0), ("process", "f32", 7)]


def _flags(api, mode):
    return api.NN_FP32 if mode == "fp32" else api.NN_TENSOR


def _mixed(api, model, mode, x, x16, blocking):
    """Runs STEPS; blocking=True turns every submit into a blocking call of the same type.  Returns (outputs, g/r of the
    process calls)."""
    e = api.Engine(S, FMAX, model, _flags(api, mode))
    outs, grs, keep, t = [], [], [], 0
    for call, fmt, n in STEPS:
        if call == "shrink":
            e.set_active(ACTIVE)
            continue
        if call == "wait":
            e.wait()
            continue
        xin = np.ascontiguousarray((x if fmt == "f32" else x16)[:e.active, t * HOP:(t + n) * HOP])
        t += n
        if call == "process" or blocking:
            out, gr = e.process(xin, want_gr=call == "process")
            if gr is not None:
                grs.append(gr)
        else:
            out = np.empty_like(xin)
            keep.append(xin)                               # alive until the round trip is complete
            e.submit(xin, out)
        outs.append(out)
    e.wait()
    e.close()
    return outs, grs


@pytest.mark.parametrize("mode", MODES)
def test_mixed_host_calls_match_blocking_calls(api, model0, mode):
    """f32 and int16, blocking and pipelined host calls on one engine, with the active range shrunk in the middle."""
    from percepnet_b200.synth import to_int16
    x = _signal(S, 8, 31)
    x16 = to_int16(x)
    ref_out, ref_gr = _mixed(api, model0, mode, x, x16, blocking=True)
    out, gr = _mixed(api, model0, mode, x, x16, blocking=False)
    assert len(out) == len(ref_out) and len(gr) == len(ref_gr) == 3
    for k, (a, b) in enumerate(zip(ref_out, out)):
        assert a.dtype == b.dtype and np.array_equal(a, b), f"call {k}"
    for k, (a, b) in enumerate(zip(ref_gr, gr)):
        assert np.array_equal(a, b), f"g/r of process call {k}"
    assert out[-1].shape[0] == ACTIVE and np.abs(ref_out[-1]).max() > 0


def _pairs(n_pairs, n_frames, seed):
    """[n_pairs, n_frames*480] int16 speech and noisy mixtures: a few synthetic pairs, shifted and scaled per row."""
    from percepnet_b200.synth import synth_pairs
    clean, noisy = synth_pairs(6, n_frames, seed=seed)
    rng = np.random.RandomState(seed)
    rows, shift = rng.randint(0, 6, n_pairs), rng.randint(0, 5, n_pairs) * HOP
    level = 0.3 + 0.7 * rng.rand(n_pairs)

    def pick(a):
        return np.stack([(np.roll(a[r], s) * g).astype(np.int16) for r, s, g in zip(rows, shift, level)])
    return pick(clean), pick(noisy)


def test_train_records_mixed_calls_match_blocking_calls(api):
    """pnb_train_records_host between pnb_submit_train_records calls (three in flight) on one engine."""
    fmax, N = 12, S // 2
    steps = [("host", 12), ("submit", 12), ("submit", 7), ("submit", 12), ("host", 5), ("submit", 12), ("host", 9)]
    speech, noisy = _pairs(N, sum(n for _, n in steps), 5)

    def run(blocking):
        e = api.Engine(S, fmax, None, api.TRAIN_DATA)
        outs, keep, t = [], [], 0
        for call, n in steps:
            s = np.ascontiguousarray(speech[:, t * HOP:(t + n) * HOP])
            y = np.ascontiguousarray(noisy[:, t * HOP:(t + n) * HOP])
            t += n
            if call == "host" or blocking:
                outs.append(e.train_records(s, y))
                continue
            rec = np.empty((N, n, 138), np.float32)
            keep.append((s, y))
            rc = e.L.pnb_submit_train_records(e.h, s.ctypes.data, s.shape[1], y.ctypes.data, y.shape[1], n,
                                              rec.ctypes.data, n * 138)
            assert rc == 0, e.L.pnb_last_error()
            outs.append(rec)
        e.wait()
        e.close()
        return np.concatenate(outs, axis=1)

    ref, got = run(True), run(False)
    assert np.array_equal(ref.view(np.int32), got.view(np.int32))
    assert np.abs(ref).max() > 0

