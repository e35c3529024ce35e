"""Host-buffer calls share the engine's device staging.  Blocking and pipelined calls of either wire format, mixed on
one engine, give the bits of blocking calls of the same types on a twin engine; so do the training-record calls.  Every
call entry point refuses bad arguments with PNB_ERR_ARG before it enqueues anything, and the engine goes on as if the
refused call had never been made."""
import numpy as np
import pytest

from test_gpu_lifecycle import HOP, _signal
from test_gpu_parity import api  # noqa: F401

pytestmark = pytest.mark.gpu

MODES = ["fp32", "tensor"]
S = 270                       # not a multiple of the 128-row tile
ACTIVE = 201                  # rows after the shrink in the middle of the mixed sequence
FMAX = 8
PNB_ERR_ARG = -1
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


# ---- refusals -------------------------------------------------------------------------------------------------------
ENHANCE = ["pnb_process_host_f32", "pnb_process_host_i16", "pnb_submit_host_f32", "pnb_submit_host_i16",
           "pnb_process_device_f32", "pnb_process_device_i16", "pnb_submit_device_f32", "pnb_submit_device_i16"]
TRAIN = ["pnb_train_records_host", "pnb_submit_train_records", "pnb_train_records_device"]


def _enhance_call(L, name, h, a, stream):
    f = getattr(L, name)
    if name.startswith("pnb_process_host"):
        return f(h, a["in"], a["in_stride"], a["out"], a["out_stride"], a["F"], None)
    if name.startswith("pnb_submit_host"):
        return f(h, a["in"], a["in_stride"], a["out"], a["out_stride"], a["F"])
    if name.startswith("pnb_process_device"):
        return f(h, a["in"], a["in_stride"], a["out"], a["out_stride"], a["F"], None, stream)
    return f(h, a["in"], a["in_stride"], a["out"], a["out_stride"], a["F"], stream)


def _train_call(L, name, h, a, stream):
    args = [h, a["speech"], a["speech_stride"], a["noisy"], a["noisy_stride"], a["F"], a["records"], a["records_stride"]]
    return getattr(L, name)(*args, *([stream] if name.endswith("device") else []))


def _refuse(L, call, name, h, valid, faults, stream):
    for fault in faults:
        rc = call(L, name, h, {**valid, **fault}, stream)
        assert rc == PNB_ERR_ARG, (name, fault, rc, L.pnb_last_error())


@pytest.mark.parametrize("mode", MODES)
def test_refused_calls_enqueue_nothing(api, model0, mode):
    """Each of the eleven call entry points refuses F = 0, F > max_frames, a NULL buffer, a short stride and the
    wrong engine mode with PNB_ERR_ARG; the next valid call of each engine then gives its twin's bits."""
    import torch
    from percepnet_b200.synth import to_int16
    x = _signal(S, 2, 41)
    speech, noisy = _pairs(S // 2, 2 * FMAX, 6)
    enh, enh_twin = (api.Engine(S, FMAX, model0, _flags(api, mode)) for _ in range(2))
    trn, trn_twin = (api.Engine(S, FMAX, None, api.TRAIN_DATA) for _ in range(2))
    first = np.ascontiguousarray(x[:, :FMAX * HOP])
    for e in (enh, enh_twin):
        e.process(first)
    for e in (trn, trn_twin):
        e.train_records(np.ascontiguousarray(speech[:, :FMAX * HOP]), np.ascontiguousarray(noisy[:, :FMAX * HOP]))

    row = FMAX * HOP
    h32, h16 = np.zeros((S, row), np.float32), np.zeros((S, row), np.int16)
    d32, d16 = torch.zeros((2, S, row), dtype=torch.float32, device="cuda"), torch.zeros((2, S, row), dtype=torch.int16, device="cuda")
    hsp, hrec = np.zeros((S // 2, row), np.int16), np.zeros((S // 2, FMAX * 138), np.float32)
    dsp, drec = torch.zeros((2, S // 2, row), dtype=torch.int16, device="cuda"), torch.zeros((S // 2, FMAX * 138), device="cuda")
    stream = torch.cuda.current_stream().cuda_stream
    torch.cuda.synchronize()
    short = FMAX * HOP - 1
    for name in ENHANCE:
        if "host" in name:
            buf = h32 if name.endswith("f32") else h16
            i, o = buf.ctypes.data, buf.ctypes.data
        else:
            buf = d32 if name.endswith("f32") else d16
            i, o = buf[0].data_ptr(), buf[1].data_ptr()
        valid = {"in": i, "in_stride": row, "out": o, "out_stride": row, "F": FMAX}
        _refuse(enh.L, _enhance_call, name, enh.h, valid,
                [{"F": 0}, {"F": FMAX + 1}, {"in": None}, {"out": None}, {"in_stride": short}, {"out_stride": short}], stream)
        _refuse(trn.L, _enhance_call, name, trn.h, valid, [{}], stream)
    for name in TRAIN:
        if "host" in name or "submit" in name:
            s, n, r = hsp.ctypes.data, hsp.ctypes.data, hrec.ctypes.data
        else:
            s, n, r = dsp[0].data_ptr(), dsp[1].data_ptr(), drec.data_ptr()
        valid = {"speech": s, "speech_stride": row, "noisy": n, "noisy_stride": row, "F": FMAX, "records": r,
                 "records_stride": FMAX * 138}
        _refuse(trn.L, _train_call, name, trn.h, valid,
                [{"F": 0}, {"F": FMAX + 1}, {"speech": None}, {"noisy": None}, {"records": None},
                 {"speech_stride": short}, {"noisy_stride": short}, {"records_stride": FMAX * 138 - 1}], stream)
        _refuse(enh.L, _train_call, name, enh.h, valid, [{}], stream)
    torch.cuda.synchronize()

    nxt = np.ascontiguousarray(x[:, FMAX * HOP:])
    (a, ga), (b, gb) = enh.process(nxt, want_gr=True), enh_twin.process(nxt, want_gr=True)
    assert np.array_equal(a, b) and np.array_equal(ga, gb)
    assert np.abs(a).max() > 0
    s, y = np.ascontiguousarray(speech[:, FMAX * HOP:]), np.ascontiguousarray(noisy[:, FMAX * HOP:])
    ra, rb = trn.train_records(s, y), trn_twin.train_records(s, y)
    assert np.array_equal(ra.view(np.int32), rb.view(np.int32))
    for e in (enh, enh_twin, trn, trn_twin):
        e.check()
        e.close()
