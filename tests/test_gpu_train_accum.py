"""Gradient accumulation on the trainer (pnb_train_accumulate / pnb_train_finish / PNB_TRAIN_ACCUM): one micro-batch
finishes to the call's own gradient bit for bit, splits of a batch meet the float64 bars of the whole batch (and, for
gradients of the forward and backward halves, also split batches; and
weighting by windows instead of hops does not), exported accumulators sum across engines bit for bit, a NaN in any
micro-batch skips the step, and every refusal leaves every bit as it was."""
import ctypes as C

import numpy as np
import pytest
import torch

from percepnet_b200 import api
from percepnet_b200.weights import N_PARAMS, PackedModel, pack_state_dict, synth_state_dict, unpack_state_dict
from test_gpu_train import moderate_records, ragged_frames, trainer
import train_oracle as O

pytestmark = pytest.mark.gpu

ARG = -1   # PNB_ERR_ARG


def bits(a):
    return np.ascontiguousarray(a).view(np.int32 if a.dtype == np.float32 else np.int64)


def same_bits(a, b):
    return a.dtype == b.dtype and np.array_equal(bits(a), bits(b))


def state(eng):
    return {k: eng.train_export(k) for k in ("weights", "m", "v", "gradient", "accum")}


def halves(eng, rec):
    """pnb_train_forward_device and pnb_train_backward_device on the records' full windows, with dL/d(out) torch
    autograd of CustomLoss (the mean over these windows) at the fp32 out: returns that out."""
    B, T = rec.shape[:2]
    x = torch.from_numpy(O.features(rec)).cuda()
    y = torch.from_numpy(np.ascontiguousarray(rec[..., 70:])).cuda()
    out = torch.empty((B, T, 68), device="cuda")
    eng.train_forward_device(x.data_ptr(), T * 70, T, 0, out.data_ptr(), T * 68)
    o = out.clone().requires_grad_(True)
    O.loss(o, y).backward()
    eng.train_backward_device(o.grad.data_ptr(), T * 68)
    eng.wait()
    return out.cpu().numpy()


@pytest.mark.parametrize("B,T,frames", [(3, 40, [40, 23, 40]), (10, 500, "ragged"), (3, 40, "halves")],
                         ids=["3x40", "10x500", "3x40-halves"])
def test_one_micro_batch_is_the_call(B, T, frames):
    """grad -> accumulate -> finish holds the call's own gradient, bit for bit, and Adam after it gives the same
    weights, m and v; accumulate issues one launch and finish two.  "halves": the gradient of a backward after its
    forward instead of a gradient call's."""
    sd = synth_state_dict(1)
    rec = moderate_records(B, T, 200 + B)
    if frames == "ragged":
        frames = ragged_frames(B, T, 201 + B)
    plain, acc = trainer(sd, B, T), trainer(sd, B, T)
    out = {}
    for name, eng in (("plain", plain), ("accumulated", acc)):
        s = halves(eng, rec) if frames == "halves" else eng.train_grad(rec, frames)
        if eng is acc:
            n0 = eng.launches
            eng.train_accumulate()
            n1 = eng.launches
            eng.train_finish()
            assert (n1 - n0, eng.launches - n1) == (1, 2)
            a = eng.train_export("accum")
            assert not np.any(a), "finish leaves the accumulator empty"
        g = eng.train_export("gradient")
        eng.train_adam(1e-3, 1)
        eng.wait()
        out[name] = (s, g) + tuple(eng.train_export(k) for k in ("weights", "m", "v"))
    for k, name in enumerate(("sums or out", "gradient", "weights", "m", "v")):
        assert same_bits(out["plain"][k], out["accumulated"][k]), name
    assert np.any(out["plain"][1] != 0)
    plain.close()
    acc.close()


SPLIT_FRAMES = [500, 1, 7, 30, 500, 250, 499, 100]   # windows 1..3: the short micro-batch of the {1, 3, 4} split


def rel_errors(g, g64):
    err = {}
    for k, w in g64.items():
        d = np.asarray(g[k], np.float64) - w
        err[k] = (np.linalg.norm(d) / max(np.linalg.norm(w), 1e-300), np.abs(d).max() / max(np.abs(w).max(), 1e-300))
    return err


def failing(err):
    return {k: e for k, e in err.items() if not (e[0] <= 1e-4 and e[1] <= 1e-3)}


def test_splits_against_float64():
    """8 x 500 moderate records split as {8}, {4, 4} and {1, 3, 4} (the 3 holding windows of 1, 7 and 30 hops): every
    finished gradient meets the float64 bars of the whole batch and is close to the one-call gradient, and equals the
    hop-weighted float64 combination of the micro-batches' own gradients bit for bit.  Weighting the same gradients by
    windows misses the bars.  The full windows cut {4, 4} through the halves, each half seeded with CustomLoss's mean
    over its own windows, meet the float64 bars of the whole batch."""
    sd = synth_state_dict(1)
    B, T = 8, 500
    rec = moderate_records(B, T, 210)
    frames = np.asarray(SPLIT_FRAMES, np.int32)
    _, g64 = O.grads(sd, rec, frames.tolist(), torch.float64, "cuda")
    eng = trainer(sd, B, T)
    eng.train_grad(rec, frames)
    whole = unpack_state_dict(PackedModel.from_flat(eng.train_export("gradient")))
    print()
    for split in ((8,), (4, 4), (1, 3, 4)):
        parts, b0 = [], 0
        for n in split:
            eng.set_active(n)
            eng.train_grad(np.ascontiguousarray(rec[b0:b0 + n]), frames[b0:b0 + n])
            parts.append((eng.train_export("gradient").astype(np.float64), int(frames[b0:b0 + n].sum()), n))
            eng.train_accumulate()
            b0 += n
        eng.train_finish()
        flat = eng.train_export("gradient")
        A, Csum = np.zeros(N_PARAMS), 0.0
        for g, c, _ in parts:
            A = A + g * float(c)
            Csum += c
        assert same_bits(flat, (A / Csum).astype(np.float32)), split
        g = unpack_state_dict(PackedModel.from_flat(flat))
        err = rel_errors(g, g64)
        worst = max(err, key=lambda k: err[k][0])
        near = max(np.linalg.norm(np.asarray(g[k], np.float64) - whole[k]) / np.linalg.norm(whole[k]) for k in whole)
        print(f"split {split}: worst {worst} {err[worst][0]:.2e} / {err[worst][1]:.2e} against float64; "
              f"{near:.2e} from the one-call gradient")
        assert not failing(err), (split, failing(err))
        assert near <= 1e-5, split
        if len(split) == 3:
            by_windows = sum(gk * n for gk, _, n in parts) / B
            wrong = failing(rel_errors(unpack_state_dict(PackedModel.from_flat(by_windows.astype(np.float32))), g64))
            print(f"  weighted by windows instead of hops: {len(wrong)} of {len(g64)} tensors miss the bars")
            assert len(wrong) > 0
    _, g64 = O.grads(sd, rec, None, torch.float64, "cuda")
    eng.set_active(4)
    for b0 in (0, 4):
        halves(eng, np.ascontiguousarray(rec[b0:b0 + 4]))
        eng.train_accumulate()
    eng.train_finish()
    err = rel_errors(unpack_state_dict(PackedModel.from_flat(eng.train_export("gradient"))), g64)
    worst = max(err, key=lambda k: err[k][0])
    print(f"halves {{4, 4}}, full windows: worst {worst} {err[worst][0]:.2e} / {err[worst][1]:.2e} against float64")
    assert not failing(err), failing(err)
    eng.close()


def test_exchange_through_exported_accumulators():
    """The accumulator exported to numpy and to a torch CUDA tensor is the same; imported into a fresh trainer of the
    same weights, either finishes to the exporter's gradient bit for bit; the sum a + b of two engines' accumulators,
    imported, equals one engine accumulating both calls."""
    sd = synth_state_dict(1)
    B, T = 4, 60
    r1, r2 = moderate_records(B, T, 220), moderate_records(B, T, 221)
    f1, f2 = ragged_frames(B, T, 222), [T, 3, 17, 40]
    one = trainer(sd, B, T)
    for r, f in ((r1, f1), (r2, f2)):
        one.train_grad(r, f)
        one.train_accumulate()
    a_np = one.train_export("accum")
    assert a_np.dtype == np.float64 and a_np.shape == (N_PARAMS + 1,)
    assert a_np[-1] == sum(f1) + sum(f2)
    a_dev = torch.full((N_PARAMS + 1,), float("nan"), dtype=torch.float64, device="cuda")
    one.train_export_ptr("accum", a_dev.data_ptr(), a_dev.numel() * 8)
    assert same_bits(a_dev.cpu().numpy(), a_np)
    one.train_finish()
    want = one.train_export("gradient")
    one.close()
    for label, load in (("numpy", lambda e: e.train_import("accum", a_np)),
                        ("torch CUDA tensor", lambda e: e.train_import_ptr("accum", a_dev.data_ptr(), a_dev.numel() * 8))):
        fresh = trainer(sd, B, T)
        load(fresh)
        fresh.train_finish()
        assert same_bits(fresh.train_export("gradient"), want), label
        fresh.close()
    parts = []
    for r, f in ((r1, f1), (r2, f2)):
        e = trainer(sd, B, T)
        e.train_grad(r, f)
        e.train_accumulate()
        parts.append(e.train_export("accum"))
        e.close()
    for a, b in ((0, 1), (1, 0)):
        e = trainer(sd, B, T)
        e.train_import("accum", parts[a] + parts[b])
        e.train_finish()
        assert same_bits(e.train_export("gradient"), want), (a, b)
        e.close()


def test_nonfinite_micro_batch_skips_the_step():
    """A NaN inside one micro-batch's window: its gradient call reports PNB_ERR_DOMAIN as before, a clean call after it
    clears the call's own flag, and finish flags the combined gradient again, so Adam is skipped (weights, m and v keep
    their bits) and wait() reports PNB_ERR_DOMAIN."""
    sd = synth_state_dict(0)
    rec = moderate_records(2, 20, 230)
    eng = trainer(sd, 2, 20)
    eng.train_grad(rec)
    eng.train_adam(1e-3, 1)
    eng.wait()
    before = {k: eng.train_export(k) for k in ("weights", "m", "v")}
    bad = rec.copy()
    bad[1, 7, 5] = np.nan
    with pytest.raises(api.PnbError, match=r"\(-5\)"):
        eng.train_grad(bad)
    eng.train_accumulate()
    with pytest.raises(api.PnbError, match=r"\(-5\)"):   # sticky until pnb_reset
        eng.train_grad(rec)
    assert np.all(np.isfinite(eng.train_export("gradient")))
    eng.train_accumulate()
    eng.train_finish()
    assert np.isnan(eng.train_export("gradient")).any()
    eng.train_adam(1e-3, 2)
    with pytest.raises(api.PnbError, match=r"\(-5\)"):
        eng.wait()
    for k, a in before.items():
        assert same_bits(eng.train_export(k), a), k
    eng.close()


def test_refusals_change_nothing():
    L = api.load_library()
    sd = synth_state_dict(0)
    rec = moderate_records(2, 10, 240)
    other = api.Engine(2, 10, pack_state_dict(sd), api.NETWORK_ONLY)
    buf = np.zeros(N_PARAMS + 1, np.float64)
    assert L.pnb_train_accumulate(other.h, None) == ARG
    assert L.pnb_train_finish(other.h, None) == ARG
    assert L.pnb_train_export(other.h, 4, buf.ctypes.data, buf.nbytes) == ARG
    assert L.pnb_train_import(other.h, 4, buf.ctypes.data, buf.nbytes) == ARG
    other.close()

    eng = trainer(sd, 2, 10)
    bytes0 = int(L.pnb_engine_bytes(eng.h))
    n0 = eng.launches
    assert L.pnb_train_accumulate(eng.h, None) == ARG       # no gradient call yet
    assert L.pnb_train_finish(eng.h, None) == ARG           # nothing accumulated
    assert eng.launches == n0
    assert int(L.pnb_engine_bytes(eng.h)) == bytes0         # refused before the accumulator exists
    eng.train_grad(rec)
    eng.train_accumulate()
    assert int(L.pnb_engine_bytes(eng.h)) == bytes0 + (N_PARAMS + 1) * 8
    eng.train_grad(rec, [10, 4])
    eng.train_accumulate()
    eng.wait()
    snap = state(eng)
    n0 = eng.launches
    assert L.pnb_train_accumulate(eng.h, None) == ARG       # the held gradient is already counted
    assert L.pnb_train_adam(eng.h, C.c_double(1e-3), 1, None) == ARG   # unfinished accumulation
    assert L.pnb_train_import(eng.h, 4, buf.ctypes.data, buf.nbytes - 8) == ARG
    assert L.pnb_train_import(eng.h, 4, buf.ctypes.data, buf.nbytes + 8) == ARG
    assert L.pnb_train_export(eng.h, 4, buf.ctypes.data, buf.nbytes - 8) == ARG
    assert L.pnb_train_export(eng.h, 5, buf.ctypes.data, buf.nbytes) == ARG
    assert L.pnb_train_export(eng.h, 4, None, buf.nbytes) == ARG
    assert eng.launches == n0
    for k, a in state(eng).items():
        assert same_bits(a, snap[k]), k
    assert snap["accum"][-1] == 2 * 10 + 10 + 4
    eng.train_finish()
    eng.wait()
    snap = state(eng)
    assert L.pnb_train_finish(eng.h, None) == ARG           # nothing since the last finish
    assert L.pnb_train_accumulate(eng.h, None) == ARG       # the finished gradient is no call's own
    for k, a in state(eng).items():
        assert same_bits(a, snap[k]), k
    eng.train_adam(1e-3, 1)
    # pnb_reset empties the accumulator and keeps the held gradient, still due
    eng.train_grad(rec)
    eng.train_accumulate()
    g = eng.train_export("gradient")
    eng.reset()
    assert not np.any(eng.train_export("accum"))
    assert L.pnb_train_finish(eng.h, None) == ARG
    assert same_bits(eng.train_export("gradient"), g)
    eng.train_adam(1e-3, 2)
    eng.wait()
    eng.close()
