"""BASELINE.json's full single-GPU size (config 3: 16 384 concurrent streams, tensor-core network; and 8 192
file pairs for the training-data generator) checked through properties that do not need 16 384 oracle runs:
every replica of a base stream must come out bit-identical wherever it sits in the batch (every tile, CTA pair and
row position computes the same thing), and the base streams themselves are anchored to the oracle.  At this size the
tensor path's GRU chain runs hop-major (util.first_hop_major); the benchmark's own shape, max_frames = 100, is run on
device buffers and tied bit for bit to a 48-stream engine, which runs the chain in anti-diagonal order."""
import numpy as np
import pytest

from util import same_bits

pytestmark = pytest.mark.gpu

S_FULL, N_BASE, F = 16384, 48, 8


@pytest.fixture(scope="module")
def api():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device")
    from percepnet_b200 import api
    api.load_library()
    return api


def test_full_batch_enhancement_replicas_and_oracle(api, oracle, model0):
    from percepnet_b200.synth import synth_pcm
    base = synth_pcm(N_BASE, 2 * F, seed=2468)
    idx = np.arange(S_FULL) % N_BASE
    x = base[idx]
    eng = api.Engine(S_FULL, F, model0, api.NN_TENSOR)
    outs, grs = [], []
    for c in range(2):                                        # two calls: the carried state is exercised at full size
        o, g = eng.process(np.ascontiguousarray(x[:, c * F * 480:(c + 1) * F * 480]), want_gr=True)
        outs.append(o); grs.append(g)
    eng.close()
    out, gr = np.concatenate(outs, axis=1), np.concatenate(grs, axis=0)          # [S, 16*480], [16, S, 68]
    assert same_bits(out, out[:N_BASE][idx]), "replicas of a stream differ across the batch"
    assert same_bits(gr, gr[:, :N_BASE][:, idx]), "replica g/r differ across the batch"
    for s in range(6):                                        # anchor: the oracle on the base streams
        h = oracle.create(model0)
        ref, ref_gr, _ = oracle.process_stream(h, base[s], True)
        oracle.destroy(h)
        rel = np.abs(gr[:, s] - ref_gr) / np.maximum(np.abs(ref_gr), 1e-6)
        assert rel.max() < 1e-4, (s, rel.max())
        lsb = np.abs(np.trunc(out[s].astype(np.float64) * 32768) - np.trunc(ref.astype(np.float64) * 32768)).max()
        assert lsb <= 1, (s, lsb)
    assert np.abs(out).max() > 1e-3                            # the batch did produce audio


def test_full_batch_training_records_replicas_and_oracle(api, oracle):
    from percepnet_b200.synth import synth_pairs
    N = S_FULL // 2
    clean, noisy = synth_pairs(N_BASE, F, seed=1357)
    idx = np.arange(N) % N_BASE
    eng = api.Engine(2 * N, F, None, api.TRAIN_DATA)
    rec = eng.train_records(clean[idx], noisy[idx])
    eng.close()
    assert same_bits(rec, rec[:N_BASE][idx])
    for k in range(4):
        want = oracle.train_records(clean[k], noisy[k])
        assert same_bits(rec[k][:, :70], want[:, :70]) and same_bits(rec[k][:, 104:], want[:, 104:])
        assert np.allclose(rec[k][:, 70:104], want[:, 70:104], rtol=1e-6, atol=1e-12)


# ------------------------------------------------------------------------------------------------ bench.py's shape
HOP = 480
F_BENCH = 100          # bench.py's hops per call: one history slide per call, the spectrum ring wraps on the second call
N_ANCHOR = 4
BENCH_LEGS = [  # (id, streams, flags, input scale, calls)
    ("tensor", S_FULL, "tensor", 1.0, 3),
    ("wide-int16", S_FULL, "wide", 32768.0, 3),     # bench.py's second timed run
    ("fp32", S_FULL, "fp32", 1.0, 2),
]


def _same_bits_dev(a, b):
    """torch tensors equal bit for bit (+-0 folded, as util.same_bits)"""
    import torch
    return bool(((a.view(torch.int32) == b.view(torch.int32)) | ((a == 0) & (b == 0))).all())


def _replicas_match(d, idx, dim, chunk=2048):
    """rows n_base.. of d (along dim) equal their base rows idx[row], compared in chunks on the device"""
    n = d.shape[dim]
    for r0 in range(N_BASE, n, chunk):
        r1 = min(n, r0 + chunk)
        if not _same_bits_dev(d.narrow(dim, r0, r1 - r0), d.index_select(dim, idx[r0:r1])):
            return False
    return True


@pytest.mark.parametrize("leg", BENCH_LEGS, ids=[b[0] for b in BENCH_LEGS])
def test_benchmark_shape_replicas_twin_and_oracle(api, oracle, model0, leg):
    """16 384 streams, max_frames = 100, calls of 100 hops from device buffers (pnb_process_device with a device g/r
    buffer): 48 base streams uploaded once and expanded on the device.  Every replica is bit-identical to its base row;
    the base rows are bit-identical to a 48-stream engine with max_frames = 100 fed the same calls; four anchors stay
    within 1 LSB of the oracle's PCM and within 1e-4 of the float64 network's g/r fed the oracle's features."""
    import time

    import torch
    from percepnet_b200.synth import synth_pcm
    from test_gpu_parity import _lsb_diff, _oracle_run
    from test_gpu_layer_bounds import DOMAIN
    cid, S, kind, scale, n_calls = leg
    flags = {"tensor": api.NN_TENSOR, "wide": api.NN_TENSOR | api.CONV_WIDE, "fp32": api.NN_FP32}[kind]
    L = F_BENCH * HOP
    base = synth_pcm(N_BASE, n_calls * F_BENCH, seed=8642, scale=scale)
    need = (2 * S * L + F_BENCH * S * 68 + N_BASE * n_calls * L) * 4 + (1 << 30)   # in, out, g/r, bases, compare slack
    free, total = torch.cuda.mem_get_info()
    if free < need:
        pytest.fail(f"{cid}: {free / 1e9:.1f} GB of {total / 1e9:.1f} GB free on the device; the test tensors alone need "
                    f"{need / 1e9:.1f} GB, before the engine")
    eng = api.Engine(S, F_BENCH, model0, flags)
    try:
        free1, _ = torch.cuda.mem_get_info()
        print(f"\n  {cid}: engine of {S} streams x {F_BENCH} hops takes {(free - free1) / 1e9:.1f} GB")
        if free1 < need:
            pytest.fail(f"{cid}: {free1 / 1e9:.1f} GB free after creating the engine, the test tensors need {need / 1e9:.1f} GB")
        d_base = torch.from_numpy(base).cuda()
        idx = torch.arange(S, device="cuda") % N_BASE
        d_out = torch.empty((S, L), device="cuda")
        d_gr = torch.empty((F_BENCH, S, 68), device="cuda")
        st = torch.cuda.current_stream().cuda_stream
        outs, grs = [], []
        t0 = time.perf_counter()
        for c in range(n_calls):
            d_in = d_base[:, c * L:(c + 1) * L].index_select(0, idx)
            eng.process_device(d_in.data_ptr(), L, d_out.data_ptr(), L, F_BENCH, d_gr.data_ptr(), stream=st)
            eng.check(st)
            del d_in
            assert _replicas_match(d_out, idx, 0), f"{cid}: call {c}: replicas of a stream differ across the batch"
            assert _replicas_match(d_gr, idx, 1), f"{cid}: call {c}: replica g/r differ across the batch"
            outs.append(d_out[:N_BASE].cpu().numpy())
            grs.append(d_gr[:, :N_BASE].cpu().numpy())
        print(f"  {cid}: {n_calls} calls of {F_BENCH} hops with their checks in {time.perf_counter() - t0:.1f} s")
    finally:
        eng.close()
    del d_out, d_gr
    out, gr = np.concatenate(outs, axis=1), np.concatenate(grs, axis=0)
    twin = api.Engine(N_BASE, F_BENCH, model0, flags)
    try:
        for c in range(n_calls):
            o, g = twin.process(np.ascontiguousarray(base[:, c * L:(c + 1) * L]), want_gr=True)
            assert same_bits(out[:, c * L:(c + 1) * L], o), f"{cid}: call {c}: PCM differs from the 48-stream engine"
            assert same_bits(gr[c * F_BENCH:(c + 1) * F_BENCH], g), f"{cid}: call {c}: g/r differ from the 48-stream engine"
        twin.check()
    finally:
        twin.close()
    # anchors: base rows on which the reference's own fp32 arithmetic stays within 1e-4 of the float64 network.  At
    # int16 scale some streams reach pre-activations ~1e7 where the reference's table activations are ill-conditioned
    # and its own g/r drift ~1e-3 from float64 over a few hundred hops; float64 is no yardstick for those.
    worst_rel, worst_lsb, anchors, skipped = 0.0, 0.0, [], []
    for s in [0, 17, 30, 47] + list(range(1, 17)):
        if len(anchors) == N_ANCHOR:
            break
        ref, gr32, taps = _oracle_run(oracle, model0, base[s:s + 1])
        g, r, mp = oracle.rnn_f64(model0, np.stack([t.np("features") for t in taps[0]]))
        assert mp.max() < DOMAIN, (cid, s, mp.max())
        t64 = np.concatenate([g, r], 1)
        den = np.maximum(np.abs(t64), 1e-6)
        e_ref = float((np.abs(gr32[:, 0] - t64) / den).max())
        if e_ref >= 1e-4:
            skipped.append((s, e_ref))
            continue
        anchors.append(s)
        worst_rel = max(worst_rel, float((np.abs(gr[:, s] - t64) / den).max()))
        worst_lsb = max(worst_lsb, float(_lsb_diff(out[s], ref[0], scale == 1.0)))
    print(f"  {cid}: anchors {anchors} over {n_calls * F_BENCH} hops: g/r within {worst_rel:.2e} of float64, PCM within "
          f"{worst_lsb:g} LSB of the oracle; skipped (row, reference fp32 vs float64): {skipped}")
    assert len(anchors) == N_ANCHOR, skipped
    assert worst_rel < 1e-4 and worst_lsb <= 1
    assert np.abs(out).max() > 1e-3 * scale
