"""CPU side of the network-only calls (pnb_compute_rnn_*) and of the model-scoring CLI (percepnet_b200.eval_records).

The premise: a training record is a network input once scaled.  {30 * rec[0..67], rec[68], rec[69]} of the records
train() writes for (speech, noisy) are, bit for bit, the features rnnoise_process_frame computes on noisy as float
(create_features, denoise.cpp:487-496; NORM_RATIO is 1, denoise.cpp:41, so there is no /32768).
"""
import numpy as np
import pytest

from util import same_bits


@pytest.mark.parametrize("div", [1, 16])
def test_scaled_records_are_the_network_input(oracle, model0, div):
    from percepnet_b200.synth import synth_pairs
    clean, noisy = synth_pairs(3, 30, seed=401)
    clean, noisy = (clean // div).astype(np.int16), (noisy // div).astype(np.int16)
    for k in range(3):
        rec = oracle.train_records(clean[k], noisy[k])
        h = oracle.create(model0)
        _, _, taps = oracle.process_stream(h, noisy[k].astype(np.float32), True, taps=True)
        oracle.destroy(h)
        feats = np.stack([t.np("features") for t in taps])
        scaled = np.concatenate([rec[:, :68] * np.float32(30), rec[:, 68:70]], axis=1)
        assert scaled.dtype == np.float32
        assert same_bits(scaled, feats), k


def test_arguments():
    from percepnet_b200 import eval_records as E
    a = E.parse_args(["--model", "m.pnbw", "a.f32", "b.f32"])
    assert a.files == ["a.f32", "b.f32"] and not a.tensor and a.batch == 4096 and a.chunk == 100 and a.pred_dir is None
    for bad in (["a.f32"], ["--model", "m.pnbw"], ["--model", "m", "--chunk", "0", "a"], ["--model", "m", "--conv-wide", "a"]):
        with pytest.raises(SystemExit):
            E.parse_args(bad)


def test_list_file(tmp_path):
    from percepnet_b200 import eval_records as E
    lst = tmp_path / "files.txt"
    lst.write_text("x.f32\n\n  y.f32  \n")
    a = E.parse_args(["--model", "m", "--list", str(lst), "--tensor", "--conv-wide", "--batch", "2", "--chunk", "7",
                      "--pred-dir", "out", "w.f32"])
    assert a.files == ["w.f32", "x.f32", "y.f32"] and a.tensor and a.conv_wide and (a.batch, a.chunk) == (2, 7)
    assert a.pred_dir == "out"


def test_read_records(tmp_path):
    from percepnet_b200 import eval_records as E
    rec = np.arange(5 * 138, dtype=np.float32).reshape(5, 138)
    rec.tofile(tmp_path / "r.f32")
    assert np.array_equal(E.read_records(str(tmp_path / "r.f32")), rec)
    rec.ravel()[:137].tofile(tmp_path / "bad.f32")
    with pytest.raises(ValueError):
        E.read_records(str(tmp_path / "bad.f32"))
    open(tmp_path / "empty.f32", "wb").close()
    with pytest.raises(ValueError):
        E.read_records(str(tmp_path / "empty.f32"))


def test_batches_and_padding():
    from percepnet_b200 import eval_records as E
    lengths = [3, 9, 1, 9, 4]
    groups = E.plan_batches(lengths, 2)
    assert groups == [[1, 3], [4, 0], [2]]                     # longest first, stable among equals
    assert sorted(i for g in groups for i in g) == list(range(5))
    assert E.plan_batches(lengths, 10) == [[1, 3, 4, 0, 2]]
    rng = np.random.RandomState(5)
    recs = [rng.rand(n, 138).astype(np.float32) for n in (4, 7, 2)]
    x = E.pad_batch(recs)
    assert x.shape == (3, 7, 138) and x.dtype == np.float32
    for k, r in enumerate(recs):
        assert np.array_equal(x[k, :len(r)], r) and not x[k, len(r):].any()


def _custom_loss(outputs, targets):
    """rnn_train.py:153-176 (CustomLoss.forward), transcribed in float64 torch."""
    import torch
    gamma, C4 = 0.5, 10
    gb_hat, rb_hat = outputs[:, :, :34], outputs[:, :, 34:68]
    gb, rb = targets[:, :, :34], targets[:, :, 34:68]
    return ((torch.mean(torch.pow((torch.pow(gb, gamma) - torch.pow(gb_hat, gamma)), 2))),
            C4 * torch.mean(torch.pow(torch.pow(gb, gamma) - torch.pow(gb_hat, gamma), 4)),
            torch.mean(torch.pow(torch.pow((1 - rb), gamma) - torch.pow((1 - rb_hat), gamma), 2)))


def test_loss_is_the_training_loss():
    import torch
    from percepnet_b200 import eval_records as E
    rng = np.random.RandomState(9)
    lengths = (13, 5, 21)
    preds = [rng.rand(n, 68).astype(np.float32) for n in lengths]
    recs = [rng.rand(n, 138).astype(np.float32) for n in lengths]
    recs[1][2, 70:104] = 0.0                                   # silent bands: g = 0 labels
    recs[2][4, 104:] = 1.0                                     # r = 1 labels
    total = np.zeros(4)
    for p, r in zip(preds, recs):
        s = E.loss_sums(p, r)
        total += s
        t = E.loss_terms(s)
        want = _custom_loss(torch.from_numpy(p[None].astype(np.float64)), torch.from_numpy(r[None, :, 70:].astype(np.float64)))
        got = (t["g2"], t["g4"], t["r2"])
        assert np.allclose(got, [float(w) for w in want], rtol=1e-12, atol=0)
        assert t["total"] == pytest.approx(sum(float(w) for w in want), rel=1e-12)
    # overall: the means over every frame of every file, i.e. the loss of the files concatenated along time
    t = E.loss_terms(total)
    cat = lambda xs: torch.from_numpy(np.concatenate(xs)[None].astype(np.float64))
    want = _custom_loss(cat(preds), cat([r[:, 70:] for r in recs]))
    assert np.allclose((t["g2"], t["g4"], t["r2"]), [float(w) for w in want], rtol=1e-12, atol=0)
