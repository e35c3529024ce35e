"""The waveform-training CLI (python -m percepnet_b200.train_wave) and SignalPath's state export / import on the GPU:
the CLI's first step is a hand-written SignalPath + PercepNet + Adam loop bit for bit, a resumed run is an uninterrupted
one bit for bit, training lowers the loss, and the dev score in the deployed arithmetic meets the training path's loss."""
import re

import numpy as np
import pytest

from percepnet_b200 import train_wave as TW

pytestmark = pytest.mark.gpu

FRAME = 480
# |deployed dev L1 - training-path L1| / training-path L1 at the initial weights: measured 2.0e-7 (plain) and 2.3e-7
# (post-filter) on an H100 80GB HBM3 at a 700 W power limit; the SNRs differed by 1e-5 dB
DEV_BAR, SNR_BAR_DB = 2e-6, 1e-3


@pytest.fixture(scope="module")
def torch():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device")
    return torch


def write_pairs(d, hops, seed, name="p"):
    """Synthetic pairs (synth.synth_pairs) of the given hops as raw int16 files, the first with a trailing partial hop;
    returns the list file and the pairs as the CLI reads them."""
    from percepnet_b200.synth import synth_pairs
    clean, noisy = synth_pairs(len(hops), max(hops) + 1, seed=seed)
    lines = []
    for k, n in enumerate(hops):
        c, x = d / f"{name}{k}_clean.pcm", d / f"{name}{k}_noisy.pcm"
        end = n * FRAME + (100 if k == 0 else 0)
        clean[k, :end].astype("<i2").tofile(c)
        noisy[k, :end].astype("<i2").tofile(x)
        lines.append(f"{c} {x}")
    lst = d / f"{name}.txt"
    lst.write_text("\n".join(lines) + "\n")
    data = [TW.load_pair(*line.split(), n) for line, n in zip(lines, hops)]
    return str(lst), data


def run(capsys, lst, out, steps, W, B, seed, lr="1e-3", extra=()):
    argv = ["--list", lst, "--window", str(W), "--batch", str(B), "--steps", str(steps), "--lr", lr, "--seed",
            str(seed), "--out", out, *extra]
    assert TW.main(argv) == 0
    log = capsys.readouterr().out
    with capsys.disabled():
        print(log)
    return log


def losses(log):
    return re.findall(r"\] loss (\S+)", log)


def test_first_step_is_the_hand_written_loop(torch, tmp_path, capsys):
    """Step 1 of the CLI: the logged loss and the weights after it equal, bit for bit, SignalPath + PercepNet + Adam
    written out here on the same schedule inputs."""
    from percepnet_b200.torch_module import STATE_FLOATS, PercepNet
    from percepnet_b200.torch_signal import SignalPath
    from percepnet_b200.weights import pack_state_dict, synth_state_dict
    hops, W, B, seed, lr = [20, 27, 13], 8, 2, 3, 1e-3
    lst, data = write_pairs(tmp_path, hops, 900)
    out = str(tmp_path / "o.pnbw")
    log = run(capsys, lst, out, 1, W, B, seed, lr=str(lr))
    assert re.search(r"\[1,      1\] loss \S+  counted \d+", log)

    cur = TW.first_cursor(len(hops), B, seed)
    x, tgt, lo, hi = TW.step_inputs(data, cur, W)
    count = int((hi - lo).sum())
    net = PercepNet()
    net.load_state_dict({k: torch.from_numpy(v) for k, v in synth_state_dict(seed).items()})
    net = net.cuda()
    opt = torch.optim.Adam(net.parameters(), lr=lr)
    sp = SignalPath(B, W, device="cuda")
    state = torch.zeros((B, STATE_FLOATS), device="cuda")
    features, ops = sp.analyze(torch.from_numpy(x).cuda().float())
    gr, _ = net(features, state, return_state=True)
    y = sp.synthesize(gr, ops)
    j = torch.arange(W * FRAME, device="cuda")
    mask = (j >= torch.from_numpy(lo).cuda()[:, None]) & (j < torch.from_numpy(hi).cuda()[:, None])
    loss = torch.where(mask, (y - torch.from_numpy(tgt).cuda().float()).abs(), 0).sum() / (32768.0 * count)
    opt.zero_grad()
    loss.backward()
    opt.step()
    print(f"hand-written loop: loss {float(loss)!r}, {count} counted")
    assert np.float32(losses(log)[0]) == np.float32(loss.item())   # 9 digits: a float32 round trip
    assert f"counted {count}" in log
    want = pack_state_dict({k: v.detach().cpu().numpy() for k, v in net.state_dict().items()}).flat()
    got = TW.read_blob(out).flat()
    assert np.array_equal(got.view(np.int32), want.view(np.int32))
    assert not np.array_equal(want, pack_state_dict(synth_state_dict(seed)).flat())
    sp.close()
    net.close()


@pytest.mark.parametrize("post", [False, True], ids=["plain", "postfilter"])
def test_resumed_run_equals_uninterrupted_run(torch, tmp_path, capsys, post):
    """2k steps straight against k steps and k more resumed from --checkpoint, the checkpoint with every row in the
    middle of its track: the same --out bytes, Adam state, network and signal state and logged losses."""
    hops, W, B, seed, k = [20, 27, 13, 35], 8, 2, 7, 2
    lst, _ = write_pairs(tmp_path, hops, 910)
    cur = TW.cursor_at(hops, B, W, seed, k)
    assert np.all(cur.offset > 0)
    assert np.any(TW.cursor_at(hops, B, W, seed, k + 1).offset == 0)   # a row starts a track after the resume
    extra = ["--postfilter"] if post else []
    full, part = str(tmp_path / "full.pnbw"), str(tmp_path / "part.pnbw")
    ck_full, ck = str(tmp_path / "full.npz"), str(tmp_path / "ck.npz")
    log_full = run(capsys, lst, full, 2 * k, W, B, seed, extra=extra + ["--checkpoint", ck_full])
    log_a = run(capsys, lst, part, k, W, B, seed, extra=extra + ["--checkpoint", ck])
    mid = dict(np.load(ck))
    log_b = run(capsys, lst, part, 2 * k, W, B, seed, extra=extra + ["--checkpoint", ck])
    assert f"resumed {ck} at step {k}" in log_b
    assert np.any(mid["net_state"] != 0) and np.any(mid["signal_state"] != 0)
    assert np.array_equal(mid["row_offset"], cur.offset) and np.array_equal(mid["row_pair"], cur.pair)
    assert len(losses(log_full)) == 2 * k and losses(log_a) + losses(log_b) == losses(log_full)
    with open(full, "rb") as f1, open(part, "rb") as f2:
        assert f1.read() == f2.read()
    a, b = np.load(ck_full), np.load(ck)
    for key in a.files:
        assert a[key].tobytes() == b[key].tobytes(), key
    assert int(a["step"]) == int(a["adam_step"]) == 2 * k


def test_training_lowers_the_loss(torch, tmp_path, capsys):
    """Four pairs of 34 hops in windows of 40 hops on four rows: each step sees the four whole files (in the epoch's
    row order), so the losses compare; the last five of 30 Adam steps are below the first."""
    lst, _ = write_pairs(tmp_path, [34] * 4, 920)
    log = run(capsys, lst, str(tmp_path / "o.pnbw"), 30, 40, 4, 1)
    v = [float(s) for s in losses(log)]
    assert len(v) == 30 and len(set(re.findall(r"counted (\d+)", log))) == 1
    print("losses:", " ".join(f"{x:.5f}" for x in v))
    assert max(v[-5:]) < v[0]


def test_dev_score_meets_the_training_path(torch, tmp_path, capsys):
    """At the initial weights the deployed dev L1 (fp32 engine, tansig tables) is within DEV_BAR of the training path's
    forward loss on the same tracks (SignalPath + PercepNet, exact tanh and sigmoid), with and without the post-filter;
    the CLI prints the noisy input's SNR as numpy computes it, and a dev line per --eval-every."""
    from percepnet_b200.torch_module import STATE_FLOATS, PercepNet
    from percepnet_b200.torch_signal import SignalPath
    from percepnet_b200.weights import synth_state_dict
    hops, W, seed = [30, 17, 45], 16, 2
    dev_lst, dev = write_pairs(tmp_path, hops, 930, name="dev")
    sd = synth_state_dict(seed)
    net = PercepNet()
    net.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()})
    net = net.cuda()
    B = len(hops)
    n_win = max(TW.track_hops(n, W) for n in hops) // W
    for post in (False, True):
        d = TW.score_dev(sd, dev, W, post)
        sp = SignalPath(B, W, postfilter=post, device="cuda")
        state = torch.zeros((B, STATE_FLOATS), device="cuda")
        s1 = s2 = s3 = 0.0
        count = 0
        with torch.no_grad():
            for w in range(n_win):
                x, tgt, lo, hi = TW.step_inputs(dev, TW.Cursor(0, 0, np.arange(B), np.full(B, w * W)), W)
                features, ops = sp.analyze(torch.from_numpy(x).cuda().float())
                gr, state = net(features, state, return_state=True)
                y = sp.synthesize(gr, ops).double().cpu().numpy()
                for b in range(B):
                    c = tgt[b, lo[b]:hi[b]].astype(np.float64)
                    e = y[b, lo[b]:hi[b]] - c
                    s1, s2, s3 = s1 + np.abs(e).sum(), s2 + (c * c).sum(), s3 + (e * e).sum()
                count += int((hi - lo).sum())
        sp.close()
        assert count == d["count"] == sum(n * FRAME for n in hops)
        l1 = s1 / (32768.0 * count)
        snr = 10 * np.log10(s2 / s3)
        gap = abs(d["l1"] - l1) / l1
        print(f"post={post}: deployed L1 {d['l1']:.9g} SNR {d['snr']:.5f} dB; training path L1 {l1:.9g} SNR "
              f"{snr:.5f} dB; L1 gap {gap:.3e}")
        assert gap < DEV_BAR
        assert abs(d["snr"] - snr) < SNR_BAR_DB
    net.close()

    lst, _ = write_pairs(tmp_path, [20, 25], 931)
    log = run(capsys, lst, str(tmp_path / "o.pnbw"), 2, 8, 2, seed,
              extra=["--dev-list", dev_lst, "--eval-every", "1"])
    num = sum(float(np.sum(c.astype(np.float64) ** 2)) for c, _ in dev)
    den = sum(float(np.sum((x.astype(np.float64) - c.astype(np.float64)) ** 2)) for c, x in dev)
    want = 10 * np.log10(num / den)
    got = re.findall(r"dev noisy input: SNR (\S+) dB", log)
    assert got == [f"{want:.4f}"]
    assert len(re.findall(r"dev \(deployed arithmetic\) L1 \S+  SNR \S+ dB  counted \d+", log)) == 2


def test_signal_path_state_round_trip(torch):
    """Export, reset and import a row between windows: the next window's features and output equal an untouched path's
    bit for bit (a reset alone does not); both calls are refused before the first analyze and while an analysis is
    pending."""
    from percepnet_b200.synth import synth_pcm
    from percepnet_b200.torch_signal import SignalPath
    B, T = 3, 8
    x = torch.from_numpy(synth_pcm(B, 3 * T, seed=940, scale=32768.0)).cuda()
    gen = torch.Generator(device="cuda").manual_seed(941)
    grs = [torch.rand((B, T, 68), device="cuda", generator=gen) for _ in range(3)]
    paths = [SignalPath(B, T, postfilter=True, device="cuda") for _ in range(3)]   # untouched, round trip, reset only
    fresh = SignalPath(B, T, device="cuda")
    some = torch.zeros((1, 8), dtype=torch.uint8, device="cuda")   # refused before the blobs are looked at
    with pytest.raises(RuntimeError, match="first analyze"):
        fresh.export_states([0])
    with pytest.raises(RuntimeError, match="first analyze"):
        fresh.import_states([0], some)
    res = []
    for w in range(3):
        xw = x[:, w * T * FRAME:(w + 1) * T * FRAME]
        if w == 2:
            blobs = paths[1].export_states([1])
            assert blobs.dtype == torch.uint8 and blobs.is_cuda and blobs.shape[0] == 1
            paths[1].reset([1])
            paths[1].import_states([1], blobs)
            paths[2].reset([1])
        res = []
        for sp in paths:
            f, ops = sp.analyze(xw)
            if w == 1 and sp is paths[0]:
                with pytest.raises(RuntimeError, match="pending"):
                    sp.export_states([0])
                with pytest.raises(RuntimeError, match="pending"):
                    sp.import_states([0], some)
            res.append((f, sp.synthesize(grs[w], ops)))
    torch.cuda.synchronize()
    (f0, y0), (f1, y1), (f2, y2) = res
    assert torch.equal(f0, f1) and torch.equal(y0, y1)
    assert not torch.equal(f0[1], f2[1]) and torch.equal(f0[0], f2[0])
    for sp in paths + [fresh]:
        sp.close()

