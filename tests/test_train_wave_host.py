"""The waveform-training CLI's host side (python -m percepnet_b200.train_wave): its refusals come before any engine, its
schedule visits every pair once per epoch with no idle row and resumes where it stopped, and its targets put every
clean sample of every pair exactly once at output index clean index + 2880."""
import numpy as np
import pytest

from percepnet_b200 import api, train_wave as TW

FRAME, LAG = 480, 2880


def write_pair(tmp_path, name, n_clean, n_noisy=None, seed=0):
    """A pair of raw int16 files of n_clean and n_noisy samples."""
    rng = np.random.RandomState(seed)
    c, x = tmp_path / f"{name}_clean.pcm", tmp_path / f"{name}_noisy.pcm"
    rng.randint(-3000, 3000, n_clean).astype("<i2").tofile(c)
    rng.randint(-3000, 3000, n_clean if n_noisy is None else n_noisy).astype("<i2").tofile(x)
    return f"{c} {x}"


def write_list(tmp_path, name, lines):
    p = tmp_path / name
    p.write_text("\n".join(lines) + "\n")
    return str(p)


@pytest.fixture
def no_engine(monkeypatch):
    def refuse(*a, **k):
        raise AssertionError("an engine was created before the refusal")
    monkeypatch.setattr(api, "Engine", refuse)


def run(argv):
    """The CLI's exit code: main's return value, or argparse's SystemExit code."""
    try:
        return TW.main(argv)
    except SystemExit as ex:
        return ex.code


def test_refusals_before_any_engine(tmp_path, capsys, no_engine):
    good = [write_pair(tmp_path, f"p{k}", (20 + k) * FRAME + k, seed=k) for k in range(3)]
    lst = write_list(tmp_path, "good.txt", good)
    base = ["--window", "8", "--batch", "2", "--steps", "1", "--out", str(tmp_path / "o.pnbw")]
    cases = {
        "hop counts differ": ["--list", write_list(tmp_path, "a.txt", good + [write_pair(tmp_path, "d", 10 * FRAME,
                                                                                         9 * FRAME + 479)])] + base,
        "shorter than one hop": ["--list", write_list(tmp_path, "b.txt", good + [write_pair(tmp_path, "s", 479)])] + base,
        "dev hop counts differ": ["--list", lst, "--dev-list", write_list(tmp_path, "c.txt", [
            write_pair(tmp_path, "e", 5 * FRAME, 6 * FRAME)]), "--eval-every", "1"] + base,
        "fewer pairs than --batch": ["--list", lst, "--window", "8", "--batch", "4", "--steps", "1", "--out", "o"],
        "window 6": ["--list", lst, "--window", "6", "--batch", "2", "--steps", "1", "--out", "o"],
        "window 1": ["--list", lst, "--window", "1", "--batch", "2", "--steps", "1", "--out", "o"],
        "window 0": ["--list", lst, "--window", "0", "--batch", "2", "--steps", "1", "--out", "o"],
        "batch 0": ["--list", lst, "--window", "8", "--batch", "0", "--steps", "1", "--out", "o"],
        "steps -1": ["--list", lst, "--window", "8", "--batch", "2", "--steps", "-1", "--out", "o"],
        "lr nan": ["--list", lst, "--lr", "nan"] + base,
        "lr < 0": ["--list", lst, "--lr", "-1e-4"] + base,
        "dev list without --eval-every": ["--list", lst, "--dev-list", lst] + base,
        "no --out": ["--list", lst, "--window", "8", "--batch", "2", "--steps", "1"],
        "a line of three paths": ["--list", write_list(tmp_path, "t.txt", good + ["a b c"])] + base,
        "a missing file": ["--list", write_list(tmp_path, "m.txt", good + [f"{tmp_path}/none.pcm {tmp_path}/n.pcm"])]
        + base,
    }
    for what, argv in cases.items():
        assert run(argv) == 2, what
        err = capsys.readouterr().err
        assert err.strip(), what
        print(f"{what}: {err.strip().splitlines()[-1]}")


def test_window_count_is_never_zero():
    """For W >= 7 every window of every track counts at least one sample (W = 6 does not: a first window lies wholly
    within the lag); the track is the pair, the six lag hops and padding to whole windows."""
    rng = np.random.RandomState(1)
    lengths = [1, 2, 5, 6, 7, 13, 40] + rng.randint(1, 300, 40).tolist()
    for W in (7, 8, 13, 50, 500):
        for n in lengths:
            L = TW.track_hops(n, W)
            assert L % W == 0 and n + 6 <= L < n + 6 + W
            clean = np.arange(n * FRAME, dtype=np.int16)
            for o in range(0, L, W):
                _, _, lo, hi = TW.window_of(clean, clean, o, W)
                assert hi > lo, (W, n, o)
    _, _, lo, hi = TW.window_of(np.ones(FRAME, np.int16), np.ones(FRAME, np.int16), 0, 6)
    assert hi == lo


def walk(hops, B, W, seed, steps):
    """The cursors before steps 0 .. steps and, in order, the pairs the rows start (row order within a step)."""
    curs = [TW.first_cursor(len(hops), B, seed)]
    starts = []
    for _ in range(steps):
        cur = curs[-1]
        starts += [int(cur.pair[b]) for b in range(B) if cur.offset[b] == 0]
        curs.append(TW.next_cursor(cur, hops, W, seed))
    return curs, starts


@pytest.mark.parametrize("B", [1, 3, 7])
def test_schedule_visits_each_pair_once_per_epoch(B):
    """The pairs the rows start, in order, are epoch 0's permutation, then epoch 1's, ...; every row is inside a track
    at every step; the cursor's (epoch, pos) counts the pairs taken."""
    rng = np.random.RandomState(2)
    hops = rng.randint(1, 60, 9).tolist()
    W, seed = 8, 5
    curs, starts = walk(hops, B, W, seed, 300)
    n = len(hops)
    epochs = len(starts) // n
    assert epochs >= 3
    for e in range(epochs):
        assert starts[e * n:(e + 1) * n] == np.random.default_rng([seed, e]).permutation(n).tolist(), e
    taken = B
    for s, cur in enumerate(curs):
        assert all(0 <= o < TW.track_hops(hops[p], W) and o % W == 0 for p, o in zip(cur.pair, cur.offset)), s
        taken += int(np.sum(cur.offset == 0)) if s else 0
        assert cur.epoch * n + cur.pos == taken, s


def test_resumed_cursor_continues_the_sequence(tmp_path):
    """A cursor saved at step k and read back (as the checkpoint holds it) continues exactly as the uninterrupted run,
    step for step, inputs included; cursor_at is the same pure function of (hops, B, W, seed, step)."""
    rng = np.random.RandomState(3)
    hops = rng.randint(1, 40, 6).tolist()
    data = [(rng.randint(-99, 99, n * FRAME).astype(np.int16), rng.randint(-99, 99, n * FRAME).astype(np.int16))
            for n in hops]
    B, W, seed, k = 3, 7, 11, 9
    straight, _ = walk(hops, B, W, seed, 2 * k)
    cur = TW.cursor_at(hops, B, W, seed, k)
    assert np.any(cur.offset > 0)      # rows in the middle of a track
    np.savez(tmp_path / "c.npz", epoch=np.int64(cur.epoch), pos=np.int64(cur.pos), row_pair=cur.pair,
             row_offset=cur.offset)
    z = np.load(tmp_path / "c.npz")
    cur = TW.Cursor(int(z["epoch"]), int(z["pos"]), z["row_pair"].astype(np.int64), z["row_offset"].astype(np.int64))
    for s in range(k, 2 * k + 1):
        want = straight[s]
        assert (cur.epoch, cur.pos) == (want.epoch, want.pos), s
        assert np.array_equal(cur.pair, want.pair) and np.array_equal(cur.offset, want.offset), s
        for a, b in zip(TW.step_inputs(data, cur, W), TW.step_inputs(data, want, W)):
            assert np.array_equal(a, b), s
        again = TW.cursor_at(hops, B, W, seed, s)
        assert (again.epoch, again.pos) == (cur.epoch, cur.pos) and np.array_equal(again.pair, cur.pair)
        assert np.array_equal(again.offset, cur.offset)
        cur = TW.next_cursor(cur, hops, W, seed)


@pytest.mark.parametrize("W", [7, 10, 32])
def test_targets_hold_every_clean_sample_once(W):
    """Over epoch 0's tracks, the counted targets are every clean sample of every pair exactly once, at track output
    index j = clean index + 2880, and the inputs are the noisy file followed by zeros: a numpy restatement on random
    pair lengths, some shorter than a window."""
    rng = np.random.RandomState(4 + W)
    hops = [1, 3, W - 1] + rng.randint(1, 4 * W, 7).tolist()
    data = [(rng.randint(-30000, 30000, n * FRAME).astype(np.int16), rng.randint(-30000, 30000, n * FRAME)
             .astype(np.int16)) for n in hops]
    B, seed = 4, 6
    n = len(hops)
    cur = TW.first_cursor(n, B, seed)
    track = [None] * B          # the epoch-0 draw each row is on (None: a later epoch's)
    draws = 0
    seen = [np.zeros(h * FRAME, np.int64) for h in hops]
    finished = set()
    while len(finished) < n:
        for b in range(B):
            if cur.offset[b] == 0:
                track[b] = draws if draws < n else None
                draws += 1
        x, tgt, lo, hi = TW.step_inputs(data, cur, W)
        assert x.shape == tgt.shape == (B, W * FRAME) and x.dtype == tgt.dtype == np.int16
        for b in range(B):
            p, o = int(cur.pair[b]), int(cur.offset[b])
            j = o * FRAME + np.arange(W * FRAME)       # output index in the track
            clean, noisy = data[p]
            counted = (j >= LAG) & (j < clean.size + LAG)
            assert np.array_equal(np.arange(W * FRAME)[counted], np.arange(lo[b], hi[b])), (p, o)
            want_x = np.where(j < noisy.size, noisy[np.minimum(j, noisy.size - 1)], 0)
            assert np.array_equal(x[b], want_x), (p, o)
            assert np.all(tgt[b][~counted] == 0)
            if track[b] is not None:
                ci = j[counted] - LAG
                assert np.array_equal(tgt[b][counted], clean[ci]), (p, o)
                seen[p][ci] += 1
                if o + W == TW.track_hops(hops[p], W):
                    finished.add(track[b])
        cur = TW.next_cursor(cur, hops, W, seed)
    for p, s in enumerate(seen):
        assert np.all(s == 1), (p, hops[p], np.unique(s))
