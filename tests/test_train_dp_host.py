"""The host side of the training CLI's accumulation and ranks (percepnet_b200.train), on the CPU: the slice plan of a
step, its arguments and refusals, and the choice of the exchange's backend."""
import numpy as np
import pytest

from percepnet_b200 import train
from test_train_host import write_records


def test_one_rank_one_micro_batch_is_the_plain_batch():
    """World 1 and --accum 1: each step's one micro-batch is batches()'s batch, the windows of the plain loop."""
    plain, step = train.batches(11, 3, 5), train.batches(11, 1 * 1 * 3, 5)
    for _ in range(9):
        (e0, idx0), (e1, idx1) = next(plain), next(step)
        parts = train.micro_batches(idx1, 3, 1, 0)
        assert e0 == e1 and len(parts) == 1 and np.array_equal(parts[0], idx0)


@pytest.mark.parametrize("world,accum,batch", [(2, 1, 3), (1, 4, 2), (2, 3, 4), (4, 2, 1)])
def test_slices_partition_the_step(world, accum, batch):
    """Rank r's micro-batch j is slice r accum + j; over all ranks the slices are the step's windows, each once."""
    n = 3 * world * accum * batch + 1
    _, idx = next(train.batches(n, world * accum * batch, 7))
    got = []
    for r in range(world):
        parts = train.micro_batches(idx, batch, accum, r)
        assert len(parts) == accum and all(len(p) == batch for p in parts)
        for j, p in enumerate(parts):
            s = r * accum + j
            assert np.array_equal(p, idx[s * batch:(s + 1) * batch])
        got += [int(i) for p in parts for i in p]
    assert got == idx.tolist() and len(set(got)) == len(got)


def test_resume_skips_whole_steps():
    """A run resumed at step s takes the windows an uninterrupted run takes from step s + 1 on, for every rank."""
    world, accum, batch, n, s = 2, 2, 3, 29, 5
    full = train.batches(n, world * accum * batch, 3)
    steps = [next(full) for _ in range(9)]
    resumed = train.batches(n, world * accum * batch, 3)
    for _ in range(s):
        next(resumed)
    for k in range(s, 9):
        e, idx = next(resumed)
        assert e == steps[k][0]
        for r in range(world):
            for a, b in zip(train.micro_batches(idx, batch, accum, r), train.micro_batches(steps[k][1], batch, accum, r)):
                assert np.array_equal(a, b)


def test_accum_argument(capsys):
    base = ["--list", "l.txt", "--steps", "1", "--out", "o.pnbw"]
    assert train.parse_args(base).accum == 1
    assert train.parse_args(base + ["--accum", "4"]).accum == 4
    for bad in ("0", "-2"):
        with pytest.raises(SystemExit) as ex:
            train.parse_args(base + ["--accum", bad])
        assert ex.value.code == 2
        assert "--accum" in capsys.readouterr().err


@pytest.mark.parametrize("world,accum,batch,want", [
    (1, 1, 4, "3 windows, fewer than --batch 4"),
    (1, 2, 2, "3 windows, fewer than one step's 4 (world 1 x --accum 2 x --batch 2)"),
    (2, 1, 2, "3 windows, fewer than one step's 4 (world 2 x --accum 1 x --batch 2)"),
])
def test_more_windows_per_step_than_there_are(tmp_path, capsys, monkeypatch, world, accum, batch, want):
    """Three windows: a step of world x --accum x --batch > 3 windows returns 2 before any engine or process group
    exists."""
    for name, n in (("a.f32", 5), ("b.f32", 3)):
        write_records(tmp_path / name, n, 23)
    lst = tmp_path / "list.txt"
    lst.write_text(f"{tmp_path / 'a.f32'}\n{tmp_path / 'b.f32'}\n")
    out = tmp_path / "o.pnbw"
    monkeypatch.setenv("WORLD_SIZE", str(world))
    argv = ["--list", str(lst), "--window", "4", "--batch", str(batch), "--accum", str(accum), "--steps", "1",
            "--out", str(out)]
    assert train.main(argv) == 2
    assert want in capsys.readouterr().err
    assert not out.exists()
    assert train.too_few_windows(3, batch, accum, world) == want
    assert train.too_few_windows(world * accum * batch, batch, accum, world) is None


def test_exchange_backend():
    """NCCL when every rank has a device of its own (on one host or several), gloo as soon as two ranks share one."""
    assert train.exchange_backend([("a", "GPU-0"), ("a", "GPU-1")]) == "nccl"
    assert train.exchange_backend([("a", "GPU-0"), ("b", "GPU-0")]) == "nccl"
    assert train.exchange_backend([("a", "GPU-0"), ("a", "GPU-0")]) == "gloo"
    assert train.exchange_backend([("a", "GPU-0"), ("a", "GPU-1"), ("a", "GPU-1")]) == "gloo"
    assert train.exchange_backend([("a", "GPU-0")]) == "nccl"


def test_digest_tells_weights_apart():
    w = np.arange(10, dtype=np.float32)
    v = w.copy()
    v[3] = np.nextafter(v[3], np.float32(100))
    assert train.digest(w) == train.digest(w.copy()) and train.digest(w) != train.digest(v)
