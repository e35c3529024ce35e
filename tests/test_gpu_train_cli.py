"""The training CLI (python -m percepnet_b200.train) end to end on the GPU: a run resumed from its --checkpoint
trains on the same windows and ends at the same bits as an uninterrupted run, and the loss it prints is the trainer's
loss of its first batch."""
import re

import numpy as np
import pytest

from percepnet_b200 import api, train
from percepnet_b200.eval_records import loss_terms
from percepnet_b200.weights import pack_state_dict, synth_state_dict

pytestmark = pytest.mark.gpu

WINDOW, BATCH, SEED = 20, 3, 4


def write_files(tmp_path):
    """Three record files of 45, 30 and 17 frames (moderate scale): six windows, three of them shorter than 20."""
    rng = np.random.RandomState(40)
    paths = []
    for k, n in enumerate((45, 30, 17)):
        rec = rng.rand(n, 138).astype(np.float32)
        rec[:, :68] *= np.float32(0.05)
        p = tmp_path / f"r{k}.f32"
        rec.astype("<f4").tofile(p)
        paths.append(str(p))
    lst = tmp_path / "list.txt"
    lst.write_text("\n".join(paths) + "\n")
    return str(lst), paths


def run(capsys, lst, out, steps, checkpoint=None):
    argv = ["--list", lst, "--window", str(WINDOW), "--batch", str(BATCH), "--steps", str(steps), "--lr", "1e-3",
            "--seed", str(SEED), "--out", out]
    if checkpoint:
        argv += ["--checkpoint", checkpoint]
    assert train.main(argv) == 0
    return capsys.readouterr().out


def test_resumed_run_equals_uninterrupted_run(tmp_path, capsys):
    lst, paths = write_files(tmp_path)
    x, frames = train.windows_of(paths, WINDOW)
    assert x.shape[0] == 6 and sorted(frames.tolist()) == [5, 10, 17, 20, 20, 20]
    full, part = str(tmp_path / "full.pnbw"), str(tmp_path / "part.pnbw")
    ck_full, ck = str(tmp_path / "full.npz"), str(tmp_path / "ck.npz")
    log_full = run(capsys, lst, full, 6, ck_full)
    log_a = run(capsys, lst, part, 3, ck)
    log_b = run(capsys, lst, part, 6, ck)
    print(log_full, log_a, log_b, sep="\n")
    assert "resumed" in log_b and "at step 3" in log_b
    losses = lambda log: re.findall(r"\] loss (\S+)", log)
    assert len(losses(log_full)) == 6 and losses(log_a) + losses(log_b) == losses(log_full)
    with open(full, "rb") as f1, open(part, "rb") as f2:
        assert f1.read() == f2.read()
    a, b = np.load(ck_full), np.load(ck)
    for k in ("weights", "m", "v"):
        assert np.array_equal(a[k].view(np.int32), b[k].view(np.int32)), k
    assert int(a["step"]) == int(b["step"]) == 6
    assert not np.array_equal(a["weights"], pack_state_dict(synth_state_dict(SEED)).flat())

    # the first printed loss is the trainer's loss of the first batch, from the initial weights
    _, idx = next(train.batches(x.shape[0], BATCH, SEED))
    eng = api.Engine(BATCH, WINDOW, pack_state_dict(synth_state_dict(SEED)), api.TRAIN_NETWORK)
    first = loss_terms(eng.train_grad(x[idx], frames[idx]).sum(0))["total"]
    eng.close()
    print(f"first batch {idx.tolist()}: direct train_grad loss {first:.9f}")
    assert losses(log_full)[0] == f"{first:.6f}"
