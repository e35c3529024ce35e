"""The training CLI under a torchrun-style launch: two ranks (torch.multiprocessing.spawn) train one model.  Two ranks of
one micro-batch each end at the bits of one process with --accum 2 (the same --out blob, the same printed losses, the
same weights on both ranks); two ranks of two micro-batches are within rounding of one process of four.  On one
device the ranks exchange over gloo; with two devices visible the same runs go over NCCL."""
import os
import re
import socket

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

from percepnet_b200 import train

pytestmark = pytest.mark.gpu

WINDOW, BATCH, SEED, STEPS = 20, 3, 5, 3


def write_files(tmp_path):
    """Seven record files (moderate scale) of 15 windows at --window 20, five of them shorter than 20 frames."""
    rng = np.random.RandomState(50)
    paths = []
    for k, n in enumerate((45, 30, 17, 60, 41, 20, 33)):
        rec = rng.rand(n, 138).astype(np.float32)
        rec[:, :68] *= np.float32(0.05)
        p = tmp_path / f"r{k}.f32"
        rec.astype("<f4").tofile(p)
        paths.append(str(p))
    lst = tmp_path / "list.txt"
    lst.write_text("\n".join(paths) + "\n")
    return str(lst)


def argv(lst, out, accum):
    return ["--list", lst, "--window", str(WINDOW), "--batch", str(BATCH), "--accum", str(accum), "--steps", str(STEPS),
            "--lr", "1e-3", "--seed", str(SEED), "--out", out]


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    p = s.getsockname()[1]
    s.close()
    return p


def _rank(rank, world, port, shared, lst, out, accum, out_dir):
    """One rank of a launch: torchrun's environment, the CLI's stdout in a file, and its final weights saved from the
    engine as it closes."""
    os.environ.update(WORLD_SIZE=str(world), RANK=str(rank), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1",
                      MASTER_PORT=str(port))
    if shared:
        os.environ["CUDA_VISIBLE_DEVICES"] = "0"
    import contextlib
    from percepnet_b200 import api
    from percepnet_b200 import train as T
    close = api.Engine.close

    def close_saving(self):
        if getattr(self, "h", None) and self.flags & api.TRAIN_NETWORK:
            np.save(os.path.join(out_dir, f"w{rank}.npy"), self.train_export("weights"))
        close(self)
    api.Engine.close = close_saving
    with open(os.path.join(out_dir, f"log{rank}.txt"), "w") as f, contextlib.redirect_stdout(f):
        rc = T.main(argv(lst, out, accum))
    with open(os.path.join(out_dir, f"rc{rank}.txt"), "w") as f:
        f.write(str(rc))


def launch(tmp_path, capsys, tag, lst, accum, shared):
    d = tmp_path / tag
    d.mkdir()
    out = str(d / "out.pnbw")
    mp.spawn(_rank, args=(2, _free_port(), shared, lst, out, accum, str(d)), nprocs=2, join=True)
    rcs = [int((d / f"rc{r}.txt").read_text()) for r in range(2)]
    logs = [(d / f"log{r}.txt").read_text() for r in range(2)]
    w = [np.load(d / f"w{r}.npy") for r in range(2)]
    with capsys.disabled():
        print(f"\n{tag}: return codes {rcs}\n{logs[0]}")
    assert rcs == [0, 0]
    assert logs[1] == "", "only rank 0 prints"
    assert np.array_equal(w[0].view(np.int32), w[1].view(np.int32)), "the ranks' weights differ"
    with open(out, "rb") as f:
        return f.read(), logs[0], w[0]


def single(tmp_path, capsys, tag, lst, accum):
    out = str(tmp_path / f"{tag}.pnbw")
    capsys.readouterr()
    assert train.main(argv(lst, out, accum)) == 0
    log = capsys.readouterr().out
    with capsys.disabled():
        print(f"\none process, --accum {accum}:\n{log}")
    with open(out, "rb") as f:
        return f.read(), log


losses = lambda log: re.findall(r"\] loss .*", log)


def blob_weights(raw: bytes) -> np.ndarray:
    """The flat float32 weights of a PNBW blob (magic, then each array as a uint64 count and its floats)."""
    parts, at = [], 8
    while at < len(raw):
        n = int(np.frombuffer(raw, "<u8", 1, at)[0])
        parts.append(np.frombuffer(raw, "<f4", n, at + 8))
        at += 8 + 4 * n
    return np.concatenate(parts)


def test_two_ranks_on_one_device_over_gloo(tmp_path, capsys):
    run_both(tmp_path, capsys, shared=True, tag="gloo")


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="NCCL between ranks needs two visible devices")
def test_two_ranks_on_two_devices_over_nccl(tmp_path, capsys):
    run_both(tmp_path, capsys, shared=False, tag="nccl")


def run_both(tmp_path, capsys, shared, tag):
    lst = write_files(tmp_path)
    # W = 2, K = 1 against one process, K = 2: bit for bit
    blob1, log1, w1 = launch(tmp_path, capsys, f"{tag}_w2k1", lst, 1, shared)
    blob_ref, log_ref = single(tmp_path, capsys, f"{tag}_w1k2", lst, 2)
    assert len(losses(log_ref)) == STEPS
    assert losses(log1) == losses(log_ref), "printed losses differ"
    assert blob1 == blob_ref, "--out differs from one process with --accum 2"
    # W = 2, K = 2 against one process, K = 4: the same windows, sums in another order
    blob2, log2, w2 = launch(tmp_path, capsys, f"{tag}_w2k2", lst, 2, shared)
    blob4, log4 = single(tmp_path, capsys, f"{tag}_w1k4", lst, 4)
    w4 = blob_weights(blob4)
    assert np.array_equal(blob_weights(blob2).view(np.int32), w2.view(np.int32))
    rel = np.linalg.norm(w2.astype(np.float64) - w4) / np.linalg.norm(w4.astype(np.float64))
    moved = np.linalg.norm(w4.astype(np.float64) - blob_weights(blob_ref)) / np.linalg.norm(w4.astype(np.float64))
    with capsys.disabled():
        print(f"W = 2, K = 2 against W = 1, K = 4: weights {rel:.2e} apart (relative norm); {np.count_nonzero(w2 != w4)} "
              f"of {w4.size} differ; a different batch moves them {moved:.2e}")
    assert losses(log2)[0] == losses(log4)[0], "the first step's loss is the loss of the same windows"
    assert rel <= 1e-6
