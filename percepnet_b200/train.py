"""Train the gain network on the GPU: rnn_train.py's loop on a PNB_TRAIN_NETWORK engine.

  python -m percepnet_b200.train --list files.txt --window 500 --batch 10 --steps N --lr 1e-4 --seed 0
                                 [--accum K] [--init model.pnbw] --out model.pnbw [--checkpoint ck.npz]
                                 [--dev-list dev.txt --eval-every K]
  torchrun --nproc-per-node W -m percepnet_b200.train ...   (the same arguments: W ranks train one model)

Record files (138 float32 per frame, eval_records.read_records) are cut into --window-frame windows
(eval_records.window_plan; the last window of a file may be shorter and counts only its own frames).  Every epoch the
windows are shuffled with a permutation seeded by (--seed, epoch), and each step takes the next W x K x --batch of them
(W ranks, K = --accum micro-batches per rank), cut into slices of --batch: rank r's micro-batch j is slice r K + j.
Each micro-batch is one gradient call (rnn_train.py's CustomLoss on exact activations, every window from zero state)
accumulated on the engine in float64, weighted by the hops it counted; with several ranks the accumulators are summed
by an all-reduce; then one Adam step with torch.optim.Adam's defaults on the whole batch's gradient.  With W = K = 1
that is exactly one gradient call and one Adam step per --batch windows.  Each step logs the three loss terms of the
whole batch as eval_records.loss_terms reports them (every rank's per-window sums, added in slice order).  With
--dev-list, every --eval-every steps the dev files are scored with eval_records.score on the deployed fp32 arithmetic
(the reference's tansig tables).  The initial weights are weights.synth_state_dict(--seed), torch's default init
bounds, or --init.  --out receives a PNBW blob; --checkpoint an npz of the weights, Adam's m and v and the step, from
which --checkpoint resumes when the file exists.  There is no CPU path.

Under torchrun (WORLD_SIZE > 1) each rank trains on the device LOCAL_RANK (modulo the visible devices; --device is
ignored).  The accumulators are summed over NCCL on device buffers when every rank has a device of its own, and over
gloo on host copies when ranks share a device.  Rank 0 alone prints, scores the dev files and writes --out and
--checkpoint; every rank resumes from --checkpoint.  The ranks compare a digest of their weights at the start and
before writing, and stop on a mismatch.
"""
from __future__ import annotations

import argparse
import hashlib
import os
import sys

import numpy as np

from .eval_records import loss_terms, read_records, score, window_plan

RECORD = 138


def read_list(path: str):
    with open(path) as f:
        return [line.strip() for line in f if line.strip()]


def windows_of(files, window: int):
    """[n, window, 138] float32 windows (zero-padded) and their frame counts."""
    recs = [read_records(p) for p in files]
    plan = window_plan([r.shape[0] for r in recs], window)
    out = np.zeros((len(plan), window, RECORD), np.float32)
    frames = np.empty(len(plan), np.int32)
    for i, (k, t0, n) in enumerate(plan):
        out[i, :n] = recs[k][t0:t0 + n]
        frames[i] = n
    return out, frames


def batches(n_windows: int, batch: int, seed: int):
    """Endless (epoch, indices) of `batch` windows: each epoch a seeded permutation, cut into full batches."""
    epoch = 0
    while True:
        perm = np.random.default_rng([seed, epoch]).permutation(n_windows)
        for b0 in range(0, n_windows - batch + 1, batch):
            yield epoch, perm[b0:b0 + batch]
        epoch += 1


def micro_batches(idx, batch: int, accum: int, rank: int):
    """Rank `rank`'s `accum` micro-batches of one step's windows idx (world x accum x batch of them, from batches()):
    slices rank x accum + j of `batch` windows each, j = 0 .. accum - 1."""
    return [idx[(rank * accum + j) * batch:(rank * accum + j + 1) * batch] for j in range(accum)]


def exchange_backend(placements) -> str:
    """The all-reduce of the accumulators: "nccl" when every rank has a device of its own (placements: one
    (host, device id) per rank), "gloo" on host copies when some ranks share a device."""
    return "nccl" if len(set(placements)) == len(placements) else "gloo"


def digest(a: np.ndarray) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


class Ranks:
    """The ranks of a run: one process, or a torchrun launch (WORLD_SIZE > 1) with a gloo process group for the host
    exchanges and, when every rank has a device of its own, an NCCL group for the accumulators."""

    def __init__(self, device: int):
        self.world = int(os.environ.get("WORLD_SIZE", "1"))
        self.rank, self.device, self.backend = 0, device, None
        if self.world <= 1:
            self.world = 1
            return
        import socket

        import torch
        import torch.distributed as dist
        self.dist, self.torch = dist, torch
        n_dev = torch.cuda.device_count()
        if n_dev < 1:
            raise RuntimeError("no CUDA device visible")
        self.device = int(os.environ.get("LOCAL_RANK", "0")) % n_dev
        dist.init_process_group("gloo")   # env://: MASTER_ADDR, MASTER_PORT, RANK, WORLD_SIZE
        self.rank = dist.get_rank()
        places = [None] * self.world
        dist.all_gather_object(places, (socket.gethostname(), str(torch.cuda.get_device_properties(self.device).uuid)))
        self.backend = exchange_backend(places)
        if self.backend == "nccl":
            torch.cuda.set_device(self.device)
            self.nccl = dist.new_group(backend="nccl")
            self.buf = None

    def sum_accumulators(self, eng):
        """Every rank's accumulator replaced by the sum over ranks (nothing with one process)."""
        if self.world == 1:
            return
        if self.backend == "gloo":
            a = eng.train_export("accum")
            self.dist.all_reduce(self.torch.from_numpy(a))
            eng.train_import("accum", a)
            return
        from .weights import N_PARAMS
        if self.buf is None:
            self.buf = self.torch.empty(N_PARAMS + 1, dtype=self.torch.float64, device=f"cuda:{self.device}")
        nbytes = self.buf.numel() * 8
        eng.train_export_ptr("accum", self.buf.data_ptr(), nbytes)
        self.dist.all_reduce(self.buf, group=self.nccl)
        self.torch.cuda.current_stream(self.device).synchronize()
        eng.train_import_ptr("accum", self.buf.data_ptr(), nbytes)

    def gather_rows(self, rows: np.ndarray) -> np.ndarray:
        """Every rank's rows (the same shape on each), concatenated in rank order."""
        if self.world == 1:
            return rows
        parts = [self.torch.empty(rows.shape, dtype=self.torch.float64) for _ in range(self.world)]
        self.dist.all_gather(parts, self.torch.from_numpy(np.ascontiguousarray(rows, np.float64)))
        return np.concatenate([p.numpy() for p in parts])

    def check_same(self, w: np.ndarray, when: str):
        """Raises when the ranks' weights differ."""
        if self.world == 1:
            return
        got = [None] * self.world
        self.dist.all_gather_object(got, digest(w))
        if len(set(got)) != 1:
            raise RuntimeError(f"ranks hold different weights {when}: digests {[g[:12] for g in got]}")

    def close(self):
        if self.world > 1 and self.dist.is_initialized():
            self.dist.destroy_process_group()


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--list", required=True, help="text file, one training record file per line")
    ap.add_argument("--window", type=int, default=500, help="frames per window (rnn_train.py: 500)")
    ap.add_argument("--batch", type=int, default=10, help="windows per gradient call (rnn_train.py: 10)")
    ap.add_argument("--accum", type=int, default=1, help="micro-batches of --batch windows per rank and step")
    ap.add_argument("--steps", type=int, required=True)
    ap.add_argument("--lr", type=float, default=1e-4)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--init", help="initial weights (PNBW blob); default synth_state_dict(--seed)")
    ap.add_argument("--out", required=True, help="PNBW blob of the trained weights")
    ap.add_argument("--checkpoint", help="npz of weights, m, v and step; resumed from when it exists")
    ap.add_argument("--dev-list", help="text file of dev record files, scored on the deployed arithmetic")
    ap.add_argument("--eval-every", type=int, default=0)
    ap.add_argument("--device", type=int, default=0, help="the device of a single-process run")
    a = ap.parse_args(argv)
    if a.window < 1 or a.batch < 1 or a.steps < 0:
        ap.error("--window and --batch must be >= 1, --steps >= 0")
    if a.accum < 1:
        ap.error("--accum must be >= 1")
    if not (a.lr >= 0 and np.isfinite(a.lr)):
        ap.error("--lr must be a finite number >= 0")
    if a.dev_list and a.eval_every < 1:
        ap.error("--dev-list needs --eval-every >= 1")
    return a


def too_few_windows(n_windows: int, batch: int, accum: int, world: int):
    """The refusal of a run whose step needs more windows than there are, or None."""
    need = world * accum * batch
    if n_windows >= need:
        return None
    if need == batch:
        return f"{n_windows} windows, fewer than --batch {batch}"
    return f"{n_windows} windows, fewer than one step's {need} (world {world} x --accum {accum} x --batch {batch})"


def main(argv=None) -> int:
    a = parse_args(argv)
    from . import api
    from .weights import PackedModel, pack_state_dict, synth_state_dict
    x, frames = windows_of(read_list(a.list), a.window)
    world = max(1, int(os.environ.get("WORLD_SIZE", "1")))
    refusal = too_few_windows(x.shape[0], a.batch, a.accum, world)
    if refusal:
        sys.stderr.write(refusal + "\n")
        return 2
    ranks = Ranks(a.device)
    lead = ranks.rank == 0
    say = print if lead else (lambda *_, **__: None)
    model = api.BlobModel(a.init) if a.init else pack_state_dict(synth_state_dict(a.seed))
    eng = api.Engine(a.batch, a.window, model, api.TRAIN_NETWORK, device=ranks.device)
    if a.init:
        model.free()
    step = 0
    if a.checkpoint and os.path.exists(a.checkpoint):
        ck = np.load(a.checkpoint)
        for k in ("weights", "m", "v"):
            eng.train_import(k, ck[k])
        step = int(ck["step"])
        say(f"resumed {a.checkpoint} at step {step}")
    dev = [read_records(p) for p in read_list(a.dev_list)] if a.dev_list and lead else None
    it = batches(x.shape[0], world * a.accum * a.batch, a.seed)
    for _ in range(step):  # the same windows as an uninterrupted run
        next(it)
    try:
        ranks.check_same(eng.train_export("weights"), "at the start")
        while step < a.steps:
            epoch, idx = next(it)
            sums = []
            for part in micro_batches(idx, a.batch, a.accum, ranks.rank):
                sums.append(eng.train_grad(x[part], frames[part]))
                eng.train_accumulate()
            ranks.sum_accumulators(eng)
            eng.train_finish()
            t = loss_terms(ranks.gather_rows(np.concatenate(sums)).sum(0))
            step += 1
            eng.train_adam(a.lr, step)
            say(f"[{epoch + 1}, {step:6d}] loss {t['total']:.6f}  g2 {t['g2']:.6f}  g4 {t['g4']:.6f}  r2 {t['r2']:.6f}")
            if dev is not None and step % a.eval_every == 0:
                pm = PackedModel.from_flat(eng.train_export("weights"))
                dsums, _ = score(dev, pm, api.NN_FP32, 4096, 100, ranks.device)
                d = loss_terms(dsums.sum(0))
                say(f"  dev (deployed arithmetic) loss {d['total']:.6f}  g2 {d['g2']:.6f}  g4 {d['g4']:.6f}  r2 {d['r2']:.6f}")
        eng.wait()
        w = eng.train_export("weights")
        ranks.check_same(w, "before writing")
        if lead:
            PackedModel.from_flat(w).save_blob(a.out)
            if a.checkpoint:
                np.savez(a.checkpoint, weights=w, m=eng.train_export("m"), v=eng.train_export("v"), step=np.int64(step))
    except (api.PnbError, RuntimeError) as ex:
        sys.stderr.write(f"{ex}\n")
        return 2
    finally:
        eng.close()
        ranks.close()
    say(f"wrote {a.out} after {step} steps")
    return 0


if __name__ == "__main__":
    sys.exit(main())
