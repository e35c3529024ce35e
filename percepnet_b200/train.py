"""Train the gain network on the GPU: rnn_train.py's loop on a PNB_TRAIN_NETWORK engine.

  python -m percepnet_b200.train --list files.txt --window 500 --batch 10 --steps N --lr 1e-4 --seed 0
                                 [--init model.pnbw] --out model.pnbw [--checkpoint ck.npz]
                                 [--dev-list dev.txt --eval-every K]

Record files (138 float32 per frame, eval_records.read_records) are cut into --window-frame windows
(eval_records.window_plan; the last window of a file may be shorter and counts only its own frames).  Every epoch the
windows are shuffled with a permutation seeded by (--seed, epoch), and each step takes the next --batch of them: one
gradient call (rnn_train.py's CustomLoss on exact activations, every window from zero state) and one Adam step with
torch.optim.Adam's defaults.  Each step logs the three loss terms as eval_records.loss_terms reports them.  With
--dev-list, every --eval-every steps the dev files are scored with eval_records.score on the deployed fp32 arithmetic
(the reference's tansig tables).  The initial weights are weights.synth_state_dict(--seed), torch's default init
bounds, or --init.  --out receives a PNBW blob; --checkpoint an npz of the weights, Adam's m and v and the step, from
which --checkpoint resumes when the file exists.  There is no CPU path.
"""
from __future__ import annotations

import argparse
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


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--list", required=True, help="text file, one training record file per line")
    ap.add_argument("--window", type=int, default=500, help="frames per window (rnn_train.py: 500)")
    ap.add_argument("--batch", type=int, default=10, help="windows per step (rnn_train.py: 10)")
    ap.add_argument("--steps", type=int, required=True)
    ap.add_argument("--lr", type=float, default=1e-4)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--init", help="initial weights (PNBW blob); default synth_state_dict(--seed)")
    ap.add_argument("--out", required=True, help="PNBW blob of the trained weights")
    ap.add_argument("--checkpoint", help="npz of weights, m, v and step; resumed from when it exists")
    ap.add_argument("--dev-list", help="text file of dev record files, scored on the deployed arithmetic")
    ap.add_argument("--eval-every", type=int, default=0)
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args(argv)
    if a.window < 1 or a.batch < 1 or a.steps < 0:
        ap.error("--window and --batch must be >= 1, --steps >= 0")
    if not (a.lr >= 0 and np.isfinite(a.lr)):
        ap.error("--lr must be a finite number >= 0")
    if a.dev_list and a.eval_every < 1:
        ap.error("--dev-list needs --eval-every >= 1")
    return a


def main(argv=None) -> int:
    a = parse_args(argv)
    from . import api
    from .weights import PackedModel, pack_state_dict, synth_state_dict
    x, frames = windows_of(read_list(a.list), a.window)
    if x.shape[0] < a.batch:
        sys.stderr.write(f"{x.shape[0]} windows, fewer than --batch {a.batch}\n")
        return 2
    model = api.BlobModel(a.init) if a.init else pack_state_dict(synth_state_dict(a.seed))
    eng = api.Engine(a.batch, a.window, model, api.TRAIN_NETWORK, device=a.device)
    if a.init:
        model.free()
    step = 0
    if a.checkpoint and os.path.exists(a.checkpoint):
        ck = np.load(a.checkpoint)
        for k in ("weights", "m", "v"):
            eng.train_import(k, ck[k])
        step = int(ck["step"])
        print(f"resumed {a.checkpoint} at step {step}")
    dev = [read_records(p) for p in read_list(a.dev_list)] if a.dev_list else None
    it = batches(x.shape[0], a.batch, a.seed)
    for _ in range(step):  # the same windows as an uninterrupted run
        next(it)
    try:
        while step < a.steps:
            epoch, idx = next(it)
            t = loss_terms(eng.train_grad(x[idx], frames[idx]).sum(0))
            step += 1
            eng.train_adam(a.lr, step)
            print(f"[{epoch + 1}, {step:6d}] loss {t['total']:.6f}  g2 {t['g2']:.6f}  g4 {t['g4']:.6f}  r2 {t['r2']:.6f}")
            if dev is not None and step % a.eval_every == 0:
                pm = PackedModel.from_flat(eng.train_export("weights"))
                sums, _ = score(dev, pm, api.NN_FP32, 4096, 100, a.device)
                d = loss_terms(sums.sum(0))
                print(f"  dev (deployed arithmetic) loss {d['total']:.6f}  g2 {d['g2']:.6f}  g4 {d['g4']:.6f}  r2 {d['r2']:.6f}")
        eng.wait()
        w = eng.train_export("weights")
        PackedModel.from_flat(w).save_blob(a.out)
        if a.checkpoint:
            np.savez(a.checkpoint, weights=w, m=eng.train_export("m"), v=eng.train_export("v"), step=np.int64(step))
    except api.PnbError as ex:
        sys.stderr.write(f"{ex}\n")
        return 2
    finally:
        eng.close()
    print(f"wrote {a.out} after {step} steps")
    return 0


if __name__ == "__main__":
    sys.exit(main())
