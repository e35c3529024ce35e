"""Score a model on training records: the network as this engine runs it, on the records ``gen_features`` /
``train()`` write, with the loss ``rnn_train.py`` trains on.

  python -m percepnet_b200.eval_records --model model.pnbw rec1.f32 rec2.f32 ...
  python -m percepnet_b200.eval_records --model model.pnbw --list files.txt [--tensor [--conv-wide]] [--batch 4096]
                                        [--chunk 100] [--window N] [--pred-dir DIR]

Each record file (138 float32 per frame: Ey_lookahead[34] Ephaty[34] T pitchcorr g[34] r[34], denoise.cpp:761-773)
is one stream that starts from a fresh network state.  With ``--window N`` each file is instead cut into consecutive
N-frame windows (the last one may be shorter), and every window is a stream of its own that starts fresh: that is how
``rnn_train.py`` sees its data (``CppRawListDataset`` reshapes every file to 500-frame sequences, ``h5Dataset`` cuts
windows of 500), so ``--window 500`` on 500-frame files gives the loss a training run logs.  A file's sums are the sums
of its windows.  Streams are batched like ``gen_features.run_jobs``: sorted by length, ``--batch`` streams per engine,
the shorter ones zero-padded to the longest.  The padding is exact: the network is causal and the streams are
independent, so frames after a stream's end cannot change its earlier outputs, and they are left out of its loss.  A
batch is fed in calls of ``--chunk`` frames with the state carried between calls, on a network-only engine
(PNB_NETWORK_ONLY, which holds none of the signal path's buffers).

The network input is {30 * rec[0..67], rec[68], rec[69]}: the device scales the records exactly as ``create_features``
(denoise.cpp:487-496) and ``rnn_train.py``'s ``CppRawListDataset`` (rnn_train.py:44-48) do, so the model sees what the
deployed network sees.  ``utils/bin2h5.py`` -> ``h5Dataset`` does NOT apply the x30; a model trained through that path
saw unscaled band energies, and the reference is inconsistent with itself there.  This tool follows the deployed one.

For every file and over all files it prints the three terms of ``rnn_train.py``'s ``CustomLoss`` (rnn_train.py:153-176,
gamma = 0.5, C4 = 10; means over frames and bands) and their total:

  g2 = mean((g^0.5 - g_hat^0.5)^2)   g4 = C4 * mean((g^0.5 - g_hat^0.5)^4)   r2 = mean(((1-r)^0.5 - (1-r_hat)^0.5)^2)

The sums behind the means are reduced in float64 on the device from the predictions and the labels rec[70..137]
(pnb_score_records_host), so only four numbers per stream and call come back; the host adds them per file in float64,
in chunk order.  ``loss_sums`` is the same reduction in numpy, kept as the reference it is checked against.  "overall"
takes the same means over every frame of every file.  With ``--pred-dir`` the predictions of each file (frames x 68
float32: 34 g then 34 r) are fetched too and go to DIR/<file name>.pred.f32.  There is no CPU path.
"""
from __future__ import annotations

import argparse
import os
import sys

import numpy as np

RECORD = 138
GAMMA, C4 = 0.5, 10.0


def read_records(path: str) -> np.ndarray:
    """A record file as [frames, 138] float32."""
    raw = np.fromfile(path, dtype="<f4")
    if raw.size == 0 or raw.size % RECORD:
        raise ValueError(f"{path}: {raw.size} floats, not a positive multiple of {RECORD}")
    return raw.reshape(-1, RECORD).astype(np.float32, copy=False)


def plan_batches(lengths, batch: int):
    """Indices of the files in each batch: longest first (similar lengths share a batch), `batch` files at most."""
    order = sorted(range(len(lengths)), key=lambda k: -lengths[k])
    return [order[b0:b0 + batch] for b0 in range(0, len(order), batch)]


def pad_batch(recs) -> np.ndarray:
    """[len(recs), longest, 138] float32: each file's records, zeros after its end."""
    F = max(r.shape[0] for r in recs)
    out = np.zeros((len(recs), F, RECORD), np.float32)
    for k, r in enumerate(recs):
        out[k, :r.shape[0]] = r
    return out


def loss_sums(pred: np.ndarray, rec: np.ndarray) -> np.ndarray:
    """float64 sums over frames and bands of the three CustomLoss terms (before the means and the C4 factor), and the
    number of terms each sum has: [sum dg^2, sum dg^4, sum dr^2, count]."""
    p = np.asarray(pred, np.float64).reshape(-1, 68)
    y = np.asarray(rec, np.float64).reshape(-1, RECORD)[:, 70:]
    dg = y[:, :34] ** GAMMA - p[:, :34] ** GAMMA
    dr = (1 - y[:, 34:]) ** GAMMA - (1 - p[:, 34:]) ** GAMMA
    return np.array([np.sum(dg ** 2), np.sum(dg ** 4), np.sum(dr ** 2), dg.size], np.float64)


def loss_terms(sums: np.ndarray) -> dict:
    """CustomLoss from loss_sums (summed over any number of files): {g2, g4, r2, total}."""
    n = sums[3]
    t = {"g2": sums[0] / n, "g4": C4 * sums[1] / n, "r2": sums[2] / n}
    t["total"] = t["g2"] + t["g4"] + t["r2"]
    return t


def window_plan(lengths, window: int):
    """The streams of files of `lengths` frames: (file index, first frame, frames) in file order, then frame order.
    window 0: one stream per file; else consecutive `window`-frame pieces, the last one possibly shorter."""
    plan = []
    for k, n in enumerate(lengths):
        step = window if window > 0 else n
        plan += [(k, t0, min(step, n - t0)) for t0 in range(0, n, step)]
    return plan


def chunk_frames(lengths, t0: int, chunk: int) -> np.ndarray:
    """The frames of the call that starts at frame t0 which belong to each stream of `lengths` frames (int32)."""
    return np.clip(np.asarray(lengths, np.int64) - t0, 0, chunk).astype(np.int32)


def score(recs, model, flags: int, batch: int, chunk: int, device: int = 0, want_pred: bool = False):
    """Loss sums [len(recs), 4] float64 of every record array in `recs`, each from a fresh stream, and its g/r
    [frames, 68] float32 (None unless want_pred)."""
    from . import api
    sums = np.zeros((len(recs), 4), np.float64)
    preds = [None] * len(recs)
    for group in plan_batches([r.shape[0] for r in recs], batch):
        x = pad_batch([recs[k] for k in group])
        lengths = [recs[k].shape[0] for k in group]
        N, F = x.shape[0], x.shape[1]
        eng = api.Engine(N, min(chunk, F), model, flags | api.NETWORK_ONLY, device=device)
        parts = []
        try:
            for t0 in range(0, F, chunk):
                s, gr = eng.score_records(x[:, t0:min(F, t0 + chunk)], chunk_frames(lengths, t0, chunk), want_pred)
                sums[group] += s
                parts.append(gr)
        finally:
            eng.close()
        if want_pred:
            gr = np.concatenate(parts, axis=1)
            for i, k in enumerate(group):
                preds[k] = gr[i, :recs[k].shape[0]]
    return sums, preds


def parse_args(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("files", nargs="*", help="record files (138 float32 per frame)")
    ap.add_argument("--model", required=True, help="binary weight file (PackedModel.save_blob, PNBW0001)")
    ap.add_argument("--list", help="text file, one record file per line")
    ap.add_argument("--tensor", action="store_true", help="run the tensor-core network (PNB_NN_TENSOR) instead of fp32")
    ap.add_argument("--conv-wide", action="store_true", help="with --tensor: three bf16 terms in conv1 / conv2 (PNB_CONV_WIDE)")
    ap.add_argument("--batch", type=int, default=4096, help="files (streams) per engine")
    ap.add_argument("--chunk", type=int, default=100, help="frames per GPU call")
    ap.add_argument("--window", type=int, default=0,
                    help="cut each file into N-frame windows, each a fresh stream (0: whole files)")
    ap.add_argument("--pred-dir", help="write each file's predictions to DIR/<file name>.pred.f32")
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args(argv)
    if a.list:
        with open(a.list) as f:
            a.files += [line.strip() for line in f if line.strip()]
    if not a.files:
        ap.error("no record files given")
    if a.batch < 1 or a.chunk < 1:
        ap.error("--batch and --chunk must be >= 1")
    if a.window < 0:
        ap.error("--window must be >= 0")
    if a.conv_wide and not a.tensor:
        ap.error("--conv-wide applies to --tensor")
    return a


def engine_flags(a) -> int:
    from . import api
    return (api.NN_TENSOR | (api.CONV_WIDE if a.conv_wide else 0)) if a.tensor else api.NN_FP32


def main(argv=None) -> int:
    a = parse_args(argv)
    from . import api
    recs = [read_records(p) for p in a.files]
    plan = window_plan([r.shape[0] for r in recs], a.window)
    model = api.BlobModel(a.model)
    try:
        sums, preds = score([recs[k][t0:t0 + n] for k, t0, n in plan], model, engine_flags(a), a.batch, a.chunk,
                            a.device, bool(a.pred_dir))
    except api.PnbError as ex:
        sys.stderr.write(f"{ex}\n")
        return 2
    finally:
        model.free()
    file_sums = np.zeros((len(recs), 4), np.float64)
    for (k, _, _), s in zip(plan, sums):          # in window order
        file_sums[k] += s
    if a.pred_dir:
        os.makedirs(a.pred_dir, exist_ok=True)
        for k, path in enumerate(a.files):
            pred = np.concatenate([p for (j, _, _), p in zip(plan, preds) if j == k])
            pred.astype("<f4").tofile(os.path.join(a.pred_dir, os.path.basename(path) + ".pred.f32"))
    total = np.zeros(4, np.float64)
    print(f"{'file':<40} {'frames':>7} {'g2':>12} {'g4':>12} {'r2':>12} {'total':>12}")
    for path, rec, s in zip(a.files, recs, file_sums):
        total += s
        t = loss_terms(s)
        print(f"{path:<40} {rec.shape[0]:>7} {t['g2']:12.6e} {t['g4']:12.6e} {t['r2']:12.6e} {t['total']:12.6e}")
    t = loss_terms(total)
    print(f"{'overall':<40} {sum(r.shape[0] for r in recs):>7} {t['g2']:12.6e} {t['g4']:12.6e} {t['r2']:12.6e} "
          f"{t['total']:12.6e}")
    return 0


if __name__ == "__main__":
    sys.exit(main())
