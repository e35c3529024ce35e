"""Train the gain network on the enhanced waveform: clean/noisy PCM pairs through the bit-exact analysis, the network
and a synthesis differentiable in g/r (torch_signal.SignalPath around torch_module.PercepNet), in consecutive windows.

  python -m percepnet_b200.train_wave --list pairs.txt --window 500 --batch 10 --steps N --lr 1e-4 --seed 0
                                      [--postfilter] [--init model.pnbw] --out model.pnbw [--checkpoint ck.npz]
                                      [--dev-list dev_pairs.txt --eval-every K] [--device 0]

Each line of --list and --dev-list is "<clean.pcm> <noisy.pcm>": raw 48 kHz int16 files, the pair gen_features reads.
A pair of n = samples // 480 hops becomes a track of L = ceil((n + 6) / W) * W hops (W = --window): its noisy PCM, six
hops of zeros that flush the output's lag (torch_signal.LATENCY_FRAMES), then zeros up to a whole number of windows.
Output sample j of a track is compared with clean sample j - 2880 for 2880 <= j < n * 480 + 2880; every other sample
is left out of the loss.  As W > 6, every window of a track counts at least one sample.

Schedule: --batch rows B.  Epoch e visits the pairs in np.random.default_rng([seed, e]).permutation(n_pairs); a row
whose track ends takes the next pair of that order, which runs on into the next epoch, so no row is ever idle.  Each
step advances every row by one window.  A row that starts a track starts from fresh signal streams and zero network
state; otherwise both carry over from its previous window, the network state detached (truncated backpropagation
through time along the file; the overlap-add memory that crosses a window's edge takes no gradient either).  A step is
analysis, PercepNet, synthesis, the loss sum(|out - target| over counted samples) / (32768 * count) in float32 on the
device, backward and one torch.optim.Adam step (torch's defaults, --lr).  Each step logs its loss and counted samples.

The initial weights are weights.synth_state_dict(--seed) or --init.  --postfilter turns on the envelope post-filter in
training and dev scoring alike.  With --dev-list, every --eval-every steps the dev pairs are enhanced in the deployed
arithmetic (an fp32 PCM engine, the reference's tansig tables) from fresh streams, with the tracks and targets above,
and the masked L1 and the SNR 10 log10(sum c^2 / sum (y - c)^2) over the whole dev set are printed, summed in float64
on the device; the noisy input's SNR is printed once as the baseline.  --out receives a PNBW blob.  --checkpoint is an
npz of the weights, Adam's moments and step, the schedule cursor and each row's network and signal state, written at
the end of the run and resumed from when it exists: a resumed run continues bit for bit.  There is no CPU path.
"""
from __future__ import annotations

import argparse
import functools
import os
import sys
from typing import NamedTuple

import numpy as np

from .torch_signal import FRAME, LATENCY_FRAMES as LAG_HOPS, LATENCY_SAMPLES as LAG

DEV_ROWS = 256                # dev pairs per enhancement engine


# ---- data -------------------------------------------------------------------------------------------------------------
def read_pairs(path: str):
    """The (clean, noisy) paths of a pair list, one "<clean> <noisy>" per line."""
    pairs = []
    with open(path) as f:
        for k, line in enumerate(f, 1):
            p = line.split()
            if not p:
                continue
            if len(p) != 2:
                raise ValueError(f"{path}:{k}: a line is '<clean.pcm> <noisy.pcm>', not {line.strip()!r}")
            pairs.append((p[0], p[1]))
    return pairs


def pair_hops(clean: str, noisy: str) -> int:
    """The whole hops of a pair; raises ValueError when its files differ in hops or hold less than one."""
    n_c, n_n = os.path.getsize(clean) // (2 * FRAME), os.path.getsize(noisy) // (2 * FRAME)
    if n_c != n_n:
        raise ValueError(f"{clean} has {n_c} hops and {noisy} {n_n}: a pair's files must have as many")
    if n_c < 1:
        raise ValueError(f"{clean}: shorter than one hop of {FRAME} samples")
    return n_c


def load_pair(clean: str, noisy: str, n: int):
    """The first n hops of both files as int16 arrays."""
    return (np.fromfile(clean, dtype="<i2", count=n * FRAME).astype(np.int16),
            np.fromfile(noisy, dtype="<i2", count=n * FRAME).astype(np.int16))


def track_hops(n: int, window: int) -> int:
    """L = ceil((n + 6) / W) * W: the hops of a pair of n hops with the lag flushed, in whole windows."""
    return -(-(n + LAG_HOPS) // window) * window


def window_of(clean: np.ndarray, noisy: np.ndarray, offset: int, window: int):
    """Hops [offset, offset + W) of a pair's track: (noisy input int16 [W*480], target int16 [W*480], lo, hi), where
    samples [lo, hi) of the window are counted and target[i] = clean[offset*480 + i - 2880] there (0 elsewhere)."""
    s0, s1 = offset * FRAME, (offset + window) * FRAME
    x = np.zeros(window * FRAME, np.int16)
    src = noisy[s0:s1]
    x[:src.size] = src
    lo, hi = max(s0, LAG), min(s1, clean.size + LAG)
    tgt = np.zeros(window * FRAME, np.int16)
    if hi > lo:
        tgt[lo - s0:hi - s0] = clean[lo - LAG:hi - LAG]
    else:
        lo = hi = s0
    return x, tgt, lo - s0, hi - s0


# ---- schedule: pure functions of (pair hops, B, W, seed, step) ----------------------------------------------------------
class Cursor(NamedTuple):
    """Where a run stands between steps: the next pair to take is position `pos` of epoch `epoch`'s order; row b is at
    hop `offset[b]` of pair `pair[b]`'s track (a multiple of W; 0: the row starts that track at the next step)."""
    epoch: int
    pos: int
    pair: np.ndarray
    offset: np.ndarray


@functools.lru_cache(maxsize=8)
def _order(n_pairs: int, seed: int, epoch: int) -> tuple:
    """The pairs in the order epoch `epoch` visits them."""
    return tuple(int(k) for k in np.random.default_rng([seed, epoch]).permutation(n_pairs))


def _take(epoch: int, pos: int, n_pairs: int, seed: int):
    if pos == n_pairs:
        epoch, pos = epoch + 1, 0
    return _order(n_pairs, seed, epoch)[pos], epoch, pos + 1


def first_cursor(n_pairs: int, batch: int, seed: int) -> Cursor:
    """Step 0: rows 0 .. B-1 take the first B pairs of epoch 0's order."""
    if batch > n_pairs:
        raise ValueError(f"{n_pairs} pairs, fewer than --batch {batch}")
    epoch, pos, pair = 0, 0, np.empty(batch, np.int64)
    for b in range(batch):
        pair[b], epoch, pos = _take(epoch, pos, n_pairs, seed)
    return Cursor(epoch, pos, pair, np.zeros(batch, np.int64))


def next_cursor(cur: Cursor, hops, window: int, seed: int) -> Cursor:
    """The cursor after one step: every row one window further; rows whose track ended take the next pairs of the
    order, in row order."""
    epoch, pos = cur.epoch, cur.pos
    pair, offset = cur.pair.copy(), cur.offset + window
    for b in range(len(pair)):
        if offset[b] == track_hops(hops[pair[b]], window):
            pair[b], epoch, pos = _take(epoch, pos, len(hops), seed)
            offset[b] = 0
    return Cursor(epoch, pos, pair, offset)


def cursor_at(hops, batch: int, window: int, seed: int, step: int) -> Cursor:
    """The cursor before step `step` (counted from 0) of a run on pairs of `hops` hops."""
    cur = first_cursor(len(hops), batch, seed)
    for _ in range(step):
        cur = next_cursor(cur, hops, window, seed)
    return cur


def step_inputs(data, cur: Cursor, window: int):
    """One step's host inputs from the pairs' (clean, noisy) int16 arrays: noisy windows int16 [B, W*480], targets int16
    [B, W*480], and each row's counted samples [lo, hi) (int64 [B] each)."""
    rows = [window_of(*data[p], o, window) for p, o in zip(cur.pair, cur.offset)]
    return (np.stack([r[0] for r in rows]), np.stack([r[1] for r in rows]),
            np.array([r[2] for r in rows], np.int64), np.array([r[3] for r in rows], np.int64))


# ---- device side ------------------------------------------------------------------------------------------------------
def masked_l1(out, target, lo, hi, count: int):
    """sum(|out - target| over samples [lo, hi) of each row) / (32768 * count), float32 on out's device."""
    import torch
    j = torch.arange(out.shape[1], device=out.device)
    mask = (j >= lo[:, None]) & (j < hi[:, None])
    return torch.where(mask, (out - target).abs(), 0).sum() / (32768.0 * count)


def score_dev(state_dict, data, window: int, postfilter: bool, device: int = 0):
    """The dev pairs' (clean, noisy) int16 arrays enhanced by an fp32 PCM engine with the weights of `state_dict`
    (numpy arrays by rnn_train.PercepNet's names), each from a fresh stream on its track: {"l1": masked L1 as the
    training loss takes it, "snr": 10 log10(sum c^2 / sum (y - c)^2) in dB, "count": counted samples}, summed in
    float64 on the device.  The enhanced PCM stays there."""
    import torch
    from . import api
    from .weights import pack_state_dict
    model = pack_state_dict(state_dict)
    flags = api.NN_FP32 | (api.POSTFILTER if postfilter else 0)
    dev = torch.device("cuda", device)
    sums = torch.zeros(3, dtype=torch.float64, device=dev)   # sum |y - c|, sum c^2, sum (y - c)^2
    count = 0
    tracks = [track_hops(c.size // FRAME, window) for c, _ in data]
    by_length = sorted(range(len(data)), key=lambda k: -tracks[k])
    with torch.cuda.device(dev):
        st = torch.cuda.current_stream().cuda_stream
        for g0 in range(0, len(by_length), DEV_ROWS):
            group = by_length[g0:g0 + DEV_ROWS]
            eng = api.Engine(len(group), window, model, flags, device)
            try:
                for t0 in range(0, tracks[group[0]], window):
                    n = sum(1 for k in group if tracks[k] > t0)   # the tracks (longest first) not yet ended
                    if n != eng.active:
                        eng.set_active(n, st)
                    x, tgt, lo, hi = step_inputs(data, Cursor(0, 0, np.array(group[:n]), np.full(n, t0)), window)
                    x = torch.from_numpy(x).to(dev).float()
                    y = torch.empty_like(x)
                    eng.process_device(x.data_ptr(), window * FRAME, y.data_ptr(), window * FRAME, window, 0, st)
                    j = torch.arange(window * FRAME, device=dev)
                    mask = (j >= torch.from_numpy(lo).to(dev)[:, None]) & (j < torch.from_numpy(hi).to(dev)[:, None])
                    c = torch.from_numpy(tgt).to(dev).double()
                    e = torch.where(mask, y.double() - c, 0)
                    sums += torch.stack([e.abs().sum(), (c * c).sum(), (e * e).sum()])
                    count += int((hi - lo).sum())
                eng.check(st)
            finally:
                eng.close()
    s = sums.cpu().numpy()
    return {"l1": s[0] / (32768.0 * count), "snr": 10 * np.log10(s[1] / s[2]), "count": count}


def noisy_snr(data) -> float:
    """The SNR of the noisy inputs against the clean ones, 10 log10(sum c^2 / sum (x - c)^2) over every dev sample."""
    num = sum(float(np.sum(c.astype(np.float64) ** 2)) for c, _ in data)
    den = sum(float(np.sum((x.astype(np.float64) - c) ** 2)) for c, x in data)
    return 10 * np.log10(num / den)


# ---- weights and checkpoints ------------------------------------------------------------------------------------------
def read_blob(path: str):
    """A PNBW blob (PackedModel.save_blob) as a PackedModel."""
    from .weights import PackedModel
    raw = open(path, "rb").read()
    if raw[:8] != PackedModel.BLOB_MAGIC:
        raise ValueError(f"{path}: not a PNBW blob (magic {raw[:8]!r})")
    parts, at = [], 8
    for _ in PackedModel.blob_keys():
        if at + 8 > len(raw):
            raise ValueError(f"{path}: truncated")
        n = int(np.frombuffer(raw, "<u8", 1, at)[0])
        if at + 8 + 4 * n > len(raw):
            raise ValueError(f"{path}: truncated")
        parts.append(np.frombuffer(raw, "<f4", n, at + 8))
        at += 8 + 4 * n
    if at != len(raw):
        raise ValueError(f"{path}: {len(raw) - at} bytes after the last array")
    return PackedModel.from_flat(np.concatenate(parts))


def _flat(tensors: dict) -> np.ndarray:
    """Tensors by parameter name as one blob-order float32 vector (weights.pack_state_dict's permutation)."""
    from .weights import pack_state_dict
    return pack_state_dict({k: v.detach().cpu().numpy() for k, v in tensors.items()}).flat()


def _unflat(v: np.ndarray) -> dict:
    from .weights import PackedModel, unpack_state_dict
    return unpack_state_dict(PackedModel.from_flat(v))


def save_checkpoint(path, net, opt, step: int, cur: Cursor, state, signal_state, window: int):
    """The run's whole state between two steps: weights, Adam's moments and step (blob order), the CLI step, the
    cursor, the network state rows [B, STATE_FLOATS] and the rows' signal state blobs [B, pnb_state_size()]."""
    from .weights import N_PARAMS
    params = dict(net.named_parameters())
    adam = [opt.state.get(p) for p in params.values()]
    adam_step = int(adam[0]["step"]) if adam[0] else 0
    zeros = np.zeros(N_PARAMS, np.float32)
    m = _flat({k: a["exp_avg"] for k, a in zip(params, adam)}) if adam_step else zeros
    v = _flat({k: a["exp_avg_sq"] for k, a in zip(params, adam)}) if adam_step else zeros
    np.savez(path, weights=_flat(params), exp_avg=m, exp_avg_sq=v, adam_step=np.int64(adam_step),
             step=np.int64(step), epoch=np.int64(cur.epoch), pos=np.int64(cur.pos), row_pair=cur.pair,
             row_offset=cur.offset, net_state=state.cpu().numpy(), signal_state=signal_state.cpu().numpy(),
             batch=np.int64(len(cur.pair)), window=np.int64(window))


def load_checkpoint(ck, net, opt):
    """Weights and Adam's state from a checkpoint into the module and the optimizer."""
    import torch
    params = dict(net.named_parameters())
    w = _unflat(ck["weights"])
    with torch.no_grad():
        for k, p in params.items():
            p.copy_(torch.from_numpy(w[k]))
    adam_step = int(ck["adam_step"])
    if adam_step:
        m, v = _unflat(ck["exp_avg"]), _unflat(ck["exp_avg_sq"])
        sd = opt.state_dict()
        sd["state"] = {i: {"step": torch.tensor(float(adam_step), dtype=torch.float32),
                           "exp_avg": torch.from_numpy(m[k]), "exp_avg_sq": torch.from_numpy(v[k])}
                       for i, k in enumerate(params)}
        opt.load_state_dict(sd)


# ---- the CLI ----------------------------------------------------------------------------------------------------------
def parse_args(argv=None):
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--list", required=True, help="text file, one '<clean.pcm> <noisy.pcm>' pair per line")
    ap.add_argument("--window", type=int, default=500, help="hops per window, > 6")
    ap.add_argument("--batch", type=int, default=10, help="rows: pairs trained side by side")
    ap.add_argument("--steps", type=int, required=True)
    ap.add_argument("--lr", type=float, default=1e-4)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--postfilter", action="store_true", help="the envelope post-filter on g (PNB_POSTFILTER)")
    ap.add_argument("--init", help="initial weights (PNBW blob); default synth_state_dict(--seed)")
    ap.add_argument("--out", required=True, help="PNBW blob of the trained weights")
    ap.add_argument("--checkpoint", help="npz of the run's whole state; resumed from when it exists")
    ap.add_argument("--dev-list", help="text file of dev pairs, scored in the deployed arithmetic")
    ap.add_argument("--eval-every", type=int, default=0)
    ap.add_argument("--device", type=int, default=0)
    a = ap.parse_args(argv)
    if a.window < 1 or a.batch < 1 or a.steps < 0:
        ap.error("--window and --batch must be >= 1, --steps >= 0")
    if a.window <= LAG_HOPS:
        ap.error(f"--window must be above {LAG_HOPS} hops, so that every window counts a sample of its track")
    if not (a.lr >= 0 and np.isfinite(a.lr)):
        ap.error("--lr must be a finite number >= 0")
    if a.dev_list and a.eval_every < 1:
        ap.error("--dev-list needs --eval-every >= 1")
    return a


def _refuse(msg: str) -> int:
    sys.stderr.write(msg + "\n")
    return 2


def main(argv=None) -> int:
    a = parse_args(argv)
    try:
        pairs = read_pairs(a.list)
        hops = [pair_hops(*p) for p in pairs]
        dev_pairs = read_pairs(a.dev_list) if a.dev_list else []
        dev_hops = [pair_hops(*p) for p in dev_pairs]
    except (OSError, ValueError) as ex:
        return _refuse(str(ex))
    if len(pairs) < a.batch:
        return _refuse(f"{len(pairs)} pairs, fewer than --batch {a.batch}")
    ck = None
    if a.checkpoint and os.path.exists(a.checkpoint):
        ck = np.load(a.checkpoint)
        if int(ck["batch"]) != a.batch or int(ck["window"]) != a.window:
            return _refuse(f"{a.checkpoint} was taken with --batch {int(ck['batch'])} --window {int(ck['window'])}")
    try:
        init = read_blob(a.init) if a.init else None
    except (OSError, ValueError) as ex:
        return _refuse(str(ex))

    import torch
    from . import api
    from .torch_module import STATE_FLOATS, PercepNet
    from .torch_signal import SignalPath
    from .weights import pack_state_dict, synth_state_dict, unpack_state_dict
    data = [load_pair(c, x, n) for (c, x), n in zip(pairs, hops)]
    dev_data = [load_pair(c, x, n) for (c, x), n in zip(dev_pairs, dev_hops)]
    dev = torch.device("cuda", a.device)
    torch.cuda.set_device(dev)
    B, W = a.batch, a.window
    net = PercepNet()
    sd = unpack_state_dict(init) if init is not None else synth_state_dict(a.seed)
    net.load_state_dict({k: torch.from_numpy(v) for k, v in sd.items()})
    net.to(dev)
    opt = torch.optim.Adam(net.parameters(), lr=a.lr)
    sp = SignalPath(B, W, postfilter=a.postfilter, device=dev)
    sp._engine(dev)   # created up front, not at the first analyze: a resumed run imports its rows' states before that
    step, cur = 0, first_cursor(len(pairs), B, a.seed)
    state = torch.zeros((B, STATE_FLOATS), dtype=torch.float32, device=dev)
    if ck is not None:
        load_checkpoint(ck, net, opt)
        step = int(ck["step"])
        cur = Cursor(int(ck["epoch"]), int(ck["pos"]), ck["row_pair"].astype(np.int64),
                     ck["row_offset"].astype(np.int64))
        state.copy_(torch.from_numpy(ck["net_state"]))
        sp.import_states(list(range(B)), torch.from_numpy(ck["signal_state"]).to(dev))
        print(f"resumed {a.checkpoint} at step {step}")
    if dev_data:
        print(f"  dev noisy input: SNR {noisy_snr(dev_data):.4f} dB")
    try:
        while step < a.steps:
            new = [b for b in range(B) if cur.offset[b] == 0]
            if new:
                sp.reset(new)
                state[new] = 0
            x, tgt, lo, hi = step_inputs(data, cur, W)
            count = int((hi - lo).sum())
            features, ops = sp.analyze(torch.from_numpy(x).to(dev).float())
            gr, state_out = net(features, state, return_state=True)
            out = sp.synthesize(gr, ops)
            loss = masked_l1(out, torch.from_numpy(tgt).to(dev).float(), torch.from_numpy(lo).to(dev),
                             torch.from_numpy(hi).to(dev), count)
            opt.zero_grad()
            loss.backward()
            opt.step()
            state = state_out.detach()
            step += 1
            print(f"[{cur.epoch + 1}, {step:6d}] loss {loss.item():.9g}  counted {count}", flush=True)
            cur = next_cursor(cur, hops, W, a.seed)
            if dev_data and step % a.eval_every == 0:
                d = score_dev({k: v.detach().cpu().numpy() for k, v in net.state_dict().items()}, dev_data, W,
                              a.postfilter, a.device)
                print(f"  dev (deployed arithmetic) L1 {d['l1']:.9g}  SNR {d['snr']:.4f} dB  counted {d['count']}")
        pack_state_dict({k: v.detach().cpu().numpy() for k, v in net.state_dict().items()}).save_blob(a.out)
        if a.checkpoint:
            save_checkpoint(a.checkpoint, net, opt, step, cur, state, sp.export_states(list(range(B))), W)
    except api.PnbError as ex:
        return _refuse(str(ex))
    finally:
        sp.close()
        net.close()
    print(f"wrote {a.out} after {step} steps")
    return 0


if __name__ == "__main__":
    sys.exit(main())
