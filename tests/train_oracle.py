"""rnn_train.py's model, loss and optimiser restated in torch, as the truth the GPU trainer is checked against.

Written from the layer list of rnn_train.PercepNet (rnn_train.py:105-145) and CustomLoss (rnn_train.py:153-176), not
copied; test_train_host.py pins it to the reference's own classes where the reference tree exists.  Parameter names and
shapes are the reference's state_dict, so weights.synth_state_dict / unpack_state_dict feed it directly.  A window may
end before the batch does (frames): its later hops are zeroed at the input (the network is causal, so that changes
nothing before them) and left out of the loss's means.
"""
from __future__ import annotations

import numpy as np
import torch
import torch.nn as nn

GAMMA, C4 = 0.5, 10.0


class Net(nn.Module):
    def __init__(self):
        super().__init__()
        self.fc = nn.Sequential(nn.Linear(70, 128), nn.ReLU())
        self.conv1 = nn.Sequential(nn.Conv1d(128, 512, 5, padding=4), nn.ReLU())   # four zero history taps
        self.conv2 = nn.Sequential(nn.Conv1d(512, 512, 3, padding=2), nn.Tanh())   # two
        self.gru1 = nn.GRU(512, 512, 1, batch_first=True)
        self.gru2 = nn.GRU(512, 512, 1, batch_first=True)
        self.gru3 = nn.GRU(512, 512, 1, batch_first=True)
        self.gru_gb = nn.GRU(512, 512, 1, batch_first=True)
        self.gru_rb = nn.GRU(1024, 128, 1, batch_first=True)
        self.fc_gb = nn.Sequential(nn.Linear(2560, 34), nn.Sigmoid())
        self.fc_rb = nn.Sequential(nn.Linear(128, 34), nn.Sigmoid())

    def forward(self, x):                                     # x [B, T, 70] -> [B, T, 68] = 34 g, 34 r
        y = self.fc(x).permute(0, 2, 1)
        y = self.conv1(y)[:, :, :-4]                          # causal: output t sees inputs t-4 .. t
        c = self.conv2(y)[:, :, :-2].permute(0, 2, 1)
        return self.head(c)

    def head(self, c):                                        # conv2's output c [B, T, 512] -> [B, T, 68]
        h1, _ = self.gru1(c)
        h2, _ = self.gru2(h1)
        h3, _ = self.gru3(h2)
        hg, _ = self.gru_gb(h3)
        g = self.fc_gb(torch.cat((c, h1, h2, h3, hg), -1))
        hr, _ = self.gru_rb(torch.cat((h3, c), -1))
        return torch.cat((g, self.fc_rb(hr)), -1)


def model(sd: dict, dtype=torch.float32, device="cpu") -> Net:
    m = Net().to(device=device, dtype=dtype)
    m.load_state_dict({k: torch.from_numpy(np.asarray(v, np.float32)) for k, v in sd.items()})
    return m


def features(rec: np.ndarray) -> np.ndarray:
    """The network input of records [B, T, 138]: {30 rec[0..67], rec[68], rec[69]} in float32 (CppRawListDataset)."""
    x = np.array(rec[..., :70], np.float32)
    x[..., :68] *= np.float32(30)
    return x


def loss(out, y, frames=None):
    """CustomLoss of out against the labels y ([B, T, 68]); with frames, the means run over each window's first
    frames[b] hops only."""
    gb_hat, rb_hat, gb, rb = out[..., :34], out[..., 34:], y[..., :34], y[..., 34:]
    # each term builds its own graph, as CustomLoss does: autograd then adds the same partial gradients in its order
    dg = torch.pow(torch.pow(gb, GAMMA) - torch.pow(gb_hat, GAMMA), 2)
    dg4 = torch.pow(torch.pow(gb, GAMMA) - torch.pow(gb_hat, GAMMA), 4)
    dr = torch.pow(torch.pow(1 - rb, GAMMA) - torch.pow(1 - rb_hat, GAMMA), 2)
    if frames is None:
        return torch.mean(dg) + C4 * torch.mean(dg4) + torch.mean(dr)
    T = out.shape[1]
    w = (torch.arange(T, device=out.device)[None, :] < torch.as_tensor(frames, device=out.device)[:, None]).to(out.dtype)
    n = w.sum() * 34
    w = w[..., None]
    return (dg * w).sum() / n + C4 * (dg4 * w).sum() / n + (dr * w).sum() / n


def grads(sd: dict, rec: np.ndarray, frames=None, dtype=torch.float64, device="cpu", chunk=None):
    """(loss, {state_dict name: gradient as numpy}) of the records' windows, by autograd in `dtype`.  chunk: windows
    per autograd pass (None: all in one).  The loss is a mean over every counted hop x 34 bands of the whole batch, so
    chunk c's loss is its own mean times count_c / count_total; the passes' gradients add up in .grad."""
    m = model(sd, dtype, device)
    B, T = rec.shape[:2]
    chunk = chunk or B
    counts = np.full(B, T, np.int64) if frames is None else np.asarray(frames, np.int64)
    total = float(counts.sum())
    L = 0.0
    for c0 in range(0, B, chunk):
        part = slice(c0, min(B, c0 + chunk))
        xt, y, fr = _inputs(rec, counts, part, frames, dtype, device)
        Lc = loss(m(xt), y, fr)
        if chunk < B:
            Lc = Lc * (float(counts[part].sum()) / total)
        Lc.backward()
        L += float(Lc.detach())
        del xt, y, Lc
    return L, {k: p.grad.detach().cpu().numpy() for k, p in m.named_parameters()}


def _inputs(rec, counts, part, frames, dtype, device):
    """The network input and labels of windows rec[part], hops past each window's end zeroed; and their frames."""
    fr = None if frames is None else [int(f) for f in counts[part]]
    x = features(rec[part])
    if fr is not None:
        for b, f in enumerate(fr):
            x[b, f:] = 0
    xt = torch.from_numpy(x).to(device=device, dtype=dtype)
    y = torch.from_numpy(np.ascontiguousarray(rec[part, :, 70:])).to(device=device, dtype=dtype)
    return xt, y, fr


def forward_taps(sd: dict, rec: np.ndarray, frames=None, dtype=torch.float64, device="cpu"):
    """The fc output, conv1 output and conv2 pre-activation of the records' windows in `dtype`, as numpy arrays laid out
    as the trainer's taps are: [T][B][width], hops past a window's end computed from its zeroed input."""
    m = model(sd, dtype, device)
    B, T = rec.shape[:2]
    counts = np.full(B, T, np.int64) if frames is None else np.asarray(frames, np.int64)
    with torch.no_grad():
        x, _, _ = _inputs(rec, counts, slice(0, B), frames, dtype, device)
        fc = m.fc(x)
        c1 = m.conv1(fc.permute(0, 2, 1))[:, :, :-4]
        c2p = m.conv2[0](c1)[:, :, :-2]
    hop_major = lambda a: np.ascontiguousarray(a.detach().cpu().numpy().transpose(1, 0, 2))
    return hop_major(fc), hop_major(c1.permute(0, 2, 1)), hop_major(c2p.permute(0, 2, 1))


class TanhAtPre(torch.autograd.Function):
    """tanh whose derivative is taken from the pre-activation a in closed form, 4 e / (1 + e)^2 with e = exp(-2|a|), as
    the trainer's kEpiDTanh takes it: torch's 1 - y^2 of the output y loses every digit of tanh'(a) where y rounds to
    +-1 (|a| > 19 in float64), and most of them from |a| of about 9 on.  factor: tanh'(a) given instead (same shape)."""

    @staticmethod
    def forward(ctx, a, factor=None):
        ctx.save_for_backward(a, factor)
        return torch.tanh(a)

    @staticmethod
    def backward(ctx, g):
        a, factor = ctx.saved_tensors
        if factor is None:
            e = torch.exp(-2 * a.abs())
            factor = 4 * e / ((1 + e) * (1 + e))
        return g * factor, None


def grads_at(sd: dict, rec: np.ndarray, frames, fc32, c1_32, c2p32, chunk=None, device="cpu", dtanh=None, dout=None,
             want_dx=False):
    """grads at the trainer's own forward values: float64 autograd as `grads`, with fc's and conv1's outputs and conv2's
    pre-activation pinned to fc32, c1_32 and c2p32 ([T][B][128 | 512 | 512], the PNB_TAP_TRAIN_* taps) by
    straight-through substitution.  fc = fc64 m + (fc32 - fc64 m).detach(), m = fc32 > 0 (the saved output's sign is the
    ReLU mask, as in kEpiDRelu), fc64 the float64 pre-activation; conv1 the same from that fc; c2p = c2p64 + (c2p32 -
    c2p64).detach(), then c = tanh(c2p) (TanhAtPre) and the rest of Net.forward.  The values are the trainer's; the
    gradient still flows through the float64 weights and the masks, with tanh' at the trainer's own pre-activation.
    Hops past a window's end take the tapped values like any other.  dtanh: tanh' as [T][B][512] float64 instead of its
    closed form at c2p32.  dout: dL/d(out) as [B][T][68] float64, seeding the backward (out.backward(dout)) instead of
    CustomLoss, as pnb_train_backward_device takes the caller's.  want_dx: also dL/dx ([B][T][70], through the masked fc64
    path to the network input).
    Returns (loss or None when dout is given, {name: gradient}, out at the own values [B][T][68], dL/dx or None)."""
    m = model(sd, torch.float64, device)
    B, T = rec.shape[:2]
    chunk = chunk or B
    counts = np.full(B, T, np.int64) if frames is None else np.asarray(frames, np.int64)
    total = float(counts.sum())
    L, outs, dxs = 0.0, [], []
    for c0 in range(0, B, chunk):
        part = slice(c0, min(B, c0 + chunk))
        x, y, fr = _inputs(rec, counts, part, frames, torch.float64, device)
        x.requires_grad_(want_dx)
        # [T][B][w] taps -> [b, w, T] of this chunk, as float64
        tap = lambda a: torch.from_numpy(np.ascontiguousarray(np.asarray(a)[:, part].transpose(1, 2, 0))).to(
            device=device, dtype=torch.float64)
        fc_t, c1_t, c2p_t = tap(fc32), tap(c1_32), tap(c2p32)
        fc64 = m.fc[0](x).permute(0, 2, 1)
        mk = (fc_t > 0).to(torch.float64)
        fc = fc64 * mk + (fc_t - fc64 * mk).detach()
        c1_64 = m.conv1[0](fc)[:, :, :-4]
        mk = (c1_t > 0).to(torch.float64)
        c1 = c1_64 * mk + (c1_t - c1_64 * mk).detach()
        c2p64 = m.conv2[0](c1)[:, :, :-2]
        c2p = c2p64 + (c2p_t - c2p64).detach()
        c = TanhAtPre.apply(c2p, None if dtanh is None else tap(dtanh))
        out = m.head(c.permute(0, 2, 1))
        outs.append(out.detach().cpu().numpy())
        if dout is None:
            Lc = loss(out, y, fr)
            if chunk < B:
                Lc = Lc * (float(counts[part].sum()) / total)
            Lc.backward()
            L += float(Lc.detach())
            del Lc
        else:
            out.backward(torch.as_tensor(np.asarray(dout)[part], dtype=torch.float64, device=device))
        if want_dx:
            dxs.append(x.grad.detach().cpu().numpy())
        del x, y, out
    return (None if dout is not None else L, {k: p.grad.detach().cpu().numpy() for k, p in m.named_parameters()},
            np.concatenate(outs), np.concatenate(dxs) if want_dx else None)


def dloss_dpre(p: np.ndarray, y: np.ndarray, count: int) -> np.ndarray:
    """CustomLoss's gradient at the sigmoid inputs of predictions p [..., 68] against labels y, in closed form (float64):
    g: -dg (1 + 2 C4 dg^2) sqrt(p) (1 - p), r: dr p sqrt(1 - p), over `count` terms of each mean."""
    p = np.asarray(p, np.float64)
    y = np.asarray(y, np.float64)
    dg = np.sqrt(y[..., :34]) - np.sqrt(p[..., :34])
    g = -dg * (1 + 2 * C4 * dg * dg) * np.sqrt(p[..., :34]) * (1 - p[..., :34])
    dr = np.sqrt(1 - y[..., 34:]) - np.sqrt(1 - p[..., 34:])
    r = dr * p[..., 34:] * np.sqrt(1 - p[..., 34:])
    return np.concatenate([g, r], -1) / count


def adam_step(p, g, m, v, lr: float, step: int):
    """torch.optim.Adam's single-tensor CPU step (defaults) in numpy float32, with ATen's roundings: lerp and addcmul
    fused (their products are exact in float64, so one float64 add rounded once is the fused result), the rest one
    rounding per operation.  Returns the new (p, m, v)."""
    f32, f64 = np.float32, np.float64
    w1, s2 = f32(1 - 0.9), f32(1 - 0.999)
    m = (m.astype(f64) + f64(w1) * (g - m).astype(f32).astype(f64)).astype(f32)
    v = ((s2 * g).astype(f32).astype(f64) * g.astype(f64) + (v * f32(0.999)).astype(f32).astype(f64)).astype(f32)
    bc1, bc2 = 1 - 0.9 ** step, 1 - 0.999 ** step
    den = ((np.sqrt(v) / f32(bc2 ** 0.5)).astype(f32) + f32(1e-8)).astype(f32)
    p = (p + ((f32(-(lr / bc1)) * m).astype(f32) / den).astype(f32)).astype(f32)
    return p, m, v
