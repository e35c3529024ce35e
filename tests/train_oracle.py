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
        fr = None if frames is None else [int(f) for f in counts[part]]
        x = features(rec[part])
        if fr is not None:
            for b, f in enumerate(fr):
                x[b, f:] = 0
        xt = torch.from_numpy(x).to(device=device, dtype=dtype)
        y = torch.from_numpy(np.ascontiguousarray(rec[part, :, 70:])).to(device=device, dtype=dtype)
        Lc = loss(m(xt), y, fr)
        if chunk < B:
            Lc = Lc * (float(counts[part].sum()) / total)
        Lc.backward()
        L += float(Lc.detach())
        del xt, y, Lc
    return L, {k: p.grad.detach().cpu().numpy() for k, p in m.named_parameters()}


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
