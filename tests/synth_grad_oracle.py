"""A float64 torch restatement of the synthesis on its operands (include/pnb_synth_grad.h): pitch mix, interp_band_gain,
gain, inverse transform, window and overlap-add, and optionally the envelope post-filter, for rows of hops.  Its
autograd is the oracle of pnb_synthesis_backward_device.

    ops [B, T, 1636]: X (bins 0..399, re/im interleaved), P, the band energies Ex, the silence flag
    gr  [B, T, 68]: 34 g then 34 r per hop
    out [B, T*480]: hop t = first half of hop t's windowed inverse transform + second half of hop t-1's (of `mem` for
        hop 0); the second half of hop T-1 is returned as the memory the call leaves

The tables are the engine's (pnb_engine.cu build_tables, from the reference's expressions): the half window and the
ERB borders from the C oracle, frac = (float)j / width and 1 - frac rounded to float32, as the synthesis kernel reads
them.  In float64 the result agrees with tests/synthesis_oracle.py (the float32 synthesis, bit-exact to the reference)
to float32 rounding.
"""
import math

import numpy as np
import torch

FRAME, WIN, BINS, NBANDS, OPS = 480, 960, 400, 34, 1636
BETA = 0.02


class Tables:
    """float64 tensors of the synthesis's constants: hw [480], frac / omf / band_of [400], the inverse transform's
    cosine and sine rows [400, 960] with the Hermitian fold's factor (1 for bin 0, 2 above)."""

    def __init__(self, oracle):
        hw, _ = oracle.tables()
        border = [int(b) for b in oracle.erb_borders()]
        frac, omf, band = np.zeros(BINS, np.float32), np.zeros(BINS, np.float32), np.zeros(BINS, np.int64)
        for b in range(NBANDS - 1):
            width = border[b + 1] - border[b]
            for j in range(width):
                k = border[b] + j
                if k < BINS:
                    frac[k] = np.float32(j) / np.float32(width)
                    omf[k] = np.float32(1) - frac[k]
                    band[k] = b
        self.hw = torch.from_numpy(hw.astype(np.float64))
        self.frac, self.omf = torch.from_numpy(frac.astype(np.float64)), torch.from_numpy(omf.astype(np.float64))
        self.band = torch.from_numpy(band)
        k = np.arange(BINS)[:, None]
        n = np.arange(WIN)[None, :]
        c = np.where(k == 0, 1.0, 2.0)
        self.cos = torch.from_numpy(c * np.cos(2 * np.pi * k * n / WIN))
        self.sin = torch.from_numpy(c * np.sin(2 * np.pi * k * n / WIN))


def post_filter(g, Ey):
    """g [..., 34] -> the filtered g (denoise.cpp:216-250, beta 0.02) in float64.  Where G is 0 (every g zero) the
    filtered gains vanish to second order: the square root is taken at a safe point there, so that the gradient is 0
    rather than inf * 0."""
    gw = g * torch.sin(math.pi / 2 * g)
    e0 = (g * Ey).sum(-1, keepdim=True)
    e1 = (gw * Ey).sum(-1, keepdim=True)
    q = e0 / (e1 + 1e-6)
    live = q != 0
    qs = torch.where(live, q, torch.ones_like(q))
    G = torch.where(live, torch.sqrt((1 + BETA) * qs / (1 + BETA * qs * qs)), torch.zeros_like(q))
    return G * gw


def synthesize(tab, ops, gr, postfilter, mem=None):
    """ops [B, T, 1636], gr [B, T, 68] (float64; gr may require grad), mem [B, 480] or None (zeros) ->
    (out [B, T*480], the memory left for the next call [B, 480])."""
    B, T = gr.shape[:2]
    Xr, Xi = ops[..., 0:2 * BINS:2], ops[..., 1:2 * BINS:2]
    Pr, Pi = ops[..., 2 * BINS:4 * BINS:2], ops[..., 2 * BINS + 1:4 * BINS:2]
    Ey = ops[..., 4 * BINS:4 * BINS + NBANDS]
    silent = (ops[..., 4 * BINS + NBANDS] != 0)[..., None]
    g, r = gr[..., :NBANDS], gr[..., NBANDS:]
    gu = post_filter(g, Ey) if postfilter else g
    b = tab.band
    interp = lambda v: tab.omf * v[..., b] + tab.frac * v[..., b + 1]   # noqa: E731  interp_band_gain, :162
    gf = interp(gu)
    rfx, rfp = interp(1 - r), interp(r)                                   # pitch_filter, :436-485
    Zr = torch.where(silent, Xr, rfx * Xr + rfp * Pr)
    Zi = torch.where(silent, Xi, rfx * Xi + rfp * Pi)
    x = (gf * Zr) @ tab.cos - (gf * Zi) @ tab.sin                         # inverse_transform, :306-324
    first = x[..., :FRAME] * tab.hw
    second = x[..., FRAME:] * tab.hw.flip(0)                              # x[480 + m] * hw[479 - m]
    prev = torch.zeros((B, 1, FRAME), dtype=x.dtype) if mem is None else mem.reshape(B, 1, FRAME)
    prev = torch.cat([prev, second[:, :-1]], 1)
    return (first + prev).reshape(B, T * FRAME), second[:, -1]


def grad(tab, ops, gr, dout, postfilter):
    """dL/d(g, r) [B, T, 68] of L = sum(out * dout), all float64 numpy or torch: the gradient
    pnb_synthesis_backward_device computes."""
    ops, dout = torch.as_tensor(ops, dtype=torch.float64), torch.as_tensor(dout, dtype=torch.float64)
    gr = torch.as_tensor(gr, dtype=torch.float64).clone().requires_grad_(True)
    out, _ = synthesize(tab, ops, gr, postfilter)
    (d,) = torch.autograd.grad((out * dout.reshape(out.shape)).sum(), gr)
    return d
