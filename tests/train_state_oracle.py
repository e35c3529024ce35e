"""train_oracle.Net run from a network state: the float64 truth of torch_module.PercepNet's forward with state.

A state row is [fc_hist 4 x 128][c1_hist 2 x 512][gru1, gru2, gru3, gru_gb 512 each][gru_rb 128] (include/
pnb_train_state.h).  Net.forward pads conv1's input with four zero hops and conv2's with two; here those hops are the
state's histories, and the GRUs start from its h0 instead of zeros.  The state out is the last four fc outputs, the last
two conv1 outputs and each GRU's h_n, so that a forward from the state out of hops [0, T1) over hops [T1, T2) is the
forward over [0, T2).
"""
from __future__ import annotations

import torch
import torch.nn.functional as F

STATE_FLOATS = 3712
GRUS = ("gru1", "gru2", "gru3", "gru_gb", "gru_rb")


def forward(m, x, state=None):
    """(out [B, T, 68], state_out [B, STATE_FLOATS]) of Net m on x [B, T, 70] from state [B, STATE_FLOATS] (None: zero
    state), in m's dtype."""
    B = x.shape[0]
    if state is None:
        state = x.new_zeros((B, STATE_FLOATS))
    h0 = [state[:, 1536 + 512 * l:1536 + 512 * l + (512 if l < 4 else 128)][None].contiguous() for l in range(5)]
    fcs = torch.cat([state[:, :512].reshape(B, 4, 128), m.fc(x)], 1)                 # [B, 4 + T, 128]
    c1 = torch.relu(F.conv1d(fcs.permute(0, 2, 1), m.conv1[0].weight, m.conv1[0].bias)).permute(0, 2, 1)
    c1s = torch.cat([state[:, 512:1536].reshape(B, 2, 512), c1], 1)                  # [B, 2 + T, 512]
    c = torch.tanh(F.conv1d(c1s.permute(0, 2, 1), m.conv2[0].weight, m.conv2[0].bias)).permute(0, 2, 1)
    h1, n1 = m.gru1(c, h0[0])
    h2, n2 = m.gru2(h1, h0[1])
    h3, n3 = m.gru3(h2, h0[2])
    hg, ng = m.gru_gb(h3, h0[3])
    hr, nr = m.gru_rb(torch.cat((h3, c), -1), h0[4])
    out = torch.cat((m.fc_gb(torch.cat((c, h1, h2, h3, hg), -1)), m.fc_rb(hr)), -1)
    state_out = torch.cat([fcs[:, -4:].reshape(B, -1), c1s[:, -2:].reshape(B, -1)] + [h[0] for h in (n1, n2, n3, ng, nr)], 1)
    return out, state_out


def random_state(B: int, seed: int, dtype=torch.float32) -> torch.Tensor:
    """A nonzero state of the kind a stream reaches: histories after ReLU (in [0, 0.5)), GRU states in (-0.9, 0.9)."""
    g = torch.Generator().manual_seed(seed)
    s = torch.rand((B, STATE_FLOATS), generator=g, dtype=torch.float64)
    s[:, :1536] *= 0.5
    s[:, 1536:] = (2 * s[:, 1536:] - 1) * 0.9
    return s.to(dtype)
