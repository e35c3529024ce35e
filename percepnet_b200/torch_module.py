"""rnn_train.py's PercepNet as a torch.nn.Module whose forward and backward run on the GPU trainer.

``PercepNet`` has rnn_train.PercepNet's submodules, so its parameter names and shapes are that model's: a rnn_train.py
checkpoint loads with ``load_state_dict``, and ``weights.pack_state_dict`` of its ``state_dict()`` is the PNBW blob the
enhancement engines load.  Its forward is one ``pnb_train_forward_state_device`` call and its backward one
``pnb_train_backward_state_device`` call (include/pnb_train_state.h; without state or lengths they are the calls of
include/pnb_train_device.h): the trainer's own kernels, with the loss, the optimizer and anything before the network
left to torch.  Gradients arrive as ordinary ``.grad`` tensors.

Like ``nn.GRU`` it takes an initial state and returns the final one (``m(x, state, return_state=True)``), and windows of
their own lengths (``lengths=``), so that truncated backpropagation through time runs over consecutive windows of one
stream: pass each call's ``state_out`` (detached, to cut the graph there) as the next call's ``state``.

The submodules only hold the parameters; they never run.  There is no CPU path: a CPU input raises.

Memory: one trainer engine per module and device, created on the first forward, recreated when the batch B or the
length T grows (and set active to B when B shrinks).  It keeps the activations of one forward for its backward, about
70 KB per window and hop: the engine takes 0.5 GB at 10 x 500 and 18 GB at 128 x 2000.  Weights travel with every
forward, so recreating an engine loses nothing; the optimizer's state lives in torch.
"""
from __future__ import annotations

import itertools

import numpy as np
import torch
import torch.nn as nn
from torch.autograd.function import once_differentiable

from . import api
from .weights import N_PARAMS, PackedModel, pack_state_dict

MAX_ROWS = 65535 * 64   # windows x hops of one trainer engine: its contractions put the rows on gridDim.y
STATE_FLOATS = api.TRAIN_STATE_FLOATS   # one window's network state (include/pnb_train_state.h)
# The columns of each piece of a state row [B, STATE_FLOATS]: the last four fc outputs and the last two conv1 outputs
# (after ReLU, oldest first; conv1's and conv2's input histories), then the five GRU states
STATE_LAYOUT = {"fc_hist": slice(0, 512), "c1_hist": slice(512, 1536), "gru1": slice(1536, 2048),
                "gru2": slice(2048, 2560), "gru3": slice(2560, 3072), "gru_gb": slice(3072, 3584),
                "gru_rb": slice(3584, 3712)}


def blob_index(shapes) -> torch.Tensor:
    """The permutation from the parameters to the PNBW blob: for parameters (name, shape) in order, flattened and
    concatenated into `flat`, blob = flat[index].  Derived by packing a state dict whose entries are their own flat
    positions (all below 2^24, so exact in float32): weights.pack_state_dict stays the one statement of the layout."""
    sd, at = {}, 0
    for name, shape in shapes:
        n = int(np.prod(shape))
        sd[name] = np.arange(at, at + n, dtype=np.float32).reshape(shape)
        at += n
    if at >= 2 ** 24:
        raise ValueError(f"{at} parameters: positions from 2^24 on are not exact in float32")
    return torch.from_numpy(pack_state_dict(sd).flat().astype(np.int64))


def to_blob(flat: torch.Tensor, index: torch.Tensor) -> torch.Tensor:
    """The concatenated parameters `flat` in blob order."""
    return flat[index]


def from_blob(blob: torch.Tensor, index: torch.Tensor) -> torch.Tensor:
    """The inverse of to_blob: a blob-order vector back to the concatenated parameters."""
    flat = torch.empty_like(blob)
    flat[index] = blob
    return flat


class _Trainer:
    """One trainer engine of a module on one device, and which forward's backward it holds (None: none)."""

    def __init__(self, B: int, T: int, blob: torch.Tensor, device: int):
        self.eng = api.Engine(B, T, PackedModel.from_flat(blob.cpu().numpy()), api.TRAIN_NETWORK, device)
        self.B, self.T, self.pending = B, T, None

    def fits(self, B: int, T: int) -> bool:
        return B <= self.B and T <= self.T

    def activate(self, B: int):
        if self.eng.active != B:
            self.eng.set_active(B, torch.cuda.current_stream().cuda_stream)
            self.pending = None   # the engine's pending forward ran on the old rows


_forward_ids = itertools.count(1)


class _TrainerFunction(torch.autograd.Function):
    """out = PercepNet(x) on the trainer, or (out, state_out) with want_state: from the state rows `state` (None: zero
    state), each window over its own lengths (a CPU int32 tensor, or None: all T hops).  Saves x, the packed weights,
    state and lengths, so that a backward whose forward is no longer the engine's pending one runs that forward again
    first."""

    @staticmethod
    @torch.amp.custom_fwd(device_type="cuda", cast_inputs=torch.float32)
    def forward(ctx, module, x, state, lengths, want_state, *params):
        blob = to_blob(torch.cat([p.detach().reshape(-1) for p in params]), module._index_on(x.device))
        out, state_out = module._run_forward(x, blob, state, lengths, want_state)
        ctx.module, ctx.fid = module, module._trainer(x).pending
        ctx.save_for_backward(x, blob, state, lengths)
        ctx.set_materialize_grads(False)   # an output the loss does not use passes NULL, not zeros
        return (out, state_out) if want_state else out

    @staticmethod
    @once_differentiable
    @torch.amp.custom_bwd(device_type="cuda")
    def backward(ctx, dout, dstate_out=None):
        x, blob, state, lengths = ctx.saved_tensors
        m = ctx.module
        B, T = x.shape[:2]
        with torch.cuda.device(x.device):
            if m._trainers.get(x.device) is None or m._trainer(x).pending != ctx.fid:
                m._run_forward(x, blob, state, lengths, False)   # another forward ran since, or a backward used this one
            tr = m._trainer(x)
            st = torch.cuda.current_stream().cuda_stream
            if dout is None:
                dout = torch.zeros((B, T, 68), dtype=torch.float32, device=x.device)
            dout = dout.to(torch.float32).contiguous()
            dso = None if dstate_out is None else dstate_out.to(torch.float32).contiguous()
            dx = torch.empty((B, T, 70), dtype=torch.float32, device=x.device) if ctx.needs_input_grad[1] else None
            ds = torch.empty((B, STATE_FLOATS), dtype=torch.float32, device=x.device) if ctx.needs_input_grad[2] else None
            grad = torch.empty(N_PARAMS, dtype=torch.float32, device=x.device)
            tr.eng.train_backward_state_device(dout.data_ptr(), T * 68, _addr(dso), STATE_FLOATS, _addr(dx), T * 70,
                                               _addr(ds), STATE_FLOATS, grad.data_ptr(), st)
            tr.pending = None
            flat = from_blob(grad, m._index_on(x.device))
        grads, at = [], 0
        for p in m._params:
            grads.append(flat[at:at + p.numel()].view_as(p))
            at += p.numel()
        return (None, dx, ds, None, None, *grads)


def _addr(t) -> int:
    """A tensor's device address, or 0 (NULL) for None."""
    return 0 if t is None else t.data_ptr()


def _lengths(lengths, B: int, T: int) -> torch.Tensor:
    """lengths as pack_padded_sequence takes them (a CPU tensor or a sequence of B ints) as a CPU int32 tensor, each
    in [1, T]."""
    if isinstance(lengths, torch.Tensor):
        if lengths.device.type != "cpu":
            raise ValueError(f"lengths must be on the CPU (as pack_padded_sequence takes them), not {lengths.device}")
        a = lengths.detach().numpy()
    else:
        a = np.asarray(lengths)
    if a.ndim != 1 or a.shape[0] != B:
        raise ValueError(f"lengths needs one entry per window: {B}, not shape {list(a.shape)}")
    if a.dtype.kind not in "iu":
        raise TypeError(f"lengths must be integers, not {a.dtype}")
    if a.min() < 1 or a.max() > T:
        raise ValueError(f"lengths must be in [1, {T}], not [{a.min()}, {a.max()}]")
    return torch.from_numpy(np.ascontiguousarray(a, np.int32))


class PercepNet(nn.Module):
    """rnn_train.PercepNet (rnn_train.py:105-145) on the GPU trainer: x [B, T, 70] float32 CUDA -> [B, T, 68], 34 g then
    34 r per hop, every window from zero GRU state and zero conv history unless a state is given (forward).  Exact
    tanh and sigmoid, fp32 FMA."""

    def __init__(self):
        super().__init__()
        self.fc = nn.Sequential(nn.Linear(70, 128), nn.ReLU())
        self.conv1 = nn.Sequential(nn.Conv1d(128, 512, 5, padding=4), nn.ReLU())
        self.conv2 = nn.Sequential(nn.Conv1d(512, 512, 3, padding=2), nn.Tanh())
        self.gru1 = nn.GRU(512, 512, 1, batch_first=True)
        self.gru2 = nn.GRU(512, 512, 1, batch_first=True)
        self.gru3 = nn.GRU(512, 512, 1, batch_first=True)
        self.gru_gb = nn.GRU(512, 512, 1, batch_first=True)
        self.gru_rb = nn.GRU(1024, 128, 1, batch_first=True)
        self.fc_gb = nn.Sequential(nn.Linear(2560, 34), nn.Sigmoid())
        self.fc_rb = nn.Sequential(nn.Linear(128, 34), nn.Sigmoid())
        self._index = blob_index([(k, tuple(p.shape)) for k, p in self.named_parameters()])
        self._indices: dict = {}    # device -> the index there
        self._trainers: dict = {}   # device -> _Trainer

    @property
    def _params(self):
        return list(self.parameters())

    def _index_on(self, device) -> torch.Tensor:
        if device not in self._indices:
            self._indices[device] = self._index.to(device)
        return self._indices[device]

    def _trainer(self, x) -> _Trainer:
        return self._trainers[x.device]

    def _run_forward(self, x: torch.Tensor, blob: torch.Tensor, state=None, lengths=None, want_state=False):
        """One pnb_train_forward_state_device of x with the weights blob on the current stream, from state (or zero
        state) over lengths (or all T hops): (out, the state out or None).  Its backward becomes due."""
        B, T = x.shape[:2]
        with torch.cuda.device(x.device):
            tr = self._trainers.get(x.device)
            if tr is None or not tr.fits(B, T):
                if tr is not None:
                    tr.eng.close()
                tr = self._trainers[x.device] = _Trainer(max(B, tr.B if tr else 0), max(T, tr.T if tr else 0), blob,
                                                         x.device.index)
            tr.activate(B)
            x = x.contiguous()
            state = None if state is None else state.contiguous()
            out = torch.empty((B, T, 68), dtype=torch.float32, device=x.device)
            state_out = torch.empty((B, STATE_FLOATS), dtype=torch.float32, device=x.device) if want_state else None
            tr.eng.train_forward_state_device(x.data_ptr(), T * 70, T, None if lengths is None else lengths.numpy(),
                                              blob.data_ptr(), _addr(state), STATE_FLOATS, out.data_ptr(), T * 68,
                                              _addr(state_out), STATE_FLOATS, torch.cuda.current_stream().cuda_stream)
            tr.pending = next(_forward_ids)
        return out, state_out

    def forward(self, x: torch.Tensor, state: torch.Tensor | None = None, *, lengths=None, return_state: bool = False):
        """x [B, T, 70] -> out [B, T, 68], or (out, state_out) with return_state.  state: None (every window from zero
        state) or [B, STATE_FLOATS] on x's device, the state each window starts from (STATE_LAYOUT); differentiable, as
        state_out is, so that chained calls backpropagate through time unless the state is detached.  lengths: None,
        or B hop counts in [1, T] (a CPU tensor or a sequence, as pack_padded_sequence takes them): window b ends
        after lengths[b] hops, its out rows past that are zeros and take no gradient, and state_out is its state there."""
        autocast = torch.is_autocast_enabled("cuda")
        lens = None
        if x.dim() == 3:   # state and lengths are refused alike on any device
            B, T = x.shape[:2]
            if state is not None:
                if tuple(state.shape) != (B, STATE_FLOATS):
                    raise ValueError(f"state must be [B, {STATE_FLOATS}] = [{B}, {STATE_FLOATS}], not {list(state.shape)}")
                if state.device != x.device:
                    raise ValueError(f"state must be on x's device {x.device}, not {state.device}")
                if not autocast and state.dtype != torch.float32:
                    raise TypeError(f"state must be float32, not {state.dtype} (under autocast it is cast to float32)")
            lens = None if lengths is None else _lengths(lengths, B, T)
        if not x.is_cuda:
            raise RuntimeError("percepnet_b200.torch_module.PercepNet runs on the GPU trainer only: x must be a CUDA "
                               "tensor (there is no CPU path)")
        if x.dim() != 3 or x.shape[2] != 70 or x.shape[0] < 1 or x.shape[1] < 1:
            raise ValueError(f"x must be [B, T, 70] with B, T >= 1, not {list(x.shape)}")
        if not autocast and x.dtype != torch.float32:
            raise TypeError(f"x must be float32, not {x.dtype} (under autocast it is cast to float32)")
        B, T = x.shape[:2]
        if B * T > MAX_ROWS:
            raise ValueError(f"B x T = {B} x {T} is above the trainer's {MAX_ROWS} rows (65535 x 64): split the batch")
        params = self._params
        if any(p.device != x.device or p.dtype != torch.float32 for p in params):
            raise TypeError(f"the parameters must be float32 on {x.device}: call .to(x.device) first")
        return _TrainerFunction.apply(self, x, state, lens, return_state, *params)

    def close(self):
        """Frees the trainer engines (they are recreated by the next forward)."""
        for tr in self._trainers.values():
            tr.eng.close()
        self._trainers.clear()
