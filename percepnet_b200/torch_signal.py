"""The bit-exact signal path around the gain network as PyTorch operations, differentiable in g/r: a model trains on a
loss on the enhanced waveform through the same DSP arithmetic it is deployed with.

    features, ops = sp.analyze(noisy)       # pnb_analyze_device_* + pnb_synthesis_operands_device; not differentiable
    gr = net(features)                      # e.g. torch_module.PercepNet: [B, T, 70] -> [B, T, 68]
    out = sp.synthesize(gr, ops)            # pnb_synthesize_device_f32; backward: pnb_synthesis_backward_device
    loss = (out - clean_delayed).abs().mean()

``SignalPath`` holds one PNB_SIGNAL_ONLY engine.  Its streams carry their signal state (history, pitch memory, spectra,
overlap-add memory) from call to call, so consecutive windows of a file continue exactly as a deployed engine would;
``reset`` starts new streams.  The gradient of a call stops at its edges: nothing flows into the PCM input (the pitch
search and the silence decision are not differentiable), and the second half of the call's last hop, which goes to the
overlap-add memory of the next call, takes no gradient, as truncated backpropagation through time cuts the graph.

Two facts a user will otherwise trip over:

* Scale.  The engine takes PCM at the C API's scale.  At unit-scale float input (|x| <= 1) every hop is silent (the
  analysis's sum of band energies is below 0.1), so the pitch filter never runs and r receives no gradient (dL/dr is
  exactly 0).  Feed int16-scale floats, as ``train()`` does; int16 tensors are read as s / 32768, as the CLI reads
  its input, and are unit scale too.
* Latency.  The output lags the input by ``LATENCY_SAMPLES`` = PNB_LATENCY_FRAMES x 480 = 2880 samples (five hops of
  look-ahead and one of overlap-add): compare ``out`` against the clean signal delayed by that many samples.

There is no CPU path: a CPU input raises.
"""
from __future__ import annotations

import torch

from . import api

FRAME = api.FRAME
FEATURES = 70
OPS_FLOATS = api.SYNTH_OPS_FLOATS
LATENCY_FRAMES = 6                      # PNB_LATENCY_FRAMES: five hops of look-ahead, one of overlap-add
LATENCY_SAMPLES = LATENCY_FRAMES * FRAME


class _Synthesis(torch.autograd.Function):
    """out = the pending synthesis of `path` with g/r `gr`; the backward reads only the saved g/r and operands, so it
    may run after later analyses and syntheses of the same path."""

    @staticmethod
    @torch.amp.custom_fwd(device_type="cuda", cast_inputs=torch.float32)
    def forward(ctx, path, gr, ops):
        B, T = gr.shape[:2]
        gr = gr.contiguous()
        out = torch.empty((B, T * FRAME), dtype=torch.float32, device=gr.device)
        with torch.cuda.device(gr.device):
            path._eng.synthesize_device(gr.data_ptr(), T * 68, T, out.data_ptr(), T * FRAME,
                                        torch.cuda.current_stream().cuda_stream)
        path._pending = None
        ctx.postfilter = path.postfilter
        ctx.save_for_backward(gr, ops)
        return out

    @staticmethod
    @torch.autograd.function.once_differentiable
    @torch.amp.custom_bwd(device_type="cuda")
    def backward(ctx, dout):
        gr, ops = ctx.saved_tensors
        B, T = gr.shape[:2]
        dout = dout.to(torch.float32).contiguous()
        dgr = torch.empty((B, T, 68), dtype=torch.float32, device=gr.device)
        with torch.cuda.device(gr.device):
            api.synthesis_backward_device(ops.data_ptr(), T * OPS_FLOATS, gr.data_ptr(), T * 68, B, T, ctx.postfilter,
                                          dout.data_ptr(), T * FRAME, dgr.data_ptr(), T * 68,
                                          torch.cuda.current_stream().cuda_stream)
        return None, dgr, None


class SignalPath:
    """The signal path of `rows` streams of at most `max_frames` hops per call on one CUDA device: analyze(pcm) then
    synthesize(gr, ops), alternately.  postfilter: the envelope post-filter on g (PNB_POSTFILTER).  The engine is created
    on the first analyze; a call with B < rows advances streams [0, B) (a change of B restarts the streams that enter
    the range)."""

    def __init__(self, rows: int, max_frames: int, postfilter: bool = False, device=None):
        if rows < 1 or max_frames < 1:
            raise ValueError(f"rows and max_frames must be >= 1, not {rows} and {max_frames}")
        self.rows, self.max_frames, self.postfilter = int(rows), int(max_frames), bool(postfilter)
        self.device = None if device is None else torch.device(device)
        if self.device is not None and self.device.type != "cuda":
            raise RuntimeError(f"SignalPath runs on a CUDA device only, not {self.device}")
        self._eng = None
        self._pending = None   # the operands tensor of the analysis whose synthesis is due

    def _engine(self, device: torch.device) -> api.Engine:
        if self._eng is None:
            flags = api.SIGNAL_ONLY | (api.POSTFILTER if self.postfilter else 0)
            self._eng = api.Engine(self.rows, self.max_frames, None, flags, device.index)
            self.device = device
        return self._eng

    def _check_device(self, t: torch.Tensor, name: str):
        if not t.is_cuda:
            raise RuntimeError(f"percepnet_b200.torch_signal.SignalPath runs on the GPU only: {name} must be a CUDA "
                               "tensor (there is no CPU path)")
        if self.device is not None and self.device.index is not None and t.device != self.device:
            raise ValueError(f"{name} must be on the path's device {self.device}, not {t.device}")

    def _check_rows(self, B: int, T: int):
        if B > self.rows or T > self.max_frames:
            raise ValueError(f"B x T = {B} x {T} is above the path's {self.rows} rows x {self.max_frames} hops")

    def analyze(self, pcm: torch.Tensor):
        """pcm [B, T*480] float32 (the C API's scale: pass int16-scale floats) or int16 (read as s / 32768) CUDA ->
        (features [B, T, 70], ops [B, T, OPS_FLOATS]) float32: the network input of each hop and the operands its
        synthesis will read.  Not differentiable.  Leaves the synthesis of these T hops pending: synthesize(gr, ops)
        comes next."""
        autocast = torch.is_autocast_enabled("cuda")
        if pcm.dim() != 2 or pcm.shape[0] < 1 or pcm.shape[1] < FRAME or pcm.shape[1] % FRAME:
            raise ValueError(f"pcm must be [B, T*480] with B, T >= 1, not {list(pcm.shape)}")
        if pcm.dtype != torch.int16 and pcm.dtype != torch.float32:
            if not (autocast and pcm.is_floating_point()):
                raise TypeError(f"pcm must be float32 or int16, not {pcm.dtype} (under autocast floats are cast to "
                                "float32)")
            pcm = pcm.float()
        B, T = pcm.shape[0], pcm.shape[1] // FRAME
        self._check_rows(B, T)
        self._check_device(pcm, "pcm")
        pcm = pcm.detach().contiguous()
        with torch.cuda.device(pcm.device):
            eng = self._engine(pcm.device)
            st = torch.cuda.current_stream().cuda_stream
            if eng.active != B:
                eng.set_active(B, st)
            features = torch.empty((B, T, FEATURES), dtype=torch.float32, device=pcm.device)
            ops = torch.empty((B, T, OPS_FLOATS), dtype=torch.float32, device=pcm.device)
            eng.analyze_device(pcm.data_ptr(), T * FRAME, T, features.data_ptr(), T * FEATURES, st,
                               int16=pcm.dtype == torch.int16)
            eng.synthesis_operands_device(ops.data_ptr(), T * OPS_FLOATS, st)
        self._pending = ops
        return features, ops

    def synthesize(self, gr: torch.Tensor, ops: torch.Tensor) -> torch.Tensor:
        """gr [B, T, 68] float32 CUDA (34 g then 34 r per hop), ops: the operands the pending analysis returned ->
        out [B, T*480] float32, differentiable in gr.  Completes the pending hops and advances the streams."""
        autocast = torch.is_autocast_enabled("cuda")
        if gr.dim() != 3 or gr.shape[2] != 68 or gr.shape[0] < 1 or gr.shape[1] < 1:
            raise ValueError(f"gr must be [B, T, 68] with B, T >= 1, not {list(gr.shape)}")
        if not autocast and gr.dtype != torch.float32:
            raise TypeError(f"gr must be float32, not {gr.dtype} (under autocast it is cast to float32)")
        if self._pending is None or ops is not self._pending:
            raise ValueError("ops must be the operands of the pending analysis: call analyze first, and synthesize "
                             "each analysis once")
        if tuple(gr.shape[:2]) != tuple(ops.shape[:2]):
            raise ValueError(f"gr must be [B, T, 68] = {[*ops.shape[:2], 68]} as the pending analysis, not "
                             f"{list(gr.shape)}")
        self._check_device(gr, "gr")
        return _Synthesis.apply(self, gr, ops)

    def reset(self, rows=None):
        """Starts new streams: every stream (rows None; a pending analysis is cancelled), or the listed ones of the
        last call's [0, B)."""
        if self._eng is None:
            return
        if rows is None:
            self._eng.reset()
            self._pending = None
        else:
            with torch.cuda.device(self.device):
                self._eng.reset_streams(rows, torch.cuda.current_stream().cuda_stream)

    def _check_states(self, what: str):
        if self._eng is None:
            raise RuntimeError(f"SignalPath.{what}: the path has no streams before its first analyze")
        if self._pending is not None:
            raise RuntimeError(f"SignalPath.{what}: an analysis is pending (its streams are mid-hop): synthesize it "
                               "first")

    def export_states(self, rows) -> torch.Tensor:
        """The state blobs of the listed streams of the last call's [0, B): CUDA uint8 [len(rows), pnb_state_size()]
        (pnb_export_states; the signal part, the network part zero), e.g. to checkpoint a run between windows.
        Refused before the first analyze and while an analysis is pending."""
        self._check_states("export_states")
        with torch.cuda.device(self.device):
            return self._eng.export_states(rows, None, stream=torch.cuda.current_stream().cuda_stream)

    def import_states(self, rows, blobs: torch.Tensor):
        """The listed streams continue from the blobs of export_states (CUDA uint8 [len(rows), pnb_state_size()], on
        the path's device; pnb_import_states, the network part ignored).  Refused as export_states."""
        self._check_states("import_states")
        with torch.cuda.device(self.device):
            self._eng.import_states(rows, blobs, stream=torch.cuda.current_stream().cuda_stream)

    def close(self):
        """Frees the engine (the next analyze creates a fresh one)."""
        if self._eng is not None:
            self._eng.close()
        self._eng, self._pending = None, None
