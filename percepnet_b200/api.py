"""Python host mirror of the C-ABI in include/percepnet_b200.h, include/pnb_train_device.h, include/pnb_train_state.h and
include/pnb_synth_grad.h (ctypes; no compute here).

``Engine`` is the batched-streams counterpart of the reference's ``DenoiseState``
(/root/reference/src/rnnoise.h:49-60): ``Engine.process`` advances S independent 48 kHz streams by F
hops of 480 samples, i.e. S x F calls of ``rnnoise_process_frame``.  The CUDA library is mandatory:
there is no CPU path, and a missing ``libpercepnet_b200.so`` raises at import of the symbol table.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from .weights import PackedModel

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(HERE, "libpercepnet_b200.so")

FRAME = 480
NN_FP32, NN_TENSOR, POSTFILTER, KEEP_TAPS, TRAIN_DATA, CONV_WIDE, TRAIN_AUDIO, NETWORK_ONLY = 0, 1, 2, 4, 8, 16, 32, 64
SIGNAL_ONLY = 128
TRAIN_NETWORK = 256
TRAIN_ARRAYS = {"weights": 0, "gradient": 1, "m": 2, "v": 3, "accum": 4}   # pnb_train_export / pnb_train_import
RECORD = 138
RNN_FEATURES, RNN_RECORDS = 0, 1   # pnb_compute_rnn_* formats: 70 features or 138 record floats per hop
TAPS = {"features": (0, np.float32, 70), "pitch": (1, np.int32, 4), "pitchf": (2, np.float32, 2),
        "X": (3, np.float32, 800), "P": (4, np.float32, 800), "Ex": (5, np.float32, 34), "gr": (6, np.float32, 68),
        "g_used": (13, np.float32, 34),
        # TRAIN_NETWORK: fc / conv1 outputs and conv2's pre-activation of the last train_grad or train_forward_device,
        # and the gradient at the output pre-activations of the last train_grad or train_backward_device,
        # [F][active rows][width]
        "train_fc": (14, np.float32, 128), "train_c1": (15, np.float32, 512), "train_c2pre": (16, np.float32, 512),
        "train_dpre": (17, np.float32, 68)}
# read_nn_state: the network state after the last hop, [n_streams][width] (PNB_TAP_NN_C2, PNB_TAP_NN_H0 + 0..4)
_NN_STATE = {"c2": (7, np.float32, 512), "gru1": (8, np.float32, 512), "gru2": (9, np.float32, 512),
             "gru3": (10, np.float32, 512), "gru_gb": (11, np.float32, 512), "gru_rb": (12, np.float32, 128)}

_lib = None


class PnbError(RuntimeError):
    pass


_PCM = (np.float32, np.int16)   # the wire formats of the PCM entry points
_vp, _sz, _i, _ll = C.c_void_p, C.c_size_t, C.c_int, C.c_longlong


def _f32_i16(name: str, *argtypes) -> dict:
    """Signatures of the f32 and the i16 form of `name` ({} marks the suffix); both take the same types."""
    return {name.format(t): (_i, argtypes) for t in ("f32", "i16")}


# Every symbol of include/percepnet_b200.h, in the header's order: name -> (restype, argtypes).  Every pointer is a
# c_void_p, so callers pass addresses as ints (0 or None for NULL).
_SIGNATURES = {
    "pnb_create": (_i, (C.POINTER(_vp), _i, _i, _vp, C.c_uint, _i)),
    "pnb_destroy": (None, (_vp,)),
    "pnb_reset": (_i, (_vp,)),
    "pnb_resolve_device": (_i, (_i,)),
    "pnb_model_load_blob": (_i, (C.c_char_p, C.POINTER(_vp))),
    "pnb_model_load_stream": (_i, (_vp, C.POINTER(_vp))),
    "pnb_model_free": (None, (_vp,)),
    **_f32_i16("pnb_process_host_{}", _vp, _vp, _sz, _vp, _sz, _i, _vp),
    **_f32_i16("pnb_submit_host_{}", _vp, _vp, _sz, _vp, _sz, _i),
    "pnb_wait": (_i, (_vp,)),
    "pnb_check": (_i, (_vp, _vp)),
    **_f32_i16("pnb_process_device_{}", _vp, _vp, _sz, _vp, _sz, _i, _vp, _vp),
    **_f32_i16("pnb_submit_device_{}", _vp, _vp, _sz, _vp, _sz, _i, _vp),
    "pnb_flush": (_i, (_vp, _vp)),
    "pnb_train_records_host": (_i, (_vp, _vp, _sz, _vp, _sz, _i, _vp, _sz)),
    "pnb_submit_train_records": (_i, (_vp, _vp, _sz, _vp, _sz, _i, _vp, _sz)),
    "pnb_train_records_device": (_i, (_vp, _vp, _sz, _vp, _sz, _i, _vp, _sz, _vp)),
    "pnb_train_audio_host": (_i, (_vp, _vp, _sz, _vp, _sz, _i, _vp, _sz, _vp, _sz)),
    "pnb_train_audio_device": (_i, (_vp, _vp, _sz, _vp, _sz, _i, _vp, _sz, _vp, _sz, _vp)),
    "pnb_compute_rnn_device": (_i, (_vp, _i, _vp, _sz, _i, _vp, _sz, _vp)),
    "pnb_compute_rnn_host": (_i, (_vp, _i, _vp, _sz, _i, _vp, _sz)),
    "pnb_score_records_device": (_i, (_vp, _vp, _sz, _i, _vp, _vp, _vp, _sz, _vp)),
    "pnb_score_records_host": (_i, (_vp, _vp, _sz, _i, _vp, _vp, _vp, _sz)),
    "pnb_train_grad_host": (_i, (_vp, _vp, _sz, _i, _vp, _vp)),
    "pnb_train_grad_device": (_i, (_vp, _vp, _sz, _i, _vp, _vp, _vp)),
    "pnb_train_adam": (_i, (_vp, C.c_double, _ll, _vp)),
    "pnb_train_accumulate": (_i, (_vp, _vp)),
    "pnb_train_finish": (_i, (_vp, _vp)),
    "pnb_train_export": (_i, (_vp, _i, _vp, _sz)),
    "pnb_train_import": (_i, (_vp, _i, _vp, _sz)),
    **_f32_i16("pnb_analyze_host_{}", _vp, _vp, _sz, _i, _vp, _sz),
    **_f32_i16("pnb_analyze_device_{}", _vp, _vp, _sz, _i, _vp, _sz, _vp),
    **_f32_i16("pnb_synthesize_host_{}", _vp, _vp, _sz, _i, _vp, _sz),
    **_f32_i16("pnb_synthesize_device_{}", _vp, _vp, _sz, _i, _vp, _sz, _vp),
    "pnb_state_size": (_sz, ()),
    "pnb_get_state": (_i, (_vp, _i, _vp, _sz)),
    "pnb_set_state": (_i, (_vp, _i, _vp, _sz)),
    "pnb_reset_streams": (_i, (_vp, _vp, _i, _vp)),
    "pnb_export_states": (_i, (_vp, _vp, _i, _vp, _sz, _vp)),
    "pnb_import_states": (_i, (_vp, _vp, _i, _vp, _sz, _vp)),
    "pnb_set_active_streams": (_i, (_vp, _i, _vp)),
    "pnb_active_streams": (_i, (_vp,)),
    "pnb_sessions_reserve": (_i, (_vp, _i)),
    **_f32_i16("pnb_process_sessions_device_{}", _vp, _vp, _i, _vp, _sz, _vp, _sz, _i, _vp, _vp),
    **_f32_i16("pnb_process_sessions_host_{}", _vp, _vp, _i, _vp, _sz, _vp, _sz, _i, _vp),
    **_f32_i16("pnb_process_sessions_ragged_device_{}", _vp, _vp, _vp, _i, _vp, _sz, _vp, _sz, _vp, _vp),
    **_f32_i16("pnb_process_sessions_ragged_host_{}", _vp, _vp, _vp, _i, _vp, _sz, _vp, _sz, _vp),
    "pnb_reset_sessions": (_i, (_vp, _vp, _i, _vp)),
    "pnb_export_sessions": (_i, (_vp, _vp, _i, _vp, _sz, _vp)),
    "pnb_import_sessions": (_i, (_vp, _vp, _i, _vp, _sz, _vp)),
    "pnb_session_stats": (_i, (_vp, _vp)),
    **_f32_i16("pnb_analyze_sessions_device_{}", _vp, _vp, _vp, _i, _vp, _sz, _i, _vp, _sz, _vp),
    **_f32_i16("pnb_analyze_sessions_host_{}", _vp, _vp, _vp, _i, _vp, _sz, _i, _vp, _sz),
    **_f32_i16("pnb_synthesize_sessions_device_{}", _vp, _vp, _i, _vp, _sz, _i, _vp, _sz, _vp),
    **_f32_i16("pnb_synthesize_sessions_host_{}", _vp, _vp, _i, _vp, _sz, _i, _vp, _sz),
    "pnb_compute_rnn_sessions_device": (_i, (_vp, _vp, _vp, _i, _i, _vp, _sz, _i, _vp, _sz, _vp)),
    "pnb_compute_rnn_sessions_host": (_i, (_vp, _vp, _vp, _i, _i, _vp, _sz, _i, _vp, _sz)),
    "pnb_pitch_only_device": (_i, (_vp, _sz, _ll, _vp, _vp, _vp, _vp, _vp, _vp, _vp)),
    "pnb_pitch_only_host": (_i, (_vp, _sz, _ll, _vp, _vp, _vp, _vp, _vp, _vp)),
    "pnb_read_tap": (_i, (_vp, _i, _vp, _sz)),
    "pnb_profile_enable": (_i, (_vp, _i)),
    "pnb_profile_read": (_i, (_vp, _vp, _vp)),
    "pnb_profile_timeline": (_i, (_vp, _vp, _vp, _vp, _i)),
    "pnb_kernel_class_name": (C.c_char_p, (_i,)),
    "pnb_launch_count": (_ll, (_vp,)),
    "pnb_launches_per_call": (_i, (_vp, _i)),
    "pnb_engine_bytes": (_sz, (_vp,)),
    "pnb_n_streams": (_i, (_vp,)),
    "pnb_max_frames": (_i, (_vp,)),
    "pnb_last_error": (C.c_char_p, ()),
    "pnb_version": (C.c_char_p, ()),
}
EXPORTS = tuple(_SIGNATURES)
# Every symbol of include/pnb_train_device.h (the trainer's calls with the caller's loss), the same way.
_TRAIN_DEVICE_SIGNATURES = {
    "pnb_train_forward_device": (_i, (_vp, _vp, _sz, _i, _vp, _vp, _sz, _vp)),
    "pnb_train_backward_device": (_i, (_vp, _vp, _sz, _vp, _sz, _vp, _vp)),
}
TRAIN_DEVICE_EXPORTS = tuple(_TRAIN_DEVICE_SIGNATURES)
# Every symbol of include/pnb_train_state.h (the same calls with network state and per-window lengths), the same way.
_TRAIN_STATE_SIGNATURES = {
    "pnb_train_forward_state_device": (_i, (_vp, _vp, _sz, _i, _vp, _vp, _vp, _sz, _vp, _sz, _vp, _sz, _vp)),
    "pnb_train_backward_state_device": (_i, (_vp, _vp, _sz, _vp, _sz, _vp, _sz, _vp, _sz, _vp, _vp)),
}
TRAIN_STATE_EXPORTS = tuple(_TRAIN_STATE_SIGNATURES)
TRAIN_STATE_FLOATS = 3712   # PNB_TRAIN_STATE_FLOATS: one window's network state
# Every symbol of include/pnb_synth_grad.h (the operands of a pending synthesis and its gradient), the same way.
_SYNTH_GRAD_SIGNATURES = {
    "pnb_synthesis_operands_device": (_i, (_vp, _vp, _sz, _vp)),
    "pnb_synthesis_backward_device": (_i, (_vp, _sz, _vp, _sz, _ll, _i, _i, _vp, _sz, _vp, _sz, _vp)),
}
SYNTH_GRAD_EXPORTS = tuple(_SYNTH_GRAD_SIGNATURES)
SYNTH_OPS_FLOATS = 1636     # PNB_SYNTH_OPS_FLOATS: one hop's synthesis operands


def load_library() -> C.CDLL:
    """dlopen the in-tree CUDA library; raises if it has not been built (no fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise PnbError(f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                       "(nvcc, sm_90a).  There is no CPU implementation to fall back to.")
    L = C.CDLL(LIB_PATH)
    for name, (restype, argtypes) in {**_SIGNATURES, **_TRAIN_DEVICE_SIGNATURES, **_TRAIN_STATE_SIGNATURES,
                                    **_SYNTH_GRAD_SIGNATURES}.items():
        f = getattr(L, name)
        f.restype, f.argtypes = restype, argtypes
    _lib = L
    return L


def _call_lib(name: str, *args) -> int:
    """The library's `name` on args; a negative return (every status is PNB_OK or a negative error code) raises with
    pnb_last_error()'s text.  Returns what the call returned."""
    L = load_library()
    rc = getattr(L, name)(*args)
    if rc < 0:
        raise PnbError(f"{name} failed ({rc}): {L.pnb_last_error().decode()}")
    return rc


def _typed(name: str, int16: bool) -> str:
    """The int16 or the float32 form of an entry point."""
    return f"{name}_i16" if int16 else f"{name}_f32"


def _ptr(a):
    """A host array's address for the library, or NULL for None."""
    return None if a is None else a.ctypes.data


def _int32s(values, what: str) -> np.ndarray:
    """A host list (slots, session ids, hops, frames) as a contiguous int32 array.  An entry that is not an integer, or
    that int32 cannot hold, is refused rather than truncated or wrapped to another valid value."""
    a = np.asarray(values).reshape(-1)
    if a.size and a.dtype.kind not in "iu":
        raise PnbError(f"{what}: entries must be integers, not {a.dtype}")
    if a.size and (a.min() < -2 ** 31 or a.max() >= 2 ** 31):
        raise PnbError(f"{what}: entries must fit in int32")
    return np.ascontiguousarray(a, np.int32)


def _session_ids(ids):
    """A call's session list as int32 and the infix of its entry points' names; (None, "") for a call on the active
    slots (ids None)."""
    return (None, "") if ids is None else (_int32s(ids, "ids"), "_sessions")


def _hops(hops, n: int, F) -> np.ndarray | None:
    """Per-session hop counts as int32, one per listed session with max(hops) = F hops (F None: not checked); None
    when every session runs the call's hops."""
    if hops is None:
        return None
    hp = _int32s(hops, "hops")
    if len(hp) != n or (F is not None and int(hp.max(initial=0)) != F):
        raise PnbError("hops needs one entry per session, and the call must be max(hops) hops long")
    return hp


def _host_array(a: np.ndarray, name: str, rows: int, label: str, widths=None, dtypes=(np.float32,), copy: bool = True):
    """`a` checked against what a host entry point will read: `rows` rows (`label` names them) of PCM, [rows, F*480],
    or with `widths`, [rows, F, W] of F hops of W values, W in widths.  A dtype outside `dtypes` raises TypeError, any
    other mismatch PnbError.  Returns (a, F): a C-contiguous copy where a is not, or with copy=False `a` itself, whose
    rows must then be contiguous and in order, for the caller to pass with its own row stride."""
    if a.dtype not in dtypes:
        raise TypeError(f"{name} must be " + " or ".join(np.dtype(d).name for d in dtypes))
    if widths is None:
        shape, ok = f"[{label}, F*480]", a.ndim == 2 and a.shape[1] % FRAME == 0
    else:
        shape, ok = f"[{label}, F, {' | '.join(map(str, widths))}]", a.ndim == 3 and a.shape[2] in widths
    if not ok:
        raise PnbError(f"{name} must be {shape}")
    if not copy and a.size and (a.strides[1] != a.itemsize or a.strides[0] % a.itemsize
                                or a.strides[0] < a.shape[1] * a.itemsize):
        raise PnbError(f"{name} must have contiguous rows, each behind the one before")
    if a.shape[0] != rows:
        raise PnbError(f"{name} must be {shape}: {a.shape[0]} rows for {rows}")
    F = a.shape[1] // FRAME if widths is None else a.shape[1]
    return (np.ascontiguousarray(a) if copy else a), F


def pitch_only_device(d_buf: int, stride: int, n_units: int, d_period: int, d_corr: int, d_gain: int, d_lag: int = 0,
                      d_prev_period: int = 0, d_prev_gain: int = 0, stream: int = 0):
    """pnb_pitch_only_device on raw device pointers (BASELINE.json config 5: the pitch analysis alone)."""
    _call_lib("pnb_pitch_only_device", d_buf, stride, n_units, d_prev_period, d_prev_gain, d_period, d_corr, d_gain,
              d_lag, stream)


def synthesis_backward_device(d_ops: int, ops_stride: int, d_gr: int, gr_stride: int, n_rows: int, n_frames: int,
                              postfilter: bool, d_dout: int, dout_stride: int, d_dgr: int, dgr_stride: int,
                              stream: int = 0):
    """pnb_synthesis_backward_device on raw device pointers (strides in floats): dL/d(g, r) [n_rows, n_frames, 68] of
    the synthesis whose operands (Engine.synthesis_operands_device) and g/r are given, from dL/d(out) [n_rows,
    n_frames*480]; postfilter: the POSTFILTER setting of the engine that synthesised.  Needs no engine."""
    _call_lib("pnb_synthesis_backward_device", d_ops, ops_stride, d_gr, gr_stride, n_rows, n_frames, 1 if postfilter else 0,
              d_dout, dout_stride, d_dgr, dgr_stride, stream)


def pitch_only(bufs: np.ndarray, prev_period=None, prev_gain=None):
    """pnb_pitch_only_host: [n, 1728] float32 pitch buffers -> (period int32 [n], corr [n], gain [n], lag int32 [n])"""
    b = np.ascontiguousarray(bufs, np.float32)
    n = b.shape[0]
    T, lag = np.empty(n, np.int32), np.empty(n, np.int32)
    corr, gain = np.empty(n, np.float32), np.empty(n, np.float32)
    pp = None if prev_period is None else np.ascontiguousarray(prev_period, np.int32)
    pg = None if prev_gain is None else np.ascontiguousarray(prev_gain, np.float32)
    _call_lib("pnb_pitch_only_host", _ptr(b), b.shape[1], n, _ptr(pp), _ptr(pg), _ptr(T), _ptr(corr), _ptr(gain),
              _ptr(lag))
    return T, corr, gain, lag


class BlobModel:
    """A model read from a binary weight file by the C loader (pnb_model_load_blob)."""

    def __init__(self, path: str):
        self.L = load_library()
        self.ptr = C.c_void_p()
        _call_lib("pnb_model_load_blob", path.encode(), C.byref(self.ptr))

    def free(self):
        if self.ptr:
            self.L.pnb_model_free(self.ptr)
            self.ptr = C.c_void_p()


class Engine:
    def __init__(self, n_streams: int, max_frames: int, model, flags: int = NN_FP32, device: int = 0):
        self.L = load_library()
        self.n_streams, self.max_frames, self.flags, self.device = n_streams, max_frames, flags, device
        self._model = model
        h = C.c_void_p()
        mptr = None if model is None else (model.ptr if isinstance(model, BlobModel) else C.addressof(model.as_c_model()))
        _call_lib("pnb_create", C.byref(h), n_streams, max_frames, mptr, flags, device)
        self.h = h

    def _call(self, name: str, *args) -> int:
        """The library's `name` on this engine (see _call_lib)."""
        return _call_lib(name, self.h, *args)

    def _rows(self, ids):
        """The rows of a call: (ids as int32 or None, n, label, name infix) for the listed sessions or, with ids None,
        the active slots."""
        a, infix = _session_ids(ids)
        if a is None:
            return a, self.active, "active", infix
        return a, len(a), "len(ids)", infix

    def close(self):
        if getattr(self, "h", None):
            self.L.pnb_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def reset(self):
        self._call("pnb_reset")

    @property
    def active(self) -> int:
        """Streams the next call advances: slots [0, active) (pnb_active_streams; n_streams unless set_active changed it)."""
        return int(self.L.pnb_active_streams(self.h))

    def set_active(self, n: int, stream: int = 0):
        """pnb_set_active_streams: later calls advance slots [0, n) only.  Slots entering the range start as fresh streams
        (reset asynchronously on `stream`); slots leaving it lose their state."""
        self._call("pnb_set_active_streams", n, stream)

    def process(self, x: np.ndarray, want_gr: bool = False):
        """x: [active, F*480] float32 (C-API scale) or int16 (CLI wire format) host array.
        Returns (out like x, gr [F, active, 68] or None)."""
        n = self.active
        x, F = _host_array(x, "x", n, "active", dtypes=_PCM)
        out = np.empty_like(x)
        gr = np.empty((F, n, 68), np.float32) if want_gr else None
        self._call(_typed("pnb_process_host", x.dtype == np.int16), _ptr(x), x.shape[1], _ptr(out), x.shape[1], F,
                   _ptr(gr))
        return out, gr

    def process_stream_chunks(self, x: np.ndarray, want_gr: bool = False):
        """Any number of hops: walks x ([active, F*480]) in calls of at most max_frames hops."""
        F = x.shape[1] // FRAME
        outs, grs = [], []
        for t0 in range(0, F, self.max_frames):
            t1 = min(F, t0 + self.max_frames)
            o, g = self.process(x[:, t0 * FRAME:t1 * FRAME], want_gr)
            outs.append(o)
            grs.append(g)
        return np.concatenate(outs, axis=1), (np.concatenate(grs, axis=0) if want_gr else None)

    def process_device(self, d_in: int, in_stride: int, d_out: int, out_stride: int, n_frames: int,
                       d_gr: int = 0, stream: int = 0, int16: bool = False):
        self._call(_typed("pnb_process_device", int16), d_in, in_stride, d_out, out_stride, n_frames, d_gr, stream)

    def submit_device(self, d_in: int, in_stride: int, d_out: int, out_stride: int, n_frames: int, stream: int = 0,
                      int16: bool = False):
        """pnb_submit_device_*: process_device without g/r; flush(other_stream) or wait() orders other work behind it."""
        self._call(_typed("pnb_submit_device", int16), d_in, in_stride, d_out, out_stride, n_frames, stream)

    # ---- the network alone, on the active slots or a session list (see pnb_compute_rnn_device in the header) --------
    def _compute_rnn(self, ids, x, hops):
        a, n, label, infix = self._rows(ids)
        x, F = _host_array(x, "x", n, label, widths=(70, RECORD))
        W = x.shape[2]
        lead = () if a is None else (_ptr(a), _ptr(_hops(hops, n, F)), n)
        gr = np.empty((n, F, 68), np.float32)
        self._call(f"pnb_compute_rnn{infix}_host", *lead, RNN_FEATURES if W == 70 else RNN_RECORDS, _ptr(x), F * W, F,
                   _ptr(gr), F * 68)
        return gr

    def _compute_rnn_device(self, ids, hops, format, d_in, in_stride, n_frames, d_gr, gr_stride, stream):
        a, infix = _session_ids(ids)
        lead = () if a is None else (_ptr(a), _ptr(_hops(hops, len(a), n_frames)), len(a))
        self._call(f"pnb_compute_rnn{infix}_device", *lead, format, d_in, in_stride, n_frames, d_gr, gr_stride, stream)

    def compute_rnn(self, x: np.ndarray) -> np.ndarray:
        """pnb_compute_rnn_host: the network alone.  x: [active, F, 70] float32 features (as create_features makes them)
        or [active, F, 138] float32 training records (scaled x30 on the device like rnn_train.py's CppRawListDataset;
        the labels are ignored); the last dimension selects the format.  Advances the slots' network state by F hops
        and leaves their signal state alone.  Returns g/r [active, F, 68], hop t of row i beside record t's labels."""
        return self._compute_rnn(None, x, None)

    def compute_rnn_device(self, format: int, d_in: int, in_stride: int, n_frames: int, d_gr: int, gr_stride: int,
                           stream: int = 0):
        """pnb_compute_rnn_device on raw device pointers (format RNN_FEATURES or RNN_RECORDS; strides in floats)."""
        self._compute_rnn_device(None, None, format, d_in, in_stride, n_frames, d_gr, gr_stride, stream)

    def _frames(self, frames, what: str = "frames"):
        """frames (None, or one count per active row) as int32 or None."""
        fr = None if frames is None else _int32s(frames, what)
        if fr is not None and len(fr) != self.active:
            raise PnbError(f"{what} needs one entry per active row")
        return fr

    def score_records(self, x: np.ndarray, frames=None, want_gr: bool = False):
        """pnb_score_records_host: compute_rnn on records x ([active, F, 138] float32) with rnn_train.py's CustomLoss
        reduced on the device against their labels.  frames: None, or one count in [0, F] per row: row i's loss counts
        its first frames[i] hops (every row still advances F hops).  Returns (sums [active, 4] float64 = {sum dg^2,
        sum dg^4, sum dr^2, count} per row, as eval_records.loss_sums computes them; g/r [active, F, 68] or None)."""
        n = self.active
        x, F = _host_array(x, "x", n, "active", widths=(RECORD,))
        fr = self._frames(frames)
        sums = np.empty((n, 4), np.float64)
        gr = np.empty((n, F, 68), np.float32) if want_gr else None
        self._call("pnb_score_records_host", _ptr(x), F * RECORD, F, _ptr(fr), _ptr(sums), _ptr(gr), F * 68)
        return sums, gr

    def score_records_device(self, d_rec: int, rec_stride: int, n_frames: int, frames, d_sums: int, d_gr: int = 0,
                             gr_stride: int = 0, stream: int = 0):
        """pnb_score_records_device on raw device pointers (strides in floats); frames: None or a host sequence of one
        count per active row; d_sums: [active, 4] float64; d_gr: 0 for no g/r."""
        self._call("pnb_score_records_device", d_rec, rec_stride, n_frames, _ptr(self._frames(frames)), d_sums, d_gr,
                   gr_stride, stream)

    # ---- training (TRAIN_NETWORK engines; see pnb_train_grad_host in the header) -----------------------------------
    def train_grad(self, rec: np.ndarray, frames=None) -> np.ndarray:
        """pnb_train_grad_host: rnn_train.py's CustomLoss on the windows rec ([active, F, 138] float32 records, one window
        per row) and its gradient with respect to every parameter, kept on the engine for train_adam.  frames: None, or
        one count in [1, F] per window (its hops after that are ignored).  Returns the loss sums [active, 4] float64 as
        score_records returns them (eval_records.loss_terms of their sum gives the loss)."""
        n = self.active
        rec, F = _host_array(rec, "rec", n, "active", widths=(RECORD,))
        fr = self._frames(frames)
        sums = np.empty((n, 4), np.float64)
        self._call("pnb_train_grad_host", _ptr(rec), F * RECORD, F, _ptr(fr), _ptr(sums))
        return sums

    def train_grad_device(self, d_rec: int, rec_stride: int, n_frames: int, frames, d_sums: int, stream: int = 0):
        """pnb_train_grad_device on raw device pointers (rec_stride in floats); frames: None or a host sequence of one
        count per active row; d_sums: [active, 4] float64."""
        self._call("pnb_train_grad_device", d_rec, rec_stride, n_frames, _ptr(self._frames(frames)), d_sums, stream)

    def train_forward_device(self, d_x: int, x_stride: int, n_frames: int, d_weights: int, d_out: int, out_stride: int,
                             stream: int = 0):
        """pnb_train_forward_device on raw device pointers (strides in floats): features [active, n_frames, 70] (not
        scaled) through the trainer's forward into g/r [active, n_frames, 68]; d_weights: 0, or N_PARAMS floats in blob
        order that replace the weights first.  Its backward (train_backward_device) is then due."""
        self._call("pnb_train_forward_device", d_x, x_stride, n_frames, d_weights, d_out, out_stride, stream)

    def train_backward_device(self, d_dout: int, dout_stride: int, d_dx: int = 0, dx_stride: int = 0, d_grad: int = 0,
                              stream: int = 0):
        """pnb_train_backward_device on raw device pointers (strides in floats): dL/d(out) of the last
        train_forward_device in; dL/dx (d_dx, or 0 for none) and the blob-order gradient (d_grad, or 0) out.  The
        gradient is also the held one, for train_adam / train_accumulate."""
        self._call("pnb_train_backward_device", d_dout, dout_stride, d_dx, dx_stride, d_grad, stream)

    def train_forward_state_device(self, d_x: int, x_stride: int, n_frames: int, lengths=None, d_weights: int = 0,
                                   d_state_in: int = 0, state_in_stride: int = TRAIN_STATE_FLOATS, d_out: int = 0,
                                   out_stride: int = 0, d_state_out: int = 0,
                                   state_out_stride: int = TRAIN_STATE_FLOATS, stream: int = 0):
        """pnb_train_forward_state_device on raw device pointers (strides in floats): train_forward_device from the
        state rows d_state_in (0: zero state), the state at each window's end out to d_state_out (0: none); lengths: None,
        or a host sequence of one hop count in [1, n_frames] per active row."""
        self._call("pnb_train_forward_state_device", d_x, x_stride, n_frames, _ptr(self._frames(lengths, "lengths")),
                   d_weights, d_state_in, state_in_stride, d_out, out_stride, d_state_out, state_out_stride, stream)

    def train_backward_state_device(self, d_dout: int, dout_stride: int, d_dstate_out: int = 0,
                                    dstate_out_stride: int = TRAIN_STATE_FLOATS, d_dx: int = 0, dx_stride: int = 0,
                                    d_dstate_in: int = 0, dstate_in_stride: int = TRAIN_STATE_FLOATS, d_grad: int = 0,
                                    stream: int = 0):
        """pnb_train_backward_state_device on raw device pointers (strides in floats): train_backward_device with
        dL/d(state out) in (d_dstate_out, or 0 for none) and dL/d(state in) out (d_dstate_in, or 0 for none)."""
        self._call("pnb_train_backward_state_device", d_dout, dout_stride, d_dstate_out, dstate_out_stride, d_dx,
                   dx_stride, d_dstate_in, dstate_in_stride, d_grad, stream)

    def train_adam(self, lr: float, step: int, stream: int = 0):
        """pnb_train_adam: one torch.optim.Adam step (defaults) with the gradient of the last train_grad; step counts
        from 1.  Skipped on the device when that gradient was not finite."""
        self._call("pnb_train_adam", float(lr), int(step), stream)

    def train_accumulate(self, stream: int = 0):
        """pnb_train_accumulate: the gradient of the last gradient call or backward, weighted by the hops it counted, into
        the engine's float64 accumulator (micro-batches and ranks summed before one train_adam)."""
        self._call("pnb_train_accumulate", stream)

    def train_finish(self, stream: int = 0):
        """pnb_train_finish: the accumulated batch's gradient (sum c_k g_k / sum c_k) becomes the held gradient for
        train_adam, and the accumulator is emptied."""
        self._call("pnb_train_finish", stream)

    def train_export(self, what: str) -> np.ndarray:
        """pnb_train_export: 'weights', 'gradient', 'm' or 'v' as one float32 vector in PNBW blob order
        (weights.PackedModel.from_flat turns it into a model), or 'accum', the accumulator's N + 1 float64 values."""
        from .weights import N_PARAMS
        a = np.empty(N_PARAMS + 1, np.float64) if what == "accum" else np.empty(N_PARAMS, np.float32)
        self.train_export_ptr(what, _ptr(a), a.nbytes)
        return a

    def train_import(self, what: str, a: np.ndarray):
        """pnb_train_import: 'weights', 'm' or 'v' from a flat float32 vector in PNBW blob order (resuming a run), or
        'accum' from N + 1 float64 values (a sum of several engines' accumulators)."""
        a = np.ascontiguousarray(a, np.float64 if what == "accum" else np.float32)
        self.train_import_ptr(what, _ptr(a), a.nbytes)

    def train_export_ptr(self, what: str, ptr: int, nbytes: int):
        """pnb_train_export into raw memory: 'accum' may be device memory of the engine's device (a torch CUDA tensor's
        data_ptr(), N + 1 float64), the other arrays host memory.  Returns when the copy is complete."""
        self._call("pnb_train_export", TRAIN_ARRAYS[what], ptr, nbytes)

    def train_import_ptr(self, what: str, ptr: int, nbytes: int):
        """pnb_train_import from raw memory, as train_export_ptr."""
        self._call("pnb_train_import", TRAIN_ARRAYS[what], ptr, nbytes)

    # ---- the signal path without the network, on the active slots or a session list (see pnb_analyze_host_f32) -------
    def _analyze(self, ids, x, hops):
        a, n, label, infix = self._rows(ids)
        x, F = _host_array(x, "x", n, label, dtypes=_PCM)
        lead = () if a is None else (_ptr(a), _ptr(_hops(hops, n, F)), n)
        feat = np.empty((n, F, 70), np.float32)
        self._call(_typed(f"pnb_analyze{infix}_host", x.dtype == np.int16), *lead, _ptr(x), x.shape[1], F, _ptr(feat),
                   F * 70)
        return feat

    def _analyze_device(self, ids, hops, d_in, in_stride, n_frames, d_feat, feat_stride, stream, int16):
        a, infix = _session_ids(ids)
        lead = () if a is None else (_ptr(a), _ptr(_hops(hops, len(a), n_frames)), len(a))
        self._call(_typed(f"pnb_analyze{infix}_device", int16), *lead, d_in, in_stride, n_frames, d_feat, feat_stride,
                   stream)

    def _synthesize(self, ids, gr, int16):
        a, n, label, infix = self._rows(ids)
        gr, F = _host_array(gr, "gr", n, label, widths=(68,))
        lead = () if a is None else (_ptr(a), n)
        out = np.empty((n, F * FRAME), np.int16 if int16 else np.float32)
        self._call(_typed(f"pnb_synthesize{infix}_host", int16), *lead, _ptr(gr), F * 68, F, _ptr(out), F * FRAME)
        return out

    def _synthesize_device(self, ids, d_gr, gr_stride, n_frames, d_out, out_stride, stream, int16):
        a, infix = _session_ids(ids)
        lead = () if a is None else (_ptr(a), len(a))
        self._call(_typed(f"pnb_synthesize{infix}_device", int16), *lead, d_gr, gr_stride, n_frames, d_out, out_stride,
                   stream)

    def analyze(self, x: np.ndarray) -> np.ndarray:
        """pnb_analyze_host_*: the analysis half of process.  x: [active, F*480] float32 (C-API scale) or int16 (CLI wire
        format).  Returns the network input [active, F, 70] float32 (the features tap of a process call on x) and leaves
        a synthesis of F hops pending: the next call must be synthesize (or compute_rnn, or reset)."""
        return self._analyze(None, x, None)

    def synthesize(self, gr: np.ndarray, int16: bool = False) -> np.ndarray:
        """pnb_synthesize_host_*: the synthesis half of process, with the caller's gains.  gr: [active, F, 68] float32
        (34 g then 34 r per hop), F the hops of the pending analysis.  Returns [active, F*480] float32, or int16 with
        the CLI's conversion."""
        return self._synthesize(None, gr, int16)

    def analyze_device(self, d_in: int, in_stride: int, n_frames: int, d_feat: int, feat_stride: int, stream: int = 0,
                       int16: bool = False):
        """pnb_analyze_device_* on raw device pointers (strides in elements)."""
        self._analyze_device(None, None, d_in, in_stride, n_frames, d_feat, feat_stride, stream, int16)

    def synthesize_device(self, d_gr: int, gr_stride: int, n_frames: int, d_out: int, out_stride: int, stream: int = 0,
                          int16: bool = False):
        """pnb_synthesize_device_* on raw device pointers (strides in elements)."""
        self._synthesize_device(None, d_gr, gr_stride, n_frames, d_out, out_stride, stream, int16)

    def synthesis_operands_device(self, d_ops: int, ops_stride: int, stream: int = 0):
        """pnb_synthesis_operands_device: the operands of the pending synthesis, [active, F, SYNTH_OPS_FLOATS] at d_ops
        (ops_stride in floats); the synthesis stays pending."""
        self._call("pnb_synthesis_operands_device", d_ops, ops_stride, stream)

    @property
    def device_bytes(self) -> int:
        """pnb_engine_bytes: the engine's fixed-size device buffers, in bytes."""
        return int(self.L.pnb_engine_bytes(self.h))

    def flush(self, stream: int = 0):
        self._call("pnb_flush", stream)

    def submit(self, x: np.ndarray, out: np.ndarray):
        """Pipelined host call (pnb_submit_host_*): returns at once; x/out ([active, F*480] float32 or int16, ideally
        pinned) must stay alive until wait()."""
        if x.shape != out.shape or x.dtype != out.dtype:
            raise PnbError("submit: x and out must have the same shape and dtype")
        n = self.active
        x, F = _host_array(x, "x", n, "active", dtypes=_PCM, copy=False)
        out, _ = _host_array(out, "out", n, "active", dtypes=_PCM, copy=False)
        self._call(_typed("pnb_submit_host", x.dtype == np.int16), _ptr(x), x.strides[0] // x.itemsize, _ptr(out),
                   out.strides[0] // out.itemsize, F)

    def wait(self):
        self._call("pnb_wait")

    def check(self, stream: int = 0):
        """pnb_check: waits for the engine's work (and `stream`) and raises on PNB_ERR_DOMAIN / PNB_ERR_CUDA."""
        self._call("pnb_check", stream)

    def _read_tap(self, tap, *rows) -> np.ndarray:
        """One tap (code, dtype, width) into a new [*rows, width] array."""
        code, dt, width = tap
        a = np.empty((*rows, width), dt)
        self._call("pnb_read_tap", code, _ptr(a), a.nbytes)
        return a

    def read_tap(self, name: str, n_frames: int, rows: int = None) -> np.ndarray:
        """pnb_read_tap: [n_frames][rows][width], rows n_streams by default; the train_* taps of a train_grad call
        take that call's active rows."""
        return self._read_tap(TAPS[name], n_frames, self.n_streams if rows is None else rows)

    def get_state(self, stream: int) -> bytes:
        buf = C.create_string_buffer(self.L.pnb_state_size())
        self._call("pnb_get_state", stream, buf, len(buf))
        return buf.raw

    def set_state(self, stream: int, blob: bytes):
        self._call("pnb_set_state", stream, blob, len(blob))

    # ---- batched stream recycling, on slots or sessions (asynchronous on `stream`; see pnb_reset_streams) -----------
    @property
    def state_size(self) -> int:
        return int(self.L.pnb_state_size())

    def _reset_rows(self, name, idx, what, stream):
        a = _int32s(idx, what)
        self._call(name, _ptr(a), len(a), stream)

    def _export_rows(self, name, idx, what, d_blobs, stride, stream):
        a = _int32s(idx, what)
        out = None
        if d_blobs is None:
            import torch
            out = torch.empty((len(a), self.state_size), dtype=torch.uint8, device=f"cuda:{self.device}")
            d_blobs, stride = out.data_ptr(), self.state_size
        self._call(name, _ptr(a), len(a), d_blobs, stride or self.state_size, stream)
        return out

    def _import_rows(self, name, idx, what, d_blobs, stride, stream):
        a = _int32s(idx, what)
        if not isinstance(d_blobs, int) and d_blobs is not None:
            t = d_blobs
            if t.dtype.itemsize != 1 or t.dim() != 2 or t.shape[0] != len(a) or t.stride(1) != 1 or not t.is_cuda:
                raise PnbError(f"{name}: blobs must be a CUDA byte tensor [len({what}), pnb_state_size()] with "
                               "contiguous rows")
            d_blobs, stride = t.data_ptr(), t.stride(0)
        self._call(name, _ptr(a), len(a), d_blobs, stride or self.state_size, stream)

    def reset_streams(self, idx, stream: int = 0):
        """pnb_reset_streams: the slots in `idx` start over as fresh streams; the others are untouched."""
        self._reset_rows("pnb_reset_streams", idx, "idx", stream)

    def export_states(self, idx, d_blobs, stride: int = 0, stream: int = 0):
        """pnb_export_states.  d_blobs: a raw device pointer (blob i at d_blobs + i*stride, stride 0 = pnb_state_size()),
        or None to get a new CUDA uint8 torch tensor [len(idx), pnb_state_size()] back."""
        return self._export_rows("pnb_export_states", idx, "idx", d_blobs, stride, stream)

    def import_states(self, idx, d_blobs, stride: int = 0, stream: int = 0):
        """pnb_import_states.  d_blobs: a raw device pointer (as export_states) or a CUDA uint8 tensor
        [len(idx), >= pnb_state_size()] whose rows are blobs; the tensor must stay alive until `stream` has run the import."""
        self._import_rows("pnb_import_states", idx, "idx", d_blobs, stride, stream)

    # ---- session pool (see pnb_sessions_reserve in the header) ---------------------------------------------------------
    def reserve_sessions(self, n_sessions: int):
        """pnb_sessions_reserve: session mode with sessions [0, n_sessions), all fresh (the first call resets the engine);
        a later, larger call grows the pool and keeps every session's state."""
        self._call("pnb_sessions_reserve", n_sessions)

    def process_sessions(self, ids, x: np.ndarray, want_gr: bool = False, hops=None):
        """pnb_process_sessions_host_*: advances exactly the listed sessions.  x: [len(ids), F*480] float32 or int16 host
        array, row i for ids[i].  Returns (out like x, gr [F, len(ids), 68] or None).
        hops: None, or one hop count per session (pnb_process_sessions_ragged_host_*): session ids[i] advances by
        hops[i], F = max(hops) must be x's width in hops, and row i of out / gr[:, i] is zero after hops[i] hops."""
        a = _int32s(ids, "ids")
        n = len(a)
        x, F = _host_array(x, "x", n, "len(ids)", dtypes=_PCM)
        hp = _hops(hops, n, F)
        out = np.empty_like(x)
        gr = np.empty((F, n, 68), np.float32) if want_gr else None
        i16, pcm = x.dtype == np.int16, (_ptr(x), x.shape[1], _ptr(out), x.shape[1])
        if hp is None:
            self._call(_typed("pnb_process_sessions_host", i16), _ptr(a), n, *pcm, F, _ptr(gr))
        else:
            self._call(_typed("pnb_process_sessions_ragged_host", i16), _ptr(a), _ptr(hp), n, *pcm, _ptr(gr))
        return out, gr

    def process_sessions_device(self, ids, d_in: int, in_stride: int, d_out: int, out_stride: int, n_frames: int = 0,
                                d_gr: int = 0, stream: int = 0, int16: bool = False, hops=None):
        """pnb_process_sessions_device_*: raw device pointers, row i of in / out and d_gr[t][i] for ids[i].
        hops: None, or one hop count per session (pnb_process_sessions_ragged_device_*; n_frames is then max(hops) and
        need not be given)."""
        a = _int32s(ids, "ids")
        hp = _hops(hops, len(a), n_frames or None)
        if hp is None:
            self._call(_typed("pnb_process_sessions_device", int16), _ptr(a), len(a), d_in, in_stride, d_out,
                       out_stride, n_frames, d_gr, stream)
        else:
            self._call(_typed("pnb_process_sessions_ragged_device", int16), _ptr(a), _ptr(hp), len(a), d_in, in_stride,
                       d_out, out_stride, d_gr, stream)

    def reset_sessions(self, ids, stream: int = 0):
        """pnb_reset_sessions: the listed sessions start over as fresh streams."""
        self._reset_rows("pnb_reset_sessions", ids, "ids", stream)

    def export_sessions(self, ids, d_blobs, stride: int = 0, stream: int = 0):
        """pnb_export_sessions, with the conventions of export_states (None: returns a new CUDA uint8 tensor)."""
        return self._export_rows("pnb_export_sessions", ids, "ids", d_blobs, stride, stream)

    def import_sessions(self, ids, d_blobs, stride: int = 0, stream: int = 0):
        """pnb_import_sessions, with the conventions of import_states (a raw pointer or a CUDA uint8 tensor of blob rows)."""
        self._import_rows("pnb_import_sessions", ids, "ids", d_blobs, stride, stream)

    def session_stats(self) -> dict:
        """pnb_session_stats: cumulative {parks, unparks, relocations} of the session pool."""
        c = (C.c_longlong * 3)()
        self._call("pnb_session_stats", c)
        return {"parks": int(c[0]), "unparks": int(c[1]), "relocations": int(c[2])}

    # ---- split and network calls on a session list (see pnb_analyze_sessions_device_f32 in the header) ---------------
    def analyze_sessions(self, ids, x: np.ndarray, hops=None) -> np.ndarray:
        """pnb_analyze_sessions_host_*: the analysis half of process_sessions.  x: [len(ids), F*480] float32 or int16, row
        i for ids[i]; hops: None or one count per session (ragged, F = max(hops)).  Returns the features [len(ids), F, 70]
        (zero after a session's own hops) and leaves a synthesis pending: synthesize_sessions with the same ids next (or
        compute_rnn_sessions on them, or reset)."""
        return self._analyze(ids, x, hops)

    def synthesize_sessions(self, ids, gr: np.ndarray, int16: bool = False) -> np.ndarray:
        """pnb_synthesize_sessions_host_*: the synthesis half, on the pending list (same ids, same order).  gr:
        [len(ids), F, 68] float32, read for each session's own hops.  Returns [len(ids), F*480] float32 (or int16): a
        session's hops of output, then zeros."""
        return self._synthesize(ids, gr, int16)

    def compute_rnn_sessions(self, ids, x: np.ndarray, hops=None) -> np.ndarray:
        """pnb_compute_rnn_sessions_host: compute_rnn on the listed sessions.  x: [len(ids), F, 70 | 138] float32 (the
        last dimension selects the format); hops: None or one count per session (F = max(hops)).  Returns g/r
        [len(ids), F, 68], zero after a session's own hops.  Between the halves of a session split it must list the
        pending sessions, hops and F."""
        return self._compute_rnn(ids, x, hops)

    def analyze_sessions_device(self, ids, d_in: int, in_stride: int, n_frames: int, d_feat: int, feat_stride: int,
                                stream: int = 0, int16: bool = False, hops=None):
        """pnb_analyze_sessions_device_* on raw device pointers (strides in elements); hops: None or one count per
        session, with n_frames = max(hops)."""
        self._analyze_device(ids, hops, d_in, in_stride, n_frames, d_feat, feat_stride, stream, int16)

    def synthesize_sessions_device(self, ids, d_gr: int, gr_stride: int, n_frames: int, d_out: int, out_stride: int,
                                   stream: int = 0, int16: bool = False):
        """pnb_synthesize_sessions_device_* on raw device pointers (strides in elements)."""
        self._synthesize_device(ids, d_gr, gr_stride, n_frames, d_out, out_stride, stream, int16)

    def compute_rnn_sessions_device(self, ids, format: int, d_in: int, in_stride: int, n_frames: int, d_gr: int,
                                    gr_stride: int, stream: int = 0, hops=None):
        """pnb_compute_rnn_sessions_device on raw device pointers (format RNN_FEATURES or RNN_RECORDS; strides in floats)."""
        self._compute_rnn_device(ids, hops, format, d_in, in_stride, n_frames, d_gr, gr_stride, stream)

    def read_nn_state(self) -> dict:
        """fp32 network state after the last hop: conv2 output and the five GRU states, [S, width]."""
        return {name: self._read_tap(tap, self.n_streams) for name, tap in _NN_STATE.items()}

    # ---- training-data generator (TRAIN_DATA engines; see pnb_train_records_host in the header) ----------------------
    def _train_data(self, name, speech, noisy, with_audio):
        N = self.n_streams // 2
        if speech.shape != noisy.shape:
            raise PnbError(f"{name}: speech and noisy must have the same shape")
        speech, F = _host_array(speech, "speech", N, "n_pairs", dtypes=(np.int16,))
        noisy, _ = _host_array(noisy, "noisy", N, "n_pairs", dtypes=(np.int16,))
        rec = np.empty((N, F, RECORD), np.float32)
        audio = np.empty((N, F * FRAME), np.int16) if with_audio else None
        self._call(name, _ptr(speech), speech.shape[1], _ptr(noisy), noisy.shape[1], F, _ptr(rec), F * RECORD,
                   *((_ptr(audio), F * FRAME) if with_audio else ()))
        return rec, audio

    def train_records(self, speech: np.ndarray, noisy: np.ndarray) -> np.ndarray:
        """speech, noisy: [n_pairs, F*480] int16 -> [n_pairs, F, 138] float32, the records the reference's train()
        (src/denoise.cpp:600-787) writes for each pair of files.  Engine must have flags=TRAIN_DATA and
        n_streams = 2*n_pairs; state carries over, so call repeatedly with consecutive chunks."""
        return self._train_data("pnb_train_records_host", speech, noisy, False)[0]

    def train_records_device(self, d_speech: int, speech_stride: int, d_noisy: int, noisy_stride: int, n_frames: int,
                             d_records: int, records_stride: int, stream: int = 0):
        self._call("pnb_train_records_device", d_speech, speech_stride, d_noisy, noisy_stride, n_frames, d_records,
                   records_stride, stream)

    def train_audio(self, speech: np.ndarray, noisy: np.ndarray):
        """speech, noisy: [n_pairs, F*480] int16 -> (records [n_pairs, F, 138] float32, audio [n_pairs, F*480] int16):
        the records of train_records and, for each pair, what the reference's train() writes to test_output.pcm over
        these frames (src/denoise.cpp:742-759: the noisy file resynthesised with its own labels, clamped to int16).
        Engine must have flags=TRAIN_DATA | TRAIN_AUDIO; state carries over, so call repeatedly with consecutive chunks."""
        return self._train_data("pnb_train_audio_host", speech, noisy, True)

    def train_audio_device(self, d_speech: int, speech_stride: int, d_noisy: int, noisy_stride: int, n_frames: int,
                           d_records: int, records_stride: int, d_audio: int, audio_stride: int, stream: int = 0):
        self._call("pnb_train_audio_device", d_speech, speech_stride, d_noisy, noisy_stride, n_frames, d_records,
                   records_stride, d_audio, audio_stride, stream)

    def profile(self, on: bool):
        self._call("pnb_profile_enable", 1 if on else 0)

    def profile_read(self) -> dict:
        """{kernel class name: (total ms, launches)} since the last read; waits for the device."""
        n = 10
        ms = (C.c_double * n)()
        cnt = (C.c_longlong * n)()
        self._call("pnb_profile_read", ms, cnt)
        return {self.L.pnb_kernel_class_name(k).decode(): (ms[k], int(cnt[k])) for k in range(n) if cnt[k]}

    def profile_timeline(self, cap: int = 4096):
        """[(class name, start ms, end ms)] of every launch since profiling was enabled / last read."""
        cls = (C.c_int * cap)()
        t0 = (C.c_double * cap)()
        t1 = (C.c_double * cap)()
        n = self._call("pnb_profile_timeline", cls, t0, t1, cap)
        return [(self.L.pnb_kernel_class_name(cls[k]).decode(), t0[k], t1[k]) for k in range(n)]

    def overlap_info(self) -> dict:
        """Every call runs its kernels one after the other on all SMs; no SM partition exists.  Kept as this constant
        because bench.py reports it as the schedule."""
        return {"net_sms": 0, "dsp_sms": 0, "chunk_hops": 0}

    @property
    def launches(self) -> int:
        return int(self.L.pnb_launch_count(self.h))

    def launches_per_call(self, n_frames: int) -> int:
        return int(self.L.pnb_launches_per_call(self.h, n_frames))
