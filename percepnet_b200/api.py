"""Python host mirror of the C-ABI in include/percepnet_b200.h (ctypes; no compute here).

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
TRAIN_ARRAYS = {"weights": 0, "gradient": 1, "m": 2, "v": 3}   # pnb_train_export / pnb_train_import
RECORD = 138
RNN_FEATURES, RNN_RECORDS = 0, 1   # pnb_compute_rnn_* formats: 70 features or 138 record floats per hop
TAPS = {"features": (0, np.float32, 70), "pitch": (1, np.int32, 4), "pitchf": (2, np.float32, 2),
        "X": (3, np.float32, 800), "P": (4, np.float32, 800), "Ex": (5, np.float32, 34), "gr": (6, np.float32, 68),
        "g_used": (13, np.float32, 34)}

_lib = None


class PnbError(RuntimeError):
    pass


def load_library() -> C.CDLL:
    """dlopen the in-tree CUDA library; raises if it has not been built (no fallback)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise PnbError(f"{LIB_PATH} is missing: run `python -c 'import __graft_entry__ as g; g.build()'` "
                       "(nvcc, sm_90a).  There is no CPU implementation to fall back to.")
    L = C.CDLL(LIB_PATH)
    vp, sz, i = C.c_void_p, C.c_size_t, C.c_int
    L.pnb_create.argtypes = [C.POINTER(vp), i, i, vp, C.c_uint, i]
    L.pnb_model_load_blob.argtypes = [C.c_char_p, C.POINTER(vp)]
    L.pnb_model_free.argtypes = [vp]
    L.pnb_model_free.restype = None
    L.pnb_train_records_host.argtypes = [vp, vp, sz, vp, sz, i, vp, sz]
    L.pnb_submit_train_records.argtypes = [vp, vp, sz, vp, sz, i, vp, sz]
    L.pnb_train_records_device.argtypes = [vp, vp, sz, vp, sz, i, vp, sz, vp]
    L.pnb_train_audio_host.argtypes = [vp, vp, sz, vp, sz, i, vp, sz, vp, sz]
    L.pnb_train_audio_device.argtypes = [vp, vp, sz, vp, sz, i, vp, sz, vp, sz, vp]
    L.pnb_destroy.argtypes = [vp]
    L.pnb_destroy.restype = None
    L.pnb_reset.argtypes = [vp]
    L.pnb_resolve_device.argtypes = [i]
    L.pnb_process_host_f32.argtypes = [vp, vp, sz, vp, sz, i, vp]
    L.pnb_process_host_i16.argtypes = [vp, vp, sz, vp, sz, i, vp]
    L.pnb_process_device_f32.argtypes = [vp, vp, sz, vp, sz, i, vp, vp]
    L.pnb_process_device_i16.argtypes = [vp, vp, sz, vp, sz, i, vp, vp]
    L.pnb_submit_host_f32.argtypes = [vp, vp, sz, vp, sz, i]
    L.pnb_submit_host_i16.argtypes = [vp, vp, sz, vp, sz, i]
    L.pnb_submit_device_f32.argtypes = [vp, vp, sz, vp, sz, i, vp]
    L.pnb_submit_device_i16.argtypes = [vp, vp, sz, vp, sz, i, vp]
    L.pnb_compute_rnn_device.argtypes = [vp, i, vp, sz, i, vp, sz, vp]
    L.pnb_compute_rnn_host.argtypes = [vp, i, vp, sz, i, vp, sz]
    L.pnb_score_records_device.argtypes = [vp, vp, sz, i, vp, vp, vp, sz, vp]
    L.pnb_score_records_host.argtypes = [vp, vp, sz, i, vp, vp, vp, sz]
    for name in ("pnb_analyze_host_f32", "pnb_analyze_host_i16", "pnb_synthesize_host_f32", "pnb_synthesize_host_i16"):
        getattr(L, name).argtypes = [vp, vp, sz, i, vp, sz]
    for name in ("pnb_analyze_device_f32", "pnb_analyze_device_i16", "pnb_synthesize_device_f32", "pnb_synthesize_device_i16"):
        getattr(L, name).argtypes = [vp, vp, sz, i, vp, sz, vp]
    L.pnb_train_grad_host.argtypes = [vp, vp, sz, i, vp, vp]
    L.pnb_train_grad_device.argtypes = [vp, vp, sz, i, vp, vp, vp]
    L.pnb_train_adam.argtypes = [vp, C.c_double, C.c_longlong, vp]
    L.pnb_train_export.argtypes = [vp, i, vp, sz]
    L.pnb_train_import.argtypes = [vp, i, vp, sz]
    L.pnb_engine_bytes.argtypes = [vp]
    L.pnb_engine_bytes.restype = sz
    L.pnb_flush.argtypes = [vp, vp]
    L.pnb_wait.argtypes = [vp]
    L.pnb_check.argtypes = [vp, vp]
    L.pnb_read_tap.argtypes = [vp, i, vp, sz]
    L.pnb_state_size.restype = sz
    L.pnb_get_state.argtypes = [vp, i, vp, sz]
    L.pnb_set_state.argtypes = [vp, i, vp, sz]
    L.pnb_reset_streams.argtypes = [vp, vp, i, vp]
    L.pnb_export_states.argtypes = [vp, vp, i, vp, sz, vp]
    L.pnb_import_states.argtypes = [vp, vp, i, vp, sz, vp]
    L.pnb_set_active_streams.argtypes = [vp, i, vp]
    L.pnb_active_streams.argtypes = [vp]
    L.pnb_sessions_reserve.argtypes = [vp, i]
    L.pnb_process_sessions_device_f32.argtypes = [vp, vp, i, vp, sz, vp, sz, i, vp, vp]
    L.pnb_process_sessions_device_i16.argtypes = [vp, vp, i, vp, sz, vp, sz, i, vp, vp]
    L.pnb_process_sessions_host_f32.argtypes = [vp, vp, i, vp, sz, vp, sz, i, vp]
    L.pnb_process_sessions_host_i16.argtypes = [vp, vp, i, vp, sz, vp, sz, i, vp]
    L.pnb_process_sessions_ragged_device_f32.argtypes = [vp, vp, vp, i, vp, sz, vp, sz, vp, vp]
    L.pnb_process_sessions_ragged_device_i16.argtypes = [vp, vp, vp, i, vp, sz, vp, sz, vp, vp]
    L.pnb_process_sessions_ragged_host_f32.argtypes = [vp, vp, vp, i, vp, sz, vp, sz, vp]
    L.pnb_process_sessions_ragged_host_i16.argtypes = [vp, vp, vp, i, vp, sz, vp, sz, vp]
    L.pnb_reset_sessions.argtypes = [vp, vp, i, vp]
    L.pnb_export_sessions.argtypes = [vp, vp, i, vp, sz, vp]
    L.pnb_import_sessions.argtypes = [vp, vp, i, vp, sz, vp]
    L.pnb_session_stats.argtypes = [vp, vp]
    L.pnb_pitch_only_device.argtypes = [vp, sz, C.c_longlong, vp, vp, vp, vp, vp, vp, vp]
    L.pnb_pitch_only_host.argtypes = [vp, sz, C.c_longlong, vp, vp, vp, vp, vp, vp]
    L.pnb_launch_count.argtypes = [vp]
    L.pnb_launch_count.restype = C.c_longlong
    L.pnb_launches_per_call.argtypes = [vp, i]
    L.pnb_n_streams.argtypes = [vp]
    L.pnb_max_frames.argtypes = [vp]
    L.pnb_profile_enable.argtypes = [vp, i]
    L.pnb_profile_read.argtypes = [vp, vp, vp]
    L.pnb_profile_timeline.argtypes = [vp, vp, vp, vp, i]
    L.pnb_kernel_class_name.argtypes = [i]
    L.pnb_kernel_class_name.restype = C.c_char_p
    L.pnb_last_error.restype = C.c_char_p
    L.pnb_version.restype = C.c_char_p
    _lib = L
    return L


EXPORTS = ("pnb_create", "pnb_destroy", "pnb_reset", "pnb_resolve_device", "pnb_process_host_f32", "pnb_process_host_i16",
           "pnb_model_load_blob", "pnb_model_load_stream", "pnb_model_free", "pnb_train_records_host", "pnb_train_records_device", "pnb_submit_train_records", "pnb_train_audio_host", "pnb_train_audio_device", "pnb_process_device_f32", "pnb_process_device_i16", "pnb_submit_host_f32", "pnb_submit_host_i16", "pnb_submit_device_f32", "pnb_submit_device_i16", "pnb_flush", "pnb_wait", "pnb_check",
           "pnb_compute_rnn_device", "pnb_compute_rnn_host", "pnb_score_records_device", "pnb_score_records_host",
           "pnb_analyze_host_f32", "pnb_analyze_host_i16", "pnb_analyze_device_f32", "pnb_analyze_device_i16",
           "pnb_synthesize_host_f32", "pnb_synthesize_host_i16", "pnb_synthesize_device_f32", "pnb_synthesize_device_i16",
           "pnb_train_grad_host", "pnb_train_grad_device", "pnb_train_adam", "pnb_train_export", "pnb_train_import",
           "pnb_engine_bytes",
           "pnb_read_tap", "pnb_state_size", "pnb_get_state", "pnb_set_state",
           "pnb_reset_streams", "pnb_export_states", "pnb_import_states", "pnb_set_active_streams", "pnb_active_streams",
           "pnb_sessions_reserve", "pnb_process_sessions_device_f32", "pnb_process_sessions_device_i16",
           "pnb_process_sessions_host_f32", "pnb_process_sessions_host_i16", "pnb_process_sessions_ragged_device_f32",
           "pnb_process_sessions_ragged_device_i16", "pnb_process_sessions_ragged_host_f32",
           "pnb_process_sessions_ragged_host_i16", "pnb_reset_sessions", "pnb_export_sessions",
           "pnb_import_sessions", "pnb_session_stats", "pnb_pitch_only_device", "pnb_pitch_only_host", "pnb_launch_count",
           "pnb_launches_per_call", "pnb_profile_enable", "pnb_profile_read", "pnb_profile_timeline", "pnb_kernel_class_name", "pnb_n_streams", "pnb_max_frames", "pnb_last_error", "pnb_version")


def pitch_only_device(d_buf: int, stride: int, n_units: int, d_period: int, d_corr: int, d_gain: int, d_lag: int = 0,
                      d_prev_period: int = 0, d_prev_gain: int = 0, stream: int = 0):
    """pnb_pitch_only_device on raw device pointers (BASELINE.json config 5: the pitch analysis alone)."""
    L = load_library()
    rc = L.pnb_pitch_only_device(d_buf, stride, n_units, d_prev_period or None, d_prev_gain or None, d_period, d_corr,
                                 d_gain, d_lag or None, stream or None)
    if rc != 0:
        raise PnbError(f"pnb_pitch_only_device failed ({rc}): {L.pnb_last_error().decode()}")


def pitch_only(bufs: np.ndarray, prev_period=None, prev_gain=None):
    """pnb_pitch_only_host: [n, 1728] float32 pitch buffers -> (period int32 [n], corr [n], gain [n], lag int32 [n])"""
    L = load_library()
    b = np.ascontiguousarray(bufs, np.float32)
    n = b.shape[0]
    T, lag = np.empty(n, np.int32), np.empty(n, np.int32)
    corr, gain = np.empty(n, np.float32), np.empty(n, np.float32)
    pp = None if prev_period is None else np.ascontiguousarray(prev_period, np.int32)
    pg = None if prev_gain is None else np.ascontiguousarray(prev_gain, np.float32)
    rc = L.pnb_pitch_only_host(b.ctypes.data, b.shape[1], n, None if pp is None else pp.ctypes.data,
                               None if pg is None else pg.ctypes.data, T.ctypes.data, corr.ctypes.data, gain.ctypes.data,
                               lag.ctypes.data)
    if rc != 0:
        raise PnbError(f"pnb_pitch_only_host failed ({rc}): {L.pnb_last_error().decode()}")
    return T, corr, gain, lag


class BlobModel:
    """A model read from a binary weight file by the C loader (pnb_model_load_blob)."""

    def __init__(self, path: str):
        self.L = load_library()
        self.ptr = C.c_void_p()
        rc = self.L.pnb_model_load_blob(path.encode(), C.byref(self.ptr))
        if rc != 0:
            raise PnbError(f"pnb_model_load_blob failed ({rc}): {self.L.pnb_last_error().decode()}")

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
        rc = self.L.pnb_create(C.byref(h), n_streams, max_frames, mptr, flags, device)
        if rc != 0:
            raise PnbError(f"pnb_create failed ({rc}): {self.L.pnb_last_error().decode()}")
        self.h = h

    def _ck(self, rc, what):
        if rc != 0:
            raise PnbError(f"{what} failed ({rc}): {self.L.pnb_last_error().decode()}")

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
        self._ck(self.L.pnb_reset(self.h), "pnb_reset")

    @property
    def active(self) -> int:
        """Streams the next call advances: slots [0, active) (pnb_active_streams; n_streams unless set_active changed it)."""
        return int(self.L.pnb_active_streams(self.h))

    def set_active(self, n: int, stream: int = 0):
        """pnb_set_active_streams: later calls advance slots [0, n) only.  Slots entering the range start as fresh streams
        (reset asynchronously on `stream`); slots leaving it lose their state."""
        self._ck(self.L.pnb_set_active_streams(self.h, n, stream or None), "pnb_set_active_streams")

    def process(self, x: np.ndarray, want_gr: bool = False):
        """x: [active, F*480] float32 (C-API scale) or int16 (CLI wire format) host array.
        Returns (out like x, gr [F, active, 68] or None)."""
        n = self.active
        assert x.ndim == 2 and x.shape[0] == n and x.shape[1] % FRAME == 0
        F = x.shape[1] // FRAME
        x = np.ascontiguousarray(x)
        out = np.empty_like(x)
        gr = np.empty((F, n, 68), np.float32) if want_gr else None
        grp = gr.ctypes.data if want_gr else None
        if x.dtype == np.float32:
            rc = self.L.pnb_process_host_f32(self.h, x.ctypes.data, x.shape[1], out.ctypes.data, x.shape[1], F, grp)
        elif x.dtype == np.int16:
            rc = self.L.pnb_process_host_i16(self.h, x.ctypes.data, x.shape[1], out.ctypes.data, x.shape[1], F, grp)
        else:
            raise TypeError("x must be float32 or int16")
        self._ck(rc, "pnb_process_host")
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
        f = self.L.pnb_process_device_i16 if int16 else self.L.pnb_process_device_f32
        self._ck(f(self.h, d_in, in_stride, d_out, out_stride, n_frames, d_gr or None, stream or None),
                 "pnb_process_device")

    def submit_device(self, d_in: int, in_stride: int, d_out: int, out_stride: int, n_frames: int, stream: int = 0,
                      int16: bool = False):
        """pnb_submit_device_*: process_device without g/r; flush(other_stream) or wait() orders other work behind it."""
        f = self.L.pnb_submit_device_i16 if int16 else self.L.pnb_submit_device_f32
        self._ck(f(self.h, d_in, in_stride, d_out, out_stride, n_frames, stream or None), "pnb_submit_device")

    def compute_rnn(self, x: np.ndarray) -> np.ndarray:
        """pnb_compute_rnn_host: the network alone.  x: [active, F, 70] float32 features (as create_features makes them)
        or [active, F, 138] float32 training records (scaled x30 on the device like rnn_train.py's CppRawListDataset;
        the labels are ignored); the last dimension selects the format.  Advances the slots' network state by F hops
        and leaves their signal state alone.  Returns g/r [active, F, 68], hop t of row i beside record t's labels."""
        n = self.active
        if x.dtype != np.float32:
            raise TypeError("x must be float32")
        assert x.ndim == 3 and x.shape[0] == n and x.shape[2] in (70, RECORD), "x must be [active, F, 70 | 138]"
        F, W = x.shape[1], x.shape[2]
        x = np.ascontiguousarray(x)
        gr = np.empty((n, F, 68), np.float32)
        fmt = RNN_FEATURES if W == 70 else RNN_RECORDS
        self._ck(self.L.pnb_compute_rnn_host(self.h, fmt, x.ctypes.data, F * W, F, gr.ctypes.data, F * 68),
                 "pnb_compute_rnn_host")
        return gr

    def compute_rnn_device(self, format: int, d_in: int, in_stride: int, n_frames: int, d_gr: int, gr_stride: int,
                           stream: int = 0):
        """pnb_compute_rnn_device on raw device pointers (format RNN_FEATURES or RNN_RECORDS; strides in floats)."""
        self._ck(self.L.pnb_compute_rnn_device(self.h, format, d_in or None, in_stride, n_frames, d_gr or None, gr_stride,
                                               stream or None), "pnb_compute_rnn_device")

    def score_records(self, x: np.ndarray, frames=None, want_gr: bool = False):
        """pnb_score_records_host: compute_rnn on records x ([active, F, 138] float32) with rnn_train.py's CustomLoss
        reduced on the device against their labels.  frames: None, or one count in [0, F] per row: row i's loss counts
        its first frames[i] hops (every row still advances F hops).  Returns (sums [active, 4] float64 = {sum dg^2,
        sum dg^4, sum dr^2, count} per row, as eval_records.loss_sums computes them; g/r [active, F, 68] or None)."""
        n = self.active
        if x.dtype != np.float32:
            raise TypeError("x must be float32")
        assert x.ndim == 3 and x.shape[0] == n and x.shape[2] == RECORD, "x must be [active, F, 138]"
        F = x.shape[1]
        x = np.ascontiguousarray(x)
        fr = None if frames is None else self._slots(frames)[0]
        if fr is not None and len(fr) != n:
            raise PnbError("score_records: frames needs one entry per active row")
        sums = np.empty((n, 4), np.float64)
        gr = np.empty((n, F, 68), np.float32) if want_gr else None
        self._ck(self.L.pnb_score_records_host(self.h, x.ctypes.data, F * RECORD, F, None if fr is None else fr.ctypes.data,
                                               sums.ctypes.data, gr.ctypes.data if want_gr else None, F * 68),
                 "pnb_score_records_host")
        return sums, gr

    def score_records_device(self, d_rec: int, rec_stride: int, n_frames: int, frames, d_sums: int, d_gr: int = 0,
                             gr_stride: int = 0, stream: int = 0):
        """pnb_score_records_device on raw device pointers (strides in floats); frames: None or a host sequence of one
        count per active row; d_sums: [active, 4] float64; d_gr: 0 for no g/r."""
        fr = None if frames is None else self._slots(frames)[0]
        self._ck(self.L.pnb_score_records_device(self.h, d_rec or None, rec_stride, n_frames,
                                                 None if fr is None else fr.ctypes.data, d_sums or None, d_gr or None,
                                                 gr_stride, stream or None), "pnb_score_records_device")

    # ---- training (TRAIN_NETWORK engines; see pnb_train_grad_host in the header) -----------------------------------
    def train_grad(self, rec: np.ndarray, frames=None) -> np.ndarray:
        """pnb_train_grad_host: rnn_train.py's CustomLoss on the windows rec ([active, F, 138] float32 records, one window
        per row) and its gradient with respect to every parameter, kept on the engine for train_adam.  frames: None, or
        one count in [1, F] per window (its hops after that are ignored).  Returns the loss sums [active, 4] float64 as
        score_records returns them (eval_records.loss_terms of their sum gives the loss)."""
        n = self.active
        if rec.dtype != np.float32:
            raise TypeError("rec must be float32")
        assert rec.ndim == 3 and rec.shape[0] == n and rec.shape[2] == RECORD, "rec must be [active, F, 138]"
        F = rec.shape[1]
        rec = np.ascontiguousarray(rec)
        fr = None if frames is None else self._slots(frames)[0]
        if fr is not None and len(fr) != n:
            raise PnbError("train_grad: frames needs one entry per active row")
        sums = np.empty((n, 4), np.float64)
        self._ck(self.L.pnb_train_grad_host(self.h, rec.ctypes.data, F * RECORD, F, None if fr is None else fr.ctypes.data,
                                            sums.ctypes.data), "pnb_train_grad_host")
        return sums

    def train_grad_device(self, d_rec: int, rec_stride: int, n_frames: int, frames, d_sums: int, stream: int = 0):
        """pnb_train_grad_device on raw device pointers (rec_stride in floats); frames: None or a host sequence of one
        count per active row; d_sums: [active, 4] float64."""
        fr = None if frames is None else self._slots(frames)[0]
        self._ck(self.L.pnb_train_grad_device(self.h, d_rec or None, rec_stride, n_frames,
                                              None if fr is None else fr.ctypes.data, d_sums or None, stream or None),
                 "pnb_train_grad_device")

    def train_adam(self, lr: float, step: int, stream: int = 0):
        """pnb_train_adam: one torch.optim.Adam step (defaults) with the gradient of the last train_grad; step counts
        from 1.  Skipped on the device when that gradient was not finite."""
        self._ck(self.L.pnb_train_adam(self.h, float(lr), int(step), stream or None), "pnb_train_adam")

    def train_export(self, what: str) -> np.ndarray:
        """pnb_train_export: 'weights', 'gradient', 'm' or 'v' as one float32 vector in PNBW blob order
        (weights.PackedModel.from_flat turns it into a model)."""
        from .weights import N_PARAMS
        a = np.empty(N_PARAMS, np.float32)
        self._ck(self.L.pnb_train_export(self.h, TRAIN_ARRAYS[what], a.ctypes.data, a.nbytes), "pnb_train_export")
        return a

    def train_import(self, what: str, a: np.ndarray):
        """pnb_train_import: 'weights', 'm' or 'v' from a flat float32 vector in PNBW blob order (resuming a run)."""
        a = np.ascontiguousarray(a, np.float32)
        self._ck(self.L.pnb_train_import(self.h, TRAIN_ARRAYS[what], a.ctypes.data, a.nbytes), "pnb_train_import")

    def analyze(self, x: np.ndarray) -> np.ndarray:
        """pnb_analyze_host_*: the analysis half of process.  x: [active, F*480] float32 (C-API scale) or int16 (CLI wire
        format).  Returns the network input [active, F, 70] float32 (the features tap of a process call on x) and leaves
        a synthesis of F hops pending: the next call must be synthesize (or compute_rnn, or reset)."""
        n = self.active
        assert x.ndim == 2 and x.shape[0] == n and x.shape[1] % FRAME == 0
        F = x.shape[1] // FRAME
        x = np.ascontiguousarray(x)
        feat = np.empty((n, F, 70), np.float32)
        if x.dtype == np.float32:
            f = self.L.pnb_analyze_host_f32
        elif x.dtype == np.int16:
            f = self.L.pnb_analyze_host_i16
        else:
            raise TypeError("x must be float32 or int16")
        self._ck(f(self.h, x.ctypes.data, x.shape[1], F, feat.ctypes.data, F * 70), "pnb_analyze_host")
        return feat

    def synthesize(self, gr: np.ndarray, int16: bool = False) -> np.ndarray:
        """pnb_synthesize_host_*: the synthesis half of process, with the caller's gains.  gr: [active, F, 68] float32
        (34 g then 34 r per hop), F the hops of the pending analysis.  Returns [active, F*480] float32, or int16 with
        the CLI's conversion."""
        n = self.active
        if gr.dtype != np.float32:
            raise TypeError("gr must be float32")
        assert gr.ndim == 3 and gr.shape[0] == n and gr.shape[2] == 68, "gr must be [active, F, 68]"
        F = gr.shape[1]
        gr = np.ascontiguousarray(gr)
        out = np.empty((n, F * FRAME), np.int16 if int16 else np.float32)
        f = self.L.pnb_synthesize_host_i16 if int16 else self.L.pnb_synthesize_host_f32
        self._ck(f(self.h, gr.ctypes.data, F * 68, F, out.ctypes.data, F * FRAME), "pnb_synthesize_host")
        return out

    def analyze_device(self, d_in: int, in_stride: int, n_frames: int, d_feat: int, feat_stride: int, stream: int = 0,
                       int16: bool = False):
        """pnb_analyze_device_* on raw device pointers (strides in elements)."""
        f = self.L.pnb_analyze_device_i16 if int16 else self.L.pnb_analyze_device_f32
        self._ck(f(self.h, d_in or None, in_stride, n_frames, d_feat or None, feat_stride, stream or None),
                 "pnb_analyze_device")

    def synthesize_device(self, d_gr: int, gr_stride: int, n_frames: int, d_out: int, out_stride: int, stream: int = 0,
                          int16: bool = False):
        """pnb_synthesize_device_* on raw device pointers (strides in elements)."""
        f = self.L.pnb_synthesize_device_i16 if int16 else self.L.pnb_synthesize_device_f32
        self._ck(f(self.h, d_gr or None, gr_stride, n_frames, d_out or None, out_stride, stream or None),
                 "pnb_synthesize_device")

    @property
    def device_bytes(self) -> int:
        """pnb_engine_bytes: the engine's fixed-size device buffers, in bytes."""
        return int(self.L.pnb_engine_bytes(self.h))

    def flush(self, stream: int = 0):
        self._ck(self.L.pnb_flush(self.h, stream or None), "pnb_flush")

    def submit(self, x: np.ndarray, out: np.ndarray):
        """Pipelined host call (pnb_submit_host_*): returns at once; x/out ([active, F*480] float32 or int16, ideally
        pinned) must stay alive until wait()."""
        assert x.shape == out.shape and x.dtype == out.dtype and x.shape[0] == self.active
        F = x.shape[1] // FRAME
        f = self.L.pnb_submit_host_f32 if x.dtype == np.float32 else self.L.pnb_submit_host_i16
        self._ck(f(self.h, x.ctypes.data, x.strides[0] // x.itemsize, out.ctypes.data, out.strides[0] // out.itemsize, F),
                 "pnb_submit_host")

    def wait(self):
        self._ck(self.L.pnb_wait(self.h), "pnb_wait")

    def check(self, stream: int = 0):
        """pnb_check: waits for the engine's work (and `stream`) and raises on PNB_ERR_DOMAIN / PNB_ERR_CUDA."""
        self._ck(self.L.pnb_check(self.h, stream or None), "pnb_check")

    def read_tap(self, name: str, n_frames: int) -> np.ndarray:
        code, dt, width = TAPS[name]
        a = np.empty((n_frames, self.n_streams, width), dt)
        self._ck(self.L.pnb_read_tap(self.h, code, a.ctypes.data, a.nbytes), f"pnb_read_tap({name})")
        return a

    def get_state(self, stream: int) -> bytes:
        buf = C.create_string_buffer(self.L.pnb_state_size())
        self._ck(self.L.pnb_get_state(self.h, stream, buf, len(buf)), "pnb_get_state")
        return buf.raw

    def set_state(self, stream: int, blob: bytes):
        self._ck(self.L.pnb_set_state(self.h, stream, blob, len(blob)), "pnb_set_state")

    # ---- batched stream recycling (asynchronous on `stream`; see pnb_reset_streams in the header) ----------------
    @staticmethod
    def _slots(idx):
        a = np.ascontiguousarray(np.asarray(idx, dtype=np.int64).reshape(-1).astype(np.int32))
        return a, len(a)

    @property
    def state_size(self) -> int:
        return int(self.L.pnb_state_size())

    def reset_streams(self, idx, stream: int = 0):
        """pnb_reset_streams: the slots in `idx` start over as fresh streams; the others are untouched."""
        a, n = self._slots(idx)
        self._ck(self.L.pnb_reset_streams(self.h, a.ctypes.data if n else None, n, stream or None), "pnb_reset_streams")

    def export_states(self, idx, d_blobs, stride: int = 0, stream: int = 0):
        """pnb_export_states.  d_blobs: a raw device pointer (blob i at d_blobs + i*stride, stride 0 = pnb_state_size()),
        or None to get a new CUDA uint8 torch tensor [len(idx), pnb_state_size()] back."""
        a, n = self._slots(idx)
        out = None
        if d_blobs is None:
            import torch
            out = torch.empty((n, self.state_size), dtype=torch.uint8, device=f"cuda:{self.device}")
            d_blobs, stride = out.data_ptr(), self.state_size
        self._ck(self.L.pnb_export_states(self.h, a.ctypes.data if n else None, n, d_blobs or None, stride or self.state_size,
                                          stream or None), "pnb_export_states")
        return out

    def import_states(self, idx, d_blobs, stride: int = 0, stream: int = 0):
        """pnb_import_states.  d_blobs: a raw device pointer (as export_states) or a CUDA uint8 tensor
        [len(idx), >= pnb_state_size()] whose rows are blobs; the tensor must stay alive until `stream` has run the import."""
        a, n = self._slots(idx)
        d_blobs, stride = self._blob_rows(d_blobs, stride, n, "import_states")
        self._ck(self.L.pnb_import_states(self.h, a.ctypes.data if n else None, n, d_blobs or None, stride or self.state_size,
                                          stream or None), "pnb_import_states")

    @staticmethod
    def _blob_rows(d_blobs, stride, n, what):
        if not isinstance(d_blobs, int) and d_blobs is not None:
            t = d_blobs
            if t.dtype.itemsize != 1 or t.dim() != 2 or t.shape[0] != n or t.stride(1) != 1 or not t.is_cuda:
                raise PnbError(f"{what}: blobs must be a CUDA byte tensor [len(idx), pnb_state_size()] with contiguous rows")
            d_blobs, stride = t.data_ptr(), t.stride(0)
        return d_blobs, stride

    # ---- session pool (see pnb_sessions_reserve in the header) ---------------------------------------------------------
    def reserve_sessions(self, n_sessions: int):
        """pnb_sessions_reserve: session mode with sessions [0, n_sessions), all fresh (the first call resets the engine);
        a later, larger call grows the pool and keeps every session's state."""
        self._ck(self.L.pnb_sessions_reserve(self.h, n_sessions), "pnb_sessions_reserve")

    def process_sessions(self, ids, x: np.ndarray, want_gr: bool = False, hops=None):
        """pnb_process_sessions_host_*: advances exactly the listed sessions.  x: [len(ids), F*480] float32 or int16 host
        array, row i for ids[i].  Returns (out like x, gr [F, len(ids), 68] or None).
        hops: None, or one hop count per session (pnb_process_sessions_ragged_host_*): session ids[i] advances by
        hops[i], F = max(hops) must be x's width in hops, and row i of out / gr[:, i] is zero after hops[i] hops."""
        a, n = self._slots(ids)
        assert x.ndim == 2 and x.shape[0] == n and x.shape[1] % FRAME == 0
        F = x.shape[1] // FRAME
        x = np.ascontiguousarray(x)
        out = np.empty_like(x)
        gr = np.empty((F, n, 68), np.float32) if want_gr else None
        grp = gr.ctypes.data if want_gr else None
        if x.dtype not in (np.float32, np.int16):
            raise TypeError("x must be float32 or int16")
        i16 = x.dtype == np.int16
        if hops is None:
            f = self.L.pnb_process_sessions_host_i16 if i16 else self.L.pnb_process_sessions_host_f32
            self._ck(f(self.h, a.ctypes.data, n, x.ctypes.data, x.shape[1], out.ctypes.data, x.shape[1], F, grp),
                     "pnb_process_sessions_host")
            return out, gr
        hp, nh = self._slots(hops)
        if nh != n or int(hp.max(initial=0)) != F:
            raise PnbError("process_sessions: hops needs one entry per session, and x must be max(hops) hops wide")
        f = self.L.pnb_process_sessions_ragged_host_i16 if i16 else self.L.pnb_process_sessions_ragged_host_f32
        self._ck(f(self.h, a.ctypes.data, hp.ctypes.data, n, x.ctypes.data, x.shape[1], out.ctypes.data, x.shape[1], grp),
                 "pnb_process_sessions_ragged_host")
        return out, gr

    def process_sessions_device(self, ids, d_in: int, in_stride: int, d_out: int, out_stride: int, n_frames: int = 0,
                                d_gr: int = 0, stream: int = 0, int16: bool = False, hops=None):
        """pnb_process_sessions_device_*: raw device pointers, row i of in / out and d_gr[t][i] for ids[i].
        hops: None, or one hop count per session (pnb_process_sessions_ragged_device_*; n_frames is then max(hops) and
        need not be given)."""
        a, n = self._slots(ids)
        if hops is None:
            f = self.L.pnb_process_sessions_device_i16 if int16 else self.L.pnb_process_sessions_device_f32
            self._ck(f(self.h, a.ctypes.data, n, d_in, in_stride, d_out, out_stride, n_frames, d_gr or None, stream or None),
                     "pnb_process_sessions_device")
            return
        hp, nh = self._slots(hops)
        if nh != n or (n_frames and int(hp.max(initial=0)) != n_frames):
            raise PnbError("process_sessions_device: hops needs one entry per session, and n_frames (if given) = max(hops)")
        f = self.L.pnb_process_sessions_ragged_device_i16 if int16 else self.L.pnb_process_sessions_ragged_device_f32
        self._ck(f(self.h, a.ctypes.data, hp.ctypes.data, n, d_in, in_stride, d_out, out_stride, d_gr or None,
                   stream or None), "pnb_process_sessions_ragged_device")

    def reset_sessions(self, ids, stream: int = 0):
        """pnb_reset_sessions: the listed sessions start over as fresh streams."""
        a, n = self._slots(ids)
        self._ck(self.L.pnb_reset_sessions(self.h, a.ctypes.data if n else None, n, stream or None), "pnb_reset_sessions")

    def export_sessions(self, ids, d_blobs, stride: int = 0, stream: int = 0):
        """pnb_export_sessions, with the conventions of export_states (None: returns a new CUDA uint8 tensor)."""
        a, n = self._slots(ids)
        out = None
        if d_blobs is None:
            import torch
            out = torch.empty((n, self.state_size), dtype=torch.uint8, device=f"cuda:{self.device}")
            d_blobs, stride = out.data_ptr(), self.state_size
        self._ck(self.L.pnb_export_sessions(self.h, a.ctypes.data if n else None, n, d_blobs or None,
                                            stride or self.state_size, stream or None), "pnb_export_sessions")
        return out

    def import_sessions(self, ids, d_blobs, stride: int = 0, stream: int = 0):
        """pnb_import_sessions, with the conventions of import_states (a raw pointer or a CUDA uint8 tensor of blob rows)."""
        a, n = self._slots(ids)
        d_blobs, stride = self._blob_rows(d_blobs, stride, n, "import_sessions")
        self._ck(self.L.pnb_import_sessions(self.h, a.ctypes.data if n else None, n, d_blobs or None,
                                            stride or self.state_size, stream or None), "pnb_import_sessions")

    def session_stats(self) -> dict:
        """pnb_session_stats: cumulative {parks, unparks, relocations} of the session pool."""
        c = (C.c_longlong * 3)()
        self._ck(self.L.pnb_session_stats(self.h, c), "pnb_session_stats")
        return {"parks": int(c[0]), "unparks": int(c[1]), "relocations": int(c[2])}

    def read_nn_state(self) -> dict:
        """fp32 network state after the last hop: conv2 output and the five GRU states, [S, width]."""
        out = {}
        for name, code, width in (("c2", 7, 512), ("gru1", 8, 512), ("gru2", 9, 512), ("gru3", 10, 512),
                                  ("gru_gb", 11, 512), ("gru_rb", 12, 128)):
            a = np.empty((self.n_streams, width), np.float32)
            self._ck(self.L.pnb_read_tap(self.h, code, a.ctypes.data, a.nbytes), f"pnb_read_tap({name})")
            out[name] = a
        return out

    def train_records(self, speech: np.ndarray, noisy: np.ndarray) -> np.ndarray:
        """speech, noisy: [n_pairs, F*480] int16 -> [n_pairs, F, 138] float32, the records the reference's train()
        (src/denoise.cpp:600-787) writes for each pair of files.  Engine must have flags=TRAIN_DATA and
        n_streams = 2*n_pairs; state carries over, so call repeatedly with consecutive chunks."""
        N = self.n_streams // 2
        assert speech.shape == noisy.shape and speech.shape[0] == N and speech.shape[1] % FRAME == 0
        assert speech.dtype == np.int16 and noisy.dtype == np.int16
        F = speech.shape[1] // FRAME
        speech, noisy = np.ascontiguousarray(speech), np.ascontiguousarray(noisy)
        rec = np.empty((N, F, RECORD), np.float32)
        self._ck(self.L.pnb_train_records_host(self.h, speech.ctypes.data, speech.shape[1], noisy.ctypes.data,
                                               noisy.shape[1], F, rec.ctypes.data, F * RECORD), "pnb_train_records_host")
        return rec

    def train_records_device(self, d_speech: int, speech_stride: int, d_noisy: int, noisy_stride: int, n_frames: int,
                             d_records: int, records_stride: int, stream: int = 0):
        self._ck(self.L.pnb_train_records_device(self.h, d_speech, speech_stride, d_noisy, noisy_stride, n_frames,
                                                 d_records, records_stride, stream), "pnb_train_records_device")

    def train_audio(self, speech: np.ndarray, noisy: np.ndarray):
        """speech, noisy: [n_pairs, F*480] int16 -> (records [n_pairs, F, 138] float32, audio [n_pairs, F*480] int16):
        the records of train_records and, for each pair, what the reference's train() writes to test_output.pcm over
        these frames (src/denoise.cpp:742-759: the noisy file resynthesised with its own labels, clamped to int16).
        Engine must have flags=TRAIN_DATA | TRAIN_AUDIO; state carries over, so call repeatedly with consecutive chunks."""
        N = self.n_streams // 2
        assert speech.shape == noisy.shape and speech.shape[0] == N and speech.shape[1] % FRAME == 0
        assert speech.dtype == np.int16 and noisy.dtype == np.int16
        F = speech.shape[1] // FRAME
        speech, noisy = np.ascontiguousarray(speech), np.ascontiguousarray(noisy)
        rec = np.empty((N, F, RECORD), np.float32)
        audio = np.empty((N, F * FRAME), np.int16)
        self._ck(self.L.pnb_train_audio_host(self.h, speech.ctypes.data, speech.shape[1], noisy.ctypes.data, noisy.shape[1],
                                             F, rec.ctypes.data, F * RECORD, audio.ctypes.data, F * FRAME),
                 "pnb_train_audio_host")
        return rec, audio

    def train_audio_device(self, d_speech: int, speech_stride: int, d_noisy: int, noisy_stride: int, n_frames: int,
                           d_records: int, records_stride: int, d_audio: int, audio_stride: int, stream: int = 0):
        self._ck(self.L.pnb_train_audio_device(self.h, d_speech, speech_stride, d_noisy, noisy_stride, n_frames, d_records,
                                               records_stride, d_audio, audio_stride, stream), "pnb_train_audio_device")

    def profile(self, on: bool):
        self._ck(self.L.pnb_profile_enable(self.h, 1 if on else 0), "pnb_profile_enable")

    def profile_read(self) -> dict:
        """{kernel class name: (total ms, launches)} since the last read; waits for the device."""
        n = 10
        ms = (C.c_double * n)()
        cnt = (C.c_longlong * n)()
        self._ck(self.L.pnb_profile_read(self.h, ms, cnt), "pnb_profile_read")
        return {self.L.pnb_kernel_class_name(k).decode(): (ms[k], int(cnt[k])) for k in range(n) if cnt[k]}

    def profile_timeline(self, cap: int = 4096):
        """[(class name, start ms, end ms)] of every launch since profiling was enabled / last read."""
        cls = (C.c_int * cap)()
        t0 = (C.c_double * cap)()
        t1 = (C.c_double * cap)()
        n = self.L.pnb_profile_timeline(self.h, cls, t0, t1, cap)
        if n < 0:
            self._ck(n, "pnb_profile_timeline")
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
