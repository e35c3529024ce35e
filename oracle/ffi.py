"""ctypes bindings for the oracle libraries -- TEST INFRASTRUCTURE ONLY.

Importable only from tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
``--impl reference`` legs.  Two libraries:

* ``libpn_oracle.so``  -- the C restatement (oracle/pn_oracle.c), always buildable.
* ``_ref/libpercepnet_ref.so`` -- the unmodified reference compiled from /root/reference/src
  plus oracle/ref_harness.cpp; exists when it was built in the container that has the
  reference (it is git-ignored but travels to the GPU box with the snapshot).
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ORACLE_SO = os.path.join(HERE, "libpn_oracle.so")
REF_SO = os.path.join(HERE, "_ref", "libpercepnet_ref.so")

F32P = C.POINTER(C.c_float)
I32P = C.POINTER(C.c_int)
I16P = C.POINTER(C.c_short)


def build(force: bool = False) -> None:
    """Compile the restatement (and the reference library when /root/reference exists)."""
    args = ["make", "-C", HERE, "-s"] + (["-B"] if force else [])
    subprocess.run(args, check=True)


def _f(a):
    a = np.ascontiguousarray(a, dtype=np.float32)
    return a, a.ctypes.data_as(F32P)


class Taps(C.Structure):
    _fields_ = [
        ("X", C.c_float * 962), ("P", C.c_float * 962), ("Y", C.c_float * 962), ("Xout", C.c_float * 962),
        ("Ex", C.c_float * 34), ("Ep", C.c_float * 34), ("Exp", C.c_float * 34), ("Ex_look", C.c_float * 34),
        ("features", C.c_float * 70), ("g", C.c_float * 34), ("r", C.c_float * 34), ("g_used", C.c_float * 34),
        ("lp", C.c_float * 864), ("xcorr_coarse", C.c_float * 147), ("best_coarse", C.c_int * 2),
        ("pitch_search", C.c_int), ("pitch_corr", C.c_float), ("pitch_index", C.c_int),
        ("pitch_gain", C.c_float), ("silence", C.c_int),
    ]

    def np(self, name):
        return np.ctypeslib.as_array(getattr(self, name)).copy()


class Oracle:
    """The C restatement."""

    def __init__(self, path: str = ORACLE_SO):
        if not os.path.exists(path):
            build()
        self.lib = L = C.CDLL(path)
        L.pn_oracle_create.restype = C.c_void_p
        L.pn_oracle_create.argtypes = [C.c_void_p]
        L.pn_oracle_destroy.argtypes = [C.c_void_p]
        L.pn_oracle_reset.argtypes = [C.c_void_p]
        L.pn_oracle_process_frame.argtypes = [C.c_void_p, F32P, F32P, C.c_void_p, C.c_int]
        L.pn_oracle_process_stream.argtypes = [C.c_void_p, F32P, F32P, C.c_int, F32P, C.c_int]
        L.pn_oracle_run_pcm16.argtypes = [C.c_void_p, I16P, C.c_int, I16P, F32P]
        L.pn_oracle_process_streams.argtypes = [C.c_void_p, C.c_int, C.c_int, F32P, F32P, C.c_int, C.c_int]
        L.pn_oracle_tansig.restype = C.c_float
        L.pn_oracle_tansig.argtypes = [C.c_float]
        L.pn_oracle_sigmoid.restype = C.c_float
        L.pn_oracle_sigmoid.argtypes = [C.c_float]
        L.pn_oracle_remove_doubling.restype = C.c_float
        L.pn_oracle_remove_doubling.argtypes = [F32P, I32P, C.c_int, C.c_float]

    # -- training-data path (row f1) ----------------------------------------------------
    def train_records(self, speech16, noisy16):
        """[count*480] int16 each -> [count, 138] float32 (train(), denoise.cpp:600-787)."""
        speech16 = np.ascontiguousarray(speech16, np.int16)
        noisy16 = np.ascontiguousarray(noisy16, np.int16)
        count = speech16.size // 480
        rec = np.empty((count, 138), np.float32)
        self.lib.pn_oracle_train_records.argtypes = [I16P, I16P, C.c_int, F32P]
        self.lib.pn_oracle_train_records(speech16.ctypes.data_as(I16P), noisy16.ctypes.data_as(I16P), count,
                                         rec.ctypes.data_as(F32P))
        return rec

    def ideal_labels(self, Ex, Ey, Exp, Ephaty):
        a = [np.ascontiguousarray(v, np.float32) for v in (Ex, Ey, Exp, Ephaty)]
        g, r = np.empty(34, np.float32), np.empty(34, np.float32)
        self.lib.pn_oracle_ideal_labels.argtypes = [F32P] * 6
        self.lib.pn_oracle_ideal_labels(*[v.ctypes.data_as(F32P) for v in a + [g, r]])
        return g, r

    # -- engine -------------------------------------------------------------------------
    def create(self, model):
        self._model = model  # keep the weight arrays alive
        return self.lib.pn_oracle_create(C.byref(model.as_c_model()))

    def destroy(self, h):
        self.lib.pn_oracle_destroy(h)

    def process_stream(self, h, x, want_gr=False, flags=0, taps=False):
        """x: [n_frames*480] float32 -> (out, gr or None, [Taps] or None)"""
        x, xp = _f(x)
        n = x.size // 480
        out = np.empty_like(x)
        if taps:
            tl = []
            gr = np.empty((n, 68), np.float32)
            for t in range(n):
                tp = Taps()
                self.lib.pn_oracle_process_frame(h, out[480 * t:].ctypes.data_as(F32P),
                                                 x[480 * t:].ctypes.data_as(F32P), C.byref(tp), flags)
                gr[t, :34] = tp.np("g")
                gr[t, 34:] = tp.np("r")
                tl.append(tp)
            return out, gr, tl
        gr = np.empty((n, 68), np.float32) if want_gr else None
        self.lib.pn_oracle_process_stream(h, out.ctypes.data_as(F32P), xp, n,
                                          gr.ctypes.data_as(F32P) if want_gr else None, flags)
        return out, gr, None

    def run_pcm16(self, model, pcm16):
        pcm16 = np.ascontiguousarray(pcm16, dtype=np.int16)
        n = pcm16.size // 480
        out = np.zeros((n - 1) * 480, np.int16)
        gr = np.empty((n, 68), np.float32)
        self.lib.pn_oracle_run_pcm16(C.byref(model.as_c_model()), pcm16.ctypes.data_as(I16P), n,
                                     out.ctypes.data_as(I16P), gr.ctypes.data_as(F32P))
        return out, gr

    def process_streams(self, model, x, n_threads=1, flags=0):
        """x: [S, n_frames*480] -> out same shape (fresh state per stream)"""
        x = np.ascontiguousarray(x, dtype=np.float32)
        S, T = x.shape
        out = np.empty_like(x)
        self.lib.pn_oracle_process_streams(C.byref(model.as_c_model()), S, T // 480,
                                           x.ctypes.data_as(F32P), out.ctypes.data_as(F32P), n_threads, flags)
        return out

    # -- stages -------------------------------------------------------------------------
    def erb_borders(self):
        b = np.zeros(34, np.int32)
        self.lib.pn_oracle_erb_borders(b.ctypes.data_as(I32P))
        return b

    def tables(self):
        hw, cw = np.zeros(480, np.float32), np.zeros(7, np.float32)
        self.lib.pn_oracle_tables(hw.ctypes.data_as(F32P), cw.ctypes.data_as(F32P))
        return hw, cw

    def fft960(self, x_ri):
        x, xp = _f(x_ri)
        y = np.empty(1920, np.float32)
        self.lib.pn_oracle_fft960(xp, y.ctypes.data_as(F32P))
        return y

    def band_energy(self, X):
        X, p = _f(X)
        e = np.empty(34, np.float32)
        self.lib.pn_oracle_band_energy(e.ctypes.data_as(F32P), p)
        return e

    def band_corr(self, X, P):
        X, xp = _f(X)
        P, pp = _f(P)
        e = np.empty(34, np.float32)
        self.lib.pn_oracle_band_corr(e.ctypes.data_as(F32P), xp, pp)
        return e

    def interp_band_gain(self, bandE):
        b, bp = _f(bandE)
        g = np.zeros(481, np.float32)
        self.lib.pn_oracle_interp_band_gain(g.ctypes.data_as(F32P), bp)
        return g

    def pitch_filter(self, X, P, r):
        X = np.array(X, dtype=np.float32, copy=True)
        P, pp = _f(P)
        r, rp = _f(r)
        self.lib.pn_oracle_pitch_filter(X.ctypes.data_as(F32P), pp, rp)
        return X

    def post_filter(self, g, Ey):
        g = np.array(g, dtype=np.float32, copy=True)
        Ey, ep = _f(Ey)
        self.lib.pn_oracle_post_filter(g.ctypes.data_as(F32P), ep)
        return g

    def pitch_downsample(self, buf1728):
        b, bp = _f(buf1728)
        lp = np.empty(864, np.float32)
        self.lib.pn_oracle_pitch_downsample(bp, lp.ctypes.data_as(F32P))
        return lp

    def autocorr_lpc(self, x):
        x, xp = _f(x)
        ac, lpc = np.empty(5, np.float32), np.empty(4, np.float32)
        self.lib.pn_oracle_autocorr_lpc(xp, x.size, ac.ctypes.data_as(F32P), lpc.ctypes.data_as(F32P))
        return ac, lpc

    def pitch_xcorr(self, x, y, max_pitch):
        x, xp = _f(x)
        y, yp = _f(y)
        out = np.empty(max_pitch, np.float32)
        self.lib.pn_oracle_pitch_xcorr(xp, yp, out.ctypes.data_as(F32P), x.size, max_pitch)
        return out

    def pitch_search(self, lp):
        lp, p = _f(lp)
        pitch, corr = C.c_int(), C.c_float()
        coarse = np.empty(147, np.float32)
        best = np.zeros(2, np.int32)
        self.lib.pn_oracle_pitch_search(p, C.byref(pitch), C.byref(corr), coarse.ctypes.data_as(F32P),
                                        best.ctypes.data_as(I32P))
        return pitch.value, corr.value, coarse, best

    def remove_doubling(self, lp, T0, prev_period, prev_gain):
        lp, p = _f(lp)
        t = C.c_int(T0)
        g = self.lib.pn_oracle_remove_doubling(p, C.byref(t), prev_period, prev_gain)
        return t.value, g

    def tansig(self, x):
        return np.array([self.lib.pn_oracle_tansig(float(v)) for v in np.asarray(x, np.float32).ravel()], np.float32)

    def sigmoid(self, x):
        return np.array([self.lib.pn_oracle_sigmoid(float(v)) for v in np.asarray(x, np.float32).ravel()], np.float32)

    def _vec(self, fn, x):
        a = np.ascontiguousarray(x, np.float32)
        y = np.empty_like(a)
        fn.argtypes = [F32P, F32P, C.c_long]
        fn(a.ctypes.data_as(F32P), y.ctypes.data_as(F32P), a.size)
        return y

    def tansig_n(self, x):
        """tansig_approx (vec.h:53-71) of every element, same shape; one call for the whole array."""
        return self._vec(self.lib.pn_oracle_tansig_n, x)

    def sigmoid_n(self, x):
        return self._vec(self.lib.pn_oracle_sigmoid_n, x)

    def dense_layer(self, layer, x, n_out):
        x, xp = _f(x)
        out = np.empty(n_out, np.float32)
        self.lib.pn_oracle_dense_layer(C.byref(layer), out.ctypes.data_as(F32P), xp)
        return out

    def conv1d_layer(self, layer, mem, x, n_out):
        x, xp = _f(x)
        out = np.empty(n_out, np.float32)
        self.lib.pn_oracle_conv1d_layer(C.byref(layer), out.ctypes.data_as(F32P), mem.ctypes.data_as(F32P), xp)
        return out

    def gru_layer(self, layer, state, x):
        x, xp = _f(x)
        self.lib.pn_oracle_gru_layer(C.byref(layer), state.ctypes.data_as(F32P), xp)
        return state

    def compute_rnn(self, model, state, features):
        f, fp = _f(features)
        g, r = np.empty(34, np.float32), np.empty(34, np.float32)
        self.lib.pn_oracle_compute_rnn(C.byref(model.as_c_model()), state.ctypes.data_as(F32P),
                                       g.ctypes.data_as(F32P), r.ctypes.data_as(F32P), fp)
        return g, r


    def pitch_batch(self, bufs, n_threads=1):
        """[n, 1728] pitch buffers -> (T int32 [n], corr [n], gain [n]) with zero previous period / gain"""
        b, bp = _f(bufs)
        n = b.shape[0]
        T, corr, gain = np.empty(n, np.int32), np.empty(n, np.float32), np.empty(n, np.float32)
        self.lib.pn_oracle_pitch_batch.argtypes = [F32P, C.c_size_t, C.c_int, C.c_void_p, C.c_void_p, I32P, F32P, F32P, C.c_int]
        self.lib.pn_oracle_pitch_batch(bp, b.shape[1], n, None, None, T.ctypes.data_as(I32P), corr.ctypes.data_as(F32P),
                                       gain.ctypes.data_as(F32P), n_threads)
        return T, corr, gain

    NN_STATE = 512 + 1024 + 4 * 512 + 128  # [conv1 mem 4 x 128][conv2 mem 2 x 512][gru1 gru2 gru3 gru_gb][gru_rb]

    def rnn_f64(self, model, features, state=None):
        """features [F, 70] of one stream -> (g [F, 34], r [F, 34] in float64, max |pre-activation| per frame):
        the network in double precision (pn_oracle_compute_rnn_f64) from `state` ([NN_STATE], the conv memories
        oldest first, then the five GRU states; not modified), or from a zero state."""
        feats = np.ascontiguousarray(features, dtype=np.float32)
        F = feats.shape[0]
        st = np.zeros(self.NN_STATE, np.float64)
        if state is not None:
            st[:] = np.asarray(state, np.float64).reshape(self.NN_STATE)
        g, r, mp = np.empty((F, 34), np.float64), np.empty((F, 34), np.float64), np.empty(F, np.float64)
        D = C.POINTER(C.c_double)
        self.lib.pn_oracle_compute_rnn_f64.restype = C.c_double
        cm = model.as_c_model()
        for t in range(F):
            mp[t] = self.lib.pn_oracle_compute_rnn_f64(C.byref(cm), st.ctypes.data_as(D), g[t].ctypes.data_as(D),
                                                       r[t].ctypes.data_as(D), feats[t].ctypes.data_as(F32P))
        return g, r, mp


class Reference:
    """The compiled, unmodified reference behind oracle/ref_harness.cpp."""

    @staticmethod
    def available() -> bool:
        return os.path.exists(REF_SO)

    def __init__(self, path: str = REF_SO):
        self.lib = L = C.CDLL(path)
        L.ref_create.restype = C.c_void_p
        L.ref_destroy.argtypes = [C.c_void_p]
        L.ref_set_model.argtypes = [C.c_void_p]
        L.ref_process_frame.argtypes = [C.c_void_p, F32P, F32P, F32P]
        L.ref_process_stream.argtypes = [C.c_void_p, F32P, F32P, C.c_int, F32P]
        L.ref_run_pcm16.argtypes = [I16P, C.c_int, I16P, F32P]
        L.ref_process_streams_omp.argtypes = [C.c_int, C.c_int, F32P, F32P, C.c_int]
        L.ref_remove_doubling.restype = C.c_float
        L.ref_remove_doubling.argtypes = [F32P, I32P, C.c_int, C.c_float]

    def train_files(self, speech_path, noisy_path, count, out_path):
        """The reference's own train() (denoise.cpp:600) on files."""
        self.lib.ref_train_files.argtypes = [C.c_char_p, C.c_char_p, C.c_int, C.c_char_p]
        return self.lib.ref_train_files(speech_path.encode(), noisy_path.encode(), count, out_path.encode())

    def set_model(self, model):
        self._model = model
        self.lib.ref_set_model(C.byref(model.as_c_model()))

    def create(self):
        return self.lib.ref_create()

    def destroy(self, h):
        self.lib.ref_destroy(h)

    def process_stream(self, h, x, want_gr=False):
        x, xp = _f(x)
        n = x.size // 480
        out = np.empty_like(x)
        gr = np.empty((n, 68), np.float32) if want_gr else None
        self.lib.ref_process_stream(h, out.ctypes.data_as(F32P), xp, n, gr.ctypes.data_as(F32P) if want_gr else None)
        return out, gr

    def run_pcm16(self, pcm16):
        pcm16 = np.ascontiguousarray(pcm16, dtype=np.int16)
        n = pcm16.size // 480
        out = np.zeros((n - 1) * 480, np.int16)
        gr = np.empty((n, 68), np.float32)
        self.lib.ref_run_pcm16(pcm16.ctypes.data_as(I16P), n, out.ctypes.data_as(I16P), gr.ctypes.data_as(F32P))
        return out, gr

    def process_streams(self, x, n_threads=1):
        x = np.ascontiguousarray(x, dtype=np.float32)
        S, T = x.shape
        out = np.empty_like(x)
        self.lib.ref_process_streams_omp(S, T // 480, x.ctypes.data_as(F32P), out.ctypes.data_as(F32P), n_threads)
        return out

    def erb_borders(self):
        b = np.zeros(34, np.int32)
        self.lib.ref_erb_borders(b.ctypes.data_as(I32P))
        return b

    def fft960(self, x_ri):
        x, xp = _f(x_ri)
        y = np.empty(1920, np.float32)
        self.lib.ref_fft960(xp, y.ctypes.data_as(F32P))
        return y

    def band_energy(self, X):
        X, p = _f(X)
        e = np.empty(34, np.float32)
        self.lib.ref_band_energy(e.ctypes.data_as(F32P), p)
        return e

    def band_corr(self, X, P):
        X, xp = _f(X)
        P, pp = _f(P)
        e = np.empty(34, np.float32)
        self.lib.ref_band_corr(e.ctypes.data_as(F32P), xp, pp)
        return e

    def interp_band_gain(self, bandE):
        b, bp = _f(bandE)
        g = np.zeros(481, np.float32)  # zero-initialised like the reference's callers
        self.lib.ref_interp_band_gain(g.ctypes.data_as(F32P), bp)
        return g

    def pitch_filter(self, X, P, r):
        X = np.array(X, dtype=np.float32, copy=True)
        P, pp = _f(P)
        g = np.zeros(34, np.float32)
        r, rp = _f(r)
        self.lib.ref_pitch_filter(X.ctypes.data_as(F32P), pp, g.ctypes.data_as(F32P), rp)
        return X

    def pitch_downsample(self, buf1728):
        b = np.array(buf1728, dtype=np.float32, copy=True)
        lp = np.empty(864, np.float32)
        self.lib.ref_pitch_downsample(b.ctypes.data_as(F32P), lp.ctypes.data_as(F32P))
        return lp

    def autocorr_lpc(self, x):
        x, xp = _f(x)
        ac, lpc = np.empty(5, np.float32), np.empty(4, np.float32)
        self.lib.ref_autocorr_lpc(xp, x.size, ac.ctypes.data_as(F32P), lpc.ctypes.data_as(F32P))
        return ac, lpc

    def pitch_xcorr(self, x, y, max_pitch):
        x, xp = _f(x)
        y, yp = _f(y)
        out = np.empty(max_pitch, np.float32)
        self.lib.ref_pitch_xcorr(xp, yp, out.ctypes.data_as(F32P), x.size, max_pitch)
        return out

    def pitch_search(self, lp):
        lp = np.array(lp, dtype=np.float32, copy=True)
        pitch, corr = C.c_int(), C.c_float()
        self.lib.ref_pitch_search(lp.ctypes.data_as(F32P), C.byref(pitch), C.byref(corr))
        return pitch.value, corr.value

    def remove_doubling(self, lp, T0, prev_period, prev_gain):
        lp = np.array(lp, dtype=np.float32, copy=True)
        t = C.c_int(T0)
        g = self.lib.ref_remove_doubling(lp.ctypes.data_as(F32P), C.byref(t), prev_period, prev_gain)
        return t.value, g

    def dense_layer(self, layer, x, n_out):
        x, xp = _f(x)
        out = np.empty(n_out, np.float32)
        self.lib.ref_dense_layer(C.byref(layer), out.ctypes.data_as(F32P), xp)
        return out

    def conv1d_layer(self, layer, mem, x, n_out):
        x, xp = _f(x)
        out = np.empty(n_out, np.float32)
        self.lib.ref_conv1d_layer(C.byref(layer), out.ctypes.data_as(F32P), mem.ctypes.data_as(F32P), xp)
        return out

    def gru_layer(self, layer, state, x):
        x, xp = _f(x)
        self.lib.ref_gru_layer(C.byref(layer), state.ctypes.data_as(F32P), xp)
        return state

    def compute_rnn(self, state, features):
        f, fp = _f(features)
        g, r = np.empty(34, np.float32), np.empty(34, np.float32)
        self.lib.ref_compute_rnn(state.ctypes.data_as(F32P), g.ctypes.data_as(F32P), r.ctypes.data_as(F32P), fp)
        return g, r
