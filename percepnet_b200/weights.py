"""Weight containers for the hot path, in the reference's own two vocabularies.

* ``synth_state_dict`` builds a random-init parameter set with the names and shapes of the
  reference's ``rnn_train.PercepNet`` ``state_dict`` (/root/reference/rnn_train.py:111-121).
  The generator is a counter-based splitmix64 written with numpy integer ops, so the same
  seed gives bit-identical weights on every machine (the GPU box has no /root/reference and
  no checkpoint; see BASELINE.json "random-init weights of that architecture").
* ``pack_state_dict`` applies the layout transforms of the reference's exporter
  (/root/reference/dump_percepnet.py:56-126) and returns the arrays exactly as the generated
  ``src/nnet_data.cpp`` would hold them (SURVEY.md App. B).
* ``PackedModel.as_c_model`` exposes them as a ``pnb_model`` (include/pnb_nnet_layout.h), which
  is layout-compatible with the reference's ``RNNModel`` (/root/reference/src/nnet_data.h:6-26).

Only numpy is needed here; nothing in this module touches the GPU.
"""
from __future__ import annotations

import ctypes as C
import hashlib
from dataclasses import dataclass, field

import numpy as np

ACT_LINEAR, ACT_SIGMOID, ACT_TANH, ACT_RELU = 0, 1, 2, 3

# (name, kind, dims...) in RNNModel field order (nnet_data.h:6-26 == named_children order)
LAYERS = (
    ("fc", "dense", 70, 128, ACT_RELU),
    ("conv1", "conv", 128, 5, 512, ACT_RELU),
    ("conv2", "conv", 512, 3, 512, ACT_TANH),
    ("gru1", "gru", 512, 512),
    ("gru2", "gru", 512, 512),
    ("gru3", "gru", 512, 512),
    ("gru_gb", "gru", 512, 512),
    ("gru_rb", "gru", 1024, 128),
    ("fc_gb", "dense", 2560, 34, ACT_SIGMOID),
    ("fc_rb", "dense", 128, 34, ACT_SIGMOID),
)

N_PARAMS = 7_962_564          # SURVEY.md 0.3
MACS_PER_FRAME = 7_948_288    # SURVEY.md 8(d)


# ----------------------------------------------------------------------------- C structs
class DenseLayerC(C.Structure):
    _fields_ = [("bias", C.POINTER(C.c_float)), ("input_weights", C.POINTER(C.c_float)),
                ("nb_inputs", C.c_int), ("nb_neurons", C.c_int), ("activation", C.c_int)]


class GRULayerC(C.Structure):
    _fields_ = [("bias", C.POINTER(C.c_float)), ("input_weights", C.POINTER(C.c_float)),
                ("recurrent_weights", C.POINTER(C.c_float)), ("nb_inputs", C.c_int),
                ("nb_neurons", C.c_int), ("activation", C.c_int), ("reset_after", C.c_int)]


class Conv1DLayerC(C.Structure):
    _fields_ = [("bias", C.POINTER(C.c_float)), ("input_weights", C.POINTER(C.c_float)),
                ("nb_inputs", C.c_int), ("kernel_size", C.c_int), ("nb_neurons", C.c_int),
                ("activation", C.c_int)]


class ModelC(C.Structure):
    _fields_ = [("fc", C.POINTER(DenseLayerC)), ("conv1", C.POINTER(Conv1DLayerC)),
                ("conv2", C.POINTER(Conv1DLayerC)), ("gru1", C.POINTER(GRULayerC)),
                ("gru2", C.POINTER(GRULayerC)), ("gru3", C.POINTER(GRULayerC)),
                ("gru_gb", C.POINTER(GRULayerC)), ("gru_rb", C.POINTER(GRULayerC)),
                ("fc_gb", C.POINTER(DenseLayerC)), ("fc_rb", C.POINTER(DenseLayerC))]


def _fptr(a: np.ndarray):
    assert a.dtype == np.float32 and a.flags["C_CONTIGUOUS"]
    return a.ctypes.data_as(C.POINTER(C.c_float))


# ----------------------------------------------------------------------------- RNG
_MASK = np.uint64(0xFFFFFFFFFFFFFFFF)


def _splitmix64(x: np.ndarray) -> np.ndarray:
    with np.errstate(over="ignore"):
        z = (x + np.uint64(0x9E3779B97F4A7C15)) & _MASK
        z = ((z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)) & _MASK
        z = ((z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)) & _MASK
        return z ^ (z >> np.uint64(31))


def uniform_pm(shape, seed: int, tag: int, bound: float) -> np.ndarray:
    """float32 uniform in [-bound, bound), element k depends only on (seed, tag, k)."""
    n = int(np.prod(shape))
    with np.errstate(over="ignore"):
        base = _splitmix64(np.array([(seed << 20) ^ (tag * 0x51ED27)], dtype=np.uint64))[0]
        idx = np.arange(n, dtype=np.uint64) + base
    bits = _splitmix64(idx) >> np.uint64(40)                     # 24 random bits
    u = bits.astype(np.float32) * np.float32(2.0 ** -24)         # exact in float32
    return ((u * np.float32(2.0) - np.float32(1.0)) * np.float32(bound)).reshape(shape)


def synth_state_dict(seed: int = 0, gain: float = 1.0) -> dict[str, np.ndarray]:
    """Random-init parameters with PyTorch names/shapes and PyTorch's default init bounds
    (U(+-1/sqrt(fan_in)) for Linear/Conv1d, U(+-1/sqrt(H)) for GRU).  ``gain`` > 1 scales the
    weight matrices (not the biases) to drive activations into saturation for coverage."""
    sd: dict[str, np.ndarray] = {}
    tag = 0

    def nxt(shape, bound, is_weight):
        nonlocal tag
        tag += 1
        return uniform_pm(shape, seed, tag, bound * (gain if is_weight else 1.0))

    for spec in LAYERS:
        name, kind = spec[0], spec[1]
        if kind == "dense":
            m, n = spec[2], spec[3]
            b = 1.0 / np.sqrt(m)
            sd[f"{name}.0.weight"] = nxt((n, m), b, True)
            sd[f"{name}.0.bias"] = nxt((n,), b, False)
        elif kind == "conv":
            c, k, n = spec[2], spec[3], spec[4]
            b = 1.0 / np.sqrt(c * k)
            sd[f"{name}.0.weight"] = nxt((n, c, k), b, True)
            sd[f"{name}.0.bias"] = nxt((n,), b, False)
        else:
            m, h = spec[2], spec[3]
            b = 1.0 / np.sqrt(h)
            sd[f"{name}.weight_ih_l0"] = nxt((3 * h, m), b, True)
            sd[f"{name}.weight_hh_l0"] = nxt((3 * h, h), b, True)
            sd[f"{name}.bias_ih_l0"] = nxt((3 * h,), b, False)
            sd[f"{name}.bias_hh_l0"] = nxt((3 * h,), b, False)
    return sd


# ----------------------------------------------------------------------------- packing
def _gru_kernel(w: np.ndarray) -> np.ndarray:
    """torch [3H, M] with gate rows (r, z, n) -> [M, 3H] with gate columns (z, r, n)
    (dump_percepnet.py:67-76)."""
    r, z, n = np.vsplit(w, 3)
    return np.ascontiguousarray(np.hstack([z.T, r.T, n.T]), dtype=np.float32)


def _gru_bias(b_ih: np.ndarray, b_hh: np.ndarray) -> np.ndarray:
    """cat(bias_ih, bias_hh) -> [b_iz b_ir b_in b_hz b_hr b_hn] (dump_percepnet.py:78-87)."""
    b = np.concatenate([b_ih, b_hh]).reshape(2, 3, -1)
    return np.ascontiguousarray(b[:, [1, 0, 2], :].reshape(-1), dtype=np.float32)


@dataclass
class PackedModel:
    """Arrays in nnet_data.cpp layout, keyed '<layer>_weights' / '_recurrent_weights' / '_bias'."""
    arrays: dict[str, np.ndarray]
    _keep: list = field(default_factory=list, repr=False)
    _c_model: ModelC | None = field(default=None, repr=False)

    def as_c_model(self) -> ModelC:
        if self._c_model is not None:
            return self._c_model
        m = ModelC()
        for spec in LAYERS:
            name, kind = spec[0], spec[1]
            a = self.arrays
            if kind == "dense":
                l = DenseLayerC(_fptr(a[name + "_bias"]), _fptr(a[name + "_weights"]), spec[2], spec[3], spec[4])
            elif kind == "conv":
                l = Conv1DLayerC(_fptr(a[name + "_bias"]), _fptr(a[name + "_weights"]), spec[2], spec[3],
                                 spec[4], spec[5])
            else:
                l = GRULayerC(_fptr(a[name + "_bias"]), _fptr(a[name + "_weights"]),
                              _fptr(a[name + "_recurrent_weights"]), spec[2], spec[3], ACT_TANH, 1)
            self._keep.append(l)
            setattr(m, name, C.pointer(l))
        self._c_model = m
        return m

    BLOB_MAGIC = b"PNBW0001"

    def save_blob(self, path: str) -> None:
        """Binary weight file: magic, then for each of the ten layers in RNNModel order the arrays of the
        generated nnet_data.cpp as float32 (dense/conv: weights, bias; gru: weights, recurrent_weights, bias).
        32 MB instead of the 180 MB C source; read by pnb_model_load_blob / rnnoise_model_from_file."""
        with open(path, "wb") as f:
            f.write(self.BLOB_MAGIC)
            for spec in LAYERS:
                name, kind = spec[0], spec[1]
                keys = [name + "_weights"] + ([name + "_recurrent_weights"] if kind == "gru" else []) + [name + "_bias"]
                for k in keys:
                    a = np.ascontiguousarray(self.arrays[k], dtype="<f4")
                    f.write(np.array([a.size], dtype="<u8").tobytes())
                    f.write(a.tobytes())

    def digest(self) -> str:
        h = hashlib.sha256()
        for k in sorted(self.arrays):
            h.update(k.encode())
            h.update(self.arrays[k].tobytes())
        return h.hexdigest()

    def n_params(self) -> int:
        return int(sum(v.size for v in self.arrays.values()))

    @staticmethod
    def blob_keys() -> list[str]:
        """The array names in PNBW blob order: layers in RNNModel order, each weights, recurrent weights, bias."""
        keys = []
        for spec in LAYERS:
            name = spec[0]
            keys += [name + "_weights"] + ([name + "_recurrent_weights"] if spec[1] == "gru" else []) + [name + "_bias"]
        return keys

    def flat(self) -> np.ndarray:
        """All arrays as one float32 vector in blob order (what pnb_train_export / pnb_train_import move)."""
        return np.concatenate([np.asarray(self.arrays[k], np.float32).reshape(-1) for k in self.blob_keys()])

    @classmethod
    def from_flat(cls, v: np.ndarray) -> "PackedModel":
        """The inverse of flat(): a model from a blob-order vector of N_PARAMS floats."""
        v = np.asarray(v, np.float32).reshape(-1)
        if v.size != N_PARAMS:
            raise ValueError(f"{v.size} floats, a PercepNet model has {N_PARAMS}")
        out, at = {}, 0
        for spec in LAYERS:
            name, kind = spec[0], spec[1]
            if kind == "dense":
                shapes = [(spec[2], spec[3]), (spec[3],)]
            elif kind == "conv":
                shapes = [(spec[3], spec[2], spec[4]), (spec[4],)]
            else:
                shapes = [(spec[2], 3 * spec[3]), (spec[3], 3 * spec[3]), (6 * spec[3],)]
            keys = [name + "_weights"] + ([name + "_recurrent_weights"] if kind == "gru" else []) + [name + "_bias"]
            for k, shp in zip(keys, shapes):
                n = int(np.prod(shp))
                out[k] = v[at:at + n].reshape(shp).copy()
                at += n
        return cls(out)


def pack_state_dict(sd: dict[str, np.ndarray]) -> PackedModel:
    out: dict[str, np.ndarray] = {}
    for spec in LAYERS:
        name, kind = spec[0], spec[1]
        if kind == "dense":       # [N, M] -> [M, N]                     (dump_percepnet.py:62)
            out[name + "_weights"] = np.ascontiguousarray(np.asarray(sd[f"{name}.0.weight"], np.float32).T)
            out[name + "_bias"] = np.ascontiguousarray(sd[f"{name}.0.bias"], dtype=np.float32)
        elif kind == "conv":      # [N, C, K] -> [K, C, N]               (dump_percepnet.py:113)
            out[name + "_weights"] = np.ascontiguousarray(
                np.transpose(np.asarray(sd[f"{name}.0.weight"], np.float32), (2, 1, 0)))
            out[name + "_bias"] = np.ascontiguousarray(sd[f"{name}.0.bias"], dtype=np.float32)
        else:
            out[name + "_weights"] = _gru_kernel(np.asarray(sd[f"{name}.weight_ih_l0"], np.float32))
            out[name + "_recurrent_weights"] = _gru_kernel(np.asarray(sd[f"{name}.weight_hh_l0"], np.float32))
            out[name + "_bias"] = _gru_bias(np.asarray(sd[f"{name}.bias_ih_l0"], np.float32),
                                            np.asarray(sd[f"{name}.bias_hh_l0"], np.float32))
    return PackedModel(out)


def _gru_unkernel(w: np.ndarray) -> np.ndarray:
    """The inverse of _gru_kernel: [M, 3H] with gate columns (z, r, n) -> torch [3H, M] with gate rows (r, z, n)."""
    z, r, n = np.hsplit(np.asarray(w, np.float32), 3)
    return np.ascontiguousarray(np.vstack([r.T, z.T, n.T]), dtype=np.float32)


def unpack_state_dict(pm: PackedModel) -> dict[str, np.ndarray]:
    """The inverse of pack_state_dict: nnet_data.cpp layout back to rnn_train.PercepNet's state_dict names and shapes
    (float32 numpy arrays; torch.from_numpy of each is what dump_percepnet.py reads).  Every transform is a permutation,
    so unpack_state_dict(pack_state_dict(sd)) equals sd bit for bit."""
    a, sd = pm.arrays, {}
    for spec in LAYERS:
        name, kind = spec[0], spec[1]
        if kind == "dense":
            sd[f"{name}.0.weight"] = np.ascontiguousarray(np.asarray(a[name + "_weights"], np.float32).T)
            sd[f"{name}.0.bias"] = np.ascontiguousarray(a[name + "_bias"], dtype=np.float32)
        elif kind == "conv":
            sd[f"{name}.0.weight"] = np.ascontiguousarray(np.transpose(np.asarray(a[name + "_weights"], np.float32), (2, 1, 0)))
            sd[f"{name}.0.bias"] = np.ascontiguousarray(a[name + "_bias"], dtype=np.float32)
        else:
            sd[f"{name}.weight_ih_l0"] = _gru_unkernel(a[name + "_weights"])
            sd[f"{name}.weight_hh_l0"] = _gru_unkernel(a[name + "_recurrent_weights"])
            b = np.asarray(a[name + "_bias"], np.float32).reshape(2, 3, -1)[:, [1, 0, 2], :]
            sd[f"{name}.bias_ih_l0"] = np.ascontiguousarray(b[0].reshape(-1))
            sd[f"{name}.bias_hh_l0"] = np.ascontiguousarray(b[1].reshape(-1))
    return sd


def synth_model(seed: int = 0, gain: float = 1.0) -> PackedModel:
    return pack_state_dict(synth_state_dict(seed, gain))
