"""Pooled rnnoise shim (PNB_SHIM_POOL=<slots>): handles of one model, network mode and device are sessions of one shared
engine, and frames of concurrent threads are batched into one session call.  librnnoise_b200.so is driven through the
C++-mangled names an unmodified src/main.cpp imports, with synth_model weights as the model and a libc FILE* for the
g/r file.  Every pooled handle is compared bit for bit -- PCM and g/r -- against an unpooled handle created in the same
process (one engine per handle, the shim's default) and fed the same frames."""
import ctypes as C
import os
import subprocess
import threading

import numpy as np
import pytest

from conftest import ROOT

pytestmark = pytest.mark.gpu

FRAME = 480
SHIM_PATH = os.path.join(ROOT, "percepnet_b200", "librnnoise_b200.so")
REF_BIN = os.path.join(ROOT, "oracle", "_ref", "percepNet_run_ref")
B200_BIN = os.path.join(ROOT, "oracle", "_ref", "percepNet_run_b200")


class Shim:
    def __init__(self):
        L = C.CDLL(SHIM_PATH)
        vp = C.c_void_p
        self.get_size = L._Z16rnnoise_get_sizev
        self.get_size.restype = C.c_int
        self.init = L._Z12rnnoise_initP12DenoiseStateP8RNNModel
        self.init.argtypes, self.init.restype = [vp, vp], C.c_int
        self.create = L._Z14rnnoise_createP8RNNModel
        self.create.argtypes, self.create.restype = [vp], vp
        self.destroy = L._Z15rnnoise_destroyP12DenoiseState
        self.destroy.argtypes, self.destroy.restype = [vp], None
        self.process = L._Z21rnnoise_process_frameP12DenoiseStatePfPKfP8_IO_FILE
        self.process.argtypes, self.process.restype = [vp, vp, vp, vp], C.c_float
        self.pool_stats = L.pnb_shim_pool_stats
        self.pool_stats.argtypes = [vp]
        libc = C.CDLL(None)
        self.fopen, self.fclose = libc.fopen, libc.fclose
        self.fopen.argtypes, self.fopen.restype = [C.c_char_p, C.c_char_p], vp
        self.fclose.argtypes = [vp]
        self.malloc, self.free = libc.malloc, libc.free
        self.malloc.argtypes, self.malloc.restype = [C.c_size_t], vp
        self.free.argtypes = [vp]

    def stats(self) -> dict:
        a = (C.c_longlong * 6)()
        assert self.pool_stats(a) == 0
        return dict(zip(("groups", "calls", "frames", "largest", "parks", "unparks"), (int(v) for v in a)))


@pytest.fixture(scope="module")
def shim():
    import torch
    if not torch.cuda.is_available():
        pytest.fail("-m gpu tests need a CUDA device")
    from percepnet_b200 import build
    build.build()
    return Shim()


@pytest.fixture
def env():
    """Sets PNB_SHIM_POOL / PNB_SHIM_NN between creates and restores them afterwards."""
    saved = {k: os.environ.get(k) for k in ("PNB_SHIM_POOL", "PNB_SHIM_NN")}

    def setenv(pool=None, nn=None):
        for k, v in (("PNB_SHIM_POOL", pool), ("PNB_SHIM_NN", nn)):
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = str(v)
    yield setenv
    setenv(saved["PNB_SHIM_POOL"], saved["PNB_SHIM_NN"])


def _addr(model):
    return C.addressof(model.as_c_model())


class Handle:
    """A shim handle with its own g/r file; feed() runs one frame the way src/main.cpp does (in == out)."""

    def __init__(self, shim, model, path, st=None):
        self.shim = shim
        self.st = st if st is not None else shim.create(_addr(model))
        assert self.st, "rnnoise_create returned NULL"
        self.path = path
        self.f = shim.fopen(path.encode(), b"wb")
        assert self.f
        self.buf = np.zeros(FRAME, np.float32)
        self.out = []

    def feed(self, frame):
        self.buf[:] = frame
        self.shim.process(self.st, self.buf.ctypes.data, self.buf.ctypes.data, self.f)
        self.out.append(self.buf.copy())

    def close(self):
        self.shim.fclose(self.f)
        self.shim.destroy(self.st)
        pcm = np.concatenate(self.out) if self.out else np.zeros(0, np.float32)
        gr = np.fromfile(self.path, dtype=np.float32).reshape(-1, 68)
        return pcm, gr


def _signals(n, n_frames, seed):
    """n distinct signals, half at the CLI's amplitude scale, half at int16 scale (pitch_filter's comb branch runs)."""
    from percepnet_b200.synth import synth_pcm
    a = synth_pcm(n, n_frames, seed=seed)
    b = synth_pcm(n, n_frames, seed=seed, scale=32768.0)
    return np.where((np.arange(n) % 2 == 0)[:, None], a, b).astype(np.float32)


def _feed_threaded(groups, frames):
    """groups: one list of (handle, row) per thread; every thread feeds its handles frame by frame."""
    n_frames = frames.shape[1] // FRAME
    errors = []

    def work(items):
        try:
            for t in range(n_frames):
                for h, row in items:
                    h.feed(frames[row, t * FRAME:(t + 1) * FRAME])
        except Exception as ex:  # re-raised in the main thread
            errors.append(ex)

    th = [threading.Thread(target=work, args=(g,)) for g in groups]
    for t in th:
        t.start()
    for t in th:
        t.join()
    assert not errors, errors


def _assert_same(a, b, what):
    assert a[0].shape == b[0].shape and a[1].shape == b[1].shape, what
    assert np.array_equal(a[0].view(np.int32), b[0].view(np.int32)), f"{what}: PCM differs"
    assert np.array_equal(a[1].view(np.int32), b[1].view(np.int32)), f"{what}: g/r differs"


def _unpooled(shim, env, model, frames, tmp_path, tag, nn=None):
    env(pool=None, nn=nn)
    res = []
    for k in range(frames.shape[0]):
        h = Handle(shim, model, str(tmp_path / f"{tag}_plain{k}.raw"))
        for t in range(frames.shape[1] // FRAME):
            h.feed(frames[k, t * FRAME:(t + 1) * FRAME])
        res.append(h.close())
    return res


@pytest.mark.parametrize("nn", ["fp32", "tensor"])
def test_pooled_threads_match_unpooled(shim, env, model0, tmp_path, nn):
    n_thr, per, n_frames = 8, 4, 150
    frames = _signals(n_thr * per, n_frames, seed=3100 if nn == "fp32" else 3200)
    want = _unpooled(shim, env, model0, frames, tmp_path, nn, nn=nn)
    s0 = shim.stats()
    assert s0["groups"] == 0
    env(pool=16, nn=nn)
    handles = [Handle(shim, model0, str(tmp_path / f"{nn}_pool{k}.raw")) for k in range(n_thr * per)]
    assert shim.stats()["groups"] == 1
    _feed_threaded([[(handles[t * per + j], t * per + j) for j in range(per)] for t in range(n_thr)], frames)
    s1 = shim.stats()
    for k, h in enumerate(handles):
        _assert_same(h.close(), want[k], f"{nn} handle {k}")
    assert shim.stats()["groups"] == 0
    assert s1["frames"] - s0["frames"] == n_thr * per * n_frames
    assert s1["largest"] <= max(16, s0["largest"])   # the hook's largest batch is process-wide


def test_more_handles_than_slots(shim, env, model0, tmp_path):
    n, n_frames = 24, 60
    frames = _signals(n, n_frames, seed=3300)
    want = _unpooled(shim, env, model0, frames, tmp_path, "many")
    s0 = shim.stats()
    env(pool=8)
    handles = [Handle(shim, model0, str(tmp_path / f"many_pool{k}.raw")) for k in range(n)]
    _feed_threaded([[(handles[k], k)] for k in range(n)], frames)
    s1 = shim.stats()
    for k, h in enumerate(handles):
        _assert_same(h.close(), want[k], f"handle {k}")
    calls, advanced = s1["calls"] - s0["calls"], s1["frames"] - s0["frames"]
    assert advanced == n * n_frames
    assert s1["parks"] > 0, "24 sessions on 8 slots never parked"
    assert calls < advanced, "24 threads never shared a call"
    assert s1["largest"] <= max(8, s0["largest"])


def test_lifecycle(shim, env, model0, tmp_path):
    from percepnet_b200.weights import synth_model
    model1 = synth_model(1)
    n_frames = 20
    frames = _signals(10, 2 * n_frames, seed=3400)
    half = n_frames * FRAME
    assert shim.stats()["groups"] == 0

    # reference runs, one engine per handle: rows 0..5 over both halves; rows 6, 7 (the recycled handles) and row 8
    # (the caller-buffer handle) over the second half only, from a fresh start; row 9 on model1
    want = _unpooled(shim, env, model0, frames[:6], tmp_path, "life_a")
    want += _unpooled(shim, env, model0, frames[6:9, half:], tmp_path, "life_b")
    want += _unpooled(shim, env, model1, frames[9:10], tmp_path, "life_c")

    env(pool=4)                                      # 6 handles on a pool of 4 sessions: the pool grows to 8
    hs = [Handle(shim, model0, str(tmp_path / f"life_pool{k}.raw")) for k in range(6)]
    other = Handle(shim, model1, str(tmp_path / "life_pool9.raw"))
    assert shim.stats()["groups"] == 2               # two models, two groups
    _feed_threaded([[(hs[k], k)] for k in range(6)] + [[(other, 9)]], frames[:, :half])

    # destroy two handles mid-run; two new handles get their ids back and must start fresh
    gone = [hs[1].close(), hs[3].close()]
    new = [Handle(shim, model0, str(tmp_path / f"life_new{k}.raw")) for k in range(2)]
    # rnnoise_init on a caller-owned buffer of rnnoise_get_size() bytes (malloc'd: rnnoise_destroy frees it)
    buf = shim.malloc(shim.get_size())
    assert shim.init(buf, _addr(model0)) == 0
    mine = Handle(shim, model0, str(tmp_path / "life_init.raw"), st=buf)
    assert shim.stats()["groups"] == 2

    items = [[(hs[k], k)] for k in (0, 2, 4, 5)] + [[(new[0], 6)], [(new[1], 7)], [(mine, 8)], [(other, 9)]]
    _feed_threaded(items, frames[:, half:])

    for k in (0, 2, 4, 5):
        _assert_same(hs[k].close(), want[k], f"handle {k}")
    for k, g in zip((1, 3), gone):                   # the destroyed handles ran the first half exactly
        pcm, gr = want[k]
        _assert_same(g, (pcm[:half], gr[:n_frames]), f"destroyed handle {k}")
    _assert_same(new[0].close(), want[6], "recycled handle 0")
    _assert_same(new[1].close(), want[7], "recycled handle 1")
    _assert_same(mine.close(), want[8], "rnnoise_init handle")
    assert shim.stats()["groups"] == 1
    _assert_same(other.close(), want[9], "model1 handle")
    assert shim.stats()["groups"] == 0


def test_refused_pool_values(shim, env, model0):
    g0 = shim.stats()["groups"]
    for bad in ("-1", "abc", "4097", "3x", ""):
        env(pool=bad)
        assert not shim.create(_addr(model0)), bad
        buf = shim.malloc(shim.get_size())
        assert shim.init(buf, _addr(model0)) != 0, bad
        shim.free(buf)
    env(pool=0)                                      # 0 is the default: one engine per handle, no group
    st = shim.create(_addr(model0))
    assert st and shim.stats()["groups"] == g0
    shim.destroy(st)


def _run_cli(binary, pcm16, workdir, extra_env):
    os.makedirs(workdir, exist_ok=True)
    pcm16.tofile(os.path.join(workdir, "in.pcm"))
    e = {k: v for k, v in os.environ.items() if k not in ("PNB_SHIM_POOL", "PNB_SHIM_NN")}
    e.update(extra_env)
    subprocess.run([binary, "in.pcm", "out.pcm"], cwd=workdir, check=True, timeout=300, env=e)
    with open(os.path.join(workdir, "out.pcm"), "rb") as f:
        out = f.read()
    with open(os.path.join(workdir, "feature_test.raw"), "rb") as f:
        gr = f.read()
    return out, gr


@pytest.mark.skipif(not (os.path.exists(REF_BIN) and os.path.exists(B200_BIN)), reason="make -C oracle refbin not run")
def test_unmodified_cli_pooled(tmp_path):
    from percepnet_b200.synth import synth_pcm, to_int16
    x16 = to_int16(synth_pcm(1, 60, seed=2024)[0])
    ref_out, ref_gr = _run_cli(REF_BIN, x16, str(tmp_path / "ref"), {})
    ref_out = np.frombuffer(ref_out, np.int16).astype(np.int32)
    ref_gr = np.frombuffer(ref_gr, np.float32)
    for nn in ("fp32", "tensor"):
        plain = _run_cli(B200_BIN, x16, str(tmp_path / f"plain_{nn}"), {"PNB_SHIM_NN": nn})
        pooled = _run_cli(B200_BIN, x16, str(tmp_path / f"pool_{nn}"), {"PNB_SHIM_NN": nn, "PNB_SHIM_POOL": "4"})
        assert pooled[0] == plain[0] and pooled[1] == plain[1], nn   # out.pcm and feature_test.raw byte for byte
        out = np.frombuffer(pooled[0], np.int16).astype(np.int32)
        gr = np.frombuffer(pooled[1], np.float32)
        assert out.shape == ref_out.shape == ((60 - 1) * 480,)
        assert np.abs(out - ref_out).max() <= 1, nn
        assert (np.abs(gr - ref_gr) / np.maximum(np.abs(ref_gr), 1e-6)).max() < 1e-4, nn
