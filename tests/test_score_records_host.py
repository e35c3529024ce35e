"""CPU side of device-side scoring (pnb_score_records_*, PNB_NETWORK_ONLY engines) and of eval_records' window and
chunk plans: which frames of which file each stream and each call carries."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT


def _covers(plan, lengths, window):
    """Every file's frames exactly once, in order, in pieces of `window` frames (the last one possibly shorter)."""
    for k, n in enumerate(lengths):
        mine = [(t0, m) for j, t0, m in plan if j == k]
        assert [t0 for t0, _ in mine] == list(np.cumsum([0] + [m for _, m in mine])[:-1])
        assert sum(m for _, m in mine) == n
        step = window or n
        assert all(m == step for _, m in mine[:-1]) and 1 <= mine[-1][1] <= step
    assert [j for j, _, _ in plan] == sorted(j for j, _, _ in plan)   # file order, then frame order


@pytest.mark.parametrize("window", [0, 1, 3, 5, 7, 100])
def test_window_plan_covers_each_file_once(window):
    from percepnet_b200 import eval_records as E
    lengths = [10, 5, 1, 7, 15]
    plan = E.window_plan(lengths, window)
    _covers(plan, lengths, window)
    if window == 0 or window >= max(lengths):
        assert plan == [(k, 0, n) for k, n in enumerate(lengths)]


def test_window_plan_pieces():
    from percepnet_b200 import eval_records as E
    assert E.window_plan([10, 3], 4) == [(0, 0, 4), (0, 4, 4), (0, 8, 2), (1, 0, 3)]
    assert E.window_plan([8], 4) == [(0, 0, 4), (0, 4, 4)]                 # no empty tail
    assert E.window_plan([500, 500], 500) == [(0, 0, 500), (1, 0, 500)]


def test_chunk_frames():
    from percepnet_b200 import eval_records as E
    lengths = [25, 20, 19, 21, 3]
    got = [E.chunk_frames(lengths, t0, 10).tolist() for t0 in range(0, 25, 10)]
    assert got == [[10, 10, 10, 10, 3], [10, 10, 9, 10, 0], [5, 0, 0, 1, 0]]
    assert E.chunk_frames(lengths, 0, 10).dtype == np.int32
    # summed over the calls of a batch, every stream counts exactly its own frames
    assert np.array_equal(sum(E.chunk_frames(lengths, t0, 10) for t0 in range(0, 25, 10)), lengths)
    # a file shorter than one chunk: one call, its own length
    assert E.chunk_frames([4, 2], 0, 100).tolist() == [4, 2]


def test_window_argument():
    from percepnet_b200 import eval_records as E
    assert E.parse_args(["--model", "m", "a"]).window == 0
    assert E.parse_args(["--model", "m", "--window", "500", "a"]).window == 500
    for bad in (["--model", "m", "--window", "-1", "a"], ["--model", "m", "--window", "x", "a"]):
        with pytest.raises(SystemExit):
            E.parse_args(bad)


def test_score_symbols_build_for_sm_90a():
    """The normal build exports the new entry points, and the loss kernel is in the library's sm_90a code."""
    from percepnet_b200 import api, build
    lib = build.build()
    L = api.load_library()
    for name in ("pnb_score_records_device", "pnb_score_records_host", "pnb_engine_bytes"):
        assert hasattr(L, name) and name in api.EXPORTS, name
    assert api.NETWORK_ONLY == 64
    assert L.pnb_engine_bytes(None) == 0
    cuobjdump = os.path.join(os.path.dirname(build._nvcc()), "cuobjdump")
    out = subprocess.run([cuobjdump, "--list-text", lib], capture_output=True, text=True, check=True).stdout
    sections = [ln for ln in out.splitlines() if "loss_sums_kernel" in ln]
    assert len(sections) == 1 and sections[0].rstrip().endswith(".sm_90a.elf.bin"), sections
    name = sections[0].split("-", 1)[1].split(".sm_90a")[0]
    sass = subprocess.run([cuobjdump, "-sass", "-fun", name, lib], capture_output=True, text=True).stdout
    assert "DADD" in sass and "MUFU.RSQ64H" in sass and "SHFL.DOWN" in sass   # float64 sqrt and sums, shuffle tree


def test_header_documents_the_flag():
    hdr = open(os.path.join(ROOT, "include", "percepnet_b200.h")).read()
    assert "PNB_NETWORK_ONLY = 64" in hdr
