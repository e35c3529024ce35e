"""CPU side of the split and network calls on a session pool (pnb_analyze_sessions_*, pnb_synthesize_sessions_*,
pnb_compute_rnn_sessions_*): the symbols are declared, mirrored by the Python layer and exported, the row-mapped layout
kernels are in the library's sm_90a code, and the calls refuse an engine handle of NULL without a GPU."""
import os
import re
import subprocess

from conftest import ROOT

NEW = ("pnb_analyze_sessions_device_f32", "pnb_analyze_sessions_device_i16", "pnb_analyze_sessions_host_f32",
       "pnb_analyze_sessions_host_i16", "pnb_synthesize_sessions_device_f32", "pnb_synthesize_sessions_device_i16",
       "pnb_synthesize_sessions_host_f32", "pnb_synthesize_sessions_host_i16", "pnb_compute_rnn_sessions_device",
       "pnb_compute_rnn_sessions_host")


def test_session_split_symbols_are_declared_and_exported():
    from percepnet_b200 import api, build
    lib = build.build()
    hdr = open(os.path.join(ROOT, "include", "percepnet_b200.h")).read()
    declared = set(re.findall(r"\b(pnb_[a-z0-9_]+)\s*\(", hdr))
    out = subprocess.run(["nm", "-D", "--defined-only", lib], capture_output=True, text=True, check=True).stdout
    L = api.load_library()
    for name in NEW:
        assert name in declared and name in api.EXPORTS, name
        assert re.search(r"\bT " + name + r"\b", out), name
        assert hasattr(L, name), name
    for name in ("analyze_sessions", "synthesize_sessions", "compute_rnn_sessions"):
        assert hasattr(api.Engine, name) and hasattr(api.Engine, name + "_device"), name


def test_null_engine_is_refused():
    from percepnet_b200 import api
    L = api.load_library()
    assert L.pnb_analyze_sessions_host_f32(None, None, None, 1, None, 480, 1, None, 70) == -1
    assert L.pnb_synthesize_sessions_host_f32(None, None, 1, None, 68, 1, None, 480) == -1
    assert L.pnb_compute_rnn_sessions_host(None, None, None, 1, 0, None, 70, 1, None, 68) == -1
    assert b"NULL" in L.pnb_last_error()


def test_row_mapped_layout_kernels_build_for_sm_90a():
    """rows_stage_kernel and rows_store_kernel each have the plain and the row-mapped form, for features (70) and g/r
    (68), all in sm_90a code; the row-mapped forms read the map."""
    from percepnet_b200 import build
    lib = build.build()
    cuobjdump = os.path.join(os.path.dirname(build._nvcc()), "cuobjdump")
    listing = subprocess.run([cuobjdump, "--list-text", lib], capture_output=True, text=True, check=True).stdout
    for kernel in ("rows_stage_kernel", "rows_store_kernel"):
        sections = [ln for ln in listing.splitlines() if kernel in ln]
        assert len(sections) == 4, (kernel, sections)                  # W in {68, 70} x map absent / present
        assert all(s.rstrip().endswith(".sm_90a.elf.bin") for s in sections), sections
        names = [s.split("-", 1)[1].split(".sm_90a")[0] for s in sections]
        mapped = [n for n in names if re.search(r"ILi(68|70)ELb1E", n)]
        plain = [n for n in names if re.search(r"ILi(68|70)ELb0E", n)]
        assert len(mapped) == 2 and len(plain) == 2, names
        for name in names:
            sass = subprocess.run([cuobjdump, "-sass", "-fun", name, lib], capture_output=True, text=True).stdout
            assert "STG" in sass and "LDG" in sass, name
