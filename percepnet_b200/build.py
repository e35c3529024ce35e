"""In-tree build of the CUDA libraries for sm_90a (H100; nvcc cross-compiles without a GPU).

  percepnet_b200/libpercepnet_b200.so   kernels + C-ABI (include/percepnet_b200.h), static cudart
  percepnet_b200/librnnoise_b200.so     the reference's rnnoise.h API (C++ linkage) on top of it
"""
from __future__ import annotations

import os
import shutil
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OBJ = os.path.join(HERE, "_build")
LIB = os.path.join(HERE, "libpercepnet_b200.so")
SHIM = os.path.join(HERE, "librnnoise_b200.so")

ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]
COMMON = ["-O3", "-std=c++17", "-lineinfo", "-Xcompiler", "-fPIC", "-Xptxas", "-v"]
# per-file extra flags: the DSP unit must not contract a*b+c (bit-exact pitch decisions, SURVEY.md H1)
SOURCES = {
    "pnb_dsp.cu": ["-fmad=false"],
    "pnb_nn_f32.cu": [],
    "pnb_nn_tc.cu": [],
    "pnb_engine.cu": [],
    "pnb_state.cu": [],
    "pnb_rnn_io.cu": [],
    "pnb_train.cu": [],
}


def _nvcc() -> str:
    for c in (os.environ.get("NVCC"), "/usr/local/cuda/bin/nvcc", shutil.which("nvcc")):
        if c and os.path.exists(c):
            return c
    raise RuntimeError("nvcc not found")


def _newer(src_list, out):
    if not os.path.exists(out):
        return True
    t = os.path.getmtime(out)
    return any(os.path.getmtime(s) > t for s in src_list)


def build(force: bool = False, verbose: bool = False) -> str:
    os.makedirs(OBJ, exist_ok=True)
    nvcc = _nvcc()
    headers = [os.path.join(CSRC, f) for f in os.listdir(CSRC) if f.endswith((".h", ".cuh"))]
    headers += [os.path.join(HERE, "..", "include", f) for f in os.listdir(os.path.join(HERE, "..", "include"))]
    objs = []
    log = []
    for src, extra in SOURCES.items():
        sp = os.path.join(CSRC, src)
        op = os.path.join(OBJ, src.replace(".cu", ".o"))
        objs.append(op)
        if force or _newer([sp] + headers + [__file__], op):
            cmd = [nvcc, *ARCH, *COMMON, *extra, "-c", sp, "-o", op]
            r = subprocess.run(cmd, capture_output=True, text=True)
            log.append(f"$ {' '.join(cmd)}\n{r.stdout}{r.stderr}")
            if r.returncode != 0:
                sys.stderr.write(log[-1])
                raise RuntimeError(f"nvcc failed on {src}")
    if force or _newer(objs, LIB):
        cmd = [nvcc, *ARCH, "-shared", "-cudart", "static", "-o", LIB, *objs]
        r = subprocess.run(cmd, capture_output=True, text=True)
        log.append(f"$ {' '.join(cmd)}\n{r.stdout}{r.stderr}")
        if r.returncode != 0:
            sys.stderr.write(log[-1])
            raise RuntimeError("link failed")
    shim_src = os.path.join(CSRC, "rnnoise_shim.cpp")
    if force or _newer([shim_src, os.path.join(CSRC, "pnb_shim_batcher.h"), LIB, __file__], SHIM):
        cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
        # -pthread: pooled handles (PNB_SHIM_POOL) batch frames of concurrent threads under std::mutex
        cmd = [cxx, "-O2", "-std=c++11", "-pthread", "-fPIC", "-shared", "-o", SHIM, shim_src, "-L" + HERE,
               "-lpercepnet_b200", "-Wl,-rpath,$ORIGIN"]
        r = subprocess.run(cmd, capture_output=True, text=True)
        log.append(f"$ {' '.join(cmd)}\n{r.stdout}{r.stderr}")
        if r.returncode != 0:
            sys.stderr.write(log[-1])
            raise RuntimeError("shim link failed")
    with open(os.path.join(OBJ, "build.log"), "a") as f:
        f.write("\n".join(log))
    if verbose:
        print("\n".join(log))
    return LIB


def build_timing() -> str:
    """libpercepnet_b200_timing.so: the same library with -DPNB_ANA_TIMING in pnb_dsp.cu (per-section cycle
    accounting of analysis_kernel, read by tools/analysis_sections.py).  Debug aid, not loaded by the product."""
    build()
    nvcc = _nvcc()
    obj = os.path.join(OBJ, "pnb_dsp_timing.o")
    out = os.path.join(HERE, "libpercepnet_b200_timing.so")
    subprocess.run([nvcc, *ARCH, *COMMON, *SOURCES["pnb_dsp.cu"], "-DPNB_ANA_TIMING", "-c", os.path.join(CSRC, "pnb_dsp.cu"),
                    "-o", obj], check=True, capture_output=True)
    others = [os.path.join(OBJ, f.replace(".cu", ".o")) for f in SOURCES if f != "pnb_dsp.cu"]
    subprocess.run([nvcc, *ARCH, "-shared", "-cudart", "static", "-o", out, obj, *others], check=True, capture_output=True)
    return out


if __name__ == "__main__":
    if "--timing" in sys.argv:
        print(build_timing())
    else:
        build(force="--force" in sys.argv, verbose=True)
