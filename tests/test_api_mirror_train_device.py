"""The Python mirror of include/pnb_train_device.h, on the CPU: its signature table agrees with every prototype of that
header, the library exports each symbol, the header compiles as strict C99 and as C++11 on its own and through
percepnet_b200.h, and none of its symbols is declared in percepnet_b200.h as well."""
import ctypes as C
import os
import re
import subprocess

import pytest

from conftest import ROOT

INC = os.path.join(ROOT, "include")
KINDS = {"int": (C.c_int,), "size_t": (C.c_size_t,)}


@pytest.fixture(scope="module")
def api():
    from percepnet_b200 import api, build
    build.build()
    return api


def _prototypes(header):
    """{name: (return type, [parameter types])} of every pnb_* prototype in the header, with '*' for any pointer."""
    hdr = open(os.path.join(INC, header)).read()
    hdr = re.sub(r"/\*.*?\*/", " ", hdr, flags=re.S)
    hdr = "\n".join(line for line in hdr.splitlines() if not line.lstrip().startswith("#"))

    def kind(decl, named):
        decl = re.sub(r"\bconst\b", " ", decl)
        if "*" in decl:
            return "*"
        words = decl.split()
        return " ".join(words[:-1] if named else words)

    protos = {}
    for ret, name, params in re.findall(r"([\w\s*]+?)\b(pnb_[a-z0-9_]+)\s*\(([^()]*)\)\s*;", hdr):
        params = [p for p in params.split(",") if p.strip() not in ("", "void")]
        protos[name] = (kind(ret, False), [kind(p, True) for p in params])
    return protos


def test_library_types_match_every_prototype(api):
    protos = _prototypes("pnb_train_device.h")
    assert set(protos) == {"pnb_train_forward_device", "pnb_train_backward_device"} == set(api.TRAIN_DEVICE_EXPORTS)
    assert not set(protos) & set(_prototypes("percepnet_b200.h")) and not set(protos) & set(api.EXPORTS)
    L = api.load_library()
    for name, (ret, params) in protos.items():
        f = getattr(L, name)
        assert ret == "int" and f.restype is C.c_int, name
        assert len(f.argtypes) == len(params), (name, params, f.argtypes)
        for k, (p, t) in enumerate(zip(params, f.argtypes)):
            assert (t is C.c_void_p) if p == "*" else t in KINDS[p], (name, k, p, t)


@pytest.mark.parametrize("first", ["pnb_train_device.h", "percepnet_b200.h"])
def test_header_is_plain_c(tmp_path, first):
    """Either header first: both declare everything, as C99 and as C++11."""
    src = tmp_path / "hdr.c"
    src.write_text(f'#include "{first}"\n'
                   "int main(void) { int (*f)(pnb_engine *, const float *, size_t, float *, size_t, float *, void *) = "
                   "pnb_train_backward_device; (void)f; (void)pnb_train_forward_device; return PNB_TAP_TRAIN_DPRE; }\n")
    cc = "/usr/bin/gcc" if os.path.exists("/usr/bin/gcc") else "gcc"
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.run([cc, "-std=c99", "-pedantic", "-Wall", "-Werror", "-fsyntax-only", "-I", INC, str(src)], check=True)
    subprocess.run([cxx, "-std=c++11", "-Wall", "-Werror", "-fsyntax-only", "-x", "c++", "-I", INC, str(src)], check=True)
