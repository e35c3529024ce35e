"""The Python mirror of the C ABI, on the CPU: its signature table agrees with every prototype of
include/percepnet_b200.h, and the host methods refuse arrays and lists the library would misread before the library
is called.  The refusals run on an Engine whose handle is NULL: the library answers every call on it with "engine is
NULL", so any other refusal was made in Python."""
import ctypes as C
import os
import re

import numpy as np
import pytest

from conftest import ROOT

# C parameter and return types -> the ctypes types that pass them unchanged
KINDS = {"int": (C.c_int,), "unsigned": (C.c_uint,), "size_t": (C.c_size_t,), "long long": (C.c_longlong,),
         "double": (C.c_double,)}


@pytest.fixture(scope="module")
def api():
    from percepnet_b200 import api, build
    build.build()
    return api


def _prototypes():
    """{name: (return type, [parameter types])} of every pnb_* prototype in the header, with '*' for any pointer."""
    hdr = open(os.path.join(ROOT, "include", "percepnet_b200.h")).read()
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


def _same_kind(c_type, ctype):
    if c_type == "*":
        return ctype in (C.c_void_p, C.c_char_p) or issubclass(ctype, C._Pointer)
    return ctype in KINDS[c_type]


def test_library_types_match_every_prototype(api):
    """What load_library() sets on each symbol: as many parameters as the prototype, each of the same kind, and the
    same kind of return value."""
    protos = _prototypes()
    assert len(protos) == 87 and set(protos) == set(api.EXPORTS)
    L = api.load_library()
    for name, (ret, params) in protos.items():
        f = getattr(L, name)
        assert (f.restype is None) if ret == "void" else _same_kind(ret, f.restype), (name, ret, f.restype)
        assert f.argtypes is not None and len(f.argtypes) == len(params), (name, params, f.argtypes)
        for k, (p, t) in enumerate(zip(params, f.argtypes)):
            assert _same_kind(p, t), (name, k, p, t)


@pytest.fixture()
def null(api):
    """An Engine on a NULL handle: no active rows, and every library call refused with "engine is NULL"."""
    e = object.__new__(api.Engine)
    e.L, e.h = api.load_library(), None
    assert e.active == 0
    return e


def _refused(api, exc, call, *words):
    with pytest.raises(exc) as ei:
        call()
    msg = str(ei.value)
    assert "engine is NULL" not in msg, msg
    for w in words:
        assert w in msg, msg


def _reaches_library(api, call):
    with pytest.raises(api.PnbError, match="engine is NULL"):
        call()


def test_submit_refuses_what_it_cannot_pass_through(api, null):
    f64 = np.zeros((0, 480))
    _refused(api, TypeError, lambda: null.submit(f64, f64.copy()), "float32 or int16")
    strided = np.zeros((1, 960), np.float32)[:, ::2]
    _refused(api, api.PnbError, lambda: null.submit(strided, strided.copy()), "contiguous")
    odd = np.zeros((0, 500), np.float32)
    _refused(api, api.PnbError, lambda: null.submit(odd, odd.copy()), "F*480")
    _refused(api, api.PnbError, lambda: null.submit(np.zeros((0, 480), np.float32), np.zeros((0, 480), np.int16)),
             "same shape and dtype")
    _reaches_library(api, lambda: null.submit(np.zeros((0, 480), np.int16), np.zeros((0, 480), np.int16)))


@pytest.mark.parametrize("method, rows, width, good", [
    ("process", (1, 480), (0, 500), (0, 480)),
    ("analyze", (1, 480), (0, 500), (0, 480)),
    ("synthesize", (1, 2, 68), (0, 2, 67), (0, 2, 68)),
    ("compute_rnn", (1, 2, 70), (0, 2, 71), (0, 2, 138)),
    ("score_records", (1, 2, 138), (0, 2, 137), (0, 2, 138)),
    ("train_grad", (1, 2, 138), (0, 2, 137), (0, 2, 138)),
])
def test_host_arrays_are_checked_before_the_call(api, null, method, rows, width, good):
    f = getattr(null, method)
    _refused(api, api.PnbError, lambda: f(np.zeros(rows, np.float32)), "1 rows for 0")
    _refused(api, api.PnbError, lambda: f(np.zeros(width, np.float32)), "must be [active, F")
    _reaches_library(api, lambda: f(np.zeros(good, np.float32)))


@pytest.mark.parametrize("bad", [2 ** 32 + 3, 1.7])
def test_list_entries_are_not_wrapped_or_truncated(api, null, bad):
    F = int(bad) % 2 ** 32                       # the hop count the entry would have become
    _refused(api, api.PnbError, lambda: null.reset_streams([0, bad]), "idx")
    _refused(api, api.PnbError, lambda: null.reset_sessions([bad]), "ids")
    _refused(api, api.PnbError, lambda: null.process_sessions([0], np.zeros((1, F * 480), np.float32), hops=[bad]),
             "hops")
    _refused(api, api.PnbError, lambda: null.score_records_device(0, 138, 1, [bad], 0), "frames")


def test_valid_lists_reach_the_library(api, null):
    for idx in ([], [0], [2 ** 31 - 1, -2 ** 31], np.arange(3), np.arange(3, dtype=np.uint16), (np.int64(5),)):
        _reaches_library(api, lambda: null.reset_streams(idx))
    _reaches_library(api, lambda: null.process_sessions(np.array([4, 1]), np.zeros((2, 960), np.int16), hops=[2, 1]))
    _reaches_library(api, lambda: null.score_records_device(0, 138, 1, None, 0))
