"""The pitch stage at its decision boundaries, on CPU: the edge corpus of tests/golden/make_pitch_edges.py.

* On every corpus row, the oracle's pitch_downsample -> pitch_search -> remove_doubling returns the lag, corr, T and
  gain the reference returned (stored in the fixture), and the live reference still returns them where it is built.
* Every comparison mutant of tests/pitch_mutants.py, compiled from pn_oracle.c with oracle/Makefile's flags, is told
  apart from the original by some row, so an edit that weakens the fixture fails here rather than going unnoticed.
"""
import os

import numpy as np
import pytest

import pitch_mutants as pm
from conftest import GOLDEN
from util import same_bits


@pytest.fixture(scope="module")
def corpus():
    return dict(np.load(os.path.join(GOLDEN, "pitch_edges.npz")))


def _stored(c):
    return c["lag"], c["corr"], c["T"], c["gain"]


def test_corpus_shape(corpus):
    n = corpus["buf"].shape[0]
    assert corpus["buf"].shape == (n, 1728) and corpus["buf"].dtype == np.float32
    assert np.isfinite(corpus["buf"]).all()
    for k in ("prev_period", "prev_gain", "lag", "corr", "T", "gain"):
        assert corpus[k].shape == (n,)


def test_oracle_matches_reference_outputs(oracle, corpus):
    got = pm.pitch_outputs(oracle, corpus["buf"], corpus["prev_period"], corpus["prev_gain"])
    for name, a, b in zip(("lag", "corr", "T", "gain"), got, _stored(corpus)):
        ok = same_bits(a, b) if a.dtype.kind == "f" else np.array_equal(a, b)
        assert ok, (name, np.nonzero(a != b)[0])


def test_live_reference_matches_stored(reference, corpus):
    got = pm.pitch_outputs(reference, corpus["buf"], corpus["prev_period"], corpus["prev_gain"])
    assert not pm.differs(got, _stored(corpus)).any()


@pytest.fixture(scope="module")
def mutant_libs(tmp_path_factory):
    from oracle.ffi import Oracle
    d = tmp_path_factory.mktemp("pitch_mutants")
    return {k: Oracle(v) for k, v in pm.build_all(str(d)).items()}


def test_unmutated_build_matches_stored(mutant_libs, corpus):
    """the temporary build itself is the oracle: without a mutation it reproduces the stored outputs"""
    got = pm.pitch_outputs(mutant_libs[None], corpus["buf"], corpus["prev_period"], corpus["prev_gain"])
    assert not pm.differs(got, _stored(corpus)).any()


@pytest.mark.parametrize("name", list(pm.MUTANTS))
def test_corpus_kills_mutant(mutant_libs, corpus, name):
    got = pm.pitch_outputs(mutant_libs[name], corpus["buf"], corpus["prev_period"], corpus["prev_gain"])
    killed = pm.differs(got, _stored(corpus))
    assert killed.any(), f"mutant {name} ({pm.MUTANTS[name][2]}) survives the pitch edge corpus"
