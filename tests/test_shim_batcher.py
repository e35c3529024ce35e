"""Group commit of the pooled rnnoise shim (percepnet_b200/csrc/pnb_shim_batcher.h), compiled on its own with g++ -pthread
and driven by a mock call that sleeps at random and records its batches: every request is in exactly one batch, no batch
exceeds the slot limit, each thread's requests keep their order, no caller returns before its own frame is complete
(input and output are the same buffer), calls never overlap, a failed call reaches every request of its batch, and
the run ends with nothing pending and no leader marked."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "percepnet_b200", "csrc")

FRAME, GRW = 4, 2

WRAP = r"""
#include "pnb_shim_batcher.h"
#include <atomic>
#include <chrono>
#include <random>
#include <thread>
using namespace pnb;

static const int FRAME = 4, GRW = 2;

struct Log {
  std::atomic<int> in_call{0};
  std::atomic<int> overlap{0}, bad_ids{0};
  int fail_every = 0;
  long long n_calls = 0;
  std::vector<int> sizes, entries, rcs;   // per call: size, rc; per batch row: t * n_req + s
};

struct Mock {
  Log *log;
  unsigned seed;
  int operator()(const int *ids, int k, const float *in, float *out, float *gr, std::string &err) const {
    if (log->in_call.fetch_add(1) != 0) log->overlap++;
    std::mt19937 rng(seed + (unsigned)log->n_calls * 7919u);
    int us = (int)(rng() % 120);
    if (us > 20) std::this_thread::sleep_for(std::chrono::microseconds(us));
    const long long call = log->n_calls++;
    const int rc = (log->fail_every && call % log->fail_every == 3) ? -7 : 0;
    log->sizes.push_back(k);
    log->rcs.push_back(rc);
    for (int i = 0; i < k; i++) {
      const float *x = in + i * FRAME;
      if (ids[i] != (int)x[0]) log->bad_ids++;
      log->entries.push_back((int)x[0] * 100000 + (int)x[1]);
      for (int j = 0; j < FRAME; j++) out[i * FRAME + j] = 2.f * x[j] + 1.f;
      gr[i * GRW] = x[0];
      gr[i * GRW + 1] = x[1];
    }
    if (rc) err = "mock call " + std::to_string(call) + " failed";
    log->in_call.fetch_sub(1);
    return rc;
  }
};

extern "C" {
// Runs n_thr threads x n_req requests through one batcher of `slots`.  Outputs: sizes[calls], entries[frames],
// call_rc[calls]; req_rc[n_thr * n_req] the code each caller got; req_err[n_thr * n_req] 1 when a failed request's text
// names its call; checks[0..5] = {overlapping calls, wrong ids, callers that returned before their frame was complete,
// pending at the end, leader marked at the end, largest batch in the stats}, stats[3] = calls, frames, largest.
// Returns the number of calls.
int run(int n_thr, int n_req, int slots, unsigned seed, int fail_every, int *sizes, int *entries, int *call_rc,
        int *req_rc, int *req_err, long long *checks, long long *stats) {
  Log log;
  log.fail_every = fail_every;
  FrameBatcher<Mock> b(Mock{&log, seed}, slots, FRAME, GRW);
  std::atomic<int> early{0};
  std::vector<std::thread> th;
  for (int t = 0; t < n_thr; t++)
    th.emplace_back([&, t]() {
      std::mt19937 rng(seed * 31u + (unsigned)t);
      for (int s = 0; s < n_req; s++) {
        float buf[FRAME] = {(float)t, (float)s, 7.f, -1.f};
        float gr[GRW] = {-5.f, -5.f};
        std::string err;
        int rc = b.process(t, buf, buf, gr, &err);   // in == out, as src/main.cpp passes them
        req_rc[t * n_req + s] = rc;
        req_err[t * n_req + s] = 0;
        if (rc == 0) {
          bool ok = buf[0] == 2.f * t + 1.f && buf[1] == 2.f * s + 1.f && buf[2] == 15.f && buf[3] == -1.f &&
                    gr[0] == (float)t && gr[1] == (float)s;
          if (!ok) early++;
        } else {
          req_err[t * n_req + s] = err.compare(0, 10, "mock call ") == 0;
        }
        int us = (int)(rng() % 60);
        if (us > 30) std::this_thread::sleep_for(std::chrono::microseconds(us - 30));
      }
    });
  for (auto &x : th) x.join();
  for (size_t i = 0; i < log.sizes.size(); i++) { sizes[i] = log.sizes[i]; call_rc[i] = log.rcs[i]; }
  for (size_t i = 0; i < log.entries.size(); i++) entries[i] = log.entries[i];
  BatcherStats st = b.stats();
  checks[0] = log.overlap; checks[1] = log.bad_ids; checks[2] = early;
  checks[3] = b.pending(); checks[4] = b.leading(); checks[5] = st.largest;
  stats[0] = st.calls; stats[1] = st.frames; stats[2] = st.largest;
  return (int)log.sizes.size();
}
}
"""


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    d = tmp_path_factory.mktemp("batcher")
    src, so = d / "batcher.cpp", d / "libbatcher.so"
    src.write_text(WRAP)
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    # the shim builds as C++11; the mock uses C++11 only too
    subprocess.run([cxx, "-O2", "-std=c++11", "-pthread", "-Wall", "-Werror", "-fPIC", "-shared", "-I", CSRC, str(src),
                    "-o", str(so)], check=True)
    L = C.CDLL(str(so))
    L.run.argtypes = [C.c_int, C.c_int, C.c_int, C.c_uint, C.c_int] + [C.c_void_p] * 7
    return L


def _run(L, n_thr, n_req, slots, seed, fail_every=0):
    total = n_thr * n_req
    sizes, call_rc = np.zeros(total, np.int32), np.zeros(total, np.int32)
    entries = np.zeros(total, np.int32)
    req_rc, req_err = np.zeros(total, np.int32), np.zeros(total, np.int32)
    checks, stats = np.zeros(6, np.int64), np.zeros(3, np.int64)
    n_calls = L.run(n_thr, n_req, slots, seed, fail_every, sizes.ctypes.data, entries.ctypes.data, call_rc.ctypes.data,
                    req_rc.ctypes.data, req_err.ctypes.data, checks.ctypes.data, stats.ctypes.data)
    sizes, call_rc = sizes[:n_calls], call_rc[:n_calls]
    assert sizes.sum() == total
    return sizes, entries, call_rc, req_rc.reshape(n_thr, n_req), req_err.reshape(n_thr, n_req), checks, stats


@pytest.mark.parametrize("slots", [1, 3, 64])
def test_group_commit_under_contention(lib, slots):
    n_thr, n_req = 64, 500
    sizes, entries, call_rc, req_rc, _, checks, stats = _run(lib, n_thr, n_req, slots, seed=1000 + slots)
    overlap, bad_ids, early, pending, leading, largest = checks.tolist()
    assert overlap == 0 and bad_ids == 0
    assert early == 0, "a caller returned before its own frame was complete"
    assert pending == 0 and leading == 0, "the run ended with requests pending or a leader marked"
    assert (call_rc == 0).all() and (req_rc == 0).all()
    # every request in exactly one batch
    t, s = entries // 100000, entries % 100000
    key = t * n_req + s
    assert np.array_equal(np.sort(key), np.arange(n_thr * n_req))
    # no batch above the slot limit; the stats agree with the log
    assert sizes.max() <= slots and sizes.min() >= 1
    assert stats.tolist() == [len(sizes), n_thr * n_req, sizes.max()] and largest == sizes.max()
    # each thread's requests in its own order, within and across batches
    for th in range(n_thr):
        assert np.array_equal(s[t == th], np.arange(n_req)), th
    # a thread has at most one request pending, so a batch never holds two of one thread
    bounds = np.concatenate([[0], np.cumsum(sizes)])
    for a, b in zip(bounds[:-1], bounds[1:]):
        assert len(np.unique(t[a:b])) == b - a
    if slots > 1:
        assert sizes.max() > 1, "64 contending threads never shared a call"


def test_failed_call_reaches_its_whole_batch(lib):
    n_thr, n_req = 16, 60
    sizes, entries, call_rc, req_rc, req_err, checks, _ = _run(lib, n_thr, n_req, 5, seed=7, fail_every=5)
    assert checks[3] == 0 and checks[4] == 0 and checks[0] == 0 and checks[2] == 0
    assert (call_rc != 0).any() and (call_rc == 0).any()
    t, s = entries // 100000, entries % 100000
    want = np.repeat(call_rc, sizes)                 # the code of the call each request went through
    got = req_rc[t, s]
    assert np.array_equal(got, want)
    assert (req_err[t, s][want != 0] == 1).all()     # with the failing call's text
