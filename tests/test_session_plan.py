"""Residency plan of the session pool (percepnet_b200/csrc/pnb_session_plan.h), compiled on its own with g++: after every
plan the listed sessions occupy slots [0, k) once each, no session is both resident and parked, the row map is a
bijection onto the list, and only sessions that change membership move."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "percepnet_b200", "csrc")

WRAP = r"""
#include "pnb_session_plan.h"
using namespace pnb;
extern "C" {
void *pool_new(int slots, int cap) { SessionPool *p = new SessionPool(); p->init(slots, cap); return p; }
void pool_free(void *p) { delete static_cast<SessionPool *>(p); }
void pool_evict(void *p, int id) { static_cast<SessionPool *>(p)->evict(id); }
int pool_duplicate(void *p, const int *ids, int k) { return static_cast<SessionPool *>(p)->duplicate(ids, k); }
// row: [k]; moves: [slots][4]; where: [cap]; occupant: [slots]; stats: [3]; returns the number of moves
int pool_plan(void *vp, const int *ids, int k, int *row, int *moves, int *where, int *occupant, long long *stats) {
  SessionPool &p = *static_cast<SessionPool *>(vp);
  std::vector<int> r;
  std::vector<SessionMove> m;
  p.plan(ids, k, r, m);
  for (int i = 0; i < k; i++) row[i] = r[i];
  for (size_t j = 0; j < m.size(); j++) { moves[4 * j] = m[j].slot; moves[4 * j + 1] = m[j].park; moves[4 * j + 2] = m[j].fill; moves[4 * j + 3] = m[j].src; }
  for (int s = 0; s < p.capacity(); s++) where[s] = p.where[s];
  for (size_t s = 0; s < p.occupant.size(); s++) occupant[s] = p.occupant[s];
  stats[0] = p.parks; stats[1] = p.unparks; stats[2] = p.relocations;
  return (int)m.size();
}
}
"""

FILL_NONE, FILL_BLOB, FILL_SLOT = 0, 1, 2


@pytest.fixture(scope="module")
def lib(tmp_path_factory):
    d = tmp_path_factory.mktemp("plan")
    src, so = d / "plan.cpp", d / "libplan.so"
    src.write_text(WRAP)
    cxx = "/usr/bin/g++" if os.path.exists("/usr/bin/g++") else "g++"
    subprocess.run([cxx, "-O2", "-std=c++17", "-Wall", "-Werror", "-fPIC", "-shared", "-I", CSRC, str(src), "-o", str(so)],
                   check=True)
    L = C.CDLL(str(so))
    vp, i = C.c_void_p, C.c_int
    L.pool_new.restype = vp
    L.pool_new.argtypes = [i, i]
    L.pool_free.argtypes = [vp]
    L.pool_evict.argtypes = [vp, i]
    L.pool_duplicate.argtypes = [vp, vp, i]
    L.pool_plan.argtypes = [vp, vp, i, vp, vp, vp, vp, vp]
    return L


class Pool:
    def __init__(self, L, slots, cap):
        self.L, self.S, self.cap = L, slots, cap
        self.h = L.pool_new(slots, cap)
        self.where = np.full(cap, -1, np.int32)
        self.occupant = np.full(slots, -1, np.int32)
        self.stats = np.zeros(3, np.int64)

    def plan(self, ids):
        ids = np.ascontiguousarray(ids, np.int32)
        k = len(ids)
        row = np.empty(k, np.int32)
        moves = np.empty((self.S, 4), np.int32)
        stats = np.zeros(3, np.int64)
        nm = self.L.pool_plan(self.h, ids.ctypes.data, k, row.ctypes.data, moves.ctypes.data, self.where.ctypes.data,
                              self.occupant.ctypes.data, stats.ctypes.data)
        delta = stats - self.stats
        self.stats = stats
        return row, moves[:nm].copy(), delta

    def evict(self, id_):
        self.L.pool_evict(self.h, id_)
        s = self.where[id_]                                     # the mirrors (the next plan reads them back)
        if s >= 0:
            self.occupant[s] = -1
            self.where[id_] = -1

    def close(self):
        self.L.pool_free(self.h)


def _check(pool, ids, row, moves, before_where, before_occ, k_prev):
    k = len(ids)
    S, cap = pool.S, pool.cap
    ids = np.asarray(ids)
    # listed sessions occupy [0, k) once each; nothing else is resident
    assert np.array_equal(pool.occupant[:k], ids[row])        # slot p computes list row row[p]
    assert (pool.occupant[k:] == -1).all()
    assert np.array_equal(pool.where[ids[row]], np.arange(k))
    resident = pool.where >= 0
    assert resident.sum() == k and set(np.flatnonzero(resident)) == set(ids.tolist())
    # no session both resident and parked: where and occupant agree exactly
    for s in range(S):
        if pool.occupant[s] >= 0:
            assert pool.where[pool.occupant[s]] == s
    # the row map is a bijection onto the list
    assert sorted(row.tolist()) == list(range(k))
    # the moves: one per slot, fills target [0, k), relocation sources in [k, k_prev), parks are the departed residents
    slots = moves[:, 0]
    assert len(set(slots.tolist())) == len(slots)
    listed = set(ids.tolist())
    parked = {int(m[1]) for m in moves if m[1] >= 0}
    departed = {int(o) for o in before_occ if o >= 0 and int(o) not in listed}
    assert parked == departed
    for slot, park, fill, src in moves:
        if park >= 0:
            assert before_occ[slot] == park
        if fill == FILL_NONE:
            assert slot >= k and park >= 0
        else:
            assert slot < k
            entering = ids[row[slot]]
            if fill == FILL_SLOT:
                assert k <= src < max(k_prev, k) and before_where[entering] == src
            else:
                assert src == entering and before_where[entering] < 0
    stays = sum(1 for i, s in enumerate(ids) if 0 <= before_where[s] < k)
    assert len([m for m in moves if m[2] != FILL_NONE]) == k - stays


def test_random_schedules_keep_the_invariants(lib):
    rng = np.random.RandomState(20261015)
    for S in (1, 2, 7, 64):
        cap = 3 * S
        pool = Pool(lib, S, cap)
        k_prev = 0
        for step in range(10_000 if S == 64 else 1_000):
            r = rng.rand()
            if r < 0.05 and k_prev:                                # an import / reset takes a session out of its slot
                pool.evict(int(rng.choice(np.flatnonzero(pool.where >= 0))))
            prev = np.flatnonzero(pool.where >= 0)
            if r < 0.3 and len(prev):                              # the same set, permuted
                ids = rng.permutation(prev)
            elif r < 0.5 and len(prev):                            # a few dropped, a few added
                keep = rng.permutation(prev)[:max(1, len(prev) - rng.randint(0, 3))]
                new = rng.choice(np.setdiff1d(np.arange(cap), keep), size=min(S - len(keep), rng.randint(0, 3)), replace=False)
                ids = rng.permutation(np.concatenate([keep, new]))
            else:                                                  # any list of 1..S out of 3S
                ids = rng.choice(cap, size=rng.randint(1, S + 1), replace=False)
            bw, bo = pool.where.copy(), pool.occupant.copy()
            row, moves, _ = pool.plan(ids)
            _check(pool, ids, row, moves, bw, bo, max(k_prev, int(np.max(np.flatnonzero(bo >= 0), initial=-1)) + 1))
            k_prev = len(ids)
        pool.close()


def test_move_counts_are_minimal(lib):
    S = 16
    pool = Pool(lib, S, 3 * S)
    base = np.arange(10, 22)                                   # 12 sessions
    _, moves, d = pool.plan(base)
    assert list(d) == [0, 12, 0] and len(moves) == 12         # every session enters once (fresh)
    for perm in range(5):                                      # the same set in any order: nothing moves
        _, moves, d = pool.plan(np.random.RandomState(perm).permutation(base))
        assert len(moves) == 0 and list(d) == [0, 0, 0]
    # one session dropped: one park; listed residents of slots >= k relocate, and nothing else
    cur = pool.occupant[:12].copy()
    drop = cur[3]
    ids = cur[cur != drop]
    _, moves, d = pool.plan(ids)
    assert d[0] == 1 and d[1] == 0 and d[2] == (1 if cur[11] != drop else 0)
    # one session added: one unpark
    ids = np.append(pool.occupant[:11], 40)
    _, moves, d = pool.plan(ids)
    assert list(d) == [0, 1, 0] and len(moves) == 1
    # k shrinking under listed residents: relocations exactly for the listed residents of slots [k, k_prev)
    cur = pool.occupant[:12].copy()
    ids = np.concatenate([cur[:4], cur[8:]])                   # k = 8: cur[8:12] sit in [k, k_prev), cur[4:8] leave
    _, moves, d = pool.plan(ids)
    assert list(d) == [4, 0, 4]
    # a session listed again after a skip comes back from its blob
    _, moves, d = pool.plan(np.append(pool.occupant[:8], cur[5]))
    assert list(d) == [0, 1, 0]
    pool.close()


def test_duplicates_are_found(lib):
    pool = Pool(lib, 8, 24)
    for ids, want in (([1, 2, 3], -1), ([1, 2, 1], 2), ([5, 5], 1), ([0], -1), ([7, 3, 9, 3, 7], 3)):
        a = np.ascontiguousarray(ids, np.int32)
        assert lib.pool_duplicate(pool.h, a.ctypes.data, len(a)) == want
    # the scratch is clean again: a plan afterwards sees no stale marks
    row, moves, d = pool.plan([1, 2, 3])
    assert list(d) == [0, 3, 0]
    pool.close()
