// pnb_session_plan.h -- the residency plan of a session pool (pnb_sessions_reserve / pnb_process_sessions_*): which slot
// each listed session computes in, which residents are parked, which are moved between slots.  Host code only, with no
// CUDA dependency, so that it can be compiled and tested on its own.
//
// A session is resident in one slot or parked as a blob.  After every call the residents are exactly that call's list,
// in slots [0, k).  A call with a list of k sessions keeps every listed resident of a slot < k where it is, parks every
// resident that is not listed, moves a listed resident of a slot >= k into a freed slot < k, and unparks every other
// listed session into a freed slot.  The same set in another order moves nothing: the row map (slot -> list row) absorbs
// the order.
#pragma once
#include <vector>

namespace pnb {

// How a slot is filled after its occupant was parked (if any): not at all, from the entering session's parking blob
// (a fresh or rejected session's blob says so, and the slot is reset), or by a raw copy of another slot.
enum SessionFill : int { kFillNone = 0, kFillBlob = 1, kFillSlot = 2 };
// One slot's part of a call's state launch; four ints, uploaded as they are.
struct SessionMove {
  int slot;  // the engine slot written (and read first when park >= 0)
  int park;  // the session parked from `slot` before it is filled, or -1
  int fill;  // SessionFill
  int src;   // kFillBlob: the entering session; kFillSlot: the source slot (>= k, so nothing in the launch writes it)
};

struct SessionPool {
  std::vector<int> where;     // [capacity] slot of a resident session, -1 when parked
  std::vector<int> occupant;  // [slots] session resident in a slot, -1 when free
  std::vector<int> listed;    // [capacity] scratch of plan(): list row of a session, -1 when not listed
  int hi = 0;                 // every occupied slot is below hi
  long long parks = 0, unparks = 0, relocations = 0;

  // Every session parked (and fresh: the engine marks its blobs), every slot free.
  void init(int slots, int capacity) {
    where.assign(capacity, -1);
    listed.assign(capacity, -1);
    occupant.assign(slots, -1);
    hi = 0;
  }
  // More sessions, all parked; the existing ones keep their places.
  void grow(int capacity) {
    if (capacity <= (int)where.size()) return;
    where.resize(capacity, -1);
    listed.resize(capacity, -1);
  }
  int capacity() const { return (int)where.size(); }
  // The first i whose ids[i] repeats an earlier entry of ids[0..k) (all in range), or -1.
  int duplicate(const int *ids, int k) {
    int dup = -1;
    for (int i = 0; i < k && dup < 0; i++) {
      if (listed[ids[i]] >= 0) dup = i;
      else listed[ids[i]] = i;
    }
    for (int i = 0; i < k; i++) listed[ids[i]] = -1;
    return dup;
  }
  // The session no longer has a slot (its slot's content is abandoned): its state is its blob from now on.
  void evict(int id) {
    const int s = where[id];
    if (s < 0) return;
    occupant[s] = -1;
    where[id] = -1;
  }

  // The plan of a call that advances the k distinct sessions ids[0..k) (in range: the caller checks).  row[p] = list row
  // computed in slot p, p < k; moves: one entry per slot that is written or parked, slots < k first.  Applies the plan.
  void plan(const int *ids, int k, std::vector<int> &row, std::vector<SessionMove> &moves) {
    row.assign(k, -1);
    moves.clear();
    for (int i = 0; i < k; i++) {
      listed[ids[i]] = i;
      const int s = where[ids[i]];
      if (s >= 0 && s < k) row[s] = i;  // stays
    }
    int p = 0;  // next free slot < k
    for (int i = 0; i < k; i++) {
      const int id = ids[i], s = where[id];
      if (s >= 0 && s < k) continue;
      while (row[p] >= 0) p++;
      const int o = occupant[p];  // not listed: a listed occupant of a slot < k stays there
      moves.push_back(SessionMove{p, o, s >= 0 ? kFillSlot : kFillBlob, s >= 0 ? s : id});
      row[p] = i;
    }
    const size_t n_fill = moves.size();
    for (int q = k; q < hi; q++) {
      const int o = occupant[q];
      if (o >= 0 && listed[o] < 0) moves.push_back(SessionMove{q, o, kFillNone, -1});
    }
    // apply
    for (size_t j = 0; j < moves.size(); j++) {
      const SessionMove &m = moves[j];
      if (m.park >= 0) {
        where[m.park] = -1;
        parks++;
      }
      if (m.fill == kFillSlot) {
        occupant[m.src] = -1;
        relocations++;
      } else if (m.fill == kFillBlob) {
        unparks++;
      }
      if (j < n_fill) {
        const int id = ids[row[m.slot]];
        occupant[m.slot] = id;
        where[id] = m.slot;
      } else {
        occupant[m.slot] = -1;
      }
    }
    for (int i = 0; i < k; i++) listed[ids[i]] = -1;
    hi = k;
  }
};

}  // namespace pnb
