// pnb_chain.cuh -- the schedule both persistent GRU chains share (gru_chain_kernel, pnb_nn_tc.cu; gru_chain_f32_kernel,
// pnb_nn_f32.cu): which layer feeds which, the order in which the blocks of a chain walk its units, and the completion
// counters that make a unit wait for its inputs.
//
// A unit is (hop t, layer l, row block, tile of hidden units).  It depends only on units of the same row block: every
// tile of layer chain_dep(l) at hop t and every tile of its own layer at hop t-1.  Each (layer, row block) has a
// counter that the unit's writers bump with red.release once its stores are issued and that its readers poll with
// ld.acquire.  The grid is fully co-resident and walks the units round-robin in an order in which everything a unit
// waits for comes earlier, so the waits cannot deadlock and no grid barrier or launch boundary is needed between layers
// or hops.
#pragma once
#include "pnb_engine.h"

namespace pnb {

// The layer whose state after hop t is layer l's input at hop t (rnn.cpp:58-71): gru2 <- gru1, gru3 <- gru2, gru_gb
// and gru_rb <- gru3; -1 for gru1, whose input (conv2's output) is complete before the launch.
__host__ __device__ constexpr int chain_dep(int l) { return l == 0 ? -1 : l < 4 ? l - 1 : 2; }

__device__ __forceinline__ unsigned ld_acquire_gpu(const unsigned *p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void red_release_gpu_add(unsigned *p, unsigned v) {
  asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
// Polls the counter at p until it reaches target.  2^26 polls take tens of seconds: a broken schedule becomes a launch
// error, not a hang.
__device__ __forceinline__ void chain_wait(const unsigned *p, unsigned target) {
  unsigned spins = 0;
  while (ld_acquire_gpu(p) < target)
    if (++spins > (1u << 26)) __trap();
}

// The order of a chain's units.  Inside a layer-hop both orders walk row block by row block, tile by tile.
//   hop-major (diag = 0): hop by hop, layer by layer inside a hop.
//   anti-diagonal (diag = 1): (hop t, layer l) sits on diagonal t + depth(l), depth = chain_dep(l) + 1 = 0,1,2,3,3, and
//   the diagonals ascend, layers ascending inside one.  Everything a unit waits for lies on an earlier diagonal, and a
//   diagonal holds up to five layer-hops of mutually independent units -- with few streams one layer-hop alone cannot
//   occupy the blocks.
struct ChainOrder {
  int F;              // hops
  int n_rb;           // row blocks
  int tiles_log2[5];  // log2(tiles of layer l)
  int unit0[5];       // first unit of layer l inside a hop
  int units_per_hop;
  int diag;
  __host__ __device__ int units() const { return F * units_per_hop; }
};
struct ChainUnit { int t, l, rb, tile; };

// F hops of n_rb row blocks whose tiles are ht hidden units wide
inline ChainOrder chain_order(int F, int n_rb, int ht, int diag) {
  ChainOrder o = {};
  o.F = F; o.n_rb = n_rb; o.diag = diag;
  int u = 0;
  for (int l = 0; l < 5; l++) {
    const int tiles = kGruH[l] / ht;
    o.tiles_log2[l] = __builtin_ctz(tiles);
    o.unit0[l] = u;
    u += n_rb * tiles;
  }
  o.units_per_hop = u;
  return o;
}

__device__ __forceinline__ int chain_diag_size(const ChainOrder &o, int d) {
  int n = 0;
#pragma unroll
  for (int l = 0; l < 5; l++) {
    const int t = d - (chain_dep(l) + 1);
    n += (t >= 0 && t < o.F) ? (o.n_rb << o.tiles_log2[l]) : 0;
  }
  return n;
}
__device__ __forceinline__ ChainUnit chain_decode_diag(const ChainOrder &o, int u) {
  int d = 0, r = u;
  bool found = false;
  for (; d < 3 && !found; d++) {  // ramp-up diagonals
    const int sz = chain_diag_size(o, d);
    if (r < sz) { found = true; break; }
    r -= sz;
  }
  if (!found && o.F > 3) {        // full diagonals 3 .. F-1 all hold units_per_hop units
    const int q = r / o.units_per_hop;
    if (q < o.F - 3) { d = 3 + q; r -= q * o.units_per_hop; found = true; }
    else { r -= (o.F - 3) * o.units_per_hop; d = o.F; }
  }
  for (; !found; d++) {           // ramp-down diagonals
    const int sz = chain_diag_size(o, d);
    if (r < sz) break;
    r -= sz;
  }
  ChainUnit x;
  x.l = 0; x.t = 0;
  bool hit = false;
#pragma unroll
  for (int l = 0; l < 5; l++) {
    const int t = d - (chain_dep(l) + 1);
    const int nl = (t >= 0 && t < o.F) ? (o.n_rb << o.tiles_log2[l]) : 0;
    if (!hit) {
      if (r < nl) { x.l = l; x.t = t; hit = true; }
      else r -= nl;
    }
  }
  const int sh = o.tiles_log2[x.l];
  x.rb = r >> sh;
  x.tile = r & ((1 << sh) - 1);
  return x;
}
__device__ __forceinline__ ChainUnit chain_decode(const ChainOrder &o, int u) {
  if (o.diag) return chain_decode_diag(o, u);
  ChainUnit x;
  x.t = u / o.units_per_hop;
  int r = u - x.t * o.units_per_hop;
  x.l = 0;
#pragma unroll
  for (int i = 1; i < 5; i++) x.l = (r >= o.unit0[i]) ? i : x.l;
  r -= o.unit0[x.l];
  const int sh = o.tiles_log2[x.l];
  x.rb = r >> sh;
  x.tile = r & ((1 << sh) - 1);
  return x;
}

}  // namespace pnb
