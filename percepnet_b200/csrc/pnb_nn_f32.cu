// pnb_nn_f32.cu -- the gain network in fp32 FMA (BASELINE.json config 2), batched over streams.
//
// The reference evaluates the network one stream at a time as 35 GEMVs per hop
// (/root/reference/src/nnet.cpp:59-72, vec.h:102-135, rnn.cpp:42-81) and re-reads all 31.9 MB of
// weights for every hop.  Here the rows of every contraction are the concurrent streams, so each
// weight tile is reused across 128 streams from shared memory; activations use the reference's
// tansig table approximation (vec.h:53-76).  Per chunk of hops: fc, conv1, conv2 over all rows of the chunk
// (gemm_f32_kernel), the five GRUs of all its hops in one persistent launch (gru_chain_f32_kernel), the output layers,
// and a carry.  The host side at the end of the file is the path's part of the engine: its weights and buffers
// (pnb_f32_state), and the hooks the engine calls (f32_prepare, f32_network, f32_state_segs).
#include <string.h>

#include <string>

#include "pnb_chain.cuh"
#include "pnb_engine.h"

namespace pnb {

// One contraction  C[M x N] = epilogue( sum_seg A_seg[M x K_seg] * B_seg[K_seg x N] ).
// A segments are activation matrices (row = stream), B segments are slices of the reference's
// input-major weight arrays (row = input j, column = output i: W[j*ldb + i]).  With an active range the rows are the
// first M of each of n_slots hop slots.
struct GemmSeg {
  const float *A;
  int lda;
  const float *B;
  int ldb;
  int K;  // multiple of 16
};
struct GemmArgs {
  GemmSeg seg[5];
  int n_seg;
  int M, N;           // M: rows per hop slot (all n_slots x M rows when n_slots = 1 and the rows are one flat range)
  int n_slots;        // hop slots; the rows of slot k start at row k * slot_stride of A and C
  int slot_stride;
  float *C;
  int ldc;
  const float *bias;  // null -> raw sums
  int act;            // PNB_ACT_* applied when bias != null
  const float *tansig;
};

// The five GRUs of a chunk of hops in one persistent fp32 launch.  Slot buffers: hop t of the chunk
// reads state slot t and writes slot t+1; inputs are conv2's output slot t or the layer below's slot t+1.
struct F32ChainLayer {
  int H, n_x, dep;            // hidden size; input segments (1 or 2); chain_dep of the layer
  const float *x[2];          // input buffers [slots][S][x_ld]
  int x_ld[2], x_K[2], x_slot1[2];
  size_t x_slot_stride[2];    // floats per hop slot of the input buffer
  const float *W, *U, *bias;  // reference layout: W [K_in][3H], U [H][3H], bias [6H]
  int ldw, w_row0[2];         // 3H; first row of W for each input segment
  float *h;                   // [(n+1) slots][S][H]
};
constexpr int kF32ChainMaxHops = 32;  // hops per launch of the fp32 chain (longer chunks amortise the ramp diagonals)
struct F32ChainArgs {
  F32ChainLayer L[5];
  ChainOrder order;  // anti-diagonal: the chunk's hops of the active streams' blocks, 32-unit tiles
  int S, n;          // rows per slot; active streams [0, n)
  unsigned *cnt;     // [5][order.n_rb] finished tiles per (layer, stream block), zero at launch
  const float *tansig;
};

__device__ __forceinline__ float tansig_approx(float x, const float *__restrict__ tbl) {  // vec.h:53-71
  float sign = 1.f;
  if (x < 0.f) { x = -x; sign = -1.f; }
  float fi = floorf(.5f + 25.f * x);
  // the reference converts with x86 cvttss2si, which yields INT_MIN when out of range or NaN (then the
  // clamp below lands on 0, not 200): keep that for |x| >= 8.6e7 so both sides leave the table the same way
  int i = (fi < 2147483648.f) ? (int)fi : (int)0x80000000;
  i = i < 200 ? i : 200;
  i = i > 0 ? i : 0;
  x -= .04f * i;
  float y = __ldg(tbl + i);
  float dy = 1.f - y * y;
  y = y + x * dy * (1.f - y * x);
  return sign * y;
}
__device__ __forceinline__ float sigmoid_approx(float x, const float *__restrict__ tbl) {  // vec.h:73-76
  return .5f + .5f * tansig_approx(.5f * x, tbl);
}
__device__ __forceinline__ float activate(float v, int act, const float *__restrict__ tbl) {
  if (act == PNB_ACT_SIGMOID) return sigmoid_approx(v, tbl);
  if (act == PNB_ACT_TANH) return tansig_approx(v, tbl);
  if (act == PNB_ACT_RELU) return v < 0.f ? 0.f : v;
  return v;
}

// Pairs of neighbouring accumulators / columns: two IEEE fp32 FMAs, one per element (Hopper has no packed fp32 FMA).
typedef float2 f32x2;
__device__ __forceinline__ void ffma2(f32x2 &d, f32x2 a, f32x2 b) {
  d.x = fmaf(a.x, b.x, d.x);
  d.y = fmaf(a.y, b.y, d.y);
}
__device__ __forceinline__ f32x2 pack2(float x, float y) { return make_float2(x, y); }
__device__ __forceinline__ float2 unpack2(f32x2 v) { return v; }

constexpr int BM = 128, BN = 64, BK = 16, APAD = 4;

template <bool VEC_B>
__global__ void __launch_bounds__(256) gemm_f32_kernel(GemmArgs g) {
  __shared__ __align__(16) float As[2][BK][BM + APAD];
  __shared__ __align__(16) float Bs[2][BK][BN];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  // row tiles per hop slot; rows [m_lim - M, m_lim) are the slot's (one flat range when n_slots = 1)
  const int tiles_slot = (int)(gridDim.y / (unsigned)g.n_slots), slot = blockIdx.y / tiles_slot;
  const int m0 = slot * g.slot_stride + (blockIdx.y - slot * tiles_slot) * BM, n0 = blockIdx.x * BN;
  const int m_lim = slot * g.slot_stride + g.M;

  f32x2 acc[8][2];  // 8 rows x 2 pairs of columns
#pragma unroll
  for (int i = 0; i < 8; i++) { acc[i][0] = make_float2(0.f, 0.f); acc[i][1] = acc[i][0]; }

  // global->register staging: A 2 x float4 per thread, B 1 x float4 per thread
  const int a_row = tid >> 2, a_kq = (tid & 3) * 4;  // rows a_row and a_row+64
  const int b_k = tid >> 4, b_n = (tid & 15) * 4;
  float4 ra0, ra1, rb;

  int seg = 0, koff = 0;
  int total_tiles = 0;
  for (int i = 0; i < g.n_seg; i++) total_tiles += g.seg[i].K / BK;

  auto fetch = [&](int sg, int k0) {
    const GemmSeg &S = g.seg[sg];
    int r0 = m0 + a_row, r1 = r0 + 64;
    ra0 = r0 < m_lim ? *reinterpret_cast<const float4 *>(S.A + (size_t)r0 * S.lda + k0 + a_kq)
                   : make_float4(0.f, 0.f, 0.f, 0.f);
    ra1 = r1 < m_lim ? *reinterpret_cast<const float4 *>(S.A + (size_t)r1 * S.lda + k0 + a_kq)
                   : make_float4(0.f, 0.f, 0.f, 0.f);
    const float *bp = S.B + (size_t)(k0 + b_k) * S.ldb + n0 + b_n;
    if (VEC_B) {
      rb = (n0 + b_n < g.N) ? __ldg(reinterpret_cast<const float4 *>(bp)) : make_float4(0.f, 0.f, 0.f, 0.f);
    } else {
      rb.x = (n0 + b_n + 0 < g.N) ? __ldg(bp + 0) : 0.f;
      rb.y = (n0 + b_n + 1 < g.N) ? __ldg(bp + 1) : 0.f;
      rb.z = (n0 + b_n + 2 < g.N) ? __ldg(bp + 2) : 0.f;
      rb.w = (n0 + b_n + 3 < g.N) ? __ldg(bp + 3) : 0.f;
    }
  };
  auto stash = [&](int buf) {
    As[buf][a_kq + 0][a_row] = ra0.x; As[buf][a_kq + 1][a_row] = ra0.y;
    As[buf][a_kq + 2][a_row] = ra0.z; As[buf][a_kq + 3][a_row] = ra0.w;
    As[buf][a_kq + 0][a_row + 64] = ra1.x; As[buf][a_kq + 1][a_row + 64] = ra1.y;
    As[buf][a_kq + 2][a_row + 64] = ra1.z; As[buf][a_kq + 3][a_row + 64] = ra1.w;
    *reinterpret_cast<float4 *>(&Bs[buf][b_k][b_n]) = rb;
  };

  fetch(0, 0);
  stash(0);
  __syncthreads();
  for (int tile = 0; tile < total_tiles; tile++) {
    const int buf = tile & 1;
    // advance (seg, koff) to the next tile and prefetch it
    int nseg = seg, nk = koff + BK;
    if (nk >= g.seg[seg].K) { nseg = seg + 1; nk = 0; }
    const bool more = tile + 1 < total_tiles;
    if (more) fetch(nseg, nk);
#pragma unroll
    for (int k = 0; k < BK; k++) {
      float4 a0 = *reinterpret_cast<const float4 *>(&As[buf][k][ty * 8]);
      float4 a1 = *reinterpret_cast<const float4 *>(&As[buf][k][ty * 8 + 4]);
      const float4 b4 = *reinterpret_cast<const float4 *>(&Bs[buf][k][tx * 4]);  // columns {0,1} and {2,3} as pairs
      const f32x2 bx = make_float2(b4.x, b4.y), by = make_float2(b4.z, b4.w);
      const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
#pragma unroll
      for (int i = 0; i < 8; i++) {
        const f32x2 aa = pack2(av[i], av[i]);
        ffma2(acc[i][0], aa, bx);
        ffma2(acc[i][1], aa, by);
      }
    }
    if (more) stash(buf ^ 1);
    __syncthreads();
    seg = nseg;
    koff = nk;
  }

#pragma unroll
  for (int i = 0; i < 8; i++) {
    int r = m0 + ty * 8 + i;
    if (r >= m_lim) continue;
    const float2 p0 = unpack2(acc[i][0]), p1 = unpack2(acc[i][1]);
    const float accv[4] = {p0.x, p0.y, p1.x, p1.y};
#pragma unroll
    for (int j = 0; j < 4; j++) {
      int c = n0 + tx * 4 + j;
      if (c >= g.N) continue;
      float v = accv[j];
      if (g.bias) v = activate(v + __ldg(g.bias + c), g.act, g.tansig);
      g.C[(size_t)r * g.ldc + c] = v;
    }
  }
}

void launch_gemm_f32(const GemmArgs &g, cudaStream_t st) {
  dim3 grid((g.N + BN - 1) / BN, g.n_slots * ((g.M + BM - 1) / BM));
  bool vec = true;
  for (int i = 0; i < g.n_seg; i++)
    if ((g.seg[i].ldb & 3) || (reinterpret_cast<uintptr_t>(g.seg[i].B) & 15)) vec = false;
  if (vec) gemm_f32_kernel<true><<<grid, 256, 0, st>>>(g);
  else gemm_f32_kernel<false><<<grid, 256, 0, st>>>(g);
}

// fc 70 -> 128 (+relu): one thread per (stream, output); the 70-float feature row is broadcast, the
// weight row W[j*128 + i] is coalesced over i.
__global__ void __launch_bounds__(128) fc_f32_kernel(const float *__restrict__ feat, const float *__restrict__ W,
                                                     const float *__restrict__ bias, float *__restrict__ out,
                                                     int M, int K, int N, size_t slot_stride) {
  __shared__ float f[4][72];
  const int r0 = blockIdx.x * 4;
  feat += blockIdx.y * slot_stride * K;  // hop slot blockIdx.y
  out += blockIdx.y * slot_stride * N;
  for (int i = threadIdx.x; i < 4 * K; i += blockDim.x) {
    int rr = i / K, kk = i % K;
    f[rr][kk] = (r0 + rr < M) ? feat[(size_t)(r0 + rr) * K + kk] : 0.f;
  }
  __syncthreads();
  const int n = threadIdx.x;
  if (n >= N) return;
  float a0 = bias[n], a1 = a0, a2 = a0, a3 = a0;
  for (int k = 0; k < K; k++) {
    float w = __ldg(W + (size_t)k * N + n);
    a0 = fmaf(w, f[0][k], a0);
    a1 = fmaf(w, f[1][k], a1);
    a2 = fmaf(w, f[2][k], a2);
    a3 = fmaf(w, f[3][k], a3);
  }
  float a[4] = {a0, a1, a2, a3};
  for (int rr = 0; rr < 4; rr++)
    if (r0 + rr < M) out[(size_t)(r0 + rr) * N + n] = a[rr] < 0.f ? 0.f : a[rr];
}

void launch_fc_f32(const float *feat, const float *W, const float *bias, float *out, int M, int K, int N, int n_slots,
                   size_t slot_stride, cudaStream_t st) {
  fc_f32_kernel<<<dim3((M + 3) / 4, n_slots), 128, 0, st>>>(feat, W, bias, out, M, K, N, slot_stride);
}

// ------------------------------------------------------------------------------------------------------------------
// The five GRUs of a chunk of hops in ONE persistent fp32 launch (BASELINE.json config 2: "persistent-kernel GRU, fp32").
//
// Unit of work = (hop t, layer l, block of BM streams, tile of 32 hidden units): the four gate sums z, r, W_n x, U_n h of
// 32 hidden units for BM streams (nnet.cpp:120-180 keeps the last two apart), as one register-tiled FMA contraction over
// [x ; h], then the gate math and the state update in the same thread -- no pre-activation ever goes to memory.
// State slot t of h_all[l] is the state BEFORE hop t of the chunk, slot t+1 the state after it: a layer reads slot t of
// its own buffer and slot t+1 of the layer below (the freshly updated state, rnn.cpp:58-71), so nothing is overwritten
// inside a launch.  Dependencies, counters and the unit order are the tensor chain's (pnb_chain.cuh), always in
// anti-diagonal order.
// The accumulation order of every sum (ascending k, x segments first, then h, one FMA per term) is the one the
// per-layer kernels above use.
// ------------------------------------------------------------------------------------------------------------------
namespace {
constexpr int CH_BK = 32, CH_HT = 32, CH_BN = 3 * CH_HT, CH_STAGES = 3, CH_THREADS = 256;  // 32-k tiles: one block barrier per 32 k
constexpr int CH_APAD = CH_BK + 4;  // row stride of the A tile in floats: 16-byte aligned rows, conflict-free 128-bit reads

__device__ __forceinline__ void cp_async16(void *smem, const void *gmem, bool valid) {
  const unsigned sa = (unsigned)__cvta_generic_to_shared(smem);
  const int n = valid ? 16 : 0;  // src-size 0: the 16 bytes are zero-filled, nothing is read
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(sa), "l"(gmem), "r"(n) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory"); }

template <int RT>  // rows per thread: 8 (128-stream blocks) or 1 (16-stream blocks, for a handful of streams)
struct ChainSmem {
  static constexpr int BM = 16 * RT;
  float A[CH_STAGES][BM][CH_APAD];
  float B[CH_STAGES][CH_BK][CH_BN];
};

// one k-tile of FMAs: acc_z/acc_r/acc_n[i] (pairs of hidden units) += A[row i][k] * B[k][gate][pair]
template <int RT>
__device__ __forceinline__ void chain_tile_fma(const float (*As)[CH_APAD], const float (*Bs)[CH_BN], int ty, int tx,
                                               f32x2 (&az)[RT], f32x2 (&ar)[RT], f32x2 (&an)[RT]) {
#pragma unroll
  for (int kk = 0; kk < CH_BK; kk += 4) {
    float4 a[RT];
#pragma unroll
    for (int i = 0; i < RT; i++) a[i] = *reinterpret_cast<const float4 *>(&As[ty + 16 * i][kk]);  // rows ty, ty+16, ..: a warp's two rows are neighbours (different banks)
#pragma unroll
    for (int q = 0; q < 4; q++) {
      const f32x2 bz = *reinterpret_cast<const f32x2 *>(&Bs[kk + q][2 * tx]);
      const f32x2 br = *reinterpret_cast<const f32x2 *>(&Bs[kk + q][CH_HT + 2 * tx]);
      const f32x2 bn = *reinterpret_cast<const f32x2 *>(&Bs[kk + q][2 * CH_HT + 2 * tx]);
#pragma unroll
      for (int i = 0; i < RT; i++) {
        const float av = q == 0 ? a[i].x : q == 1 ? a[i].y : q == 2 ? a[i].z : a[i].w;
        const f32x2 aa = pack2(av, av);
        ffma2(az[i], aa, bz);
        ffma2(ar[i], aa, br);
        ffma2(an[i], aa, bn);
      }
    }
  }
}

template <int RT>
__global__ void __launch_bounds__(CH_THREADS, RT == 8 ? 2 : 4) gru_chain_f32_kernel(const __grid_constant__ F32ChainArgs args) {
  using SM = ChainSmem<RT>;
  constexpr int BM = SM::BM;
  extern __shared__ __align__(16) unsigned char chain_smem_raw[];
  SM &sm = *reinterpret_cast<SM *>(chain_smem_raw);
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int S = args.S, n_rb = args.order.n_rb;

  for (int u = blockIdx.x; u < args.order.units(); u += gridDim.x) {
    const ChainUnit un = chain_decode(args.order, u);
    const int t = un.t, l = un.l, rb = un.rb;
    const F32ChainLayer &L = args.L[l];
    const int tiles = L.H / CH_HT;
    const int j0 = un.tile * CH_HT, m0 = rb * BM;

    // ---- dependencies (one thread polls; the barrier publishes the result to the block)
    if (tid == 0) {
      if (L.dep >= 0) chain_wait(args.cnt + L.dep * n_rb + rb, (unsigned)(t + 1) * (unsigned)(args.L[L.dep].H / CH_HT));
      if (t > 0) chain_wait(args.cnt + l * n_rb + rb, (unsigned)t * (unsigned)tiles);
    }
    __syncthreads();

    // ---- the contraction over [x segments ; h]
    f32x2 az[RT], ar[RT], anx[RT], anh[RT];  // pairs of neighbouring hidden units
#pragma unroll
    for (int i = 0; i < RT; i++) { az[i] = make_float2(0.f, 0.f); ar[i] = az[i]; anx[i] = az[i]; anh[i] = az[i]; }

    const int n_seg = L.n_x + 1;
    int kt_total = 0;
    for (int sg = 0; sg < n_seg; sg++) kt_total += (sg < L.n_x ? L.x_K[sg] : L.H) / CH_BK;

    // issue the loads of k-tile `kt` (global tile index over all segments) into stage kt % CH_STAGES
    auto issue = [&](int kt) {
      int sg = 0, k0 = kt * CH_BK;
      while (sg < L.n_x && k0 >= L.x_K[sg]) { k0 -= L.x_K[sg]; sg++; }
      const bool rec = sg == L.n_x;
      const float *Ab = rec ? L.h + (size_t)t * S * L.H : L.x[sg] + (size_t)(t + L.x_slot1[sg]) * L.x_slot_stride[sg];
      const int lda = rec ? L.H : L.x_ld[sg];
      const float *Bb = rec ? L.U : L.W + (size_t)L.w_row0[sg] * L.ldw;
      const int st = kt % CH_STAGES;
      // A: BM rows x CH_BK/4 chunks of 16 bytes
      constexpr int CPR = CH_BK / 4;
      for (int c = tid; c < BM * CPR; c += CH_THREADS) {
        const int r = c / CPR, q = c - r * CPR;
        const bool ok = m0 + r < args.n;
        cp_async16(&sm.A[st][r][q * 4], Ab + (size_t)(ok ? m0 + r : 0) * lda + k0 + q * 4, ok);
      }
      // B: CH_BK k-rows x 3 gates x 8 chunks
      for (int c = tid; c < CH_BK * 24; c += CH_THREADS) {
        const int kr = c / 24, rem = c - kr * 24, g = rem >> 3, q = rem & 7;
        cp_async16(&sm.B[st][kr][g * CH_HT + q * 4], Bb + (size_t)(k0 + kr) * L.ldw + g * L.H + j0 + q * 4, true);
      }
    };
    for (int p = 0; p < CH_STAGES - 1; p++) {
      if (p < kt_total) issue(p);
      cp_async_commit();
    }
    const int kt_x = kt_total - L.H / CH_BK;  // tiles before the recurrent segment
    for (int kt = 0; kt < kt_total; kt++) {
      cp_async_wait<CH_STAGES - 2>();
      __syncthreads();  // tile kt has landed for every thread; the stage read in iteration kt-1 is free again
      if (kt + CH_STAGES - 1 < kt_total) issue(kt + CH_STAGES - 1);
      cp_async_commit();
      const int st = kt % CH_STAGES;
      if (kt < kt_x) chain_tile_fma<RT>(sm.A[st], sm.B[st], ty, tx, az, ar, anx);
      else chain_tile_fma<RT>(sm.A[st], sm.B[st], ty, tx, az, ar, anh);
    }
    cp_async_wait<0>();

    // ---- gates and state update (nnet.cpp:120-180 with reset_after: z, r from the summed sums, n = tanh(b_n + (b'_n + U_n h) r + W_n x))
    {
      const float *b = L.bias;
      const int H = L.H;
      const float *h_old = L.h + (size_t)t * S * H;
      float *h_new = L.h + (size_t)(t + 1) * S * H;
      const int j = j0 + 2 * tx;
      float bz[2], br[2], bn[2], bnh[2];
#pragma unroll
      for (int c = 0; c < 2; c++) {
        bz[c] = __ldg(b + j + c) + __ldg(b + 3 * H + j + c);
        br[c] = __ldg(b + H + j + c) + __ldg(b + 4 * H + j + c);
        bn[c] = __ldg(b + 2 * H + j + c);
        bnh[c] = __ldg(b + 5 * H + j + c);
      }
#pragma unroll
      for (int i = 0; i < RT; i++) {
        const int m = m0 + ty + 16 * i;
        if (m >= args.n) continue;
        const float2 ho = __ldcg(reinterpret_cast<const float2 *>(h_old + (size_t)m * H + j));
        const float2 sz = unpack2(az[i]), sr = unpack2(ar[i]), snx = unpack2(anx[i]), snh = unpack2(anh[i]);
        float out[2];
#pragma unroll
        for (int c = 0; c < 2; c++) {
          const float z = sigmoid_approx(bz[c] + (c == 0 ? sz.x : sz.y), args.tansig);
          const float r = sigmoid_approx(br[c] + (c == 0 ? sr.x : sr.y), args.tansig);
          const float tmp = bnh[c] + (c == 0 ? snh.x : snh.y);
          float cc = bn[c] + tmp * r;
          cc = cc + (c == 0 ? snx.x : snx.y);
          const float n = tansig_approx(cc, args.tansig);
          const float h = c == 0 ? ho.x : ho.y;
          out[c] = z * h + (1.f - z) * n;
        }
        *reinterpret_cast<float2 *>(h_new + (size_t)m * H + j) = make_float2(out[0], out[1]);
      }
    }
    __syncthreads();  // every thread's stores are issued (and the tile buffers are free for the next unit)
    if (tid == 0) {
      __threadfence();
      red_release_gpu_add(args.cnt + l * n_rb + rb, 1u);
    }
  }
}
}  // namespace

size_t f32_chain_smem(int rt) { return rt == 8 ? sizeof(ChainSmem<8>) : sizeof(ChainSmem<1>); }

// Returns false, launching nothing, when the kernel cannot be configured.
bool launch_gru_chain_f32(const F32ChainArgs &a, int rt, int sm_count, cudaStream_t st) {
  static int occ8 = 0, occ1 = 0;
  int &occ = rt == 8 ? occ8 : occ1;
  const size_t smem = f32_chain_smem(rt);
  if (!occ) {
    cudaError_t e1, e2;
    if (rt == 8) {
      e1 = cudaFuncSetAttribute(gru_chain_f32_kernel<8>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      e2 = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, gru_chain_f32_kernel<8>, CH_THREADS, smem);
    } else {
      e1 = cudaFuncSetAttribute(gru_chain_f32_kernel<1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      e2 = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, gru_chain_f32_kernel<1>, CH_THREADS, smem);
    }
    if (e1 != cudaSuccess || e2 != cudaSuccess || occ < 1) { occ = 0; return false; }
  }
  // the dependency waits need every block of the grid resident: never more blocks than fit at once
  int grid = occ * sm_count;
  if (grid > a.order.units()) grid = a.order.units();
  if (rt == 8) gru_chain_f32_kernel<8><<<grid, CH_THREADS, smem, st>>>(a);
  else gru_chain_f32_kernel<1><<<grid, CH_THREADS, smem, st>>>(a);
  return true;
}

}  // namespace pnb

// ------------------------------------------------------------------------------------------ host state
using namespace pnb;

struct pnb_f32_state {
  // weights in the reference's layout (SURVEY.md App. B); fc is the engine's, the tensor path reads it too
  struct { float *W = nullptr, *b = nullptr; } conv1, conv2, fc_gb, fc_rb;
  struct { float *W = nullptr, *U = nullptr, *b = nullptr; } gru[5];  // gru1..3, gru_gb, gru_rb
  // Hop-slot buffers of one chunk of at most chunk_hops(e) hops.  Slots 0.. of the fc / conv1 buffers hold the conv
  // histories (oldest first), slot 0 of every GRU state buffer e->h[l] ([chunk+1][S][H]) the state before the chunk's
  // first hop; the chunk's carry moves the last slots back there, so between calls the state lives at the front.
  float *ring_fc = nullptr;  // [chunk+4][S][128] fc outputs: slots 0..3 the last four hops (oldest first), 4.. the chunk's
  float *ring_c1 = nullptr;  // [chunk+2][S][512] conv1 outputs, likewise
  float *c2_all = nullptr;   // [chunk][S][512] conv2 outputs of the chunk
  unsigned *cnt = nullptr;   // [5][rb] dependency counters of the persistent GRU chain
  int rt = 8, rb = 0;        // rows per thread of the chain kernel (8: 128-stream blocks, 1: 16-stream blocks); stream blocks
};

// hops per chunk of the network
static int chunk_hops(const pnb_engine *e) { return e->Fmax < kF32ChainMaxHops ? e->Fmax : kF32ChainMaxHops; }

#define FCK(call)                                                                                                   \
  do {                                                                                                              \
    cudaError_t _e = (call);                                                                                        \
    if (_e != cudaSuccess)                                                                                          \
      return engine_fail(_e == cudaErrorMemoryAllocation ? PNB_ERR_ALLOC : PNB_ERR_CUDA,                            \
                         (std::string(#call) + " failed: " + cudaGetErrorString(_e)).c_str());                      \
  } while (0)

int f32_prepare(pnb_engine *e, const pnb_model *model) {
  e->f32 = std::make_shared<pnb_f32_state>();
  pnb_f32_state &f = *e->f32;
  FCK(engine_upload(e, &f.conv1.W, model->conv1->input_weights, 5 * 128 * 512));
  FCK(engine_upload(e, &f.conv1.b, model->conv1->bias, 512));
  FCK(engine_upload(e, &f.conv2.W, model->conv2->input_weights, 3 * 512 * 512));
  FCK(engine_upload(e, &f.conv2.b, model->conv2->bias, 512));
  const pnb_gru_layer *g5[5] = {model->gru1, model->gru2, model->gru3, model->gru_gb, model->gru_rb};
  for (int i = 0; i < 5; i++) {
    const size_t M = g5[i]->nb_inputs, H = kGruH[i];
    FCK(engine_upload(e, &f.gru[i].W, g5[i]->input_weights, M * 3 * H));
    FCK(engine_upload(e, &f.gru[i].U, g5[i]->recurrent_weights, H * 3 * H));
    FCK(engine_upload(e, &f.gru[i].b, g5[i]->bias, 6 * H));
  }
  FCK(engine_upload(e, &f.fc_gb.W, model->fc_gb->input_weights, 2560 * 34));
  FCK(engine_upload(e, &f.fc_gb.b, model->fc_gb->bias, 34));
  FCK(engine_upload(e, &f.fc_rb.W, model->fc_rb->input_weights, 128 * 34));
  FCK(engine_upload(e, &f.fc_rb.b, model->fc_rb->bias, 34));
  const size_t S = e->S, C = chunk_hops(e);
  f.rt = S <= 64 ? 1 : 8;
  f.rb = (int)((S + 16 * f.rt - 1) / (16 * f.rt));
  FCK(engine_alloc(e, &f.ring_fc, (C + 4) * S * 128, kStreamState));
  FCK(engine_alloc(e, &f.ring_c1, (C + 2) * S * 512, kStreamState));
  FCK(engine_alloc(e, &f.c2_all, C * S * 512, kScratch));
  for (int i = 0; i < 5; i++) FCK(engine_alloc(e, &e->h[i], (C + 1) * S * kGruH[i], kStreamState));
  FCK(engine_alloc(e, &f.cnt, (size_t)5 * f.rb, kStreamState));
  return PNB_OK;
}

static GemmSeg seg(const float *A, int lda, const float *B, int ldb, int K) {
  GemmSeg s;
  s.A = A; s.lda = lda; s.B = B; s.ldb = ldb; s.K = K;
  return s;
}

// The network of hops [h0, h0 + n) of a call (n <= chunk_hops(e)) in fp32 FMA (rnn.cpp:42-81): the non-recurrent layers
// once over the active rows of all n hop slots, the five GRUs of all n hops in one persistent launch, the output layers
// over the same rows, and the carry that moves the conv histories and the states back to the front of their slot buffers.
// hops: the per-slot hops of a ragged call (device), or null.
static int run_chunk(pnb_engine *e, int h0, int n, const int *hops, cudaStream_t st) {
  const pnb_f32_state &f = *e->f32;
  const int S = e->S, na = e->n_active;
  // all streams active: the rows of the n slots are one flat range; otherwise the first na rows of each slot
  const int rows = na == S ? n * S : na, slots = na == S ? 1 : n;
  const float *tbl = e->tansig();
  // fc -> slots 4.. (slots 0..3 hold the last four hops' outputs)
  { LaunchScope m(e, PNB_K_FC, st); launch_fc_f32(e->d_feat + (size_t)h0 * S * kFeat, e->fc.W, e->fc.b, f.ring_fc + (size_t)4 * S * 128, rows, 70, 128, slots, S, st); }
  GemmArgs g;
  memset(&g, 0, sizeof g);
  g.M = rows; g.n_slots = slots; g.slot_stride = S; g.tansig = tbl;
  // conv1: tap q of hop t reads fc slot t + q (oldest first, nnet.cpp:182-200; weights [tap][c][n]) -> c1 slots 2..
  for (int q = 0; q < 5; q++) g.seg[q] = seg(f.ring_fc + (size_t)q * S * 128, 128, f.conv1.W + (size_t)q * 128 * 512, 512, 128);
  g.n_seg = 5; g.N = 512; g.C = f.ring_c1 + (size_t)2 * S * 512; g.ldc = 512; g.bias = f.conv1.b; g.act = PNB_ACT_RELU;
  { LaunchScope m(e, PNB_K_GEMM_F32, st); launch_gemm_f32(g, st); }
  for (int q = 0; q < 3; q++) g.seg[q] = seg(f.ring_c1 + (size_t)q * S * 512, 512, f.conv2.W + (size_t)q * 512 * 512, 512, 512);
  g.n_seg = 3; g.N = 512; g.C = f.c2_all; g.ldc = 512; g.bias = f.conv2.b; g.act = PNB_ACT_TANH;
  { LaunchScope m(e, PNB_K_GEMM_F32, st); launch_gemm_f32(g, st); }

  // stacked GRUs: each consumes the freshly updated state of the one below (SURVEY.md App. C.10)
  F32ChainArgs a;
  memset(&a, 0, sizeof a);
  const int n_rb = (int)(((size_t)na + 16 * f.rt - 1) / (16 * f.rt));  // stream blocks of the active streams
  a.order = chain_order(n, n_rb, CH_HT, 1);
  a.S = S; a.n = na; a.cnt = f.cnt; a.tansig = tbl;
  for (int li = 0; li < 5; li++) {
    F32ChainLayer &L = a.L[li];
    const int H = kGruH[li];
    L.H = H; L.W = f.gru[li].W; L.U = f.gru[li].U; L.bias = f.gru[li].b; L.ldw = 3 * H; L.h = e->h[li];
    L.dep = chain_dep(li);
    if (li == 0) {          // gru1 <- conv2 out
      L.n_x = 1; L.x[0] = f.c2_all; L.x_ld[0] = 512; L.x_K[0] = 512; L.x_slot1[0] = 0; L.x_slot_stride[0] = (size_t)S * 512;
    } else if (li < 4) {    // gru2 <- gru1, gru3 <- gru2, gru_gb <- gru3
      L.n_x = 1; L.x[0] = e->h[li - 1]; L.x_ld[0] = 512; L.x_K[0] = 512; L.x_slot1[0] = 1; L.x_slot_stride[0] = (size_t)S * 512;
    } else {                // gru_rb <- [gru3 state, conv2 out] (rnn.cpp:69-71)
      L.n_x = 2;
      L.x[0] = e->h[2]; L.x_ld[0] = 512; L.x_K[0] = 512; L.x_slot1[0] = 1; L.x_slot_stride[0] = (size_t)S * 512; L.w_row0[0] = 0;
      L.x[1] = f.c2_all;  L.x_ld[1] = 512; L.x_K[1] = 512; L.x_slot1[1] = 0; L.x_slot_stride[1] = (size_t)S * 512; L.w_row0[1] = 512;
    }
  }
  {
    LaunchScope m(e, PNB_K_GEMM_F32, st);
    if (!launch_gru_chain_f32(a, f.rt, e->sm_count, st)) return engine_fail(PNB_ERR_CUDA, "cannot configure the fp32 GRU chain kernel");
  }
  // fc_gb on [conv2, gru1, gru2, gru3, gru_gb] (rnn.cpp:73-78), fc_rb on gru_rb (rnn.cpp:80); state after hop t = slot t+1
  float *gr = e->d_gr + (size_t)h0 * S * 68;
  g.seg[0] = seg(f.c2_all, 512, f.fc_gb.W, 34, 512);
  for (int q = 1; q < 5; q++) g.seg[q] = seg(e->h[q - 1] + (size_t)S * 512, 512, f.fc_gb.W + (size_t)q * 512 * 34, 34, 512);
  g.n_seg = 5; g.N = 34; g.C = gr; g.ldc = 68; g.bias = f.fc_gb.b; g.act = PNB_ACT_SIGMOID;
  { LaunchScope m(e, PNB_K_GEMM_F32, st); launch_gemm_f32(g, st); }
  g.seg[0] = seg(e->h[4] + (size_t)S * 128, 128, f.fc_rb.W, 34, 128);
  g.n_seg = 1; g.N = 34; g.C = gr + 34; g.ldc = 68; g.bias = f.fc_rb.b; g.act = PNB_ACT_SIGMOID;
  { LaunchScope m(e, PNB_K_GEMM_F32, st); launch_gemm_f32(g, st); }
  // carry: the last 4 fc / 2 conv1 slots and the last state slot move to the front, conv2's output of the last hop is
  // kept for the tap.  In a ragged call a row that stopped inside the chunk takes its own last hop's slots, one that
  // stopped in an earlier chunk keeps its front slots
  SlotCarry c;
  memset(&c, 0, sizeof c);
  c.hops = hops; c.h0 = h0; c.n = n; c.cnt = f.cnt; c.n_cnt = 5 * f.rb;
  add_carry_seg(c, f.ring_fc, f.ring_fc, 128 * 4, na, S, 4, n);
  add_carry_seg(c, f.ring_c1, f.ring_c1, 512 * 4, na, S, 2, n);
  for (int li = 0; li < 5; li++) add_carry_seg(c, e->h[li], e->h[li], kGruH[li] * 4, na, S, 1, n);
  add_carry_seg(c, e->c2, f.c2_all, 512 * 4, na, S, 1, n - 1);
  { LaunchScope m(e, PNB_K_F32_CARRY, st); launch_slot_carry(c, e->sm_count, st); }
  return PNB_OK;
}

// The network of a call of F hops: chunks of up to chunk_hops(e) hops, in order.
int f32_network(pnb_engine *e, int F, const int *hops, cudaStream_t st) {
  const int C = chunk_hops(e);
  for (int h0 = 0; h0 < F; h0 += C)
    if (int rc = run_chunk(e, h0, F - h0 < C ? F - h0 : C, hops, st)) return rc;
  return PNB_OK;
}

int f32_network_launches(const pnb_engine *e, int F) {
  const int C = chunk_hops(e);
  return 7 * ((F + C - 1) / C);  // per chunk: fc, conv1, conv2, GRU chain, fc_gb, fc_rb, carry
}

// The fp32 path's part of a stream's state: the conv histories at slots 0..3 / 0..1 of the hop-slot buffers (where
// run_chunk's carry leaves them); the blob's bf16 term planes, which only tensor engines fill, are written as zeros.
int f32_state_segs(const pnb_engine *e, StateSeg *seg, int ns) {
  const pnb_f32_state &f = *e->f32;
  const size_t S = e->S;
  for (int k = 0; k < 4; k++)
    add_words(seg, ns, kSegCopy, f.ring_fc + (size_t)k * S * 128, 128 * 4, offsetof(StreamState, fc_hist) + (size_t)k * 128 * 4, 128);
  for (int k = 0; k < 2; k++)
    add_words(seg, ns, kSegCopy, f.ring_c1 + (size_t)k * S * 512, 512 * 4, offsetof(StreamState, c1_hist) + (size_t)k * 512 * 4, 512);
  add_words(seg, ns, kSegBlobZero, nullptr, 0, offsetof(StreamState, fc_terms), (sizeof(StreamState) - offsetof(StreamState, fc_terms)) / 4);
  return ns;
}

// The path's weights as the PNBW blob orders them (RNNModel layer order; per layer weights, recurrent weights, bias):
// the 25 device arrays and their float counts.  A PNB_TRAIN_NETWORK engine trains these in place.
int f32_params(const pnb_engine *e, float **p, size_t *count) {
  const pnb_f32_state &f = *e->f32;
  int k = 0;
  auto put = [&](float *a, size_t n) { p[k] = a; count[k] = n; k++; };
  put(e->fc.W, 70 * 128); put(e->fc.b, 128);
  put(f.conv1.W, 5 * 128 * 512); put(f.conv1.b, 512);
  put(f.conv2.W, 3 * 512 * 512); put(f.conv2.b, 512);
  for (int i = 0; i < 5; i++) {
    const size_t H = kGruH[i], M = i == 4 ? 1024 : 512;
    put(f.gru[i].W, M * 3 * H); put(f.gru[i].U, H * 3 * H); put(f.gru[i].b, 6 * H);
  }
  put(f.fc_gb.W, 2560 * 34); put(f.fc_gb.b, 34);
  put(f.fc_rb.W, 128 * 34); put(f.fc_rb.b, 34);
  return PNB_OK;
}
