// pnb_nn_tc.cu -- the gain network on Hopper tensor cores (wgmma + TMA + mbarrier), batched over streams.
//
// Replaces the reference's 35 scalar GEMVs per hop (src/nnet.cpp:59-200, src/rnn.cpp:42-81 of the reference)
// for the layers that carry 99.9 % of the MACs: conv1, conv2, the five GRUs and the two output layers.  The rows
// of every contraction are the concurrent streams (M = S), so the operation is genuinely dense.
//
// Precision.  The parity bar (1e-4 relative on g/r, +-1 LSB on PCM) rules out plain 16-bit operands.
// Every fp32 operand is therefore split into two 16-bit terms whose sum reproduces it to ~2^-22, and the three
// significant products are issued as separate tensor-core MMAs into the same fp32 register accumulator:
//   x w ~= xh wh + xh wl + xl wh
//   GRUs / output layers (inputs bounded by tanh): fp16 terms, both sides pre-scaled by powers of two
//   conv1 / conv2 (ReLU inputs, unbounded):        bf16 terms
//
// Three kernels, all persistent and warp-specialised, one CTA of three warpgroups per SM:
//   conv_pair_kernel conv1 or conv2 over all F hops of a call.  A tile is two neighbouring hops of 128 streams:
//                    each weight stage feeds both hops, each input hop slot feeds tap j of the first hop and tap
//                    j - 1 of the second.
//   tc_gemm_kernel   one 34-wide output layer over all rows (fc_gb, fc_rb run once per call over F*S rows)
//   gru_chain_kernel the five GRUs of all F hops of a call in ONE launch.  A tile (hop, layer, 128 streams,
//                    64 hidden units) depends only on tiles of the same 128 streams (layer below at this hop,
//                    own layer at the previous hop), so the recurrence is a per-(layer, row tile) counter that
//                    the consumer warps bump (release) and the TMA producer polls (acquire) -- no grid barrier,
//                    no launch boundary between layers or hops.
// Warpgroup roles per CTA: warpgroup 0 = TMA producer (one thread: cp.async.bulk.tensor into a ring of stages guarded
// by full / empty mbarriers; output layers SWIZZLE_128B boxes of 64 k, the conv layers and the chain SWIZZLE_64B
// boxes of 32 k),
// warpgroups 1 and 2 = consumers: each issues wgmma for 64 of the tile's 128 rows (m64nNk16, fp32 accumulators in
// registers; the conv and output layers take both operands from shared memory, the chain loads its activation operand into
// registers with ldmatrix once per stage) and runs the epilogue of its rows.  The producer streams the next tile's
// operands while the consumers finish the current one.
//
// The GRU tile holds, for 64 hidden units, three accumulators per unit: z and r summed over [x ; h], and the
// candidate's W_n x and U_n h apart (nnet.cpp:136-173 needs the last two apart) -- 256 accumulator columns in three
// register blocks nx (64), zr (128), nh (64).  Weight rows are packed [z|r|n] per tile in both parts, so one TMA box
// brings a tile's rows; per product the input part issues N = 128 into zr and N = 64 into nx, the recurrent part
// N = 128 into zr and N = 64 into nh.  The six MMAs of a 16-wide k-step read only two 64 x 16 activation blocks (the
// hi and lo terms), so those are loaded from shared memory into registers once (wgmma's A-from-registers form)
// instead of being read again by every MMA.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <math.h>
#include <stdio.h>
#include <string.h>

#include <string>
#include <vector>

#include "../../include/percepnet_b200.h"
#include "pnb_chain.cuh"
#include "pnb_engine.h"

using namespace pnb;

namespace {

constexpr int TM = 128;   // streams per CTA tile: two consumer warpgroups of 64 rows
constexpr int BK = 64;    // k per pipeline stage of the output layers: 128-byte rows, SWIZZLE_128B
constexpr int CBK = 32;   // k per pipeline stage of the conv layers and the GRU chain: 64-byte rows, SWIZZLE_64B
constexpr int HT = 64;    // hidden units per GRU tile
constexpr int GRU_BN = 3 * HT;  // weight rows per GRU tile (z|r|n)
constexpr int kConsumerWGs = 2;
constexpr int kTcThreads = 128 * (1 + kConsumerWGs);
constexpr int kPubWarps = 4 * kConsumerWGs;  // warps that bump a GRU tile's completion counter
constexpr int DENSE_BN = 128;   // output columns per conv tile
// Registers per thread after the producer warpgroup hands its surplus to the consumers (setmaxnreg, in the conv
// layers and the GRU chain): the launch gives 168 to each of the 384 threads; 128 x (168 - 40) = 256 x (232 - 168).
constexpr int kProducerRegs = 40, kConsumerRegs = 232;
constexpr float kActScale = 1024.f;  // fp16 activations are stored x 2^10 (keeps the low term normal)
// |pre-activation| from which the reference's tansig_approx (vec.h:63) overflows its float->int conversion
constexpr float kTanhDomain = 8.5e7f;

// ------------------------------------------------------------------------------------------ PTX
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_LOOP:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra WAIT_DONE;\n\t"
      "bra WAIT_LOOP;\n\t"
      "WAIT_DONE:\n\t}" ::"r"(bar), "r"(parity)
      : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap *map, uint32_t bar, int x, int y) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint"
      " [%0], [%1, {%3, %4}], [%2], %5;" ::"r"(dst),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(x), "r"(y),
      "l"(0x1000000000000000ull)  // EVICT_NORMAL
      : "memory");
}
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async;" ::: "memory"); }

// Shared-memory matrix descriptor (wgmma), K-major operand, SWIZZLE_128B: rows of 128 bytes, 8-row groups 1024 bytes
// apart: start>>4 [0,14), LBO [16,30) (unused for swizzled K-major, 1), SBO>>4 [32,46) = 64, layout [62,64) = 1 (SW128).
// The high word is a constant; the low word is (address >> 4) | LBO and advances by plain addition, 32 bytes per
// 16-wide k-step inside the 128-byte row and 1024 bytes per 8 rows (the shared window is < 256 KB, so the 14-bit
// field never carries).  Tiles are 1024-byte aligned (the swizzle is a function of the address bits).
// SWIZZLE_64B (the GRU chain): rows of 64 bytes, 8-row groups 512 bytes apart, SBO>>4 = 32, layout = 2; the k-step
// advance is the same 32 bytes.
constexpr uint32_t kDescHi = (uint32_t)(1024 >> 4) | (1u << 30);
constexpr uint32_t kDescHi64 = (uint32_t)(512 >> 4) | (2u << 30);
__device__ __forceinline__ uint32_t desc_lo(uint32_t saddr) { return ((saddr >> 4) & 0x3FFF) | (1u << 16); }
__device__ __forceinline__ uint64_t desc64(uint32_t lo, uint32_t hi = kDescHi) { return ((uint64_t)hi << 32) | lo; }

__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// Keeps the compiler from moving accesses of accumulator registers across a wgmma fence / wait.
template <int R>
__device__ __forceinline__ void acc_fence(float *d) {
#pragma unroll
  for (int i = 0; i < R; i++) asm volatile("" : "+f"(d[i])::"memory");
}

// D[64 x N] = (acc ? D : 0) + A[64 x 16] B[N x 16]^T, fp32 accumulators in registers (m64nNk16 fragment: register
// 4j + q holds row 16 warp + lane/4 + 8 (q/2), column 8j + 2 (lane%4) + q%2).  acc = 0 starts a sum without a
// zero fill of the registers: a fill that the compiler places while earlier MMAs are in flight serialises them.
template <int N, bool BF16>
__device__ __forceinline__ void wgmma(float *d, uint64_t da, uint64_t db, uint32_t acc = 1);
#define PNB_WGMMA_PRED(ACC) "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %" #ACC ", 0;\n\t"
template <>
__device__ __forceinline__ void wgmma<128, true>(float *d, uint64_t da, uint64_t db, uint32_t acc) {
  asm volatile(PNB_WGMMA_PRED(66)
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, "
      "%15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, "
      "%39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, "
      "%63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
        "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),
        "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),
        "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]),
        "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]),
        "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]),
        "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(acc));
}
template <>
__device__ __forceinline__ void wgmma<48, false>(float *d, uint64_t da, uint64_t db, uint32_t acc) {
  asm volatile(PNB_WGMMA_PRED(26)
      "wgmma.mma_async.sync.aligned.m64n48k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, "
      "%15, %16, %17, %18, %19, %20, %21, %22, %23}, %24, %25, p, 1, 1, 0, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
        "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),
        "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
      : "l"(da), "l"(db), "r"(acc));
}
// The same MMA with A from registers (the GRU chain): a[0..3] is this thread's share of the 64 x 16 A block -- rows
// 16 warp + lane/4 (+8 in a[1], a[3]), k 2 (lane%4) (+8 in a[2], a[3]), two fp16 per register, as ldmatrix.x4
// leaves it.  The registers are read asynchronously: they must not be rewritten before the MMA has completed.
template <int N>
__device__ __forceinline__ void wgmma_rs(float *d, const uint32_t *a, uint64_t db, uint32_t acc = 1);
template <>
__device__ __forceinline__ void wgmma_rs<128>(float *d, const uint32_t *a, uint64_t db, uint32_t acc) {
  asm volatile(PNB_WGMMA_PRED(69)
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, "
      "%15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, "
      "%39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, "
      "%63}, {%64, %65, %66, %67}, %68, p, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
        "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),
        "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),
        "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]),
        "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]),
        "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]),
        "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(acc));
}
template <>
__device__ __forceinline__ void wgmma_rs<64>(float *d, const uint32_t *a, uint64_t db, uint32_t acc) {
  asm volatile(PNB_WGMMA_PRED(37)
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, "
      "%15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1, 0;\n\t}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
        "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),
        "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),
        "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(db), "r"(acc));
}
#undef PNB_WGMMA_PRED
__device__ __forceinline__ void ldsm_x4(uint32_t *r, uint32_t addr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr)
               : "memory");
}
template <int R>
__device__ __forceinline__ void reg_fence(uint32_t *r) {  // acc_fence for the A fragments
#pragma unroll
  for (int i = 0; i < R; i++) asm volatile("" : "+r"(r[i])::"memory");
}

// ------------------------------------------------------------------------------------------ activations
// tansig_approx of vec.h:53-71 on the FMA/ALU pipes only.  The reference forms the table index with
// floor(.5f + 25 x) -> (int); here t + 2^23 rounded toward -inf leaves floor(t) in the low mantissa bits (exact for
// 0 <= t < 2^23), which replaces FRND + F2I + I2F (quarter-rate conversion pipe) by one FADD.RM and one FADD.
// |x| is clamped at 8: from there on the reference returns exactly +-1 (index clamped at 200, where dy = 0).
// NaN propagates (min.NaN); beyond |x| = 8.6e7 the reference's conversion overflows (undefined behaviour, x86
// returns its argument) -- callers whose pre-activations can get there raise the engine's domain flag instead.
__device__ __forceinline__ float tansig_s(float x, const float *tbl) {
  float ax;
  asm("min.NaN.f32 %0, %1, %2;" : "=f"(ax) : "f"(fabsf(x)), "f"(8.0f));
  const float t = fmaf(25.f, ax, .5f);
  const float r = __fadd_rd(t, 8388608.f);
  const int idx = __float_as_int(r) & 0xFF;           // floor(t) <= 200 (255 at most for a NaN payload; table has 256 slots)
  const float fi = r - 8388608.f;
  const float xr = fmaf(-.04f, fi, ax);
  const float y = tbl[idx];
  const float dy = fmaf(-y, y, 1.f);
  const float u = fmaf(-y, xr, 1.f);
  const float v = fmaf(xr * dy, u, y);
  return __int_as_float(__float_as_int(v) | (__float_as_int(x) & 0x80000000));
}
__device__ __forceinline__ float sigmoid_s(float x, const float *tbl) { return fmaf(.5f, tansig_s(.5f * x, tbl), .5f); }

// fp16 two-term split of two neighbouring values (x 2^10)
__device__ __forceinline__ void store_split_h2(float v0, float v1, __half *hi_p, __half *lo_p) {
  const float s0 = v0 * kActScale, s1 = v1 * kActScale;
  const __half2 h = __floats2half2_rn(s0, s1);
  const float2 hf = __half22float2(h);
  *reinterpret_cast<__half2 *>(hi_p) = h;
  *reinterpret_cast<__half2 *>(lo_p) = __floats2half2_rn(s0 - hf.x, s1 - hf.y);
}
// The conv layers' splits of four neighbouring values, one 8-byte store per term: fp16 two-term split (x 2^10), the
// roundings of store_split_h2, and bf16 three-term split into planes `plane` elements apart
__device__ __forceinline__ uint32_t h2_bits(__half2 h) { return *reinterpret_cast<uint32_t *>(&h); }
__device__ __forceinline__ uint32_t b2_bits(__nv_bfloat162 h) { return *reinterpret_cast<uint32_t *>(&h); }
__device__ __forceinline__ void store_split_h4(const float *v, __half *hi_p, __half *lo_p) {
  uint32_t hi[2], lo[2];
#pragma unroll
  for (int i = 0; i < 2; i++) {
    const float s0 = v[2 * i] * kActScale, s1 = v[2 * i + 1] * kActScale;
    const __half2 h = __floats2half2_rn(s0, s1);
    const float2 hf = __half22float2(h);
    hi[i] = h2_bits(h);
    lo[i] = h2_bits(__floats2half2_rn(s0 - hf.x, s1 - hf.y));
  }
  *reinterpret_cast<uint2 *>(hi_p) = make_uint2(hi[0], hi[1]);
  *reinterpret_cast<uint2 *>(lo_p) = make_uint2(lo[0], lo[1]);
}
__device__ __forceinline__ void store_split_b4(const float *v, __nv_bfloat16 *t0_p, size_t plane) {
  uint32_t t[3][2];
#pragma unroll
  for (int i = 0; i < 2; i++) {
    const float v0 = v[2 * i], v1 = v[2 * i + 1];
    const __nv_bfloat162 h = __floats2bfloat162_rn(v0, v1);
    const float2 hf = __bfloat1622float2(h);
    const float r0 = v0 - hf.x, r1 = v1 - hf.y;
    const __nv_bfloat162 l = __floats2bfloat162_rn(r0, r1);
    const float2 lf = __bfloat1622float2(l);
    t[0][i] = b2_bits(h);
    t[1][i] = b2_bits(l);
    t[2][i] = b2_bits(__floats2bfloat162_rn(r0 - lf.x, r1 - lf.y));
  }
#pragma unroll
  for (int k = 0; k < 3; k++) *reinterpret_cast<uint2 *>(t0_p + k * plane) = make_uint2(t[k][0], t[k][1]);
}

// ------------------------------------------------------------------------------------------ shared kernel pieces
template <int BN, int NT = 2, int KB = BK>
struct StageLayout {  // NT terms of A (the tile's 128 rows), then NT terms of the BN rows of B, KB k each
  static constexpr int kABytes = TM * KB * 2;
  static constexpr int kBBytes = BN * KB * 2;
  static constexpr int kBytes = NT * (kABytes + kBBytes);
};

struct Pipe {  // position in an mbarrier ring
  uint32_t st = 0, ph = 0;
  __device__ __forceinline__ void advance(uint32_t stages) {
    if (++st == stages) { st = 0; ph ^= 1; }
  }
};

struct SmemCarve {
  uint8_t *stages;
  uint32_t full, empty;  // shared-window addresses of the barrier arrays
  float *tbl;
};
template <int STAGES, int REGION_BYTES>  // REGION_BYTES: the stage ring (the barriers sit behind it)
__device__ __forceinline__ SmemCarve carve(uint8_t *smem_raw) {
  // the swizzled tiles need 1024-byte (SW128) alignment; align the carve-up by hand
  uint8_t *smem = smem_raw + ((1024u - (smem_u32(smem_raw) & 1023u)) & 1023u);
  SmemCarve c;
  c.stages = smem;
  uint64_t *bars = reinterpret_cast<uint64_t *>(smem + REGION_BYTES);
  c.full = smem_u32(bars);
  c.empty = c.full + 8 * STAGES;
  c.tbl = reinterpret_cast<float *>(bars + 2 * STAGES);
  return c;
}
template <int STAGES, int REGION_BYTES>
constexpr size_t tc_smem_bytes() {
  return (size_t)REGION_BYTES + 2 * STAGES * 8 + 256 * 4 + 1024;
}
// common prologue: barriers and the activation table
template <int STAGES>
__device__ __forceinline__ void tc_prologue(const SmemCarve &c, const float *tansig) {
  if (threadIdx.x == 0) {
    for (int i = 0; i < STAGES; i++) {
      mbar_init(c.full + 8 * i, 1);
      mbar_init(c.empty + 8 * i, kConsumerWGs);  // one arrival per consumer warpgroup
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  for (int i = threadIdx.x; i < 256; i += blockDim.x) c.tbl[i] = i < 201 ? tansig[i] : 1.f;
  __syncthreads();
}

// The products of one pass over K, as (A term, B term) pairs in issue order.  Two terms per operand: hi hi, hi lo,
// lo hi.  Three terms (t0 t1 t2, each 8 bits below the previous): the six products of total order <= 2.
// The conv layers' ReLU inputs are unbounded, so the K loop runs once per product order, smallest products first
// (three terms: PASS 0 order 2, PASS 1 order 1, PASS 2 t0 t0; two terms: PASS 1, PASS 2).  The tensor core adds
// into the fp32 accumulator with truncation at the accumulator's magnitude, so correction products added to an already
// large sum lose exactly the bits they were meant to supply; summed among themselves first, they do not.  The output
// layers use the same two passes.  (The GRU chain, whose operands are bounded by 1, issues all products of a k-block
// at once: gru_mma_kblock.)
template <int PASS, typename F>
__device__ __forceinline__ void pass_products(F &&mma) {
  if (PASS == 0) { mma(1, 1); mma(0, 2); mma(2, 0); }
  else if (PASS == 1) { mma(0, 1); mma(1, 0); }
  else mma(0, 0);
}

// Consumer side of one stage: wait for the operands, issue the k-block's MMAs, and free the stage the PREVIOUS k-block
// read once its MMAs have completed (one k-block of MMAs stays in flight).  `prev_empty` is 0 before a tile's first
// k-block.  ACC_REGS: the accumulator registers the MMAs write (fenced around the asynchronous updates).
template <int ACC_REGS>
struct Consumer {
  uint32_t prev_empty = 0;
  __device__ __forceinline__ void begin(float *acc, uint32_t full_bar, uint32_t parity) {
    mbar_wait(full_bar, parity);
    fence(acc);
  }
  // orders the MMAs after every register write before them (accumulators, A fragments loaded after the barrier wait)
  __device__ __forceinline__ void fence(float *acc) {
    acc_fence<ACC_REGS>(acc);
    wgmma_fence();
  }
  __device__ __forceinline__ void end(float *acc, uint32_t empty_bar) {
    wgmma_commit();
    wgmma_wait<1>();
    acc_fence<ACC_REGS>(acc);
    if (prev_empty && threadIdx.x % 128 == 0) mbar_arrive(prev_empty);
    prev_empty = empty_bar;
  }
  __device__ __forceinline__ void drain(float *acc) {  // end of a tile: every MMA has completed
    wgmma_wait<0>();
    acc_fence<ACC_REGS>(acc);
    if (prev_empty && threadIdx.x % 128 == 0) mbar_arrive(prev_empty);
    prev_empty = 0;
  }
};

// ------------------------------------------------------------------------------------------ output layers
struct TcSeg {
  int a_map, b_map;  // indices into TcArgs::maps
  int k_blocks;      // K / BK
  int a_k0, b_k0;    // starting k (elements) in the A / B matrices
  int a_row0;        // row of the A matrix that holds tile row 0 (hop offset inside a multi-hop buffer)
  int a_term_rows;   // row distance between the split terms inside this A buffer
};

struct TcArgs {
  CUtensorMap maps[8];
  TcSeg seg[5];
  int n_seg;
  int M;                // rows per hop slot: rows [k slot_stride, k slot_stride + M) of slot k (one slot: a flat range)
  int slot_stride;      // row distance between hop slots (unused with one slot)
  int tiles_slot;       // row tiles per hop slot: tiles never straddle two slots
  int tiles_m, tiles_n; // tile grid (tiles_m = slots x tiles_slot); a CTA walks tiles blockIdx.x, blockIdx.x + gridDim.x, ...
  int b_term_rows;      // row distance between the split terms inside a packed weight matrix
  float out_scale;      // 2^-(activation scale + weight scale)
  const float *tansig;  // 201-entry table (global)
  const float *bias;    // padded to a multiple of 16 entries
  int *status;          // engine status word: bit 0 = an activation left the reference's defined domain
  int N;                // valid output columns
  int ldc;              // row stride of out_f32
  float *out_f32;       // sigmoid outputs [rows][ldc]
};

// First row of row tile mt, the end of its hop slot's rows in *lim
__device__ __forceinline__ int dense_tile_row0(const TcArgs &args, int mt, int *lim) {
  const int slot = mt / args.tiles_slot;
  *lim = slot * args.slot_stride + args.M;
  return slot * args.slot_stride + (mt - slot * args.tiles_slot) * TM;
}

// ===== TMA producer (one thread): the tile's A rows and B rows, one pass over K per product order =====
template <int BN, int STAGES>
__device__ __forceinline__ void dense_producer(const TcArgs &args, const SmemCarve &c, uint32_t stage0, int total_tiles) {
  using SL = StageLayout<BN>;
  Pipe p;
  for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    int lim;
    const int n_tile = tile % args.tiles_n, m0 = dense_tile_row0(args, tile / args.tiles_n, &lim);
    // pass 1 (hi lo, lo hi) needs both terms of either operand, pass 2 (hi hi) the first
    for (int nt = 2; nt > 0; nt--) {
      for (int s = 0; s < args.n_seg; s++) {
        const TcSeg &sg = args.seg[s];
        const CUtensorMap *ma = &args.maps[sg.a_map], *mb = &args.maps[sg.b_map];
        const int arow = sg.a_row0 + m0, brow = n_tile * BN;
        for (int kb = 0; kb < sg.k_blocks; kb++) {
          mbar_wait(c.empty + 8 * p.st, p.ph ^ 1);  // fresh barrier: passes immediately
          const uint32_t fb = c.full + 8 * p.st;
          mbar_expect_tx(fb, nt * (SL::kABytes + SL::kBBytes));
          const uint32_t sp = stage0 + p.st * SL::kBytes;
          for (int tm = 0; tm < nt; tm++) {
            tma_load_2d(sp + tm * SL::kABytes, ma, fb, sg.a_k0 + kb * BK, tm * sg.a_term_rows + arow);
            tma_load_2d(sp + 2 * SL::kABytes + tm * SL::kBBytes, mb, fb, sg.b_k0 + kb * BK, tm * args.b_term_rows + brow);
          }
          p.advance(STAGES);
        }
      }
    }
  }
}

// One k-block of a tile on the MMA side (one consumer warpgroup, its 64 rows): the pass's products of the four 16-wide
// k-steps.  `a_lo` is the descriptor low word of this warpgroup's rows in the stage's first A term, `b_lo` that of the
// stage's first B term.
template <int BN, int PASS>
__device__ __forceinline__ void mma_kblock(float *acc, uint32_t a_lo, uint32_t b_lo) {
  using SL = StageLayout<BN>;
  constexpr uint32_t A = SL::kABytes >> 4, B = SL::kBBytes >> 4;
#pragma unroll
  for (int ks = 0; ks < BK / 16; ks++) {
    const uint32_t a = a_lo + ks * 2, b = b_lo + ks * 2;
    pass_products<PASS>([&](int ta, int tb) { wgmma<BN, false>(acc, desc64(a + ta * A), desc64(b + tb * B)); });
  }
}

// ===== consumer warpgroup: MMAs of its 64 rows, then the epilogue (bias, sigmoid, fp32 stores) =====
template <int BN, int STAGES>
__device__ __forceinline__ void dense_consumer(const TcArgs &args, const SmemCarve &c, uint32_t stage0, int total_tiles, int wg) {
  using SL = StageLayout<BN>;
  constexpr int R = BN / 2;  // accumulator registers per thread
  const uint32_t a_lo0 = desc_lo(stage0) + (uint32_t)(wg * 64 * 128 >> 4);
  const uint32_t b_lo0 = desc_lo(stage0) + (uint32_t)(2 * SL::kABytes >> 4);
  const int warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
  const float sc = args.out_scale;
  const float *tbl = c.tbl;
  const int N = args.N;
  Pipe p;
  Consumer<R> cons;
  for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    int lim;  // rows from lim on (padding up to the tile's end) are computed but neither stored nor checked
    const int n_tile = tile % args.tiles_n, m0 = dense_tile_row0(args, tile / args.tiles_n, &lim);
    float acc[R];
#pragma unroll
    for (int i = 0; i < R; i++) acc[i] = 0.f;
    int nkb = 0;
    for (int s = 0; s < args.n_seg; s++) nkb += args.seg[s].k_blocks;
#pragma unroll
    for (int pass = 1; pass < 3; pass++) {
      for (int kb = 0; kb < nkb; kb++) {
        cons.begin(acc, c.full + 8 * p.st, p.ph);
        const uint32_t so = p.st * (SL::kBytes >> 4);
        if (pass == 1) mma_kblock<BN, 1>(acc, a_lo0 + so, b_lo0 + so);
        else mma_kblock<BN, 2>(acc, a_lo0 + so, b_lo0 + so);
        cons.end(acc, c.empty + 8 * p.st);
        p.advance(STAGES);
      }
    }
    cons.drain(acc);
    bool bad = false;
#pragma unroll
    for (int h = 0; h < 2; h++) {  // the thread's two rows of the fragment
      const int row = m0 + wg * 64 + warp * 16 + (lane >> 2) + 8 * h;
      if (row >= lim) continue;
#pragma unroll
      for (int j = 0; j < BN / 8; j++) {
        const int col = n_tile * BN + 8 * j + 2 * (lane & 3);
        if (col >= N) continue;  // N is even: a pair is entirely in or out
        const float2 bb = __ldg(reinterpret_cast<const float2 *>(args.bias + col));
        float *op = args.out_f32 + (size_t)row * args.ldc + col;
#pragma unroll
        for (int q = 0; q < 2; q++) {
          const float x = fmaf(acc[4 * j + 2 * h + q], sc, q ? bb.y : bb.x);
          op[q] = sigmoid_s(x, tbl);
          bad |= fabsf(x) >= 2.f * kTanhDomain;
        }
      }
    }
    if (bad) atomicOr(args.status, 1);
  }
}

// fc_gb / fc_rb: fp16 two-term operands, STAGES stages
template <int BN, int STAGES>
__global__ void __launch_bounds__(kTcThreads, 1) tc_gemm_kernel(const __grid_constant__ TcArgs args) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const SmemCarve c = carve<STAGES, STAGES * StageLayout<BN>::kBytes>(smem_raw);
  const int wg = threadIdx.x >> 7;
  const int total_tiles = args.tiles_m * args.tiles_n;
  tc_prologue<STAGES>(c, args.tansig);
  const uint32_t stage0 = smem_u32(c.stages);
  if (wg == 0) {
    if (threadIdx.x == 0) dense_producer<BN, STAGES>(args, c, stage0, total_tiles);
  } else {
    dense_consumer<BN, STAGES>(args, c, stage0, total_tiles, wg - 1);
  }
}

// ------------------------------------------------------------------------------------------ conv layers
// conv_pair_kernel<Q>: conv1 (Q = 5 taps over the fc outputs) or conv2 (Q = 3 taps over the conv1 outputs) for all F
// hops of a call, 512 outputs, bf16 terms.  Tap q of hop t reads input slot t + q, and every hop uses the same weight
// rows for tap q.  A tile is (hop pair t0 = 2p, t0 + 1; 128 streams; 128 output columns), with two accumulator sets:
// acc0 for hop t0, acc1 for hop t0 + 1.  Input slot t0 + j feeds tap j of hop t0 and tap j - 1 of hop t0 + 1, and
// weight tap q feeds both, so per pass and 32-k block the tile loads Q + 1 input slots and Q weight taps where two
// one-hop tiles loaded 2 Q of each.
// The ring carries, per pass and k-block, Q + 1 stages: stage j holds the pass's terms of input slot t0 + j and of
// weight tap j (stage Q: the input slot alone).  Unit j, on the stage j barrier, issues tap j - 1 of hop t0 + 1
// (acc1 += A_j W_{j-1}, weights of stage j - 1) and tap j of hop t0 (acc0 += A_j W_j).  Stage j - 1 is read for the
// last time by unit j and stage Q by unit Q, so stages are freed in ring order, and the consumers hold at most three
// at once (two for the units being issued, one for the unit in flight).
// A tile whose second hop is past the call's end (odd F) loads stages 0 .. Q - 1 only and issues acc0 alone.
// Tiles are walked column tile fastest, then hop pair, then row tile: the CTAs running at once read the input slots of
// one or two row tiles, which neighbouring pairs share, so they come from L2.  (With the row tile before the pair, the
// input slots of one pair over all rows -- 75 MB for conv1 at 16 384 streams -- overflow L2 and every pair reads its
// slots from HBM again.)
// Summation order, identical for every hop whichever accumulator or tile it is in: passes (pass_products), then 32-k
// blocks, then taps, then 16-wide k-steps.  A hop's bits depend on nothing but its own row.
struct ConvArgs {
  CUtensorMap a_map;    // input hop slots, [3 terms][slots x S][K]: boxes of 128 rows x 32 k, SWIZZLE_64B
  CUtensorMap w_map;    // packed weights, [3 terms][512][Q K]: the same boxes
  int k_blocks;         // K / CBK
  int a_term_rows;      // rows per term plane of the input
  int S;                // rows per hop slot
  int n;                // active streams: rows [0, n) of every slot
  int F;                // hops of the call
  int pairs;            // hop pairs, ceil(F / 2)
  int tiles;            // row tiles (ceil(n / 128)) x pairs x column tiles
  const float *tansig;
  const float *bias;
  int *status;          // engine status word: bit 0 = an activation left the reference's defined domain
  const int *wide;      // device word: non-zero = three operand terms (six products) instead of two
  const int *hops;      // ragged calls: [n] hops of each row, or null.  Hop t of row r with t >= hops[r] is computed
                        // but neither stored nor checked; out_f32 takes the row's hop hops[r] - 1 (else F - 1)
  int act;              // PNB_ACT_RELU (conv1) or PNB_ACT_TANH (conv2)
  __nv_bfloat16 *out_b; // conv1: three bf16 terms, hop t at row out_row0 + t S of planes out_plane_rows apart
  __half *out_h;        // conv2: fp16 two-term split (x 2^10), hop t at row out_row0 + t S
  float *out_f32;       // conv2: fp32 copy of each row's last hop, [n][512], or null
  int out_row0;
  int out_plane_rows;
};
constexpr int CONV_N = 512;
constexpr int CONV_TILES_N = CONV_N / DENSE_BN;
// 7 stages of 32 KB (two terms) or 4 of 48 KB (three terms): three held by the consumers, the rest in flight
constexpr int CONV_ST2 = 7, CONV_ST3 = 4;
constexpr int kConvRegion = CONV_ST2 * StageLayout<DENSE_BN, 2, CBK>::kBytes > CONV_ST3 * StageLayout<DENSE_BN, 3, CBK>::kBytes
                                ? CONV_ST2 * StageLayout<DENSE_BN, 2, CBK>::kBytes
                                : CONV_ST3 * StageLayout<DENSE_BN, 3, CBK>::kBytes;
constexpr int kConvStages = CONV_ST2 > CONV_ST3 ? CONV_ST2 : CONV_ST3;

struct ConvTile {
  int n_tile, m0, t0;
  bool pair;  // hop t0 + 1 is inside the call
  __device__ __forceinline__ ConvTile(const ConvArgs &a, int tile) {
    n_tile = tile % CONV_TILES_N;
    const int rp = tile / CONV_TILES_N;
    t0 = 2 * (rp % a.pairs);
    m0 = (rp / a.pairs) * TM;
    pair = t0 + 1 < a.F;
  }
};

// ===== TMA producer (one thread): per pass, k-block and unit j, input slot t0 + j and weight tap j =====
template <int Q, int NT, int STAGES>
__device__ __forceinline__ void conv_producer(const ConvArgs &args, const SmemCarve &c, uint32_t stage0) {
  using SL = StageLayout<DENSE_BN, NT, CBK>;
  const int K = args.k_blocks * CBK;
  Pipe p;
  for (int tile = blockIdx.x; tile < args.tiles; tile += gridDim.x) {
    const ConvTile tl(args, tile);
    const int units = tl.pair ? Q + 1 : Q;
    const int arow = tl.t0 * args.S + tl.m0, brow = tl.n_tile * DENSE_BN;
    // with q passes still to go after this one, the pass needs the first q + 1 terms of either operand
    for (int nt = NT; nt > 0; nt--) {
      for (int kb = 0; kb < args.k_blocks; kb++) {
        for (int j = 0; j < units; j++) {
          mbar_wait(c.empty + 8 * p.st, p.ph ^ 1);  // fresh barrier: passes immediately
          const uint32_t fb = c.full + 8 * p.st;
          mbar_expect_tx(fb, nt * (SL::kABytes + (j < Q ? SL::kBBytes : 0)));
          const uint32_t sp = stage0 + p.st * SL::kBytes;
          for (int tm = 0; tm < nt; tm++) {
            tma_load_2d(sp + tm * SL::kABytes, &args.a_map, fb, kb * CBK, tm * args.a_term_rows + j * args.S + arow);
            if (j < Q)
              tma_load_2d(sp + NT * SL::kABytes + tm * SL::kBBytes, &args.w_map, fb, j * K + kb * CBK, tm * CONV_N + brow);
          }
          p.advance(STAGES);
        }
      }
    }
  }
}

// The consumer's side of the conv ring: `full` is the next stage to wait for, `freed` the oldest stage not yet freed,
// `pending` the stages the unit in flight is the last reader of.
struct ConvRing {
  Pipe full, freed;
  int pending = 0;
  template <int STAGES>
  __device__ __forceinline__ void release(const SmemCarve &c) {
    for (; pending > 0; pending--) {
      if (threadIdx.x % 128 == 0) mbar_arrive(c.empty + 8 * freed.st);
      freed.advance(STAGES);
    }
  }
};

// One unit on one consumer warpgroup: wait for its stage, issue acc1 (if HOP1: A of this stage, weights of the
// stage before) and acc0 (if HOP0: A and weights of this stage) per k-step and product, alternating so that
// neighbouring MMAs do not wait on each other's accumulators, then free the stages the previous unit read last once
// its MMAs have completed (one unit stays in flight).  RETIRE: stages this unit is the last reader of.
template <int NT, int PASS, int STAGES, int R, bool HOP0, bool HOP1, int RETIRE>
__device__ __forceinline__ void conv_unit(float *acc, uint32_t a_lo0, uint32_t b_lo0, const SmemCarve &c, ConvRing &ring) {
  using SL = StageLayout<DENSE_BN, NT, CBK>;
  constexpr uint32_t A = SL::kABytes >> 4, B = SL::kBBytes >> 4, ST = SL::kBytes >> 4;
  const uint32_t st = ring.full.st;
  mbar_wait(c.full + 8 * st, ring.full.ph);
  acc_fence<R>(acc);
  wgmma_fence();
  const uint32_t so = st * ST, sp = (st ? st - 1 : STAGES - 1) * ST;
#pragma unroll
  for (int ks = 0; ks < CBK / 16; ks++) {
    const uint32_t a = a_lo0 + so + ks * 2, b = b_lo0 + so + ks * 2, bp = b_lo0 + sp + ks * 2;
    pass_products<PASS>([&](int ta, int tb) {
      if (HOP1) wgmma<DENSE_BN, true>(acc + 64, desc64(a + ta * A, kDescHi64), desc64(bp + tb * B, kDescHi64));
      if (HOP0) wgmma<DENSE_BN, true>(acc, desc64(a + ta * A, kDescHi64), desc64(b + tb * B, kDescHi64));
    });
  }
  wgmma_commit();
  wgmma_wait<1>();
  acc_fence<R>(acc);
  ring.release<STAGES>(c);
  ring.pending = RETIRE;
  ring.full.advance(STAGES);
}

// One pass over K of a tile: k-blocks, and per k-block the units in ring order
template <int Q, int NT, int PASS, int STAGES, bool PAIR>
__device__ __forceinline__ void conv_pass(float *acc, int k_blocks, uint32_t a_lo0, uint32_t b_lo0, const SmemCarve &c,
                                          ConvRing &ring) {
  constexpr int R = PAIR ? 128 : 64;
  for (int kb = 0; kb < k_blocks; kb++) {
    if (PAIR) {
      conv_unit<NT, PASS, STAGES, R, true, false, 0>(acc, a_lo0, b_lo0, c, ring);
#pragma unroll
      for (int j = 1; j < Q; j++) conv_unit<NT, PASS, STAGES, R, true, true, 1>(acc, a_lo0, b_lo0, c, ring);
      conv_unit<NT, PASS, STAGES, R, false, true, 2>(acc, a_lo0, b_lo0, c, ring);
    } else {
#pragma unroll
      for (int j = 0; j < Q; j++) conv_unit<NT, PASS, STAGES, R, true, false, 1>(acc, a_lo0, b_lo0, c, ring);
    }
  }
}
template <int Q, int NT, int STAGES, bool PAIR>
__device__ __forceinline__ void conv_tile_mmas(float *acc, int k_blocks, uint32_t a_lo0, uint32_t b_lo0, const SmemCarve &c,
                                               ConvRing &ring) {
  if (NT == 3) conv_pass<Q, NT, 0, STAGES, PAIR>(acc, k_blocks, a_lo0, b_lo0, c, ring);
  conv_pass<Q, NT, 1, STAGES, PAIR>(acc, k_blocks, a_lo0, b_lo0, c, ring);
  conv_pass<Q, NT, 2, STAGES, PAIR>(acc, k_blocks, a_lo0, b_lo0, c, ring);
  wgmma_wait<0>();
  acc_fence<PAIR ? 128 : 64>(acc);
  ring.release<STAGES>(c);
}

// Epilogue of hop t for this thread's two rows: bias, activation, stores.  Returns whether a pre-activation left the
// reference's tanh domain.  In the MMA fragment a lane holds two neighbouring columns of every 8-column group, so a
// warp's stores would cover half a 32-byte sector per row; the four lanes of a row (a quad) first exchange the
// activated values of column groups 2 jj and 2 jj + 1, after which lane q holds columns 16 jj + 4 q .. + 3 and the
// quad writes whole sectors.  Lanes of a quad share their row, so rows that store nothing still take part in the
// exchange.
__device__ __forceinline__ bool conv_epilogue(const ConvArgs &args, const float *acc, const ConvTile &tl, int t, int wg,
                                              const float *tbl) {
  const int warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31, q = lane & 3;
  const int src = (lane & ~3) | ((q & 1) << 1);  // the quad lane holding the first two of this lane's columns
  bool bad = false;
#pragma unroll
  for (int h = 0; h < 2; h++) {  // the thread's two rows of the fragment
    const int row = tl.m0 + wg * 64 + warp * 16 + (lane >> 2) + 8 * h;
    bool ok = row < args.n;  // padding rows of the last row tile are computed only
    bool last = t == args.F - 1;
    if (args.hops && ok) {   // a ragged call: the row's frozen hops are padding too
      const int hr = __ldg(args.hops + row);
      ok = t < hr;
      last = t == hr - 1;
    }
    const size_t orow = (size_t)args.out_row0 + (size_t)t * args.S + row;
#pragma unroll
    for (int jj = 0; jj < DENSE_BN / 16; jj++) {
      float v[2][2];  // columns 8 j + 2 q, + 1 of j = 2 jj, 2 jj + 1
#pragma unroll
      for (int g = 0; g < 2; g++) {
        const int j = 2 * jj + g;
        const float2 bb = __ldg(reinterpret_cast<const float2 *>(args.bias + tl.n_tile * DENSE_BN + 8 * j + 2 * q));
#pragma unroll
        for (int e = 0; e < 2; e++) {
          const float x = acc[4 * j + 2 * h + e] + (e ? bb.y : bb.x);
          if (args.act == PNB_ACT_TANH) { v[g][e] = tansig_s(x, tbl); bad |= ok && fabsf(x) >= kTanhDomain; }
          else v[g][e] = x < 0.f ? 0.f : x;
        }
      }
      float w[4];  // columns 16 jj + 4 q .. + 3
#pragma unroll
      for (int e = 0; e < 2; e++) {
        const float a0 = __shfl_sync(0xffffffffu, v[0][e], src), b0 = __shfl_sync(0xffffffffu, v[1][e], src);
        const float a1 = __shfl_sync(0xffffffffu, v[0][e], src + 1), b1 = __shfl_sync(0xffffffffu, v[1][e], src + 1);
        w[e] = q < 2 ? a0 : b0;
        w[2 + e] = q < 2 ? a1 : b1;
      }
      if (!ok) continue;
      const int col = tl.n_tile * DENSE_BN + 16 * jj + 4 * q;
      if (args.out_f32 && last) {
        float *op = args.out_f32 + (size_t)row * CONV_N + col;
#pragma unroll
        for (int e = 0; e < 4; e++) op[e] = w[e];
      }
      if (args.out_h)
        store_split_h4(w, args.out_h + orow * CONV_N + col, args.out_h + ((size_t)args.out_plane_rows + orow) * CONV_N + col);
      if (args.out_b) store_split_b4(w, args.out_b + orow * CONV_N + col, (size_t)args.out_plane_rows * CONV_N);
    }
  }
  return bad;
}

// ===== consumer warpgroup: MMAs of its 64 rows of both hops, then the epilogue of each hop =====
template <int Q, int NT, int STAGES>
__device__ __forceinline__ void conv_consumer(const ConvArgs &args, const SmemCarve &c, uint32_t stage0, int wg) {
  using SL = StageLayout<DENSE_BN, NT, CBK>;
  const uint32_t a_lo0 = desc_lo(stage0) + (uint32_t)(wg * 64 * CBK * 2 >> 4);
  const uint32_t b_lo0 = desc_lo(stage0) + (uint32_t)(NT * SL::kABytes >> 4);
  ConvRing ring;
  for (int tile = blockIdx.x; tile < args.tiles; tile += gridDim.x) {
    const ConvTile tl(args, tile);
    float acc[128];  // acc0 = acc[0, 64), acc1 = acc[64, 128)
#pragma unroll
    for (int i = 0; i < 128; i++) acc[i] = 0.f;
    if (tl.pair) conv_tile_mmas<Q, NT, STAGES, true>(acc, args.k_blocks, a_lo0, b_lo0, c, ring);
    else conv_tile_mmas<Q, NT, STAGES, false>(acc, args.k_blocks, a_lo0, b_lo0, c, ring);
    bool bad = conv_epilogue(args, acc, tl, tl.t0, wg, c.tbl);
    if (tl.pair) bad |= conv_epilogue(args, acc + 64, tl, tl.t0 + 1, wg, c.tbl);
    if (bad) atomicOr(args.status, 1);
  }
}

template <int Q>
__global__ void __launch_bounds__(kTcThreads, 1) conv_pair_kernel(const __grid_constant__ ConvArgs args) {
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const SmemCarve c = carve<kConvStages, kConvRegion>(smem_raw);
  const int wg = threadIdx.x >> 7;
  tc_prologue<kConvStages>(c, args.tansig);
  const uint32_t stage0 = smem_u32(c.stages);
  // the same word for every thread of the launch (written by an earlier launch): every role takes the same branch
  const bool wide = *args.wide != 0;
  if (wg == 0) {
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kProducerRegs));
    if (threadIdx.x != 0) return;
    if (wide) conv_producer<Q, 3, CONV_ST3>(args, c, stage0);
    else conv_producer<Q, 2, CONV_ST2>(args, c, stage0);
  } else {
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kConsumerRegs));
    if (wide) conv_consumer<Q, 3, CONV_ST3>(args, c, stage0, wg - 1);
    else conv_consumer<Q, 2, CONV_ST2>(args, c, stage0, wg - 1);
  }
}

// ------------------------------------------------------------------------------------------ the GRU chain
struct ChainLayer {
  int n_x;              // input segments (2 for gru_rb: [gru3 state, conv2 out])
  int x_map[2];         // A tensor maps of the input segments
  int x_kb[2];          // their k-blocks
  int x_bk0[2];         // starting k in the packed input weights
  int x_row1[2];        // 0: the segment is indexed by hop (conv2 out, slot t); 1: state slots (slot t+1 = after hop t)
  int x_term_rows[2];   // row distance between the two split terms in that buffer
  int h_map, w_map, u_map;
  int h_kb;             // H / CBK
  int H;
  int b_term_rows;      // rows of one term plane of the packed weights
  int dep;              // chain_dep of this layer
  float scale;          // 2^-(10 + weight scale)
  const float4 *bias4;  // per unit {b_z + b'_z, b_r + b'_r, b_n, b'_n}
  float *h32;           // fp32 state [S][H], updated in place
  __half *h_hl;         // fp16 terms [2][(Fmax+1) S][H]
  int h_term_rows;      // (Fmax+1) S
};
struct ChainArgs {
  CUtensorMap maps[16];  // 0: conv2 out, 1..5: state slots of the five GRUs, 6..10: input weights, 11..15: recurrent weights
  ChainLayer L[5];
  ChainOrder order;      // F hops of the row tiles of the active streams (128 streams each), 64-unit tiles
  int S;                 // rows per hop slot of the buffers
  int n;                 // active streams: rows [0, n) of every slot
  const int *hops;       // ragged calls: [n] hops of each row, or null.  Hop t of row r with t >= hops[r] is computed
                         // but stores nothing: the fp32 state keeps that of the row's last hop
  unsigned *cnt;         // [5][order.n_rb] consumer-warp completions, zero at launch
  const float *tansig;
};

// all consumer warps of every tile of (layer, row tile) have finished `hops` hops
__device__ __forceinline__ void wait_layer(const ChainArgs &a, int layer, int rb, int hops) {
  chain_wait(a.cnt + layer * a.order.n_rb + rb, (unsigned)hops * kPubWarps << a.order.tiles_log2[layer]);
}

constexpr int GRU_STAGES = 5;
using GruStage = StageLayout<GRU_BN, 2, CBK>;  // 2 x 8 KB of A + 2 x 12 KB of B = 40 KB

// A fragments of one k-block (CBK = two 16-wide k-steps, both terms of A) for one consumer warp: 16 registers,
// fa[8 term + 4 ks + i] (wgmma_rs layout).  `a_addr[ks]` is this lane's ldmatrix row address for k-step ks in the first A term of stage
// 0 (gru_a_addr); `so` the stage's byte offset.
constexpr int kFragRegs = 2 * (CBK / 16) * 4;
__device__ __forceinline__ void gru_load_a(uint32_t *fa, const uint32_t *a_addr, uint32_t so) {
#pragma unroll
  for (int t = 0; t < 2; t++)
#pragma unroll
    for (int ks = 0; ks < CBK / 16; ks++) ldsm_x4(fa + 8 * t + 4 * ks, a_addr[ks] + so + t * GruStage::kABytes);
}
// ldmatrix.x4 row addresses: lanes 8m .. 8m+7 address the rows of 8x8 matrix m = (rows +8 (m&1), k +8 (m>>1)) of the
// warp's 16 rows, which puts the fragment in the order wgmma_rs reads it.  The TMA box wrote the 64-byte rows with
// SWIZZLE_64B: the 16-byte chunk index XOR address bits 7-8, i.e. XOR (row / 2) % 4 (the stage is 1024-byte aligned).
__device__ __forceinline__ void gru_a_addr(uint32_t *a_addr, uint32_t stage0, int cw, int warp, int lane) {
  const int row = cw * 64 + warp * 16 + (lane & 7) + 8 * ((lane >> 3) & 1);
#pragma unroll
  for (int ks = 0; ks < CBK / 16; ks++) {
    const int chunk = 2 * ks + (lane >> 4);
    a_addr[ks] = stage0 + row * (CBK * 2) + ((chunk ^ ((row >> 1) & 3)) << 4);
  }
}

// One k-block of a GRU tile on one consumer warpgroup: per k-step the three products hi hi, hi lo, lo hi of weight
// rows [z|r] (N = 128) into `zr` and of rows [n] (N = 64) into `n`, the two register blocks alternating so that
// consecutive MMAs do not wait on each other's accumulators.  A (the activations) comes from the fragments `fa`
// (gru_load_a), B from the stage.  zr_acc / n_acc = 0: the k-block starts the block's sum (its first MMA overwrites
// the registers).
__device__ __forceinline__ void gru_mma_kblock(float *zr, float *n, const uint32_t *fa, uint32_t b_lo, uint32_t zr_acc, uint32_t n_acc) {
  constexpr uint32_t B = GruStage::kBBytes >> 4;
  constexpr uint32_t BN = (2 * HT * CBK * 2) >> 4;  // the n rows follow the 2 HT rows of [z|r]
#pragma unroll
  for (int ks = 0; ks < CBK / 16; ks++) {
    const uint32_t *hi = fa + 4 * ks, *lo = fa + 8 + 4 * ks;
    const uint32_t b = b_lo + ks * 2;
    wgmma_rs<128>(zr, hi, desc64(b, kDescHi64), ks ? 1u : zr_acc);
    wgmma_rs<64>(n, hi, desc64(b + BN, kDescHi64), ks ? 1u : n_acc);
    wgmma_rs<128>(zr, hi, desc64(b + B, kDescHi64));
    wgmma_rs<64>(n, hi, desc64(b + B + BN, kDescHi64));
    wgmma_rs<128>(zr, lo, desc64(b, kDescHi64));
    wgmma_rs<64>(n, lo, desc64(b + BN, kDescHi64));
  }
}

// Consumer side of one k-block of a GRU unit: wait for the stage, load its A fragments into `fa`, issue the MMAs into
// `zr` and `n` (the nx or nh block of `acc`), free the previous stage.  One k-block stays in flight and reads its
// fragments asynchronously, so consecutive k-blocks use different `fa`: gru_chain_kernel alternates two, k-blocks
// in pairs.  Every part of a unit has an even number of k-blocks (inputs are 512 wide, H a multiple of HT).
constexpr int kChainAccRegs = 4 * HT / 2;  // nx (64 columns), zr (128), nh (64)
constexpr int NX = 0, ZR = HT / 2, NH = 3 * HT / 2;
static_assert(512 % (2 * CBK) == 0 && HT % (2 * CBK) == 0, "the chain's k-blocks are consumed in pairs");
__device__ __forceinline__ void gru_consume_kblock(float *acc, float *n, uint32_t *fa, uint32_t zr_acc, uint32_t n_acc,
                                                   const uint32_t *a_addr, uint32_t b_lo0, const SmemCarve &c, Pipe &p,
                                                   Consumer<kChainAccRegs> &cons) {
  mbar_wait(c.full + 8 * p.st, p.ph);
  const uint32_t so = p.st * GruStage::kBytes;
  gru_load_a(fa, a_addr, so);
  reg_fence<kFragRegs>(fa);
  cons.fence(acc);
  gru_mma_kblock(acc + ZR, n, fa, b_lo0 + (so >> 4), zr_acc, n_acc);
  cons.end(acc, c.empty + 8 * p.st);
  p.advance(GRU_STAGES);
}

__global__ void __launch_bounds__(kTcThreads, 1) gru_chain_kernel(const __grid_constant__ ChainArgs args) {
  using SL = GruStage;
  constexpr int STAGES = GRU_STAGES;
  // accumulator registers per thread, three blocks: nx = W_n x (64 columns), zr = [z | r] over [x ; h] (128 columns),
  // nh = U_n h (64 columns).  The blocks never overlap partially: wgmma into partly overlapping register ranges
  // would serialise the MMA pipeline.
  constexpr int R = kChainAccRegs;
  extern __shared__ __align__(1024) uint8_t smem_raw[];
  const SmemCarve c = carve<STAGES, STAGES * SL::kBytes>(smem_raw);
  const int wg = threadIdx.x >> 7;
  const int total_units = args.order.units();
  const int S = args.S;
  tc_prologue<STAGES>(c, args.tansig);
  const uint32_t stage0 = smem_u32(c.stages);

  if (wg == 0) {
    // ===== TMA producer: waits for the rows it is about to read, then streams the tile's operands =====
    asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(kProducerRegs));
    if (threadIdx.x != 0) return;
    Pipe p;
    for (int u = blockIdx.x; u < total_units; u += gridDim.x) {
      const ChainUnit un = chain_decode(args.order, u);
      const ChainLayer &L = args.L[un.l];
      if (L.dep >= 0) wait_layer(args, L.dep, un.rb, un.t + 1);  // input: layer below, this hop
      if (un.t > 0) wait_layer(args, un.l, un.rb, un.t);        // own state after the previous hop
      fence_proxy_async();  // the rows were written with st.global by other SMs; TMA reads them through the async proxy
      const int m0 = un.rb * TM;
      const int brow = un.tile * GRU_BN;
      for (int s = 0; s <= L.n_x; s++) {
        const bool rec = s == L.n_x;
        const CUtensorMap *ma = &args.maps[rec ? L.h_map : L.x_map[s]], *mb = &args.maps[rec ? L.u_map : L.w_map];
        const int nkb = rec ? L.h_kb : L.x_kb[s];
        const int arow = (rec ? un.t : un.t + L.x_row1[s]) * S + m0;
        const int aterm = rec ? L.h_term_rows : L.x_term_rows[s];
        const int bk0 = rec ? 0 : L.x_bk0[s];
        for (int kb = 0; kb < nkb; kb++) {
          mbar_wait(c.empty + 8 * p.st, p.ph ^ 1);
          const uint32_t fb = c.full + 8 * p.st;
          mbar_expect_tx(fb, SL::kBytes);
          const uint32_t sp = stage0 + p.st * SL::kBytes;
          tma_load_2d(sp, ma, fb, kb * CBK, arow);
          tma_load_2d(sp + SL::kABytes, ma, fb, kb * CBK, aterm + arow);
          tma_load_2d(sp + 2 * SL::kABytes, mb, fb, bk0 + kb * CBK, brow);
          tma_load_2d(sp + 2 * SL::kABytes + SL::kBBytes, mb, fb, bk0 + kb * CBK, L.b_term_rows + brow);
          p.advance(STAGES);
        }
      }
    }
  } else {
    // ===== consumer warpgroup: MMAs of its 64 streams, then the gate math of nnet.cpp:136-178 (reset_after) =====
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(kConsumerRegs));
    const int cw = wg - 1, warp = (threadIdx.x >> 5) & 3, lane = threadIdx.x & 31;
    const uint32_t b_lo0 = desc_lo(stage0) + (uint32_t)(2 * SL::kABytes >> 4);
    uint32_t a_addr[CBK / 16];
    gru_a_addr(a_addr, stage0, cw, warp, lane);
    const float *tbl = c.tbl;
    Pipe p;
    Consumer<R> cons;
    for (int u = blockIdx.x; u < total_units; u += gridDim.x) {
      const ChainUnit un = chain_decode(args.order, u);
      const ChainLayer &L = args.L[un.l];
      const int H = L.H;
      float acc[R];  // no zero fill: the first k-block of either part starts its blocks' sums
      uint32_t fa0[kFragRegs], fa1[kFragRegs];  // A fragments of the even / odd k-blocks
      // input part: [z|r] rows into zr, n rows into nx; recurrent part: [z|r] rows into zr, n rows into nh
      int nkb = 0;
      for (int s = 0; s < L.n_x; s++) nkb += L.x_kb[s];
      for (int kb = 0; kb < nkb; kb += 2) {
        gru_consume_kblock(acc, acc + NX, fa0, kb != 0, kb != 0, a_addr, b_lo0, c, p, cons);
        gru_consume_kblock(acc, acc + NX, fa1, 1u, 1u, a_addr, b_lo0, c, p, cons);
      }
      for (int kb = 0; kb < L.h_kb; kb += 2) {
        gru_consume_kblock(acc, acc + NH, fa0, 1u, kb != 0, a_addr, b_lo0, c, p, cons);
        gru_consume_kblock(acc, acc + NH, fa1, 1u, 1u, a_addr, b_lo0, c, p, cons);
      }
      cons.drain(acc);
      // the previous hop's state of these rows is complete (other SMs wrote it): acquire before reading it.  The fp32
      // state is updated in place: this thread alone reads and writes these (row, unit) pairs at this hop, and whoever
      // touches them at the next hop waits for this unit's counter bump first.
      if (un.t > 0) {
        if (lane == 0) wait_layer(args, un.l, un.rb, un.t);
        __syncwarp();
      }
      const float sc = L.scale;
#pragma unroll
      for (int h = 0; h < 2; h++) {  // the thread's two rows of the fragment
        const int row = un.rb * TM + cw * 64 + warp * 16 + (lane >> 2) + 8 * h;
        if (row >= args.n || (args.hops && un.t >= __ldg(args.hops + row))) continue;
        float *h32 = L.h32 + (size_t)row * H;
        __half *ph = L.h_hl + ((size_t)(un.t + 1) * S + row) * H;
#pragma unroll
        for (int j = 0; j < HT / 8; j++) {
          const int unit = un.tile * HT + 8 * j + 2 * (lane & 3);
          const float2 ho = __ldcg(reinterpret_cast<const float2 *>(h32 + unit));
          float hn[2];
#pragma unroll
          for (int q = 0; q < 2; q++) {
            const int i = 4 * j + 2 * h + q;  // fragment register of this (row, unit) inside a 64-column group
            const float4 bb = __ldg(L.bias4 + unit + q);
            const float z = sigmoid_s(fmaf(acc[ZR + i], sc, bb.x), tbl);
            const float r = sigmoid_s(fmaf(acc[ZR + HT / 2 + i], sc, bb.y), tbl);
            const float tmp = fmaf(acc[NH + i], sc, bb.w);
            float cnd = fmaf(tmp, r, bb.z);
            cnd = fmaf(acc[NX + i], sc, cnd);
            const float n = tansig_s(cnd, tbl);
            hn[q] = fmaf(z, (q ? ho.y : ho.x) - n, n);  // z h + (1 - z) n
          }
          *reinterpret_cast<float2 *>(h32 + unit) = make_float2(hn[0], hn[1]);
          store_split_h2(hn[0], hn[1], ph + unit, ph + (size_t)L.h_term_rows * H + unit);
        }
      }
      // publish: every store of this warp for this tile is ordered before the counter bump
      __syncwarp();
      if (lane == 0) {
        __threadfence();
        red_release_gpu_add(args.cnt + un.l * args.order.n_rb + un.rb, 1u);
      }
    }
  }
}

constexpr int SMALL_BN = 48, SMALL_STAGES = 5;
// conv layers: fc / conv1 outputs and the conv weights are stored as THREE bf16 terms.  The launches use the first
// two (three products, corrections summed before the main product) unless the engine's `wide` word is set
// (PNB_CONV_WIDE at pnb_create: all three terms, six products).  The mode is the same for every row of every call,
// so a stream's result never depends on what its neighbours in the batch carry.
constexpr int kConvTerms = 3;
constexpr size_t kConvSmem = tc_smem_bytes<kConvStages, kConvRegion>();
constexpr size_t kSmallSmem = tc_smem_bytes<SMALL_STAGES, SMALL_STAGES * StageLayout<SMALL_BN>::kBytes>();
static_assert(kConvSmem <= 227 * 1024, "the conv ring fits a Hopper block's shared memory");

// fc 70 -> 128 relu in fp32 FMA (0.1 % of the MACs; K = 70 is no tensor-core shape), emitting the three bf16
// terms conv1 consumes.  One block per 16 rows, one thread per output: the 16 feature rows sit in shared memory and are
// read four k at a time (one broadcast 128-bit load per row and four FMAs), the weight column comes through L1.
// Every output is bias + sum over ascending k, one fmaf per term, like the fp32 path's fc kernel.  grid.y walks hop slots
// of M rows each, slot_stride rows apart (one slot: M is all rows of the call's hops).
constexpr int FC_ROWS = 16;
__global__ void __launch_bounds__(128) fc_split_kernel(const float *__restrict__ feat, const float *__restrict__ W,
                                                       const float *__restrict__ bias, __nv_bfloat16 *__restrict__ out,
                                                       int M, size_t plane_rows, size_t slot_stride) {
  __shared__ __align__(16) float f[FC_ROWS][72];
  const int r0 = blockIdx.x * FC_ROWS;
  feat += blockIdx.y * slot_stride * 70;  // hop slot blockIdx.y: M rows of it
  out += blockIdx.y * slot_stride * 128;
  for (int i = threadIdx.x; i < FC_ROWS * 72; i += blockDim.x) {
    const int rr = i / 72, kk = i - rr * 72;
    f[rr][kk] = (kk < 70 && r0 + rr < M) ? feat[(size_t)(r0 + rr) * 70 + kk] : 0.f;
  }
  __syncthreads();
  const int n = threadIdx.x;
  float a[FC_ROWS];
  const float b0 = bias[n];
#pragma unroll
  for (int rr = 0; rr < FC_ROWS; rr++) a[rr] = b0;
#pragma unroll 1
  for (int k = 0; k < 68; k += 4) {
    const float w0 = __ldg(W + (size_t)k * 128 + n), w1 = __ldg(W + (size_t)(k + 1) * 128 + n);
    const float w2 = __ldg(W + (size_t)(k + 2) * 128 + n), w3 = __ldg(W + (size_t)(k + 3) * 128 + n);
#pragma unroll
    for (int rr = 0; rr < FC_ROWS; rr++) {
      const float4 fv = *reinterpret_cast<const float4 *>(&f[rr][k]);
      a[rr] = fmaf(w0, fv.x, a[rr]);
      a[rr] = fmaf(w1, fv.y, a[rr]);
      a[rr] = fmaf(w2, fv.z, a[rr]);
      a[rr] = fmaf(w3, fv.w, a[rr]);
    }
  }
  {
    const float w0 = __ldg(W + (size_t)68 * 128 + n), w1 = __ldg(W + (size_t)69 * 128 + n);
#pragma unroll
    for (int rr = 0; rr < FC_ROWS; rr++) {
      a[rr] = fmaf(w0, f[rr][68], a[rr]);
      a[rr] = fmaf(w1, f[rr][69], a[rr]);
    }
  }
  const size_t plane = plane_rows * 128;
#pragma unroll
  for (int rr = 0; rr < FC_ROWS; rr++) {
    if (r0 + rr >= M) break;
    float v = a[rr] < 0.f ? 0.f : a[rr];
    __nv_bfloat16 t0 = __float2bfloat16_rn(v);
    float r = v - __bfloat162float(t0);
    __nv_bfloat16 t1 = __float2bfloat16_rn(r);
    __nv_bfloat16 t2 = __float2bfloat16_rn(r - __bfloat162float(t1));
    size_t o = (size_t)(r0 + rr) * 128 + n;
    out[o] = t0; out[plane + o] = t1; out[2 * plane + o] = t2;
  }
}

}  // namespace

// ------------------------------------------------------------------------------------------ host state
struct pnb_tc_state {
  // split activations
  // Multi-hop buffers: rows are (hop slot, stream).  The conv layers carry no recurrence, so they run once per
  // call over all F hops (M = F S rows); a tap is the same buffer read `tap` slots later.  Slots 0..3 (0..1) hold
  // the last hops of the previous call.
  __nv_bfloat16 *fc_all = nullptr;   // [3][(Fmax+4) S][128]  fc outputs, bf16 terms
  __nv_bfloat16 *c1_all = nullptr;   // [3][(Fmax+2) S][512]  conv1 outputs
  __half *c2_h = nullptr;            // [2][Fmax S][512]      conv2 outputs, fp16 terms
  __half *h_all[5] = {};             // [2][(Fmax+1) S][H]    GRU states as fp16 terms, slot t+1 = after hop t,
                                     //                       slot 0 = carried from the previous call
  // packed weights
  __nv_bfloat16 *w_conv1 = nullptr, *w_conv2 = nullptr;  // [3][512][K]
  __half *w_gru[5] = {}, *u_gru[5] = {};                 // [2][tiles*192][K]
  float scale_gru[5] = {};                               // 2^-(10 + e)
  float4 *bias4[5] = {};                                 // per unit {b_z + b'_z, b_r + b'_r, b_n, b'_n}
  __half *w_gb = nullptr, *w_rb = nullptr;               // [2][48][2560], [2][48][128] (34 rows used)
  float scale_gb = 0.f, scale_rb = 0.f;
  float *bias_pad = nullptr;                             // conv1 [512] | conv2 [512] | fc_gb [48] | fc_rb [48]
  unsigned *cnt = nullptr;                               // chain dependency counters [5][tiles_mp]
  int *wide = nullptr;                                   // see kConvTerms
  int tiles_mp = 0;
  // tensor maps
  CUtensorMap m_c2, m_h[5], m_wgb, m_wrb;                  // output layers: 64-k boxes, SW128
  CUtensorMap m_fc_all, m_c1_all, m_wconv1, m_wconv2;     // conv layers: 32-k boxes, SW64
  CUtensorMap m_c2_ch, m_h_ch[5], m_w[5], m_u[5];         // GRU chain: 32-k boxes, SW64
};

typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn g_encode = nullptr;
static std::string g_tc_err;

// boxes of box_k x box_rows; the output layers read 64 k (SWIZZLE_128B), the conv layers and the GRU chain 32 k
// (SWIZZLE_64B)
static int make_map(CUtensorMap *m, const void *base, bool bf16, uint64_t rows, uint64_t cols, uint32_t box_rows,
                    uint32_t box_k = BK, CUtensorMapSwizzle swizzle = CU_TENSOR_MAP_SWIZZLE_128B) {
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {cols * 2};
  cuuint32_t box[2] = {box_k, box_rows};
  cuuint32_t estr[2] = {1, 1};
  CUresult r = g_encode(m, bf16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2,
                        const_cast<void *>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                        swizzle, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return r == CUDA_SUCCESS ? 0 : (int)r;
}

static float pow2_scale_for(const float *a, size_t na, const float *b, size_t nb, int *e_out) {
  float mx = 0.f;
  for (size_t i = 0; i < na; i++) mx = fmaxf(mx, fabsf(a[i]));
  for (size_t i = 0; i < nb; i++) mx = fmaxf(mx, fabsf(b[i]));
  int e = 0;
  if (mx > 0.f && isfinite(mx)) {
    int ex;
    frexpf(mx, &ex);  // mx = f * 2^ex, f in [0.5, 1)
    e = 14 - ex;      // mx * 2^e in [2^13, 2^14)
  }
  *e_out = e;
  return ldexpf(1.f, e);
}

#define TCK(call)                                                                          \
  do {                                                                                     \
    cudaError_t _e = (call);                                                               \
    if (_e != cudaSuccess) {                                                               \
      g_tc_err = std::string(#call) + ": " + cudaGetErrorString(_e);                       \
      return engine_fail(PNB_ERR_CUDA, g_tc_err.c_str());                                      \
    }                                                                                      \
  } while (0)

// GRU weights: reference layout W[j*3H + g*H + i] -> K-major rows ordered [tile][gate z, r, n][HT units], scaled,
// split into two fp16 terms.  Input and recurrent weights alike: the first 2 HT rows of a tile are the N = 128 MMA
// onto the zr accumulators, the last HT rows the N = 64 MMA onto nx (input) or nh (recurrent).
static void pack_gru(const float *W, int K, int H, float scale, std::vector<__half> &out) {
  const int tiles = H / HT, rows = tiles * GRU_BN;
  out.assign((size_t)2 * rows * K, __float2half(0.f));
  for (int tl = 0; tl < tiles; tl++)
    for (int g = 0; g < 3; g++)
      for (int ii = 0; ii < HT; ii++) {
        const int row = tl * GRU_BN + g * HT + ii, i = tl * HT + ii;
        for (int j = 0; j < K; j++) {
          float w = W[(size_t)j * 3 * H + g * H + i] * scale;
          __half hi = __float2half_rn(w);
          __half lo = __float2half_rn(w - __half2float(hi));
          out[(size_t)row * K + j] = hi;
          out[((size_t)rows + row) * K + j] = lo;
        }
      }
}
// dense/conv weights: W[k*N + n] -> [n][k], three bf16 terms
static void pack_dense_b3(const float *W, int K, int N, std::vector<__nv_bfloat16> &out) {
  out.assign((size_t)3 * N * K, __float2bfloat16(0.f));
  for (int n = 0; n < N; n++)
    for (int k = 0; k < K; k++) {
      float w = W[(size_t)k * N + n];
      __nv_bfloat16 t0 = __float2bfloat16_rn(w);
      float r = w - __bfloat162float(t0);
      __nv_bfloat16 t1 = __float2bfloat16_rn(r);
      out[(size_t)n * K + k] = t0;
      out[((size_t)N + n) * K + k] = t1;
      out[((size_t)2 * N + n) * K + k] = __float2bfloat16_rn(r - __bfloat162float(t1));
    }
}

// 34-wide output layers: W[k*34 + n] -> [48 rows (34 used)][K], scaled, two fp16 terms
static void pack_small_h2(const float *W, int K, int N, float scale, std::vector<__half> &out) {
  out.assign((size_t)2 * SMALL_BN * K, __float2half(0.f));
  for (int n = 0; n < N; n++)
    for (int k = 0; k < K; k++) {
      float w = W[(size_t)k * N + n] * scale;
      __half hi = __float2half_rn(w);
      out[(size_t)n * K + k] = hi;
      out[((size_t)SMALL_BN + n) * K + k] = __float2half_rn(w - __half2float(hi));
    }
}

// Largest |pre-activation| a layer can form from inputs bounded by 1 (tanh outputs / GRU states): the row sums of
// |W| (+ |U|) plus |b|.  The tensor path is validated inside the reference's defined domain only (tansig_approx
// overflows its float->int conversion from 8.6e7 on, vec.h:63); weights that could leave it are refused up front.
static double max_preact(const float *W, int K, int N, int ld, const float *U, int KU, const float *b0, const float *b1) {
  std::vector<double> acc(N, 0.0);
  for (int k = 0; k < K; k++)
    for (int n = 0; n < N; n++) acc[n] += fabs((double)W[(size_t)k * ld + n]);
  if (U)
    for (int k = 0; k < KU; k++)
      for (int n = 0; n < N; n++) acc[n] += fabs((double)U[(size_t)k * ld + n]);
  double mx = 0.0;
  for (int n = 0; n < N; n++) {
    double v = acc[n] + (b0 ? fabs((double)b0[n]) : 0.0) + (b1 ? fabs((double)b1[n]) : 0.0);
    if (!(v <= mx)) mx = v;  // NaN-propagating max
  }
  return mx;
}

int tc_prepare(pnb_engine *e, const pnb_model *model) {
  if (!g_encode) {
    void *fn = nullptr;
    cudaDriverEntryPointQueryResult qr;
    cudaError_t r = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qr);
    if (r != cudaSuccess || !fn) return engine_fail(PNB_ERR_CUDA, "cuTensorMapEncodeTiled is not available from the driver");
    g_encode = (EncodeTiledFn)fn;
  }
  const pnb_gru_layer *g5[5] = {model->gru1, model->gru2, model->gru3, model->gru_gb, model->gru_rb};
  {  // inputs of the GRUs and output layers are bounded by 1 inside the reference's domain: bound their pre-activations
    double mx = 0.0;
    for (int i = 0; i < 5; i++) {
      const int K = g5[i]->nb_inputs, H = g5[i]->nb_neurons;
      for (int g = 0; g < 3; g++) {
        double v = max_preact(g5[i]->input_weights + g * H, K, H, 3 * H, g5[i]->recurrent_weights + g * H, H,
                              g5[i]->bias + g * H, g5[i]->bias + (3 + g) * H);
        if (!(v <= mx)) mx = v;
      }
    }
    double v = max_preact(model->fc_gb->input_weights, 2560, 34, 34, nullptr, 0, model->fc_gb->bias, nullptr);
    if (!(v <= mx)) mx = v;
    v = max_preact(model->fc_rb->input_weights, 128, 34, 34, nullptr, 0, model->fc_rb->bias, nullptr);
    if (!(v <= mx)) mx = v;
    if (!(mx < kTanhDomain))
      return engine_fail(PNB_ERR_ARG, "PNB_NN_TENSOR: a GRU / output layer can form pre-activations >= 8.5e7 (or NaN), outside the "
                                  "domain of the reference's tansig_approx; use PNB_NN_FP32 for this model");
  }
  e->tc = std::make_shared<pnb_tc_state>();
  pnb_tc_state *t = e->tc.get();
  const size_t S = e->S;
  const size_t Fm = e->Fmax;
  for (int i = 0; i < 5; i++) TCK(engine_alloc(e, &e->h[i], S * kGruH[i], kStreamState));
  TCK(engine_alloc(e, &t->fc_all, kConvTerms * (Fm + 4) * S * 128, kStreamState));
  TCK(engine_alloc(e, &t->c1_all, kConvTerms * (Fm + 2) * S * 512, kStreamState));
  {
    int w = (e->flags & PNB_CONV_WIDE) ? 1 : 0;
    if (const char *ct = getenv("PNB_CONV_TERMS")) w = atoi(ct) == 3 ? 1 : atoi(ct) == 2 ? 0 : w;  // experiments
    TCK(engine_upload(e, &t->wide, &w, 1));
  }
  TCK(engine_alloc(e, &t->c2_h, 2 * Fm * S * 512, kStreamState));
  for (int i = 0; i < 5; i++) TCK(engine_alloc(e, &t->h_all[i], 2 * (Fm + 1) * S * kGruH[i], kStreamState));
  t->tiles_mp = (int)((S + TM - 1) / TM);
  TCK(engine_alloc(e, &t->cnt, (size_t)5 * t->tiles_mp, kStreamState));
  {
    std::vector<__nv_bfloat16> p;
    pack_dense_b3(model->conv1->input_weights, 640, 512, p);
    TCK(engine_upload(e, &t->w_conv1, p.data(), p.size()));
    pack_dense_b3(model->conv2->input_weights, 1536, 512, p);
    TCK(engine_upload(e, &t->w_conv2, p.data(), p.size()));
  }
  for (int i = 0; i < 5; i++) {
    const int K = g5[i]->nb_inputs, H = g5[i]->nb_neurons;
    int ex;
    float sc = pow2_scale_for(g5[i]->input_weights, (size_t)K * 3 * H, g5[i]->recurrent_weights, (size_t)H * 3 * H, &ex);
    t->scale_gru[i] = ldexpf(1.f, -(10 + ex));
    std::vector<__half> p;
    pack_gru(g5[i]->input_weights, K, H, sc, p);
    TCK(engine_upload(e, &t->w_gru[i], p.data(), p.size()));
    pack_gru(g5[i]->recurrent_weights, H, H, sc, p);
    TCK(engine_upload(e, &t->u_gru[i], p.data(), p.size()));
    // nnet.cpp:136-160: z and r start from b + b' (one float add), the candidate keeps b_n and b'_n apart
    const float *b = g5[i]->bias;
    std::vector<float4> b4(H);
    for (int j = 0; j < H; j++) b4[j] = make_float4(b[j] + b[3 * H + j], b[H + j] + b[4 * H + j], b[2 * H + j], b[5 * H + j]);
    TCK(engine_upload(e, &t->bias4[i], b4.data(), b4.size()));
  }
  {
    int ex;
    std::vector<__half> p;
    float sc = pow2_scale_for(model->fc_gb->input_weights, (size_t)2560 * 34, nullptr, 0, &ex);
    t->scale_gb = ldexpf(1.f, -(10 + ex));
    pack_small_h2(model->fc_gb->input_weights, 2560, 34, sc, p);
    TCK(engine_upload(e, &t->w_gb, p.data(), p.size()));
    sc = pow2_scale_for(model->fc_rb->input_weights, (size_t)128 * 34, nullptr, 0, &ex);
    t->scale_rb = ldexpf(1.f, -(10 + ex));
    pack_small_h2(model->fc_rb->input_weights, 128, 34, sc, p);
    TCK(engine_upload(e, &t->w_rb, p.data(), p.size()));
    std::vector<float> bp(512 + 512 + 48 + 48, 0.f);
    memcpy(bp.data(), model->conv1->bias, 512 * 4);
    memcpy(bp.data() + 512, model->conv2->bias, 512 * 4);
    memcpy(bp.data() + 1024, model->fc_gb->bias, 34 * 4);
    memcpy(bp.data() + 1072, model->fc_rb->bias, 34 * 4);
    TCK(engine_upload(e, &t->bias_pad, bp.data(), bp.size()));
  }
  int bad = 0;
  bad |= make_map(&t->m_wgb, t->w_gb, false, 2 * SMALL_BN, 2560, SMALL_BN);
  bad |= make_map(&t->m_wrb, t->w_rb, false, 2 * SMALL_BN, 128, SMALL_BN);
  bad |= make_map(&t->m_c2, t->c2_h, false, 2 * Fm * S, 512, TM);
  for (int i = 0; i < 5; i++)
    bad |= make_map(&t->m_h[i], t->h_all[i], false, 2 * (Fm + 1) * S, kGruH[i], TM);
  // the conv layers' and the chain's operands: boxes of 32 k
  const CUtensorMapSwizzle sw64 = CU_TENSOR_MAP_SWIZZLE_64B;
  bad |= make_map(&t->m_fc_all, t->fc_all, true, kConvTerms * (Fm + 4) * S, 128, TM, CBK, sw64);
  bad |= make_map(&t->m_c1_all, t->c1_all, true, kConvTerms * (Fm + 2) * S, 512, TM, CBK, sw64);
  bad |= make_map(&t->m_wconv1, t->w_conv1, true, kConvTerms * 512, 640, DENSE_BN, CBK, sw64);
  bad |= make_map(&t->m_wconv2, t->w_conv2, true, kConvTerms * 512, 1536, DENSE_BN, CBK, sw64);
  bad |= make_map(&t->m_c2_ch, t->c2_h, false, 2 * Fm * S, 512, TM, CBK, sw64);
  for (int i = 0; i < 5; i++) {
    const int rows = (kGruH[i] / HT) * GRU_BN;
    bad |= make_map(&t->m_h_ch[i], t->h_all[i], false, 2 * (Fm + 1) * S, kGruH[i], TM, CBK, sw64);
    bad |= make_map(&t->m_w[i], t->w_gru[i], false, 2 * rows, g5[i]->nb_inputs, GRU_BN, CBK, sw64);
    bad |= make_map(&t->m_u[i], t->u_gru[i], false, 2 * rows, kGruH[i], GRU_BN, CBK, sw64);
  }
  if (bad) return engine_fail(PNB_ERR_CUDA, "cuTensorMapEncodeTiled failed");
  TCK(cudaFuncSetAttribute(gru_chain_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                           (int)tc_smem_bytes<GRU_STAGES, GRU_STAGES * GruStage::kBytes>()));
  TCK(cudaFuncSetAttribute(conv_pair_kernel<5>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kConvSmem));
  TCK(cudaFuncSetAttribute(conv_pair_kernel<3>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kConvSmem));
  TCK(cudaFuncSetAttribute(tc_gemm_kernel<SMALL_BN, SMALL_STAGES>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                           (int)kSmallSmem));
  return PNB_OK;
}

// The tensor path's part of a stream's state: the conv input histories (the last 4 fc / 2 conv1 outputs, oldest first)
// as the three bf16 term planes of hop slots 0..3 / 0..1, and the fp16 hi / lo terms of the GRU states at slot 0.
// Export writes the terms and their fp32 sums; import restores the raw terms, or splits blobs without them (fp32-mode
// engines) with the roundings of store_split_b4 / store_split_h2.
int tc_state_segs(const pnb_engine *e, StateSeg *seg, int ns) {
  static_assert(kConvTerms == 3, "StreamState carries three bf16 terms per conv history value");
  const pnb_tc_state *t = e->tc.get();
  const size_t S = e->S, Fm = e->Fmax;
  auto hist = [&](const __nv_bfloat16 *base, size_t plane, int slots, int width, size_t sum_off, size_t terms_off) {
    for (int i = 0; i < slots; i++) {
      StateSeg g = StateSeg();
      g.kind = kSegSumBf16; g.eng = (char *)(base + (size_t)i * S * width); g.eng_stride = (size_t)width * 2;
      g.plane = plane * 2; g.blob_off = (unsigned)(sum_off + (size_t)i * width * 4); g.n = width;
      seg[ns++] = g;
      for (int tm = 0; tm < kConvTerms; tm++) {
        g.kind = kSegTermBf16; g.eng = (char *)(base + (size_t)tm * plane + (size_t)i * S * width); g.plane = 0;
        g.blob_off = (unsigned)(terms_off + ((size_t)tm * slots + i) * width * 2);
        g.aux_off = (unsigned)(sum_off + (size_t)i * width * 4); g.term = (short)tm;
        seg[ns++] = g;
      }
    }
  };
  hist(t->fc_all, (Fm + 4) * S * 128, 4, 128, offsetof(StreamState, fc_hist), offsetof(StreamState, fc_terms));
  hist(t->c1_all, (Fm + 2) * S * 512, 2, 512, offsetof(StreamState, c1_hist), offsetof(StreamState, c1_terms));
  size_t off = 0;
  for (int li = 0; li < 5; li++) {
    const size_t H = kGruH[li];
    for (int tm = 0; tm < 2; tm++) {
      StateSeg g = StateSeg();
      g.kind = kSegSplitF16; g.eng = (char *)(t->h_all[li] + (size_t)tm * (Fm + 1) * S * H); g.eng_stride = H * 2;
      g.blob_off = (unsigned)(offsetof(StreamState, h) + off * 4); g.n = (unsigned)H; g.scale = kActScale; g.term = (short)tm;
      seg[ns++] = g;
    }
    off += H;
  }
  return ns;
}

// One persistent tensor-core launch: a conv layer, an output layer or the GRU chain, each a tc_gemm_kernel record in the
// profile.
template <typename K, typename A>
static int tc_launch(pnb_engine *e, K kernel, const A &a, int units, size_t smem, cudaStream_t st) {
  int grid = units < e->sm_count ? units : e->sm_count;  // persistent: one CTA per SM
  if (grid < 1) grid = 1;
  LaunchScope m(e, PNB_K_TC_GEMM, st);
  kernel<<<grid, kTcThreads, smem, st>>>(a);
  TCK(cudaGetLastError());
  return PNB_OK;
}
// An output layer over the active rows of `slots` hop slots.  With every stream active the rows are one flat range of
// slots x S; otherwise each slot has its own ceil(n / 128) row tiles.
static int tc_launch_out(pnb_engine *e, TcArgs &a, int slots, cudaStream_t st) {
  const int n = e->n_active;
  if (n == e->S) {
    a.M = slots * n; a.slot_stride = 0; a.tiles_slot = (a.M + TM - 1) / TM; a.tiles_m = a.tiles_slot;
  } else {
    a.M = n; a.slot_stride = e->S; a.tiles_slot = (n + TM - 1) / TM; a.tiles_m = slots * a.tiles_slot;
  }
  a.tiles_n = 1;
  a.status = e->d_status;
  return tc_launch(e, tc_gemm_kernel<SMALL_BN, SMALL_STAGES>, a, a.tiles_m, kSmallSmem, st);
}
// A conv layer over the active rows of the call's F hops: ceil(n / 128) row tiles per hop pair
template <int Q>
static int tc_launch_conv(pnb_engine *e, ConvArgs &a, int F, cudaStream_t st) {
  a.S = e->S; a.n = e->n_active; a.F = F;
  a.pairs = (F + 1) / 2;
  a.tiles = (a.n + TM - 1) / TM * a.pairs * CONV_TILES_N;
  a.status = e->d_status;
  return tc_launch(e, conv_pair_kernel<Q>, a, a.tiles, kConvSmem, st);
}

static TcSeg mkseg(int a_map, int b_map, int K, int a_k0, int b_k0, int a_row0, int a_term_rows) {
  TcSeg s;
  s.a_map = a_map; s.b_map = b_map; s.k_blocks = K / BK; s.a_k0 = a_k0; s.b_k0 = b_k0;
  s.a_row0 = a_row0; s.a_term_rows = a_term_rows;
  return s;
}

// ---- the network of a call of F hops, in phases; each returns PNB_OK or a negative error --------------------------
// The non-recurrent front (rnn.cpp:50-52 on F S rows): fc -> conv1 -> conv2.  Hop t of the call lives in slot t of the
// per-call buffers.
static int tc_front(pnb_engine *e, int F, const int *hops, cudaStream_t st) {
  pnb_tc_state *t = e->tc.get();
  const int S = e->S, Fm = e->Fmax, na = e->n_active;
  const float *tbl = e->tansig();
  {  // fc (fp32 FMA on the CUDA cores) -> bf16 terms at slots 4 ..
    const int rows = na == S ? F * S : na, slots = na == S ? 1 : F;  // per grid.y slot
    LaunchScope m(e, PNB_K_TC_AUX, st);
    fc_split_kernel<<<dim3((rows + FC_ROWS - 1) / FC_ROWS, slots), 128, 0, st>>>(e->d_feat, e->fc.W, e->fc.b,
                                                    t->fc_all + (size_t)4 * S * 128, rows, (size_t)(Fm + 4) * S, (size_t)S);
  }
  // conv1: tap q of hop t reads fc slot t + q (oldest first, nnet.cpp:182-200); output -> c1 slots 2 + t
  ConvArgs a;
  memset(&a, 0, sizeof a);
  a.a_map = t->m_fc_all; a.w_map = t->m_wconv1;
  a.k_blocks = 128 / CBK; a.a_term_rows = (Fm + 4) * S;
  a.tansig = tbl; a.bias = t->bias_pad; a.wide = t->wide; a.act = PNB_ACT_RELU;
  a.out_b = t->c1_all; a.out_row0 = 2 * S; a.out_plane_rows = (Fm + 2) * S;
  if (int rc = tc_launch_conv<5>(e, a, F, st)) return rc;
  // conv2: three taps -> tanh -> fp16 terms (gru1 / gru_rb / fc_gb inputs); fp32 copy of the call's last hop (of each
  // row's last hop in a ragged call, whose frozen hops neither store nor raise the domain bit)
  memset(&a, 0, sizeof a);
  a.a_map = t->m_c1_all; a.w_map = t->m_wconv2;
  a.k_blocks = 512 / CBK; a.a_term_rows = (Fm + 2) * S;
  a.tansig = tbl; a.bias = t->bias_pad + 512; a.wide = t->wide; a.act = PNB_ACT_TANH;
  a.out_h = t->c2_h; a.out_f32 = e->c2; a.out_row0 = 0; a.out_plane_rows = Fm * S;
  a.hops = hops;
  return tc_launch_conv<3>(e, a, F, st);
}

// The recurrent part: five GRUs per hop (rnn.cpp:58-71) in one persistent launch.  State slot t holds the state
// BEFORE hop t of the call; the fp32 state e->h is updated in place.
static int tc_gru_chain(pnb_engine *e, int F, const int *hops, cudaStream_t st) {
  pnb_tc_state *t = e->tc.get();
  const int S = e->S, Fm = e->Fmax;
  ChainArgs a;
  memset(&a, 0, sizeof a);
  a.maps[0] = t->m_c2_ch;
  for (int i = 0; i < 5; i++) { a.maps[1 + i] = t->m_h_ch[i]; a.maps[6 + i] = t->m_w[i]; a.maps[11 + i] = t->m_u[i]; }
  // only the active streams' row tiles are units; the counters of the others stay zero.  With many streams one
  // layer-hop fills the machine and hop-major order keeps a layer's fresh output in L2 for the layer above; with few,
  // only the anti-diagonal order exposes enough independent units
  const int tiles_mp = (e->n_active + TM - 1) / TM;
  a.order = chain_order(F, tiles_mp, HT, (tiles_mp * (512 / HT) < e->sm_count) ? 1 : 0);
  a.S = S; a.n = e->n_active; a.cnt = t->cnt; a.tansig = e->tansig();
  a.hops = hops;
  const int c2_terms = Fm * S, h_terms = (Fm + 1) * S;
  for (int li = 0; li < 5; li++) {
    ChainLayer &L = a.L[li];
    const int H = kGruH[li], tiles = H / HT;
    L.H = H; L.h_kb = H / CBK;
    L.b_term_rows = tiles * GRU_BN;
    L.h_map = 1 + li; L.w_map = 6 + li; L.u_map = 11 + li;
    L.dep = chain_dep(li);
    L.scale = t->scale_gru[li];
    L.bias4 = t->bias4[li];
    L.h32 = e->h[li];
    L.h_hl = t->h_all[li]; L.h_term_rows = h_terms;
    // each GRU consumes the freshly written state (slot t+1) of the layer below (rnn.cpp:58-71, SURVEY.md App. C.10)
    if (li == 0) {          // gru1 <- conv2 out
      L.n_x = 1; L.x_map[0] = 0; L.x_kb[0] = 512 / CBK; L.x_bk0[0] = 0; L.x_row1[0] = 0; L.x_term_rows[0] = c2_terms;
    } else if (li < 4) {    // gru2 <- gru1, gru3 <- gru2, gru_gb <- gru3
      L.n_x = 1; L.x_map[0] = li; L.x_kb[0] = 512 / CBK; L.x_bk0[0] = 0; L.x_row1[0] = 1; L.x_term_rows[0] = h_terms;
    } else {                // gru_rb <- [gru3 state, conv2 out]
      L.n_x = 2;
      L.x_map[0] = 3; L.x_kb[0] = 512 / CBK; L.x_bk0[0] = 0; L.x_row1[0] = 1; L.x_term_rows[0] = h_terms;
      L.x_map[1] = 0; L.x_kb[1] = 512 / CBK; L.x_bk0[1] = 512; L.x_row1[1] = 0; L.x_term_rows[1] = c2_terms;
    }
  }
  return tc_launch(e, gru_chain_kernel, a, a.order.units(), tc_smem_bytes<GRU_STAGES, GRU_STAGES * GruStage::kBytes>(), st);
}

// The two 34-wide output layers (rnn.cpp:73-80; N padded to 48, fp16 two-term split, sigmoid epilogue).
static int tc_out(pnb_engine *e, int F, const int *, cudaStream_t st) {
  pnb_tc_state *t = e->tc.get();
  const int S = e->S, Fm = e->Fmax;
  const float *tbl = e->tansig();
  const int h_terms = (Fm + 1) * S;
  TcArgs a;
  memset(&a, 0, sizeof a);
  a.maps[0] = t->m_c2;
  for (int q = 0; q < 4; q++) a.maps[1 + q] = t->m_h[q];
  a.maps[5] = t->m_wgb;
  a.seg[0] = mkseg(0, 5, 512, 0, 0, 0, Fm * S);
  for (int q = 1; q < 5; q++) a.seg[q] = mkseg(q, 5, 512, 0, q * 512, S, h_terms);  // state after hop t = slot t+1
  a.n_seg = 5; a.b_term_rows = SMALL_BN; a.out_scale = t->scale_gb; a.tansig = tbl;
  a.bias = t->bias_pad + 1024; a.N = 34; a.ldc = 68; a.out_f32 = e->d_gr;
  if (int rc = tc_launch_out(e, a, F, st)) return rc;
  memset(&a, 0, sizeof a);
  a.maps[0] = t->m_h[4];
  a.maps[1] = t->m_wrb;
  a.seg[0] = mkseg(0, 1, 128, 0, 0, S, h_terms);
  a.n_seg = 1; a.b_term_rows = SMALL_BN; a.out_scale = t->scale_rb; a.tansig = tbl;
  a.bias = t->bias_pad + 1072; a.N = 34; a.ldc = 68; a.out_f32 = e->d_gr + 34;
  return tc_launch_out(e, a, F, st);
}

// End of a call of F hops: the last 4 fc / 2 conv1 hop slots and the last state slot move to the front (in a ragged
// call those of each row's own last hop), and the chain's dependency counters return to zero, in one launch.
static int tc_carry(pnb_engine *e, int F, const int *hops, cudaStream_t st) {
  pnb_tc_state *t = e->tc.get();
  const int S = e->S, Fm = e->Fmax, na = e->n_active;
  SlotCarry c;
  memset(&c, 0, sizeof c);
  c.hops = hops; c.h0 = 0; c.n = F; c.cnt = t->cnt; c.n_cnt = 5 * t->tiles_mp;
  for (int tm = 0; tm < kConvTerms; tm++) {
    __nv_bfloat16 *bf = t->fc_all + (size_t)tm * (Fm + 4) * S * 128, *bc = t->c1_all + (size_t)tm * (Fm + 2) * S * 512;
    add_carry_seg(c, bf, bf, 128 * 2, na, S, 4, F);
    add_carry_seg(c, bc, bc, 512 * 2, na, S, 2, F);
  }
  for (int li = 0; li < 5; li++)
    for (int tm = 0; tm < 2; tm++) {
      __half *b = t->h_all[li] + (size_t)tm * (Fm + 1) * S * kGruH[li];
      add_carry_seg(c, b, b, kGruH[li] * 2, na, S, 1, F);
    }
  LaunchScope m(e, PNB_K_TC_AUX, st);
  launch_slot_carry(c, e->sm_count, st);
  return PNB_OK;
}

int tc_network(pnb_engine *e, int F, const int *hops, cudaStream_t st) {
  for (int (*phase)(pnb_engine *, int, const int *, cudaStream_t) : {tc_front, tc_gru_chain, tc_out, tc_carry})
    if (int rc = phase(e, F, hops, st)) return rc;
  return PNB_OK;
}

int tc_network_launches(const pnb_engine *, int) { return 7; }  // fc, conv1, conv2, GRU chain, fc_gb, fc_rb, carry
