// pnb_train.cu -- the gradient of rnn_train.py's CustomLoss with respect to every parameter of its PercepNet, and an
// Adam step, on a PNB_TRAIN_NETWORK engine (the fp32 path's weight buffers are the parameters).
//
// One pnb_train_grad_* call of B windows x F hops, rows r = t*B + b (hop-major, like the engine's per-call buffers):
//   stage    rows_stage (records -> {30 rec[0..67], rec[68], rec[69]}), then the hops past each window's end set to zero
//   forward  fc, conv1, conv2 over all rows (train_gemm_kernel); per GRU its input products for all hops as one
//            contraction, then the recurrence in one persistent launch (gru_fwd_rec_kernel) that saves h, z, r, n and
//            W_hn h + b_hn; fc_gb / fc_rb.  Activations are exact tanhf / expf sigmoids (torch's), not the tansig table.
//   loss     loss_sums_kernel (pnb_rnn_io.cu) on the predictions; train_dpre_kernel the loss gradient at the output
//            pre-activations in closed form
//   backward output layers, then the GRUs in reverse dependency order (gru_rb, gru_gb, gru3, gru2, gru1): each layer's
//            gradient from its non-recurrent consumers is one contraction, its recurrence runs backwards in one
//            persistent launch (gru_bwd_rec_kernel); conv2, conv1, fc.  Weight gradients are contractions over the rows
//            (split over the rows into a fixed number of parts, then summed part by part in order).
//   check    one pass over the gradient: a non-finite value raises the engine's domain bit and makes the next Adam
//            step a no-op on the device
// No floating-point atomics anywhere: every sum has one fixed order, so a call's loss and gradient are the same bits
// whatever stream it runs on.
#include <math.h>
#include <string.h>

#include <string>

#include "pnb_chain.cuh"
#include "pnb_engine.h"

namespace pnb {
namespace {

constexpr int kParams = 25;  // parameter arrays in PNBW blob order: 5 dense / conv layers x 2, 5 GRUs x 3

// ---------------------------------------------------------------------------------------------------- contraction
// C[M x N] = epilogue(sum over segments of op(A_s)[M x K_s] * op(B_s)[K_s x N]).  op(A)(m, k) = A[m*lda + k], or
// A[k*lda + m] when TA; A == null is a matrix of ones (the column sums of a bias gradient).  op(B)(k, n) = B[k*ldb + n],
// or B[n*ldb + k] when TB.  X*W is <false, false>, dY*W^T <false, true>, X^T*dY <true, false>.
// With parts > 1 (X^T*dY only) the K range of one segment is cut into `parts` slices, slice z goes to C + z*M*N
// (ldc = N) and train_parts_kernel adds the slices in order.
enum { kEpiNone = 0, kEpiRelu, kEpiTanh, kEpiSigmoid, kEpiDRelu, kEpiDTanh };
struct TSeg {
  const float *A;
  size_t lda;
  const float *B;
  size_t ldb;
  int K;
};
struct TGemm {
  TSeg seg[5];
  int n_seg, M, N, parts;
  float *C;
  size_t ldc;
  int accumulate;      // C += instead of C =
  const float *bias;   // or null
  int epi;             // kEpi*: activations of the forward, or the activation derivative at aux
  const float *aux;    // kEpiDRelu: the saved output; kEpiDTanh: the saved pre-activation
  size_t ld_aux;
  float *pre;          // or null: the pre-activation (before epi) is also stored here, at ld_aux
};

constexpr int TBM = 64, TBN = 64, TBK = 16;

template <bool TA, bool TB>
__global__ void __launch_bounds__(256) train_gemm_kernel(const __grid_constant__ TGemm g) {
  __shared__ float As[TBK][TBM + 4];
  __shared__ float Bs[TBK][TBN + 4];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int m0 = blockIdx.y * TBM, n0 = blockIdx.x * TBN;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; i++)
#pragma unroll
    for (int j = 0; j < 4; j++) acc[i][j] = 0.f;
  for (int s = 0; s < g.n_seg; s++) {
    const TSeg S = g.seg[s];
    int k_lo = 0, k_hi = S.K;
    if (g.parts > 1) {
      const int per = (S.K + g.parts - 1) / g.parts;
      k_lo = min(S.K, (int)blockIdx.z * per);
      k_hi = min(S.K, k_lo + per);
    }
    for (int k0 = k_lo; k0 < k_hi; k0 += TBK) {
#pragma unroll
      for (int e = tid; e < TBM * TBK; e += 256) {
        const int mm = TA ? e % TBM : e / TBK, kk = TA ? e / TBM : e % TBK;
        const int m = m0 + mm, k = k0 + kk;
        float v = 0.f;
        if (m < g.M && k < k_hi) v = S.A ? __ldg(S.A + (TA ? (size_t)k * S.lda + m : (size_t)m * S.lda + k)) : 1.f;
        As[kk][mm] = v;
      }
#pragma unroll
      for (int e = tid; e < TBN * TBK; e += 256) {
        const int nn = TB ? e / TBK : e % TBN, kk = TB ? e % TBK : e / TBN;
        const int n = n0 + nn, k = k0 + kk;
        Bs[kk][nn] = (n < g.N && k < k_hi) ? __ldg(S.B + (TB ? (size_t)n * S.ldb + k : (size_t)k * S.ldb + n)) : 0.f;
      }
      __syncthreads();
#pragma unroll
      for (int kk = 0; kk < TBK; kk++) {
        float a[4], b[4];
#pragma unroll
        for (int i = 0; i < 4; i++) { a[i] = As[kk][ty * 4 + i]; b[i] = Bs[kk][tx * 4 + i]; }
#pragma unroll
        for (int i = 0; i < 4; i++)
#pragma unroll
          for (int j = 0; j < 4; j++) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
      }
      __syncthreads();
    }
  }
  float *C = g.C + (size_t)blockIdx.z * g.M * g.N;
#pragma unroll
  for (int i = 0; i < 4; i++) {
    const int m = m0 + ty * 4 + i;
    if (m >= g.M) continue;
#pragma unroll
    for (int j = 0; j < 4; j++) {
      const int n = n0 + tx * 4 + j;
      if (n >= g.N) continue;
      float *c = C + (size_t)m * g.ldc + n;
      float v = acc[i][j];
      if (g.accumulate) v += *c;
      if (g.bias) v += __ldg(g.bias + n);
      if (g.pre) g.pre[(size_t)m * g.ld_aux + n] = v;
      switch (g.epi) {
        case kEpiRelu: v = v < 0.f ? 0.f : v; break;
        case kEpiTanh: v = tanhf(v); break;
        case kEpiSigmoid: v = 1.f / (1.f + expf(-v)); break;
        case kEpiDRelu: v = g.aux[(size_t)m * g.ld_aux + n] > 0.f ? v : 0.f; break;  // selected, not multiplied
        case kEpiDTanh: {
          // tanh'(a) = 4 e / (1 + e)^2, e = exp(-2|a|), from the pre-activation: 1 - y^2 from the rounded output y would
          // lose every digit where tanh saturates (y = +-1 in fp32 from |a| > 9, tanh'(a) still up to 6e-8)
          const float e = expf(-2.f * fabsf(g.aux[(size_t)m * g.ld_aux + n]));
          v = v * (4.f * e / ((1.f + e) * (1.f + e)));
          break;
        }
        default: break;
      }
      *c = v;
    }
  }
}

// dst[i] = sum_{p < parts} part[p][i], in order
__global__ void train_parts_kernel(const float *__restrict__ part, int parts, size_t n, float *__restrict__ dst) {
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    float s = part[i];
    for (int p = 1; p < parts; p++) s += part[(size_t)p * n + i];
    dst[i] = s;
  }
}

// ---------------------------------------------------------------------------------------------------- recurrences
// One GRU layer over F hops, persistent: CTA c owns hidden units [c*JU, (c+1)*JU) and keeps their slice of U (forward:
// the 3*JU columns; backward: the JU rows) in shared memory for the whole launch.  A hop needs the whole state (the
// whole gate gradient) of the hop before it, written by every CTA: the CTAs bump one counter per hop (red.release) and
// wait for G of them (chain_wait, pnb_chain.cuh) -- the grid is sized to be co-resident.  A warp takes one row at a time;
// its lanes split the contraction and add their partials with a shuffle butterfly, which leaves the same sum in every
// lane (a + b == b + a), so lane ju finishes unit ju.
struct RecArgs {
  int H, n, F;
  const float *U, *bh;      // U [H][3H], b_hh [3H], gate order z, r, n (the reference's layout)
  const float *gx;          // [F][n][3H] input products + b_ih
  float *h;                 // [F+1][n][H], slot 0 zero: the state before hop t is slot t
  float *z, *r, *nn, *hn;   // [F][n][H]: the gates and W_hn h + b_hn
  const float *dh_ext;      // [F][n][H] gradient of the layer's output from its non-recurrent consumers
  float *dgx, *dgh;         // [F][n][3H]: gradient at the input products (z, r, n) and at the state products (z, r, hn)
  float *carry;             // [n][H]: dh * z of the hop after, per unit
  const int *frames;        // [n] hops per window (device), or null: F
  unsigned *cnt;            // hops finished x CTAs, zero at launch
};

__device__ __forceinline__ float sigm(float x) { return 1.f / (1.f + expf(-x)); }

template <int JU>
__global__ void __launch_bounds__(256) gru_fwd_rec_kernel(const __grid_constant__ RecArgs a) {
  extern __shared__ float Us[];  // [H][3 JU + 1]
  constexpr int NC = 3 * JU, SP = NC + 1;
  const int H = a.H, H3 = 3 * H, n = a.n, j0 = blockIdx.x * JU, G = gridDim.x;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  for (int i = tid; i < H * NC; i += blockDim.x) {
    const int k = i / NC, c = i - k * NC;
    Us[k * SP + c] = a.U[(size_t)k * H3 + (c / JU) * H + j0 + c % JU];
  }
  __syncthreads();
  for (int t = 0; t < a.F; t++) {
    if (t > 0) {
      if (tid == 0) chain_wait(a.cnt, (unsigned)t * G);
      __syncthreads();
    }
    const float *hp = a.h + (size_t)t * n * H;
    for (int b = warp; b < n; b += blockDim.x >> 5) {
      float acc[NC];
#pragma unroll
      for (int c = 0; c < NC; c++) acc[c] = 0.f;
      for (int k = lane; k < H; k += 32) {
        const float hv = __ldcg(hp + (size_t)b * H + k);
#pragma unroll
        for (int c = 0; c < NC; c++) acc[c] = fmaf(hv, Us[k * SP + c], acc[c]);
      }
#pragma unroll
      for (int c = 0; c < NC; c++)
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) acc[c] += __shfl_xor_sync(0xffffffffu, acc[c], o);
#pragma unroll
      for (int ju = 0; ju < JU; ju++) {
        if (lane != ju) continue;
        const int j = j0 + ju;
        const size_t row = (size_t)t * n + b;
        const float *x = a.gx + row * H3;
        const float z = sigm(x[j] + (acc[ju] + a.bh[j]));
        const float r = sigm(x[H + j] + (acc[JU + ju] + a.bh[H + j]));
        const float hn = acc[2 * JU + ju] + a.bh[2 * H + j];
        const float nv = tanhf(x[2 * H + j] + r * hn);
        const float ho = __ldcg(hp + (size_t)b * H + j);
        a.h[(row + n) * H + j] = (1.f - z) * nv + z * ho;
        a.z[row * H + j] = z; a.r[row * H + j] = r; a.nn[row * H + j] = nv; a.hn[row * H + j] = hn;
      }
    }
    __syncthreads();
    if (tid == 0) {
      __threadfence();
      red_release_gpu_add(a.cnt, 1u);
    }
  }
}

template <int JU>
__global__ void __launch_bounds__(256) gru_bwd_rec_kernel(const __grid_constant__ RecArgs a) {
  extern __shared__ float Ur[];  // [JU][3H]: rows j0.. of U
  const int H = a.H, H3 = 3 * H, n = a.n, j0 = blockIdx.x * JU, G = gridDim.x;
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  for (int i = tid; i < JU * H3; i += blockDim.x) Ur[i] = a.U[(size_t)j0 * H3 + i];
  __syncthreads();
  for (int s = 0; s < a.F; s++) {
    const int t = a.F - 1 - s;
    if (s > 0) {
      if (tid == 0) chain_wait(a.cnt, (unsigned)s * G);
      __syncthreads();
    }
    for (int b = warp; b < n; b += blockDim.x >> 5) {
      const int fr = a.frames ? a.frames[b] : a.F;
      const bool live = t < fr, rec = t + 1 < fr;  // hop t counts; hop t+1 counts (else nothing flows back from it)
      float acc[JU];
#pragma unroll
      for (int ju = 0; ju < JU; ju++) acc[ju] = 0.f;
      if (rec) {
        const float *gp = a.dgh + ((size_t)(t + 1) * n + b) * H3;
        for (int c = lane; c < H3; c += 32) {
          const float d = __ldcg(gp + c);
#pragma unroll
          for (int ju = 0; ju < JU; ju++) acc[ju] = fmaf(d, Ur[ju * H3 + c], acc[ju]);
        }
#pragma unroll
        for (int ju = 0; ju < JU; ju++)
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) acc[ju] += __shfl_xor_sync(0xffffffffu, acc[ju], o);
      }
#pragma unroll
      for (int ju = 0; ju < JU; ju++) {
        if (lane != ju) continue;
        const int j = j0 + ju;
        const size_t row = (size_t)t * n + b;
        float *gx = a.dgx + row * H3, *gh = a.dgh + row * H3, *cr = a.carry + (size_t)b * H + j;
        if (!live) {  // past the window's end: zeros, written, whatever the saved activations hold
          gx[j] = 0.f; gx[H + j] = 0.f; gx[2 * H + j] = 0.f;
          gh[j] = 0.f; gh[H + j] = 0.f; gh[2 * H + j] = 0.f;
          *cr = 0.f;
          continue;
        }
        float dh = a.dh_ext[row * H + j];
        if (rec) dh += acc[ju] + *cr;
        const float z = a.z[row * H + j], r = a.r[row * H + j], nv = a.nn[row * H + j], hn = a.hn[row * H + j];
        const float hp = a.h[row * H + j];  // slot t: the state before hop t
        const float dan = dh * (1.f - z) * (1.f - nv * nv);
        const float daz = dh * (hp - nv) * z * (1.f - z);
        const float dar = dan * hn * r * (1.f - r);
        gx[j] = daz; gx[H + j] = dar; gx[2 * H + j] = dan;
        gh[j] = daz; gh[H + j] = dar; gh[2 * H + j] = dan * r;
        *cr = dh * z;
      }
    }
    __syncthreads();
    if (tid == 0) {
      __threadfence();
      red_release_gpu_add(a.cnt, 1u);
    }
  }
}

// ---------------------------------------------------------------------------------------------------- elementwise
// x [F][n][70]: the hops t >= frames[b] of window b become zeros, so that nothing past a window's end (NaN included)
// reaches any activation the gradient multiplies
__global__ void train_mask_kernel(float *__restrict__ x, const int *__restrict__ frames, int n, int F) {
  const size_t total = (size_t)F * n * kFeat;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t row = i / kFeat;
    const int b = (int)(row % n), t = (int)(row / n);
    if (frames && t >= frames[b]) x[i] = 0.f;
  }
}

// CustomLoss's gradient at the output pre-activations (sigmoid inputs), in closed form, in float64: with p the
// prediction and y the label of a counted hop,
//   g: d/da = -dg (1 + 2 C4 dg^2) sqrt(p) (1 - p),  dg = sqrt(y) - sqrt(p)
//   r: d/da =  dr p sqrt(1 - p),                    dr = sqrt(1 - y) - sqrt(1 - p)
// times 1/count of the means.  Finite at p = 0 and p = 1, where torch's autograd of the same loss multiplies an
// infinite d/dp by a zero sigmoid derivative and returns NaN.  Hops past a window's end get zeros.
__global__ void train_dpre_kernel(const float *__restrict__ pred, const float *__restrict__ rec, size_t rec_stride,
                                  const int *__restrict__ frames, int n, int F, double inv_count, float *__restrict__ d) {
  const size_t total = (size_t)F * n * 68;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int k = (int)(i % 68);
    const size_t row = i / 68;
    const int b = (int)(row % n), t = (int)(row / n);
    if (t >= (frames ? frames[b] : F)) { d[i] = 0.f; continue; }
    const double p = pred[i], y = rec[(size_t)b * rec_stride + (size_t)t * PNB_RECORD_FLOATS + 70 + k];
    double v;
    if (k < kBands) {
      const double dg = sqrt(y) - sqrt(p);
      v = -dg * (1.0 + 20.0 * dg * dg) * sqrt(p) * (1.0 - p);
    } else {
      v = (sqrt(1.0 - y) - sqrt(1.0 - p)) * p * sqrt(1.0 - p);
    }
    d[i] = (float)(v * inv_count);
  }
}

// bad = 1 (and the engine's domain bit) when any of the n gradient values is not finite; bad is zeroed before
__global__ void train_check_kernel(const float *__restrict__ g, size_t n, int *bad, int *status) {
  bool found = false;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    found |= !isfinite(g[i]);
  if (__syncthreads_or(found) && threadIdx.x == 0) {
    *bad = 1;
    atomicOr(status, 1);
  }
}

struct AdamArgs {
  float *p[kParams];
  size_t off[kParams + 1];
  const float *g;
  float *m, *v;
  const int *bad;
  float w1, s2, bc2_sqrt, neg_step, eps;
};
// torch.optim.Adam's single-tensor step (defaults, no weight decay / amsgrad) with torch's own roundings on the CPU:
//   m.lerp_(g, 1 - b1)                       m + w1 (g - m), fused (ATen's vectorised lerp)
//   v.mul_(b2).addcmul_(g, g, value=1 - b2)  (s2 g) g + (v b2), fused
//   p.addcdiv_(m, sqrt(v) / sqrt(bc2) + eps, value=-lr/bc1)   p + (-step m) / denom
// skipped entirely when the gradient pass flagged a non-finite value
__global__ void train_adam_kernel(const __grid_constant__ AdamArgs a) {
  if (*a.bad) return;
  const int s = blockIdx.y;
  const size_t n = a.off[s + 1] - a.off[s];
  float *p = a.p[s];
  const float *g = a.g + a.off[s];
  float *m = a.m + a.off[s], *v = a.v + a.off[s];
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const float gi = g[i];
    const float mi = fmaf(a.w1, __fsub_rn(gi, m[i]), m[i]);
    const float vi = fmaf(__fmul_rn(a.s2, gi), gi, __fmul_rn(v[i], 0.999f));
    const float den = __fadd_rn(__fdiv_rn(sqrtf(vi), a.bc2_sqrt), a.eps);
    p[i] = __fadd_rn(p[i], __fdiv_rn(__fmul_rn(a.neg_step, mi), den));
    m[i] = mi;
    v[i] = vi;
  }
}

unsigned blocks_for(size_t total, unsigned cap = 4096) {
  const size_t b = (total + 255) / 256;
  return (unsigned)(b < cap ? (b ? b : 1) : cap);
}

}  // namespace
}  // namespace pnb

// ------------------------------------------------------------------------------------------ host state
using namespace pnb;

struct pnb_train_state {
  float *param[kParams];
  size_t off[kParams + 1];
  float *grad = nullptr, *m = nullptr, *v = nullptr;  // [N] flat, blob order
  float *part = nullptr;                               // partial sums of the split weight-gradient contractions
  int *bad = nullptr;
  unsigned *cnt = nullptr;                             // [10] counters of the recurrences, zeroed per call
  // activations and gradients of one call, rows r = t*n + b; sized for S windows x Fmax hops
  float *x = nullptr;       // [F][n][70]
  float *fc = nullptr;      // [F+4][n][128]: slots 0..3 zero (conv1's history), hop t in slot t+4
  float *c1 = nullptr;      // [F+2][n][512]: slots 0..1 zero, hop t in slot t+2
  float *c2 = nullptr;      // [F][n][512]
  float *c2p = nullptr;     // [F][n][512]: conv2's pre-activation, for tanh' in the backward
  float *h[5] = {}, *z[5] = {}, *r[5] = {}, *nn[5] = {}, *hn[5] = {};  // [F+1][n][H] (slot 0 zero) / [F][n][H]
  float *pred = nullptr, *dpre = nullptr;  // [F][n][68]
  float *g1 = nullptr, *g2 = nullptr;      // [F][n][1536]: input products (forward); dgx, dgh (backward)
  float *ea = nullptr, *eb = nullptr;      // [F+4][n][512]: layer gradients, trailing zero slots for the conv backward
  float *dc2 = nullptr;                    // [F+2][n][512]
  float *carry = nullptr;                  // [S][512]
  int G512 = 0, G128 = 0;                  // CTAs of the recurrences (a power of two, co-resident)
};

constexpr size_t kPartFloats = (size_t)1 << 21;

#define TCK(call)                                                                                                   \
  do {                                                                                                              \
    cudaError_t _e = (call);                                                                                        \
    if (_e != cudaSuccess)                                                                                          \
      return engine_fail(_e == cudaErrorMemoryAllocation ? PNB_ERR_ALLOC : PNB_ERR_CUDA,                            \
                         (std::string(#call) + " failed: " + cudaGetErrorString(_e)).c_str());                      \
  } while (0)

template <int JU>
static cudaError_t rec_attr(size_t fwd, size_t bwd) {
  cudaError_t e1 = cudaFuncSetAttribute(gru_fwd_rec_kernel<JU>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)fwd);
  cudaError_t e2 = cudaFuncSetAttribute(gru_bwd_rec_kernel<JU>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bwd);
  return e1 != cudaSuccess ? e1 : e2;
}
static size_t fwd_smem(int H, int JU) { return (size_t)H * (3 * JU + 1) * sizeof(float); }
static size_t bwd_smem(int H, int JU) { return (size_t)JU * 3 * H * sizeof(float); }

// The most CTAs (a power of two, at most 128 and at most H) of which every one fits on the device at once with the
// shared memory its slice of U takes.
static int rec_grid(const pnb_engine *e, int H) {
  for (int G = 128; G >= 8; G >>= 1) {
    if (G > H) continue;
    const int JU = H / G;
    if (JU > 16) return 0;
    int occ = 0;
    const size_t sm = fwd_smem(H, JU) > bwd_smem(H, JU) ? fwd_smem(H, JU) : bwd_smem(H, JU);
    cudaError_t ce;
    switch (JU) {
      case 1: ce = rec_attr<1>(fwd_smem(H, 1), bwd_smem(H, 1)); if (!ce) ce = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, gru_bwd_rec_kernel<1>, 256, sm); break;
      case 2: ce = rec_attr<2>(fwd_smem(H, 2), bwd_smem(H, 2)); if (!ce) ce = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, gru_bwd_rec_kernel<2>, 256, sm); break;
      case 4: ce = rec_attr<4>(fwd_smem(H, 4), bwd_smem(H, 4)); if (!ce) ce = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, gru_bwd_rec_kernel<4>, 256, sm); break;
      case 8: ce = rec_attr<8>(fwd_smem(H, 8), bwd_smem(H, 8)); if (!ce) ce = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, gru_bwd_rec_kernel<8>, 256, sm); break;
      default: ce = rec_attr<16>(fwd_smem(H, 16), bwd_smem(H, 16)); if (!ce) ce = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, gru_bwd_rec_kernel<16>, 256, sm); break;
    }
    if (ce != cudaSuccess) return 0;
    if (occ * e->sm_count >= G) return G;
  }
  return 0;
}

int train_prepare(pnb_engine *e) {
  e->train = std::make_shared<pnb_train_state>();
  pnb_train_state &s = *e->train;
  size_t count[kParams];
  { const int rc = f32_params(e, s.param, count); if (rc) return rc; }
  s.off[0] = 0;
  for (int i = 0; i < kParams; i++) s.off[i + 1] = s.off[i] + count[i];
  const size_t N = s.off[kParams], S = e->S, F = e->Fmax, R = S * F;
  if (R > (size_t)65535 * TBM)  // the contractions put the rows on gridDim.y
    return engine_fail(PNB_ERR_ARG, "PNB_TRAIN_NETWORK: n_streams x max_frames_per_call above 65535 x 64 rows");
  TCK(engine_alloc(e, &s.grad, N, kScratch));  // kScratch: pnb_reset keeps the gradient and Adam's moments
  TCK(engine_alloc(e, &s.m, N, kScratch));
  TCK(engine_alloc(e, &s.v, N, kScratch));
  TCK(engine_alloc(e, &s.part, kPartFloats, kScratch));
  TCK(engine_alloc(e, &s.bad, 1, kScratch));
  TCK(engine_alloc(e, &s.cnt, 10, kScratch));
  TCK(engine_alloc(e, &s.x, R * kFeat, kScratch));
  TCK(engine_alloc(e, &s.fc, (F + 4) * S * 128, kScratch));
  TCK(engine_alloc(e, &s.c1, (F + 2) * S * 512, kScratch));
  TCK(engine_alloc(e, &s.c2, R * 512, kScratch));
  TCK(engine_alloc(e, &s.c2p, R * 512, kScratch));
  for (int l = 0; l < 5; l++) {
    const size_t H = kGruH[l];
    TCK(engine_alloc(e, &s.h[l], (F + 1) * S * H, kScratch));
    TCK(engine_alloc(e, &s.z[l], R * H, kScratch));
    TCK(engine_alloc(e, &s.r[l], R * H, kScratch));
    TCK(engine_alloc(e, &s.nn[l], R * H, kScratch));
    TCK(engine_alloc(e, &s.hn[l], R * H, kScratch));
  }
  TCK(engine_alloc(e, &s.pred, R * 68, kScratch));
  TCK(engine_alloc(e, &s.dpre, R * 68, kScratch));
  TCK(engine_alloc(e, &s.g1, R * 1536, kScratch));
  TCK(engine_alloc(e, &s.g2, R * 1536, kScratch));
  TCK(engine_alloc(e, &s.ea, (F + 4) * S * 512, kScratch));
  TCK(engine_alloc(e, &s.eb, (F + 4) * S * 512, kScratch));
  TCK(engine_alloc(e, &s.dc2, (F + 2) * S * 512, kScratch));
  TCK(engine_alloc(e, &s.carry, S * 512, kScratch));
  s.G512 = rec_grid(e, 512);
  s.G128 = rec_grid(e, 128);
  if (!s.G512 || !s.G128) return engine_fail(PNB_ERR_CUDA, "cannot configure the training recurrence kernels");
  return PNB_OK;
}

// ---- launch helpers
namespace {
TSeg tseg(const float *A, size_t lda, const float *B, size_t ldb, int K) { return {A, lda, B, ldb, K}; }

struct Launcher {
  pnb_engine *e;
  cudaStream_t st;
  int n = 0;
  cudaError_t err = cudaSuccess;
  void check() { if (err == cudaSuccess) err = cudaGetLastError(); }

  // C[M x N] (=, or += with acc) epi(sum_s A_s W_s + bias): forward products and dY W^T
  void gemm(bool tb, const TSeg *segs, int n_seg, int M, int N, float *C, size_t ldc, const float *bias = nullptr,
            int epi = kEpiNone, bool acc = false, const float *aux = nullptr, size_t ld_aux = 0, float *pre = nullptr) {
    TGemm g;
    memset(&g, 0, sizeof g);
    for (int i = 0; i < n_seg; i++) g.seg[i] = segs[i];
    g.n_seg = n_seg; g.M = M; g.N = N; g.parts = 1; g.C = C; g.ldc = ldc; g.accumulate = acc; g.bias = bias;
    g.epi = epi; g.aux = aux; g.ld_aux = ld_aux; g.pre = pre;
    dim3 grid((N + TBN - 1) / TBN, (M + TBM - 1) / TBM, 1);
    if (tb) train_gemm_kernel<false, true><<<grid, 256, 0, st>>>(g);
    else train_gemm_kernel<false, false><<<grid, 256, 0, st>>>(g);
    n++;
    check();
  }
  // dst[M x N] (contiguous) = X^T dY over R rows: X [R][ldx] (null: ones, a bias gradient with M = 1), dY [R][ldy].
  // The rows are cut into parts (a function of the shapes only), summed in order by a second launch.
  void wgrad(const float *X, size_t ldx, int M, const float *dY, size_t ldy, int N, int R, float *dst) {
    const int tiles = ((N + TBN - 1) / TBN) * ((M + TBM - 1) / TBM);
    int parts = (2 * e->sm_count + tiles - 1) / tiles;
    const int by_k = (R + 1023) / 1024;
    if (parts > by_k) parts = by_k;
    const int by_mem = (int)(kPartFloats / ((size_t)M * N));
    if (parts > by_mem) parts = by_mem;
    if (parts > 64) parts = 64;
    if (parts < 1) parts = 1;
    TGemm g;
    memset(&g, 0, sizeof g);
    g.seg[0] = tseg(X, ldx, dY, ldy, R);
    g.n_seg = 1; g.M = M; g.N = N; g.parts = parts; g.C = e->train->part; g.ldc = N;
    dim3 grid((N + TBN - 1) / TBN, (M + TBM - 1) / TBM, parts);
    train_gemm_kernel<true, false><<<grid, 256, 0, st>>>(g);
    const size_t cnt = (size_t)M * N;
    train_parts_kernel<<<blocks_for(cnt), 256, 0, st>>>(e->train->part, parts, cnt, dst);
    n += 2;
    check();
  }
  template <int JU>
  void rec_launch(const RecArgs &a, int G, bool fwd) {
    if (fwd) gru_fwd_rec_kernel<JU><<<G, 256, fwd_smem(a.H, JU), st>>>(a);
    else gru_bwd_rec_kernel<JU><<<G, 256, bwd_smem(a.H, JU), st>>>(a);
  }
  void rec(const RecArgs &a, bool fwd) {
    const int G = a.H == 512 ? e->train->G512 : e->train->G128, JU = a.H / G;
    switch (JU) {
      case 1: rec_launch<1>(a, G, fwd); break;
      case 2: rec_launch<2>(a, G, fwd); break;
      case 4: rec_launch<4>(a, G, fwd); break;
      case 8: rec_launch<8>(a, G, fwd); break;
      default: rec_launch<16>(a, G, fwd); break;
    }
    n++;
    check();
  }
};
}  // namespace

// The parameter arrays in blob order: fc W, b (0, 1); conv1 (2, 3); conv2 (4, 5); GRU k = 0..4 (gru1, gru2, gru3,
// gru_gb, gru_rb) W, U, b at 6 + 3k .. 8 + 3k; fc_gb (21, 22); fc_rb (23, 24).
int train_grad(pnb_engine *e, const float *rec, size_t rec_stride, const int *frames, const int *h_frames, double *sums,
               int F, cudaStream_t st) {
  pnb_train_state &s = *e->train;
  const int n = e->n_active, R = F * n;
  const size_t nb = (size_t)n;
  Launcher L{e, st};
  float *const *P = s.param;
  float *G = s.grad;
  const size_t *O = s.off;
  // per call: the counters, the flag and the zero slots (the row stride n changes from call to call)
  TCK(cudaMemsetAsync(s.cnt, 0, 10 * sizeof(unsigned), st));
  TCK(cudaMemsetAsync(s.bad, 0, sizeof(int), st));
  TCK(cudaMemsetAsync(s.fc, 0, 4 * nb * 128 * sizeof(float), st));
  TCK(cudaMemsetAsync(s.c1, 0, 2 * nb * 512 * sizeof(float), st));
  for (int l = 0; l < 5; l++) TCK(cudaMemsetAsync(s.h[l], 0, nb * kGruH[l] * sizeof(float), st));
  TCK(cudaMemsetAsync(s.dc2 + (size_t)R * 512, 0, 2 * nb * 512 * sizeof(float), st));
  TCK(cudaMemsetAsync(s.ea + (size_t)R * 512, 0, 4 * nb * 512 * sizeof(float), st));

  // ---- stage: {30 rec[0..67], rec[68], rec[69]}, zero past each window's end
  L.n += launch_rows_stage(s.x, kFeat, rec, rec_stride, PNB_RECORD_FLOATS, 68, n, n, F, st);
  train_mask_kernel<<<blocks_for((size_t)R * kFeat), 256, 0, st>>>(s.x, frames, n, F);
  L.n++;
  L.check();

  // ---- forward
  float *fc_out = s.fc + 4 * nb * 128, *c1_out = s.c1 + 2 * nb * 512;
  { TSeg a[1] = {tseg(s.x, kFeat, P[0], 128, kFeat)}; L.gemm(false, a, 1, R, 128, fc_out, 128, P[1], kEpiRelu); }
  {
    TSeg a[5];
    for (int q = 0; q < 5; q++) a[q] = tseg(s.fc + q * nb * 128, 128, P[2] + (size_t)q * 128 * 512, 512, 128);
    L.gemm(false, a, 5, R, 512, c1_out, 512, P[3], kEpiRelu);
  }
  {
    TSeg a[3];
    for (int q = 0; q < 3; q++) a[q] = tseg(s.c1 + q * nb * 512, 512, P[4] + (size_t)q * 512 * 512, 512, 512);
    L.gemm(false, a, 3, R, 512, s.c2, 512, P[5], kEpiTanh, false, nullptr, 512, s.c2p);
  }
  auto rec_args = [&](int l) {
    RecArgs a;
    memset(&a, 0, sizeof a);
    a.H = kGruH[l]; a.n = n; a.F = F;
    a.U = P[7 + 3 * l]; a.bh = P[8 + 3 * l] + 3 * kGruH[l];
    a.gx = s.g1; a.h = s.h[l]; a.z = s.z[l]; a.r = s.r[l]; a.nn = s.nn[l]; a.hn = s.hn[l];
    a.dgx = s.g1; a.dgh = s.g2; a.carry = s.carry; a.frames = frames;
    return a;
  };
  auto out_of = [&](int l) { return s.h[l] + nb * kGruH[l]; };  // the layer's output at hop t: slot t+1
  for (int l = 0; l < 5; l++) {
    const int H = kGruH[l], H3 = 3 * H;
    const float *W = P[6 + 3 * l], *b = P[8 + 3 * l];
    if (l == 0) { TSeg a[1] = {tseg(s.c2, 512, W, H3, 512)}; L.gemm(false, a, 1, R, H3, s.g1, H3, b); }
    else if (l < 4) { TSeg a[1] = {tseg(out_of(l - 1), 512, W, H3, 512)}; L.gemm(false, a, 1, R, H3, s.g1, H3, b); }
    else {
      TSeg a[2] = {tseg(out_of(2), 512, W, H3, 512), tseg(s.c2, 512, W + (size_t)512 * H3, H3, 512)};
      L.gemm(false, a, 2, R, H3, s.g1, H3, b);
    }
    RecArgs a = rec_args(l);
    a.cnt = s.cnt + l;
    L.rec(a, true);
  }
  {
    TSeg a[5] = {tseg(s.c2, 512, P[21], 34, 512)};
    for (int q = 1; q < 5; q++) a[q] = tseg(out_of(q - 1), 512, P[21] + (size_t)q * 512 * 34, 34, 512);
    L.gemm(false, a, 5, R, 34, s.pred, 68, P[22], kEpiSigmoid);
    TSeg c[1] = {tseg(out_of(4), 128, P[23], 34, 128)};
    L.gemm(false, c, 1, R, 34, s.pred + 34, 68, P[24], kEpiSigmoid);
  }

  // ---- loss and its gradient at the output pre-activations
  L.n += launch_loss_sums(s.pred, rec, rec_stride, frames, sums, n, n, F, st);
  long long counted = 0;
  for (int i = 0; i < n; i++) counted += h_frames ? h_frames[i] : F;
  train_dpre_kernel<<<blocks_for((size_t)R * 68), 256, 0, st>>>(s.pred, rec, rec_stride, frames, n, F,
                                                                1.0 / ((double)counted * kBands), s.dpre);
  L.n++;
  L.check();

  // ---- backward.  Weight gradients go straight into the flat gradient at their blob offsets.
  const float *dg = s.dpre, *dr = s.dpre + 34;
  // fc_rb
  L.wgrad(out_of(4), 128, 128, dr, 68, 34, R, G + O[23]);
  L.wgrad(nullptr, 0, 1, dr, 68, 34, R, G + O[24]);
  { TSeg a[1] = {tseg(dr, 68, P[23], 34, 34)}; L.gemm(true, a, 1, R, 128, s.ea, 128); }
  // a GRU's recurrence backwards and its weight gradients; X segments: its inputs
  auto gru_back = [&](int l, const float *ext, const float *X0, const float *X1) {
    const int H = kGruH[l], H3 = 3 * H;
    RecArgs a = rec_args(l);
    a.dh_ext = ext;
    a.cnt = s.cnt + 5 + l;
    L.rec(a, false);
    L.wgrad(X0, 512, 512, s.g1, H3, H3, R, G + O[6 + 3 * l]);
    if (X1) L.wgrad(X1, 512, 512, s.g1, H3, H3, R, G + O[6 + 3 * l] + (size_t)512 * H3);
    L.wgrad(s.h[l], H, H, s.g2, H3, H3, R, G + O[7 + 3 * l]);  // slot t: the state before hop t
    L.wgrad(nullptr, 0, 1, s.g1, H3, H3, R, G + O[8 + 3 * l]);
    L.wgrad(nullptr, 0, 1, s.g2, H3, H3, R, G + O[8 + 3 * l] + H3);
  };
  const float *Wfg = P[21];
  auto fcgb_rows = [&](int q) { return tseg(dg, 68, Wfg + (size_t)q * 512 * 34, 34, 34); };  // dY_g W_fcgb[q]^T
  // gru_rb: its inputs are [gru3, conv2]
  gru_back(4, s.ea, out_of(2), s.c2);
  {
    const float *W = P[18];
    TSeg a[1] = {tseg(s.g1, 384, W, 384, 384)};
    L.gemm(true, a, 1, R, 512, s.eb, 512);                                    // gru3's share
    TSeg c[1] = {tseg(s.g1, 384, W + (size_t)512 * 384, 384, 384)};
    L.gemm(true, c, 1, R, 512, s.dc2, 512);                                   // conv2's share
  }
  // fc_gb
  L.wgrad(s.c2, 512, 512, dg, 68, 34, R, G + O[21]);
  for (int q = 1; q < 5; q++) L.wgrad(out_of(q - 1), 512, 512, dg, 68, 34, R, G + O[21] + (size_t)q * 512 * 34);
  L.wgrad(nullptr, 0, 1, dg, 68, 34, R, G + O[22]);
  { TSeg a[1] = {fcgb_rows(0)}; L.gemm(true, a, 1, R, 512, s.dc2, 512, nullptr, kEpiNone, true); }
  // gru_gb
  { TSeg a[1] = {fcgb_rows(4)}; L.gemm(true, a, 1, R, 512, s.ea, 512); }
  gru_back(3, s.ea, out_of(2), nullptr);
  { TSeg a[2] = {tseg(s.g1, 1536, P[15], 1536, 1536), fcgb_rows(3)}; L.gemm(true, a, 2, R, 512, s.eb, 512, nullptr, kEpiNone, true); }
  // gru3, gru2, gru1: each one's input gradient plus fc_gb's share is the layer below's
  gru_back(2, s.eb, out_of(1), nullptr);
  { TSeg a[2] = {tseg(s.g1, 1536, P[12], 1536, 1536), fcgb_rows(2)}; L.gemm(true, a, 2, R, 512, s.ea, 512); }
  gru_back(1, s.ea, out_of(0), nullptr);
  { TSeg a[2] = {tseg(s.g1, 1536, P[9], 1536, 1536), fcgb_rows(1)}; L.gemm(true, a, 2, R, 512, s.eb, 512); }
  gru_back(0, s.eb, s.c2, nullptr);
  // conv2: its output gradient through tanh
  { TSeg a[1] = {tseg(s.g1, 1536, P[6], 1536, 1536)}; L.gemm(true, a, 1, R, 512, s.dc2, 512, nullptr, kEpiDTanh, true, s.c2p, 512); }
  for (int q = 0; q < 3; q++) L.wgrad(s.c1 + q * nb * 512, 512, 512, s.dc2, 512, 512, R, G + O[4] + (size_t)q * 512 * 512);
  L.wgrad(nullptr, 0, 1, s.dc2, 512, 512, R, G + O[5]);
  {  // conv1 output gradient: hop t gets tap q of hop t + 2 - q (the trailing zero slots end the sum)
    TSeg a[3];
    for (int q = 0; q < 3; q++) a[q] = tseg(s.dc2 + (2 - q) * nb * 512, 512, P[4] + (size_t)q * 512 * 512, 512, 512);
    L.gemm(true, a, 3, R, 512, s.ea, 512, nullptr, kEpiDRelu, false, c1_out, 512);
  }
  for (int q = 0; q < 5; q++) L.wgrad(s.fc + q * nb * 128, 128, 128, s.ea, 512, 512, R, G + O[2] + (size_t)q * 128 * 512);
  L.wgrad(nullptr, 0, 1, s.ea, 512, 512, R, G + O[3]);
  {
    TSeg a[5];
    for (int q = 0; q < 5; q++) a[q] = tseg(s.ea + (4 - q) * nb * 512, 512, P[2] + (size_t)q * 128 * 512, 512, 512);
    L.gemm(true, a, 5, R, 128, s.eb, 128, nullptr, kEpiDRelu, false, fc_out, 128);
  }
  L.wgrad(s.x, kFeat, kFeat, s.eb, 128, 128, R, G + O[0]);
  L.wgrad(nullptr, 0, 1, s.eb, 128, 128, R, G + O[1]);

  const size_t N = O[kParams];
  train_check_kernel<<<blocks_for(N, 1024), 256, 0, st>>>(G, N, s.bad, e->d_status);
  L.n++;
  L.check();
  TCK(L.err);
  // pnb_launches_per_call reports train_grad_launches: the schedule above and that count must agree
  if (L.n != train_grad_launches(e)) return engine_fail(PNB_ERR_CUDA, "train_grad issued a launch count train_grad_launches does not know");
  return L.n;
}

// The launches of train_grad, which does not depend on the shape of the call: stage 2; forward 3 + 5 x 2 + 2; loss 2;
// backward 99 (fc_rb 5, gru_rb 11 + 2, fc_gb 13, gru_gb 1 + 9 + 1, gru3 and gru2 9 + 1 each, gru1 9, conv2 9, conv1 13,
// fc 5, check 1).
int train_grad_launches(const pnb_engine *) { return 118; }

int train_adam(pnb_engine *e, double lr, long long step, cudaStream_t st) {
  const pnb_train_state &s = *e->train;
  AdamArgs a;
  memset(&a, 0, sizeof a);
  for (int i = 0; i < kParams; i++) a.p[i] = s.param[i];
  for (int i = 0; i <= kParams; i++) a.off[i] = s.off[i];
  a.g = s.grad; a.m = s.m; a.v = s.v; a.bad = s.bad;
  // torch's scalars: python floats, cast to float32 by the tensor ops
  const double bc1 = 1.0 - pow(0.9, (double)step), bc2 = 1.0 - pow(0.999, (double)step);
  a.w1 = (float)(1.0 - 0.9);
  a.s2 = (float)(1.0 - 0.999);
  a.bc2_sqrt = (float)pow(bc2, 0.5);
  a.neg_step = (float)(-(lr / bc1));
  a.eps = 1e-8f;
  train_adam_kernel<<<dim3(64, kParams), 256, 0, st>>>(a);
  TCK(cudaGetLastError());
  return 1;
}

// what: 0 weights, 1 gradient, 2 Adam m, 3 Adam v; host memory of train_params(e) floats
int train_copy(pnb_engine *e, int what, void *host, bool to_host, cudaStream_t st) {
  const pnb_train_state &s = *e->train;
  float *flat = what == 1 ? s.grad : what == 2 ? s.m : s.v;
  const cudaMemcpyKind k = to_host ? cudaMemcpyDeviceToHost : cudaMemcpyHostToDevice;
  float *h = static_cast<float *>(host);
  if (what == 0) {
    for (int i = 0; i < kParams; i++) {
      const size_t bytes = (s.off[i + 1] - s.off[i]) * sizeof(float);
      TCK(to_host ? cudaMemcpyAsync(h + s.off[i], s.param[i], bytes, k, st) : cudaMemcpyAsync(s.param[i], h + s.off[i], bytes, k, st));
    }
  } else {
    const size_t bytes = s.off[kParams] * sizeof(float);
    TCK(to_host ? cudaMemcpyAsync(h, flat, bytes, k, st) : cudaMemcpyAsync(flat, h, bytes, k, st));
  }
  return PNB_OK;
}

size_t train_params(const pnb_engine *e) { return e->train ? e->train->off[kParams] : 0; }
