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
// The forward and the backward are two halves (forward_half, backward_half) that train_grad runs around its loss.
// pnb_train_forward_device runs the forward half alone on the caller's network input and weights; the backward of the
// caller's loss (pnb_train_backward_device) seeds the output pre-activations from the caller's dL/d(out)
// (train_seed_kernel), runs the backward half, and adds dL/dx = dA_fc W_fc^T when asked.  Its check skips the next
// Adam step on a non-finite gradient but raises no domain bit: the caller owns that loss, as torch's autograd does.
// Both may carry network state (pnb_train_state.h): the forward starts from the caller's state rows and gathers each
// window's state at its end (train_state_kernel), over per-window lengths; the backward takes dL/d(state out) as seeds
// and gives dL/d(state in).
// Between gradient calls and Adam, pnb_train_accumulate / pnb_train_finish sum several calls' gradients (micro-batches,
// or ranks through an exported accumulator) in float64, weighted by their counted hops (train_accum_kernel,
// train_finish_kernel), and the check runs again on the sum.
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
  // backward, each or null: dL/d(state out) of this layer (row b at seed + b * seed_stride), added to dh at each window's
  // last hop; dL/d(state in) (row b at dh0 + b * dh0_stride), one more step after hop 0
  const float *seed;
  size_t seed_stride;
  float *dh0;
  size_t dh0_stride;
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
        else if (a.seed) dh += a.seed[(size_t)b * a.seed_stride + j];  // t = fr - 1: the state the window ends in
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
  if (!a.dh0) return;
  // the state before hop 0: dh0 = dgh(0) U^T + dh(0) z(0), summed as the loop's carry is (hop 0 counts in every window)
  if (tid == 0) chain_wait(a.cnt, (unsigned)a.F * G);
  __syncthreads();
  for (int b = warp; b < n; b += blockDim.x >> 5) {
    float acc[JU];
#pragma unroll
    for (int ju = 0; ju < JU; ju++) acc[ju] = 0.f;
    const float *gp = a.dgh + (size_t)b * H3;
    for (int c = lane; c < H3; c += 32) {
      const float d = __ldcg(gp + c);
#pragma unroll
      for (int ju = 0; ju < JU; ju++) acc[ju] = fmaf(d, Ur[ju * H3 + c], acc[ju]);
    }
#pragma unroll
    for (int ju = 0; ju < JU; ju++)
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) acc[ju] += __shfl_xor_sync(0xffffffffu, acc[ju], o);
#pragma unroll
    for (int ju = 0; ju < JU; ju++)
      if (lane == ju) a.dh0[(size_t)b * a.dh0_stride + j0 + ju] = acc[ju] + a.carry[(size_t)b * H + j0 + ju];
  }
}

// ---------------------------------------------------------------------------------------------------- elementwise
// x [F][n][w]: the hops t >= frames[b] of window b become zeros, so that nothing past a window's end (NaN included)
// reaches any activation the gradient multiplies (w = 70, the network input), or the caller's output rows (w = 68)
__global__ void train_mask_kernel(float *__restrict__ x, int w, const int *__restrict__ frames, int n, int F) {
  const size_t total = (size_t)F * n * w;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const size_t row = i / w;
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

// The backward's entry point when the caller supplies dL/d(out): dout [n][F][68] rows of dout_stride floats (window-major,
// as the caller's tensors) -> d [F][n][68] (hop-major, r = t*n + b), d = dout (1 - p) p left to right, ATen's
// sigmoid_backward, so the seed is the same bits torch's autograd passes into the output layers.  Hops past a window's
// end (frames, or null: none) get zeros whatever dout holds there.
__global__ void train_seed_kernel(const float *__restrict__ dout, size_t dout_stride, const float *__restrict__ pred,
                                  const int *__restrict__ frames, int n, int F, float *__restrict__ d) {
  const size_t total = (size_t)F * n * 68;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int k = (int)(i % 68);
    const size_t row = i / 68;
    const int b = (int)(row % n), t = (int)(row / n);
    if (frames && t >= frames[b]) { d[i] = 0.f; continue; }
    const float p = pred[i];
    d[i] = __fmul_rn(__fmul_rn(dout[(size_t)b * dout_stride + (size_t)t * 68 + k], __fsub_rn(1.f, p)), p);
  }
}

// The network state of a window, PNB_TRAIN_STATE_FLOATS floats: [fc_hist 4 x 128][c1_hist 2 x 512][gru1, gru2, gru3,
// gru_gb 512 each][gru_rb 128], histories oldest first (StreamState's fc_hist, c1_hist, h).  For a window that has run L
// hops, value i of window b is fc slot L + k, c1 slot L + k or GRU slot L of the trainer's buffers: the state in is
// L = 0 (the slots before hop 0), the state out L = the window's hops.
struct StateBufs {
  float *fc, *c1, *h[5];
  int n;
};
__device__ __forceinline__ float *state_slot(const StateBufs &s, int b, int i, int L) {
  const size_t n = s.n;
  if (i < 512) return s.fc + ((L + i / 128) * n + b) * 128 + i % 128;
  if (i < 1536) return s.c1 + ((L + (i - 512) / 512) * n + b) * 512 + (i - 512) % 512;
  const int l = (i - 1536) / 512;
  return s.h[l] + ((size_t)L * n + b) * (l < 4 ? 512 : 128) + (i - 1536) % 512;
}

// out false: the caller's state rows (row b at st + b * stride) into the slots before hop 0; out true: the slots at each
// window's end (frames[b], or null: F) out to the rows
__global__ void train_state_kernel(const StateBufs s, float *st, size_t stride, const int *__restrict__ frames, int F,
                                   bool out) {
  const size_t total = (size_t)s.n * PNB_TRAIN_STATE_FLOATS;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int b = (int)(i / PNB_TRAIN_STATE_FLOATS), k = (int)(i % PNB_TRAIN_STATE_FLOATS);
    float *row = st + (size_t)b * stride + k;
    if (out) *row = *state_slot(s, b, k, frames ? frames[b] : F);
    else *state_slot(s, b, k, 0) = *row;
  }
}

// dL/d(state out) of the conv histories (row b at ds + b * ds_stride), L = frames[b] (or F): fc_hist[k] is the fc
// output of hop L - 4 + k and c1_hist[k] conv1's of hop L - 2 + k, so its seed goes to that hop's row of dfc [F][n][128]
// or dc1 [F][n][512] (zero elsewhere; their contractions add them before the ReLU derivative).  A slot before hop 0
// (L < 4, L < 2) is state in slot L + k passed through, and dsi (dL/d(state in), or null) starts from those seeds:
// every history value of it is written, zero where none passes through.
__global__ void train_hist_seed_kernel(const float *__restrict__ ds, size_t ds_stride, float *__restrict__ dsi,
                                       size_t dsi_stride, const int *__restrict__ frames, int n, int F,
                                       float *__restrict__ dfc, float *__restrict__ dc1) {
  const size_t total = (size_t)n * 1536;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (size_t)gridDim.x * blockDim.x) {
    const int b = (int)(i / 1536), k = (int)(i % 1536), L = frames ? frames[b] : F;
    const bool fc = k < 512;
    const int W = fc ? 128 : 512, D = fc ? 4 : 2, kk = fc ? k : k - 512, slot = kk / W, c = kk % W, t = L - D + slot;
    const float *row = ds + (size_t)b * ds_stride;
    if (t >= 0) (fc ? dfc : dc1)[((size_t)t * n + b) * W + c] = row[k];
    if (dsi) dsi[(size_t)b * dsi_stride + k] = slot >= L ? row[k - L * W] : 0.f;
  }
}

// bad = 1 (and, with a status word, the engine's domain bit) when any of the n gradient values is not finite; bad is
// zeroed before
__global__ void train_check_kernel(const float *__restrict__ g, size_t n, int *bad, int *status) {
  bool found = false;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    found |= !isfinite(g[i]);
  if (__syncthreads_or(found) && threadIdx.x == 0) {
    *bad = 1;
    if (status) atomicOr(status, 1);
  }
}

// Accumulation of several gradient calls (micro-batches, or ranks) before one Adam step, in float64: each call's
// gradient g_k carries 1/c_k (c_k its counted hops), so the batch's is sum c_k g_k / sum c_k.  acc[i] += g[i] * c for
// i < n, acc[n] += c.  g * c is exact in float64 (24-bit mantissa, c < 2^29), so one call finishes to its own bits and
// two add to the same bits in either order.  Four values per thread (n is the model's 7 962 564, a multiple of 4; the
// tail loop covers any other n).
__global__ void train_accum_kernel(const float *__restrict__ g, size_t n, double c, double *__restrict__ acc) {
  const size_t n4 = n / 4, stride = (size_t)gridDim.x * blockDim.x, tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const float4 *g4 = reinterpret_cast<const float4 *>(g);
  double2 *a2 = reinterpret_cast<double2 *>(acc);
  for (size_t i = tid; i < n4; i += stride) {
    const float4 v = __ldg(g4 + i);
    double2 lo = a2[2 * i], hi = a2[2 * i + 1];
    lo.x = __dadd_rn(lo.x, __dmul_rn((double)v.x, c)); lo.y = __dadd_rn(lo.y, __dmul_rn((double)v.y, c));
    hi.x = __dadd_rn(hi.x, __dmul_rn((double)v.z, c)); hi.y = __dadd_rn(hi.y, __dmul_rn((double)v.w, c));
    a2[2 * i] = lo;
    a2[2 * i + 1] = hi;
  }
  for (size_t i = 4 * n4 + tid; i < n; i += stride) acc[i] = __dadd_rn(acc[i], __dmul_rn((double)g[i], c));
  if (tid == 0) acc[n] = __dadd_rn(acc[n], c);
}

// g[i] = (float)(acc[i] / acc[n]) and acc[i] = 0 for i < n; acc[n] is read by every thread, so the caller zeroes it
// after this launch
__global__ void train_finish_kernel(double *__restrict__ acc, size_t n, float *__restrict__ g) {
  const double C = acc[n];
  const size_t n4 = n / 4, stride = (size_t)gridDim.x * blockDim.x, tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  float4 *g4 = reinterpret_cast<float4 *>(g);
  double2 *a2 = reinterpret_cast<double2 *>(acc);
  const double2 zero = make_double2(0.0, 0.0);
  for (size_t i = tid; i < n4; i += stride) {
    const double2 lo = a2[2 * i], hi = a2[2 * i + 1];
    g4[i] = make_float4((float)__ddiv_rn(lo.x, C), (float)__ddiv_rn(lo.y, C), (float)__ddiv_rn(hi.x, C), (float)__ddiv_rn(hi.y, C));
    a2[2 * i] = zero;
    a2[2 * i + 1] = zero;
  }
  for (size_t i = 4 * n4 + tid; i < n; i += stride) {
    g[i] = (float)__ddiv_rn(acc[i], C);
    acc[i] = 0.0;
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
  double *acc = nullptr;                               // [N + 1] accumulated gradients and their hops, on first use
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
  int *lens = nullptr;                     // [S] the last train_forward's hops per window, when it had lengths
  int G512 = 0, G128 = 0;                  // CTAs of the recurrences (a power of two, co-resident)
  int last_F = 0, last_n = 0;              // hops and rows of the last gradient call (0: none yet), for train_tap
  const int *fwd_frames = nullptr;         // the last train_forward's per-window hops (lens), or null: all F
  long long fwd_hops = 0;                  // and the hops they count
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
  TCK(engine_alloc(e, &s.lens, S, kScratch));
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
    {
      LaunchScope m(e, kUnprofiled, st);
      if (tb) train_gemm_kernel<false, true><<<grid, 256, 0, st>>>(g);
      else train_gemm_kernel<false, false><<<grid, 256, 0, st>>>(g);
    }
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
    { LaunchScope m(e, kUnprofiled, st); train_gemm_kernel<true, false><<<grid, 256, 0, st>>>(g); }
    const size_t cnt = (size_t)M * N;
    { LaunchScope m(e, kUnprofiled, st); train_parts_kernel<<<blocks_for(cnt), 256, 0, st>>>(e->train->part, parts, cnt, dst); }
    check();
  }
  template <int JU>
  void rec_launch(const RecArgs &a, int G, bool fwd) {
    LaunchScope m(e, kUnprofiled, st);
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
    check();
  }
};
}  // namespace

// The parameter arrays in blob order: fc W, b (0, 1); conv1 (2, 3); conv2 (4, 5); GRU k = 0..4 (gru1, gru2, gru3,
// gru_gb, gru_rb) W, U, b at 6 + 3k .. 8 + 3k; fc_gb (21, 22); fc_rb (23, 24).
namespace {
// The recurrence arguments of GRU l over the rows t*n + b of an F-hop call: forward into its saved h/z/r/n/hn, backward
// from them into g1 (dgx) and g2 (dgh).
RecArgs rec_args(const pnb_train_state &s, int l, int n, int F, const int *frames) {
  RecArgs a;
  memset(&a, 0, sizeof a);
  a.H = kGruH[l]; a.n = n; a.F = F;
  a.U = s.param[7 + 3 * l]; a.bh = s.param[8 + 3 * l] + 3 * kGruH[l];
  a.gx = s.g1; a.h = s.h[l]; a.z = s.z[l]; a.r = s.r[l]; a.nn = s.nn[l]; a.hn = s.hn[l];
  a.dgx = s.g1; a.dgh = s.g2; a.carry = s.carry; a.frames = frames;
  return a;
}
// GRU l's output at hop t: slot t+1 of its states
float *out_of(const pnb_train_state &s, int l, int n) { return s.h[l] + (size_t)n * kGruH[l]; }
StateBufs state_bufs(const pnb_train_state &s, int n) {
  StateBufs b;
  b.fc = s.fc; b.c1 = s.c1; b.n = n;
  for (int l = 0; l < 5; l++) b.h[l] = s.h[l];
  return b;
}
// where GRU l's state starts in a state row
constexpr size_t state_gru(int l) { return 1536 + 512 * (size_t)l; }
}  // namespace

// The forward half on the network input staged in s.x ([F][n][70]) from the caller's state (state_in, rows of
// state_in_stride floats) or, with state_in null, from zero state: fc, conv1, conv2, the five GRUs with everything their
// backward needs saved, fc_gb and fc_rb into s.pred.  15 launches, 16 with a state in.
static int forward_half(pnb_engine *e, Launcher &L, const int *frames, int F, const float *state_in,
                        size_t state_in_stride) {
  pnb_train_state &s = *e->train;
  const int n = e->n_active, R = F * n;
  const size_t nb = (size_t)n;
  const cudaStream_t st = L.st;
  float *const *P = s.param;
  // per call: the forward counters and the slots before hop 0 (the row stride n changes from call to call)
  TCK(cudaMemsetAsync(s.cnt, 0, 5 * sizeof(unsigned), st));
  if (state_in) {
    LaunchScope m(e, kUnprofiled, st);
    train_state_kernel<<<blocks_for(nb * PNB_TRAIN_STATE_FLOATS), 256, 0, st>>>(
        state_bufs(s, n), const_cast<float *>(state_in), state_in_stride, nullptr, 0, false);
  } else {
    TCK(cudaMemsetAsync(s.fc, 0, 4 * nb * 128 * sizeof(float), st));
    TCK(cudaMemsetAsync(s.c1, 0, 2 * nb * 512 * sizeof(float), st));
    for (int l = 0; l < 5; l++) TCK(cudaMemsetAsync(s.h[l], 0, nb * kGruH[l] * sizeof(float), st));
  }
  L.check();
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
  for (int l = 0; l < 5; l++) {
    const int H = kGruH[l], H3 = 3 * H;
    const float *W = P[6 + 3 * l], *b = P[8 + 3 * l];
    if (l == 0) { TSeg a[1] = {tseg(s.c2, 512, W, H3, 512)}; L.gemm(false, a, 1, R, H3, s.g1, H3, b); }
    else if (l < 4) { TSeg a[1] = {tseg(out_of(s, l - 1, n), 512, W, H3, 512)}; L.gemm(false, a, 1, R, H3, s.g1, H3, b); }
    else {
      TSeg a[2] = {tseg(out_of(s, 2, n), 512, W, H3, 512), tseg(s.c2, 512, W + (size_t)512 * H3, H3, 512)};
      L.gemm(false, a, 2, R, H3, s.g1, H3, b);
    }
    RecArgs a = rec_args(s, l, n, F, frames);
    a.cnt = s.cnt + l;
    L.rec(a, true);
  }
  {
    TSeg a[5] = {tseg(s.c2, 512, P[21], 34, 512)};
    for (int q = 1; q < 5; q++) a[q] = tseg(out_of(s, q - 1, n), 512, P[21] + (size_t)q * 512 * 34, 34, 512);
    L.gemm(false, a, 5, R, 34, s.pred, 68, P[22], kEpiSigmoid);
    TSeg c[1] = {tseg(out_of(s, 4, n), 128, P[23], 34, 128)};
    L.gemm(false, c, 1, R, 34, s.pred + 34, 68, P[24], kEpiSigmoid);
  }
  return PNB_OK;
}

// The backward half of the forward half's call, from the gradient at the output pre-activations in s.dpre: output
// layers, then the GRUs in reverse dependency order, conv2, conv1, fc.  Weight gradients go straight into the flat
// gradient at their blob offsets; fc's pre-activation gradient is left in s.eb.  dstate_out (or null): dL/d(state out)
// rows, which seed the GRUs' last hops and the histories' hops; dstate_in (or null): dL/d(state in) rows, written.
// 98 launches, + 1 with dstate_out (the history seeds), + 6 with dstate_in (the history gradients, one contraction per
// history slot).
static int backward_half(pnb_engine *e, Launcher &L, const int *frames, int F, const float *dstate_out,
                         size_t dstate_out_stride, float *dstate_in, size_t dstate_in_stride) {
  pnb_train_state &s = *e->train;
  const int n = e->n_active, R = F * n;
  const size_t nb = (size_t)n;
  const cudaStream_t st = L.st;
  float *const *P = s.param;
  float *G = s.grad;
  const size_t *O = s.off;
  TCK(cudaMemsetAsync(s.cnt + 5, 0, 5 * sizeof(unsigned), st));
  TCK(cudaMemsetAsync(s.dc2 + (size_t)R * 512, 0, 2 * nb * 512 * sizeof(float), st));
  TCK(cudaMemsetAsync(s.ea + (size_t)R * 512, 0, 4 * nb * 512 * sizeof(float), st));
  const float *fc_out = s.fc + 4 * nb * 128, *c1_out = s.c1 + 2 * nb * 512;
  auto out = [&](int l) { return out_of(s, l, n); };
  const float *dg = s.dpre, *dr = s.dpre + 34;
  // fc_rb
  L.wgrad(out(4), 128, 128, dr, 68, 34, R, G + O[23]);
  L.wgrad(nullptr, 0, 1, dr, 68, 34, R, G + O[24]);
  { TSeg a[1] = {tseg(dr, 68, P[23], 34, 34)}; L.gemm(true, a, 1, R, 128, s.ea, 128); }
  // a GRU's recurrence backwards and its weight gradients; X segments: its inputs
  auto gru_back = [&](int l, const float *ext, const float *X0, const float *X1) {
    const int H = kGruH[l], H3 = 3 * H;
    RecArgs a = rec_args(s, l, n, F, frames);
    a.dh_ext = ext;
    a.cnt = s.cnt + 5 + l;
    if (dstate_out) { a.seed = dstate_out + state_gru(l); a.seed_stride = dstate_out_stride; }
    if (dstate_in) { a.dh0 = dstate_in + state_gru(l); a.dh0_stride = dstate_in_stride; }
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
  gru_back(4, s.ea, out(2), s.c2);
  {
    const float *W = P[18];
    TSeg a[1] = {tseg(s.g1, 384, W, 384, 384)};
    L.gemm(true, a, 1, R, 512, s.eb, 512);                                    // gru3's share
    TSeg c[1] = {tseg(s.g1, 384, W + (size_t)512 * 384, 384, 384)};
    L.gemm(true, c, 1, R, 512, s.dc2, 512);                                   // conv2's share
  }
  // fc_gb
  L.wgrad(s.c2, 512, 512, dg, 68, 34, R, G + O[21]);
  for (int q = 1; q < 5; q++) L.wgrad(out(q - 1), 512, 512, dg, 68, 34, R, G + O[21] + (size_t)q * 512 * 34);
  L.wgrad(nullptr, 0, 1, dg, 68, 34, R, G + O[22]);
  { TSeg a[1] = {fcgb_rows(0)}; L.gemm(true, a, 1, R, 512, s.dc2, 512, nullptr, kEpiNone, true); }
  // gru_gb
  { TSeg a[1] = {fcgb_rows(4)}; L.gemm(true, a, 1, R, 512, s.ea, 512); }
  gru_back(3, s.ea, out(2), nullptr);
  { TSeg a[2] = {tseg(s.g1, 1536, P[15], 1536, 1536), fcgb_rows(3)}; L.gemm(true, a, 2, R, 512, s.eb, 512, nullptr, kEpiNone, true); }
  // gru3, gru2, gru1: each one's input gradient plus fc_gb's share is the layer below's
  gru_back(2, s.eb, out(1), nullptr);
  { TSeg a[2] = {tseg(s.g1, 1536, P[12], 1536, 1536), fcgb_rows(2)}; L.gemm(true, a, 2, R, 512, s.ea, 512); }
  gru_back(1, s.ea, out(0), nullptr);
  { TSeg a[2] = {tseg(s.g1, 1536, P[9], 1536, 1536), fcgb_rows(1)}; L.gemm(true, a, 2, R, 512, s.eb, 512); }
  gru_back(0, s.eb, s.c2, nullptr);
  // conv2: its output gradient through tanh
  { TSeg a[1] = {tseg(s.g1, 1536, P[6], 1536, 1536)}; L.gemm(true, a, 1, R, 512, s.dc2, 512, nullptr, kEpiDTanh, true, s.c2p, 512); }
  for (int q = 0; q < 3; q++) L.wgrad(s.c1 + q * nb * 512, 512, 512, s.dc2, 512, 512, R, G + O[4] + (size_t)q * 512 * 512);
  L.wgrad(nullptr, 0, 1, s.dc2, 512, 512, R, G + O[5]);
  const bool seeded = dstate_out != nullptr;  // the conv1 / fc output gradients below add the history seeds
  if (seeded) {
    TCK(cudaMemsetAsync(s.ea, 0, (size_t)R * 512 * sizeof(float), st));
    TCK(cudaMemsetAsync(s.eb, 0, (size_t)R * 128 * sizeof(float), st));
    LaunchScope m(e, kUnprofiled, st);
    train_hist_seed_kernel<<<blocks_for(nb * 1536), 256, 0, st>>>(dstate_out, dstate_out_stride, dstate_in,
                                                                  dstate_in_stride, frames, n, F, s.eb, s.ea);
  }
  {  // conv1 output gradient: hop t gets tap q of hop t + 2 - q (the trailing zero slots end the sum)
    TSeg a[3];
    for (int q = 0; q < 3; q++) a[q] = tseg(s.dc2 + (2 - q) * nb * 512, 512, P[4] + (size_t)q * 512 * 512, 512, 512);
    L.gemm(true, a, 3, R, 512, s.ea, 512, nullptr, kEpiDRelu, seeded, c1_out, 512);
  }
  for (int q = 0; q < 5; q++) L.wgrad(s.fc + q * nb * 128, 128, 128, s.ea, 512, 512, R, G + O[2] + (size_t)q * 128 * 512);
  L.wgrad(nullptr, 0, 1, s.ea, 512, 512, R, G + O[3]);
  {
    TSeg a[5];
    for (int q = 0; q < 5; q++) a[q] = tseg(s.ea + (4 - q) * nb * 512, 512, P[2] + (size_t)q * 128 * 512, 512, 512);
    L.gemm(true, a, 5, R, 128, s.eb, 128, nullptr, kEpiDRelu, seeded, fc_out, 128);
  }
  if (dstate_in) {  // history slot k (hop k - D) is conv tap q of hop k - q: the input gradients extended before hop 0
    for (int k = 0; k < 2; k++) {
      TSeg a[2];
      for (int q = 0; q <= k; q++) a[q] = tseg(s.dc2 + (k - q) * nb * 512, 512, P[4] + (size_t)q * 512 * 512, 512, 512);
      L.gemm(true, a, k + 1, n, 512, dstate_in + 512 + 512 * k, dstate_in_stride, nullptr, kEpiNone, seeded);
    }
    for (int k = 0; k < 4; k++) {
      TSeg a[4];
      for (int q = 0; q <= k; q++) a[q] = tseg(s.ea + (k - q) * nb * 512, 512, P[2] + (size_t)q * 128 * 512, 512, 512);
      L.gemm(true, a, k + 1, n, 128, dstate_in + 128 * k, dstate_in_stride, nullptr, kEpiNone, seeded);
    }
  }
  L.wgrad(s.x, kFeat, kFeat, s.eb, 128, 128, R, G + O[0]);
  L.wgrad(nullptr, 0, 1, s.eb, 128, 128, R, G + O[1]);
  return PNB_OK;
}

// The check of the held gradient: s.bad zeroed, then raised (and the domain bit in status, unless null) by a
// non-finite value.  1 launch.
static int check_grad(pnb_engine *e, Launcher &L, int *status) {
  const pnb_train_state &s = *e->train;
  const size_t N = s.off[kParams];
  TCK(cudaMemsetAsync(s.bad, 0, sizeof(int), L.st));
  { LaunchScope m(e, kUnprofiled, L.st); train_check_kernel<<<blocks_for(N, 1024), 256, 0, L.st>>>(s.grad, N, s.bad, status); }
  L.check();
  return PNB_OK;
}

int train_grad(pnb_engine *e, const float *rec, size_t rec_stride, const int *frames, const int *h_frames, double *sums,
               int F, cudaStream_t st) {
  pnb_train_state &s = *e->train;
  const int n = e->n_active, R = F * n;
  const long long launches0 = e->launches;
  Launcher L{e, st};
  // ---- stage: {30 rec[0..67], rec[68], rec[69]}, zero past each window's end
  { LaunchScope m(e, kUnprofiled, st); launch_rows_stage(s.x, kFeat, rec, rec_stride, PNB_RECORD_FLOATS, 68, n, n, F, st); }
  { LaunchScope m(e, kUnprofiled, st); train_mask_kernel<<<blocks_for((size_t)R * kFeat), 256, 0, st>>>(s.x, kFeat, frames, n, F); }
  L.check();
  if (int rc = forward_half(e, L, frames, F, nullptr, 0)) return rc;

  // ---- loss and its gradient at the output pre-activations
  { LaunchScope m(e, kUnprofiled, st); launch_loss_sums(s.pred, rec, rec_stride, frames, sums, n, n, F, st); }
  long long counted = 0;
  for (int i = 0; i < n; i++) counted += h_frames ? h_frames[i] : F;
  {
    LaunchScope m(e, kUnprofiled, st);
    train_dpre_kernel<<<blocks_for((size_t)R * 68), 256, 0, st>>>(s.pred, rec, rec_stride, frames, n, F,
                                                                  1.0 / ((double)counted * kBands), s.dpre);
  }
  L.check();

  if (int rc = backward_half(e, L, frames, F, nullptr, 0, nullptr, 0)) return rc;
  if (int rc = check_grad(e, L, e->d_status)) return rc;
  TCK(L.err);
  // pnb_launches_per_call reports train_grad_launches: the schedule above and that count must agree
  if (e->launches - launches0 != train_grad_launches(e))
    return engine_fail(PNB_ERR_CUDA, "train_grad issued a launch count train_grad_launches does not know");
  e->train_hops = counted;
  s.last_F = F;
  s.last_n = n;
  return PNB_OK;
}

// A forward of the caller's network input (70 features per hop, not scaled) on windows [0, n_active), each from the
// caller's state rows (state_in) or from zero state; weights (or null) first replace the parameters, and the predictions
// go to the caller's rows.  lengths (device, with h_lengths its host copy; or null): the hops of each window, whose
// later input is zeroed and whose later output rows are zeros; the state at each window's end goes to state_out (or
// nowhere).
int train_forward(pnb_engine *e, const float *x, size_t x_stride, const float *weights, const float *state_in,
                  size_t state_in_stride, const int *lengths, const int *h_lengths, float *out, size_t out_stride,
                  float *state_out, size_t state_out_stride, int F, cudaStream_t st) {
  pnb_train_state &s = *e->train;
  const int n = e->n_active, R = F * n;
  const long long launches0 = e->launches;
  Launcher L{e, st};
  if (weights)
    for (int i = 0; i < kParams; i++)
      TCK(cudaMemcpyAsync(s.param[i], weights + s.off[i], (s.off[i + 1] - s.off[i]) * sizeof(float),
                          cudaMemcpyDeviceToDevice, st));
  { LaunchScope m(e, kUnprofiled, st); launch_rows_stage(s.x, kFeat, x, x_stride, kFeat, 0, n, n, F, st); }
  const int *frames = nullptr;  // kept on the trainer for the backward: the staging lengths came through is reused
  if (lengths) {
    TCK(cudaMemcpyAsync(s.lens, lengths, (size_t)n * sizeof(int), cudaMemcpyDeviceToDevice, st));
    frames = s.lens;
    LaunchScope m(e, kUnprofiled, st);
    train_mask_kernel<<<blocks_for((size_t)R * kFeat), 256, 0, st>>>(s.x, kFeat, frames, n, F);
  }
  L.check();
  if (int rc = forward_half(e, L, frames, F, state_in, state_in_stride)) return rc;
  if (frames) {
    LaunchScope m(e, kUnprofiled, st);
    train_mask_kernel<<<blocks_for((size_t)R * 68), 256, 0, st>>>(s.pred, 68, frames, n, F);
  }
  { LaunchScope m(e, kUnprofiled, st); launch_rows_store(s.pred, 68, out, out_stride, n, n, F, st); }
  if (state_out) {
    LaunchScope m(e, kUnprofiled, st);
    train_state_kernel<<<blocks_for((size_t)n * PNB_TRAIN_STATE_FLOATS), 256, 0, st>>>(state_bufs(s, n), state_out,
                                                                                       state_out_stride, frames, F, true);
  }
  L.check();
  TCK(L.err);
  if (e->launches - launches0 != train_forward_launches(e, state_in, lengths, state_out))
    return engine_fail(PNB_ERR_CUDA, "train_forward issued a launch count train_forward_launches does not know");
  s.last_F = F;
  s.last_n = n;
  s.fwd_frames = frames;
  s.fwd_hops = (long long)n * F;
  if (h_lengths) {
    s.fwd_hops = 0;
    for (int i = 0; i < n; i++) s.fwd_hops += h_lengths[i];
  }
  return PNB_OK;
}

// The backward of the last train_forward from the caller's gradient at its output (and at its state out, when not null):
// the seed, the backward half, and the input and state-in gradients when asked for; the gradient becomes the held one
// (its check skips the next Adam step, but raises no domain bit: the caller owns the loss) and, when asked for, is
// copied out in blob order.
int train_backward(pnb_engine *e, const float *dout, size_t dout_stride, const float *dstate_out,
                   size_t dstate_out_stride, float *dx, size_t dx_stride, float *dstate_in, size_t dstate_in_stride,
                   float *grad, cudaStream_t st) {
  pnb_train_state &s = *e->train;
  const int n = s.last_n, F = s.last_F, R = F * n;
  const long long launches0 = e->launches;
  Launcher L{e, st};
  {
    LaunchScope m(e, kUnprofiled, st);
    train_seed_kernel<<<blocks_for((size_t)R * 68), 256, 0, st>>>(dout, dout_stride, s.pred, s.fwd_frames, n, F, s.dpre);
  }
  L.check();
  if (int rc = backward_half(e, L, s.fwd_frames, F, dstate_out, dstate_out_stride, dstate_in, dstate_in_stride)) return rc;
  if (dx) {  // dL/dx = dA_fc W_fc^T, then out to the caller's rows
    TSeg a[1] = {tseg(s.eb, 128, s.param[0], 128, 128)};
    L.gemm(true, a, 1, R, kFeat, s.g1, kFeat);
    { LaunchScope m(e, kUnprofiled, st); launch_rows_store(s.g1, kFeat, dx, dx_stride, n, n, F, st); }
    L.check();
  }
  if (int rc = check_grad(e, L, nullptr)) return rc;
  if (grad) TCK(cudaMemcpyAsync(grad, s.grad, s.off[kParams] * sizeof(float), cudaMemcpyDeviceToDevice, st));
  TCK(L.err);
  if (e->launches - launches0 != train_backward_launches(e, dx, dstate_out, dstate_in))
    return engine_fail(PNB_ERR_CUDA, "train_backward issued a launch count train_backward_launches does not know");
  e->train_hops = s.fwd_hops;
  return PNB_OK;
}

int train_tap(const pnb_engine *e, int what, const void **src, size_t *bytes) {
  if (!e->train) return engine_fail(PNB_ERR_ARG, "the PNB_TAP_TRAIN_* taps need a PNB_TRAIN_NETWORK engine");
  const pnb_train_state &s = *e->train;
  if (!s.last_F)
    return engine_fail(PNB_ERR_ARG, "the PNB_TAP_TRAIN_* taps need a pnb_train_grad_* or pnb_train_forward_device call first");
  const size_t nb = (size_t)s.last_n, rows = (size_t)s.last_F * nb;
  switch (what) {
    case PNB_TAP_TRAIN_FC: *src = s.fc + 4 * nb * 128; *bytes = rows * 128 * sizeof(float); break;
    case PNB_TAP_TRAIN_C1: *src = s.c1 + 2 * nb * 512; *bytes = rows * 512 * sizeof(float); break;
    case PNB_TAP_TRAIN_DPRE: *src = s.dpre; *bytes = rows * 68 * sizeof(float); break;
    default: *src = s.c2p; *bytes = rows * 512 * sizeof(float); break;
  }
  return PNB_OK;
}

// The launches of train_grad, which does not depend on the shape of the call: stage 2; forward 3 + 5 x 2 + 2; loss 2;
// backward 99 (fc_rb 5, gru_rb 11 + 2, fc_gb 13, gru_gb 1 + 9 + 1, gru3 and gru2 9 + 1 each, gru1 9, conv2 9, conv1 13,
// fc 5, check 1).
int train_grad_launches(const pnb_engine *) { return 118; }
// train_forward: stage 1, forward 15, store 1; a state in 1 (its scatter), lengths 2 (the masks of the input and the
// output), a state out 1 (its gather).  train_backward: seed 1, backward 98, check 1, and with the input gradient its
// contraction and store 2; a state-out gradient 1 (the history seeds), a state-in gradient 6 (the history contractions).
int train_forward_launches(const pnb_engine *, bool state_in, bool lengths, bool state_out) {
  return 17 + (state_in ? 1 : 0) + (lengths ? 2 : 0) + (state_out ? 1 : 0);
}
int train_backward_launches(const pnb_engine *, bool dx, bool dstate_out, bool dstate_in) {
  return (dx ? 102 : 100) + (dstate_out ? 1 : 0) + (dstate_in ? 6 : 0);
}

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
  { LaunchScope m(e, kUnprofiled, st); train_adam_kernel<<<dim3(64, kParams), 256, 0, st>>>(a); }
  TCK(cudaGetLastError());
  return PNB_OK;
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

// The accumulator, allocated (zeroed, and zeroed again by pnb_reset) the first time an accumulation, export or import
// needs it: engines that never accumulate do not carry its 64 MB.  engine_alloc's zeroing runs on the legacy stream,
// so the device is synchronised once before any stream of the engine's may touch the buffer.
int train_accum_prepare(pnb_engine *e) {
  pnb_train_state &s = *e->train;
  if (s.acc) return PNB_OK;
  TCK(engine_alloc(e, &s.acc, s.off[kParams] + 1, kStreamState));
  TCK(cudaDeviceSynchronize());
  return PNB_OK;
}

int train_accumulate(pnb_engine *e, cudaStream_t st) {
  const pnb_train_state &s = *e->train;
  const size_t N = s.off[kParams];
  { LaunchScope m(e, kUnprofiled, st); train_accum_kernel<<<blocks_for(N / 4), 256, 0, st>>>(s.grad, N, (double)e->train_hops, s.acc); }
  TCK(cudaGetLastError());
  return PNB_OK;
}

int train_finish(pnb_engine *e, cudaStream_t st) {
  const pnb_train_state &s = *e->train;
  const size_t N = s.off[kParams];
  { LaunchScope m(e, kUnprofiled, st); train_finish_kernel<<<blocks_for(N / 4), 256, 0, st>>>(s.acc, N, s.grad); }
  TCK(cudaMemsetAsync(s.acc + N, 0, sizeof(double), st));
  TCK(cudaMemsetAsync(s.bad, 0, sizeof(int), st));
  { LaunchScope m(e, kUnprofiled, st); train_check_kernel<<<blocks_for(N, 1024), 256, 0, st>>>(s.grad, N, s.bad, e->d_status); }
  TCK(cudaGetLastError());
  return PNB_OK;
}

// The accumulator's N + 1 doubles to or from mem, host memory or device memory of the engine's device, on st
int train_accum_copy(pnb_engine *e, void *mem, bool out, cudaStream_t st) {
  const pnb_train_state &s = *e->train;
  const size_t bytes = (s.off[kParams] + 1) * sizeof(double);
  TCK(out ? cudaMemcpyAsync(mem, s.acc, bytes, cudaMemcpyDefault, st) : cudaMemcpyAsync(s.acc, mem, bytes, cudaMemcpyDefault, st));
  return PNB_OK;
}
