// pnb_state.cu -- batched per-stream state movement: the gather (export) and scatter (import, reset) kernels behind
// pnb_export_states / pnb_import_states / pnb_reset_streams, and the one table that says where a stream's state lives
// in an engine (state_segs).  pnb_get_state / pnb_set_state are the n = 1 case of the same kernels.
//
// A stream's state is a list of pieces (StateSeg): the history line at line_off, the overlap-add memory, pitch
// continuity, the five live spectrum ring slots, and the network's conv histories and GRU states (fp32, or the tensor
// path's split terms).  One warp moves one piece of one stream with coalesced 32-bit accesses; the blob side is only
// 4-byte aligned (63 804-byte blobs packed back to back), so wider accesses would not be aligned in general.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>

#include "pnb_engine.h"
#include "pnb_state.h"

namespace pnb {
namespace {

constexpr int kWarpsPerBlock = 8;

__device__ __forceinline__ void copy_words(unsigned *__restrict__ d, const unsigned *__restrict__ s, unsigned n, unsigned lane) {
  unsigned k = lane;
  for (; k + 96 < n; k += 128) {  // four loads in flight per lane before the stores
    const unsigned v0 = s[k], v1 = s[k + 32], v2 = s[k + 64], v3 = s[k + 96];
    d[k] = v0; d[k + 32] = v1; d[k + 64] = v2; d[k + 96] = v3;
  }
  for (; k < n; k += 32) d[k] = s[k];
}
__device__ __forceinline__ void zero_words(unsigned *d, unsigned n, unsigned lane) {
  for (unsigned k = lane; k < n; k += 32) d[k] = 0u;
}

// One block per blob: magic / version and, for tensor-mode engines, the GRU bound pnb_set_state enforces.  A rejected
// blob is imported as a reset stream; the engine's status word records the rejection and the lowest rejected slot.
__global__ void __launch_bounds__(256) state_check_kernel(const __grid_constant__ StateArgs a) {
  const int i = blockIdx.x;
  const StreamState *b = reinterpret_cast<const StreamState *>(a.blobs + (size_t)i * a.blob_stride);
  bool ok = b->magic == kStateMagic && b->version == kStateVersion;
  if (a.check_gru)
    for (int k = threadIdx.x; k < 4 * 512 + 128; k += blockDim.x) ok = ok && fabsf(b->h[k]) <= kStateGruBound;  // NaN fails
  ok = __syncthreads_and(ok) != 0;
  if (threadIdx.x == 0) {
    a.ok[i] = ok ? 1 : 0;
    if (!ok) {
      atomicOr(a.status, kStatusRejected);
      atomicMin(a.status + 1, a.streams[i]);
    }
  }
}

// Warp w of the grid moves piece (w mod n_seg) of stream (w / n_seg).
__global__ void __launch_bounds__(256) state_move_kernel(const __grid_constant__ StateArgs a) {
  const unsigned lane = threadIdx.x & 31;
  const long long task = (long long)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  if (task >= (long long)a.n * a.n_seg) return;
  const int i = (int)(task / a.n_seg), j = (int)(task - (long long)i * a.n_seg);
  const StateSeg &g = a.seg[j];
  char *eng = g.eng + (size_t)a.streams[i] * g.eng_stride;
  char *blob = a.blobs ? a.blobs + (size_t)i * a.blob_stride : nullptr;
  int mode = a.mode;
  if (mode == kStateImport && !a.ok[i]) mode = kStateReset;  // a rejected blob leaves its stream fresh
  const unsigned n = g.n;
  if (mode == kStateExport && j == 0 && lane == 0) {
    StreamState *b = reinterpret_cast<StreamState *>(blob);
    b->magic = kStateMagic;
    b->version = kStateVersion;
    b->has_terms = a.has_terms;
  }
  switch (g.kind) {
    case kSegCopy: {
      unsigned *e32 = reinterpret_cast<unsigned *>(eng);
      if (mode == kStateExport) copy_words(reinterpret_cast<unsigned *>(blob + g.blob_off), e32, n, lane);
      else if (mode == kStateImport) copy_words(e32, reinterpret_cast<const unsigned *>(blob + g.blob_off), n, lane);
      else zero_words(e32, n, lane);
      break;
    }
    case kSegBlobZero:
      if (mode == kStateExport) zero_words(reinterpret_cast<unsigned *>(blob + g.blob_off), n, lane);
      break;
    case kSegEngZero:
      if (mode == kStateReset) zero_words(reinterpret_cast<unsigned *>(eng), n, lane);
      break;
    case kSegSumBf16:
      if (mode == kStateExport) {
        float *dst = reinterpret_cast<float *>(blob + g.blob_off);
        for (unsigned k = lane; k < n; k += 32) {
          float s = 0.f;
          for (int tm = 2; tm >= 0; tm--)  // smallest term first: the fp32 sum is then exact up to its last bit
            s = __fadd_rn(s, __bfloat162float(reinterpret_cast<const __nv_bfloat16 *>(eng + tm * g.plane)[k]));
          dst[k] = s;
        }
      }
      break;
    case kSegTermBf16: {
      __nv_bfloat16 *e16 = reinterpret_cast<__nv_bfloat16 *>(eng);
      unsigned short *b16 = reinterpret_cast<unsigned short *>(blob + g.blob_off);
      if (mode == kStateExport) {
        for (unsigned k = lane; k < n; k += 32) b16[k] = __bfloat16_as_ushort(e16[k]);
      } else if (mode == kStateImport) {
        if (reinterpret_cast<const StreamState *>(blob)->has_terms) {
          for (unsigned k = lane; k < n; k += 32) e16[k] = __ushort_as_bfloat16(b16[k]);
        } else {  // split the fp32 history: term t is the rounding of what terms 0..t-1 left over
          const float *src = reinterpret_cast<const float *>(blob + g.aux_off);
          for (unsigned k = lane; k < n; k += 32) {
            float r = src[k];
            __nv_bfloat16 t = __float2bfloat16_rn(r);
            for (int q = 0; q < g.term; q++) {
              r = __fsub_rn(r, __bfloat162float(t));
              t = __float2bfloat16_rn(r);
            }
            e16[k] = t;
          }
        }
      } else {
        for (unsigned k = lane; k < n; k += 32) e16[k] = __ushort_as_bfloat16((unsigned short)0);
      }
      break;
    }
    case kSegSplitF16: {
      __half *e16 = reinterpret_cast<__half *>(eng);
      if (mode == kStateImport) {
        const float *src = reinterpret_cast<const float *>(blob + g.blob_off);
        for (unsigned k = lane; k < n; k += 32) {
          const float sv = __fmul_rn(src[k], g.scale);
          const __half hi = __float2half_rn(sv);
          e16[k] = g.term == 0 ? hi : __float2half_rn(__fsub_rn(sv, __half2float(hi)));
        }
      } else if (mode == kStateReset) {
        for (unsigned k = lane; k < n; k += 32) e16[k] = __ushort_as_half((unsigned short)0);
      }
      break;
    }
  }
}

__global__ void state_clear_reject_kernel(int *status) {
  atomicAnd(status, ~kStatusRejected);
  status[1] = kNoRejectedSlot;
}

// n 32-bit words of one field, cut into pieces of at most kStateSegMax words
void add_words(StateSeg *seg, int &ns, short kind, void *eng, size_t eng_stride, size_t blob_off, size_t n) {
  for (size_t k = 0; k < n; k += kStateSegMax) {
    StateSeg &g = seg[ns++];
    g = StateSeg();
    g.kind = kind;
    g.eng = eng ? static_cast<char *>(eng) + 4 * k : nullptr;
    g.eng_stride = eng_stride;
    g.blob_off = (unsigned)(blob_off + 4 * k);
    g.n = (unsigned)(n - k < (size_t)kStateSegMax ? n - k : (size_t)kStateSegMax);
  }
}

}  // namespace

int state_segs(const pnb_engine *e, StateSeg *seg) {
  int ns = 0;
  const size_t S = e->S;
  // signal state: the history line at line_off, overlap-add memory, pitch continuity, the five live spectrum slots
  add_words(seg, ns, kSegCopy, e->d_pcm + e->line_off, e->pcm_stride * 4, offsetof(StreamState, pcm), kKeep);
  add_words(seg, ns, kSegCopy, e->d_synth, kFrame * 4, offsetof(StreamState, synth), kFrame);
  add_words(seg, ns, kSegCopy, e->d_last_period, 4, offsetof(StreamState, last_period), 1);
  add_words(seg, ns, kSegCopy, e->d_last_gain, 4, offsetof(StreamState, last_gain), 1);
  for (int k = 0; k < 5; k++) {
    const long c = e->hop - 5 + k;
    const size_t slot = (size_t)((c % e->ring + e->ring) % e->ring);
    add_words(seg, ns, kSegCopy, e->d_zring + slot * S * kBins, kBins * 8, offsetof(StreamState, spec) + (size_t)k * kBins * 8, 2 * kBins);
    add_words(seg, ns, kSegCopy, e->d_ering + slot * S * kBands, kBands * 4, offsetof(StreamState, eband) + (size_t)k * kBands * 4, kBands);
  }
  if (e->flags & PNB_TRAIN_DATA) {  // no network: its part of the blob is zero
    add_words(seg, ns, kSegBlobZero, nullptr, 0, offsetof(StreamState, fc_hist),
              (offsetof(StreamState, has_terms) - offsetof(StreamState, fc_hist)) / 4);
    add_words(seg, ns, kSegBlobZero, nullptr, 0, offsetof(StreamState, fc_terms), (sizeof(StreamState) - offsetof(StreamState, fc_terms)) / 4);
    return ns;
  }
  // GRU states in fp32 (both paths), at the parity the next call starts from
  size_t off = 0;
  for (int li = 0; li < 5; li++) {
    const size_t H = e->gru[li].H;
    add_words(seg, ns, kSegCopy, e->h[li][e->par[li]], H * 4, offsetof(StreamState, h) + off * 4, H);
    off += H;
  }
  add_words(seg, ns, kSegEngZero, e->c2, 512 * 4, 0, 512);  // the conv2 tap (PNB_TAP_NN_C2) of a fresh stream
  if (e->flags & PNB_NN_TENSOR) return tc_state_segs(e, seg, ns);
  // fp32 path: the conv histories at slots 0..3 / 0..1 of the hop-slot buffers (nn_chunk_f32's carry)
  for (int k = 0; k < 4; k++)
    add_words(seg, ns, kSegCopy, e->ring_fc + (size_t)k * S * 128, 128 * 4, offsetof(StreamState, fc_hist) + (size_t)k * 128 * 4, 128);
  for (int k = 0; k < 2; k++)
    add_words(seg, ns, kSegCopy, e->ring_c1 + (size_t)k * S * 512, 512 * 4, offsetof(StreamState, c1_hist) + (size_t)k * 512 * 4, 512);
  add_words(seg, ns, kSegBlobZero, nullptr, 0, offsetof(StreamState, fc_terms), (sizeof(StreamState) - offsetof(StreamState, fc_terms)) / 4);
  return ns;
}

int launch_state_check(const StateArgs &a, cudaStream_t st) {
  state_check_kernel<<<a.n, 256, 0, st>>>(a);
  return 1;
}
int launch_state_move(const StateArgs &a, cudaStream_t st) {
  const long long warps = (long long)a.n * a.n_seg;
  state_move_kernel<<<(unsigned)((warps + kWarpsPerBlock - 1) / kWarpsPerBlock), 32 * kWarpsPerBlock, 0, st>>>(a);
  return 1;
}
int launch_state_clear_reject(int *status, cudaStream_t st) {
  state_clear_reject_kernel<<<1, 1, 0, st>>>(status);
  return 1;
}

}  // namespace pnb
