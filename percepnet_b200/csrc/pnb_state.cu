// pnb_state.cu -- batched per-stream state movement: the gather (export) and scatter (import, reset) kernels behind
// pnb_export_states / pnb_import_states / pnb_reset_streams, and the one table that says where a stream's state lives
// in an engine (state_segs, which takes the network path's own pieces from tc_state_segs / f32_state_segs).
// pnb_get_state / pnb_set_state are the n = 1 case of the same kernels.  The session pool
// (pnb_process_sessions_*) parks, unparks and relocates sessions with the same pieces (session_move_kernel) and keeps
// its parking blobs with session_blob_kernel.  The carries that put the state back in place after a call are here
// too: the network paths' end-of-chunk carry of their hop-slot buffers (slot_carry_kernel) and a ragged call's fix-up
// of the pieces that follow the engine's counters (ragged_carry_kernel).
//
// A stream's state is a list of pieces (StateSeg): the history line at line_off, the overlap-add memory, pitch
// continuity, the five live spectrum ring slots, and the network's conv histories and GRU states (fp32, or the tensor
// path's split terms).  One warp moves one piece of one stream with coalesced 32-bit accesses; the blob side is only
// 4-byte aligned (63 804-byte blobs packed back to back), so wider accesses would not be aligned in general.
#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <string.h>

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

// One piece g of one stream: engine side at `eng`, blob at `blob` (null for a reset); `first`: the stream's first piece,
// whose warp writes the blob's header on export.
__device__ __forceinline__ void move_piece(int mode, const StateSeg &g, char *eng, char *blob, bool first, unsigned has_terms,
                                           unsigned lane) {
  const unsigned n = g.n;
  if (mode == kStateExport && first && lane == 0) {
    StreamState *b = reinterpret_cast<StreamState *>(blob);
    b->magic = kStateMagic;
    b->version = kStateVersion;
    b->has_terms = has_terms;
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
  move_piece(mode, g, eng, blob, j == 0, a.has_terms, lane);
}

// The engine-side bytes of piece g, raw, from slot src to slot dst (a session moved between slots): the bf16 term
// planes and fp16 GRU terms as they are, never through the blob's sums.
__device__ __forceinline__ void relocate_piece(const StateSeg &g, char *dst, const char *src, unsigned lane) {
  switch (g.kind) {
    case kSegCopy:
    case kSegEngZero:
      copy_words(reinterpret_cast<unsigned *>(dst), reinterpret_cast<const unsigned *>(src), g.n, lane);
      break;
    case kSegTermBf16:
    case kSegSplitF16:
      for (unsigned k = lane; k < g.n; k += 32)
        reinterpret_cast<unsigned short *>(dst)[k] = reinterpret_cast<const unsigned short *>(src)[k];
      break;
    default:
      break;
  }
}

// The state launch of a session call (pnb_session_plan.h): warp w handles piece (w mod n_seg) of move (w / n_seg).  It
// first parks the slot's occupant (export of the piece to that session's blob), then fills the piece from the entering
// session's blob (import; reset when the blob is marked fresh or rejected), or from the relocation source slot.  Parking
// and filling one piece in one warp, in that order, is what keeps the launch race-free.  The three bf16 term planes of a
// conv history are read by the sum piece as well, so the warp of the sum piece handles the whole group (the sum and its
// three terms, the next three pieces) and the warps of the term pieces do nothing.  With a.blobs set (export of resident
// sessions to the caller's blobs) `park` is the row of the caller's blob and nothing is filled.
__global__ void __launch_bounds__(256) session_move_kernel(const __grid_constant__ StateArgs a) {
  const unsigned lane = threadIdx.x & 31;
  const long long task = (long long)blockIdx.x * kWarpsPerBlock + (threadIdx.x >> 5);
  if (task >= (long long)a.n * a.n_seg) return;
  const int i = (int)(task / a.n_seg), j = (int)(task - (long long)i * a.n_seg);
  if (a.seg[j].kind == kSegTermBf16) return;  // handled with its sum piece
  const int4 mv = reinterpret_cast<const int4 *>(a.moves)[i];
  const int group = a.seg[j].kind == kSegSumBf16 ? 4 : 1;
  const size_t slot = (size_t)mv.x;
  if (mv.y >= 0) {
    char *blob = a.blobs ? a.blobs + (size_t)mv.y * a.blob_stride : a.park + (size_t)mv.y * a.park_stride;
    for (int q = 0; q < group; q++) {
      const StateSeg &g = a.seg[j + q];
      move_piece(kStateExport, g, g.eng + slot * g.eng_stride, blob, j == 0, a.has_terms, lane);
    }
  }
  if (mv.z == kFillBlob) {
    char *blob = a.park + (size_t)mv.w * a.park_stride;
    const StreamState *b = reinterpret_cast<const StreamState *>(blob);
    const int mode = b->magic == kStateMagic && b->version == kStateVersion ? kStateImport : kStateReset;
    for (int q = 0; q < group; q++) {
      const StateSeg &g = a.seg[j + q];
      move_piece(mode, g, g.eng + slot * g.eng_stride, blob, false, a.has_terms, lane);
    }
  } else if (mv.z == kFillSlot) {
    for (int q = 0; q < group; q++) {
      const StateSeg &g = a.seg[j + q];
      relocate_piece(g, g.eng + slot * g.eng_stride, g.eng + (size_t)mv.w * g.eng_stride, lane);
    }
  }
}

// Parking blobs of the listed sessions (a.streams: session ids), one block per session:
//   import  the caller's blob i becomes the session's parking blob when state_check_kernel accepted it; a rejected one
//           marks the parking blob fresh (magic 0), so the session is unparked as a reset stream
//   export  the parking blob is written to the caller's blob a.rows[i] (i when null); a blob marked fresh is written as
//           the blob of a fresh stream (zeros under the header)
//   reset   marks the parking blob fresh
__global__ void __launch_bounds__(256) session_blob_kernel(const __grid_constant__ StateArgs a) {
  const int i = blockIdx.x;
  unsigned *park = reinterpret_cast<unsigned *>(a.park + (size_t)a.streams[i] * a.park_stride);
  constexpr unsigned kWords = sizeof(StreamState) / 4;
  if (a.mode == kStateReset || (a.mode == kStateImport && !a.ok[i])) {
    if (threadIdx.x == 0) park[0] = 0u;
    return;
  }
  const int r = a.rows ? a.rows[i] : i;
  unsigned *user = reinterpret_cast<unsigned *>(a.blobs + (size_t)r * a.blob_stride);
  if (a.mode == kStateImport) {
    for (unsigned k = threadIdx.x; k < kWords; k += blockDim.x) park[k] = user[k];
    return;
  }
  const StreamState *b = reinterpret_cast<const StreamState *>(park);
  const bool fresh = !(b->magic == kStateMagic && b->version == kStateVersion);
  for (unsigned k = threadIdx.x; k < kWords; k += blockDim.x) user[k] = fresh ? 0u : park[k];
  if (fresh && threadIdx.x == 0) {
    StreamState *u = reinterpret_cast<StreamState *>(user);
    u->magic = kStateMagic;
    u->version = kStateVersion;
    u->has_terms = a.has_terms;
  }
}

// g/r of a session call in list order: dst[t][row[p]][:] = src[t][p][:] for the k computed slots (zeros for the hops
// a ragged call's slot did not run)
__global__ void gr_gather_kernel(const float *__restrict__ src, float *__restrict__ dst, const int *__restrict__ row, int k,
                                 int S, int F, const int *__restrict__ hops) {
  const long long total = (long long)F * k * 68;
  for (long long x = (long long)blockIdx.x * blockDim.x + threadIdx.x; x < total; x += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(x % 68);
    const long long tp = x / 68;
    const int p = (int)(tp % k), t = (int)(tp / k);
    dst[((size_t)t * k + row[p]) * 68 + c] = (hops && t >= hops[p]) ? 0.f : src[((size_t)t * S + p) * 68 + c];
  }
}

// The pieces of a slot's state that move with the engine's counters (see state_segs): the history window at line_off
// and the five live spectrum ring slots at hop.
struct RaggedArgs {
  float *pcm;
  size_t pcm_stride, line_off;  // the call's window: line_off + h * 480 after h hops
  float2 *zring;                // [ring][S][400]
  float *ering;                 // [ring][S][34]
  int ring, S, F;
  long hop0;                    // hop counter at the call's start
  const int *hops, *slots;      // [S] hops per slot; [gridDim.x] the slots that stopped early
};

// One block per slot that stopped after h < F hops.  Each piece is read completely before it is written, so the
// overlapping source and destination ranges (F - h < 11 hops of history, F - h < 5 ring slots) need no second buffer:
// the history window goes through registers between two block barriers, and each thread owns one word of every ring
// slot and walks the five slots from the newest down, reading a slot before it writes the one it shadows.
constexpr int kRaggedThreads = 256;
__global__ void __launch_bounds__(kRaggedThreads) ragged_carry_kernel(const __grid_constant__ RaggedArgs a) {
  const int p = a.slots[blockIdx.x], h = a.hops[p], d = a.F - h;
  const unsigned tid = threadIdx.x;
  {
    float *line = a.pcm + (size_t)p * a.pcm_stride + a.line_off;
    constexpr int kPer = (kKeep + kRaggedThreads - 1) / kRaggedThreads;
    float keep[kPer];
#pragma unroll
    for (int i = 0; i < kPer; i++) {
      const int j = tid + kRaggedThreads * i;
      keep[i] = j < kKeep ? line[(size_t)h * kFrame + j] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < kPer; i++) {
      const int j = tid + kRaggedThreads * i;
      if (j < kKeep) line[(size_t)a.F * kFrame + j] = keep[i];
    }
  }
  {
    const int R = a.ring;
    const long base = a.hop0 + h - 5;  // live slot k after h hops: base + k; after F hops: base + d + k
    constexpr unsigned kZ = 2 * kBins;
    for (unsigned w = tid; w < kZ + kBands; w += kRaggedThreads)
      for (int k = 4; k >= 0; k--) {
        const size_t src = (size_t)(((base + k) % R + R) % R), dst = (size_t)(((base + d + k) % R + R) % R);
        if (w < kZ) {
          float *z = reinterpret_cast<float *>(a.zring);
          z[(dst * a.S + p) * kZ + w] = z[(src * a.S + p) * kZ + w];
        } else {
          a.ering[(dst * a.S + p) * kBands + (w - kZ)] = a.ering[(src * a.S + p) * kBands + (w - kZ)];
        }
      }
  }
}

__global__ void __launch_bounds__(256) slot_carry_kernel(const __grid_constant__ SlotCarry a) {
  const size_t tid = (size_t)blockIdx.x * blockDim.x + threadIdx.x, nth = (size_t)gridDim.x * blockDim.x;
  for (int s = 0; s < a.n_seg; s++) {
    const SlotSeg g = a.seg[s];
    for (size_t i = tid; i < g.slot; i += nth) {
      int from = g.from;
      if (a.hops) {
        const int done = min(max(a.hops[i / g.row] - a.h0, 0), a.n);  // hops of this chunk the row ran
        from -= a.n - done;
        if (from < 0 || (from == 0 && g.dst == g.src)) continue;
      }
      const uint4 *src = g.src + (size_t)from * g.stride;
      for (int q = 0; q < g.n_slots; q++) g.dst[(size_t)q * g.stride + i] = src[(size_t)q * g.stride + i];
    }
  }
  for (size_t i = tid; i < (size_t)a.n_cnt; i += nth) a.cnt[i] = 0u;
}

__global__ void state_clear_reject_kernel(int *status) {
  atomicAnd(status, ~kStatusRejected);
  status[1] = kNoRejectedSlot;
}

}  // namespace

int state_segs(const pnb_engine *e, StateSeg *seg) {
  int ns = 0;
  const size_t S = e->S;
  if (e->flags & PNB_NETWORK_ONLY) {  // no signal path: its part of the blob is zero on export and ignored on import
    add_words(seg, ns, kSegBlobZero, nullptr, 0, offsetof(StreamState, pcm),
              (offsetof(StreamState, fc_hist) - offsetof(StreamState, pcm)) / 4);
  } else {
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
  }
  if (e->flags & (PNB_TRAIN_DATA | PNB_SIGNAL_ONLY)) {  // no network: its part of the blob is zero on export, ignored on import
    add_words(seg, ns, kSegBlobZero, nullptr, 0, offsetof(StreamState, fc_hist),
              (offsetof(StreamState, has_terms) - offsetof(StreamState, fc_hist)) / 4);
    add_words(seg, ns, kSegBlobZero, nullptr, 0, offsetof(StreamState, fc_terms), (sizeof(StreamState) - offsetof(StreamState, fc_terms)) / 4);
    return ns;
  }
  // GRU states in fp32 (both paths)
  size_t off = 0;
  for (int li = 0; li < 5; li++) {
    const size_t H = kGruH[li];
    add_words(seg, ns, kSegCopy, e->h[li], H * 4, offsetof(StreamState, h) + off * 4, H);
    off += H;
  }
  add_words(seg, ns, kSegEngZero, e->c2, 512 * 4, 0, 512);  // the conv2 tap (PNB_TAP_NN_C2) of a fresh stream
  return (e->flags & PNB_NN_TENSOR) ? tc_state_segs(e, seg, ns) : f32_state_segs(e, seg, ns);
}

void launch_state_check(const StateArgs &a, cudaStream_t st) {
  state_check_kernel<<<a.n, 256, 0, st>>>(a);
}
void launch_state_move(const StateArgs &a, cudaStream_t st) {
  const long long warps = (long long)a.n * a.n_seg;
  state_move_kernel<<<(unsigned)((warps + kWarpsPerBlock - 1) / kWarpsPerBlock), 32 * kWarpsPerBlock, 0, st>>>(a);
}
void launch_session_move(const StateArgs &a, cudaStream_t st) {
  const long long warps = (long long)a.n * a.n_seg;
  session_move_kernel<<<(unsigned)((warps + kWarpsPerBlock - 1) / kWarpsPerBlock), 32 * kWarpsPerBlock, 0, st>>>(a);
}
void launch_session_blob(const StateArgs &a, cudaStream_t st) {
  session_blob_kernel<<<a.n, 256, 0, st>>>(a);
}
void launch_gr_gather(const float *src, float *dst, const int *row, int k, int S, int F, cudaStream_t st, const int *hops) {
  const long long total = (long long)F * k * 68;
  const long long blocks = (total + 255) / 256;
  gr_gather_kernel<<<(unsigned)(blocks < 4096 ? blocks : 4096), 256, 0, st>>>(src, dst, row, k, S, F, hops);
}

// Beside state_segs: the same places, at the counters of the call's start.
void launch_ragged_carry(const pnb_engine *e, int F, const int *d_hops, const int *d_slots, int n, cudaStream_t st) {
  RaggedArgs a;
  memset(&a, 0, sizeof a);
  a.pcm = e->d_pcm; a.pcm_stride = e->pcm_stride; a.line_off = e->line_off;
  a.zring = e->d_zring; a.ering = e->d_ering; a.ring = e->ring; a.S = e->S; a.F = F; a.hop0 = e->hop;
  a.hops = d_hops; a.slots = d_slots;
  ragged_carry_kernel<<<n, kRaggedThreads, 0, st>>>(a);
}
void launch_slot_carry(const SlotCarry &c, int sm_count, cudaStream_t st) {
  slot_carry_kernel<<<2 * sm_count, 256, 0, st>>>(c);
}
void launch_state_clear_reject(int *status, cudaStream_t st) {
  state_clear_reject_kernel<<<1, 1, 0, st>>>(status);
}

}  // namespace pnb
