// pnb_state.h -- the per-stream state blob (pnb_get_state / pnb_export_states) and the descriptors of the kernels that
// gather it from and scatter it into an engine (pnb_state.cu).  Host and device code share this layout.
#pragma once
#include <stddef.h>
#include "pnb_common.cuh"

struct pnb_engine;

namespace pnb {

// The live part of the reference's DenoiseState + RNNState (src/denoise.cpp:71-85, src/nnet_data.h:28-38; SURVEY.md
// App. A.2).  A stream moved between engines at a call boundary continues exactly from these bytes.
struct StreamState {
  unsigned magic, version;
  float pcm[kKeep];          // the last 5280 input samples (comb_buf without its newest hop)
  float synth[kFrame];       // overlap-add memory
  int last_period;
  float last_gain;
  float spec[5][2 * kBins];  // spectra of the last five windowed blocks (analysis spectrum of the next five hops), oldest first
  float eband[5][kBands];    // their band energies
  float fc_hist[4][128];     // conv1 input history (last four fc outputs), oldest first
  float c1_hist[2][512];     // conv2 input history (last two conv1 outputs)
  float h[4 * 512 + 128];    // gru1, gru2, gru3, gru_gb, gru_rb
  // tensor-mode engines keep the conv histories as three bf16 terms; the sum above does not always split back into the
  // same terms (a low term of exactly half an ulp), so the raw terms travel too and a tensor-mode engine restores those
  unsigned has_terms;
  unsigned short fc_terms[3][4][128];
  unsigned short c1_terms[3][2][512];
};
constexpr unsigned kStateMagic = 0x53424E50u;  // "PNBS"
constexpr unsigned kStateVersion = 1;
constexpr float kStateGruBound = 1.0001f;      // |GRU state| a tensor-mode engine accepts (tanh outputs and their mixes)

// The blob is a wire format: its size and every offset are fixed.
static_assert(sizeof(StreamState) == 63804, "StreamState is a wire format");
static_assert(offsetof(StreamState, pcm) == 8 && offsetof(StreamState, synth) == 21128 &&
              offsetof(StreamState, last_period) == 23048 && offsetof(StreamState, last_gain) == 23052 &&
              offsetof(StreamState, spec) == 23056 && offsetof(StreamState, eband) == 39056 &&
              offsetof(StreamState, fc_hist) == 39736 && offsetof(StreamState, c1_hist) == 41784 &&
              offsetof(StreamState, h) == 45880 && offsetof(StreamState, has_terms) == 54584 &&
              offsetof(StreamState, fc_terms) == 54588 && offsetof(StreamState, c1_terms) == 57660,
              "StreamState field offsets are part of the wire format");

// One piece of a stream's state: where it sits in the engine (stream s at eng + s * eng_stride) and in the blob.
// The kinds say how each direction treats it:
//   kSegCopy      n 32-bit words, engine <-> blob; reset zeroes the engine side
//   kSegBlobZero  n words of the blob written as zero on export (parts the engine does not carry)
//   kSegEngZero   n words of the engine zeroed on reset (engine-side taps that are not part of the blob)
//   kSegSumBf16   export: n fp32 values = the sum of the three bf16 term planes (`plane` bytes apart), smallest first
//   kSegTermBf16  term `term` of n bf16 values: export copies it to the blob, import restores it from the blob's raw
//                 terms or, for a blob without them (has_terms == 0), splits it from the fp32 values at aux_off
//   kSegSplitF16  import: term `term` (0 hi, 1 lo) of the fp16 split of n fp32 values x kActScale; reset zeroes it
enum StateSegKind : short { kSegCopy = 0, kSegBlobZero, kSegEngZero, kSegSumBf16, kSegTermBf16, kSegSplitF16 };
struct StateSeg {
  char *eng;
  size_t eng_stride;
  size_t plane;
  unsigned blob_off, aux_off;
  unsigned n;
  float scale;           // kSegSplitF16: the fp16 activation scale
  short kind, term;
};
constexpr int kMaxStateSegs = 72;  // a tensor-mode engine needs 69
constexpr int kStateSegMax = 512;  // words / elements per piece: long fields are cut into pieces of at most this

// Appends the pieces of n 32-bit words of one field, cut into pieces of at most kStateSegMax words
inline void add_words(StateSeg *seg, int &ns, short kind, void *eng, size_t eng_stride, size_t blob_off, size_t n) {
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

enum StateMode { kStateExport = 0, kStateImport = 1, kStateReset = 2 };
struct StateArgs {
  StateSeg seg[kMaxStateSegs];
  int n_seg;
  int n;                 // streams in the batch
  const int *streams;    // [n] engine slots
  char *blobs;           // blob i at blobs + i * blob_stride (export: written, import: read, reset: null)
  size_t blob_stride;
  int *ok;               // [n] import: the verdict of state_check_kernel per blob
  int mode;
  unsigned has_terms;    // export: the blob's has_terms
  // import checks
  int check_gru;         // tensor-mode engines refuse GRU states outside kStateGruBound
  int *status;           // the engine's status word [2]: bit 1 of [0] = a blob was rejected, [1] = lowest rejected slot
  // session pool (session_move_kernel / session_blob_kernel): streams are then session ids
  const int *moves;      // [n][4] SessionMove (pnb_session_plan.h)
  const int *rows;       // session_blob_kernel export: caller's blob of entry i (null = i)
  char *park;            // parking blob of session s at park + s * park_stride
  size_t park_stride;
};

// Status bit raised when an import rejected a blob (reported once as PNB_ERR_ARG by the synchronising entry points).
constexpr int kStatusRejected = 2;
constexpr int kNoRejectedSlot = 0x7F7F7F7F;  // status[1] when nothing was rejected (a byte-wise memset can write it)

// The pieces of a stream's state in engine e at its current hop / line offset (host counters committed when a call is
// enqueued, so the list is right in stream order); returns their number (<= kMaxStateSegs).
int state_segs(const pnb_engine *e, StateSeg *seg);
void launch_state_check(const StateArgs &a, cudaStream_t st);
void launch_state_move(const StateArgs &a, cudaStream_t st);
void launch_state_clear_reject(int *status, cudaStream_t st);
// session pool: the state launch of a call (a.n moves), the parking-blob operations (a.n sessions), and the g/r of a
// call in list order ([F][k][68] from the engine's [F][S][68])
void launch_session_move(const StateArgs &a, cudaStream_t st);
void launch_session_blob(const StateArgs &a, cudaStream_t st);
// hops: [k] hops of each slot in a ragged call (entries t >= hops[p] are written as zeros), or null
void launch_gr_gather(const float *src, float *dst, const int *row, int k, int S, int F, cudaStream_t st,
                      const int *hops = nullptr);
// The fix-up of a ragged session call (pnb_process_sessions_ragged_*), enqueued after synthesis and before the history
// slide, with the engine's hop counter and line offset still those of the call's start.  The n slots at d_slots stopped
// after hops[p] < F hops; the pieces of their state that sit where the counters say (state_segs) move from where hop
// hops[p] left them to where hop F would have put them.  One launch.
void launch_ragged_carry(const pnb_engine *e, int F, const int *d_hops, const int *d_slots, int n, cudaStream_t st);

// The carry at the end of a network chunk of n hops (hops [h0, h0 + n) of the call), both network paths: the hop slots
// the next chunk reads first move to the front of their buffers, and the chain's counters return to zero.  Segment g
// moves the first `slot` 16-byte words of n_slots slots, `stride` words apart, from slots from.. of src to slots 0.. of
// dst.  In a ragged call a row (`row` words) that stopped after hop hops[row] takes its slots from
// from - (n - clamp(hops[row] - h0, 0, n)) on instead, and nothing moves when that is below 0 or the row is already in
// place.  A thread owns the same word of every slot and walks the slots upwards, so a slot that is both source and
// destination is read before it is overwritten.
struct SlotSeg { uint4 *dst; const uint4 *src; size_t slot, stride, row; int n_slots, from; };
struct SlotCarry {
  SlotSeg seg[16];
  int n_seg;
  const int *hops;  // [active streams] hops of each row in a ragged call, or null
  int h0, n;
  unsigned *cnt;    // [n_cnt] counters to zero
  int n_cnt;
};
// Appends the segment of the first n_rows rows (row_bytes each, a multiple of 16) of n_slots slots of S rows
inline void add_carry_seg(SlotCarry &c, void *dst, const void *src, size_t row_bytes, int n_rows, int S, int n_slots, int from) {
  c.seg[c.n_seg++] = SlotSeg{static_cast<uint4 *>(dst), static_cast<const uint4 *>(src), n_rows * row_bytes / 16,
                             S * row_bytes / 16, row_bytes / 16, n_slots, from};
}
void launch_slot_carry(const SlotCarry &c, int sm_count, cudaStream_t st);
// Parking blobs are engine-owned: padded to 16 bytes
constexpr size_t kParkStride = (sizeof(StreamState) + 15) / 16 * 16;

}  // namespace pnb
