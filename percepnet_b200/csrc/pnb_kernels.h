// pnb_kernels.h -- kernel argument blocks and launcher prototypes shared by the .cu files.
#pragma once
#include "pnb_common.cuh"

namespace pnb {

// ---- DSP (pnb_dsp.cu) -------------------------------------------------------------------
struct AnalysisArgs {
  const float *pcm;        // [S][pcm_stride]: 5280 samples of history, then the call's hops
  size_t pcm_stride;
  int n_streams, n_frames; // streams analysed: rows [0, n_streams)
  int stride;              // S: rows per hop slot of the per-call buffers and the ring (>= n_streams)
  const Tables *tab;
  float *feat;             // [F][S][70]
  float2 *zring;           // [ring][S][400] spectra of the windowed blocks, slot = hop % ring (carried state)
  float *ering;            // [ring][S][34] their band energies
  int ring;                // slots (>= n_frames + 5)
  long hop0;               // absolute index of the call's first hop
  float2 *P;               // [F][S][400] or null (training-data mode has no synthesis)
  float *Ex;               // [F][S][34] or null
  float *raw;              // [F][S][68] or null: look-ahead band energies and pitch coherence before the x30
  unsigned char *silence;  // [F][S]
  int *last_period;        // [S] carried state
  float *last_gain;        // [S]
  int *tap_pitch;          // [F][S][4] or null
  float *tap_pitchf;       // [F][S][2] or null
  const int *hops;         // [n_streams] hops of each slot (ragged session calls, each <= n_frames), or null: n_frames
};

struct SynthesisArgs {
  const float2 *zring;     // analysis spectrum of hop c is the ring slot of hop c-5
  int ring;
  long hop0;
  const float2 *P;         // [F][S][400]
  const float *gr;         // [F][S][68]
  const float *Ex;         // [F][S][34] (post-filter only)
  const unsigned char *silence;
  int n_streams, n_frames; // streams synthesised: rows [0, n_streams)
  int stride;              // S: rows per hop slot of the per-call buffers and the ring (>= n_streams)
  const Tables *tab;
  float *synth_mem;        // [S][480] carried state
  float *out;              // float output rows or null
  short *out16;            // int16 output rows or null
  size_t out_stride;
  int postfilter;
  float *tap_g;            // [F][S][34] or null: the band gains as applied (after the optional post-filter)
  const int *row;          // [n_streams] output row of each slot (session calls), or null: row s
  const int *hops;         // [n_streams] hops of each slot (ragged session calls), or null: n_frames; hops [hops[s],
                           // n_frames) of a slot's output row are written as zeros
};

// training-data records (train(), denoise.cpp:600-787): streams [0,N) are the noisy signals, [N,2N) the clean ones
struct LabelArgs {
  const float *feat;       // [F][2N][70]
  const float *raw;        // [F][2N][68]
  const float *Ex;         // [F][2N][34]
  const Tables *tab;
  int n_pairs, n_frames;
  float *records;          // pair p, frame t at records + p*pair_stride + t*138
  size_t pair_stride;
};
int launch_train_labels(const LabelArgs &a, cudaStream_t st);

// pitch analysis alone (BASELINE.json config 5): unit u reads buf[u*stride .. +1728), writes T/corr/gain (and the
// pitch_search lag when lag != null); prev_period / prev_gain null = 0 (a fresh stream)
struct PitchOnlyArgs {
  const float *buf;
  size_t stride;
  long n_units;
  const int *prev_period;
  const float *prev_gain;
  int *T;
  float *corr, *gain;
  int *lag;
};
int launch_pitch_only(const PitchOnlyArgs &a, cudaStream_t st);

cudaError_t dsp_configure();
int launch_analysis(const AnalysisArgs &a, cudaStream_t st);
int launch_synthesis(const SynthesisArgs &a, cudaStream_t st);
// row: [n_streams] input row of each slot (session calls), or null: row s.  hops: [n_streams] hops of each slot (ragged
// session calls), or null: slot s copies hops[s] * 480 samples instead of n_samples
int launch_stage_in(float *pcm, size_t pcm_stride, const float *in, const short *in16, size_t in_stride,
                    int n_streams, int n_samples, cudaStream_t st, float i16_div = 32768.f, const int *row = nullptr,
                    const int *hops = nullptr);
int launch_slide_history(float *pcm, size_t pcm_stride, int n_streams, int n_samples, cudaStream_t st);

// ---- network, fp32 FMA path (pnb_nn_f32.cu) ---------------------------------------------
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
int launch_gemm_f32(const GemmArgs &g, cudaStream_t st);

// fc: features [M x 70] -> [M x 128], relu (nnet.cpp:105 on the `fc` layer), on M rows of each of n_slots hop slots
// slot_stride rows apart
int launch_fc_f32(const float *feat, const float *W, const float *bias, float *out, int M, int K, int N, int n_slots,
                  size_t slot_stride, cudaStream_t st);

// The five GRUs of a chunk of hops in one persistent fp32 launch (pnb_nn_f32.cu).  Slot buffers: hop t of the chunk
// reads state slot t and writes slot t+1; inputs are conv2's output slot t or the layer below's slot t+1.
struct F32ChainLayer {
  int H, n_x, dep;            // hidden size; input segments (1 or 2); layer whose fresh state is the input (-1: conv2 out)
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
  int S, n, n_rb, n_units, n_lh;               // S: rows per slot; n: active streams [0, n); n_rb: their stream blocks
  unsigned char lh[5 * kF32ChainMaxHops];      // (hop << 3) | layer in anti-diagonal order
  int lh_unit0[5 * kF32ChainMaxHops + 1];      // first unit of every entry; [n_lh] = n_units
  unsigned *cnt;                               // [5][n_rb] finished tiles per (layer, stream block), zero at launch
  const float *tansig;
};
int launch_gru_chain_f32(const F32ChainArgs &a, int rows_per_thread, int sm_count, cudaStream_t st);
// The first slot4 float4s of n_slots slots stride4 apart, from slots from.. of src (slot 0 of the source buffer) to
// dst; row4: float4s per row.  In a ragged call (hops) a row that stops after hop h of the call takes its slots from
// from - (n - clamp(h - h0, 0, n)) on instead (it stopped that many slots before the chunk's end), and nothing moves
// when that is below 0 or the row is already in place.
struct F32CarrySeg { float4 *dst; const float4 *src; size_t slot4, stride4, row4; int n_slots, from; };
struct F32CarryArgs {
  F32CarrySeg seg[12];
  int n_seg;
  unsigned *cnt;
  int n_cnt;
  const int *hops;  // [active streams] hops of each row in a ragged call, or null
  int h0, n;        // the chunk: hops [h0, h0 + n) of the call
};
int launch_f32_carry(const F32CarryArgs &a, cudaStream_t st);

}  // namespace pnb
