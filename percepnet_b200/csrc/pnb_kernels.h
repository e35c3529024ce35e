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
  float2 *P;               // [F][S][400] or null (a training-data engine without PNB_TRAIN_AUDIO has no synthesis)
  int P_rows;              // P is stored for rows [0, P_rows) only (a training-data engine resynthesises the noisy rows)
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
  int clamp16;             // int16 conversion of out16: 0 truncates y*32768 (main.cpp:36), 1 clamps y to [-32768, 32767]
                           // and truncates (train()'s test_output.pcm, denoise.cpp:756-758)
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
  float *gr;               // [F][2N][68] or null: the record's g and r of pair p, frame t at row t*2N + p (its noisy row)
};
void launch_train_labels(const LabelArgs &a, cudaStream_t st);

// pitch analysis alone (BASELINE.json config 5): unit u reads buf[u*stride .. +1728), writes T/corr/gain (and the
// pitch_search lag when lag != null); prev_period / prev_gain null = 0 (a fresh stream).  Returns false, launching
// nothing, when the kernel cannot be configured.
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
bool launch_pitch_only(const PitchOnlyArgs &a, cudaStream_t st);

// The synthesis's gradient with respect to g/r (include/pnb_synth_grad.h): one warp per (row, hop) of n_rows rows of
// n_frames hops; strides in floats.  Returns false, launching nothing, when the kernel cannot be configured.
constexpr int kSynthOps = 1636;  // PNB_SYNTH_OPS_FLOATS: X [800], P [800], Ex [34], silence, padding
struct SynthGradArgs {
  const float *ops;
  size_t ops_stride;
  const float *gr;
  size_t gr_stride;
  const float *dout;
  size_t dout_stride;
  float *dgr;
  size_t dgr_stride;
  long long n_rows;
  int n_frames;
  int postfilter;
  const Tables *tab;
};
bool launch_synthesis_backward(const SynthGradArgs &a, cudaStream_t st);

cudaError_t dsp_configure();
void launch_analysis(const AnalysisArgs &a, cudaStream_t st);
void launch_synthesis(const SynthesisArgs &a, cudaStream_t st);
// row: [n_streams] input row of each slot (session calls), or null: row s.  hops: [n_streams] hops of each slot (ragged
// session calls), or null: slot s copies hops[s] * 480 samples instead of n_samples
void launch_stage_in(float *pcm, size_t pcm_stride, const float *in, const short *in16, size_t in_stride,
                     int n_streams, int n_samples, cudaStream_t st, float i16_div = 32768.f, const int *row = nullptr,
                     const int *hops = nullptr);
void launch_slide_history(float *pcm, size_t pcm_stride, int n_streams, int n_samples, cudaStream_t st);

// ---- layout moves of the network and split calls (pnb_rnn_io.cu) ---------------------------
// rows [0, n_streams) of `in` (n_frames hops of in_width floats each) -> dst [F][S][w], w = 70 (features, or records
// with in_width 138) or 68 (g/r); the first n_scaled values of each hop are multiplied by 30 (records: 68, else 0).
// row: [n_streams] the input row of each slot (session calls), or null: row s.  hops (with row only): [n_streams] hops
// of each slot, or null: n_frames; slot s gets zeros for hops >= hops[s], whose input is not read
void launch_rows_stage(float *dst, int w, const float *in, size_t in_stride, int in_width, int n_scaled, int n_streams,
                       int S, int n_frames, cudaStream_t st, const int *row = nullptr, const int *hops = nullptr);
// src [F][S][w] -> rows [0, n_streams) of `out`, n_frames x w floats each; w = 68 (g/r) or 70 (features).  slot:
// [n_streams] the slot of each output row (session calls), or null: slot r.  hops (with slot only): [n_streams] hops of
// each slot, or null: n_frames; a row is zero for the hops its slot did not run
void launch_rows_store(const float *src, int w, float *out, size_t out_stride, int n_streams, int S, int n_frames,
                       cudaStream_t st, const int *slot = nullptr, const int *hops = nullptr);
// the operands synthesis_kernel reads for the rows [0, a.n_streams) and hops [0, a.n_frames) of the synthesis `a`
// (zring, ring, hop0, P, Ex, silence, stride) -> ops rows of n_frames x kSynthOps floats
void launch_synth_ops(const SynthesisArgs &a, float *ops, size_t ops_stride, cudaStream_t st);
// rnn_train.py's CustomLoss sums of rows [0, n_streams): gr [F][S][68] against the labels rec[t][70..137] of row i's
// first frames[i] hops (frames null: all n_frames) -> sums[i] = {sum dg^2, sum dg^4, sum dr^2, count} in float64
void launch_loss_sums(const float *gr, const float *rec, size_t rec_stride, const int *frames, double *sums, int n_streams,
                      int S, int n_frames, cudaStream_t st);

}  // namespace pnb
