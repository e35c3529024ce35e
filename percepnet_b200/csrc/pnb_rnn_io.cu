// pnb_rnn_io.cu -- the layout moves between a caller's stream-major rows and the per-call buffers [F][S][w] of the
// engine: the network call's features or training records into d_feat and its g/r out of d_gr (pnb_compute_rnn_*), the
// analysis half's features out of d_feat (pnb_analyze_*) and the synthesis half's caller g/r into d_gr
// (pnb_synthesize_*), and the same on a session list (row-mapped, with per-slot hops); the operands of a pending
// synthesis out to the caller's rows (pnb_synthesis_operands_device); and the loss of a score call (pnb_score_records_*),
// reduced from the same g/r and the records' labels.
#include "../../include/percepnet_b200.h"
#include "pnb_kernels.h"

namespace pnb {

// dst[(t*S + s)*W + j] = in[r*in_stride + t*in_width + j] for the rows [0, n) of every hop t and j < W, r = s (kMapped
// false) or row[s]: the list row of slot s in a session call; the first n_scaled values of a hop are multiplied by 30,
// the others copied as they are.  With hops (kMapped only) slot s gets zeros for its hops t >= hops[s], and the caller's
// row is not read there.  Features: W = 70, in_width 70, none scaled.  Records: W = 70, in_width 138, the first 68
// scaled (create_features, denoise.cpp:487-496; rnn_train.py:44-48), T and pitchcorr as they are, the labels
// rec[70..137] never read.  g/r: W = 68, in_width 68, none scaled.  Threads walk the output in order: the writes are
// contiguous, the reads contiguous runs of W floats.
template <int W, bool kMapped>
__global__ void rows_stage_kernel(float *__restrict__ dst, const float *__restrict__ in, size_t in_stride, int in_width,
                                  int n_scaled, int n, int S, int F, const int *__restrict__ row,
                                  const int *__restrict__ hops) {
  const long long total = (long long)F * n * W;
  for (long long x = (long long)blockIdx.x * blockDim.x + threadIdx.x; x < total; x += (long long)gridDim.x * blockDim.x) {
    const int j = (int)(x % W);
    const long long ts = x / W;
    const int s = (int)(ts % n), t = (int)(ts / n);
    float *d = dst + ((size_t)t * S + s) * W + j;
    if (kMapped && hops && t >= hops[s]) {
      *d = 0.f;
      continue;
    }
    const float v = in[(size_t)(kMapped ? row[s] : s) * in_stride + (size_t)t * in_width + j];
    *d = j < n_scaled ? v * 30.f : v;
  }
}

// out[r*out_stride + t*W + c] = src[(t*S + s)*W + c] for the rows r of [0, n), s = r (kMapped false) or slot[r]: the
// slot of list row r in a session call; with hops (kMapped only) zeros for the hops t >= hops[s] the slot did not run.
// g/r (W = 68) and features (W = 70).  Threads walk the output in order: the writes are contiguous, the reads
// contiguous runs of W floats.
template <int W, bool kMapped>
__global__ void rows_store_kernel(const float *__restrict__ src, float *__restrict__ out, size_t out_stride, int n, int S,
                                  int F, const int *__restrict__ slot, const int *__restrict__ hops) {
  const long long total = (long long)n * F * W;
  for (long long x = (long long)blockIdx.x * blockDim.x + threadIdx.x; x < total; x += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(x % W);
    const long long rt = x / W;
    const int t = (int)(rt % F), r = (int)(rt / F);
    const int s = kMapped ? slot[r] : r;
    out[(size_t)r * out_stride + (size_t)t * W + c] = (kMapped && hops && t >= hops[s]) ? 0.f : src[((size_t)t * S + s) * W + c];
  }
}

// The operands of the pending synthesis (include/pnb_synth_grad.h): ops[r*ops_stride + t*1636 + j] for the rows r of
// [0, n) and hops t of [0, F), read at exactly the addresses synthesis_kernel reads for slot r at hop t: X from the ring
// slot of hop hop0 + t - 5 (a call's first five hops read spectra of the previous call), P, Ex and the silence flag from
// the per-call buffers.  Threads walk the output in order: the writes are contiguous, the reads runs of 800 or 34 floats.
__global__ void synth_ops_kernel(const float2 *__restrict__ zring, int ring, long hop0, const float2 *__restrict__ P,
                                 const float *__restrict__ Ex, const unsigned char *__restrict__ silence,
                                 float *__restrict__ ops, size_t ops_stride, int n, int S, int F) {
  const long long total = (long long)n * F * kSynthOps;
  for (long long x = (long long)blockIdx.x * blockDim.x + threadIdx.x; x < total; x += (long long)gridDim.x * blockDim.x) {
    const int j = (int)(x % kSynthOps);
    const long long rt = x / kSynthOps;
    const int t = (int)(rt % F), r = (int)(rt / F);
    const size_t fs = (size_t)t * S + r;
    float v = 0.f;
    if (j < 2 * kBins) {
      const long c = hop0 + t;
      const int slot_x = (int)(((c - 5) % ring + ring) % ring);
      const float2 z = zring[((size_t)slot_x * S + r) * kBins + j / 2];
      v = (j & 1) ? z.y : z.x;
    } else if (j < 4 * kBins) {
      const float2 p = P[fs * kBins + (j - 2 * kBins) / 2];
      v = (j & 1) ? p.y : p.x;
    } else if (j < 4 * kBins + kBands) {
      v = Ex[fs * kBands + j - 4 * kBins];
    } else if (j == 4 * kBins + kBands) {
      v = silence[fs] != 0 ? 1.f : 0.f;
    }
    ops[(size_t)r * ops_stride + (size_t)t * kSynthOps + j] = v;
  }
}

// The loss rnn_train.py trains on (CustomLoss, rnn_train.py:153-176, gamma = 0.5), before its means and its C4 factor:
// for row i, over its first frames[i] hops t and the 34 bands b, with y the label rec[t][70..137] and p the prediction
// gr[t][i] (both widened to float64),
//   dg = sqrt(y_g) - sqrt(p_g)    dr = sqrt(1 - y_r) - sqrt(1 - p_r)
//   sums[i] = {sum dg^2, sum dg^4, sum dr^2, 34 frames[i]}
// One warp per row walks its hops in order; lane l keeps the partials of bands l and l + 32 (lanes 0 and 1), and a
// fixed shuffle tree adds the lanes.  No atomics: a row's sums depend on its own predictions and labels only, in a fixed
// order, so they are the same bits whatever else the call holds.  Every product and sum is rounded on its own (no
// contraction), as numpy's `** 0.5` (sqrt), `** 2` and the sums of eval_records.loss_sums round them; NaN (a label
// r > 1, say) propagates the same way.
__global__ void __launch_bounds__(256) loss_sums_kernel(const float *__restrict__ gr, const float *__restrict__ rec,
                                                        size_t rec_stride, const int *__restrict__ frames,
                                                        double *__restrict__ sums, int n, int S, int F) {
  const int i = (int)(((long long)blockIdx.x * blockDim.x + threadIdx.x) >> 5), lane = threadIdx.x & 31;
  if (i >= n) return;
  const int T = frames ? frames[i] : F;
  double g2 = 0.0, g4 = 0.0, r2 = 0.0;
  const float *y = rec + (size_t)i * rec_stride + 70;
  const float *p = gr + (size_t)i * 68;
  auto band = [&](int t, int b) {
    const double yg = y[(size_t)t * PNB_RECORD_FLOATS + b], yr = y[(size_t)t * PNB_RECORD_FLOATS + kBands + b];
    const double pg = p[(size_t)t * S * 68 + b], pr = p[(size_t)t * S * 68 + kBands + b];
    const double dg = __dsub_rn(sqrt(yg), sqrt(pg));
    const double dr = __dsub_rn(sqrt(__dsub_rn(1.0, yr)), sqrt(__dsub_rn(1.0, pr)));
    const double dg2 = __dmul_rn(dg, dg);
    g2 = __dadd_rn(g2, dg2);
    g4 = __dadd_rn(g4, __dmul_rn(dg2, dg2));
    r2 = __dadd_rn(r2, __dmul_rn(dr, dr));
  };
#pragma unroll 4
  for (int t = 0; t < T; t++) {
    band(t, lane);
    if (lane < kBands - 32) band(t, lane + 32);
  }
  for (int o = 16; o > 0; o >>= 1) {
    g2 = __dadd_rn(g2, __shfl_down_sync(0xffffffffu, g2, o));
    g4 = __dadd_rn(g4, __shfl_down_sync(0xffffffffu, g4, o));
    r2 = __dadd_rn(r2, __shfl_down_sync(0xffffffffu, r2, o));
  }
  if (lane == 0) {
    double *s = sums + (size_t)i * 4;
    s[0] = g2; s[1] = g4; s[2] = r2; s[3] = (double)T * kBands;
  }
}

static unsigned copy_blocks(long long total) {
  const long long b = (total + 255) / 256;
  return (unsigned)(b < 8192 ? b : 8192);
}

template <int W>
static void rows_stage(unsigned blocks, float *dst, const float *in, size_t in_stride, int in_width, int n_scaled, int n,
                       int S, int F, const int *row, const int *hops, cudaStream_t st) {
  if (row) rows_stage_kernel<W, true><<<blocks, 256, 0, st>>>(dst, in, in_stride, in_width, n_scaled, n, S, F, row, hops);
  else rows_stage_kernel<W, false><<<blocks, 256, 0, st>>>(dst, in, in_stride, in_width, n_scaled, n, S, F, nullptr, nullptr);
}
void launch_rows_stage(float *dst, int w, const float *in, size_t in_stride, int in_width, int n_scaled, int n_streams,
                       int S, int n_frames, cudaStream_t st, const int *row, const int *hops) {
  const unsigned blocks = copy_blocks((long long)n_frames * n_streams * w);
  if (w == kFeat) rows_stage<kFeat>(blocks, dst, in, in_stride, in_width, n_scaled, n_streams, S, n_frames, row, hops, st);
  else rows_stage<68>(blocks, dst, in, in_stride, in_width, n_scaled, n_streams, S, n_frames, row, hops, st);
}

template <int W>
static void rows_store(unsigned blocks, const float *src, float *out, size_t out_stride, int n, int S, int F, const int *slot,
                       const int *hops, cudaStream_t st) {
  if (slot) rows_store_kernel<W, true><<<blocks, 256, 0, st>>>(src, out, out_stride, n, S, F, slot, hops);
  else rows_store_kernel<W, false><<<blocks, 256, 0, st>>>(src, out, out_stride, n, S, F, nullptr, nullptr);
}
void launch_rows_store(const float *src, int w, float *out, size_t out_stride, int n_streams, int S, int n_frames,
                       cudaStream_t st, const int *slot, const int *hops) {
  const unsigned blocks = copy_blocks((long long)n_frames * n_streams * w);
  if (w == kFeat) rows_store<kFeat>(blocks, src, out, out_stride, n_streams, S, n_frames, slot, hops, st);
  else rows_store<68>(blocks, src, out, out_stride, n_streams, S, n_frames, slot, hops, st);
}

void launch_synth_ops(const SynthesisArgs &a, float *ops, size_t ops_stride, cudaStream_t st) {
  synth_ops_kernel<<<copy_blocks((long long)a.n_streams * a.n_frames * kSynthOps), 256, 0, st>>>(
      a.zring, a.ring, a.hop0, a.P, a.Ex, a.silence, ops, ops_stride, a.n_streams, a.stride, a.n_frames);
}

void launch_loss_sums(const float *gr, const float *rec, size_t rec_stride, const int *frames, double *sums, int n_streams,
                      int S, int n_frames, cudaStream_t st) {
  loss_sums_kernel<<<(unsigned)(((long long)n_streams * 32 + 255) / 256), 256, 0, st>>>(gr, rec, rec_stride, frames, sums,
                                                                                      n_streams, S, n_frames);
}

}  // namespace pnb
