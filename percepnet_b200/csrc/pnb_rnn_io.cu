// pnb_rnn_io.cu -- the two copies of a network-only call (pnb_compute_rnn_*): the caller's stream-major rows of
// features or training records into the per-call buffer [F][S][70] the network hooks read, and the hooks' g/r
// [F][S][68] back out to stream-major rows.
#include "pnb_kernels.h"

namespace pnb {

// feat[(t*S + s)*70 + j] = in[s*in_stride + t*width + j] for the rows [0, n) of every hop t.  width = 138 (records):
// the first 68 values are scaled by 30 (create_features, denoise.cpp:487-496; rnn_train.py:44-48), T and pitchcorr
// are taken as they are, the labels rec[70..137] are never read.  Threads walk the output in order: the writes are
// contiguous, the reads contiguous runs of 70 floats.
__global__ void features_stage_kernel(float *__restrict__ feat, const float *__restrict__ in, size_t in_stride, int width,
                                      int n, int S, int F) {
  const long long total = (long long)F * n * kFeat;
  for (long long x = (long long)blockIdx.x * blockDim.x + threadIdx.x; x < total; x += (long long)gridDim.x * blockDim.x) {
    const int j = (int)(x % kFeat);
    const long long ts = x / kFeat;
    const int s = (int)(ts % n), t = (int)(ts / n);
    const float v = in[(size_t)s * in_stride + (size_t)t * width + j];
    feat[((size_t)t * S + s) * kFeat + j] = (width != kFeat && j < 68) ? v * 30.f : v;
  }
}

// out[s*out_stride + t*68 + c] = gr[(t*S + s)*68 + c] for the rows [0, n).  Threads walk the output in order: the
// writes are contiguous, the reads contiguous runs of 68 floats.
__global__ void gr_store_kernel(const float *__restrict__ gr, float *__restrict__ out, size_t out_stride, int n, int S,
                                int F) {
  const long long total = (long long)n * F * 68;
  for (long long x = (long long)blockIdx.x * blockDim.x + threadIdx.x; x < total; x += (long long)gridDim.x * blockDim.x) {
    const int c = (int)(x % 68);
    const long long st = x / 68;
    const int t = (int)(st % F), s = (int)(st / F);
    out[(size_t)s * out_stride + (size_t)t * 68 + c] = gr[((size_t)t * S + s) * 68 + c];
  }
}

static unsigned copy_blocks(long long total) {
  const long long b = (total + 255) / 256;
  return (unsigned)(b < 8192 ? b : 8192);
}

int launch_features_stage(float *feat, const float *in, size_t in_stride, int width, int n_streams, int S, int n_frames,
                          cudaStream_t st) {
  features_stage_kernel<<<copy_blocks((long long)n_frames * n_streams * kFeat), 256, 0, st>>>(feat, in, in_stride, width,
                                                                                             n_streams, S, n_frames);
  return 1;
}

int launch_gr_store(const float *gr, float *out, size_t out_stride, int n_streams, int S, int n_frames, cudaStream_t st) {
  gr_store_kernel<<<copy_blocks((long long)n_frames * n_streams * 68), 256, 0, st>>>(gr, out, out_stride, n_streams, S,
                                                                                    n_frames);
  return 1;
}

}  // namespace pnb
