// pnb_engine.cu -- host side of the C-ABI (include/percepnet_b200.h): engine lifetime, weight ingest
// from the reference's RNNModel layout, constant tables, and the per-call kernel schedule.
//
// Schedule of one pnb_process_* call with F hops on S streams:
//   stage_in -> analysis (all F hops; one warp per stream) -> F x network step -> synthesis -> slide history
// The network step is the only part that is sequential in time across the batch; analysis and synthesis
// need no network state, so hops are processed F at a time.  A network-only call (pnb_compute_rnn_*) is
//   rows_stage (features) -> F x network step -> rows_store (g/r)
// on caller-supplied features or training records.  The split call cuts the PCM call where the network sits, on slots
// and on a session list (pnb_*_sessions_*) alike, each half the fused call's (analysis_half / synthesis_half):
//   pnb_analyze_*:    [session move] -> stage_in -> analysis -> rows_store (features)
//   pnb_synthesize_*: rows_stage (caller g/r) -> synthesis [-> ragged fix-up] [-> slide history]
#include <math.h>
#include <stdarg.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <stddef.h>
#include <stdint.h>
#include <algorithm>
#include <mutex>
#include <string>
#include <vector>

#include "../../include/percepnet_b200.h"
#include "pnb_engine.h"

using namespace pnb;

static thread_local std::string g_err;
static int fail(int code, const char *fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  g_err = buf;
  return code;
}
#define CK(call)                                                                                   \
  do {                                                                                             \
    cudaError_t _e = (call);                                                                       \
    if (_e != cudaSuccess) return fail(PNB_ERR_CUDA, "%s failed: %s (%s:%d)", #call, cudaGetErrorString(_e), __FILE__, __LINE__); \
  } while (0)

int engine_fail(int code, const char *msg) { return fail(code, "%s", msg); }

extern "C" const char *pnb_last_error(void) { return g_err.c_str(); }
extern "C" const char *pnb_version(void) { return "percepnet_b200 0.1 (sm_90a)"; }

// ------------------------------------------------------------------------------------------
// constant tables, with the reference's own expressions so that they round identically
// ------------------------------------------------------------------------------------------
static void build_tables(Tables &t) {
  memset(&t, 0, sizeof t);
  for (int i = 0; i < kFrame; i++) {  // denoise.cpp:191-192
    double a = .5 * M_PI * (i + .5) / kFrame;
    t.half_window[i] = (float)sin(.5 * M_PI * sin(a) * sin(a));
  }
  {  // denoise.cpp:200-206: float running sum
    float acc = 0;
    for (int i = 1; i < 8; i++) {
      t.comb_w[i - 1] = (float)(0.5 - 0.5 * cos(2.0 * M_PI * i / 8));
      acc += t.comb_w[i - 1];
    }
    for (int i = 0; i < 7; i++) t.comb_w[i] /= acc;
  }
  for (int i = 0; i < kWin; i++) {  // kiss_fft.cpp:415-419
    const double pi = 3.14159265358979323846264338327;
    double ph = (-2 * pi / kWin) * i;
    t.tw[i].x = (float)cos(ph);
    t.tw[i].y = (float)sin(ph);
  }
  {  // erbband.h:34-99 with (960, 32, 0, 20000), denoise.cpp:87
    auto hz2erb = [](float hz) { return (float)(9.265 * log(1 + hz / (24.7 * 9.265))); };
    auto erb2hz = [](float e) { return (float)(24.7 * 9.265 * (exp(e / 9.265) - 1)); };
    float lo = hz2erb(0.f), hi = hz2erb(20000.f), step = (hi - lo) / (34.f - 1);
    int border[kBands];
    for (int i = 0; i < kBands; i++) {
      float cut = erb2hz(i < kBands - 1 ? lo + step * i : hi);
      border[i] = (int)((cut + 25) / 50.f);
    }
    for (int i = 0; i < kBands - 2; i++)
      if (border[i + 1] - border[i] < 2) border[i + 1] += 2 - (border[i + 1] - border[i]);
    for (int i = 0; i < kBands; i++) t.border[i] = (short)border[i];
    t.border[kBands] = t.border[kBands + 1] = (short)border[kBands - 1];
    for (int b = 0; b < kBands - 1; b++) {
      int width = border[b + 1] - border[b];
      for (int j = 0; j < width; j++) {
        int bin = border[b] + j;
        if (bin >= kBins) continue;
        float frac = (float)j / width;  // denoise.cpp:99
        t.frac[bin] = frac;
        t.omf[bin] = 1 - frac;
        t.band_of[bin] = (short)b;
      }
    }
  }
  // tansig_table.h: tanh(0.04 i) to six decimals; the three entries where the shipped table is not the
  // correctly rounded value carry the shipped value
  for (int i = 0; i <= 200; i++) t.tansig[i] = (float)(floor(tanh(0.04 * i) * 1e6 + 0.5) / 1e6);
  t.tansig[70] = 0.992631f;
  t.tansig[170] = 0.999997f;
  t.tansig[190] = 1.000000f;
}

// ------------------------------------------------------------------------------------------
cudaError_t engine_buffer(pnb_engine *e, void **p, size_t bytes, bool zero_on_reset, const void *src) {
  cudaError_t r = cudaMalloc(p, bytes);
  if (r != cudaSuccess) return r;
  e->buffers.push_back({*p, bytes, zero_on_reset});
  return src ? cudaMemcpy(*p, src, bytes, cudaMemcpyHostToDevice) : cudaMemset(*p, 0, bytes);
}

static int check_model(const pnb_model *m) {
  if (!m || !m->fc || !m->conv1 || !m->conv2 || !m->gru1 || !m->gru2 || !m->gru3 || !m->gru_gb || !m->gru_rb ||
      !m->fc_gb || !m->fc_rb)
    return fail(PNB_ERR_ARG, "model or one of its ten layers is NULL");
  // the architecture the hot path is built for (rnn_train.py:111-121, rnn.cpp:42-81)
  bool ok = m->fc->nb_inputs == 70 && m->fc->nb_neurons == 128 && m->conv1->nb_inputs == 128 &&
            m->conv1->kernel_size == 5 && m->conv1->nb_neurons == 512 && m->conv2->nb_inputs == 512 &&
            m->conv2->kernel_size == 3 && m->conv2->nb_neurons == 512 && m->gru_rb->nb_inputs == 1024 &&
            m->gru_rb->nb_neurons == 128 && m->fc_gb->nb_inputs == 2560 && m->fc_gb->nb_neurons == 34 &&
            m->fc_rb->nb_inputs == 128 && m->fc_rb->nb_neurons == 34;
  const pnb_gru_layer *g4[4] = {m->gru1, m->gru2, m->gru3, m->gru_gb};
  for (int i = 0; i < 4; i++) ok = ok && g4[i]->nb_inputs == 512 && g4[i]->nb_neurons == 512;
  const pnb_gru_layer *g5[5] = {m->gru1, m->gru2, m->gru3, m->gru_gb, m->gru_rb};
  for (int i = 0; i < 5; i++) ok = ok && g5[i]->reset_after == 1 && g5[i]->activation == PNB_ACT_TANH;
  if (!ok) return fail(PNB_ERR_ARG, "model dimensions are not PercepNet's (70-128-conv5x512-conv3x512-4xGRU512-GRU128-34/34)");
  // the kernels fuse each layer's activation (rnn_train.py:111-121 / dump_percepnet.py); a model that asks for
  // anything else would silently compute something the reference does not
  if (m->fc->activation != PNB_ACT_RELU || m->conv1->activation != PNB_ACT_RELU || m->conv2->activation != PNB_ACT_TANH ||
      m->fc_gb->activation != PNB_ACT_SIGMOID || m->fc_rb->activation != PNB_ACT_SIGMOID)
    return fail(PNB_ERR_ARG, "model activations are not PercepNet's (fc relu, conv1 relu, conv2 tanh, fc_gb / fc_rb sigmoid)");
  return PNB_OK;
}

extern "C" int pnb_resolve_device(int device) {
  int ndev = 0;
  cudaError_t ce = cudaGetDeviceCount(&ndev);
  if (ce != cudaSuccess || ndev == 0)
    return fail(PNB_ERR_NO_DEVICE, "no CUDA device available (%s); this library has no CPU path",
                ce == cudaSuccess ? "device count 0" : cudaGetErrorString(ce));
  if (device == -1) {  // the calling thread's current device
    ce = cudaGetDevice(&device);
    if (ce != cudaSuccess) return fail(PNB_ERR_CUDA, "cudaGetDevice failed: %s", cudaGetErrorString(ce));
  }
  if (device < 0 || device >= ndev) return fail(PNB_ERR_ARG, "device %d out of range (have %d)", device, ndev);
  return device;
}

extern "C" int pnb_create(pnb_engine **out, int n_streams, int max_frames, const pnb_model *model, unsigned flags,
                          int device) {
  if (!out) return fail(PNB_ERR_ARG, "out is NULL");
  *out = nullptr;
  if (n_streams < 1 || max_frames < 1) return fail(PNB_ERR_ARG, "n_streams and max_frames_per_call must be >= 1");
  if ((long long)n_streams * max_frames > (1ll << 24))
    return fail(PNB_ERR_ARG, "n_streams x max_frames_per_call above 2^24 rows per call: split the batch across engines");
  if ((flags & PNB_TRAIN_NETWORK) &&
      (flags & (PNB_NN_TENSOR | PNB_CONV_WIDE | PNB_TRAIN_DATA | PNB_TRAIN_AUDIO | PNB_POSTFILTER | PNB_SIGNAL_ONLY)))
    return fail(PNB_ERR_ARG, "PNB_TRAIN_NETWORK trains the fp32 network alone: combine it only with PNB_NETWORK_ONLY and PNB_KEEP_TAPS");
  if (flags & PNB_TRAIN_NETWORK) flags |= PNB_NETWORK_ONLY;  // a training engine is a network-only engine that also trains
  const bool train_mode = (flags & PNB_TRAIN_DATA) != 0, train_audio = (flags & PNB_TRAIN_AUDIO) != 0;
  if (train_audio && !train_mode) return fail(PNB_ERR_ARG, "PNB_TRAIN_AUDIO applies to PNB_TRAIN_DATA engines");
  if (train_mode && (n_streams & 1)) return fail(PNB_ERR_ARG, "PNB_TRAIN_DATA needs n_streams = 2 x pairs");
  if ((flags & PNB_CONV_WIDE) && !(flags & PNB_NN_TENSOR)) return fail(PNB_ERR_ARG, "PNB_CONV_WIDE applies to PNB_NN_TENSOR engines");
  if (train_mode && (flags & (PNB_NN_TENSOR | PNB_POSTFILTER | PNB_NETWORK_ONLY)))
    return fail(PNB_ERR_ARG, "PNB_TRAIN_DATA runs no network: combine it only with PNB_KEEP_TAPS");
  const bool net_only = (flags & PNB_NETWORK_ONLY) != 0;
  if (net_only && (flags & (PNB_TRAIN_AUDIO | PNB_POSTFILTER)))
    return fail(PNB_ERR_ARG, "PNB_NETWORK_ONLY runs no signal path: PNB_TRAIN_AUDIO and PNB_POSTFILTER do not apply");
  const bool sig_only = (flags & PNB_SIGNAL_ONLY) != 0;
  if (sig_only && (flags & (PNB_NN_TENSOR | PNB_CONV_WIDE | PNB_TRAIN_DATA | PNB_TRAIN_AUDIO | PNB_NETWORK_ONLY)))
    return fail(PNB_ERR_ARG, "PNB_SIGNAL_ONLY runs no network: combine it only with PNB_POSTFILTER and PNB_KEEP_TAPS");
  const bool has_net = !train_mode && !sig_only;
  int rc = has_net ? check_model(model) : 0;
  if (rc) return rc;
  device = pnb_resolve_device(device);
  if (device < 0) return device;
  CK(cudaSetDevice(device));
  cudaDeviceProp prop;
  CK(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0)
    return fail(PNB_ERR_NO_DEVICE, "device %d is sm_%d%d; this build carries sm_90a (Hopper) code only", device, prop.major,
                prop.minor);

  pnb_engine *e = new pnb_engine();
  e->S = n_streams;
  e->n_active = n_streams;
  e->Fmax = max_frames;
  e->device = device;
  e->flags = flags;
  e->sm_count = prop.multiProcessorCount;
  const size_t S = n_streams, F = max_frames;
#define CKD(call)                                                                                   \
  do {                                                                                              \
    cudaError_t _e = (call);                                                                        \
    if (_e != cudaSuccess) {                                                                        \
      int _rc = fail(_e == cudaErrorMemoryAllocation ? PNB_ERR_ALLOC : PNB_ERR_CUDA, "%s failed: %s", #call, cudaGetErrorString(_e)); \
      pnb_destroy(e);                                                                               \
      return _rc;                                                                                   \
    }                                                                                               \
  } while (0)

  CKD(cudaStreamCreateWithFlags(&e->stream, cudaStreamNonBlocking));
  CKD(dsp_configure());
  {
    Tables *t = new Tables();
    build_tables(*t);
    cudaError_t r = engine_upload(e, &e->d_tab, t, 1);
    delete t;
    CKD(r);
  }
  if (has_net) {  // both paths run fc from the reference's layout (SURVEY.md App. B)
    CKD(engine_upload(e, &e->fc.W, model->fc->input_weights, 70 * 128));
    CKD(engine_upload(e, &e->fc.b, model->fc->bias, 128));
  }

  // stream state
  // room for several calls' hops behind the history (advance_line): eight calls when calls are short, fewer
  // when one call already carries many hops (the move is then amortised over those hops anyway)
  const size_t line_calls = F >= 128 ? 1 : (128 / F > (size_t)kLineCalls ? (size_t)kLineCalls : 128 / F);
  if (!net_only) {  // a network-only engine has no signal path: none of its buffers, here and below
    e->pcm_stride = kKeep + line_calls * F * kFrame;
    CKD(engine_alloc(e, &e->d_pcm, S * e->pcm_stride, kStreamState));
    CKD(engine_alloc(e, &e->d_synth, S * kFrame, kStreamState));
  }
  CKD(engine_alloc(e, &e->d_status, 2, kScratch));  // pnb_reset sets it itself
  CKD(cudaMemset(e->d_status + 1, 0x7F, sizeof(int)));  // kNoRejectedSlot
  CKD(cudaHostAlloc((void **)&e->h_status, 2 * sizeof(int), cudaHostAllocDefault));
  e->h_status[0] = 0;
  e->h_status[1] = kNoRejectedSlot;
  // batched stream-state operations: staging of the slot indices, import verdicts (both grown by the session pool),
  // one blob of scratch
  CKD(cudaEventCreateWithFlags(&e->ev_call, cudaEventDisableTiming));
  for (int k = 0; k < 2; k++) {
    CKD(cudaEventCreateWithFlags(&e->ev_idx[k], cudaEventDisableTiming));
    CKD(cudaHostAlloc((void **)&e->h_idx[k], S * sizeof(int), cudaHostAllocDefault));
    CKD(cudaMalloc((void **)&e->d_idx[k], S * sizeof(int)));
  }
  e->idx_cap = S;
  CKD(cudaMalloc((void **)&e->d_ok, S * sizeof(int)));
  e->ok_cap = S;
  CKD(engine_buffer(e, &e->d_blob1, sizeof(StreamState), kScratch, nullptr));
  if (!net_only) {
    CKD(engine_alloc(e, &e->d_last_period, S, kStreamState));
    CKD(engine_alloc(e, &e->d_last_gain, S, kStreamState));
  }
  // per-call buffers
  CKD(engine_alloc(e, &e->d_feat, F * S * kFeat, kScratch));
  if (!net_only) {
    e->ring = (int)F + 5;
    CKD(engine_alloc(e, &e->d_zring, (size_t)e->ring * S * kBins, kStreamState));
    CKD(engine_alloc(e, &e->d_ering, (size_t)e->ring * S * kBands, kStreamState));
    if (!train_mode || train_audio) CKD(engine_alloc(e, &e->d_P, F * S * kBins, kScratch));  // audio: noisy rows only
    CKD(engine_alloc(e, &e->d_Ex, F * S * kBands, kScratch));
    CKD(engine_alloc(e, &e->d_sil, F * S, kScratch));
  }
  if (!train_mode || train_audio) CKD(engine_alloc(e, &e->d_gr, F * S * 68, kScratch));  // audio: the noisy rows' labels
  if (train_mode) CKD(engine_alloc(e, &e->d_raw, F * S * 68, kScratch));
  if ((flags & PNB_KEEP_TAPS) && !net_only) {  // the taps a network-only engine keeps need no buffers of their own
    CKD(engine_alloc(e, &e->d_tap_pitch, F * S * 4, kScratch));
    CKD(engine_alloc(e, &e->d_tap_pitchf, F * S * 2, kScratch));
    if (!train_mode) CKD(engine_alloc(e, &e->d_tap_g, F * S * kBands, kScratch));
  }
  if (has_net) {  // a signal-only engine has no network: no weights, network state or network buffers
    CKD(engine_alloc(e, &e->c2, S * 512, kStreamState));
    int rc = (flags & PNB_NN_TENSOR) ? tc_prepare(e, model) : f32_prepare(e, model);
    if (!rc && (flags & PNB_TRAIN_NETWORK)) rc = train_prepare(e);
    if (rc) { pnb_destroy(e); return rc; }
  }
  CKD(cudaDeviceSynchronize());
  *out = e;
  return PNB_OK;
}

extern "C" void pnb_destroy(pnb_engine *e) {
  if (!e) return;
  cudaSetDevice(e->device);
  cudaDeviceSynchronize();
  for (const auto &b : e->buffers) cudaFree(b.p);
  if (e->h_status) cudaFreeHost(e->h_status);
  for (int k = 0; k < 2; k++) {
    if (e->h_idx[k]) cudaFreeHost(e->h_idx[k]);
    if (e->d_idx[k]) cudaFree(e->d_idx[k]);
    if (e->ev_idx[k]) cudaEventDestroy(e->ev_idx[k]);
  }
  if (e->d_ok) cudaFree(e->d_ok);
  if (e->d_park) cudaFree(e->d_park);
  if (e->d_sgr) cudaFree(e->d_sgr);
  if (e->ev_call) cudaEventDestroy(e->ev_call);
  for (int k = 0; k < 2; k++) {
    if (e->stage[k].in) cudaFree(e->stage[k].in);
    if (e->stage[k].out) cudaFree(e->stage[k].out);
    if (e->ev_in[k]) cudaEventDestroy(e->ev_in[k]);
    if (e->ev_cmp[k]) cudaEventDestroy(e->ev_cmp[k]);
    if (e->ev_out[k]) cudaEventDestroy(e->ev_out[k]);
  }
  if (e->s_in) cudaStreamDestroy(e->s_in);
  if (e->s_out) cudaStreamDestroy(e->s_out);
  for (auto &r : e->prof_pending) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
  for (auto ev : e->prof_pool) cudaEventDestroy(ev);
  if (e->stream) cudaStreamDestroy(e->stream);
  delete e;
}

extern "C" int pnb_reset(pnb_engine *e) {
  if (!e) return fail(PNB_ERR_ARG, "engine is NULL");
  CK(cudaSetDevice(e->device));
  cudaDeviceSynchronize();  // a poisoned engine may carry a sticky launch error of its own; the memsets below report a dead context
  cudaGetLastError();
  for (const auto &b : e->buffers)
    if (b.zero_on_reset) CK(cudaMemset(b.p, 0, b.bytes));
  e->line_off = 0;
  CK(cudaMemset(e->d_status, 0, sizeof(int)));
  CK(cudaMemset(e->d_status + 1, 0x7F, sizeof(int)));  // kNoRejectedSlot
  e->h_status[0] = 0;
  e->h_status[1] = kNoRejectedSlot;
  e->hop = 0;
  e->pending = {};
  e->n_active = e->S;
  e->poisoned = false;
  e->train_open = false;  // the accumulator (stream state) was zeroed above; the held gradient stays, and stays due
  e->train_fwd_F = 0;
  if (e->sessions) {  // every session fresh: all parked, every blob marked fresh
    CK(cudaMemset(e->d_park, 0, (size_t)e->pool.capacity() * kParkStride));
    e->pool.init(e->S, e->pool.capacity());
  }
  CK(cudaDeviceSynchronize());
  return PNB_OK;
}

// ------------------------------------------------------------------------------------------
// per-kernel-class timing
// ------------------------------------------------------------------------------------------
static cudaEvent_t prof_event(pnb_engine *e) {
  if (!e->prof_pool.empty()) { cudaEvent_t ev = e->prof_pool.back(); e->prof_pool.pop_back(); return ev; }
  cudaEvent_t ev;
  cudaEventCreate(&ev);
  return ev;
}
LaunchScope::LaunchScope(pnb_engine *eng, int cls, cudaStream_t s) : e(eng), idx(-1), st(s) {
  e->launches++;
  if (!e->profiling || cls == kUnprofiled) return;
  pnb_engine::ProfRec r;
  r.cls = cls; r.a = prof_event(e); r.b = prof_event(e);
  cudaEventRecord(r.a, st);
  e->prof_pending.push_back(r);
  idx = (int)e->prof_pending.size() - 1;
}
LaunchScope::~LaunchScope() {
  if (idx >= 0) cudaEventRecord(e->prof_pending[idx].b, st);
}
extern "C" int pnb_profile_enable(pnb_engine *e, int on) {
  if (!e) return fail(PNB_ERR_ARG, "engine is NULL");
  e->profiling = on != 0;
  return PNB_OK;
}
extern "C" int pnb_profile_read(pnb_engine *e, double *ms, long long *counts) {
  if (!e || !ms || !counts) return fail(PNB_ERR_ARG, "NULL argument");
  CK(cudaSetDevice(e->device));
  CK(cudaDeviceSynchronize());
  for (auto &r : e->prof_pending) {
    float t = 0.f;
    CK(cudaEventElapsedTime(&t, r.a, r.b));
    e->prof_ms[r.cls] += t;
    e->prof_n[r.cls] += 1;
    e->prof_pool.push_back(r.a);
    e->prof_pool.push_back(r.b);
  }
  e->prof_pending.clear();
  for (int i = 0; i < PNB_NUM_KERNEL_CLASSES; i++) {
    ms[i] = e->prof_ms[i]; counts[i] = e->prof_n[i];
    e->prof_ms[i] = 0; e->prof_n[i] = 0;
  }
  return PNB_OK;
}
// Every launch of the profiled calls as (class, start, end) in ms relative to the first launch, in launch order;
// consumes the pending records like pnb_profile_read.  Returns the number of records written (<= cap) or a negative error.
extern "C" int pnb_profile_timeline(pnb_engine *e, int *cls, double *t0_ms, double *t1_ms, int cap) {
  if (!e || !cls || !t0_ms || !t1_ms) return fail(PNB_ERR_ARG, "NULL argument");
  CK(cudaSetDevice(e->device));
  CK(cudaDeviceSynchronize());
  int n = 0;
  for (auto &r : e->prof_pending) {
    if (n < cap) {
      float a = 0.f, b = 0.f;
      CK(cudaEventElapsedTime(&a, e->prof_pending[0].a, r.a));
      CK(cudaEventElapsedTime(&b, e->prof_pending[0].a, r.b));
      cls[n] = r.cls; t0_ms[n] = a; t1_ms[n] = b;
      n++;
    }
    e->prof_pool.push_back(r.a);
    e->prof_pool.push_back(r.b);
  }
  e->prof_pending.clear();
  return n;
}
extern "C" const char *pnb_kernel_class_name(int cls) {
  static const char *names[PNB_NUM_KERNEL_CLASSES] = {"stage_in_kernel", "analysis_kernel", "fc_f32_kernel",
      "gemm_f32_kernel", "f32_carry_kernel", "synthesis_kernel", "slide_history_kernel", "tc_gemm_kernel", "tc_aux_kernel", "train_labels_kernel"};
  return (cls >= 0 && cls < PNB_NUM_KERNEL_CLASSES) ? names[cls] : "?";
}

// ------------------------------------------------------------------------------------------
// The next call's window starts n_frames*480 samples further on; when it would not fit any more, the last 5280
// samples are moved back to the start of the rows.
static void advance_line(pnb_engine *e, int F, cudaStream_t st) {
  e->line_off += (size_t)F * kFrame;
  if (e->line_off + kKeep + (size_t)e->Fmax * kFrame <= e->pcm_stride) return;
  {
    LaunchScope m(e, PNB_K_SLIDE, st);
    launch_slide_history(e->d_pcm, e->pcm_stride, e->n_active, (int)e->line_off, st);  // inactive rows: no state to keep
  }
  e->line_off = 0;
}

static AnalysisArgs analysis_args(pnb_engine *e, int F) {
  AnalysisArgs a;
  a.pcm = e->d_pcm + e->line_off;  // this call's [history | new hops] window of every row
  a.pcm_stride = e->pcm_stride; a.n_streams = e->n_active; a.stride = e->S; a.n_frames = F; a.tab = e->d_tab;
  a.feat = e->d_feat; a.zring = e->d_zring; a.ering = e->d_ering; a.ring = e->ring; a.hop0 = e->hop;
  a.P = e->d_P; a.P_rows = e->n_active; a.Ex = e->d_Ex; a.raw = nullptr; a.silence = e->d_sil;
  a.last_period = e->d_last_period; a.last_gain = e->d_last_gain;
  a.tap_pitch = e->d_tap_pitch; a.tap_pitchf = e->d_tap_pitchf;
  a.hops = nullptr;
  return a;
}
static SynthesisArgs synthesis_args(pnb_engine *e, int F, float *d_out, short *d_out16, size_t out_stride) {
  SynthesisArgs s;
  s.zring = e->d_zring; s.ring = e->ring; s.hop0 = e->hop; s.P = e->d_P; s.gr = e->d_gr;
  s.Ex = e->d_Ex; s.silence = e->d_sil; s.n_streams = e->n_active; s.stride = e->S; s.n_frames = F;
  s.tab = e->d_tab; s.synth_mem = e->d_synth;
  s.out = d_out; s.out16 = d_out16; s.out_stride = out_stride;
  s.postfilter = (e->flags & PNB_POSTFILTER) ? 1 : 0;
  s.tap_g = e->d_tap_g;
  s.row = nullptr;
  s.hops = nullptr;
  s.clamp16 = 0;
  return s;
}

// Ordering of an engine's work (see pnb_engine.h): every call and state operation makes its stream wait for the last
// one before its first launch, and marks its own end behind its last launch once all of them were accepted.
static int wait_last_call(pnb_engine *e, cudaStream_t st) {
  if (e->call_recorded) CK(cudaStreamWaitEvent(st, e->ev_call, 0));
  return PNB_OK;
}
static int mark_call_end(pnb_engine *e, cudaStream_t st) {
  CK(cudaGetLastError());
  CK(cudaEventRecord(e->ev_call, st));
  e->call_recorded = true;
  return PNB_OK;
}

// The launches of one call or state operation, in ev_call's order; returns PNB_OK or a negative error.  Their markers
// count them as they are issued.  The enqueue itself may move host-side stream state (advance_line the line offset, a
// session operation the residency plan) and part of the work may already be enqueued, so a failure after it started
// leaves the streams' state undefined: the engine is poisoned, and refuses calls and state operations until pnb_reset.
// A failed enqueue adds nothing to the launch count.
template <typename Launches>
static int enqueue_ordered(pnb_engine *e, cudaStream_t st, Launches launches) {
  const long long launches0 = e->launches;
  int rc = wait_last_call(e, st);
  if (rc == PNB_OK) rc = launches();
  if (rc == PNB_OK) rc = mark_call_end(e, st);
  if (rc != PNB_OK) {
    e->launches = launches0;
    e->poisoned = true;
  }
  return rc;
}
// Enqueues one call of F hops on st (arguments already checked) and commits the hop counter (unless commit_hop is false:
// a network call, which leaves the signal state alone, or an analysis, whose synthesis commits it) and last_frames when
// all of it was accepted.
template <typename Launches>
static int enqueue_call(pnb_engine *e, int F, cudaStream_t st, Launches launches, bool commit_hop = true) {
  if (int rc = enqueue_ordered(e, st, launches)) return rc;
  if (commit_hop) e->hop += F;
  e->last_frames = F;
  return PNB_OK;
}

// The n ints at src through the pinned, event-guarded index staging, copied on st; *dst: their device copy, valid for
// the work enqueued on st behind it (the caller's array is free again when this returns).
static int stage_ints(pnb_engine *e, const int *src, size_t n, cudaStream_t st, const int **dst) {
  const int k = e->idx_slot;
  CK(cudaEventSynchronize(e->ev_idx[k]));  // the copy out of this slot two operations ago has run
  memcpy(e->h_idx[k], src, n * sizeof(int));
  CK(cudaMemcpyAsync(e->d_idx[k], e->h_idx[k], n * sizeof(int), cudaMemcpyHostToDevice, st));
  CK(cudaEventRecord(e->ev_idx[k], st));
  e->idx_slot = k ^ 1;
  *dst = e->d_idx[k];
  return PNB_OK;
}

// What the state kernels of every slot and session operation share: the pieces of a slot at the counters committed by
// the last call, the import verdicts and status word, and the parking area of a session pool (null without one).
static StateArgs state_args(pnb_engine *e) {
  StateArgs a;
  memset(&a, 0, sizeof a);
  a.n_seg = state_segs(e, a.seg);
  a.park = e->d_park;
  a.park_stride = kParkStride;
  a.ok = e->d_ok;
  a.status = e->d_status;
  a.has_terms = (e->flags & PNB_NN_TENSOR) ? 1u : 0u;
  a.check_gru = (e->flags & PNB_NN_TENSOR) ? 1 : 0;
  return a;
}

// The per-slot part of a ragged session call on the device: hops[p] of slot p, and the slots that stop before the
// call's last hop.  All null / 0 for every other call.
struct RaggedSlots {
  const int *hops = nullptr;
  const int *slots = nullptr;
  int n_short = 0;
};

// The rows of a session call on the device, one upload: the row map (list row of slot p), for a split or network call
// the slot map (slot of list row i: their layout kernels walk the caller's rows), and for a ragged call the hops of
// every slot and the slots with fewer than F.  n_up: the ints of that upload, [row][slot][hops][short slots].
struct SessionRows {
  const int *row = nullptr;
  const int *slot = nullptr;
  RaggedSlots rg;
  size_t n_up = 0;
};
static void point_rows(const int *d, int k, bool with_slot, bool ragged, size_t n_up, SessionRows *r) {
  size_t at = (size_t)k;
  r->row = d;
  if (with_slot) { r->slot = d + at; at += k; }
  if (ragged) {
    r->rg.hops = d + at;
    r->rg.slots = d + at + k;
    r->rg.n_short = (int)(n_up - at - k);
  }
  r->n_up = n_up;
}

// A session call's residency plan, applied (pnb_session_plan.h), its upload (the rows of SessionRows, then the moves
// 16-byte aligned), and its state launch when membership changed.  Sets the active range to the list; *r: the rows on
// the device.
static int enqueue_plan(pnb_engine *e, const int *ids, int k, const int *hops, int F, bool with_slot, cudaStream_t st,
                        SessionRows *r) {
  StateArgs a = state_args(e);  // before the plan: parking reads the pieces where the last call left them
  e->pool.plan(ids, k, e->plan_row, e->plan_moves);
  e->n_active = k;
  std::vector<int> &up = e->plan_up;
  up.assign(e->plan_row.begin(), e->plan_row.end());
  if (with_slot) {
    up.resize(2 * (size_t)k);
    for (int p = 0; p < k; p++) up[k + e->plan_row[p]] = p;
  }
  if (hops) {  // slot p runs the hops of its list row; then the slots that stop early
    for (int p = 0; p < k; p++) up.push_back(hops[e->plan_row[p]]);
    for (int p = 0; p < k; p++)
      if (hops[e->plan_row[p]] < F) up.push_back(p);
  }
  const size_t n_up = up.size();
  up.resize((n_up + 3) & ~(size_t)3, 0);  // the moves start 16-byte aligned
  const size_t at_moves = up.size();
  const int *mv = reinterpret_cast<const int *>(e->plan_moves.data());
  up.insert(up.end(), mv, mv + 4 * e->plan_moves.size());
  const int *d = nullptr;
  { int rc = stage_ints(e, up.data(), up.size(), st, &d); if (rc) return rc; }
  point_rows(d, k, with_slot, hops != nullptr, n_up, r);
  if (e->plan_moves.empty()) return PNB_OK;
  a.n = (int)e->plan_moves.size();
  a.moves = d + at_moves;
  LaunchScope m(e, kUnprofiled, st);
  launch_session_move(a, st);
  return PNB_OK;
}

// The rows of the pending session split, from its host copy (pnb_engine::pending.up): nothing is planned again.
static int stage_pending_rows(pnb_engine *e, cudaStream_t st, SessionRows *r) {
  const pnb_engine::PendingSplit &p = e->pending;
  const int *d = nullptr;
  { int rc = stage_ints(e, p.up.data(), p.up.size(), st, &d); if (rc) return rc; }
  point_rows(d, (int)p.ids.size(), true, !p.hops.empty(), p.up.size(), r);
  return PNB_OK;
}

// A session export into the caller's blobs (a: their address and stride): resident sessions from their slots
// (session_move_kernel), parked ones from their parking blobs (session_blob_kernel); nothing moves.  Its upload is
// [moves of the resident ones][ids of the parked ones][their rows].
static int enqueue_session_export(pnb_engine *e, const int *ids, int n, StateArgs a, cudaStream_t st) {
  std::vector<int> &up = e->plan_up;
  up.clear();
  std::vector<int> parked, rows;
  for (int i = 0; i < n; i++) {
    const int s = e->pool.where[ids[i]];
    if (s >= 0) up.insert(up.end(), {s, i, kFillNone, -1});
    else { parked.push_back(ids[i]); rows.push_back(i); }
  }
  const int r = (int)up.size() / 4, p = (int)parked.size();
  up.insert(up.end(), parked.begin(), parked.end());
  up.insert(up.end(), rows.begin(), rows.end());
  const int *d = nullptr;
  { int rc = stage_ints(e, up.data(), up.size(), st, &d); if (rc) return rc; }
  if (r) {
    a.n = r; a.moves = d;
    LaunchScope m(e, kUnprofiled, st);
    launch_session_move(a, st);
  }
  if (p) {
    a.n = p; a.streams = d + 4 * r; a.rows = d + 4 * r + p;
    LaunchScope m(e, kUnprofiled, st);
    launch_session_blob(a, st);
  }
  return PNB_OK;
}

// One stream-state operation (reset, export or import: mode) as its entry point received it.
struct StateOp {
  int mode;
  const int *list;     // n slots, or session ids when sessions (host)
  int n;
  void *blobs;         // blob i at blobs + i * blob_stride; a reset has none
  size_t blob_stride;
  bool sessions;
};

// Enqueues one state operation on st (arguments already checked), after every call and state operation issued earlier
// on the engine and before every one issued later.  Slots: the list through the index staging, the blob check of an
// import, the move.  Sessions: an export as enqueue_session_export; a reset or an import takes the sessions out of
// their slots on the host, then stages the ids, checks the blobs of an import and rewrites their parking blobs.
static int enqueue_state(pnb_engine *e, const StateOp &op, cudaStream_t st) {
  return enqueue_ordered(e, st, [&]() -> int {
    StateArgs a = state_args(e);
    a.mode = op.mode;
    a.blobs = static_cast<char *>(op.blobs);
    a.blob_stride = op.blob_stride;
    if (op.sessions && op.mode == kStateExport) return enqueue_session_export(e, op.list, op.n, a, st);
    if (op.sessions)
      for (int i = 0; i < op.n; i++) e->pool.evict(op.list[i]);
    { int rc = stage_ints(e, op.list, (size_t)op.n, st, &a.streams); if (rc) return rc; }
    a.n = op.n;
    if (op.mode == kStateImport) {  // a session import reports session ids
      LaunchScope m(e, kUnprofiled, st);
      launch_state_check(a, st);
    }
    LaunchScope m(e, kUnprofiled, st);
    if (op.sessions) launch_session_blob(a, st);
    else launch_state_move(a, st);
    return PNB_OK;
  });
}

// One array of a call's rows, in host or device memory by entry point: row r at p + r * stride values of `bytes` bytes
// each, `width` values per hop, or `width` values whatever the hops (per_row: a score call's sums).  `name` is the
// stride's name in its refusal.  width 0: the call has no such array.
struct Rows {
  void *p;
  size_t stride, width, bytes;
  const char *name;
  bool per_row;
  size_t values(int F) const { return per_row ? width : (size_t)F * width; }  // the values of a row of an F-hop call
};
static Rows rows(const void *p, size_t stride, size_t width, size_t bytes, const char *name = "row stride", bool per_row = false) {
  return {const_cast<void *>(p), stride, width, bytes, name, per_row};
}
template <typename T>
static Rows pcm(const T *p, size_t stride) { return rows(p, stride, kFrame, sizeof(T)); }

// One call as its entry point received it, its buffers as row arrays.  In / out: PCM / PCM of a slot, session or ragged
// call; speech, noisy / records and (pnb_train_audio_*) audio of a training-record call; features or records / g/r of a
// network call; records / g/r (when asked for) and the loss sums of a score call; PCM / features of an analysis; g/r /
// PCM of a synthesis; - / the operands of the pending synthesis (kOperands); features / g/r of a training forward; dL/d(out) / dL/dx (when asked for) of a training backward.  An analysis, synthesis or network call on a session list (pool) has ids too; its analysis and
// network forms may have hops.
struct Call {
  enum Kind { kSlots, kSessions, kRagged, kNetwork, kRecords, kAnalyze, kSynthesize, kOperands, kTrain, kTrainForward,
              kTrainBackward } kind;
  Rows in[2], out[2];
  int F;           // hops; a ragged call's is max(hops), set by check_call
  float *gr;       // enhancement calls: g/r destination [F][rows][68], or null
  const int *ids;  // session, ragged and pool calls: the session list (host), n_ids long
  int n_ids;
  const int *hops;    // ragged and pool calls: each listed session's hops (host), or null; null once check_call finds
                      // them all equal to F
  int format;         // network calls: PNB_RNN_FEATURES or PNB_RNN_RECORDS
  const int *frames;  // score and gradient calls: the hops each row's loss counts (host), or null for F; a training
                      // forward: each window's hops (lengths)
  bool status = true;  // a blocking host call reads back and reports the status word (rejected imports, PNB_ERR_DOMAIN)
  bool pool = false;   // an analysis, synthesis or network call on a session list (pnb_*_sessions_*)
  const float *weights = nullptr;  // a training forward: the parameters in blob order (device), or null
  float *grad = nullptr;           // a training backward: the gradient's destination in blob order (device), or null
};

// The rows of a call on st, *r: nothing for a slot call; on a session list the pending session split's rows staged
// again (the same list: nothing moves mid-hop), or else the call's residency plan applied, with the slot map for a
// split or network call.
static int call_rows(pnb_engine *e, const Call &c, cudaStream_t st, SessionRows *r) {
  if (!c.ids) return PNB_OK;
  if (e->pending.F) return stage_pending_rows(e, st, r);
  return enqueue_plan(e, c.ids, c.n_ids, c.hops, c.F, c.pool, st, r);
}

// The network hook of the engine's path for a call of F hops (hops: a ragged call's per-slot hops, or null).
static int network(pnb_engine *e, int F, const int *hops, cudaStream_t st) {
  return (e->flags & PNB_NN_TENSOR) ? tc_network(e, F, hops, st) : f32_network(e, F, hops, st);
}

// The signal path before the network, on st: the caller's PCM rows (in) into the history line, then the analysis of F
// hops into d_feat, over the active slots and through a session call's row map and per-slot hops (r; null for slots).
static int analysis_half(pnb_engine *e, const Rows &in, int F, const SessionRows &r, cudaStream_t st) {
  const bool i16 = in.bytes == sizeof(short);
  {
    LaunchScope m(e, PNB_K_STAGE_IN, st);
    launch_stage_in(e->d_pcm + e->line_off, e->pcm_stride, i16 ? nullptr : static_cast<const float *>(in.p),
                    i16 ? static_cast<const short *>(in.p) : nullptr, in.stride, e->n_active, F * kFrame, st, 32768.f,
                    r.row, r.rg.hops);
  }
  {
    AnalysisArgs aa = analysis_args(e, F);
    aa.hops = r.rg.hops;
    LaunchScope m(e, PNB_K_ANALYSIS, st);
    launch_analysis(aa, st);
  }
  CK(cudaGetLastError());
  return PNB_OK;
}

// The signal path after the network, on st, from the g/r in d_gr: the synthesis of F hops into the caller's PCM rows
// (out), through r as analysis_half, then the fix-up of the slots that stop short, then the history slide when it falls
// due.  The fix-up runs before the slide, which moves the window the counters of hop F point at.
static void synthesis_half(pnb_engine *e, const Rows &out, int F, const SessionRows &r, cudaStream_t st) {
  const bool i16 = out.bytes == sizeof(short);
  {
    SynthesisArgs sa = synthesis_args(e, F, i16 ? nullptr : static_cast<float *>(out.p),
                                      i16 ? static_cast<short *>(out.p) : nullptr, out.stride);
    sa.row = r.row;
    sa.hops = r.rg.hops;
    LaunchScope m(e, PNB_K_SYNTHESIS, st);
    launch_synthesis(sa, st);
  }
  if (r.rg.n_short) {
    LaunchScope m(e, PNB_K_SLIDE, st);
    launch_ragged_carry(e, F, r.rg.hops, r.rg.slots, r.rg.n_short, st);
  }
  advance_line(e, F, st);
}

// A network call on st (arguments already checked): the caller's rows into the features buffer, the network hook, its
// g/r out to the caller's rows; a score call reduces the loss from the same g/r and writes g/r only when asked.  The
// signal state (history line, overlap-add, pitch memory, spectrum ring, hop counter, line offset) is not touched.  On a
// session list row i of the caller's arrays is ids[i]'s (call_rows), and a ragged call's frozen hops stage and store
// zeros.
static int enqueue_network(pnb_engine *e, const Call &c, cudaStream_t st) {
  const int F = c.F;
  const Rows &in = c.in[0], &gr = c.out[0], &sums = c.out[1];
  return enqueue_call(e, F, st, [&]() -> int {
    SessionRows r;
    if (int rc = call_rows(e, c, st, &r)) return rc;
    const int S = e->S, na = e->n_active;
    const int *frames = nullptr;  // a score call's per-row hop counts, staged like a ragged call's hops
    if (c.frames) { int rc = stage_ints(e, c.frames, (size_t)na, st, &frames); if (rc) return rc; }
    {
      LaunchScope m(e, PNB_K_STAGE_IN, st);
      launch_rows_stage(e->d_feat, kFeat, static_cast<const float *>(in.p), in.stride, (int)in.width,
                        c.format == PNB_RNN_RECORDS ? 68 : 0, na, S, F, st, r.row, r.rg.hops);
    }
    CK(cudaGetLastError());
    if (int rc = network(e, F, r.rg.hops, st)) return rc;
    if (sums.p) {
      LaunchScope m(e, PNB_K_STAGE_IN, st);
      launch_loss_sums(e->d_gr, static_cast<const float *>(in.p), in.stride, frames, static_cast<double *>(sums.p), na, S, F, st);
    }
    if (gr.p) {
      LaunchScope m(e, PNB_K_STAGE_IN, st);
      launch_rows_store(e->d_gr, 68, static_cast<float *>(gr.p), gr.stride, na, S, F, st, r.slot, r.rg.hops);
    }
    return PNB_OK;
  }, false);
}

// One training-record call on st (arguments already checked), the training-data generator (row f1): stage both files of
// every pair, analysis over 2N streams, labels; with audio (a PNB_TRAIN_AUDIO engine) then the resynthesis of the N
// noisy streams with their labels.
static int enqueue_records(pnb_engine *e, const Call &c, cudaStream_t st) {
  const int F = c.F;
  const Rows &speech = c.in[0], &noisy = c.in[1], &records = c.out[0], &audio = c.out[1];
  return enqueue_call(e, F, st, [&]() -> int {
    const int N = e->S / 2;
    float *line = e->d_pcm + e->line_off;
    {
      LaunchScope m(e, PNB_K_STAGE_IN, st);
      launch_stage_in(line, e->pcm_stride, nullptr, static_cast<const short *>(noisy.p), noisy.stride, N, F * kFrame, st, 1.f);
    }
    {
      LaunchScope m(e, PNB_K_STAGE_IN, st);
      launch_stage_in(line + (size_t)N * e->pcm_stride, e->pcm_stride, nullptr, static_cast<const short *>(speech.p),
                      speech.stride, N, F * kFrame, st, 1.f);
    }
    AnalysisArgs a = analysis_args(e, F);  // all S streams: the active range of a training-data engine is always S
    a.raw = e->d_raw;
    a.P_rows = N;  // an audio engine's P: the noisy rows (the others have none)
    { LaunchScope m(e, PNB_K_ANALYSIS, st); launch_analysis(a, st); }
    LabelArgs l;
    l.feat = e->d_feat; l.raw = e->d_raw; l.Ex = e->d_Ex; l.tab = e->d_tab; l.n_pairs = N; l.n_frames = F;
    l.records = static_cast<float *>(records.p); l.pair_stride = records.stride;
    l.gr = audio.p ? e->d_gr : nullptr;
    { LaunchScope m(e, PNB_K_LABELS, st); launch_train_labels(l, st); }
    if (audio.p) {  // denoise.cpp:742-759 on the noisy rows, their labels post-filtered already (no PNB_POSTFILTER here)
      SynthesisArgs s = synthesis_args(e, F, nullptr, static_cast<short *>(audio.p), audio.stride);
      s.n_streams = N;
      s.clamp16 = 1;
      LaunchScope m(e, PNB_K_SYNTHESIS, st);
      launch_synthesis(s, st);
    }
    advance_line(e, F, st);
    return PNB_OK;
  });
}

// One enhancement call on st, its buffers on the device (arguments already checked): the analysis half, the network,
// the synthesis half.  A session call first applies its residency plan, and reads input row / writes output row and
// g/r row row[p] for slot p.  With hops (a ragged call) slot p runs the hops of its list row, and the slots that stop
// early are moved to the counters of hop F after synthesis.
static int enqueue_enhance(pnb_engine *e, const Call &c, cudaStream_t st) {
  const int F = c.F;
  return enqueue_call(e, F, st, [&]() -> int {
    SessionRows r;
    if (int rc = call_rows(e, c, st, &r)) return rc;
    if (int rc = analysis_half(e, c.in[0], F, r, st)) return rc;
    if (int rc = network(e, F, r.rg.hops, st)) return rc;
    synthesis_half(e, c.out[0], F, r, st);
    const int S = e->S, na = e->n_active;  // the call advances streams [0, na); per-call buffers keep the stride S
    if (c.gr && r.row) {  // [F][na][68] in list order
      LaunchScope m(e, kUnprofiled, st);
      launch_gr_gather(e->d_gr, c.gr, r.row, na, S, F, st, r.rg.hops);
    } else if (c.gr) {  // [F][na][68] from the [F][S][68] buffer
      CK(cudaMemcpy2DAsync(c.gr, (size_t)na * 68 * sizeof(float), e->d_gr, (size_t)S * 68 * sizeof(float), (size_t)na * 68 * sizeof(float), F,
                           cudaMemcpyDeviceToDevice, st));
    }
    return PNB_OK;
  });
}

// An analysis on st (arguments already checked): the rows of the call and the analysis half, as enqueue_enhance runs
// them, then the features out to the caller's rows.  Nothing bound to the hop counter or the line offset moves: the
// analysis and synthesis kernels both take hop0 = e->hop, and the synthesis that completes these hops runs the rest of
// the fused call and commits them.  The pending split keeps the hops and, on a session list, the list and the rows of
// its upload.
static int enqueue_analyze(pnb_engine *e, const Call &c, cudaStream_t st) {
  const int F = c.F;
  const Rows &feat = c.out[0];
  SessionRows r;
  const int rc = enqueue_call(e, F, st, [&]() -> int {
    if (int rc = call_rows(e, c, st, &r)) return rc;
    if (int rc = analysis_half(e, c.in[0], F, r, st)) return rc;
    LaunchScope m(e, PNB_K_STAGE_IN, st);
    launch_rows_store(e->d_feat, kFeat, static_cast<float *>(feat.p), feat.stride, e->n_active, e->S, F, st, r.slot, r.rg.hops);
    return PNB_OK;
  }, false);
  if (rc == PNB_OK)
    e->pending = {F, std::vector<int>(c.ids, c.ids + c.n_ids),
                  c.hops ? std::vector<int>(c.hops, c.hops + c.n_ids) : std::vector<int>(),
                  std::vector<int>(e->plan_up.begin(), e->plan_up.begin() + r.n_up)};
  return rc;
}

// A synthesis on st (arguments already checked, an analysis of F hops pending): the rows of the call, the caller's g/r
// rows into d_gr where the network hook would have left them, then the synthesis half of enqueue_enhance, which commits
// the hop counter.
static int enqueue_synthesize(pnb_engine *e, const Call &c, cudaStream_t st) {
  const int F = c.F;
  const Rows &gr = c.in[0];
  const int rc = enqueue_call(e, F, st, [&]() -> int {
    SessionRows r;
    if (int rc = call_rows(e, c, st, &r)) return rc;
    {
      LaunchScope m(e, PNB_K_STAGE_IN, st);
      launch_rows_stage(e->d_gr, 68, static_cast<const float *>(gr.p), gr.stride, 68, 0, e->n_active, e->S, F, st, r.row,
                        r.rg.hops);
    }
    synthesis_half(e, c.out[0], F, r, st);
    return PNB_OK;
  });
  if (rc == PNB_OK) e->pending = {};
  return rc;
}

// The operands of the pending synthesis on st (arguments already checked, an analysis of F hops pending): one launch
// that reads what synthesis_kernel will read, through the same SynthesisArgs.  Neither the signal state, the hop counter
// nor the pending synthesis changes, so it is ordered like a call but commits nothing.
static int enqueue_operands(pnb_engine *e, const Call &c, cudaStream_t st) {
  const Rows &ops = c.out[0];
  return enqueue_ordered(e, st, [&]() -> int {
    const SynthesisArgs sa = synthesis_args(e, c.F, nullptr, nullptr, 0);
    LaunchScope m(e, PNB_K_STAGE_IN, st);
    launch_synth_ops(sa, static_cast<float *>(ops.p), ops.stride, st);
    return PNB_OK;
  });
}

// A gradient call on st (arguments already checked): the trainer's forward, loss and backward on the records of windows
// [0, n_active), each from zero state; the loss sums to the caller, the gradient into the engine's buffer.  Neither the
// network state of the slots nor the signal state is touched.
static int enqueue_train(pnb_engine *e, const Call &c, cudaStream_t st) {
  e->train_fwd_F = 0;
  return enqueue_call(e, c.F, st, [&]() -> int {
    const int *frames = nullptr;
    if (c.frames) { int rc = stage_ints(e, c.frames, (size_t)e->n_active, st, &frames); if (rc) return rc; }
    return train_grad(e, static_cast<const float *>(c.in[0].p), c.in[0].stride, frames, c.frames,
                      static_cast<double *>(c.out[1].p), c.F, st);
  }, false);
}

// A training forward on st (arguments already checked): the caller's features through the trainer's forward half on
// windows [0, n_active), its g/r out; its backward becomes due.  A training backward (arguments checked, so a forward of
// F hops is due): the caller's dL/d(out) through the backward half into the held gradient, dL/dx out when asked for.
// Either may carry network state: a forward's state in / state out rows and per-window lengths (c.frames), a backward's
// dL/d(state out) / dL/d(state in) rows (in[1] / out[1], null when absent).
static int enqueue_train_forward(pnb_engine *e, const Call &c, cudaStream_t st) {
  e->train_fwd_F = 0;
  const int rc = enqueue_call(e, c.F, st, [&]() -> int {
    const int *lengths = nullptr;
    if (c.frames) { int rc = stage_ints(e, c.frames, (size_t)e->n_active, st, &lengths); if (rc) return rc; }
    return train_forward(e, static_cast<const float *>(c.in[0].p), c.in[0].stride, c.weights,
                         static_cast<const float *>(c.in[1].p), c.in[1].stride, lengths, c.frames,
                         static_cast<float *>(c.out[0].p), c.out[0].stride, static_cast<float *>(c.out[1].p),
                         c.out[1].stride, c.F, st);
  }, false);
  if (rc == PNB_OK) e->train_fwd_F = c.F;
  return rc;
}
static int enqueue_train_backward(pnb_engine *e, const Call &c, cudaStream_t st) {
  e->train_fwd_F = 0;
  return enqueue_call(e, c.F, st, [&]() -> int {
    return train_backward(e, static_cast<const float *>(c.in[0].p), c.in[0].stride,
                          static_cast<const float *>(c.in[1].p), c.in[1].stride, static_cast<float *>(c.out[0].p),
                          c.out[0].stride, static_cast<float *>(c.out[1].p), c.out[1].stride, c.grad, st);
  }, false);
}

// The call's enqueue body (arguments already checked).
static int enqueue(pnb_engine *e, const Call &c, cudaStream_t st) {
  switch (c.kind) {
    case Call::kNetwork: return enqueue_network(e, c, st);
    case Call::kRecords: return enqueue_records(e, c, st);
    case Call::kAnalyze: return enqueue_analyze(e, c, st);
    case Call::kSynthesize: return enqueue_synthesize(e, c, st);
    case Call::kOperands: return enqueue_operands(e, c, st);
    case Call::kTrain: return enqueue_train(e, c, st);
    case Call::kTrainForward: return enqueue_train_forward(e, c, st);
    case Call::kTrainBackward: return enqueue_train_backward(e, c, st);
    default: return enqueue_enhance(e, c, st);
  }
}

// Every call and state operation but pnb_synthesize_* and the network calls, while an analysis waits for its synthesis:
// a stream's state between the halves is mid-hop (its overlap-add memory lags its history), and no blob may capture it.
static int refuse_pending(const pnb_engine *e) {
  return fail(PNB_ERR_ARG, "a synthesis is pending (pnb_analyze_* of %d hops): call pnb_synthesize_* with the same n_frames, or pnb_reset",
              e->pending.F);
}

// The slot-level entry points of an engine in session mode: refused before anything is enqueued.
static int refuse_in_session_mode() {
  return fail(PNB_ERR_ARG, "engine is in session mode (pnb_sessions_reserve): slots are the pool's; use the *_sessions entry points");
}

// Every call and state operation of a poisoned engine (enqueue_ordered), with the code its entry point documents.
static int refuse_poisoned(int code) {
  return fail(code, "an earlier call failed while enqueuing work; the streams' state is undefined until pnb_reset");
}

// The entries of a slot or session list, the argument `name`: each in [0, end) and in the active range [0, active) (a
// session list passes active = end), none listed twice.  Repeats are found with the session pool's scratch, which is -1
// everywhere between calls; a slot list of an engine without a pool grows it to the number of slots.
static int check_list(pnb_engine *e, const int *list, int n, int end, int active, const char *name) {
  for (int i = 0; i < n; i++) {
    if (list[i] < 0 || list[i] >= end) return fail(PNB_ERR_ARG, "%s[%d] = %d outside [0, %d)", name, i, list[i], end);
    if (list[i] >= active) return fail(PNB_ERR_ARG, "%s[%d] = %d outside the active range [0, %d)", name, i, list[i], active);
  }
  if (e->pool.listed.size() < (size_t)end) e->pool.listed.resize(end, -1);
  const int d = e->pool.duplicate(list, n);
  if (d >= 0) return fail(PNB_ERR_ARG, "%s[%d] = %d listed twice", name, d, list[d]);
  return PNB_OK;
}

// A session list: after pnb_sessions_reserve, n in [1, n_max], distinct ids in [0, capacity).
static int check_ids(pnb_engine *e, const int *ids, int n, int n_max) {
  if (!e->sessions) return fail(PNB_ERR_ARG, "no session pool: call pnb_sessions_reserve first");
  if (!ids) return fail(PNB_ERR_ARG, "ids is NULL");
  if (n < 1 || n > n_max) return fail(PNB_ERR_ARG, "n = %d sessions outside [1, %d]", n, n_max);
  return check_list(e, ids, n, e->pool.capacity(), e->pool.capacity(), "ids");
}

// The stride refusal of each of the arrays: a row of F hops fits in its stride.
static int check_strides(const Rows (&a)[2], int F) {
  for (const Rows &r : a)
    if (r.width && r.stride < r.values(F))
      return r.per_row ? fail(PNB_ERR_ARG, "%s smaller than %zu", r.name, r.width)
                       : fail(PNB_ERR_ARG, "%s smaller than n_frames*%zu", r.name, r.width);
  return PNB_OK;
}

// A call on a session list while a session split is pending: the pending list in its order and n_frames, and for a
// network call (which passes hops) the pending hops.
static int check_pending_list(const pnb_engine *e, const Call &c) {
  const std::vector<int> &ids = e->pending.ids, &hops = e->pending.hops;
  bool same = c.n_ids == (int)ids.size() && c.F == e->pending.F && std::equal(ids.begin(), ids.end(), c.ids);
  if (same && c.kind == Call::kNetwork)
    same = c.hops ? !hops.empty() && std::equal(hops.begin(), hops.end(), c.hops) : hops.empty();
  if (!same)
    return fail(PNB_ERR_ARG, "a session split of %d sessions and %d hops is pending: pass its list in the same order, its n_frames%s",
                (int)ids.size(), e->pending.F, c.kind == Call::kNetwork ? " and its hops" : "");
  return PNB_OK;
}

// Every refusal of a call, before anything changes.  Every call checks an engine of its family (training records,
// enhancement or the network alone; a PNB_NETWORK_ONLY engine runs network calls only, a PNB_SIGNAL_ONLY engine split
// calls only) that no failed call has poisoned, 1 <= F <= Fmax, none of its arrays NULL, the input strides; a
// training-record call then that its engine has audio exactly when the call does; every call then the output strides,
// and the pending synthesis: a synthesis needs one of F hops (on a session list: the pending list), an operand export one
// whose hops it takes, a network call on a
// session list while one is pending the pending list and hops, every other call but a network call none.  After that a
// slot or split call checks session mode, a session call its list, a network call its format, then session mode, and a
// score call its frames.  A ragged call, and a split or network call on a session list, checks the list first (so
// session mode) and then the hop counts, because their largest is a ragged call's length F and must be a pool call's
// n_frames; when every session runs F hops, hops becomes null and the call is the call without hops.
static int check_call(pnb_engine *e, Call &c) {
  if (c.kind == Call::kRagged || c.pool) {
    if (!e) return fail(PNB_ERR_ARG, "engine is NULL");
    { int rc = check_ids(e, c.ids, c.n_ids, e->S); if (rc) return rc; }
    if (c.kind == Call::kRagged && !c.hops) return fail(PNB_ERR_ARG, "hops is NULL");
  }
  if (c.hops) {
    int F = 0;
    for (int i = 0; i < c.n_ids; i++) {
      if (c.hops[i] < 1 || c.hops[i] > e->Fmax) return fail(PNB_ERR_ARG, "hops[%d] = %d outside [1, %d]", i, c.hops[i], e->Fmax);
      F = c.hops[i] > F ? c.hops[i] : F;
    }
    if (c.kind == Call::kRagged) c.F = F;
    else if (c.F != F) return fail(PNB_ERR_ARG, "n_frames %d, but max(hops) = %d", c.F, F);
    bool uniform = true;
    for (int i = 0; i < c.n_ids; i++) uniform = uniform && c.hops[i] == c.F;
    if (uniform) c.hops = nullptr;
  }
  const bool trainer = c.kind == Call::kTrain || c.kind == Call::kTrainForward || c.kind == Call::kTrainBackward;
  const bool train = c.kind == Call::kRecords, network = c.kind == Call::kNetwork || trainer;
  const bool split = c.kind == Call::kAnalyze || c.kind == Call::kSynthesize || c.kind == Call::kOperands;
  if (!e) return fail(PNB_ERR_ARG, "engine is NULL");
  if (!network && (e->flags & PNB_NETWORK_ONLY))
    return fail(PNB_ERR_ARG, "engine was created with PNB_NETWORK_ONLY: use pnb_compute_rnn_* / pnb_score_records_*");
  if (!split && (e->flags & PNB_SIGNAL_ONLY))
    return fail(PNB_ERR_ARG, "engine was created with PNB_SIGNAL_ONLY: use pnb_analyze_* / pnb_synthesize_*");
  if (trainer && !(e->flags & PNB_TRAIN_NETWORK)) return fail(PNB_ERR_ARG, "engine was not created with PNB_TRAIN_NETWORK");
  if (c.kind == Call::kTrainBackward) {  // the hops of the forward it differentiates
    if (!e->train_fwd_F)
      return fail(PNB_ERR_ARG, "no pnb_train_forward_device call awaits its backward (one backward per forward; "
                               "pnb_reset, pnb_set_active_streams, pnb_train_grad_*, pnb_train_adam and "
                               "pnb_train_import of the weights end a forward's wait)");
    c.F = e->train_fwd_F;
  }
  if (train && !(e->flags & PNB_TRAIN_DATA)) return fail(PNB_ERR_ARG, "engine was not created with PNB_TRAIN_DATA");
  if (!train && (e->flags & PNB_TRAIN_DATA))
    return fail(PNB_ERR_ARG, "engine was created with PNB_TRAIN_DATA: use pnb_train_records_* / pnb_submit_train_records");
  if (e->poisoned) return refuse_poisoned(PNB_ERR_CUDA);
  if (c.kind == Call::kOperands) {  // the hops of the pending synthesis
    if (!e->pending.F) return fail(PNB_ERR_ARG, "no analysis awaits its synthesis: call pnb_analyze_* first");
    c.F = e->pending.F;
  }
  if (c.F < 1 || c.F > e->Fmax) return fail(PNB_ERR_ARG, "n_frames %d outside [1, %d]", c.F, e->Fmax);
  for (int i = 0; i < 2; i++)
    if ((c.in[i].width && !c.in[i].p) || (c.out[i].width && !c.out[i].p))
      return fail(PNB_ERR_ARG, train ? "speech/noisy/records pointer is NULL" : "input/output pointer is NULL");
  { int rc = check_strides(c.in, c.F); if (rc) return rc; }
  const bool audio = c.out[1].width != 0;
  if (train && audio && !(e->flags & PNB_TRAIN_AUDIO)) return fail(PNB_ERR_ARG, "engine was not created with PNB_TRAIN_AUDIO");
  if (train && !audio && (e->flags & PNB_TRAIN_AUDIO))
    return fail(PNB_ERR_ARG, "engine was created with PNB_TRAIN_AUDIO: use pnb_train_audio_*, so that its audio has no gaps");
  { int rc = check_strides(c.out, c.F); if (rc) return rc; }
  if (c.kind == Call::kSynthesize || c.kind == Call::kOperands) {
    if (!e->pending.F) return fail(PNB_ERR_ARG, "no analysis awaits its synthesis: call pnb_analyze_* first");
    if (c.F != e->pending.F) return fail(PNB_ERR_ARG, "n_frames %d, but the pending analysis has %d hops", c.F, e->pending.F);
    if (c.pool) { int rc = check_pending_list(e, c); if (rc) return rc; }
  } else if (e->pending.F && !network) {
    return refuse_pending(e);
  } else if (e->pending.F && c.pool) {
    int rc = check_pending_list(e, c);
    if (rc) return rc;
  }
  if (c.kind == Call::kSessions) return check_ids(e, c.ids, c.n_ids, e->S);
  if (c.kind == Call::kNetwork && c.format != PNB_RNN_FEATURES && c.format != PNB_RNN_RECORDS)
    return fail(PNB_ERR_ARG, "format %d is neither PNB_RNN_FEATURES (0) nor PNB_RNN_RECORDS (1)", c.format);
  if ((c.kind == Call::kSlots || network || split) && !c.pool && e->sessions) return refuse_in_session_mode();
  // a window of a gradient call or a training forward has at least one hop
  const int fr_lo = c.kind == Call::kTrain || c.kind == Call::kTrainForward ? 1 : 0;
  if (c.frames)  // every row's counted hops in [fr_lo, F]
    for (int i = 0; i < e->n_active; i++)
      if (c.frames[i] < fr_lo || c.frames[i] > c.F)
        return fail(PNB_ERR_ARG, "%s[%d] = %d outside [%d, %d]", c.kind == Call::kTrainForward ? "lengths" : "frames", i,
                    c.frames[i], fr_lo, c.F);
  return PNB_OK;
}

// Every device-buffer call entry point.
static int device_call(pnb_engine *e, Call c, cudaStream_t st) {
  { int rc = check_call(e, c); if (rc) return rc; }
  CK(cudaSetDevice(e->device));
  return enqueue(e, c, st);
}

extern "C" int pnb_process_device_f32(pnb_engine *e, const float *d_in, size_t in_stride, float *d_out,
                                      size_t out_stride, int n_frames, float *d_gr, void *cuda_stream) {
  return device_call(e, {Call::kSlots, {pcm(d_in, in_stride)}, {pcm(d_out, out_stride)}, n_frames, d_gr}, (cudaStream_t)cuda_stream);
}
extern "C" int pnb_process_device_i16(pnb_engine *e, const short *d_in, size_t in_stride, short *d_out,
                                      size_t out_stride, int n_frames, float *d_gr, void *cuda_stream) {
  return device_call(e, {Call::kSlots, {pcm(d_in, in_stride)}, {pcm(d_out, out_stride)}, n_frames, d_gr}, (cudaStream_t)cuda_stream);
}
// pnb_process_device_* without g/r; both names are part of the ABI.
extern "C" int pnb_submit_device_f32(pnb_engine *e, const float *d_in, size_t in_stride, float *d_out, size_t out_stride,
                                     int n_frames, void *cuda_stream) {
  return device_call(e, {Call::kSlots, {pcm(d_in, in_stride)}, {pcm(d_out, out_stride)}, n_frames}, (cudaStream_t)cuda_stream);
}
extern "C" int pnb_submit_device_i16(pnb_engine *e, const short *d_in, size_t in_stride, short *d_out, size_t out_stride,
                                     int n_frames, void *cuda_stream) {
  return device_call(e, {Call::kSlots, {pcm(d_in, in_stride)}, {pcm(d_out, out_stride)}, n_frames}, (cudaStream_t)cuda_stream);
}

// A training-record call: int16 speech and noisy rows in, records and, for pnb_train_audio_* (with_audio), audio out.  A
// blocking host call does not read the status word: a training-data engine reports a rejected pnb_import_states through
// pnb_wait / pnb_check only.
static Call records_call(const short *speech, size_t speech_stride, const short *noisy, size_t noisy_stride, int F,
                         float *records, size_t records_stride, bool with_audio = false, short *audio = nullptr,
                         size_t audio_stride = 0) {
  Call c{Call::kRecords, {pcm(speech, speech_stride), pcm(noisy, noisy_stride)},
         {rows(records, records_stride, PNB_RECORD_FLOATS, sizeof(float), "records_stride")}, F};
  if (with_audio) c.out[1] = rows(audio, audio_stride, kFrame, sizeof(short), "audio_stride");
  c.status = false;
  return c;
}

extern "C" int pnb_train_records_device(pnb_engine *e, const short *d_speech, size_t speech_stride,
                                        const short *d_noisy, size_t noisy_stride, int F, float *d_records,
                                        size_t records_stride, void *cuda_stream) {
  return device_call(e, records_call(d_speech, speech_stride, d_noisy, noisy_stride, F, d_records, records_stride),
                     (cudaStream_t)cuda_stream);
}
extern "C" int pnb_train_audio_device(pnb_engine *e, const short *d_speech, size_t speech_stride, const short *d_noisy,
                                      size_t noisy_stride, int F, float *d_records, size_t records_stride, short *d_audio,
                                      size_t audio_stride, void *cuda_stream) {
  return device_call(e, records_call(d_speech, speech_stride, d_noisy, noisy_stride, F, d_records, records_stride, true,
                                     d_audio, audio_stride), (cudaStream_t)cuda_stream);
}

// ------------------------------------------------------------------------------------------
// host-buffer calls: device staging, and the pipeline in which the H2D of call i+1 and the D2H of call i-1 overlap the
// kernels of call i
// ------------------------------------------------------------------------------------------
// Buffers of at least `bytes`: a slot grows, never shrinks.  The slot is idle when this runs.
static int grow(void **buf, size_t *cap, size_t bytes) {
  if (*cap >= bytes) return PNB_OK;
  if (*buf) CK(cudaFree(*buf));
  *buf = nullptr;
  *cap = 0;
  CK(cudaMalloc(buf, bytes));
  *cap = bytes;
  return PNB_OK;
}

// The staging slot of a host-buffer call: k = submitted & 1, the slot the next pipelined call takes.  Only pipelined
// calls advance `submitted`, so a blocking call borrows that slot, and an engine that only makes blocking calls uses
// slot 0 alone.  Creates the copy streams and their events for the first pipelined call: blocking calls do not use
// them, and with them created a blocking 16-stream tensor engine took about 15 us (4 %) longer per call (H100 80GB HBM3,
// 700 W).  Waits until the slot's last pipelined round trip is complete, and grows its buffers to in_bytes / out_bytes.
// Callers size them for an Fmax-hop call, so a slot grows at most once however f32, int16, blocking and pipelined calls
// mix.  Returns k or a negative error.
static int staging_slot(pnb_engine *e, bool pipelined, size_t in_bytes, size_t out_bytes) {
  if (pipelined && !e->s_in) {
    CK(cudaStreamCreateWithFlags(&e->s_in, cudaStreamNonBlocking));
    CK(cudaStreamCreateWithFlags(&e->s_out, cudaStreamNonBlocking));
    for (int k = 0; k < 2; k++) {
      CK(cudaEventCreateWithFlags(&e->ev_in[k], cudaEventDisableTiming));
      CK(cudaEventCreateWithFlags(&e->ev_cmp[k], cudaEventDisableTiming));
      CK(cudaEventCreateWithFlags(&e->ev_out[k], cudaEventDisableTiming));
    }
  }
  const int k = (int)(e->submitted & 1);
  if (e->submitted >= 2) CK(cudaEventSynchronize(e->ev_out[k]));  // the slot's last pipelined round trip is complete
  pnb_engine::Staging &s = e->stage[k];
  { int rc = grow(&s.in, &s.in_bytes, in_bytes); if (rc) return rc; }
  { int rc = grow(&s.out, &s.out_bytes, out_bytes); if (rc) return rc; }
  return k;
}

// One round trip through staging slot k: h2d(stream) copies the input into the slot, call() enqueues the call on the
// engine's stream, d2h(stream) copies the output back.  Pipelined, the copies go to s_in / s_out, the slot's events
// order them with the call, and the round trip is left in flight.  Blocking, all of it goes to the engine's stream, for
// the caller to synchronise.
template <typename H2D, typename Call, typename D2H>
static int round_trip(pnb_engine *e, int k, bool pipelined, H2D h2d, Call call, D2H d2h) {
  CK(h2d(pipelined ? e->s_in : e->stream));
  if (pipelined) {
    CK(cudaEventRecord(e->ev_in[k], e->s_in));
    CK(cudaStreamWaitEvent(e->stream, e->ev_in[k], 0));
  }
  { int rc = call(); if (rc) return rc; }
  if (pipelined) {
    CK(cudaEventRecord(e->ev_cmp[k], e->stream));
    CK(cudaStreamWaitEvent(e->s_out, e->ev_cmp[k], 0));
  }
  CK(d2h(pipelined ? e->s_out : e->stream));
  if (pipelined) {
    CK(cudaEventRecord(e->ev_out[k], e->s_out));
    e->submitted++;
  }
  return PNB_OK;
}

// after the stream that carried the status copy was synchronised
static int report_status(pnb_engine *e) {
  if (e->h_status[0] & kStatusRejected) {  // reported once: no other stream was affected
    const int slot = e->h_status[1];
    launch_state_clear_reject(e->d_status, e->stream);  // uncounted: part of reporting a rejection, not of a call or state operation
    CK(cudaGetLastError());
    CK(cudaStreamSynchronize(e->stream));
    e->h_status[0] &= ~kStatusRejected;
    e->h_status[1] = kNoRejectedSlot;
    if (e->sessions)
      return fail(PNB_ERR_ARG, "pnb_import_sessions rejected a blob (bad magic / version, or a GRU state outside [-1, 1] for a "
                               "tensor-mode engine); lowest rejected session %d, left fresh like every rejected one", slot);
    return fail(PNB_ERR_ARG, "pnb_import_states rejected a blob (bad magic / version, or a GRU state outside [-1, 1] for a "
                             "tensor-mode engine); lowest rejected stream %d, left reset like every rejected one", slot);
  }
  if ((e->h_status[0] & 1) && (e->flags & PNB_TRAIN_NETWORK))
    return fail(PNB_ERR_DOMAIN, "a pnb_train_grad_* call or pnb_train_finish met a non-finite gradient (non-finite records "
                                "inside a window, non-finite weights, or a non-finite imported accumulator); the Adam step "
                                "after it was skipped.  Sticky until pnb_reset");
  if (e->h_status[0] & 1)
    return fail(PNB_ERR_DOMAIN, "tensor path: a pre-activation left the domain of the reference's tansig_approx (|x| >= 8.5e7, "
                                "src/vec.h:63 is undefined there); results since the last pnb_reset are not the reference's -- "
                                "use PNB_NN_FP32 for such input");
  return PNB_OK;
}

// Lays a call's arrays out in a staging buffer, n_rows rows each at a stride of Fmax hops: sets their strides and byte
// offsets at[i] (16-byte aligned), and returns the bytes they take.
static size_t staged_layout(Rows (&a)[2], size_t n_rows, int Fmax, size_t at[2]) {
  size_t bytes = 0;
  for (int i = 0; i < 2; i++) {
    at[i] = bytes;
    a[i].stride = a[i].values(Fmax);
    bytes += (n_rows * a[i].stride * a[i].bytes + 15) & ~(size_t)15;
  }
  return bytes;
}

// F hops of n_rows rows of each array of src into the same array of dst (absent arrays: nothing).
static cudaError_t copy_rows(const Rows (&dst)[2], const Rows (&src)[2], int F, size_t n_rows, cudaMemcpyKind kind, cudaStream_t s) {
  for (int i = 0; i < 2; i++) {
    if (!src[i].p) continue;
    const size_t b = src[i].bytes;
    const cudaError_t ce = cudaMemcpy2DAsync(dst[i].p, dst[i].stride * b, src[i].p, src[i].stride * b, src[i].values(F) * b,
                                             n_rows, kind, s);
    if (ce != cudaSuccess) return ce;
  }
  return cudaSuccess;
}

// Every host-buffer call entry point: pnb_submit_host_* and pnb_submit_train_records pipelined, the others blocking.
// Each array is staged at its place in the slot's input or output buffer, laid out for the engine's most rows (its
// pairs on a training-data engine, else its slots) at Fmax hops, so a slot grows at most once per kind of call.  The
// blocking form then copies an enhancement call's g/r and (when the call reports it) the status word back on the
// engine's stream too, and synchronises it once.  Rows travel F hops wide: a ragged call's input beyond a row's hops is
// copied but not read.
static int host_call(pnb_engine *e, Call c, bool pipelined) {
  { int rc = check_call(e, c); if (rc) return rc; }
  CK(cudaSetDevice(e->device));
  const size_t S = e->S, per = (e->flags & PNB_TRAIN_DATA) ? 2 : 1;  // a training-data engine's rows are its pairs
  const size_t na = (c.ids ? c.n_ids : e->n_active) / per;       // the rows of the arrays and of gr
  Call d = c;  // the call on staging slot k
  size_t at_in[2], at_out[2];
  const int k = staging_slot(e, pipelined, staged_layout(d.in, S / per, e->Fmax, at_in), staged_layout(d.out, S / per, e->Fmax, at_out));
  if (k < 0) return k;
  if (c.ids && c.gr) { int rc = grow((void **)&e->d_sgr, &e->sgr_bytes, (size_t)e->Fmax * S * 68 * sizeof(float)); if (rc) return rc; }
  for (int i = 0; i < 2; i++) {
    if (c.in[i].p) d.in[i].p = static_cast<char *>(e->stage[k].in) + at_in[i];
    if (c.out[i].p) d.out[i].p = static_cast<char *>(e->stage[k].out) + at_out[i];
  }
  d.gr = c.ids && c.gr ? e->d_sgr : nullptr;  // session calls gather g/r in list order on the device
  const int rc = round_trip(e, k, pipelined,
      [&](cudaStream_t s) { return copy_rows(d.in, c.in, c.F, na, cudaMemcpyHostToDevice, s); },
      [&] { return enqueue(e, d, e->stream); },
      [&](cudaStream_t s) { return copy_rows(c.out, d.out, c.F, na, cudaMemcpyDeviceToHost, s); });
  if (rc || pipelined) return rc;
  if (d.gr)
    CK(cudaMemcpyAsync(c.gr, d.gr, (size_t)c.F * na * 68 * sizeof(float), cudaMemcpyDeviceToHost, e->stream));
  else if (c.gr)
    CK(cudaMemcpy2DAsync(c.gr, na * 68 * sizeof(float), e->d_gr, S * 68 * sizeof(float), na * 68 * sizeof(float), c.F, cudaMemcpyDeviceToHost,
                         e->stream));
  if (c.status) CK(cudaMemcpyAsync(e->h_status, e->d_status, 2 * sizeof(int), cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  return c.status ? report_status(e) : PNB_OK;
}

extern "C" int pnb_process_host_f32(pnb_engine *e, const float *in, size_t in_stride, float *out, size_t out_stride,
                                    int n_frames, float *gr) {
  return host_call(e, {Call::kSlots, {pcm(in, in_stride)}, {pcm(out, out_stride)}, n_frames, gr}, false);
}
extern "C" int pnb_process_host_i16(pnb_engine *e, const short *in, size_t in_stride, short *out, size_t out_stride,
                                    int n_frames, float *gr) {
  return host_call(e, {Call::kSlots, {pcm(in, in_stride)}, {pcm(out, out_stride)}, n_frames, gr}, false);
}
extern "C" int pnb_submit_host_f32(pnb_engine *e, const float *in, size_t in_stride, float *out, size_t out_stride,
                                   int n_frames) {
  return host_call(e, {Call::kSlots, {pcm(in, in_stride)}, {pcm(out, out_stride)}, n_frames}, true);
}
extern "C" int pnb_submit_host_i16(pnb_engine *e, const short *in, size_t in_stride, short *out, size_t out_stride,
                                   int n_frames) {
  return host_call(e, {Call::kSlots, {pcm(in, in_stride)}, {pcm(out, out_stride)}, n_frames}, true);
}

extern "C" int pnb_train_records_host(pnb_engine *e, const short *speech, size_t speech_stride, const short *noisy,
                                      size_t noisy_stride, int F, float *records, size_t records_stride) {
  return host_call(e, records_call(speech, speech_stride, noisy, noisy_stride, F, records, records_stride), false);
}
extern "C" int pnb_submit_train_records(pnb_engine *e, const short *speech, size_t speech_stride, const short *noisy,
                                        size_t noisy_stride, int F, float *records, size_t records_stride) {
  return host_call(e, records_call(speech, speech_stride, noisy, noisy_stride, F, records, records_stride), true);
}
extern "C" int pnb_train_audio_host(pnb_engine *e, const short *speech, size_t speech_stride, const short *noisy,
                                    size_t noisy_stride, int F, float *records, size_t records_stride, short *audio,
                                    size_t audio_stride) {
  return host_call(e, records_call(speech, speech_stride, noisy, noisy_stride, F, records, records_stride, true, audio,
                                   audio_stride), false);
}

// The network alone on caller-supplied features or training records (the batched compute_rnn, rnn.cpp:42): rows of 70
// features (any format but PNB_RNN_RECORDS, which check_call then refuses) or 138 record floats in, rows of g/r out.
static Call network_call(int format, const float *in, size_t in_stride, int n_frames, float *gr, size_t gr_stride) {
  Call c{Call::kNetwork, {rows(in, in_stride, format == PNB_RNN_RECORDS ? PNB_RECORD_FLOATS : kFeat, sizeof(float))},
         {rows(gr, gr_stride, 68, sizeof(float))}, n_frames};
  c.format = format;
  return c;
}
extern "C" int pnb_compute_rnn_device(pnb_engine *e, int format, const float *d_in, size_t in_stride, int n_frames, float *d_gr,
                                      size_t gr_stride, void *cuda_stream) {
  return device_call(e, network_call(format, d_in, in_stride, n_frames, d_gr, gr_stride), (cudaStream_t)cuda_stream);
}
extern "C" int pnb_compute_rnn_host(pnb_engine *e, int format, const float *in, size_t in_stride, int n_frames, float *gr,
                                    size_t gr_stride) {
  return host_call(e, network_call(format, in, in_stride, n_frames, gr, gr_stride), false);
}

// A network call on records that also reduces rnn_train.py's loss against their labels on the device: the sums, four
// doubles per row, are its second output; g/r its first only when asked for.
static Call score_call(const float *rec, size_t rec_stride, int n_frames, const int *frames, double *sums, float *gr,
                       size_t gr_stride) {
  Call c = network_call(PNB_RNN_RECORDS, rec, rec_stride, n_frames, gr, gr_stride);
  if (!gr) c.out[0] = {};
  c.out[1] = rows(sums, 4, 4, sizeof(double), "row stride", true);
  c.frames = frames;
  return c;
}
extern "C" int pnb_score_records_device(pnb_engine *e, const float *d_rec, size_t rec_stride, int n_frames, const int *frames,
                                        double *d_sums, float *d_gr, size_t gr_stride, void *cuda_stream) {
  return device_call(e, score_call(d_rec, rec_stride, n_frames, frames, d_sums, d_gr, gr_stride), (cudaStream_t)cuda_stream);
}
extern "C" int pnb_score_records_host(pnb_engine *e, const float *rec, size_t rec_stride, int n_frames, const int *frames,
                                      double *sums, float *gr, size_t gr_stride) {
  return host_call(e, score_call(rec, rec_stride, n_frames, frames, sums, gr, gr_stride), false);
}

// A gradient call (PNB_TRAIN_NETWORK): records in, the loss sums out, the gradient kept on the engine.
static Call train_call(const float *rec, size_t rec_stride, int n_frames, const int *frames, double *sums) {
  Call c{Call::kTrain, {rows(rec, rec_stride, PNB_RECORD_FLOATS, sizeof(float))}, {}, n_frames};
  c.out[1] = rows(sums, 4, 4, sizeof(double), "row stride", true);
  c.frames = frames;
  return c;
}
extern "C" int pnb_train_grad_device(pnb_engine *e, const float *d_rec, size_t rec_stride, int n_frames, const int *frames,
                                     double *d_sums, void *cuda_stream) {
  return device_call(e, train_call(d_rec, rec_stride, n_frames, frames, d_sums), (cudaStream_t)cuda_stream);
}
extern "C" int pnb_train_grad_host(pnb_engine *e, const float *rec, size_t rec_stride, int n_frames, const int *frames,
                                   double *sums) {
  return host_call(e, train_call(rec, rec_stride, n_frames, frames, sums), false);
}

// The trainer's forward and backward on the caller's tensors (PNB_TRAIN_NETWORK): features, and the state in and
// lengths when given, in; g/r, and the state out when asked for, out.  dL/d(out), and dL/d(state out) when given, in;
// dL/dx, dL/d(state in) and the gradient, each when asked for, out.  The calls without state are the calls with every
// state array and lengths NULL.
static Rows state_rows(const float *p, size_t stride, const char *name) {
  return p ? rows(p, stride, PNB_TRAIN_STATE_FLOATS, sizeof(float), name, true) : Rows{};
}
extern "C" int pnb_train_forward_state_device(pnb_engine *e, const float *d_x, size_t x_stride, int n_frames,
                                              const int *lengths, const float *d_weights, const float *d_state_in,
                                              size_t state_in_stride, float *d_out, size_t out_stride,
                                              float *d_state_out, size_t state_out_stride, void *cuda_stream) {
  Call c{Call::kTrainForward,
         {rows(d_x, x_stride, kFeat, sizeof(float), "x_stride"), state_rows(d_state_in, state_in_stride, "state_in_stride")},
         {rows(d_out, out_stride, 68, sizeof(float), "out_stride"),
          state_rows(d_state_out, state_out_stride, "state_out_stride")},
         n_frames};
  c.weights = d_weights;
  c.frames = lengths;
  return device_call(e, c, (cudaStream_t)cuda_stream);
}
extern "C" int pnb_train_backward_state_device(pnb_engine *e, const float *d_dout, size_t dout_stride,
                                               const float *d_dstate_out, size_t dstate_out_stride, float *d_dx,
                                               size_t dx_stride, float *d_dstate_in, size_t dstate_in_stride,
                                               float *d_grad, void *cuda_stream) {
  Call c{Call::kTrainBackward,
         {rows(d_dout, dout_stride, 68, sizeof(float), "dout_stride"),
          state_rows(d_dstate_out, dstate_out_stride, "dstate_out_stride")},
         {Rows{}, state_rows(d_dstate_in, dstate_in_stride, "dstate_in_stride")},
         0};
  if (d_dx) c.out[0] = rows(d_dx, dx_stride, kFeat, sizeof(float), "dx_stride");
  c.grad = d_grad;
  return device_call(e, c, (cudaStream_t)cuda_stream);
}
extern "C" int pnb_train_forward_device(pnb_engine *e, const float *d_x, size_t x_stride, int n_frames,
                                        const float *d_weights, float *d_out, size_t out_stride, void *cuda_stream) {
  return pnb_train_forward_state_device(e, d_x, x_stride, n_frames, nullptr, d_weights, nullptr, 0, d_out, out_stride,
                                        nullptr, 0, cuda_stream);
}
extern "C" int pnb_train_backward_device(pnb_engine *e, const float *d_dout, size_t dout_stride, float *d_dx,
                                         size_t dx_stride, float *d_grad, void *cuda_stream) {
  return pnb_train_backward_state_device(e, d_dout, dout_stride, nullptr, 0, d_dx, dx_stride, nullptr, 0, d_grad,
                                         cuda_stream);
}

// The refusals every training entry point shares: an engine of its kind that no failed call has poisoned.
static int check_trainer(pnb_engine *e) {
  if (!e) return fail(PNB_ERR_ARG, "engine is NULL");
  if (!(e->flags & PNB_TRAIN_NETWORK)) return fail(PNB_ERR_ARG, "engine was not created with PNB_TRAIN_NETWORK");
  if (e->poisoned) return refuse_poisoned(PNB_ERR_CUDA);
  return PNB_OK;
}

extern "C" int pnb_train_adam(pnb_engine *e, double lr, long long step, void *cuda_stream) {
  { int rc = check_trainer(e); if (rc) return rc; }
  if (!(lr >= 0.0) || !isfinite(lr)) return fail(PNB_ERR_ARG, "lr = %g is not a finite number >= 0", lr);
  if (step < 1) return fail(PNB_ERR_ARG, "step = %lld, Adam counts steps from 1", step);
  if (e->train_open)
    return fail(PNB_ERR_ARG, "accumulated gradients are not finished: pnb_train_finish before pnb_train_adam");
  CK(cudaSetDevice(e->device));
  if (int rc = enqueue_ordered(e, (cudaStream_t)cuda_stream, [&] { return train_adam(e, lr, step, (cudaStream_t)cuda_stream); }))
    return rc;
  e->train_fwd_F = 0;  // the step rewrote the weights a pending forward's backward would take
  return PNB_OK;
}

// Accumulation: the held gradient, weighted by the hops its call counted, into the float64 accumulator; and the
// accumulated batch's gradient back into the held gradient.  Each refuses what would count a gradient twice or step
// on a part of the batch, before anything is enqueued.
extern "C" int pnb_train_accumulate(pnb_engine *e, void *cuda_stream) {
  { int rc = check_trainer(e); if (rc) return rc; }
  if (!e->train_hops)
    return fail(PNB_ERR_ARG, "no gradient call or backward since the last pnb_train_accumulate or pnb_train_finish: the "
                             "held gradient is already counted");
  CK(cudaSetDevice(e->device));
  { int rc = train_accum_prepare(e); if (rc) return rc; }
  if (int rc = enqueue_ordered(e, (cudaStream_t)cuda_stream, [&] { return train_accumulate(e, (cudaStream_t)cuda_stream); }))
    return rc;
  e->train_hops = 0;
  e->train_open = true;
  return PNB_OK;
}
extern "C" int pnb_train_finish(pnb_engine *e, void *cuda_stream) {
  { int rc = check_trainer(e); if (rc) return rc; }
  if (!e->train_open)
    return fail(PNB_ERR_ARG, "nothing was accumulated or imported since the last pnb_train_finish");
  CK(cudaSetDevice(e->device));
  if (int rc = enqueue_ordered(e, (cudaStream_t)cuda_stream, [&] { return train_finish(e, (cudaStream_t)cuda_stream); }))
    return rc;
  e->train_hops = 0;
  e->train_open = false;
  return PNB_OK;
}

// Export / import of the trainer's arrays: weights, gradient, m and v as one flat float32 vector in PNBW blob order
// in host memory; the accumulator as its N + 1 doubles in host memory or device memory of the engine's device.  Both
// wait for the engine's earlier work and finish before they return.
static int train_transfer(pnb_engine *e, int what, void *mem, size_t bytes, bool out) {
  { int rc = check_trainer(e); if (rc) return rc; }
  if (!mem) return fail(PNB_ERR_ARG, "%s is NULL", out ? "dst" : "src");
  if (what < PNB_TRAIN_WEIGHTS || what > PNB_TRAIN_ACCUM) return fail(PNB_ERR_ARG, "what = %d is not a PNB_TRAIN_* array", what);
  if (!out && what == PNB_TRAIN_GRADIENT) return fail(PNB_ERR_ARG, "the gradient is computed, not imported");
  const bool accum = what == PNB_TRAIN_ACCUM;
  const size_t need = accum ? (train_params(e) + 1) * sizeof(double) : train_params(e) * sizeof(float);
  if ((out ? bytes < need : bytes != need) && accum)
    return fail(PNB_ERR_ARG, "%zu bytes, the accumulator is %zu doubles (%zu bytes)", bytes, train_params(e) + 1, need);
  if (out ? bytes < need : bytes != need)
    return fail(PNB_ERR_ARG, "%zu bytes, the model has %zu parameters (%zu bytes)", bytes, train_params(e), need);
  CK(cudaSetDevice(e->device));
  if (accum) { int rc = train_accum_prepare(e); if (rc) return rc; }
  const int rc = enqueue_ordered(e, e->stream, [&] {
    return accum ? train_accum_copy(e, mem, out, e->stream) : train_copy(e, what, mem, out, e->stream);
  });
  if (rc) return rc;
  CK(cudaStreamSynchronize(e->stream));
  if (accum && !out) e->train_open = true;
  if (what == PNB_TRAIN_WEIGHTS && !out) e->train_fwd_F = 0;  // as after pnb_train_adam
  return PNB_OK;
}
extern "C" int pnb_train_export(pnb_engine *e, int what, void *dst, size_t bytes) { return train_transfer(e, what, dst, bytes, true); }
extern "C" int pnb_train_import(pnb_engine *e, int what, const void *src, size_t bytes) {
  return train_transfer(e, what, const_cast<void *>(src), bytes, false);
}

// The split call: the analysis half of a slot call (PCM rows in, the network input out) and its synthesis half (the
// caller's g/r in, PCM rows out); f32 and int16 forms of either half mix freely.
static Call analyze_call(const void *in, size_t in_bytes, size_t in_stride, int n_frames, float *feat, size_t feat_stride) {
  return {Call::kAnalyze, {rows(in, in_stride, kFrame, in_bytes)}, {rows(feat, feat_stride, kFeat, sizeof(float), "feat_stride")}, n_frames};
}
static Call synthesize_call(const float *gr, size_t gr_stride, int n_frames, void *out, size_t out_bytes, size_t out_stride) {
  return {Call::kSynthesize, {rows(gr, gr_stride, 68, sizeof(float), "gr_stride")}, {rows(out, out_stride, kFrame, out_bytes)}, n_frames};
}
extern "C" int pnb_analyze_host_f32(pnb_engine *e, const float *in, size_t in_stride, int n_frames, float *feat, size_t feat_stride) {
  return host_call(e, analyze_call(in, sizeof(float), in_stride, n_frames, feat, feat_stride), false);
}
extern "C" int pnb_analyze_host_i16(pnb_engine *e, const short *in, size_t in_stride, int n_frames, float *feat, size_t feat_stride) {
  return host_call(e, analyze_call(in, sizeof(short), in_stride, n_frames, feat, feat_stride), false);
}
extern "C" int pnb_analyze_device_f32(pnb_engine *e, const float *d_in, size_t in_stride, int n_frames, float *d_feat,
                                      size_t feat_stride, void *cuda_stream) {
  return device_call(e, analyze_call(d_in, sizeof(float), in_stride, n_frames, d_feat, feat_stride), (cudaStream_t)cuda_stream);
}
extern "C" int pnb_analyze_device_i16(pnb_engine *e, const short *d_in, size_t in_stride, int n_frames, float *d_feat,
                                      size_t feat_stride, void *cuda_stream) {
  return device_call(e, analyze_call(d_in, sizeof(short), in_stride, n_frames, d_feat, feat_stride), (cudaStream_t)cuda_stream);
}
extern "C" int pnb_synthesize_host_f32(pnb_engine *e, const float *gr, size_t gr_stride, int n_frames, float *out, size_t out_stride) {
  return host_call(e, synthesize_call(gr, gr_stride, n_frames, out, sizeof(float), out_stride), false);
}
extern "C" int pnb_synthesize_host_i16(pnb_engine *e, const float *gr, size_t gr_stride, int n_frames, short *out, size_t out_stride) {
  return host_call(e, synthesize_call(gr, gr_stride, n_frames, out, sizeof(short), out_stride), false);
}
extern "C" int pnb_synthesize_device_f32(pnb_engine *e, const float *d_gr, size_t gr_stride, int n_frames, float *d_out,
                                         size_t out_stride, void *cuda_stream) {
  return device_call(e, synthesize_call(d_gr, gr_stride, n_frames, d_out, sizeof(float), out_stride), (cudaStream_t)cuda_stream);
}
extern "C" int pnb_synthesize_device_i16(pnb_engine *e, const float *d_gr, size_t gr_stride, int n_frames, short *d_out,
                                         size_t out_stride, void *cuda_stream) {
  return device_call(e, synthesize_call(d_gr, gr_stride, n_frames, d_out, sizeof(short), out_stride), (cudaStream_t)cuda_stream);
}
// The operands of the pending synthesis (include/pnb_synth_grad.h): a split call with no input, whose hops are the
// pending analysis's.
extern "C" int pnb_synthesis_operands_device(pnb_engine *e, float *d_ops, size_t ops_stride, void *cuda_stream) {
  return device_call(e, {Call::kOperands, {}, {rows(d_ops, ops_stride, kSynthOps, sizeof(float), "ops_stride")}, 0},
                     (cudaStream_t)cuda_stream);
}

// The split and network calls on a session list: row i of every array belongs to ids[i]; hops NULL, or each listed
// session's own hops (ragged, n_frames = max(hops)).  The synthesis takes the list, hops and rows of the pending analysis.
static Call on_sessions(Call c, const int *ids, const int *hops, int n) {
  c.ids = ids;
  c.n_ids = n;
  c.hops = hops;
  c.pool = true;
  return c;
}
extern "C" int pnb_analyze_sessions_device_f32(pnb_engine *e, const int *ids, const int *hops, int n, const float *d_in,
                                               size_t in_stride, int n_frames, float *d_feat, size_t feat_stride, void *cuda_stream) {
  return device_call(e, on_sessions(analyze_call(d_in, sizeof(float), in_stride, n_frames, d_feat, feat_stride), ids, hops, n),
                     (cudaStream_t)cuda_stream);
}
extern "C" int pnb_analyze_sessions_device_i16(pnb_engine *e, const int *ids, const int *hops, int n, const short *d_in,
                                               size_t in_stride, int n_frames, float *d_feat, size_t feat_stride, void *cuda_stream) {
  return device_call(e, on_sessions(analyze_call(d_in, sizeof(short), in_stride, n_frames, d_feat, feat_stride), ids, hops, n),
                     (cudaStream_t)cuda_stream);
}
extern "C" int pnb_analyze_sessions_host_f32(pnb_engine *e, const int *ids, const int *hops, int n, const float *in,
                                             size_t in_stride, int n_frames, float *feat, size_t feat_stride) {
  return host_call(e, on_sessions(analyze_call(in, sizeof(float), in_stride, n_frames, feat, feat_stride), ids, hops, n), false);
}
extern "C" int pnb_analyze_sessions_host_i16(pnb_engine *e, const int *ids, const int *hops, int n, const short *in,
                                             size_t in_stride, int n_frames, float *feat, size_t feat_stride) {
  return host_call(e, on_sessions(analyze_call(in, sizeof(short), in_stride, n_frames, feat, feat_stride), ids, hops, n), false);
}
extern "C" int pnb_synthesize_sessions_device_f32(pnb_engine *e, const int *ids, int n, const float *d_gr, size_t gr_stride,
                                                  int n_frames, float *d_out, size_t out_stride, void *cuda_stream) {
  return device_call(e, on_sessions(synthesize_call(d_gr, gr_stride, n_frames, d_out, sizeof(float), out_stride), ids, nullptr, n),
                     (cudaStream_t)cuda_stream);
}
extern "C" int pnb_synthesize_sessions_device_i16(pnb_engine *e, const int *ids, int n, const float *d_gr, size_t gr_stride,
                                                  int n_frames, short *d_out, size_t out_stride, void *cuda_stream) {
  return device_call(e, on_sessions(synthesize_call(d_gr, gr_stride, n_frames, d_out, sizeof(short), out_stride), ids, nullptr, n),
                     (cudaStream_t)cuda_stream);
}
extern "C" int pnb_synthesize_sessions_host_f32(pnb_engine *e, const int *ids, int n, const float *gr, size_t gr_stride,
                                                int n_frames, float *out, size_t out_stride) {
  return host_call(e, on_sessions(synthesize_call(gr, gr_stride, n_frames, out, sizeof(float), out_stride), ids, nullptr, n), false);
}
extern "C" int pnb_synthesize_sessions_host_i16(pnb_engine *e, const int *ids, int n, const float *gr, size_t gr_stride,
                                                int n_frames, short *out, size_t out_stride) {
  return host_call(e, on_sessions(synthesize_call(gr, gr_stride, n_frames, out, sizeof(short), out_stride), ids, nullptr, n), false);
}
extern "C" int pnb_compute_rnn_sessions_device(pnb_engine *e, const int *ids, const int *hops, int n, int format, const float *d_in,
                                               size_t in_stride, int n_frames, float *d_gr, size_t gr_stride, void *cuda_stream) {
  return device_call(e, on_sessions(network_call(format, d_in, in_stride, n_frames, d_gr, gr_stride), ids, hops, n),
                     (cudaStream_t)cuda_stream);
}
extern "C" int pnb_compute_rnn_sessions_host(pnb_engine *e, const int *ids, const int *hops, int n, int format, const float *in,
                                             size_t in_stride, int n_frames, float *gr, size_t gr_stride) {
  return host_call(e, on_sessions(network_call(format, in, in_stride, n_frames, gr, gr_stride), ids, hops, n), false);
}

extern "C" int pnb_flush(pnb_engine *e, void *cuda_stream) {
  if (!e) return fail(PNB_ERR_ARG, "engine is NULL");
  CK(cudaSetDevice(e->device));
  return wait_last_call(e, (cudaStream_t)cuda_stream);
}

extern "C" int pnb_wait(pnb_engine *e) {
  if (!e) return fail(PNB_ERR_ARG, "engine is NULL");
  CK(cudaSetDevice(e->device));
  if (e->s_in) CK(cudaStreamSynchronize(e->s_in));
  { int rc = wait_last_call(e, e->stream); if (rc) return rc; }  // the status covers every call, on any stream
  CK(cudaMemcpyAsync(e->h_status, e->d_status, 2 * sizeof(int), cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  if (e->s_out) CK(cudaStreamSynchronize(e->s_out));
  return report_status(e);
}
extern "C" int pnb_check(pnb_engine *e, void *cuda_stream) {
  if (!e) return fail(PNB_ERR_ARG, "engine is NULL");
  CK(cudaSetDevice(e->device));
  CK(cudaStreamSynchronize((cudaStream_t)cuda_stream));
  int rc = pnb_wait(e);
  if (rc) return rc;
  if (e->poisoned) return fail(PNB_ERR_CUDA, "an earlier call failed while enqueuing work; pnb_reset the engine");
  return PNB_OK;
}

extern "C" int pnb_read_tap(pnb_engine *e, int what, void *dst, size_t dst_bytes) {
  if (!e || !dst) return fail(PNB_ERR_ARG, "NULL argument");
  CK(cudaSetDevice(e->device));
  const size_t n = (size_t)e->last_frames * e->S;
  const void *src = nullptr;
  size_t bytes = 0;
  switch (what) {
    case PNB_TAP_FEATURES: src = e->d_feat; bytes = n * kFeat * 4; break;
    case PNB_TAP_PITCH: src = e->d_tap_pitch; bytes = n * 16; break;
    case PNB_TAP_PITCHF: src = e->d_tap_pitchf; bytes = n * 8; break;
    case PNB_TAP_X: {  // gather from the ring: the analysis spectrum of hop c is the slot of hop c-5
      if (!e->d_zring) return fail(PNB_ERR_ARG, "tap %d: a PNB_NETWORK_ONLY engine has no spectra", what);
      bytes = n * kBins * 8;
      if (dst_bytes < bytes) return fail(PNB_ERR_ARG, "tap %d needs %zu bytes, got %zu", what, bytes, dst_bytes);
      CK(cudaDeviceSynchronize());
      const size_t per = (size_t)e->S * kBins * 8;
      for (int k = 0; k < e->last_frames; k++) {
        long c = e->hop - e->last_frames + k;
        int slot = (int)(((c - 5) % e->ring + e->ring) % e->ring);
        CK(cudaMemcpy((char *)dst + k * per, (const char *)e->d_zring + slot * per, per, cudaMemcpyDeviceToHost));
      }
      return PNB_OK;
    }
    case PNB_TAP_P: src = e->d_P; bytes = n * kBins * 8; break;
    case PNB_TAP_EX: src = e->d_Ex; bytes = n * kBands * 4; break;
    case PNB_TAP_GR: src = e->d_gr; bytes = n * 68 * 4; break;
    case PNB_TAP_G_USED: src = e->d_tap_g; bytes = n * kBands * 4; break;
    case PNB_TAP_NN_C2: src = e->c2; bytes = (size_t)e->S * 512 * 4; break;
    case PNB_TAP_NN_H0: case PNB_TAP_NN_H0 + 1: case PNB_TAP_NN_H0 + 2: case PNB_TAP_NN_H0 + 3: case PNB_TAP_NN_H0 + 4: {
      int li = what - PNB_TAP_NN_H0;
      src = e->h[li]; bytes = (size_t)e->S * kGruH[li] * 4; break;
    }
    case PNB_TAP_TRAIN_FC: case PNB_TAP_TRAIN_C1: case PNB_TAP_TRAIN_C2PRE: case PNB_TAP_TRAIN_DPRE: {
      int rc = train_tap(e, what, &src, &bytes);
      if (rc) return rc;
      break;
    }
    default: return fail(PNB_ERR_ARG, "unknown tap %d", what);
  }
  if (!src && (e->flags & PNB_SIGNAL_ONLY) && what >= PNB_TAP_NN_C2 && what < PNB_TAP_G_USED)
    return fail(PNB_ERR_ARG, "tap %d: a PNB_SIGNAL_ONLY engine has no network state", what);
  if (!src && (e->flags & PNB_NETWORK_ONLY))
    return fail(PNB_ERR_ARG, "tap %d: a PNB_NETWORK_ONLY engine keeps the features, g/r and network state taps only", what);
  if (!src) return fail(PNB_ERR_ARG, "tap %d needs PNB_KEEP_TAPS at pnb_create", what);
  if (dst_bytes < bytes) return fail(PNB_ERR_ARG, "tap %d needs %zu bytes, got %zu", what, bytes, dst_bytes);
  CK(cudaDeviceSynchronize());
  CK(cudaMemcpy(dst, src, bytes, cudaMemcpyDeviceToHost));
  return PNB_OK;
}

// ------------------------------------------------------------------------------------------
// per-stream state export / import (the reference's DenoiseState + RNNState, src/denoise.cpp:71-85, nnet_data.h:28-38,
// reduced to what is live: SURVEY.md App. A.2) -- for moving a stream between engines / GPUs at a call boundary
// ------------------------------------------------------------------------------------------
extern "C" size_t pnb_state_size(void) { return sizeof(StreamState); }

// The blobs of a batched state operation: not NULL, blob_stride at least pnb_state_size(), both 4-byte aligned.
static int check_blobs(const void *d_blobs, size_t blob_stride) {
  if (!d_blobs) return fail(PNB_ERR_ARG, "d_blobs is NULL");
  if (blob_stride < sizeof(StreamState))
    return fail(PNB_ERR_ARG, "blob_stride %zu below pnb_state_size() = %zu", blob_stride, sizeof(StreamState));
  if ((reinterpret_cast<uintptr_t>(d_blobs) | blob_stride) & 3) return fail(PNB_ERR_ARG, "d_blobs and blob_stride must be multiples of 4 bytes");
  return PNB_OK;
}

static int state_batch(pnb_engine *e, int mode, const int *streams, int n, void *d_blobs, size_t blob_stride, void *cuda_stream) {
  if (!e) return fail(PNB_ERR_ARG, "engine is NULL");
  if (e->sessions) return refuse_in_session_mode();
  if (e->pending.F) return refuse_pending(e);
  if (n < 0) return fail(PNB_ERR_ARG, "n = %d is negative", n);
  if (n == 0) return PNB_OK;
  if (!streams) return fail(PNB_ERR_ARG, "streams is NULL");
  if (mode != kStateReset) { int rc = check_blobs(d_blobs, blob_stride); if (rc) return rc; }
  if (e->poisoned) return refuse_poisoned(PNB_ERR_ARG);
  if (n > e->S) return fail(PNB_ERR_ARG, "n = %d streams, the engine has %d", n, e->S);
  { int rc = check_list(e, streams, n, e->S, e->n_active, "streams"); if (rc) return rc; }
  CK(cudaSetDevice(e->device));
  return enqueue_state(e, {mode, streams, n, d_blobs, blob_stride, false}, (cudaStream_t)cuda_stream);
}

extern "C" int pnb_reset_streams(pnb_engine *e, const int *streams, int n, void *cuda_stream) {
  return state_batch(e, kStateReset, streams, n, nullptr, 0, cuda_stream);
}
extern "C" int pnb_export_states(pnb_engine *e, const int *streams, int n, void *d_blobs, size_t blob_stride, void *cuda_stream) {
  return state_batch(e, kStateExport, streams, n, d_blobs, blob_stride, cuda_stream);
}
extern "C" int pnb_import_states(pnb_engine *e, const int *streams, int n, const void *d_blobs, size_t blob_stride, void *cuda_stream) {
  return state_batch(e, kStateImport, streams, n, const_cast<void *>(d_blobs), blob_stride, cuda_stream);
}

// Active range: calls advance slots [0, n).  Growing it resets the entering slots like pnb_reset_streams (ordered like
// any state operation); shrinking it enqueues nothing, the leaving slots' state is simply no longer kept.
extern "C" int pnb_set_active_streams(pnb_engine *e, int n, void *cuda_stream) {
  if (!e) return fail(PNB_ERR_ARG, "engine is NULL");
  if (e->flags & PNB_TRAIN_DATA) return fail(PNB_ERR_ARG, "PNB_TRAIN_DATA engines always advance all their streams");
  if (e->sessions) return refuse_in_session_mode();
  if (e->pending.F) return refuse_pending(e);
  if (n < 1 || n > e->S) return fail(PNB_ERR_ARG, "active streams %d outside [1, %d]", n, e->S);
  if (e->poisoned) return refuse_poisoned(PNB_ERR_ARG);
  if (n > e->n_active) {
    std::vector<int> entering(n - e->n_active);
    for (int i = 0; i < n - e->n_active; i++) entering[i] = e->n_active + i;
    CK(cudaSetDevice(e->device));
    const int rc = enqueue_state(e, {kStateReset, entering.data(), (int)entering.size(), nullptr, 0, false}, (cudaStream_t)cuda_stream);
    if (rc) return rc;
  }
  e->n_active = n;
  e->train_fwd_F = 0;  // a pending training forward ran on the old rows
  return PNB_OK;
}
extern "C" int pnb_active_streams(const pnb_engine *e) { return e ? e->n_active : 0; }

static int check_one_state(pnb_engine *e, int stream, const void *buf, size_t bytes) {
  if (!e || !buf) return fail(PNB_ERR_ARG, "NULL argument");
  if (e->sessions) return refuse_in_session_mode();
  if (e->pending.F) return refuse_pending(e);
  { int rc = check_list(e, &stream, 1, e->S, e->n_active, "stream"); if (rc) return rc; }
  if (bytes < sizeof(StreamState)) return fail(PNB_ERR_ARG, "state buffer of %zu bytes, need pnb_state_size() = %zu", bytes, sizeof(StreamState));
  if (e->poisoned) return refuse_poisoned(PNB_ERR_CUDA);
  return PNB_OK;
}

// The single-stream host forms: the batched kernels through one blob of device scratch, with the engine idle before
// and after.
extern "C" int pnb_get_state(pnb_engine *e, int stream, void *dst, size_t bytes) {
  int rc = check_one_state(e, stream, dst, bytes);
  if (rc) return rc;
  CK(cudaSetDevice(e->device));
  CK(cudaDeviceSynchronize());
  if ((rc = enqueue_state(e, {kStateExport, &stream, 1, e->d_blob1, sizeof(StreamState), false}, e->stream))) return rc;
  CK(cudaMemcpyAsync(dst, e->d_blob1, sizeof(StreamState), cudaMemcpyDeviceToHost, e->stream));
  CK(cudaStreamSynchronize(e->stream));
  return PNB_OK;
}

extern "C" int pnb_set_state(pnb_engine *e, int stream, const void *src, size_t bytes) {
  int rc = check_one_state(e, stream, src, bytes);
  if (rc) return rc;
  const StreamState *st = static_cast<const StreamState *>(src);
  if (st->magic != kStateMagic || st->version != kStateVersion) return fail(PNB_ERR_ARG, "not a pnb_get_state blob (magic/version)");
  if (e->flags & PNB_NN_TENSOR)
    for (size_t i = 0; i < sizeof st->h / sizeof(float); i++)
      if (!(fabsf(st->h[i]) <= kStateGruBound))
        return fail(PNB_ERR_ARG, "GRU state value %g outside [-1, 1]: not a state the network can reach", (double)st->h[i]);
  CK(cudaSetDevice(e->device));
  CK(cudaDeviceSynchronize());
  CK(cudaMemcpyAsync(e->d_blob1, src, sizeof(StreamState), cudaMemcpyHostToDevice, e->stream));
  if ((rc = enqueue_state(e, {kStateImport, &stream, 1, e->d_blob1, sizeof(StreamState), false}, e->stream))) return rc;
  CK(cudaStreamSynchronize(e->stream));
  return PNB_OK;
}

// ------------------------------------------------------------------------------------------
// session pool: sessions [0, capacity) over the engine's slots; a call advances any listed subset (pnb_session_plan.h)
// ------------------------------------------------------------------------------------------
// Grows both buffer pairs (pinned and device) of the index staging to at least n ints; the engine is idle.
static int grow_ints(pnb_engine *e, size_t n) {
  if (n > e->idx_cap) {
    for (int k = 0; k < 2; k++) {
      int *h = nullptr, *d = nullptr;
      CK(cudaHostAlloc((void **)&h, n * sizeof(int), cudaHostAllocDefault));
      CK(cudaMalloc((void **)&d, n * sizeof(int)));
      cudaFreeHost(e->h_idx[k]);
      cudaFree(e->d_idx[k]);
      e->h_idx[k] = h;
      e->d_idx[k] = d;
    }
    e->idx_cap = n;
  }
  return PNB_OK;
}

extern "C" int pnb_sessions_reserve(pnb_engine *e, int n_sessions) {
  if (!e) return fail(PNB_ERR_ARG, "engine is NULL");
  if (e->flags & PNB_TRAIN_DATA) return fail(PNB_ERR_ARG, "PNB_TRAIN_DATA engines have no session pool");
  if (e->flags & PNB_NETWORK_ONLY) return fail(PNB_ERR_ARG, "PNB_NETWORK_ONLY engines have no session pool");
  if (e->flags & PNB_SIGNAL_ONLY) return fail(PNB_ERR_ARG, "PNB_SIGNAL_ONLY engines have no session pool");
  if (e->pending.F) return refuse_pending(e);
  if (e->poisoned) return refuse_poisoned(PNB_ERR_ARG);
  if (n_sessions < 1) return fail(PNB_ERR_ARG, "n_sessions = %d, need >= 1", n_sessions);
  if (e->sessions && n_sessions <= e->pool.capacity()) return PNB_OK;  // the pool never shrinks
  CK(cudaSetDevice(e->device));
  CK(cudaDeviceSynchronize());
  const size_t cap = (size_t)n_sessions, wide = cap > (size_t)e->S ? cap : (size_t)e->S;
  // staging: a call's row and slot maps, for a ragged call slot hops and short slots, then the moves (<= 8 S + 3 ints),
  // an export's moves, ids and rows (<= 6 n)
  { int rc = grow_ints(e, 8 * wide + 4); if (rc) return rc; }
  if (wide > e->ok_cap) {
    int *ok = nullptr;
    CK(cudaMalloc((void **)&ok, wide * sizeof(int)));
    cudaFree(e->d_ok);
    e->d_ok = ok;
    e->ok_cap = wide;
  }
  char *park = nullptr;
  cudaError_t ce = cudaMalloc((void **)&park, cap * kParkStride);
  if (ce != cudaSuccess)
    return fail(ce == cudaErrorMemoryAllocation ? PNB_ERR_ALLOC : PNB_ERR_CUDA, "parking area of %zu sessions: %s", cap,
                cudaGetErrorString(ce));
  if (e->sessions) {  // grow: the parked sessions keep their blobs, the new ones start fresh
    const size_t old = (size_t)e->pool.capacity() * kParkStride;
    CK(cudaMemcpy(park, e->d_park, old, cudaMemcpyDeviceToDevice));
    CK(cudaMemset(park + old, 0, cap * kParkStride - old));
    CK(cudaFree(e->d_park));
    e->d_park = park;
    e->pool.grow((int)cap);
    return PNB_OK;
  }
  e->d_park = park;
  e->sessions = true;
  e->pool.init(e->S, (int)cap);
  return pnb_reset(e);
}

extern "C" int pnb_session_stats(const pnb_engine *e, long long *out) {
  if (!e || !out) return fail(PNB_ERR_ARG, "NULL argument");
  out[0] = e->pool.parks;
  out[1] = e->pool.unparks;
  out[2] = e->pool.relocations;
  return PNB_OK;
}

extern "C" int pnb_process_sessions_device_f32(pnb_engine *e, const int *ids, int n, const float *d_in, size_t in_stride,
                                               float *d_out, size_t out_stride, int n_frames, float *d_gr, void *cuda_stream) {
  return device_call(e, {Call::kSessions, {pcm(d_in, in_stride)}, {pcm(d_out, out_stride)}, n_frames, d_gr, ids, n}, (cudaStream_t)cuda_stream);
}
extern "C" int pnb_process_sessions_device_i16(pnb_engine *e, const int *ids, int n, const short *d_in, size_t in_stride,
                                               short *d_out, size_t out_stride, int n_frames, float *d_gr, void *cuda_stream) {
  return device_call(e, {Call::kSessions, {pcm(d_in, in_stride)}, {pcm(d_out, out_stride)}, n_frames, d_gr, ids, n}, (cudaStream_t)cuda_stream);
}
extern "C" int pnb_process_sessions_host_f32(pnb_engine *e, const int *ids, int n, const float *in, size_t in_stride, float *out,
                                             size_t out_stride, int n_frames, float *gr) {
  return host_call(e, {Call::kSessions, {pcm(in, in_stride)}, {pcm(out, out_stride)}, n_frames, gr, ids, n}, false);
}
extern "C" int pnb_process_sessions_host_i16(pnb_engine *e, const int *ids, int n, const short *in, size_t in_stride, short *out,
                                             size_t out_stride, int n_frames, float *gr) {
  return host_call(e, {Call::kSessions, {pcm(in, in_stride)}, {pcm(out, out_stride)}, n_frames, gr, ids, n}, false);
}

// Ragged session calls: session ids[i] advances by hops[i]; the call is max(hops) hops long (check_call).
extern "C" int pnb_process_sessions_ragged_device_f32(pnb_engine *e, const int *ids, const int *hops, int n, const float *d_in,
                                                      size_t in_stride, float *d_out, size_t out_stride, float *d_gr,
                                                      void *cuda_stream) {
  return device_call(e, {Call::kRagged, {pcm(d_in, in_stride)}, {pcm(d_out, out_stride)}, 0, d_gr, ids, n, hops}, (cudaStream_t)cuda_stream);
}
extern "C" int pnb_process_sessions_ragged_device_i16(pnb_engine *e, const int *ids, const int *hops, int n, const short *d_in,
                                                      size_t in_stride, short *d_out, size_t out_stride, float *d_gr,
                                                      void *cuda_stream) {
  return device_call(e, {Call::kRagged, {pcm(d_in, in_stride)}, {pcm(d_out, out_stride)}, 0, d_gr, ids, n, hops}, (cudaStream_t)cuda_stream);
}
extern "C" int pnb_process_sessions_ragged_host_f32(pnb_engine *e, const int *ids, const int *hops, int n, const float *in,
                                                    size_t in_stride, float *out, size_t out_stride, float *gr) {
  return host_call(e, {Call::kRagged, {pcm(in, in_stride)}, {pcm(out, out_stride)}, 0, gr, ids, n, hops}, false);
}
extern "C" int pnb_process_sessions_ragged_host_i16(pnb_engine *e, const int *ids, const int *hops, int n, const short *in,
                                                    size_t in_stride, short *out, size_t out_stride, float *gr) {
  return host_call(e, {Call::kRagged, {pcm(in, in_stride)}, {pcm(out, out_stride)}, 0, gr, ids, n, hops}, false);
}

// pnb_reset_sessions / pnb_export_sessions / pnb_import_sessions.  A reset or an import takes the listed sessions out
// of their slots (the slot's content is abandoned) and rewrites their parking blobs; the next call that lists them
// unparks them.  An export writes each session from where it is; nothing moves.
static int session_batch(pnb_engine *e, int mode, const int *ids, int n, void *d_blobs, size_t blob_stride, void *cuda_stream) {
  if (!e) return fail(PNB_ERR_ARG, "engine is NULL");
  if (e->poisoned) return refuse_poisoned(PNB_ERR_ARG);
  if (e->pending.F) return refuse_pending(e);
  if (n == 0 && e->sessions) return PNB_OK;
  if (mode != kStateReset) { int rc = check_blobs(d_blobs, blob_stride); if (rc) return rc; }
  { int rc = check_ids(e, ids, n, e->pool.capacity()); if (rc) return rc; }
  CK(cudaSetDevice(e->device));
  return enqueue_state(e, {mode, ids, n, d_blobs, blob_stride, true}, (cudaStream_t)cuda_stream);
}
extern "C" int pnb_reset_sessions(pnb_engine *e, const int *ids, int n, void *cuda_stream) {
  return session_batch(e, kStateReset, ids, n, nullptr, 0, cuda_stream);
}
extern "C" int pnb_export_sessions(pnb_engine *e, const int *ids, int n, void *d_blobs, size_t blob_stride, void *cuda_stream) {
  return session_batch(e, kStateExport, ids, n, d_blobs, blob_stride, cuda_stream);
}
extern "C" int pnb_import_sessions(pnb_engine *e, const int *ids, int n, const void *d_blobs, size_t blob_stride, void *cuda_stream) {
  return session_batch(e, kStateImport, ids, n, const_cast<void *>(d_blobs), blob_stride, cuda_stream);
}

// ------------------------------------------------------------------------------------------
// binary weight file -> pnb_model (layout of the generated nnet_data.cpp, SURVEY.md App. B)
// ------------------------------------------------------------------------------------------
namespace {
struct BlobModel {
  pnb_model m;
  pnb_dense_layer fc, fc_gb, fc_rb;
  pnb_conv1d_layer conv1, conv2;
  pnb_gru_layer gru[5];
  std::vector<std::vector<float>> arrays;
};
bool read_array(FILE *f, size_t expect, std::vector<float> &dst) {
  unsigned long long n = 0;
  if (fread(&n, 8, 1, f) != 1 || n != expect) return false;
  dst.resize(n);
  return fread(dst.data(), 4, n, f) == n;
}
}  // namespace

extern "C" int pnb_model_load_blob(const char *path, pnb_model **out) {
  if (!path || !out) return fail(PNB_ERR_ARG, "NULL argument");
  *out = nullptr;
  FILE *f = fopen(path, "rb");
  if (!f) return fail(PNB_ERR_ARG, "cannot open %s", path);
  int rc = pnb_model_load_stream(f, out);
  fclose(f);
  return rc;
}

extern "C" int pnb_model_load_stream(void *file, pnb_model **out) {
  if (!file || !out) return fail(PNB_ERR_ARG, "NULL argument");
  *out = nullptr;
  FILE *f = static_cast<FILE *>(file);
  const char *path = "weight stream";
  char magic[8];
  if (fread(magic, 1, 8, f) != 8 || memcmp(magic, "PNBW0001", 8) != 0) return fail(PNB_ERR_ARG, "%s is not a PNBW0001 weight file", path);
  BlobModel *b = new BlobModel();
  b->arrays.resize(25);
  int ai = 0;
  bool ok = true;
  auto dense = [&](pnb_dense_layer &l, int M, int N, int act) {
    ok = ok && read_array(f, (size_t)M * N, b->arrays[ai]) && read_array(f, N, b->arrays[ai + 1]);
    l.input_weights = b->arrays[ai].data(); l.bias = b->arrays[ai + 1].data(); l.nb_inputs = M; l.nb_neurons = N; l.activation = act;
    ai += 2;
  };
  auto conv = [&](pnb_conv1d_layer &l, int C, int K, int N, int act) {
    ok = ok && read_array(f, (size_t)C * K * N, b->arrays[ai]) && read_array(f, N, b->arrays[ai + 1]);
    l.input_weights = b->arrays[ai].data(); l.bias = b->arrays[ai + 1].data(); l.nb_inputs = C; l.kernel_size = K; l.nb_neurons = N; l.activation = act;
    ai += 2;
  };
  auto gru = [&](pnb_gru_layer &l, int M, int H) {
    ok = ok && read_array(f, (size_t)M * 3 * H, b->arrays[ai]) && read_array(f, (size_t)H * 3 * H, b->arrays[ai + 1]) &&
         read_array(f, 6 * (size_t)H, b->arrays[ai + 2]);
    l.input_weights = b->arrays[ai].data(); l.recurrent_weights = b->arrays[ai + 1].data(); l.bias = b->arrays[ai + 2].data();
    l.nb_inputs = M; l.nb_neurons = H; l.activation = PNB_ACT_TANH; l.reset_after = 1;
    ai += 3;
  };
  dense(b->fc, 70, 128, PNB_ACT_RELU);
  conv(b->conv1, 128, 5, 512, PNB_ACT_RELU);
  conv(b->conv2, 512, 3, 512, PNB_ACT_TANH);
  for (int i = 0; i < 4; i++) gru(b->gru[i], 512, 512);
  gru(b->gru[4], 1024, 128);
  dense(b->fc_gb, 2560, 34, PNB_ACT_SIGMOID);
  dense(b->fc_rb, 128, 34, PNB_ACT_SIGMOID);
  if (!ok) { delete b; return fail(PNB_ERR_ARG, "%s is truncated or has unexpected layer sizes", path); }
  b->m.fc = &b->fc; b->m.conv1 = &b->conv1; b->m.conv2 = &b->conv2;
  b->m.gru1 = &b->gru[0]; b->m.gru2 = &b->gru[1]; b->m.gru3 = &b->gru[2]; b->m.gru_gb = &b->gru[3]; b->m.gru_rb = &b->gru[4];
  b->m.fc_gb = &b->fc_gb; b->m.fc_rb = &b->fc_rb;
  *out = &b->m;  // first member: the BlobModel is recovered from the pointer in pnb_model_free
  return PNB_OK;
}
extern "C" void pnb_model_free(pnb_model *m) {
  if (m) delete reinterpret_cast<BlobModel *>(m);
}

// ------------------------------------------------------------------------------------------
// the pitch analysis alone (BASELINE.json config 5)
// ------------------------------------------------------------------------------------------
extern "C" int pnb_pitch_only_device(const float *d_pitch_buf, size_t stride, long long n_units, const int *d_prev_period,
                                     const float *d_prev_gain, int *d_period, float *d_corr, float *d_gain, int *d_lag,
                                     void *cuda_stream) {
  if (!d_pitch_buf || !d_period || !d_corr || !d_gain) return fail(PNB_ERR_ARG, "NULL argument");
  if (n_units < 1 || stride < 1728) return fail(PNB_ERR_ARG, "n_units must be >= 1 and stride >= 1728");
  if (n_units > (1ll << 31) - 8) return fail(PNB_ERR_ARG, "n_units above 2^31");
  PitchOnlyArgs a;
  a.buf = d_pitch_buf; a.stride = stride; a.n_units = (long)n_units; a.prev_period = d_prev_period; a.prev_gain = d_prev_gain;
  a.T = d_period; a.corr = d_corr; a.gain = d_gain; a.lag = d_lag;
  // uncounted: there is no engine to count it
  if (!launch_pitch_only(a, (cudaStream_t)cuda_stream)) return fail(PNB_ERR_CUDA, "pitch_only_kernel could not be configured");
  CK(cudaGetLastError());
  return PNB_OK;
}

// ------------------------------------------------------------------------------------------
// the synthesis's gradient with respect to g/r (include/pnb_synth_grad.h)
// ------------------------------------------------------------------------------------------
// The constant tables on the current device, uploaded by the first call there and kept for the process (there is no
// engine to own them); null when the upload failed.
static const Tables *device_tables() {
  static std::mutex mu;
  static std::vector<Tables *> per_device;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return nullptr;
  std::lock_guard<std::mutex> lock(mu);
  if ((size_t)dev >= per_device.size()) per_device.resize(dev + 1, nullptr);
  if (!per_device[dev]) {
    Tables h;
    build_tables(h);
    Tables *d = nullptr;
    if (cudaMalloc((void **)&d, sizeof(Tables)) != cudaSuccess) return nullptr;
    if (cudaMemcpy(d, &h, sizeof(Tables), cudaMemcpyHostToDevice) != cudaSuccess) {
      cudaFree(d);
      return nullptr;
    }
    per_device[dev] = d;
  }
  return per_device[dev];
}

extern "C" int pnb_synthesis_backward_device(const float *d_ops, size_t ops_stride, const float *d_gr, size_t gr_stride,
                                             long long n_rows, int n_frames, int postfilter, const float *d_dout,
                                             size_t dout_stride, float *d_dgr, size_t dgr_stride, void *cuda_stream) {
  if (!d_ops || !d_gr || !d_dout || !d_dgr) return fail(PNB_ERR_ARG, "NULL argument");
  if (n_rows < 1) return fail(PNB_ERR_ARG, "n_rows %lld below 1", n_rows);
  if (n_frames < 1) return fail(PNB_ERR_ARG, "n_frames %d below 1", n_frames);
  if (postfilter != 0 && postfilter != 1) return fail(PNB_ERR_ARG, "postfilter %d is neither 0 nor 1", postfilter);
  const size_t F = (size_t)n_frames;
  if (ops_stride < F * kSynthOps) return fail(PNB_ERR_ARG, "ops_stride smaller than n_frames*%d", kSynthOps);
  if (gr_stride < F * 68) return fail(PNB_ERR_ARG, "gr_stride smaller than n_frames*68");
  if (dout_stride < F * kFrame) return fail(PNB_ERR_ARG, "dout_stride smaller than n_frames*%d", kFrame);
  if (dgr_stride < F * 68) return fail(PNB_ERR_ARG, "dgr_stride smaller than n_frames*68");
  SynthGradArgs a;
  a.ops = d_ops; a.ops_stride = ops_stride; a.gr = d_gr; a.gr_stride = gr_stride; a.dout = d_dout;
  a.dout_stride = dout_stride; a.dgr = d_dgr; a.dgr_stride = dgr_stride; a.n_rows = n_rows; a.n_frames = n_frames;
  a.postfilter = postfilter;
  a.tab = device_tables();
  if (!a.tab) return fail(PNB_ERR_CUDA, "the constant tables could not be uploaded to the current device");
  // uncounted: there is no engine to count it
  if (!launch_synthesis_backward(a, (cudaStream_t)cuda_stream))
    return fail(PNB_ERR_CUDA, "synthesis_backward_kernel could not be configured");
  CK(cudaGetLastError());
  return PNB_OK;
}

// host buffers: staging grows on demand and is kept per host thread (there is no engine to own it)
extern "C" int pnb_pitch_only_host(const float *pitch_buf, size_t stride, long long n_units, const int *prev_period,
                                   const float *prev_gain, int *period, float *corr, float *gain, int *lag) {
  if (!pitch_buf || !period || !corr || !gain) return fail(PNB_ERR_ARG, "NULL argument");
  if (n_units < 1 || stride < 1728) return fail(PNB_ERR_ARG, "n_units must be >= 1 and stride >= 1728");
  struct Staging { float *buf = nullptr; int *i4 = nullptr; float *f3 = nullptr; long long cap = 0; int dev = -1; cudaStream_t st = nullptr; };
  static thread_local Staging g;
  int dev = 0;
  CK(cudaGetDevice(&dev));
  if (g.cap < n_units || g.dev != dev) {
    if (g.buf) { cudaFree(g.buf); cudaFree(g.i4); cudaFree(g.f3); g.buf = nullptr; }
    if (!g.st || g.dev != dev) CK(cudaStreamCreateWithFlags(&g.st, cudaStreamNonBlocking));
    CK(cudaMalloc((void **)&g.buf, (size_t)n_units * 1728 * sizeof(float)));
    CK(cudaMalloc((void **)&g.i4, (size_t)n_units * 3 * sizeof(int)));
    CK(cudaMalloc((void **)&g.f3, (size_t)n_units * 3 * sizeof(float)));
    g.cap = n_units; g.dev = dev;
  }
  const size_t n = (size_t)n_units;
  int *d_T = g.i4, *d_lag = g.i4 + n, *d_pT = g.i4 + 2 * n;
  float *d_corr = g.f3, *d_gain = g.f3 + n, *d_pg = g.f3 + 2 * n;
  CK(cudaMemcpy2DAsync(g.buf, 1728 * sizeof(float), pitch_buf, stride * sizeof(float), 1728 * sizeof(float), n, cudaMemcpyHostToDevice, g.st));
  if (prev_period) CK(cudaMemcpyAsync(d_pT, prev_period, n * sizeof(int), cudaMemcpyHostToDevice, g.st));
  if (prev_gain) CK(cudaMemcpyAsync(d_pg, prev_gain, n * sizeof(float), cudaMemcpyHostToDevice, g.st));
  int rc = pnb_pitch_only_device(g.buf, 1728, n_units, prev_period ? d_pT : nullptr, prev_gain ? d_pg : nullptr, d_T, d_corr, d_gain,
                                 lag ? d_lag : nullptr, g.st);
  if (rc) return rc;
  CK(cudaMemcpyAsync(period, d_T, n * sizeof(int), cudaMemcpyDeviceToHost, g.st));
  CK(cudaMemcpyAsync(corr, d_corr, n * sizeof(float), cudaMemcpyDeviceToHost, g.st));
  CK(cudaMemcpyAsync(gain, d_gain, n * sizeof(float), cudaMemcpyDeviceToHost, g.st));
  if (lag) CK(cudaMemcpyAsync(lag, d_lag, n * sizeof(int), cudaMemcpyDeviceToHost, g.st));
  CK(cudaStreamSynchronize(g.st));
  return PNB_OK;
}

extern "C" long long pnb_launch_count(const pnb_engine *e) { return e ? e->launches : 0; }
extern "C" int pnb_launches_per_call(const pnb_engine *e, int n_frames) {
  if (!e) return 0;
  // stage_in, analysis, the network, synthesis; without the history move of advance_line (at most one more launch per
  // call), and without the fix-up of a ragged session call in which a session runs fewer hops than the call (one more);
  // the resynthesis of a PNB_TRAIN_AUDIO engine is one launch more than its records alone; a PNB_NETWORK_ONLY engine's
  // call is pnb_compute_rnn_*: rows_stage, the network, rows_store; a PNB_SIGNAL_ONLY engine's is one pnb_analyze_*
  // (stage_in, analysis, rows_store) and one pnb_synthesize_* (rows_stage, synthesis)
  if (e->flags & PNB_SIGNAL_ONLY) return 5;
  if (e->flags & PNB_TRAIN_NETWORK) return train_grad_launches(e);  // one pnb_train_grad_* call, whatever n_frames
  const int net = (e->flags & PNB_NN_TENSOR) ? tc_network_launches(e, n_frames) : f32_network_launches(e, n_frames);
  if (e->flags & PNB_NETWORK_ONLY) return 2 + net;
  return 3 + net + ((e->flags & PNB_TRAIN_AUDIO) ? 1 : 0);
}
extern "C" size_t pnb_engine_bytes(const pnb_engine *e) {
  size_t n = 0;
  if (e)
    for (const auto &b : e->buffers) n += b.bytes;
  return n;
}
extern "C" int pnb_n_streams(const pnb_engine *e) { return e ? e->S : 0; }
extern "C" int pnb_max_frames(const pnb_engine *e) { return e ? e->Fmax : 0; }
