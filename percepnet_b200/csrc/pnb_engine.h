// pnb_engine.h -- the engine object behind the opaque pnb_engine handle.
#pragma once
#include <stddef.h>
#include <memory>
#include <vector>
#include "pnb_kernels.h"
#include "pnb_session_plan.h"
#include "pnb_state.h"
#include "../../include/percepnet_b200.h"
#include "../../include/pnb_nnet_layout.h"

struct pnb_tc_state;   // tensor-core path (pnb_nn_tc.cu)
struct pnb_f32_state;  // fp32 FMA path (pnb_nn_f32.cu)
struct pnb_train_state;  // PNB_TRAIN_NETWORK: gradients, Adam's moments, saved activations (pnb_train.cu)

constexpr int kGruH[5] = {512, 512, 512, 512, 128};  // hidden sizes of gru1..3, gru_gb, gru_rb (check_model)

struct pnb_engine {
  int S = 0, Fmax = 0, device = 0, sm_count = 0;
  // Active range (pnb_set_active_streams): a call advances slots [0, n_active) only.  Per-stream buffers keep the stride
  // S (slot s of hop slot t at row t*S + s), so the active rows of every hop slot are a contiguous prefix.
  int n_active = 0;
  unsigned flags = 0;
  cudaStream_t stream = nullptr;  // used by the host-buffer entry points
  pnb::Tables *d_tab = nullptr;

  // every device buffer whose size is fixed at pnb_create (engine_buffer)
  struct Buffer { void *p; size_t bytes; bool zero_on_reset; };
  std::vector<Buffer> buffers;

  struct { float *W = nullptr, *b = nullptr; } fc;  // the fc layer in the reference's layout (SURVEY.md App. B)

  // per-stream signal state
  // [S][5280 + c*Fmax*480], c <= kLineCalls: each stream's history line.  A call appends its hops behind the history and
  // the next call simply starts F*480 samples further on (line_off); only when the row is used up are the last
  // 5280 samples moved back to its start, once every c calls instead of after every call.
  float *d_pcm = nullptr;
  size_t pcm_stride = 0;
  size_t line_off = 0;
  float *d_synth = nullptr;
  int *d_last_period = nullptr;
  float *d_last_gain = nullptr;

  // per-call intermediates [F][S][...]
  float *d_feat = nullptr;
  float2 *d_zring = nullptr;  // [ring][S][400] carried spectra (see pnb_dsp.cu), slot = hop % ring
  float *d_ering = nullptr;   // [ring][S][34]
  int ring = 0;
  float2 *d_P = nullptr;
  float *d_Ex = nullptr;
  float *d_raw = nullptr;     // [F][S][68] training-data mode only
  unsigned char *d_sil = nullptr;
  float *d_gr = nullptr;
  int *d_tap_pitch = nullptr;
  float *d_tap_pitchf = nullptr;
  float *d_tap_g = nullptr;   // [F][S][34] gains as applied (PNB_KEEP_TAPS)

  // network state both paths share: conv2's output of the last hop and the GRU states in fp32, whose rows [0, S) hold
  // the state between calls (tensor: [S][H], updated in place; fp32: the front of its hop slots [chunk+1][S][H])
  float *c2 = nullptr;       // [S][512]
  float *h[5] = {};
  long hop = 0;  // hops processed since reset

  // Device staging of the host-buffer calls (every *_host entry point, pnb_submit_host_* and pnb_submit_train_records):
  // two slots, each an input and an output buffer, allocated on first use and only ever
  // grown.  Pipelined calls take slot submitted & 1 and copy on s_in / s_out (created for the first of them), ordered
  // with the call on `stream` by the slot's events; blocking calls borrow the slot the next pipelined call will take and
  // run on `stream` alone.
  struct Staging { void *in = nullptr, *out = nullptr; size_t in_bytes = 0, out_bytes = 0; };
  Staging stage[2];
  cudaStream_t s_in = nullptr, s_out = nullptr;
  cudaEvent_t ev_in[2] = {nullptr, nullptr}, ev_cmp[2] = {nullptr, nullptr}, ev_out[2] = {nullptr, nullptr};
  long long submitted = 0;  // pipelined calls so far

  // the network path's own buffers and packed weights; shared_ptr because its deleter is bound in the path's file,
  // where the type is complete
  std::shared_ptr<pnb_tc_state> tc;
  std::shared_ptr<pnb_f32_state> f32;
  std::shared_ptr<pnb_train_state> train;
  // PNB_TRAIN_NETWORK accumulation: the hops the held gradient counted while no pnb_train_accumulate has taken it yet
  // (0: none, or taken), and whether the accumulator holds anything (accumulated or imported) not yet finished
  long long train_hops = 0;
  bool train_open = false;
  // the hops of the pnb_train_forward_device call whose backward is still due (0: none).  Cleared by its backward,
  // a gradient call, pnb_set_active_streams, pnb_reset, pnb_train_adam and pnb_train_import of the weights: one
  // backward per forward, on the rows and with the weights that forward ran.
  int train_fwd_F = 0;
  int last_frames = 0;
  // An analysis (pnb_analyze_*) whose synthesis (pnb_synthesize_*) is still due, set by the analysis and cleared by the
  // synthesis or pnb_reset.  F: its hops, or 0 when none is pending.  Between the two halves the analysed streams are
  // mid-hop, so every call and state operation but the synthesis and network calls is refused.  A session split
  // (pnb_analyze_sessions_*) also keeps its list, its hops in list order (empty when every session runs F hops) and the
  // host copy of its row upload (row map, slot map, and for a ragged call the hops of every slot and the slots that stop
  // early).  The index staging that upload went through is reused by the next call, and the plan is already applied to
  // the pool, so the synthesis and a network call between the halves stage this copy again.  All empty for a slot split.
  struct PendingSplit {
    int F = 0;
    std::vector<int> ids, hops, up;
  };
  PendingSplit pending;
  long long launches = 0;  // kernel launches of the calls and state operations so far (pnb_launch_count; LaunchScope)
  // status word on the device: bit 0 = an activation left the domain in which the reference's tansig_approx is
  // defined (tensor path only; reported as PNB_ERR_DOMAIN by the synchronising entry points, cleared by pnb_reset);
  // bit 1 = pnb_import_states rejected a blob, [1] = the lowest rejected slot (reported once, then cleared; in session
  // mode pnb_import_sessions raises it and [1] is the lowest rejected session id)
  int *d_status = nullptr;  // [2]
  int *h_status = nullptr;  // [2] pinned host copy, refreshed by the synchronising entry points

  // Ordering: every call and every state operation (of slots or sessions, pnb_get_state / pnb_set_state and a grown
  // active range included) is enqueued through one ordered enqueue (enqueue_ordered), which makes the stream it is
  // issued on wait for ev_call before its first launch and records ev_call there after its last.  Each waits for the one
  // before, so ev_call stands for everything issued earlier on the engine, whichever stream it went to; pnb_flush and
  // pnb_wait wait for it too.  A failure after that enqueue started sets `poisoned`, for every one of them.
  cudaEvent_t ev_call = nullptr;
  bool call_recorded = false;    // ev_call has been recorded at least once
  // batched stream-state operations: staging of the slot indices, import verdicts, one blob of scratch
  int *h_idx[2] = {nullptr, nullptr};  // [idx_cap] pinned staging of the slot indices (session calls: row map and moves),
  int *d_idx[2] = {nullptr, nullptr};  // double-buffered, and their device copies
  cudaEvent_t ev_idx[2] = {nullptr, nullptr};  // the copy out of h_idx[k] has run
  int idx_slot = 0;
  size_t idx_cap = 0;            // ints: S, more in session mode
  int *d_ok = nullptr;           // [ok_cap] import: per-blob verdict of the device-side check
  size_t ok_cap = 0;
  void *d_blob1 = nullptr;       // one blob of device scratch: pnb_get_state / pnb_set_state
  // a call failed after it had started to enqueue work: the streams' state is undefined until pnb_reset
  bool poisoned = false;

  // Session pool (pnb_sessions_reserve): sessions [0, capacity) are resident in a slot or parked as a blob in d_park.
  // The host-side plan says which; every session call applies its plan when it is enqueued, like hop / line_off.
  bool sessions = false;
  pnb::SessionPool pool;
  char *d_park = nullptr;        // [capacity][kParkStride] parking blobs; magic 0 = a fresh (or rejected) session
  float *d_sgr = nullptr;        // pnb_process_sessions_host_*: g/r of the call in list order, grown on first use
  size_t sgr_bytes = 0;
  std::vector<int> plan_row, plan_up;       // scratch of a session call: row map, and what is uploaded (session_rows)
  std::vector<pnb::SessionMove> plan_moves;

  // optional per-kernel-class timing (pnb_profile_enable): CUDA events around every launch
  bool profiling = false;
  struct ProfRec { int cls; cudaEvent_t a, b; };
  std::vector<ProfRec> prof_pending;
  std::vector<cudaEvent_t> prof_pool;
  double prof_ms[PNB_NUM_KERNEL_CLASSES] = {0};
  long long prof_n[PNB_NUM_KERNEL_CLASSES] = {0};

  const float *tansig() const {
    return reinterpret_cast<const float *>(reinterpret_cast<const char *>(d_tab) + offsetof(pnb::Tables, tansig));
  }
};

// A zeroed device buffer (engine_alloc: of n T) whose size is fixed for the engine's life: pnb_destroy frees it, and
// pnb_reset zeroes it again when zero_on_reset (stream state).  engine_upload fills it from host memory instead; it is
// never reset.
cudaError_t engine_buffer(pnb_engine *e, void **p, size_t bytes, bool zero_on_reset, const void *src);
template <typename T>
cudaError_t engine_alloc(pnb_engine *e, T **p, size_t n, bool zero_on_reset) {
  return engine_buffer(e, reinterpret_cast<void **>(p), n * sizeof(T), zero_on_reset, nullptr);
}
template <typename T>
cudaError_t engine_upload(pnb_engine *e, T **p, const T *src, size_t n) {
  return engine_buffer(e, reinterpret_cast<void **>(p), n * sizeof(T), false, src);
}
constexpr bool kStreamState = true, kScratch = false;  // engine_alloc's zero_on_reset
// Sets pnb_last_error to msg; returns code.
int engine_fail(int code, const char *msg);

// The network paths' hooks, tensor-core (tc_*, pnb_nn_tc.cu) and fp32 FMA (f32_*, pnb_nn_f32.cu).  Return PNB_OK /
// a negative error.
// prepare: the path's weights and buffers, and the GRU states e->h in its layout
int tc_prepare(pnb_engine *e, const pnb_model *model);
int f32_prepare(pnb_engine *e, const pnb_model *model);
// the network of a call of F hops; hops: the per-slot hops of a ragged session call (device), or null
int tc_network(pnb_engine *e, int F, const int *hops, cudaStream_t st);
int f32_network(pnb_engine *e, int F, const int *hops, cudaStream_t st);
// launches of the network of a call of F hops
int tc_network_launches(const pnb_engine *e, int F);
int f32_network_launches(const pnb_engine *e, int F);
// the path's pieces of a stream's state (state_segs, pnb_state.cu): appended to seg[ns..]; returns the new count
int tc_state_segs(const pnb_engine *e, pnb::StateSeg *seg, int ns);
int f32_state_segs(const pnb_engine *e, pnb::StateSeg *seg, int ns);

// PNB_TRAIN_NETWORK (pnb_train.cu).  prepare: after f32_prepare, the trainer's buffers.  grad: the loss sums and the
// gradient of a call of F hops on windows [0, n_active) (records on the device; frames: device / host copies of the
// hops per window, or null).  adam: one step with the held gradient.  copy: what = 0 weights,
// 1 gradient, 2 m, 3 v between the device and train_params(e) floats of host memory, on st.  accum_prepare: the
// float64 accumulator, allocated once; accumulate: the held gradient times e->train_hops into it (1 launch); finish:
// the gradient from it, the accumulator zeroed, and the non-finite check (2 launches); accum_copy: its
// train_params(e) + 1 doubles to (out) or from mem, host or device memory, on st.
int f32_params(const pnb_engine *e, float **p, size_t *count);
int train_prepare(pnb_engine *e);
int train_grad(pnb_engine *e, const float *rec, size_t rec_stride, const int *frames, const int *h_frames, double *sums,
               int F, cudaStream_t st);
int train_grad_launches(const pnb_engine *e);
// forward: the caller's network input x (rows of F x 70 floats, not scaled) of windows [0, n_active) through the
// network from the state rows state_in (PNB_TRAIN_STATE_FLOATS each, or null: zero state), weights (device, blob order,
// or null) copied into the parameters first, the predictions out to the caller's rows (F x 68) and the state at each
// window's end to state_out (or null); lengths (device, h_lengths its host copy, or null: F): each window's hops.  The
// activations are kept for one backward.  backward: from the caller's dL/d(out) rows (F x 68) and dL/d(state out) rows
// (or null) of the last forward, the held gradient (copied to grad, device, when not null) and, when not null, dL/dx to
// the caller's rows (F x 70) and dL/d(state in) to its state rows.  Their launch counts depend on nothing but which of
// the optional arrays are given.
int train_forward(pnb_engine *e, const float *x, size_t x_stride, const float *weights, const float *state_in,
                  size_t state_in_stride, const int *lengths, const int *h_lengths, float *out, size_t out_stride,
                  float *state_out, size_t state_out_stride, int F, cudaStream_t st);
int train_backward(pnb_engine *e, const float *dout, size_t dout_stride, const float *dstate_out,
                   size_t dstate_out_stride, float *dx, size_t dx_stride, float *dstate_in, size_t dstate_in_stride,
                   float *grad, cudaStream_t st);
int train_forward_launches(const pnb_engine *e, bool state_in, bool lengths, bool state_out);
int train_backward_launches(const pnb_engine *e, bool dx, bool dstate_out, bool dstate_in);
int train_adam(pnb_engine *e, double lr, long long step, cudaStream_t st);
int train_copy(pnb_engine *e, int what, void *host, bool to_host, cudaStream_t st);
size_t train_params(const pnb_engine *e);
int train_accum_prepare(pnb_engine *e);
int train_accumulate(pnb_engine *e, cudaStream_t st);
int train_finish(pnb_engine *e, cudaStream_t st);
int train_accum_copy(pnb_engine *e, void *mem, bool out, cudaStream_t st);
// The PNB_TAP_TRAIN_* tap `what` of the last gradient or forward call: its device pointer and size in bytes, or PNB_ERR_ARG (set
// as the last error) on an engine without a trainer or before its first gradient call.
int train_tap(const pnb_engine *e, int what, const void **src, size_t *bytes);

// The marker of one kernel launch on behalf of an engine, constructed right before the launch and destroyed right
// after it: it counts the launch in e->launches and, when profiling and cls is a kernel class, records an event pair
// around it for that class (kUnprofiled: counted only).  Every launch of a call or state operation has its own marker,
// and nothing else counts launches.
constexpr int kUnprofiled = -1;
struct LaunchScope {
  pnb_engine *e; int idx;
  LaunchScope(pnb_engine *eng, int cls, cudaStream_t st);
  ~LaunchScope();
  cudaStream_t st;
};
