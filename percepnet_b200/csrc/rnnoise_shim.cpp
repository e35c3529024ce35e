// rnnoise_shim.cpp -- the reference's own single-stream API on top of the batched engine.
//
// Exports, with C++ linkage exactly like /root/reference/src/rnnoise.h:52-60 (the reference sources are
// all .cpp and the header has no extern "C"; SURVEY.md 0.8), the symbols an unmodified
// /root/reference/src/main.cpp imports:
//   int rnnoise_get_size();                                   src/denoise.cpp:348
//   int rnnoise_init(DenoiseState*, RNNModel*);               src/denoise.cpp:259
//   DenoiseState* rnnoise_create(RNNModel*);                  src/denoise.cpp:252
//   void rnnoise_destroy(DenoiseState*);                      src/denoise.cpp:326
//   float rnnoise_process_frame(DenoiseState*, float*, const float*, FILE*);   src/denoise.cpp:508
// By default a stream handle is a batch of one; it exists for drop-in correctness (percepNet_run), throughput
// comes from the pnb_* batch API.  model == NULL selects `percepnet_model_orig`, the symbol the
// generated src/nnet_data.cpp defines (dump_percepnet.py:149); it is referenced weakly so that hosts
// which always pass a model do not need to link one.
//
// PNB_SHIM_POOL=<slots> (opt-in; unset or 0 keeps one engine per handle) makes every handle a session of an engine
// shared by all handles with the same model pointer, network mode and device.  The first handle of such a group creates
// the engine with <slots> slots; concurrent rnnoise_process_frame calls of the group's handles are coalesced into one
// session call per batch of at most <slots> frames (pnb_shim_batcher.h).  The last rnnoise_destroy of a group destroys
// its engine.
#include <errno.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <mutex>
#include <string>
#include <vector>

#include "../../include/percepnet_b200.h"
#include "pnb_shim_batcher.h"

struct RNNModel;      // layout == pnb_model (include/pnb_nnet_layout.h)
struct ShimGroup;
struct DenoiseState { // opaque to callers (rnnoise.h:49)
  pnb_engine *engine; // unpooled: the handle's own engine; pooled: NULL
  float gr[68];
  ShimGroup *group;   // pooled: the shared engine this handle is a session of; unpooled: NULL
  int id;             // pooled: the session id in the group
};

extern const RNNModel percepnet_model_orig __attribute__((weak));

// ---- pooled handles ----------------------------------------------------------------------------------------------
static const int kMaxPoolSlots = 4096;  // the largest PNB_SHIM_POOL accepted

struct EngineCall {
  ShimGroup *g;
  int operator()(const int *ids, int k, const float *in, float *out, float *gr, std::string &err) const;
};

struct ShimGroup {
  const RNNModel *model;  // group key: model pointer, network flags, device ordinal
  unsigned flags;
  int device;
  pnb_engine *engine;
  std::mutex engine_mu;   // serialises the leader's calls with the session resets and pool growth of new handles
  pnb::FrameBatcher<EngineCall> batcher;
  std::vector<int> free_ids;  // ids of destroyed handles, reset when handed out again
  int next_id = 0, capacity, refs = 0;
  ShimGroup(const RNNModel *m, unsigned f, int dev, pnb_engine *e, int slots)
      : model(m), flags(f), device(dev), engine(e), batcher(EngineCall{this}, slots, PNB_FRAME, 2 * PNB_BANDS),
        capacity(slots) {}
};

int EngineCall::operator()(const int *ids, int k, const float *in, float *out, float *gr, std::string &err) const {
  std::lock_guard<std::mutex> lk(g->engine_mu);
  int rc = pnb_process_sessions_host_f32(g->engine, ids, k, in, PNB_FRAME, out, PNB_FRAME, 1, gr);
  if (rc != PNB_OK) err = pnb_last_error();
  return rc;
}

// the registry of live groups and the counters of destroyed ones; g_registry_mu is taken before any engine_mu
static std::mutex g_registry_mu;
static std::vector<ShimGroup *> g_groups;
static pnb::BatcherStats g_retired;

static void fold_stats(pnb::BatcherStats &acc, const pnb::BatcherStats &s) {
  acc.calls += s.calls;
  acc.frames += s.frames;
  if (s.largest > acc.largest) acc.largest = s.largest;
}

// with g_registry_mu held
static void drop_group_if_unused(ShimGroup *g) {
  if (g->refs > 0) return;
  for (size_t i = 0; i < g_groups.size(); i++)
    if (g_groups[i] == g) {
      g_groups.erase(g_groups.begin() + i);
      break;
    }
  fold_stats(g_retired, g->batcher.stats());
  pnb_destroy(g->engine);
  delete g;
}

// PNB_SHIM_POOL: 0 when unset, the slot count, or -1 (refused; the reason goes to stderr)
static int pool_slots(const char *who) {
  const char *s = getenv("PNB_SHIM_POOL");
  if (!s) return 0;
  char *end = NULL;
  errno = 0;
  long v = strtol(s, &end, 10);
  if (end == s || *end != '\0' || errno == ERANGE || v < 0 || v > kMaxPoolSlots) {
    fprintf(stderr, "%s: PNB_SHIM_POOL=\"%s\" is not a slot count in [0, %d]\n", who, s, kMaxPoolSlots);
    return -1;
  }
  return (int)v;
}

static int pooled_init(DenoiseState *st, const RNNModel *m, unsigned flags, int device, int slots) {
  int dev = pnb_resolve_device(device);
  if (dev < 0) {
    fprintf(stderr, "rnnoise_init: %s\n", pnb_last_error());
    return dev;
  }
  std::lock_guard<std::mutex> lk(g_registry_mu);
  ShimGroup *g = NULL;
  for (size_t i = 0; i < g_groups.size() && !g; i++)
    if (g_groups[i]->model == m && g_groups[i]->flags == flags && g_groups[i]->device == dev) g = g_groups[i];
  if (!g) {  // the first handle of the group sets its slot count
    pnb_engine *e = NULL;
    int rc = pnb_create(&e, slots, 1, reinterpret_cast<const pnb_model *>(m), flags, dev);
    if (rc == PNB_OK) rc = pnb_sessions_reserve(e, slots);
    if (rc != PNB_OK) {
      fprintf(stderr, "rnnoise_init: %s\n", pnb_last_error());
      pnb_destroy(e);
      return rc;
    }
    g = new ShimGroup(m, flags, dev, e, slots);
    g_groups.push_back(g);
  }
  int id, rc = PNB_OK;
  if (!g->free_ids.empty()) {  // a recycled id: clear what its previous owner left
    id = g->free_ids.back();
    std::lock_guard<std::mutex> le(g->engine_mu);
    rc = pnb_reset_sessions(g->engine, &id, 1, NULL);
    if (rc == PNB_OK) g->free_ids.pop_back();
  } else {  // a new id: sessions are fresh from pnb_sessions_reserve; double the pool when it is full
    id = g->next_id;
    if (id == g->capacity) {
      std::lock_guard<std::mutex> le(g->engine_mu);
      rc = pnb_sessions_reserve(g->engine, 2 * g->capacity);
      if (rc == PNB_OK) g->capacity *= 2;
    }
    if (rc == PNB_OK) g->next_id++;
  }
  if (rc != PNB_OK) {
    fprintf(stderr, "rnnoise_init: %s\n", pnb_last_error());
    drop_group_if_unused(g);
    return rc;
  }
  g->refs++;
  st->group = g;
  st->id = id;
  return 0;
}

static void pooled_destroy(DenoiseState *st) {
  std::lock_guard<std::mutex> lk(g_registry_mu);
  ShimGroup *g = st->group;
  g->free_ids.push_back(st->id);
  g->refs--;
  drop_group_if_unused(g);
}

// Process-wide counters of the pooled shim, a test and measurement hook: out[0] live groups, out[1] session calls
// issued, out[2] frames advanced through them, out[3] the largest batch (these three since the process started), and
// out[4] parks, out[5] unparks summed over the live groups' engines (pnb_session_stats).
extern "C" int pnb_shim_pool_stats(long long *out) {
  if (!out) return PNB_ERR_ARG;
  std::lock_guard<std::mutex> lk(g_registry_mu);
  pnb::BatcherStats s = g_retired;
  long long parks = 0, unparks = 0;
  for (size_t i = 0; i < g_groups.size(); i++) {
    fold_stats(s, g_groups[i]->batcher.stats());
    long long ps[3] = {0, 0, 0};
    std::lock_guard<std::mutex> le(g_groups[i]->engine_mu);
    if (pnb_session_stats(g_groups[i]->engine, ps) == PNB_OK) {
      parks += ps[0];
      unparks += ps[1];
    }
  }
  out[0] = (long long)g_groups.size();
  out[1] = s.calls;
  out[2] = s.frames;
  out[3] = s.largest;
  out[4] = parks;
  out[5] = unparks;
  return PNB_OK;
}

// Declared by the reference (src/rnnoise.h:62-64) but defined nowhere in it (SURVEY.md 3.2): here they read the
// binary weight file of pnb_model_load_blob, so a host can run without compiling nnet_data.cpp.
RNNModel *rnnoise_model_from_file(FILE *f) {
  if (!f) return NULL;
  pnb_model *m = NULL;
  if (pnb_model_load_stream(f, &m) != PNB_OK) {
    fprintf(stderr, "rnnoise_model_from_file: %s\n", pnb_last_error());
    return NULL;
  }
  return reinterpret_cast<RNNModel *>(m);
}
void rnnoise_model_free(RNNModel *model) { pnb_model_free(reinterpret_cast<pnb_model *>(model)); }

int rnnoise_get_size() { return (int)sizeof(DenoiseState); }

int rnnoise_init(DenoiseState *st, RNNModel *model) {
  memset(st, 0, sizeof *st);
  const RNNModel *m = model ? model : &percepnet_model_orig;
  if (!m) {
    fprintf(stderr, "rnnoise_init: no model given and percepnet_model_orig is not linked\n");
    return -1;
  }
  // PNB_SHIM_NN=tensor runs the network on the tensor cores (2.8x lower latency per frame; g/r within 1e-5 of
  // the reference instead of 5e-7); the default keeps the fp32 network, which also reproduces the reference
  // outside tansig_approx's defined range (DESIGN.md 1)
  const char *nn = getenv("PNB_SHIM_NN");
  const unsigned flags = (nn && strcmp(nn, "tensor") == 0) ? PNB_NN_TENSOR : PNB_NN_FP32;
  // PNB_DEVICE=<ordinal> picks the GPU; otherwise the calling thread's current CUDA device (device 0 in a fresh process)
  const char *dv = getenv("PNB_DEVICE");
  // PNB_SHIM_POOL=<slots>: the handle becomes a session of its group's shared engine
  const int slots = pool_slots("rnnoise_init");
  if (slots < 0) return PNB_ERR_ARG;
  if (slots > 0) return pooled_init(st, m, flags, dv ? atoi(dv) : -1, slots);
  int rc = pnb_create(&st->engine, 1, 1, reinterpret_cast<const pnb_model *>(m), flags, dv ? atoi(dv) : -1);
  if (rc != PNB_OK) {
    fprintf(stderr, "rnnoise_init: %s\n", pnb_last_error());
    return rc;
  }
  return 0;
}

DenoiseState *rnnoise_create(RNNModel *model) {
  DenoiseState *st = (DenoiseState *)malloc(rnnoise_get_size());
  if (!st) return NULL;
  if (rnnoise_init(st, model) != 0) {  // no CPU fallback: the caller gets NULL and the reason on stderr
    free(st);
    fprintf(stderr, "rnnoise_create: cannot create the CUDA engine (there is no CPU path)\n");
    return NULL;
  }
  return st;
}

void rnnoise_destroy(DenoiseState *st) {
  if (!st) return;
  if (st->group)
    pooled_destroy(st);
  else
    pnb_destroy(st->engine);
  free(st);
}

float rnnoise_process_frame(DenoiseState *st, float *out, const float *in, FILE *f_feature) {
  if (!st || (!st->engine && !st->group)) {
    fprintf(stderr, "rnnoise_process_frame: no engine (rnnoise_create failed?)\n");
    abort();  // the reference would dereference NULL here; a frame cannot be skipped silently
  }
  if (st->group) {  // one frame of a batch of the group's concurrent callers; returns when this frame is done
    std::string err;
    if (st->group->batcher.process(st->id, in, out, st->gr, &err) != PNB_OK) {
      fprintf(stderr, "rnnoise_process_frame: %s\n", err.c_str());
      abort();
    }
  } else {
    int rc = pnb_process_host_f32(st->engine, in, PNB_FRAME, out, PNB_FRAME, 1, st->gr);
    if (rc != PNB_OK) {
      fprintf(stderr, "rnnoise_process_frame: %s\n", pnb_last_error());
      abort();
    }
  }
  if (f_feature) {  // src/denoise.cpp:533-534
    fwrite(st->gr, sizeof(float), 34, f_feature);
    fwrite(st->gr + 34, sizeof(float), 34, f_feature);
  }
  return 0;  // src/denoise.cpp:546
}
