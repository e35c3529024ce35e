/*
 * percepnet_b200.h -- C-ABI of the H100-native PercepNet enhancement hot path.
 *
 * Plain pointers and sizes only (no torch / C++ types).  Two layers of entry points:
 *
 *  1. the batched-streams engine (pnb_*): S independent 48 kHz streams advance together,
 *     F hops of 480 samples per call.  This is what a host integrates for throughput.
 *  2. the reference's own single-stream API (rnnoise_create / rnnoise_process_frame /
 *     rnnoise_destroy, C++ linkage like /root/reference/src/rnnoise.h:52-60) lives in
 *     librnnoise_b200.so (percepnet_b200/csrc/rnnoise_shim.cpp) on top of this ABI, so the
 *     unmodified /root/reference/src/main.cpp links against it.
 *
 * What each entry point replaces in the reference (paths relative to /root/reference):
 *   pnb_create          rnnoise_create + rnnoise_init            src/denoise.cpp:252-280
 *                       + check_init table construction           src/denoise.cpp:186-214
 *                       + weight ingest of `const RNNModel*`      src/nnet_data.h:6-26
 *   pnb_process_*       rnnoise_process_frame for S streams x F hops   src/denoise.cpp:508-547
 *                       (compute_frame_features :372, compute_rnn src/rnn.cpp:42,
 *                        pitch_filter :436, interp_band_gain :162, frame_synthesis :352)
 *   pnb_process_*_i16   the int16 I/O conversions of the CLI      src/main.cpp:30-39
 *   pnb_destroy         rnnoise_destroy                           src/denoise.cpp:326-331
 *   pnb_reset           the memset in rnnoise_init                src/denoise.cpp:260
 *
 * Frame contract (src/rnnoise.h:60, SURVEY.md 8b): hops of exactly 480 float samples at
 * 48 kHz, any amplitude scale; output hop t carries input hop t-6.  Streams are laid out
 * stream-major: sample n of stream s is at base[s*stride + n].
 *
 * All functions return PNB_OK (0) or a negative error code; pnb_last_error() gives text.
 * There is no CPU fallback: without a usable CUDA device pnb_create fails with
 * PNB_ERR_NO_DEVICE.
 */
#ifndef PERCEPNET_B200_H
#define PERCEPNET_B200_H

#include <stddef.h>
#include "pnb_nnet_layout.h"

#ifdef __cplusplus
extern "C" {
#endif

#define PNB_FRAME 480        /* FRAME_SIZE, src/denoise.cpp:19 */
#define PNB_BANDS 34         /* NB_BANDS,   src/denoise.cpp:35 */
#define PNB_FEATURES 70      /* NB_FEATURES, src/denoise.cpp:40 */
#define PNB_LATENCY_FRAMES 6 /* 5 hops look-ahead + 1 hop overlap-add */

enum {
  PNB_OK = 0,
  PNB_ERR_ARG = -1,
  PNB_ERR_CUDA = -2,
  PNB_ERR_NO_DEVICE = -3,
  PNB_ERR_ALLOC = -4,
  PNB_ERR_DOMAIN = -5  /* PNB_NN_TENSOR only: a pre-activation reached |x| >= 8.5e7, where the reference's tansig_approx
                          (src/vec.h:63) overflows its float->int conversion (undefined behaviour; on x86 "tanh" returns
                          its argument).  The tensor path does not reproduce that: outputs since the last pnb_reset are not
                          the reference's.  Reported by the synchronising entry points (pnb_process_host_*, pnb_wait,
                          pnb_check); sticky until pnb_reset.  The fp32 path (PNB_NN_FP32) follows the reference there too. */
};

/* pnb_create flags */
enum {
  PNB_NN_FP32 = 0,       /* network contraction in fp32 FMA (BASELINE.json config 2)                  */
  PNB_NN_TENSOR = 1,     /* network contraction on wgmma tensor cores, split-fp16 operands, fp32 accumulate */
  PNB_POSTFILTER = 2,    /* apply the envelope post-filter (src/denoise.cpp:216-250) to g; off in the reference */
  PNB_KEEP_TAPS = 4,     /* keep per-frame intermediates of the last call readable through pnb_read_tap    */
  PNB_CONV_WIDE = 16,    /* PNB_NN_TENSOR only: conv1 / conv2 with three bf16 terms per operand (six tensor-core products)
                            instead of two (three).  Two terms reproduce the double-precision network to 7e-6 on g/r for
                            input at the CLI's amplitude scale (PCM / 32768, |x| <= 1) and to 4e-4 at worst for float
                            input hundreds to thousands of times louder (the reference's own fp32 arithmetic: 3e-5 there);
                            three terms stay within 2.1e-5 at every scale and cost 8 % of the throughput.  The mode is
                            per engine, never per input, so a stream's result does not depend on its neighbours.          */
  PNB_TRAIN_DATA = 8,    /* training-data generator (pnb_train_records_*): n_streams = 2 x pairs, no network,
                            no synthesis; model may be NULL; the pnb_process_* entry points are refused      */
  PNB_TRAIN_AUDIO = 32,  /* with PNB_TRAIN_DATA only: the generator also resynthesises every noisy file with its own
                            labels, as train() writes test_output.pcm (pnb_train_audio_*, which replace
                            pnb_train_records_* / pnb_submit_train_records on such an engine)                 */
  PNB_NETWORK_ONLY = 64, /* the network alone: an engine for pnb_compute_rnn_* and pnb_score_records_*, without the
                            signal-path buffers of a PCM engine (history lines, overlap-add and pitch memory, spectrum
                            rings, per-call spectra; about 14.7 GB at 16 384 streams x 100 hops).  pnb_process_*,
                            pnb_submit_*, pnb_train_* and pnb_sessions_reserve are refused with PNB_ERR_ARG before
                            anything is enqueued.  Not with PNB_TRAIN_DATA, PNB_TRAIN_AUDIO or PNB_POSTFILTER; with
                            PNB_KEEP_TAPS the features, g/r and PNB_TAP_NN_* taps are readable and the other taps are
                            refused.  State blobs: export writes the network part and zeroes the signal part, import
                            takes the network part and ignores the signal part, so blobs move both ways between this
                            engine and a PCM engine of the same network path. */
  PNB_SIGNAL_ONLY = 128, /* the signal path alone: an engine for pnb_analyze_* / pnb_synthesize_*, with g/r from the caller.
                            model may be NULL and is ignored; no fc weights, network state or network buffers are
                            allocated.  Every other call, pnb_train_* and pnb_sessions_reserve are refused with PNB_ERR_ARG
                            before anything is enqueued.  Not with PNB_NN_TENSOR, PNB_CONV_WIDE, PNB_TRAIN_DATA,
                            PNB_TRAIN_AUDIO or PNB_NETWORK_ONLY; with PNB_POSTFILTER and PNB_KEEP_TAPS (the PNB_TAP_NN_*
                            taps are refused).  State blobs: export writes the signal part and zeroes the network part,
                            import takes the signal part and ignores the network part, so blobs move both ways between
                            this engine and a PCM engine. */
  PNB_TRAIN_NETWORK = 256 /* a PNB_NETWORK_ONLY engine that also trains its fp32 network (pnb_train_*): n_streams windows per
                            step, max_frames_per_call the window length T.  Its parameters are the fp32 path's weight
                            buffers, so pnb_compute_rnn_* / pnb_score_records_* on it run the weights of the last Adam step
                            in the deployed tansig arithmetic.  PNB_NN_FP32 only: not with PNB_NN_TENSOR, PNB_CONV_WIDE,
                            PNB_TRAIN_DATA, PNB_TRAIN_AUDIO, PNB_POSTFILTER or PNB_SIGNAL_ONLY.  Besides what a network-only
                            engine holds it keeps the gradient and Adam's two moments (3 x 31.9 MB) and the activations one
                            gradient call saves for its backward pass, about 72 KB per frame of n_streams x T (128 windows
                            x 2000 hops: 18.5 GB); n_streams x T at most 65535 x 64. */
};

typedef struct pnb_engine pnb_engine;

/* model: the reference's weight layout (a `const RNNModel*` from a compiled nnet_data.cpp may be
 * passed as is); the weights are copied to the device, the caller's arrays are not retained. */
int pnb_create(pnb_engine **out, int n_streams, int max_frames_per_call, const pnb_model *model,
               unsigned flags, int device);   /* device: CUDA ordinal, or -1 = the calling thread's current device */
void pnb_destroy(pnb_engine *e);
int pnb_reset(pnb_engine *e);
/* The CUDA ordinal pnb_create(..., device) would use (device -1 = the calling thread's current device), or the negative
 * error code pnb_create would return for it (PNB_ERR_NO_DEVICE, PNB_ERR_CUDA, PNB_ERR_ARG).  Creates nothing; lets a
 * host key per-device resources without linking the CUDA runtime itself. */
int pnb_resolve_device(int device);

/* Binary weight file (percepnet_b200.weights.PackedModel.save_blob): the arrays of the generated nnet_data.cpp
 * as raw float32, 32 MB instead of 180 MB of C source and no 46 s compile.  The returned model owns its arrays;
 * release it with pnb_model_free (after pnb_create has copied it, at any time). */
int pnb_model_load_blob(const char *path, pnb_model **out);
/* the same from an open stream (a FILE* positioned at the start of the blob; passed as void* to keep <stdio.h> out
 * of this header); the stream is left open, positioned behind the blob */
int pnb_model_load_stream(void *file, pnb_model **out);
void pnb_model_free(pnb_model *m);

/* Host buffers (pageable or pinned).  in/out: the active rows (n = pnb_active_streams(e), n_streams unless
 * pnb_set_active_streams changed it) of n_frames*480 samples, row strides in elements.  in may equal out.  gr (NULL ok)
 * receives the raw network outputs the reference fwrite()s per frame (src/denoise.cpp:533-534) as [n_frames][n][68] =
 * 34 g then 34 r.  Blocking: returns when out (and gr) are complete. */
int pnb_process_host_f32(pnb_engine *e, const float *in, size_t in_stride, float *out, size_t out_stride,
                         int n_frames, float *gr);

/* int16 PCM wire format with the CLI's conversions (src/main.cpp:34,36): x = s/32768.f in,
 * (short)(y*32768) out (C truncation; output past full scale wraps to its low 16 bits, as the CLI built for x86-64
 * does).  The first-hop drop of main.cpp:37-38 is the caller's. */
int pnb_process_host_i16(pnb_engine *e, const short *in, size_t in_stride, short *out, size_t out_stride,
                         int n_frames, float *gr);

/* Pipelined host entry for sustained throughput (in/out: the active rows, as above): enqueues host->device copy,
 * processing and device->host copy
 * on internal streams and returns; the copies of neighbouring calls overlap the kernels.  At most two calls are
 * in flight (a third blocks until the oldest completed).  Buffers must stay valid -- and should be pinned --
 * until pnb_wait() returns.  Calls are processed in submission order (the streams' state advances in order). */
int pnb_submit_host_f32(pnb_engine *e, const float *in, size_t in_stride, float *out, size_t out_stride, int n_frames);
int pnb_submit_host_i16(pnb_engine *e, const short *in, size_t in_stride, short *out, size_t out_stride, int n_frames);
/* Waits on the host for every call and state operation issued on the engine, on any stream, then reports the engine's
 * status: PNB_OK, PNB_ERR_DOMAIN, or PNB_ERR_CUDA -- or, once, PNB_ERR_ARG when pnb_import_states rejected a blob since
 * the last report. */
int pnb_wait(pnb_engine *e);
/* pnb_wait, after everything enqueued on `cuda_stream` so far has run. */
int pnb_check(pnb_engine *e, void *cuda_stream);

/* Device buffers on the engine's device; asynchronous on cuda_stream (a cudaStream_t, NULL = default
 * stream).  in/out hold the active rows as above; d_gr (NULL ok) as above, in device memory.
 * Order: the calls and state operations of one engine run in the order they are issued, on whatever streams they are
 * issued on.  A call starts after everything enqueued on its cuda_stream before it and after the engine's previous call
 * or state operation; d_out (and d_gr) are complete in cuda_stream's order behind it. */
int pnb_process_device_f32(pnb_engine *e, const float *d_in, size_t in_stride, float *d_out, size_t out_stride,
                           int n_frames, float *d_gr, void *cuda_stream);
int pnb_process_device_i16(pnb_engine *e, const short *d_in, size_t in_stride, short *d_out, size_t out_stride,
                           int n_frames, float *d_gr, void *cuda_stream);

/* pnb_process_device_* without d_gr.  pnb_flush(e, stream) makes `stream` wait for every call and state operation
 * issued on the engine so far, on any stream: d_out is then complete in that stream's order, and on the host after
 * pnb_wait / pnb_check. */
int pnb_submit_device_f32(pnb_engine *e, const float *d_in, size_t in_stride, float *d_out, size_t out_stride,
                          int n_frames, void *cuda_stream);
int pnb_submit_device_i16(pnb_engine *e, const short *d_in, size_t in_stride, short *d_out, size_t out_stride,
                          int n_frames, void *cuda_stream);
int pnb_flush(pnb_engine *e, void *cuda_stream);

/* Training-data generator: the per-frame loop of the reference's train() (src/denoise.cpp:600-787, as shipped:
 * gains fixed at 1, no biquads, the second file is the finished noisy mixture, TEST defined so g is post-filtered).
 * The engine must have been created with PNB_TRAIN_DATA and n_streams = 2 x n_pairs.  speech/noisy hold n_pairs
 * rows of int16 PCM (row strides in samples); for pair p and frame t of the call the 138 floats
 *   Ey_lookahead[34] Ephaty[34] T pitchcorr g[34] r[34]                      (src/denoise.cpp:761-773)
 * are written to records + p*records_stride + t*138 -- a row is what train() writes to its <output> file for that
 * pair of files.  State carries over between calls, so a long pair of files can be fed in chunks of at most
 * max_frames_per_call frames.  Refused on a PNB_TRAIN_AUDIO engine (its audio would have gaps): use pnb_train_audio_*. */
#define PNB_RECORD_FLOATS 138
int pnb_train_records_host(pnb_engine *e, const short *speech, size_t speech_stride, const short *noisy,
                           size_t noisy_stride, int n_frames, float *records, size_t records_stride);
/* Pipelined form (pair it with pnb_wait, like pnb_submit_host_*): the copies of neighbouring calls overlap the
 * kernels; the buffers of a call must stay untouched until pnb_wait returns or two further calls were submitted. */
int pnb_submit_train_records(pnb_engine *e, const short *speech, size_t speech_stride, const short *noisy,
                             size_t noisy_stride, int n_frames, float *records, size_t records_stride);
int pnb_train_records_device(pnb_engine *e, const short *d_speech, size_t speech_stride, const short *d_noisy,
                             size_t noisy_stride, int n_frames, float *d_records, size_t records_stride,
                             void *cuda_stream);

/* Training data with its ideal-gain audio (PNB_TRAIN_DATA | PNB_TRAIN_AUDIO engines only).  records receive exactly
 * what pnb_train_records_* writes.  Row p of audio (audio + p*audio_stride, audio_stride >= n_frames*480) receives
 * n_frames x 480 int16 samples: what train() writes to test_output.pcm for pair p over these frames
 * (src/denoise.cpp:742-759): the noisy frame resynthesised with its own labels -- g post-filtered, pitch_filter with r
 * unless the noisy frame is silent, interp_band_gain(g), frame_synthesis -- and converted by clamping, then truncating:
 * (short)fmaxf(-32768, fminf(32767, y)) at scale 1 (NaN gives 32767), not the (short)(y*32768) of pnb_process_*_i16.
 * Every frame is written (nothing is dropped); output frame t carries noisy input frame t - 6.  State carries over
 * between calls, so the audio does not depend on how frames are grouped into calls; pnb_reset and the state blob
 * cover the overlap-add memory.  train()'s test_input.pcm is the noisy input itself (its clamp is a no-op on int16).
 * Refused with PNB_ERR_ARG like pnb_train_records_*, and also on an engine without PNB_TRAIN_AUDIO, a NULL audio
 * pointer or a short audio_stride.  A call issues one launch more than pnb_train_records_*. */
int pnb_train_audio_host(pnb_engine *e, const short *speech, size_t speech_stride, const short *noisy,
                         size_t noisy_stride, int n_frames, float *records, size_t records_stride, short *audio,
                         size_t audio_stride);
int pnb_train_audio_device(pnb_engine *e, const short *d_speech, size_t speech_stride, const short *d_noisy,
                           size_t noisy_stride, int n_frames, float *d_records, size_t records_stride, short *d_audio,
                           size_t audio_stride, void *cuda_stream);

/* The network alone: the batched compute_rnn (src/rnnoise.h:68, src/rnn.cpp:42) on caller-supplied inputs, to score a
 * model on features or training records exactly as the engine runs it.
 *   format       PNB_RNN_FEATURES: 70 floats per hop, the network input as create_features makes it
 *                (src/denoise.cpp:487-496, = PNB_TAP_FEATURES).  PNB_RNN_RECORDS: 138 floats per hop, a record of
 *                train() / pnb_train_records_*; the device takes features = {30*rec[0..67], rec[68], rec[69]} (one fp32
 *                multiply, as create_features and rnn_train.py's CppRawListDataset scale them) and ignores the labels
 *                rec[70..137].
 *   in / d_in    the active rows [0, n) (n = pnb_active_streams(e)), stream-major: row i holds n_frames consecutive hops,
 *                at in + i*in_stride, in_stride >= n_frames * (70 or 138) floats.
 *   gr / d_gr    row i receives n_frames x 68 floats (34 g then 34 r per hop) at gr + i*gr_stride, gr_stride >=
 *                n_frames*68.  Unlike the [n_frames][n][68] g/r of pnb_process_*, hop t of row i lines up with the
 *                labels rec[t][70..137] of the same record row.
 * A call advances the network state of every active slot (conv histories, GRU states, conv2 output) by n_frames hops,
 * computing compute_rnn once per hop in order, exactly as a pnb_process_* call does after its analysis.  It does not
 * touch the slot's signal state (history, overlap-add memory, pitch memory, spectra), so between two pnb_process_*
 * calls it is the batched compute_rnn(&st->rnn, ...) on a DenoiseState between two frames.  PNB_TAP_FEATURES and
 * PNB_TAP_GR read the call; the other per-frame taps are unspecified after it.  Ordering and blocking are those of
 * pnb_process_device_* / pnb_process_host_*; on a PNB_NN_TENSOR engine, features that drive a pre-activation out of the
 * domain raise PNB_ERR_DOMAIN the same way (features are not otherwise validated).  Refused with PNB_ERR_ARG before
 * anything is enqueued: NULL pointers, format not 0 or 1, n_frames outside [1, max_frames], short strides, a
 * PNB_TRAIN_DATA engine, an engine in session mode; a poisoned engine returns PNB_ERR_CUDA.  A call issues the
 * network's launches plus two. */
enum { PNB_RNN_FEATURES = 0, PNB_RNN_RECORDS = 1 };
int pnb_compute_rnn_device(pnb_engine *e, int format, const float *d_in, size_t in_stride, int n_frames,
                           float *d_gr, size_t gr_stride, void *cuda_stream);
int pnb_compute_rnn_host(pnb_engine *e, int format, const float *in, size_t in_stride, int n_frames,
                         float *gr, size_t gr_stride);

/* Scoring on the device: pnb_compute_rnn_* on training records (PNB_RNN_RECORDS) with rnn_train.py's CustomLoss
 * (rnn_train.py:153-176, gamma = 0.5) reduced against the records' own labels, so only four numbers per row leave the
 * device.  The network input is staged and the network state advanced exactly as a pnb_compute_rnn_* call of the same
 * records does.
 *   rec / d_rec  the active rows [0, n) of records, as pnb_compute_rnn_* takes them; rec_stride >= n_frames * 138.
 *   frames       host array of n ints in [0, n_frames] (reusable when the call returns), or NULL for n_frames each:
 *                row i's loss counts its first frames[i] hops only (the padding of a shorter file drops out).  Every
 *                row still advances by n_frames hops.
 *   sums / d_sums  overwritten with n x 4 float64: {sum dg^2, sum dg^4, sum dr^2, count} per row, over the counted hops
 *                and the 34 bands, where dg = sqrt(g) - sqrt(g_hat), dr = sqrt(1 - r) - sqrt(1 - r_hat), the labels
 *                g, r = rec[t][70..103], rec[t][104..137] and count = 34 * frames[i].  CustomLoss's terms are
 *                sum dg^2 / count, 10 sum dg^4 / count and sum dr^2 / count.  NaN propagates (a label r > 1 makes
 *                that row's sum dr^2 NaN).  A row's sums depend on its own records only, in a fixed order: they are the
 *                same bits whatever other rows, n_streams or active range the call has.
 *   gr / d_gr    NULL, or g/r written as pnb_compute_rnn_* writes them (same bits), gr_stride >= n_frames * 68.
 * Allowed where pnb_compute_rnn_* is (PCM and PNB_NETWORK_ONLY engines); ordering, blocking, PNB_ERR_DOMAIN and the
 * refusals are pnb_compute_rnn_*'s, and also NULL sums and frames[i] outside [0, n_frames].  A call without gr issues
 * as many launches as a pnb_compute_rnn_* call of n_frames hops; with gr, one more. */
int pnb_score_records_device(pnb_engine *e, const float *d_rec, size_t rec_stride, int n_frames, const int *frames,
                             double *d_sums, float *d_gr, size_t gr_stride, void *cuda_stream);
int pnb_score_records_host(pnb_engine *e, const float *rec, size_t rec_stride, int n_frames, const int *frames,
                           double *sums, float *gr, size_t gr_stride);

/* Training (PNB_TRAIN_NETWORK engines): rnn_train.py's step -- CustomLoss (gamma = 0.5, C4 = 10) of its PercepNet on a
 * batch of windows, the gradient of every parameter, and a torch.optim.Adam step (defaults: betas 0.9 / 0.999, eps 1e-8,
 * no weight decay, no amsgrad) -- on the device, in fp32 FMA.  The model is PercepNet.forward (rnn_train.py:105-145) with
 * exact tanh and sigmoid (not the tansig table of inference), torch's GRU gate formula, and every window starting from
 * zero GRU state and zero conv history.  Nothing carries between calls; the slots' network state is not touched.
 *   pnb_train_grad_*  rec / d_rec hold the active rows [0, n) of records as pnb_score_records_* takes them (network input
 *                     {30 rec[0..67], rec[68], rec[69]}), one window per row, rec_stride >= n_frames * 138.  frames: host
 *                     array of n ints in [1, n_frames] (window i ends after frames[i] hops), or NULL for n_frames each;
 *                     the hops past a window's end contribute nothing to the loss or the gradient, whatever they hold
 *                     (NaN included).  sums / d_sums: n x 4 float64 as pnb_score_records_* writes them, for the trainer's
 *                     exact-activation predictions.  The gradient of the loss -- the mean over the counted hops x 34 bands
 *                     of all windows -- overwrites the engine's gradient buffer.  It is computed at the output
 *                     pre-activations in closed form, g: -dg (1 + 2 C4 dg^2) sqrt(p) (1 - p), r: dr p sqrt(1 - p); this
 *                     equals torch's autograd wherever that is finite, and is its finite limit where a sigmoid output
 *                     rounds to exactly 0 or 1 in fp32, where torch's autograd returns NaN (rnn_train.py:198's "CustomLoss
 *                     cause Nan error").  That is the one deliberate difference from torch.  A gradient with a non-finite
 *                     value (from non-finite records inside a window or non-finite weights) raises the domain bit: the next
 *                     synchronising entry point returns PNB_ERR_DOMAIN, sticky until pnb_reset.  No floating-point atomics:
 *                     the loss and the gradient of a call are the same bits from run to run, on any stream, host or device
 *                     entry.  Ordering, blocking and the refusals are those of pnb_score_records_* (frames in [1, n_frames]);
 *                     also refused on any engine without PNB_TRAIN_NETWORK.  A call issues pnb_launches_per_call(e, .)
 *                     launches, whatever n_frames.
 *   pnb_train_adam    one Adam step with the held gradient, lr >= 0 and finite, step >= 1 the step number (torch's
 *                     state['step'], for the bias corrections), asynchronous on cuda_stream and ordered like a call.  When
 *                     the last gradient call flagged a non-finite value the step is skipped on the device: weights and
 *                     moments stay as they are, with no host synchronisation.  The arithmetic is torch's single-tensor
 *                     CPU step: m = lerp(m, g, 0.1) (fused), v = fma(0.001 g, g, 0.999 v), p += (-lr / bc1) m / (sqrt(v) /
 *                     sqrt(bc2) + eps).  pnb_reset touches neither weights nor moments.
 *   pnb_train_export / pnb_train_import  one array as a flat float32 vector in PNBW blob order (the ten layers in
 *                     RNNModel order, each layer's weights, recurrent weights, bias; 7 962 564 floats): the weights, the
 *                     gradient (export only) or Adam's m or v.  Both wait for the engine's earlier work and return when
 *                     the copy is complete; export needs bytes >= the vector, import exactly the vector. */
enum { PNB_TRAIN_WEIGHTS = 0, PNB_TRAIN_GRADIENT = 1, PNB_TRAIN_ADAM_M = 2, PNB_TRAIN_ADAM_V = 3 };
int pnb_train_grad_host(pnb_engine *e, const float *rec, size_t rec_stride, int n_frames, const int *frames, double *sums);
int pnb_train_grad_device(pnb_engine *e, const float *d_rec, size_t rec_stride, int n_frames, const int *frames,
                          double *d_sums, void *cuda_stream);
int pnb_train_adam(pnb_engine *e, double lr, long long step, void *cuda_stream);
int pnb_train_export(pnb_engine *e, int what, void *dst, size_t bytes);
int pnb_train_import(pnb_engine *e, int what, const void *src, size_t bytes);

/* The signal path without the network: pnb_process_* cut where the network sits, so the g/r between analysis and
 * synthesis come from the caller -- another engine's pnb_compute_rnn_*, a torch model, a records file's ideal gains,
 * the reference's feature_test.raw.  Both halves work on the active rows [0, n), stream-major:
 *   in / d_in     PCM rows as pnb_process_*_* takes them (int16: s/32768.f)
 *   feat / d_feat row i receives n_frames x 70 floats, feat_stride >= n_frames*70: hop t is bit for bit
 *                 PNB_TAP_FEATURES[t][i] of a pnb_process_* call on the same input
 *   gr / d_gr     row i holds n_frames x 68 floats (34 g then 34 r per hop), gr_stride >= n_frames*68
 *   out / d_out   PCM rows as pnb_process_*_* writes them (int16: C truncation of y*32768, wrapping)
 * These are the layouts of pnb_compute_rnn_* (PNB_RNN_FEATURES in, g/r out), so the three calls chain on device
 * pointers with no reshaping; f32 and int16 forms of the two halves mix freely.
 * pnb_analyze_* advances the active slots' signal input by n_frames hops (stage-in, analysis, history bookkeeping) and
 * leaves a pending synthesis on the engine.  The next pnb_synthesize_*, with the same n_frames, completes those hops
 * with the caller's g/r in place of the network's (post-filtered on a PNB_POSTFILTER engine), writes the PCM and commits
 * the hops.  A pnb_process_* call on the same input with the same g/r produces the same output and leaves the engine in
 * the same state.  g/r are used as given: for finite values the output is the reference's synthesis arithmetic on them
 * (pitch_filter and interp_band_gain are linear in r and g; nothing is clamped); for non-finite values the affected
 * rows' output is unspecified, the call still completes and the other rows are unaffected.
 * While a synthesis is pending, only pnb_synthesize_*, pnb_compute_rnn_* / pnb_score_records_* (they touch no signal
 * state), pnb_wait, pnb_check, pnb_flush, pnb_read_tap, the profile readers and pnb_reset (which cancels it) are
 * accepted.  Every other call and state operation -- another pnb_analyze_*, pnb_process_* / pnb_submit_*,
 * pnb_set_active_streams, pnb_reset_streams / pnb_export_states / pnb_import_states, pnb_get_state / pnb_set_state,
 * pnb_sessions_reserve -- returns PNB_ERR_ARG before anything is enqueued: between the halves a stream is mid-hop (its
 * overlap-add memory lags its history), a state no blob may capture.
 * Also refused with PNB_ERR_ARG before anything is enqueued: pnb_synthesize_* with nothing pending or another n_frames,
 * an engine in session mode, PNB_TRAIN_DATA and PNB_NETWORK_ONLY engines, NULL pointers, short strides, n_frames outside
 * [1, max_frames]; a poisoned engine returns PNB_ERR_CUDA.  Ordering, blocking and poisoning are those of
 * pnb_process_device_* / pnb_process_host_*.
 * Launches: pnb_analyze_* issues three (stage-in, analysis, feature store), plus the history move on the calls where
 * pnb_process_* would issue it; pnb_synthesize_* issues two (g/r stage-in, synthesis). */
int pnb_analyze_host_f32(pnb_engine *e, const float *in, size_t in_stride, int n_frames, float *feat, size_t feat_stride);
int pnb_analyze_host_i16(pnb_engine *e, const short *in, size_t in_stride, int n_frames, float *feat, size_t feat_stride);
int pnb_analyze_device_f32(pnb_engine *e, const float *d_in, size_t in_stride, int n_frames, float *d_feat,
                           size_t feat_stride, void *cuda_stream);
int pnb_analyze_device_i16(pnb_engine *e, const short *d_in, size_t in_stride, int n_frames, float *d_feat,
                           size_t feat_stride, void *cuda_stream);
int pnb_synthesize_host_f32(pnb_engine *e, const float *gr, size_t gr_stride, int n_frames, float *out, size_t out_stride);
int pnb_synthesize_host_i16(pnb_engine *e, const float *gr, size_t gr_stride, int n_frames, short *out, size_t out_stride);
int pnb_synthesize_device_f32(pnb_engine *e, const float *d_gr, size_t gr_stride, int n_frames, float *d_out,
                              size_t out_stride, void *cuda_stream);
int pnb_synthesize_device_i16(pnb_engine *e, const float *d_gr, size_t gr_stride, int n_frames, short *d_out,
                              size_t out_stride, void *cuda_stream);

/* Per-stream state for migration between engines / GPUs (the live part of the reference's DenoiseState + RNNState,
 * src/denoise.cpp:71-85, src/nnet_data.h:28-38): input history, overlap-add memory, pitch continuity, the spectra the
 * next five hops will analyse, conv histories and GRU states -- pnb_state_size() bytes, a flat host blob.
 * Both calls wait for the engine to be idle.  A state taken from stream a of one engine and set on stream b of another
 * (any batch size, either network mode, same model) continues the stream exactly where it left off: bit for bit between
 * engines of the same mode.  PNB_TRAIN_DATA and PNB_SIGNAL_ONLY engines carry the signal part only. */
size_t pnb_state_size(void);
int pnb_get_state(pnb_engine *e, int stream, void *dst, size_t dst_bytes);
int pnb_set_state(pnb_engine *e, int stream, const void *src, size_t src_bytes);

/* Batched stream recycling inside a running engine: a session that ends frees its slot for the next one, a session that
 * moves to another engine / GPU takes its state along -- without idling the device.  All three are asynchronous on
 * cuda_stream (a cudaStream_t, NULL = default stream) and never synchronise the host.
 *   streams      host array of n distinct slots in [0, n_streams); it may be reused as soon as the call returns
 *   d_blobs      device memory on the engine's device: blob i at d_blobs + i*blob_stride, blob_stride >= pnb_state_size()
 *                (pointer and stride multiples of 4 bytes); the bytes are those of pnb_get_state / pnb_set_state, so a
 *                blob may be copied to the host and set with pnb_set_state on any engine, and the reverse
 * Order: an operation runs after everything already enqueued on cuda_stream and after every call issued earlier on the
 * engine, on any stream; every call issued later runs after it.
 *
 * pnb_reset_streams: the listed streams get the state of a stream in a freshly created engine (history, overlap-add and
 *   pitch memory, the live spectrum slots, conv histories and GRU states -- what pnb_reset clears, restricted to them).
 *   The other streams and the engine's status are not touched.  n = 0 is a no-op.
 * pnb_export_states: writes the blob of every listed stream (PNB_TRAIN_DATA engines: the signal part, the rest zero).
 * pnb_import_states: the batched pnb_set_state (any batch size, max_frames or network mode of the exporting engine).
 *   A tensor-mode engine given an fp32-mode blob splits its conv histories and GRU states on the device exactly as
 *   pnb_set_state does.  A blob with a wrong magic / version, or (tensor mode) a GRU value outside [-1.0001, 1.0001],
 *   is not loaded: its stream is left reset and the next synchronising entry point (pnb_wait, pnb_check,
 *   pnb_process_host_*) returns PNB_ERR_ARG once, naming the lowest rejected slot in pnb_last_error(); unlike
 *   PNB_ERR_DOMAIN this does not stick.
 * Refused with PNB_ERR_ARG before anything is enqueued: NULL pointers (for n > 0), a slot out of range or listed twice,
 * a short or misaligned blob_stride, and an engine poisoned by a failed call. */
int pnb_reset_streams(pnb_engine *e, const int *streams, int n, void *cuda_stream);
int pnb_export_states(pnb_engine *e, const int *streams, int n, void *d_blobs, size_t blob_stride, void *cuda_stream);
int pnb_import_states(pnb_engine *e, const int *streams, int n, const void *d_blobs, size_t blob_stride, void *cuda_stream);

/* Active range: calls issued after pnb_set_active_streams(e, n, .) advance slots [0, n) only, 1 <= n <= n_streams, and
 * cost roughly n / n_streams of a full call (rounded up to 128-stream tiles in the network).  A fresh engine, and an
 * engine after pnb_reset, has n = n_streams.  n is taken when a call is issued: calls already submitted keep theirs.
 *   Growing n: the entering slots are reset as by pnb_reset_streams, asynchronously on cuda_stream and ordered like
 *   any state operation.  pnb_import_states after the grow gives an entering slot a state.
 *   Shrinking n enqueues nothing: the leaving slots lose their state (pnb_export_states them first to keep it).
 * In and out of every pnb_process_* / pnb_submit_* call hold n rows, gr / d_gr is [n_frames][n][68]; pnb_read_tap keeps
 * its n_streams layout (rows >= n unspecified).  Live sessions stay packed in [0, n): when the session at slot k ends,
 * export slot n-1, import it at k, then shrink to n-1.
 * Refused with PNB_ERR_ARG before anything is enqueued: n outside [1, n_streams], a PNB_TRAIN_DATA engine, a poisoned
 * engine.  pnb_reset_streams / pnb_export_states / pnb_import_states / pnb_get_state / pnb_set_state refuse slots >= n. */
int pnb_set_active_streams(pnb_engine *e, int n, void *cuda_stream);
int pnb_active_streams(const pnb_engine *e);

/* Session pool: calls advance any listed subset of sessions, and sessions that sit a call out keep their state.
 * A session is a logical stream id in [0, capacity); each session is either resident in a slot of the engine or parked
 * as a blob (the bytes of pnb_export_states) in engine-owned device memory.  Only sessions that change membership
 * between two calls move: a session listed in consecutive calls stays in its slot, one that skips a call is parked once
 * and unparked once; listing the same set in another order moves nothing.
 *
 * pnb_sessions_reserve: the first call puts the engine in session mode and resets it (every session starts fresh); a
 *   later call with a larger n_sessions grows the parking area (pnb_state_size() bytes, rounded up to 16, per session)
 *   and keeps every session's state; a smaller or equal one is a no-op.  Waits for the engine to be idle.  Refused on
 *   PNB_TRAIN_DATA engines and on an engine poisoned by a failed call.
 * pnb_process_sessions_*: advances exactly the n listed sessions (distinct ids, 1 <= n <= n_streams) by n_frames hops;
 *   row i of in / out and gr[t][i] belong to ids[i], in list order; every session not listed keeps its state.  ids is
 *   host memory, reusable when the call returns.  The device forms are asynchronous and ordered like pnb_process_device_*
 *   (d_gr NULL ok); the host forms block like pnb_process_host_* (gr NULL ok).
 * pnb_reset_sessions: the listed sessions start over as fresh streams (the session-level pnb_reset_streams).
 * pnb_export_sessions / pnb_import_sessions: the blobs of pnb_export_states / pnb_import_states (same d_blobs and
 *   blob_stride rules, n <= capacity), so a session moves between pooled engines, plain engines (pnb_set_state) and
 *   the host.  An import is checked like pnb_import_states: a rejected blob leaves its session fresh, and the next
 *   synchronising entry point returns PNB_ERR_ARG once, naming the lowest rejected session id.
 *   The three are asynchronous on cuda_stream and ordered with the calls like the slot-level state operations.
 * pnb_session_stats: out[0] parks, out[1] unparks (fresh starts included), out[2] relocations (a listed session moved
 *   from a slot >= n to a free slot < n), counted since pnb_sessions_reserve.  A test and measurement hook.
 * In session mode pnb_process_* / pnb_submit_*, pnb_set_active_streams, pnb_reset_streams, pnb_export_states,
 * pnb_import_states, pnb_get_state and pnb_set_state return PNB_ERR_ARG before anything is enqueued; pnb_reset makes
 * every session fresh and keeps session mode.  The session calls refuse, before any state changes: a call before
 * pnb_sessions_reserve, NULL pointers, ids out of range or listed twice, n out of range, short strides, and n_frames
 * outside [1, max_frames].  A call that fails after it started to enqueue work poisons the engine, as the other calls. */
int pnb_sessions_reserve(pnb_engine *e, int n_sessions);
int pnb_process_sessions_device_f32(pnb_engine *e, const int *ids, int n, const float *d_in, size_t in_stride,
                                    float *d_out, size_t out_stride, int n_frames, float *d_gr, void *cuda_stream);
int pnb_process_sessions_device_i16(pnb_engine *e, const int *ids, int n, const short *d_in, size_t in_stride,
                                    short *d_out, size_t out_stride, int n_frames, float *d_gr, void *cuda_stream);
int pnb_process_sessions_host_f32(pnb_engine *e, const int *ids, int n, const float *in, size_t in_stride, float *out,
                                  size_t out_stride, int n_frames, float *gr);
int pnb_process_sessions_host_i16(pnb_engine *e, const int *ids, int n, const short *in, size_t in_stride, short *out,
                                  size_t out_stride, int n_frames, float *gr);
/* Ragged session calls: session ids[i] advances by its own hops[i] hops, 1 <= hops[i] <= max_frames (hops is host
 * memory, reusable when the call returns); the call is F = max(hops) hops long.  Row strides must be at least F*480;
 * input row i is read for its first hops[i]*480 samples only (the host forms copy F*480 samples of every row, the
 * rest is ignored); output row i holds hops[i] hops of output followed by zeros up to F*480; gr / d_gr is [F][n][68]
 * with gr[t][i] = 0 for t >= hops[i].  Each session ends in the state of its own hops[i] hops and continues bit for bit
 * like a plain engine fed the same hops back to back; sessions not listed keep their state.  Residency, ordering,
 * blocking, poisoning and error codes are those of pnb_process_sessions_*, which refuse the same arguments; a ragged
 * call also refuses hops == NULL and any hops[i] outside [1, max_frames], with PNB_ERR_ARG before anything changes.
 * When every hops[i] == F the call is pnb_process_sessions_*(..., F, ...): the same launches, the same results.  A
 * call with a shorter session adds one launch (the fix-up that moves the early finishers' state to the call's end).
 * PNB_KEEP_TAPS taps of the hops a session did not run are unspecified. */
int pnb_process_sessions_ragged_device_f32(pnb_engine *e, const int *ids, const int *hops, int n, const float *d_in,
                                           size_t in_stride, float *d_out, size_t out_stride, float *d_gr, void *cuda_stream);
int pnb_process_sessions_ragged_device_i16(pnb_engine *e, const int *ids, const int *hops, int n, const short *d_in,
                                           size_t in_stride, short *d_out, size_t out_stride, float *d_gr, void *cuda_stream);
int pnb_process_sessions_ragged_host_f32(pnb_engine *e, const int *ids, const int *hops, int n, const float *in,
                                         size_t in_stride, float *out, size_t out_stride, float *gr);
int pnb_process_sessions_ragged_host_i16(pnb_engine *e, const int *ids, const int *hops, int n, const short *in,
                                         size_t in_stride, short *out, size_t out_stride, float *gr);
int pnb_reset_sessions(pnb_engine *e, const int *ids, int n, void *cuda_stream);
int pnb_export_sessions(pnb_engine *e, const int *ids, int n, void *d_blobs, size_t blob_stride, void *cuda_stream);
int pnb_import_sessions(pnb_engine *e, const int *ids, int n, const void *d_blobs, size_t blob_stride, void *cuda_stream);
int pnb_session_stats(const pnb_engine *e, long long *out);

/* The pitch analysis alone (BASELINE.json config 5; needs no engine): for each of n_units pitch buffers of 1728
 * float samples (unit u at d_pitch_buf + u*stride; the reference's st->pitch_buf, src/denoise.cpp:80,405-411) runs
 * pitch_downsample, pitch_search and remove_doubling (src/pitch.cpp:148-216, 283-386, 423-527) exactly as the hot path
 * does, and writes the final period T in [60, 767], the raw pitch correlation (feature 69) and the pitch gain.
 * d_prev_period / d_prev_gain (NULL = 0) are the previous frame's values remove_doubling's continuity test uses;
 * d_lag (NULL ok) receives pitch_search's lag before the doubling check.  Asynchronous on cuda_stream, current device. */
int pnb_pitch_only_device(const float *d_pitch_buf, size_t stride, long long n_units, const int *d_prev_period,
                          const float *d_prev_gain, int *d_period, float *d_corr, float *d_gain, int *d_lag,
                          void *cuda_stream);

/* Host-buffer form (blocking): copies the buffers to the current device, runs the kernel, copies the results back. */
int pnb_pitch_only_host(const float *pitch_buf, size_t stride, long long n_units, const int *prev_period,
                        const float *prev_gain, int *period, float *corr, float *gain, int *lag);

/* Per-frame intermediates of the LAST call (requires PNB_KEEP_TAPS); copies to host memory.
 * Layouts are [n_frames][n_streams][...]:                                                   */
enum {
  PNB_TAP_FEATURES = 0, /* float[70]  network input (src/denoise.cpp:487-496)                */
  PNB_TAP_PITCH = 1,    /* int[4]     {pitch_search lag, final period T, silence, 0}          */
  PNB_TAP_PITCHF = 2,   /* float[2]   {pitch_corr, pitch_gain}                                */
  PNB_TAP_X = 3,        /* float[800] analysis spectrum bins 0..399 (re,im)                   */
  PNB_TAP_P = 4,        /* float[800] comb-filtered spectrum bins 0..399 (re,im)              */
  PNB_TAP_EX = 5,       /* float[34]  band energy of X                                        */
  PNB_TAP_GR = 6,       /* float[68]  g, r                                                    */
  /* network state after the last hop of the call, layout [n_streams][width] (no PNB_KEEP_TAPS needed): */
  PNB_TAP_NN_C2 = 7,    /* float[512] conv2 output                                            */
  PNB_TAP_NN_H0 = 8,    /* +0..4: float[512|128] states of gru1, gru2, gru3, gru_gb, gru_rb   */
  PNB_TAP_G_USED = 13   /* float[34]  band gains as applied: g, post-filtered under PNB_POSTFILTER (PNB_KEEP_TAPS) */
};
int pnb_read_tap(pnb_engine *e, int what, void *dst, size_t dst_bytes);

/* Per-kernel-class device timing.  While enabled, every launch of a pnb_process_* call is bracketed by
 * CUDA events on the launching stream; pnb_profile_read waits for them and returns the accumulated
 * milliseconds and launch counts per class since the last read (arrays of PNB_NUM_KERNEL_CLASSES). */
enum {
  PNB_K_STAGE_IN = 0, PNB_K_ANALYSIS = 1, PNB_K_FC = 2, PNB_K_GEMM_F32 = 3, PNB_K_F32_CARRY = 4,  /* fp32 path: the per-chunk carry (was the GRU gate kernel before the gates were fused) */
 
  PNB_K_SYNTHESIS = 5, PNB_K_SLIDE = 6, PNB_K_TC_GEMM = 7, PNB_K_TC_AUX = 8, PNB_K_LABELS = 9,
  PNB_NUM_KERNEL_CLASSES = 10
};
int pnb_profile_enable(pnb_engine *e, int on);
int pnb_profile_read(pnb_engine *e, double *ms, long long *counts);
/* The same records as a timeline: launch i of the profiled calls as (class, start ms, end ms) relative to the first
 * launch, in launch order.  Returns the count written (<= cap). */
int pnb_profile_timeline(pnb_engine *e, int *cls, double *t0_ms, double *t1_ms, int cap);
const char *pnb_kernel_class_name(int cls);

/* Number of kernels this library has launched on behalf of e since creation. */
long long pnb_launch_count(const pnb_engine *e);
/* Kernel launches one pnb_process_* call with n_frames hops issues (one more on the calls that also move the
 * streams' history back to the start of their rows, at most every call, typically every eighth; one more on a ragged
 * session call in which some session runs fewer than n_frames = max(hops) hops).  On a PNB_TRAIN_AUDIO engine it is the
 * value of a PNB_TRAIN_DATA engine of the same shape plus one: the resynthesis launch.  On a PNB_NETWORK_ONLY engine it
 * is the launch count of one pnb_compute_rnn_* call of n_frames hops (PNB_TRAIN_NETWORK: of one pnb_train_grad_* call,
 * the same for every n_frames); on a PNB_SIGNAL_ONLY engine that of one
 * pnb_analyze_* and one pnb_synthesize_* call of n_frames hops (five, without the history move). */
int pnb_launches_per_call(const pnb_engine *e, int n_frames);
/* Bytes of the engine's device buffers whose size pnb_create fixes (weights, network buffers, stream state, per-call
 * scratch); not the staging that host-buffer calls grow on first use, nor a session pool's parking area. */
size_t pnb_engine_bytes(const pnb_engine *e);
int pnb_n_streams(const pnb_engine *e);
int pnb_max_frames(const pnb_engine *e);
const char *pnb_last_error(void);
const char *pnb_version(void);

#ifdef __cplusplus
}
#endif
#endif /* PERCEPNET_B200_H */
