/*
 * pn_oracle.h -- TEST INFRASTRUCTURE ONLY.
 *
 * CPU restatement (plain C, strict IEEE single precision, no FMA contraction) of the
 * reference's per-frame enhancement path rnnoise_process_frame
 * (/root/reference/src/denoise.cpp:508-547 and everything it calls).  It is the checker the
 * CUDA path is compared against; it is never imported, linked or executed by the product
 * (percepnet_b200/), only by tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
 * --impl reference legs.
 *
 * Pinning: bit-exact against the compiled, unmodified reference (oracle/_ref, built by
 * oracle/Makefile from /root/reference/src) on every stage tap and end to end
 * (tests/test_oracle_vs_reference.py, run in the build container), and against the
 * committed golden vectors under tests/golden/ that the reference itself produced
 * (tests/golden/make_golden.py), plus the reference's own toy-layer known-answer vectors
 * (/root/reference/tests/nnet_data_test.h).
 */
#ifndef PN_ORACLE_H
#define PN_ORACLE_H

#include <stddef.h>
#include "../include/pnb_nnet_layout.h"

#ifdef __cplusplus
extern "C" {
#endif

#define PNO_FRAME 480
#define PNO_WINDOW 960
#define PNO_FREQ 481
#define PNO_BANDS 34
#define PNO_FEATURES 70
#define PNO_HIST 5760 /* = COMB_BUF_SIZE, denoise.cpp:32 */
#define PNO_NN_STATE (512 + 1024 + 4 * 512 + 128)

typedef struct pn_oracle pn_oracle;

/* Everything a parity test may want to look at for one frame. */
typedef struct pn_oracle_taps {
  float X[2 * PNO_FREQ];    /* analysis spectrum of the delayed frame (re,im interleaved) */
  float P[2 * PNO_FREQ];    /* comb-filtered ("pitch") spectrum                           */
  float Y[2 * PNO_FREQ];    /* look-ahead spectrum                                        */
  float Xout[2 * PNO_FREQ]; /* spectrum handed to the inverse transform                   */
  float Ex[PNO_BANDS], Ep[PNO_BANDS], Exp[PNO_BANDS], Ex_look[PNO_BANDS];
  float features[PNO_FEATURES];
  float g[PNO_BANDS], r[PNO_BANDS]; /* raw NN outputs (what the reference fwrite()s) */
  float g_used[PNO_BANDS];          /* gains applied (differs from g only with the post-filter on) */
  float lp[864];                    /* pitch_downsample output */
  float xcorr_coarse[147];
  int best_coarse[2];
  int pitch_search; /* lag returned by pitch_search (src/pitch.cpp:384) */
  float pitch_corr; /* src/pitch.cpp:385 */
  int pitch_index;  /* period after remove_doubling == st->last_period */
  float pitch_gain; /* == st->last_gain */
  int silence;
} pn_oracle_taps;

pn_oracle *pn_oracle_create(const pnb_model *model); /* weight arrays stay caller-owned */
void pn_oracle_destroy(pn_oracle *o);
void pn_oracle_reset(pn_oracle *o);

/* flags */
#define PNO_POSTFILTER 1 /* apply denoise.cpp:216-250 to g before it is used (off in the reference's inference path) */

/* one frame, float C-API semantics of src/rnnoise.h:60; in may alias out; taps may be NULL */
void pn_oracle_process_frame(pn_oracle *o, float *out, const float *in, pn_oracle_taps *taps, int flags);
/* n_frames on one stream; gr (NULL ok) gets n_frames*68 floats */
void pn_oracle_process_stream(pn_oracle *o, float *out, const float *in, int n_frames, float *gr, int flags);
/* src/main.cpp:30-39 I/O semantics; out16 gets (n_frames-1)*480 samples */
void pn_oracle_run_pcm16(const pnb_model *m, const short *in16, int n_frames, short *out16, float *gr);
/* independent streams, OpenMP over streams; in/out [n_streams][n_frames*480] */
void pn_oracle_process_streams(const pnb_model *m, int n_streams, int n_frames, const float *in, float *out,
                               int n_threads, int flags);

/* ---- training-data path (row f1): train() of denoise.cpp:600-787 on in-memory int16 "files" ---- */
#define PNO_RECORD 138 /* Ey_lookahead[34] Ephaty[34] T pitchcorr g[34] r[34], denoise.cpp:761-773 */
void pn_oracle_train_records(const short *speech, const short *noisy, int count, float *records);
/* labels of denoise.cpp:549-589 from clean (Ex, Exp) and noisy (Ey, Ephaty) band statistics */
void pn_oracle_ideal_labels(const float *Ex, const float *Ey, const float *Exp, const float *Ephaty, float *g, float *r);

/* ---- stage-level entry points (each pinned against the reference's function) ---- */
void pn_oracle_erb_borders(int *out34);                                   /* erbband.h:34-99         */
void pn_oracle_tables(float *half_window480, float *comb_window7);        /* denoise.cpp:186-214     */
float pn_oracle_tansig(float x);                                          /* vec.h:53-71             */
float pn_oracle_sigmoid(float x);                                         /* vec.h:73-76             */
void pn_oracle_tansig_n(const float *x, float *y, long n);                /* the same, n values      */
void pn_oracle_sigmoid_n(const float *x, float *y, long n);
void pn_oracle_fft960(const float *in_ri, float *out_ri);                 /* kiss_fft.cpp:566-586    */
void pn_oracle_band_energy(float *bandE, const float *X_ri);              /* denoise.cpp:89-123      */
void pn_oracle_band_corr(float *bandE, const float *X_ri, const float *P_ri); /* denoise.cpp:125-160 */
void pn_oracle_interp_band_gain(float *g481, const float *bandE);         /* denoise.cpp:162-182 (+ App. C.1) */
void pn_oracle_pitch_filter(float *X_ri, const float *P_ri, const float *r); /* denoise.cpp:436-485  */
void pn_oracle_post_filter(float *g, const float *Ey);                    /* denoise.cpp:216-250     */
void pn_oracle_pitch_downsample(const float *pitch_buf1728, float *lp864);/* pitch.cpp:148-216       */
void pn_oracle_autocorr_lpc(const float *x, int n, float *ac5, float *lpc4); /* celt_lpc.cpp:198,37  */
void pn_oracle_pitch_xcorr(const float *x, const float *y, float *xcorr, int len, int max_pitch); /* pitch.cpp:218 */
void pn_oracle_pitch_search(const float *lp864, int *pitch, float *corr, float *xcorr_coarse147, int *best2); /* pitch.cpp:283 */
float pn_oracle_remove_doubling(const float *lp864, int *T0, int prev_period, float prev_gain); /* pitch.cpp:424 */
void pn_oracle_dense_layer(const pnb_dense_layer *l, float *out, const float *in);               /* nnet.cpp:105 */
void pn_oracle_conv1d_layer(const pnb_conv1d_layer *l, float *out, float *mem, const float *in); /* nnet.cpp:182 */
void pn_oracle_gru_layer(const pnb_gru_layer *l, float *state, const float *in);                 /* nnet.cpp:120 */
/* state block: [conv1 mem 512][conv2 mem 1024][gru1 512][gru2 512][gru3 512][gru_gb 512][gru_rb 128] */
void pn_oracle_compute_rnn(const pnb_model *m, float *state, float *gains, float *strengths,
                           const float *features);                                               /* rnn.cpp:42 */

/* pitch_downsample + pitch_search + remove_doubling on n independent pitch buffers (unit u at bufs + u*stride),
 * OpenMP over units; prev_* NULL = 0 */
void pn_oracle_pitch_batch(const float *bufs, size_t stride, int n, const int *prev_period, const float *prev_gain,
                           int *T_out, float *corr_out, float *gain_out, int n_threads);
/* The same network evaluated in double precision (same wiring, table and correction formula): the arbiter between
 * two single-precision evaluations.  state: PNO_NN_STATE doubles, laid out like the float state block.  Returns the
 * largest |x| handed to the tanh approximation in this frame (the reference's is defined for |x| < 8.6e7 only). */
double pn_oracle_compute_rnn_f64(const pnb_model *m, double *state, double *gains, double *strengths,
                                 const float *features);

#ifdef __cplusplus
}
#endif
#endif
