/*
 * pn_oracle.c -- TEST INFRASTRUCTURE ONLY (see pn_oracle.h for the pinning statement).
 *
 * A CPU restatement of the reference's rnnoise_process_frame path.  It is organised
 * differently from the reference (one history line per stream instead of three
 * overlapping buffers, table-driven mixed-radix FFT, explicit stage functions) but every
 * floating-point expression keeps the reference's operand order and precision, so that the
 * results are bit-identical to the compiled reference (which contains no fused
 * multiply-adds and no re-associated sums, SURVEY.md 0.9).  Build with
 * -ffp-contract=off and without -ffast-math (oracle/Makefile).
 *
 * Citations are to /root/reference/src unless a path is given.
 */
#include "pn_oracle.h"

#include <math.h>
#include <stdlib.h>
#include <string.h>

typedef struct { float r, i; } cpx;

#define NB PNO_BANDS
#define FRAME PNO_FRAME
#define WIN PNO_WINDOW
#define NFREQ PNO_FREQ

/* ------------------------------------------------------------------------------------ */
/*  Constant tables (denoise.cpp:186-214, kiss_fft.cpp:406-421,434-493, erbband.h)       */
/* ------------------------------------------------------------------------------------ */
static struct {
  int ready;
  float half_window[FRAME];
  float comb_w[7];
  cpx tw[WIN];
  short perm[WIN];
  float scale;
  int border[NB];
  float tansig[201];
} K;

/* erbband.h:64-69: both helpers evaluate in double and return float */
static float hz_to_erb(float hz) { return (float)(9.265 * log(1 + hz / (24.7 * 9.265))); }
static float erb_to_hz(float e) { return (float)(24.7 * 9.265 * (exp(e / 9.265) - 1)); }

static void build_tables(void) {
  int i;
  if (K.ready) return;
  /* Vorbis power-complementary half window, denoise.cpp:191-192 (double -> float) */
  for (i = 0; i < FRAME; i++) {
    double a = .5 * M_PI * (i + .5) / FRAME;
    K.half_window[i] = (float)sin(.5 * M_PI * sin(a) * sin(a));
  }
  /* 7-tap normalised Hann used by the comb filter, denoise.cpp:200-206; the running sum is float */
  {
    float acc = 0;
    for (i = 1; i < 8; i++) {
      K.comb_w[i - 1] = (float)(0.5 - 0.5 * cos(2.0 * M_PI * i / 8));
      acc += K.comb_w[i - 1];
    }
    for (i = 0; i < 7; i++) K.comb_w[i] /= acc;
  }
  /* FFT-960 twiddles, kiss_fft.cpp:415-419 */
  for (i = 0; i < WIN; i++) {
    const double pi = 3.14159265358979323846264338327;
    double ph = (-2 * pi / WIN) * i;
    K.tw[i].r = (float)cos(ph);
    K.tw[i].i = (float)sin(ph);
  }
  K.scale = 1.f / WIN; /* kiss_fft.cpp:459 */
  /* digit-reversal of the 5.3.4.4.4 factorisation (kiss_fft.cpp:314-345 with the factor
   * order produced by kf_factor, :352-404): input n = n0 + 5(n1 + 3(n2 + 4(n3 + 4 n4)))
   * lands at 192 n0 + 64 n1 + 16 n2 + 4 n3 + n4 */
  for (i = 0; i < WIN; i++) {
    int n = i, n0, n1, n2, n3, n4;
    n0 = n % 5; n /= 5;
    n1 = n % 3; n /= 3;
    n2 = n % 4; n /= 4;
    n3 = n % 4; n /= 4;
    n4 = n;
    K.perm[i] = (short)(192 * n0 + 64 * n1 + 16 * n2 + 4 * n3 + n4);
  }
  /* ERB band edges in FFT bins, erbband.h:34-99 with (960, 32, 0, 20000) from denoise.cpp:87 */
  {
    float lo = hz_to_erb(0.f), hi = hz_to_erb(20000.f);
    float cut[NB];
    float step = (hi - lo) / (34.f - 1); /* linspace, erbband.h:6-30 */
    for (i = 0; i < NB - 1; i++) cut[i] = erb_to_hz(lo + step * i);
    cut[NB - 1] = erb_to_hz(hi);
    for (i = 0; i < NB; i++) K.border[i] = (int)((cut[i] + 25) / 50.f);
    for (i = 0; i < NB - 2; i++)
      if (K.border[i + 1] - K.border[i] < 2) K.border[i + 1] += 2 - (K.border[i + 1] - K.border[i]);
  }
  /* tanh lookup of tansig_table.h: tanh(0.04 i) printed with 6 decimals; three entries of
   * the shipped table deviate from correct rounding and are patched to the shipped values
   * (checked entry by entry against the header in tests/test_oracle_vs_reference.py) */
  for (i = 0; i <= 200; i++) K.tansig[i] = (float)(floor(tanh(0.04 * i) * 1e6 + 0.5) / 1e6);
  K.tansig[70] = 0.992631f;
  K.tansig[170] = 0.999997f;
  K.tansig[190] = 1.000000f;
  K.ready = 1;
}

void pn_oracle_erb_borders(int *out34) { build_tables(); memcpy(out34, K.border, sizeof K.border); }
void pn_oracle_tables(float *hw, float *cw) {
  build_tables();
  if (hw) memcpy(hw, K.half_window, sizeof K.half_window);
  if (cw) memcpy(cw, K.comb_w, sizeof K.comb_w);
}

/* ------------------------------------------------------------------------------------ */
/*  FFT-960 (kiss_fft.cpp:518-586): scaled digit-reversed load, then stages               */
/*  radix4(m=1) radix4(m=4) radix4(m=16) radix3(m=64) radix5(m=192)                       */
/* ------------------------------------------------------------------------------------ */
static inline cpx cmul(cpx a, cpx b) { /* C_MUL, _kiss_fft_guts.h */
  cpx m;
  m.r = a.r * b.r - a.i * b.i;
  m.i = a.r * b.i + a.i * b.r;
  return m;
}
static inline cpx cadd(cpx a, cpx b) { cpx m; m.r = a.r + b.r; m.i = a.i + b.i; return m; }
static inline cpx csub(cpx a, cpx b) { cpx m; m.r = a.r - b.r; m.i = a.i - b.i; return m; }

static void stage_r4_first(cpx *f) { /* kiss_fft.cpp:112-131, 240 butterflies on adjacent quads */
  int b;
  for (b = 0; b < 240; b++, f += 4) {
    cpx d02 = csub(f[0], f[2]);
    cpx s13, d13;
    f[0] = cadd(f[0], f[2]);
    s13 = cadd(f[1], f[3]);
    f[2] = csub(f[0], s13);
    f[0] = cadd(f[0], s13);
    d13 = csub(f[1], f[3]);
    f[1].r = d02.r + d13.i;
    f[1].i = d02.i - d13.r;
    f[3].r = d02.r - d13.i;
    f[3].i = d02.i + d13.r;
  }
}
static void stage_r4(cpx *base, int m, int groups, int tws) { /* kiss_fft.cpp:132-166 */
  int g, j;
  for (g = 0; g < groups; g++) {
    cpx *f = base + g * 4 * m;
    for (j = 0; j < m; j++, f++) {
      cpx a = cmul(f[m], K.tw[j * tws]);
      cpx b = cmul(f[2 * m], K.tw[2 * j * tws]);
      cpx c = cmul(f[3 * m], K.tw[3 * j * tws]);
      cpx d0b = csub(f[0], b);
      cpx sac, dac;
      f[0] = cadd(f[0], b);
      sac = cadd(a, c);
      dac = csub(a, c);
      f[2 * m] = csub(f[0], sac);
      f[0] = cadd(f[0], sac);
      f[m].r = d0b.r + dac.i;
      f[m].i = d0b.i - dac.r;
      f[3 * m].r = d0b.r - dac.i;
      f[3 * m].i = d0b.i + dac.r;
    }
  }
}
static void stage_r3(cpx *base, int m, int groups, int tws) { /* kiss_fft.cpp:173-228 */
  int g, j;
  float w3i = K.tw[tws * m].i; /* epi3, :194 */
  for (g = 0; g < groups; g++) {
    cpx *f = base + g * 3 * m;
    for (j = 0; j < m; j++, f++) {
      cpx a = cmul(f[m], K.tw[j * tws]);
      cpx b = cmul(f[2 * m], K.tw[2 * j * tws]);
      cpx s = cadd(a, b);
      cpx d = csub(a, b);
      f[m].r = f[0].r - s.r * .5f;
      f[m].i = f[0].i - s.i * .5f;
      d.r *= w3i;
      d.i *= w3i;
      f[0] = cadd(f[0], s);
      f[2 * m].r = f[m].r + d.i;
      f[2 * m].i = f[m].i - d.r;
      f[m].r = f[m].r - d.i;
      f[m].i = f[m].i + d.r;
    }
  }
}
static void stage_r5(cpx *base, int m, int groups, int tws) { /* kiss_fft.cpp:232-305 */
  int g, u;
  cpx ya = K.tw[tws * m], yb = K.tw[tws * 2 * m];
  for (g = 0; g < groups; g++) {
    cpx *f0 = base + g * 5 * m, *f1 = f0 + m, *f2 = f0 + 2 * m, *f3 = f0 + 3 * m, *f4 = f0 + 4 * m;
    for (u = 0; u < m; u++, f0++, f1++, f2++, f3++, f4++) {
      cpx z0 = *f0;
      cpx z1 = cmul(*f1, K.tw[u * tws]);
      cpx z2 = cmul(*f2, K.tw[2 * u * tws]);
      cpx z3 = cmul(*f3, K.tw[3 * u * tws]);
      cpx z4 = cmul(*f4, K.tw[4 * u * tws]);
      cpx s14 = cadd(z1, z4), d14 = csub(z1, z4);
      cpx s23 = cadd(z2, z3), d23 = csub(z2, z3);
      cpx p, q;
      f0->r = f0->r + (s14.r + s23.r);
      f0->i = f0->i + (s14.i + s23.i);
      p.r = z0.r + (s14.r * ya.r + s23.r * yb.r);
      p.i = z0.i + (s14.i * ya.r + s23.i * yb.r);
      q.r = d14.i * ya.i + d23.i * yb.i;
      q.i = -(d14.r * ya.i + d23.r * yb.i);
      *f1 = csub(p, q);
      *f4 = cadd(p, q);
      p.r = z0.r + (s14.r * yb.r + s23.r * ya.r);
      p.i = z0.i + (s14.i * yb.r + s23.i * ya.r);
      q.r = d23.i * ya.i - d14.i * yb.i;
      q.i = d14.r * yb.i - d23.r * ya.i;
      *f2 = cadd(p, q);
      *f3 = csub(p, q);
    }
  }
}
static void fft960(const cpx *in, cpx *out) {
  int i;
  build_tables();
  for (i = 0; i < WIN; i++) { /* kiss_fft.cpp:579-584 */
    out[K.perm[i]].r = K.scale * in[i].r;
    out[K.perm[i]].i = K.scale * in[i].i;
  }
  stage_r4_first(out);
  stage_r4(out, 4, 60, 60);
  stage_r4(out, 16, 15, 15);
  stage_r3(out, 64, 5, 5);
  stage_r5(out, 192, 1, 1);
}
void pn_oracle_fft960(const float *in_ri, float *out_ri) { fft960((const cpx *)in_ri, (cpx *)out_ri); }

/* window (denoise.cpp:282-289) + real->complex forward transform keeping bins 0..480 (:291-304) */
static void window_inplace(float *x) {
  int i;
  for (i = 0; i < FRAME; i++) {
    x[i] *= K.half_window[i];
    x[WIN - 1 - i] *= K.half_window[i];
  }
}
static void spectrum_of(const float *x960, cpx *spec481) {
  cpx a[WIN], b[WIN];
  int i;
  for (i = 0; i < WIN; i++) { a[i].r = x960[i]; a[i].i = 0; }
  fft960(a, b);
  memcpy(spec481, b, NFREQ * sizeof(cpx));
}
/* inverse via forward FFT of the Hermitian extension, read back reversed (denoise.cpp:306-324) */
static void signal_of(const cpx *spec481, float *x960) {
  cpx a[WIN], b[WIN];
  int i;
  memcpy(a, spec481, NFREQ * sizeof(cpx));
  for (i = NFREQ; i < WIN; i++) { a[i].r = a[WIN - i].r; a[i].i = -a[WIN - i].i; }
  fft960(a, b);
  x960[0] = WIN * b[0].r;
  for (i = 1; i < WIN; i++) x960[i] = WIN * b[WIN - i].r;
}

/* ------------------------------------------------------------------------------------ */
/*  ERB band pooling (denoise.cpp:89-182)                                                 */
/* ------------------------------------------------------------------------------------ */
static void band_pool(float *bandE, const cpx *A, const cpx *B) { /* A==B -> energy, else correlation */
  float acc[NB] = {0};
  int b, j;
  for (b = 0; b < NB - 1; b++) {
    int lo = K.border[b], width = K.border[b + 1] - K.border[b];
    for (j = 0; j < width; j++) {
      float frac = (float)j / width;
      float v = A[lo + j].r * B[lo + j].r;
      v += A[lo + j].i * B[lo + j].i;
      acc[b] += (1 - frac) * v;
      acc[b + 1] += frac * v;
    }
  }
  acc[0] *= 2;
  acc[NB - 1] *= 2;
  memcpy(bandE, acc, sizeof acc);
}
void pn_oracle_band_energy(float *bandE, const float *X) { build_tables(); band_pool(bandE, (const cpx *)X, (const cpx *)X); }
void pn_oracle_band_corr(float *bandE, const float *X, const float *P) { build_tables(); band_pool(bandE, (const cpx *)X, (const cpx *)P); }

/* per-bin interpolation of band values.  The reference only defines bins below the last
 * border (400); through its zero-initialised callers (denoise.cpp:440,517 and the 481-BYTE
 * memset at :164) every bin from 400 to 480 ends up 0 -- SURVEY.md App. C.1. */
static void band_to_bins(float *g, const float *bandE) {
  int b, j;
  memset(g, 0, NFREQ * sizeof(float));
  for (b = 0; b < NB - 1; b++) {
    int lo = K.border[b], width = K.border[b + 1] - K.border[b];
    for (j = 0; j < width; j++) {
      float frac = (float)j / width;
      g[lo + j] = (1 - frac) * bandE[b] + frac * bandE[b + 1];
    }
  }
}
void pn_oracle_interp_band_gain(float *g481, const float *bandE) { build_tables(); band_to_bins(g481, bandE); }

/* X <- interp(1-r) X + interp(r) P   (denoise.cpp:436-485) */
static void comb_mix(cpx *X, const cpx *P, const float *r) {
  float rf[NFREQ], one_minus[NB];
  int i;
  for (i = 0; i < NB; i++) one_minus[i] = 1 - r[i];
  band_to_bins(rf, one_minus);
  for (i = 0; i < NFREQ; i++) { X[i].r = rf[i] * X[i].r; X[i].i = rf[i] * X[i].i; }
  band_to_bins(rf, r);
  for (i = 0; i < NFREQ; i++) { X[i].r += rf[i] * P[i].r; X[i].i += rf[i] * P[i].i; }
}
void pn_oracle_pitch_filter(float *X, const float *P, const float *r) { build_tables(); comb_mix((cpx *)X, (const cpx *)P, r); }

/* envelope post-filter (denoise.cpp:216-250); beta = 0.02 (:43) */
void pn_oracle_post_filter(float *g, const float *Ey) {
  float gw[NB], e0 = 0, e1 = 0, q, G;
  const float beta = 0.02f;
  int i;
  for (i = 0; i < NB; i++) gw[i] = g[i] * sinf((float)(M_PI / 2 * g[i])); /* sinf(double->float arg), :227 */
  for (i = 0; i < NB; i++) e0 += g[i] * Ey[i];
  for (i = 0; i < NB; i++) e1 += gw[i] * Ey[i];
  q = e0 / (e1 + 1e-6f);
  G = sqrtf(((1 + beta) * q) / (1 + beta * (q * q)));
  for (i = 0; i < NB; i++) g[i] = G * gw[i];
}

/* ------------------------------------------------------------------------------------ */
/*  Pitch analysis (pitch.cpp, celt_lpc.cpp).  All sums are strict left-to-right           */
/*  multiply-then-add chains starting from 0, exactly as the reference's macros expand.   */
/* ------------------------------------------------------------------------------------ */
static float dot_seq(const float *a, const float *b, int n) { /* pitch.h:136-144 */
  float s = 0;
  int i;
  for (i = 0; i < n; i++) s = s + a[i] * b[i];
  return s;
}
/* every lag is an independent sequential dot product (pitch.cpp:218-281, pitch.h:53-117:
 * the 4-lag kernel and the scalar remainder accumulate each lag in ascending j) */
void pn_oracle_pitch_xcorr(const float *x, const float *y, float *xcorr, int len, int max_pitch) {
  int k;
  for (k = 0; k < max_pitch; k++) xcorr[k] = dot_seq(x, y + k, len);
}

void pn_oracle_autocorr_lpc(const float *x, int n, float *ac, float *lpc) {
  /* _celt_autocorr(x, ac, NULL, 0, lag=4, n), celt_lpc.cpp:198-279: bulk over n-4 samples, then the tail */
  int k, i, j, fast = n - 4;
  float work[5];
  pn_oracle_pitch_xcorr(x, x, ac, fast, 5);
  for (k = 0; k <= 4; k++) {
    float d = 0;
    for (i = k + fast; i < n; i++) d = d + x[i] * x[i - k];
    ac[k] += d;
  }
  /* _celt_lpc order 4 on a copy (celt_lpc.cpp:37-88); the divide runs in double (:61) */
  memcpy(work, ac, sizeof work);
  for (i = 0; i < 4; i++) lpc[i] = 0;
  if (work[0] != 0) {
    float err = work[0];
    for (i = 0; i < 4; i++) {
      float rr = 0, r;
      for (j = 0; j < i; j++) rr += lpc[j] * work[i - j];
      rr += work[i + 1];
      r = (float)(-rr / (err + 0.00001));
      lpc[i] = r;
      for (j = 0; j < (i + 1) >> 1; j++) {
        float t1 = lpc[j], t2 = lpc[i - 1 - j];
        lpc[j] = t1 + r * t2;
        lpc[i - 1 - j] = t2 + r * t1;
      }
      err = err - (r * r) * err;
      if (err < .001f * work[0]) break;
    }
  }
}

void pn_oracle_pitch_downsample(const float *x, float *lp) { /* pitch.cpp:148-216, len=1728, C=1 */
  float ac[5], lpc[4], fir[5], tmp = 1.f, raw[864];
  const float c1 = .8f;
  int i;
  for (i = 1; i < 864; i++) lp[i] = .5f * (.5f * (x[2 * i - 1] + x[2 * i + 1]) + x[2 * i]);
  lp[0] = .5f * (.5f * x[1] + x[0]);
  {
    float ac_in[5];
    pn_oracle_autocorr_lpc(lp, 864, ac_in, lpc); /* autocorrelation only; LPC redone below on the conditioned ac */
    memcpy(ac, ac_in, sizeof ac);
  }
  ac[0] *= 1.0001f;                                                   /* :190 */
  for (i = 1; i <= 4; i++) ac[i] -= ac[i] * (.008f * i) * (.008f * i); /* :199 */
  { /* Levinson on the conditioned autocorrelation (same code path as above, fed with ac) */
    int j;
    for (i = 0; i < 4; i++) lpc[i] = 0;
    if (ac[0] != 0) {
      float err = ac[0];
      for (i = 0; i < 4; i++) {
        float rr = 0, r;
        for (j = 0; j < i; j++) rr += lpc[j] * ac[i - j];
        rr += ac[i + 1];
        r = (float)(-rr / (err + 0.00001));
        lpc[i] = r;
        for (j = 0; j < (i + 1) >> 1; j++) {
          float t1 = lpc[j], t2 = lpc[i - 1 - j];
          lpc[j] = t1 + r * t2;
          lpc[i - 1 - j] = t2 + r * t1;
        }
        err = err - (r * r) * err;
        if (err < .001f * ac[0]) break;
      }
    }
  }
  for (i = 0; i < 4; i++) { tmp = .9f * tmp; lpc[i] = lpc[i] * tmp; } /* :204-208 */
  fir[0] = lpc[0] + .8f;                                               /* :210-214 */
  fir[1] = lpc[1] + c1 * lpc[0];
  fir[2] = lpc[2] + c1 * lpc[1];
  fir[3] = lpc[3] + c1 * lpc[2];
  fir[4] = c1 * lpc[3];
  /* celt_fir5 in place with zero history (pitch.cpp:106-145,154): taps see the unfiltered samples */
  memcpy(raw, lp, sizeof raw);
  for (i = 0; i < 864; i++) {
    float s = raw[i];
    int t;
    for (t = 0; t < 5; t++) s = s + fir[t] * (i - 1 - t >= 0 ? raw[i - 1 - t] : 0.f);
    lp[i] = s;
  }
}

/* pitch.cpp:46-104, float build */
static void best_two(const float *xcorr, const float *y, int len, int max_pitch, int *best) {
  float syy = 1, num0 = -1, num1 = -1, den0 = 0, den1 = 0;
  int i, j;
  best[0] = 0;
  best[1] = 1;
  for (j = 0; j < len; j++) syy = syy + y[j] * y[j];
  for (i = 0; i < max_pitch; i++) {
    if (xcorr[i] > 0) {
      float c = xcorr[i], num;
      c *= 1e-12f;
      num = c * c;
      if (num * den1 > num1 * syy) {
        if (num * den0 > num0 * syy) {
          num1 = num0; den1 = den0; best[1] = best[0];
          num0 = num;  den0 = syy;  best[0] = i;
        } else {
          num1 = num; den1 = syy; best[1] = i;
        }
      }
    }
    syy += y[i + len] * y[i + len] - y[i] * y[i];
    syy = 1 > syy ? 1 : syy;
  }
}

/* pitch.cpp:283-386 with x_lp = lp+384, y = lp, len = 960, max_pitch = 588 (denoise.cpp:406-407) */
void pn_oracle_pitch_search(const float *lp, int *pitch, float *corr, float *coarse_out, int *best_out) {
  const float *x = lp + 384, *y = lp;
  float x4[240], y4[387], xc[294];
  int best[2] = {0, 0}, i, off;
  for (i = 0; i < 240; i++) x4[i] = x[2 * i];
  for (i = 0; i < 387; i++) y4[i] = y[2 * i];
  pn_oracle_pitch_xcorr(x4, y4, xc, 240, 147);
  if (coarse_out) memcpy(coarse_out, xc, 147 * sizeof(float));
  best_two(xc, y4, 240, 147, best);
  if (best_out) { best_out[0] = best[0]; best_out[1] = best[1]; }
  for (i = 0; i < 294; i++) {
    float s;
    xc[i] = 0;
    if (abs(i - 2 * best[0]) > 2 && abs(i - 2 * best[1]) > 2) continue;
    s = dot_seq(x, y + i, 480);
    xc[i] = -1 > s ? -1 : s;
  }
  best_two(xc, y, 480, 294, best);
  if (best[0] > 0 && best[0] < 293) {
    float a = xc[best[0] - 1], b = xc[best[0]], c = xc[best[0] + 1];
    if ((c - a) > .7f * (b - a)) off = 1;
    else if ((a - c) > .7f * (b - c)) off = -1;
    else off = 0;
  } else off = 0;
  *pitch = 2 * best[0] - off;
  *corr = xc[best[0]];
}

static float pgain(float xy, float xx, float yy) { return xy / sqrtf(1 + xx * yy); } /* pitch.cpp:417-420 */

/* pitch.cpp:423-527 with maxperiod 768, minperiod 60, N 960 (denoise.cpp:410-411) */
float pn_oracle_remove_doubling(const float *lp, int *T0_, int prev_period, float prev_gain) {
  static const int second[16] = {0, 0, 3, 2, 3, 2, 5, 2, 3, 2, 3, 2, 5, 2, 3, 2};
  const int maxp = 384, minp = 30, N = 480, minp0 = 60;
  const float *x = lp + maxp;
  float yy_tab[385], xx, xy, xy2, yy, g, g0, pg, best_xy, best_yy, xc[3];
  int k, i, T, T0, off;
  *T0_ /= 2;
  prev_period /= 2;
  if (*T0_ >= maxp) *T0_ = maxp - 1;
  T = T0 = *T0_;
  xx = 0; xy = 0;
  for (i = 0; i < N; i++) { xx = xx + x[i] * x[i]; xy = xy + x[i] * x[i - T0]; }
  yy_tab[0] = xx;
  yy = xx;
  for (i = 1; i <= maxp; i++) {
    yy = yy + x[-i] * x[-i] - x[N - i] * x[N - i];
    yy_tab[i] = 0 > yy ? 0 : yy;
  }
  yy = yy_tab[T0];
  best_xy = xy;
  best_yy = yy;
  g = g0 = pgain(xy, xx, yy);
  for (k = 2; k <= 15; k++) {
    int T1 = (2 * T0 + k) / (2 * k), T1b;
    float g1, cont, thresh;
    if (T1 < minp) break;
    if (k == 2) T1b = (T1 + T0 > maxp) ? T0 : T0 + T1;
    else T1b = (2 * second[k] * T0 + k) / (2 * k);
    xy = 0; xy2 = 0;
    for (i = 0; i < N; i++) { xy = xy + x[i] * x[i - T1]; xy2 = xy2 + x[i] * x[i - T1b]; }
    xy = .5f * (xy + xy2);
    yy = .5f * (yy_tab[T1] + yy_tab[T1b]);
    g1 = pgain(xy, xx, yy);
    if (abs(T1 - prev_period) <= 1) cont = prev_gain;
    else if (abs(T1 - prev_period) <= 2 && 5 * k * k < T0) cont = .5f * prev_gain;
    else cont = 0;
    thresh = .3f > .7f * g0 - cont ? .3f : .7f * g0 - cont;
    if (T1 < 3 * minp) thresh = .4f > .85f * g0 - cont ? .4f : .85f * g0 - cont;
    else if (T1 < 2 * minp) thresh = .5f > .9f * g0 - cont ? .5f : .9f * g0 - cont; /* unreachable, App. C.9 */
    if (g1 > thresh) { best_xy = xy; best_yy = yy; T = T1; g = g1; }
  }
  best_xy = 0 > best_xy ? 0 : best_xy;
  if (best_yy <= best_xy) pg = 1.f;
  else pg = best_xy / (best_yy + 1);
  for (k = 0; k < 3; k++) xc[k] = dot_seq(x, x - (T + k - 1), N);
  if ((xc[2] - xc[0]) > .7f * (xc[1] - xc[0])) off = 1;
  else if ((xc[0] - xc[2]) > .7f * (xc[1] - xc[2])) off = -1;
  else off = 0;
  if (pg > g) pg = g;
  *T0_ = 2 * T + off;
  if (*T0_ < minp0) *T0_ = minp0;
  return pg;
}

/* ------------------------------------------------------------------------------------ */
/*  Network (nnet.cpp, rnn.cpp, vec.h)                                                    */
/* ------------------------------------------------------------------------------------ */
float pn_oracle_tansig(float x) { /* vec.h:53-71 */
  float y, dy, sign = 1;
  int i;
  build_tables();
  if (x < 0) { x = -x; sign = -1; }
  i = (int)floor(.5f + 25 * x);
  i = i < 200 ? i : 200;
  i = i > 0 ? i : 0;
  x -= .04f * i;
  y = K.tansig[i];
  dy = 1 - y * y;
  y = y + x * dy * (1 - y * x);
  return sign * y;
}
float pn_oracle_sigmoid(float x) { return .5f + .5f * pn_oracle_tansig(.5f * x); } /* vec.h:73-76 */
/* the two above over n values in one call (tests evaluate millions) */
void pn_oracle_tansig_n(const float *x, float *y, long n) {
  long i;
  for (i = 0; i < n; i++) y[i] = pn_oracle_tansig(x[i]);
}
void pn_oracle_sigmoid_n(const float *x, float *y, long n) {
  long i;
  for (i = 0; i < n; i++) y[i] = pn_oracle_sigmoid(x[i]);
}

static void activate(float *v, int n, int act) { /* nnet.cpp:74-103 */
  int i;
  if (act == PNB_ACT_SIGMOID) for (i = 0; i < n; i++) v[i] = pn_oracle_sigmoid(v[i]);
  else if (act == PNB_ACT_TANH) for (i = 0; i < n; i++) v[i] = pn_oracle_tansig(v[i]);
  else if (act == PNB_ACT_RELU) for (i = 0; i < n; i++) v[i] = v[i] < 0 ? 0 : v[i];
}
/* out[i] += sum_j W[j*stride+i] x[j], j ascending, mul then add (nnet.cpp:59-72, vec.h:102-135) */
static void gemv_acc(float *out, const float *W, int rows, int cols, int stride, const float *x) {
  int i, j;
  for (j = 0; j < cols; j++) {
    float xj = x[j];
    const float *w = W + (size_t)j * stride;
    for (i = 0; i < rows; i++) out[i] += w[i] * xj;
  }
}
void pn_oracle_dense_layer(const pnb_dense_layer *l, float *out, const float *in) { /* nnet.cpp:105-118 */
  int N = l->nb_neurons;
  memcpy(out, l->bias, N * sizeof(float));
  gemv_acc(out, l->input_weights, N, l->nb_inputs, N, in);
  activate(out, N, l->activation);
}
void pn_oracle_conv1d_layer(const pnb_conv1d_layer *l, float *out, float *mem, const float *in) { /* nnet.cpp:182-200 */
  int C = l->nb_inputs, Kt = l->kernel_size, N = l->nb_neurons;
  float *cat = (float *)malloc((size_t)C * Kt * sizeof(float));
  memcpy(cat, mem, (size_t)C * (Kt - 1) * sizeof(float));
  memcpy(cat + C * (Kt - 1), in, C * sizeof(float));
  memcpy(out, l->bias, N * sizeof(float));
  gemv_acc(out, l->input_weights, N, C * Kt, N, cat);
  activate(out, N, l->activation);
  memcpy(mem, cat + C, (size_t)C * (Kt - 1) * sizeof(float));
  free(cat);
}
void pn_oracle_gru_layer(const pnb_gru_layer *l, float *h, const float *in) { /* nnet.cpp:120-180, reset_after only */
  int N = l->nb_neurons, M = l->nb_inputs, S = 3 * N, i;
  float *z = (float *)malloc(4 * (size_t)N * sizeof(float)), *r = z + N, *c = r + N, *t = c + N;
  const float *b = l->bias, *W = l->input_weights, *U = l->recurrent_weights;
  for (i = 0; i < N; i++) z[i] = b[i];
  for (i = 0; i < N; i++) z[i] += b[3 * N + i];
  gemv_acc(z, W, N, M, S, in);
  gemv_acc(z, U, N, N, S, h);
  activate(z, N, PNB_ACT_SIGMOID);
  for (i = 0; i < N; i++) r[i] = b[N + i];
  for (i = 0; i < N; i++) r[i] += b[4 * N + i];
  gemv_acc(r, W + N, N, M, S, in);
  gemv_acc(r, U + N, N, N, S, h);
  activate(r, N, PNB_ACT_SIGMOID);
  for (i = 0; i < N; i++) c[i] = b[2 * N + i];
  for (i = 0; i < N; i++) t[i] = b[5 * N + i];
  gemv_acc(t, U + 2 * N, N, N, S, h);
  for (i = 0; i < N; i++) c[i] += t[i] * r[i];
  gemv_acc(c, W + 2 * N, N, M, S, in);
  activate(c, N, l->activation);
  for (i = 0; i < N; i++) c[i] = z[i] * h[i] + (1 - z[i]) * c[i];
  memcpy(h, c, N * sizeof(float));
  free(z);
}
void pn_oracle_compute_rnn(const pnb_model *m, float *st, float *gains, float *strengths, const float *feat) {
  /* rnn.cpp:42-81; later layers read the already-updated states of earlier ones (App. C.10) */
  float d0[128], c1[512], c2[512], rb_in[1024], gb_in[2560];
  float *m1 = st, *m2 = st + 512, *h1 = st + 1536, *h2 = h1 + 512, *h3 = h2 + 512, *hg = h3 + 512, *hr = hg + 512;
  pn_oracle_dense_layer(m->fc, d0, feat);
  pn_oracle_conv1d_layer(m->conv1, c1, m1, d0);
  pn_oracle_conv1d_layer(m->conv2, c2, m2, c1);
  pn_oracle_gru_layer(m->gru1, h1, c2);
  pn_oracle_gru_layer(m->gru2, h2, h1);
  pn_oracle_gru_layer(m->gru3, h3, h2);
  pn_oracle_gru_layer(m->gru_gb, hg, h3);
  memcpy(rb_in, h3, 512 * sizeof(float));
  memcpy(rb_in + 512, c2, 512 * sizeof(float));
  pn_oracle_gru_layer(m->gru_rb, hr, rb_in);
  memcpy(gb_in, c2, 512 * sizeof(float));
  memcpy(gb_in + 512, h1, 512 * sizeof(float));
  memcpy(gb_in + 1024, h2, 512 * sizeof(float));
  memcpy(gb_in + 1536, h3, 512 * sizeof(float));
  memcpy(gb_in + 2048, hg, 512 * sizeof(float));
  pn_oracle_dense_layer(m->fc_gb, gains, gb_in);
  pn_oracle_dense_layer(m->fc_rb, strengths, hr);
}

/* the pitch analysis of n independent 1728-sample pitch buffers (denoise.cpp:404-414), OpenMP over units */
void pn_oracle_pitch_batch(const float *bufs, size_t stride, int n, const int *prev_period, const float *prev_gain,
                           int *T_out, float *corr_out, float *gain_out, int n_threads) {
  int u;
#ifdef _OPENMP
#pragma omp parallel for num_threads(n_threads > 0 ? n_threads : 1) schedule(static)
#endif
  for (u = 0; u < n; u++) {
    float lp[864], corr;
    int pitch, T;
    pn_oracle_pitch_downsample(bufs + (size_t)u * stride, lp);
    pn_oracle_pitch_search(lp, &pitch, &corr, NULL, NULL);
    T = 768 - pitch;
    gain_out[u] = pn_oracle_remove_doubling(lp, &T, prev_period ? prev_period[u] : 0, prev_gain ? prev_gain[u] : 0.f);
    T_out[u] = T;
    corr_out[u] = corr;
  }
  (void)n_threads;
}

/* ------------------------------------------------------------------------------------ */
/*  The same network in double precision: the arbiter between two single-precision         */
/*  evaluations (the reference's sequential fp32 sums and the GPU's split-operand tensor    */
/*  products).  Same wiring (rnn.cpp:42-81), same tansig table and correction formula       */
/*  (vec.h:53-71) evaluated in double.  Returns through *max_pre the largest |x| handed to  */
/*  tansig_approx, so that a test can tell whether a frame stayed inside the domain in      */
/*  which the reference's float->int conversion is defined (|x| < 8.6e7, vec.h:63).         */
/* ------------------------------------------------------------------------------------ */
static double tansig_d(double x, double *max_pre) {
  double y, dy, sign = 1, fi;
  int i;
  build_tables();
  if (x < 0) { x = -x; sign = -1; }
  if (x > *max_pre) *max_pre = x;
  fi = floor(.5 + 25 * x);
  i = fi < 200 ? (int)fi : 200;
  i = i > 0 ? i : 0;
  x -= .04 * i;
  y = (double)K.tansig[i];
  dy = 1 - y * y;
  y = y + x * dy * (1 - y * x);
  return sign * y;
}
static void activate_d(double *v, int n, int act, double *mp) {
  int i;
  if (act == PNB_ACT_SIGMOID) for (i = 0; i < n; i++) v[i] = .5 + .5 * tansig_d(.5 * v[i], mp);
  else if (act == PNB_ACT_TANH) for (i = 0; i < n; i++) v[i] = tansig_d(v[i], mp);
  else if (act == PNB_ACT_RELU) for (i = 0; i < n; i++) v[i] = v[i] < 0 ? 0 : v[i];
}
static void gemv_acc_d(double *out, const float *W, int rows, int cols, int stride, const double *x) {
  int i, j;
  for (j = 0; j < cols; j++) {
    double xj = x[j];
    const float *w = W + (size_t)j * stride;
    for (i = 0; i < rows; i++) out[i] += (double)w[i] * xj;
  }
}
static void dense_d(const pnb_dense_layer *l, double *out, const double *in, double *mp) {
  int N = l->nb_neurons, i;
  for (i = 0; i < N; i++) out[i] = l->bias[i];
  gemv_acc_d(out, l->input_weights, N, l->nb_inputs, N, in);
  activate_d(out, N, l->activation, mp);
}
static void conv1d_d(const pnb_conv1d_layer *l, double *out, double *mem, const double *in, double *mp) {
  int C = l->nb_inputs, Kt = l->kernel_size, N = l->nb_neurons, i;
  double *cat = (double *)malloc((size_t)C * Kt * sizeof(double));
  memcpy(cat, mem, (size_t)C * (Kt - 1) * sizeof(double));
  memcpy(cat + C * (Kt - 1), in, C * sizeof(double));
  for (i = 0; i < N; i++) out[i] = l->bias[i];
  gemv_acc_d(out, l->input_weights, N, C * Kt, N, cat);
  activate_d(out, N, l->activation, mp);
  memcpy(mem, cat + C, (size_t)C * (Kt - 1) * sizeof(double));
  free(cat);
}
static void gru_d(const pnb_gru_layer *l, double *h, const double *in, double *mp) {
  int N = l->nb_neurons, M = l->nb_inputs, S = 3 * N, i;
  double *z = (double *)malloc(4 * (size_t)N * sizeof(double)), *r = z + N, *c = r + N, *t = c + N;
  const float *b = l->bias, *W = l->input_weights, *U = l->recurrent_weights;
  for (i = 0; i < N; i++) z[i] = (double)b[i] + (double)b[3 * N + i];
  gemv_acc_d(z, W, N, M, S, in);
  gemv_acc_d(z, U, N, N, S, h);
  activate_d(z, N, PNB_ACT_SIGMOID, mp);
  for (i = 0; i < N; i++) r[i] = (double)b[N + i] + (double)b[4 * N + i];
  gemv_acc_d(r, W + N, N, M, S, in);
  gemv_acc_d(r, U + N, N, N, S, h);
  activate_d(r, N, PNB_ACT_SIGMOID, mp);
  for (i = 0; i < N; i++) { c[i] = b[2 * N + i]; t[i] = b[5 * N + i]; }
  gemv_acc_d(t, U + 2 * N, N, N, S, h);
  for (i = 0; i < N; i++) c[i] += t[i] * r[i];
  gemv_acc_d(c, W + 2 * N, N, M, S, in);
  activate_d(c, N, l->activation, mp);
  for (i = 0; i < N; i++) h[i] = z[i] * h[i] + (1 - z[i]) * c[i];
  free(z);
}
double pn_oracle_compute_rnn_f64(const pnb_model *m, double *st, double *gains, double *strengths, const float *feat) {
  double f[PNO_FEATURES], d0[128], c1[512], c2[512], rb_in[1024], gb_in[2560], mp = 0.0;
  double *m1 = st, *m2 = st + 512, *h1 = st + 1536, *h2 = h1 + 512, *h3 = h2 + 512, *hg = h3 + 512, *hr = hg + 512;
  int i;
  for (i = 0; i < PNO_FEATURES; i++) f[i] = feat[i];
  dense_d(m->fc, d0, f, &mp);
  conv1d_d(m->conv1, c1, m1, d0, &mp);
  conv1d_d(m->conv2, c2, m2, c1, &mp);
  gru_d(m->gru1, h1, c2, &mp);
  gru_d(m->gru2, h2, h1, &mp);
  gru_d(m->gru3, h3, h2, &mp);
  gru_d(m->gru_gb, hg, h3, &mp);
  memcpy(rb_in, h3, 512 * sizeof(double));
  memcpy(rb_in + 512, c2, 512 * sizeof(double));
  gru_d(m->gru_rb, hr, rb_in, &mp);
  memcpy(gb_in, c2, 512 * sizeof(double));
  memcpy(gb_in + 512, h1, 512 * sizeof(double));
  memcpy(gb_in + 1024, h2, 512 * sizeof(double));
  memcpy(gb_in + 1536, h3, 512 * sizeof(double));
  memcpy(gb_in + 2048, hg, 512 * sizeof(double));
  dense_d(m->fc_gb, gains, gb_in, &mp);
  dense_d(m->fc_rb, strengths, hr, &mp);
  return mp;
}

/* ------------------------------------------------------------------------------------ */
/*  Per-stream engine.  hist[] is the reference's comb_buf (denoise.cpp:77,388-389); its   */
/*  pitch_buf and analysis_mem are windows of it (SURVEY.md App. A.2):                     */
/*    pitch_buf = hist[1632 .. 3360)   analysis window = hist[2400 .. 3360)                */
/*    look-ahead window = hist[4800 .. 5760)   comb taps read hist[2400 - kT + i]          */
/* ------------------------------------------------------------------------------------ */
struct pn_oracle {
  const pnb_model *model;
  float hist[PNO_HIST];
  float synth_mem[FRAME];
  int last_period;
  float last_gain;
  float nn[PNO_NN_STATE];
};

pn_oracle *pn_oracle_create(const pnb_model *model) {
  pn_oracle *o = (pn_oracle *)calloc(1, sizeof *o);
  build_tables();
  o->model = model;
  return o;
}
void pn_oracle_destroy(pn_oracle *o) { free(o); }
void pn_oracle_reset(pn_oracle *o) {
  const pnb_model *m = o->model;
  memset(o, 0, sizeof *o);
  o->model = m;
}

/* compute_frame_features (denoise.cpp:364-434) followed by compute_lookahead_band_energy (:498-506): everything
 * the enhancement path and the training-data path share. */
typedef struct {
  cpx X[NFREQ], P[NFREQ], Y[NFREQ];
  float Ex[NB], Ep[NB], Exp[NB], Ey[NB], lp[864], corr, gain;
  int pitch, T, silence;
} frame_analysis;

static void analyse_frame(pn_oracle *o, const float *in, frame_analysis *a, pn_oracle_taps *tp) {
  cpx *X = a->X, *P = a->P, *Y = a->Y;
  float *Ex = a->Ex, *Ep = a->Ep, *Exp = a->Exp, *Ey = a->Ey, *lp = a->lp;
  float buf[WIN], corr, gain, E = 0;
  int i, k, pitch, T;

  /* slide the history line and append the new hop (denoise.cpp:388-389) */
  memmove(o->hist, o->hist + FRAME, (PNO_HIST - FRAME) * sizeof(float));
  memcpy(o->hist + PNO_HIST - FRAME, in, FRAME * sizeof(float));

  /* analysis of the frame delayed by five hops (denoise.cpp:402, :333-346) */
  memcpy(buf, o->hist + 2400, sizeof buf);
  window_inplace(buf);
  spectrum_of(buf, X);
  band_pool(Ex, X, X);

  /* pitch (denoise.cpp:404-414) */
  pn_oracle_pitch_downsample(o->hist + 1632, lp);
  pn_oracle_pitch_search(lp, &pitch, &corr, tp ? tp->xcorr_coarse : NULL, tp ? tp->best_coarse : NULL);
  T = 768 - pitch;
  gain = pn_oracle_remove_doubling(lp, &T, o->last_period, o->last_gain);
  o->last_period = T;
  o->last_gain = gain;

  /* comb-filtered frame, its spectrum, band statistics (denoise.cpp:416-427) */
  for (i = 0; i < WIN; i++) buf[i] = 0;
  for (k = -3; k <= 3; k++)
    for (i = 0; i < WIN; i++) buf[i] += o->hist[2400 - T * k + i] * K.comb_w[k + 3];
  window_inplace(buf);
  spectrum_of(buf, P);
  band_pool(Ep, P, P);
  band_pool(Exp, X, P);
  for (i = 0; i < NB; i++) {
    double v = Exp[i] / sqrt(1e-15 + Ex[i] * Ep[i]); /* float product, then double (H4) */
    v = fmax(0, v);
    Exp[i] = (float)fmin(1, v);
  }
  for (i = 0; i < NB; i++) E += Ex[i];
  a->silence = E < 0.1; /* float promoted to double against the double literal, :433 */

  /* look-ahead band energies from the newest 960 samples (denoise.cpp:498-506) */
  memcpy(buf, o->hist + PNO_HIST - WIN, sizeof buf);
  window_inplace(buf);
  spectrum_of(buf, Y);
  band_pool(Ey, Y, Y);
  a->corr = corr; a->gain = gain; a->pitch = pitch; a->T = T;
}

void pn_oracle_process_frame(pn_oracle *o, float *out, const float *in, pn_oracle_taps *tp, int flags) {
  frame_analysis fa;
  cpx *X = fa.X, *P = fa.P, *Y = fa.Y;
  float *Ex = fa.Ex, *Ep = fa.Ep, *Exp = fa.Exp, *Ey = fa.Ey, *lp = fa.lp;
  float feat[PNO_FEATURES], g[NB], r[NB], gbin[NFREQ], buf[WIN], corr, gain;
  int i, T, silence;

  analyse_frame(o, in, &fa, tp);
  corr = fa.corr; gain = fa.gain; T = fa.T; silence = fa.silence;
  if (tp) tp->pitch_search = fa.pitch;

  /* features (denoise.cpp:487-496, 528-530) */
  for (i = 0; i < NB; i++) feat[i] = Ey[i] * 30;
  for (i = 0; i < NB; i++) feat[NB + i] = Exp[i] * 30;
  feat[68] = (float)o->last_period / (768 - 3 * 60);
  feat[69] = corr;

  pn_oracle_compute_rnn(o->model, o->nn, g, r, feat);

  if (tp) {
    memcpy(tp->X, X, sizeof fa.X); memcpy(tp->P, P, sizeof fa.P); memcpy(tp->Y, Y, sizeof fa.Y);
    memcpy(tp->Ex, Ex, sizeof fa.Ex); memcpy(tp->Ep, Ep, sizeof fa.Ep); memcpy(tp->Exp, Exp, sizeof fa.Exp);
    memcpy(tp->Ex_look, Ey, sizeof fa.Ey); memcpy(tp->features, feat, sizeof feat);
    memcpy(tp->g, g, sizeof g); memcpy(tp->r, r, sizeof r); memcpy(tp->lp, lp, sizeof fa.lp);
    tp->pitch_corr = corr; tp->pitch_index = T; tp->pitch_gain = gain; tp->silence = silence;
  }

  if (flags & PNO_POSTFILTER) pn_oracle_post_filter(g, Ex); /* where the paper puts it; off by default (SURVEY 0.7) */
  if (tp) memcpy(tp->g_used, g, sizeof g);

  if (!silence) comb_mix(X, P, r);  /* denoise.cpp:536-538 */
  band_to_bins(gbin, g);            /* :539 */
  for (i = 0; i < NFREQ; i++) { X[i].r *= gbin[i]; X[i].i *= gbin[i]; }
  if (tp) memcpy(tp->Xout, X, sizeof fa.X);

  /* synthesis: inverse transform, window, overlap-add (denoise.cpp:352-359) */
  signal_of(X, buf);
  window_inplace(buf);
  for (i = 0; i < FRAME; i++) out[i] = buf[i] + o->synth_mem[i];
  memcpy(o->synth_mem, buf + FRAME, FRAME * sizeof(float));
}

/* ------------------------------------------------------------------------------------ */
/*  Training-data path (SURVEY.md 8 row f1): the labels of denoise.cpp:549-589 and the      */
/*  per-frame record of train() (denoise.cpp:600-787, as shipped: gains fixed at 1, no      */
/*  biquads, the second file is the already-mixed noisy signal).  denoise.cpp is C++, so    */
/*  sqrt() of a float expression is the float overload; of a double expression, double.     */
/* ------------------------------------------------------------------------------------ */
void pn_oracle_ideal_labels(const float *Ex, const float *Ey, const float *Exp, const float *Ephaty, float *g, float *r) {
  float pna = 0, n0 = (float)0.03, Ephatp[NB];
  int i;
  build_tables();
  for (i = 0; i < 7; i++) pna += K.comb_w[i] * K.comb_w[i];                 /* denoise.cpp:207-210 */
  for (i = 0; i < NB; i++) {                                                /* calc_ideal_gain, :571-577 */
    g[i] = (float)(Ex[i] / (.0001 + Ey[i]));
    if (g[i] > 1) g[i] = 1;
    if (g[i] < 0) g[i] = 0;
  }
  for (i = 0; i < NB; i++)                                                  /* estimate_phat_corr, :549-553 */
    Ephatp[i] = (float)(Ephaty[i] / sqrt((1 - pna) * pow(Ephaty[i], 2) + pna));
  for (i = 0; i < NB; i++) {                                                /* filter_strength_calc, :555-569 */
    float a, b, c, alpha, q = Ephaty[i];
    a = Ephatp[i] * Ephatp[i] - Exp[i] * Exp[i];
    if (a < 0) a = 0;
    b = Ephatp[i] * q * (1 - Exp[i] * Exp[i]);
    c = Exp[i] * Exp[i] - q * q;
    if (c < 0) c = 0;
    alpha = (float)((sqrtf(b * b + a * c) - b) / (a + 1e-8));
    r[i] = alpha / (1 + alpha);
  }
  for (i = 0; i < NB; i++)                                                  /* adjust_gain_strength_by_condition, :579-589 */
    if (Ephatp[i] < Exp[i]) {
      float g_att = sqrtf((1 + n0 - Exp[i] * Exp[i]) / (1 + n0 - Ephatp[i] * Ephatp[i]));
      r[i] = (float)0.99;
      g[i] *= g_att;
    }
}

/* train() on in-memory files: speech/noisy hold count*480 int16 samples each (no wrap-around);
 * records gets count*138 floats: Ey_lookahead[34] Ephaty[34] T pitchcorr g[34] r[34] (denoise.cpp:761-773). */
void pn_oracle_train_records(const short *speech, const short *noisy, int count, float *records) {
  pn_oracle *st = pn_oracle_create(NULL), *ns = pn_oracle_create(NULL);
  frame_analysis *fx = (frame_analysis *)malloc(sizeof *fx), *fy = (frame_analysis *)malloc(sizeof *fy);
  float x[FRAME], xn[FRAME];
  int t, i;
  for (t = 0; t < count; t++) {
    float *rec = records + (size_t)t * 138;
    for (i = 0; i < FRAME; i++) x[i] = (float)speech[(size_t)t * FRAME + i];  /* NORM_RATIO 1, speech_gain 1 */
    for (i = 0; i < FRAME; i++) xn[i] = (float)noisy[(size_t)t * FRAME + i];
    analyse_frame(ns, xn, fy, NULL);
    analyse_frame(st, x, fx, NULL);
    memcpy(rec, fy->Ey, NB * sizeof(float));
    memcpy(rec + NB, fy->Exp, NB * sizeof(float));
    rec[68] = (float)ns->last_period / (768 - 3 * 60);
    rec[69] = fy->corr;
    pn_oracle_ideal_labels(fx->Ex, fy->Ex, fx->Exp, fy->Exp, rec + 70, rec + 104);
    /* denoise.cpp:45-46 defines TEST, so the shipped train() post-filters g in place (:742-743) before it is
     * written; the rest of the TEST block (test_input.pcm / test_output.pcm debug audio) does not touch the record. */
    pn_oracle_post_filter(rec + 70, fy->Ex);
  }
  free(fx); free(fy);
  pn_oracle_destroy(st); pn_oracle_destroy(ns);
}

void pn_oracle_process_stream(pn_oracle *o, float *out, const float *in, int n_frames, float *gr, int flags) {
  int t;
  for (t = 0; t < n_frames; t++) {
    if (gr) {
      pn_oracle_taps *tp = (pn_oracle_taps *)malloc(sizeof *tp);
      pn_oracle_process_frame(o, out + FRAME * t, in + FRAME * t, tp, flags);
      memcpy(gr + 68 * t, tp->g, NB * sizeof(float));
      memcpy(gr + 68 * t + NB, tp->r, NB * sizeof(float));
      free(tp);
    } else {
      pn_oracle_process_frame(o, out + FRAME * t, in + FRAME * t, NULL, flags);
    }
  }
}

void pn_oracle_run_pcm16(const pnb_model *m, const short *in16, int n_frames, short *out16, float *gr) {
  /* src/main.cpp:30-39: /32768.f in, truncating *32768 out, first output frame dropped */
  pn_oracle *o = pn_oracle_create(m);
  int t, i;
  for (t = 0; t < n_frames; t++) {
    float x[FRAME];
    for (i = 0; i < FRAME; i++) x[i] = ((float)in16[FRAME * t + i]) / 32768.f;
    pn_oracle_process_stream(o, x, x, 1, gr ? gr + 68 * t : NULL, 0);
    if (t > 0)
      for (i = 0; i < FRAME; i++) out16[FRAME * (t - 1) + i] = (short)(x[i] * 32768);
  }
  pn_oracle_destroy(o);
}

void pn_oracle_process_streams(const pnb_model *m, int n_streams, int n_frames, const float *in, float *out,
                               int n_threads, int flags) {
  int s;
  build_tables();
#ifdef _OPENMP
#pragma omp parallel for schedule(dynamic, 1) num_threads(n_threads)
#endif
  for (s = 0; s < n_streams; s++) {
    pn_oracle *o = pn_oracle_create(m);
    pn_oracle_process_stream(o, out + (size_t)s * n_frames * FRAME, in + (size_t)s * n_frames * FRAME, n_frames, NULL, flags);
    pn_oracle_destroy(o);
  }
  (void)n_threads;
}
