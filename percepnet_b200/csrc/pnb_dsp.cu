// pnb_dsp.cu -- analysis and synthesis kernels of the PercepNet hot path for sm_90a.
//
// One warp owns one utterance stream and walks the hops of the call in order, carrying the
// per-stream scalar state (last pitch period / gain, overlap-add memory) in registers.
// What it replaces in the reference (paths relative to /root/reference/src):
//   analysis_kernel : compute_frame_features (denoise.cpp:372-434), frame_analysis (:333),
//                     apply_window (:282), forward_transform (:291) + opus_fft_c (kiss_fft.cpp:566),
//                     compute_band_energy/corr (:89,:125), pitch_downsample / pitch_search /
//                     remove_doubling (pitch.cpp:148,283,424), _celt_autocorr/_celt_lpc
//                     (celt_lpc.cpp:198,37), comb filter (:416-427), compute_lookahead_band_energy
//                     (:498), create_features (:487)
//   synthesis_kernel: pitch_filter (:436), interp_band_gain (:162), gain apply (:539-544),
//                     post_filtering (:216), frame_synthesis (:352) + inverse_transform (:306)
//
// Numerics: this translation unit is compiled with -fmad=false and every decision-critical sum is a
// strict ascending multiply-then-add chain, so pitch decisions, spectra and features are bit-identical
// to the reference (whose objects contain no FMA and no re-associated sums, SURVEY.md 0.9 / H1).
// The two double-precision islands (denoise.cpp:427, celt_lpc.cpp:61) run in fp64 here as well.
#include <stdlib.h>
#include "pnb_kernels.h"

namespace pnb {

// ------------------------------------------------------------------------------------------
// warp-level FFT-960 over a shared-memory line (kiss_fft.cpp:518-586: factors 5,3,4,4,4 executed
// as radix-4 (m=1,4,16), radix-3 (m=64), radix-5 (m=192) on a digit-reversed, 1/960-scaled input)
// ------------------------------------------------------------------------------------------
__device__ __forceinline__ float2 cmul(float2 a, float2 b) {
  return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x);
}
__device__ __forceinline__ float2 cadd(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ float2 csub(float2 a, float2 b) { return make_float2(a.x - b.x, a.y - b.y); }

// position of input sample i after the digit reversal of the 5.3.4.4.4 factorisation
__device__ __forceinline__ int fft_slot(int i) {
  int n0 = i % 5; i /= 5;
  int n1 = i % 3; i /= 3;
  int n2 = i & 3; i >>= 2;
  int n3 = i & 3; i >>= 2;
  return 192 * n0 + 64 * n1 + 16 * n2 + 4 * n3 + i;
}

// Work-line layout: element e lives at float2 index e + 2 (e >> 4), i.e. 16 bytes of padding after every 16
// complex values, so that a lane's 128-byte block and the stride-16 / stride-192 walks of the later passes
// are free of shared-memory bank conflicts.
constexpr int kFftLine = kWin + 2 * (kWin / 16);  // 1080 float2
__device__ __forceinline__ int fpos(int e) { return e + 2 * (e >> 4); }

struct FftTw {            // per-block tables in shared memory
  float2 tw[kWin];        // exp(-2 pi i k / 960)                       (kiss_fft.cpp:415-419)
  float2 tw5[4][192];     // tw[m u], m = 1..4: the radix-5 twiddles, contiguous in u
};

// Three register-blocked passes over the five kiss_fft stages (kiss_fft.cpp:518-564: radix 4,4,4,3,5 with
// m = 1,4,16,64,192 on the digit-reversed, 1/960-scaled input).  Every butterfly performs exactly the
// reference's operations in the reference's order; only the order BETWEEN independent butterflies differs.
//   pass A: lane loads the 16 inputs of a 16-element output block straight from `load(i)` (no scatter
//           through shared memory), does radix-4 m=1 and radix-4 m=4 in registers, stores 128 contiguous bytes
//   pass B: radix-4 m=16 then radix-3 m=64 on the 12 elements {192 n0 + 64 r + 16 q + j}
//   pass C: radix-5 m=192
// The 32 lanes of a warp cooperate on one transform.
template <bool kAllOutputs, class Load>
__device__ __forceinline__ void fft960_warp(float2 *f, const FftTw &T, int lane, Load load) {
  __syncwarp();
  {  // ---------------- pass A ----------------
    const float2 t1a = T.tw[60], t1b = T.tw[120], t1c = T.tw[180];    // j = 1: tw[60 j], tw[120 j], tw[180 j]
    const float2 t2a = T.tw[120], t2b = T.tw[240], t2c = T.tw[360];   // j = 2
    const float2 t3a = T.tw[180], t3b = T.tw[360], t3c = T.tw[540];   // j = 3
    const float2 t0 = T.tw[0];
    for (int b = lane; b < 60; b += 32) {
      const int n0 = b / 12, n1 = (b >> 2) % 3, n2 = b & 3;
      const int ibase = n0 + 5 * n1 + 15 * n2;
      float2 v[16];
#pragma unroll
      for (int n3 = 0; n3 < 4; n3++)
#pragma unroll
        for (int n4 = 0; n4 < 4; n4++) v[4 * n3 + n4] = load(ibase + 60 * n3 + 240 * n4);
#pragma unroll
      for (int q = 0; q < 4; q++) {  // radix-4, m = 1 (kiss_fft.cpp:112-131)
        float2 a0 = v[4 * q], a1 = v[4 * q + 1], a2 = v[4 * q + 2], a3 = v[4 * q + 3];
        float2 d02 = csub(a0, a2);
        a0 = cadd(a0, a2);
        float2 s13 = cadd(a1, a3);
        a2 = csub(a0, s13);
        a0 = cadd(a0, s13);
        float2 d13 = csub(a1, a3);
        v[4 * q] = a0;
        v[4 * q + 2] = a2;
        v[4 * q + 1] = make_float2(d02.x + d13.y, d02.y - d13.x);
        v[4 * q + 3] = make_float2(d02.x - d13.y, d02.y + d13.x);
      }
#pragma unroll
      for (int j = 0; j < 4; j++) {  // radix-4, m = 4, twiddle stride 60 (kiss_fft.cpp:132-166)
        const float2 wa = j == 0 ? t0 : j == 1 ? t1a : j == 2 ? t2a : t3a;
        const float2 wb = j == 0 ? t0 : j == 1 ? t1b : j == 2 ? t2b : t3b;
        const float2 wc = j == 0 ? t0 : j == 1 ? t1c : j == 2 ? t2c : t3c;
        float2 a = cmul(v[j + 4], wa), bb = cmul(v[j + 8], wb), c = cmul(v[j + 12], wc);
        float2 f0 = v[j];
        float2 d0b = csub(f0, bb);
        f0 = cadd(f0, bb);
        float2 sac = cadd(a, c), dac = csub(a, c);
        v[j + 8] = csub(f0, sac);
        v[j] = cadd(f0, sac);
        v[j + 4] = make_float2(d0b.x + dac.y, d0b.y - dac.x);
        v[j + 12] = make_float2(d0b.x - dac.y, d0b.y + dac.x);
      }
      float4 *dst = reinterpret_cast<float4 *>(f + 18 * b);
#pragma unroll
      for (int k = 0; k < 8; k++) dst[k] = make_float4(v[2 * k].x, v[2 * k].y, v[2 * k + 1].x, v[2 * k + 1].y);
    }
  }
  __syncwarp();
  {  // ---------------- pass B ----------------
    const float w3i = T.tw[320].y;  // epi3, kiss_fft.cpp:194
    for (int g = lane; g < 80; g += 32) {
      const int n0 = g >> 4, jj = g & 15;
      const int e0 = 192 * n0 + jj;
      float2 v[3][4];
#pragma unroll
      for (int r = 0; r < 3; r++)
#pragma unroll
        for (int q = 0; q < 4; q++) v[r][q] = f[fpos(e0 + 64 * r + 16 * q)];
      const float2 wa = T.tw[15 * jj], wb = T.tw[30 * jj], wc = T.tw[45 * jj];
#pragma unroll
      for (int r = 0; r < 3; r++) {  // radix-4, m = 16, twiddle stride 15
        float2 a = cmul(v[r][1], wa), bb = cmul(v[r][2], wb), c = cmul(v[r][3], wc);
        float2 f0 = v[r][0];
        float2 d0b = csub(f0, bb);
        f0 = cadd(f0, bb);
        float2 sac = cadd(a, c), dac = csub(a, c);
        v[r][2] = csub(f0, sac);
        v[r][0] = cadd(f0, sac);
        v[r][1] = make_float2(d0b.x + dac.y, d0b.y - dac.x);
        v[r][3] = make_float2(d0b.x - dac.y, d0b.y + dac.x);
      }
#pragma unroll
      for (int q = 0; q < 4; q++) {  // radix-3, m = 64, twiddle stride 5 (kiss_fft.cpp:173-228)
        const int j64 = jj + 16 * q;
        float2 a = cmul(v[1][q], T.tw[5 * j64]);
        float2 bb = cmul(v[2][q], T.tw[10 * j64]);
        float2 s = cadd(a, bb), d = csub(a, bb);
        float2 f0 = v[0][q];
        float2 f1 = make_float2(f0.x - s.x * .5f, f0.y - s.y * .5f);
        d.x *= w3i;
        d.y *= w3i;
        v[0][q] = cadd(f0, s);
        v[2][q] = make_float2(f1.x + d.y, f1.y - d.x);
        v[1][q] = make_float2(f1.x - d.y, f1.y + d.x);
      }
#pragma unroll
      for (int r = 0; r < 3; r++)
#pragma unroll
        for (int q = 0; q < 4; q++) f[fpos(e0 + 64 * r + 16 * q)] = v[r][q];
    }
  }
  __syncwarp();
  {  // ---------------- pass C: radix-5, m = 192 (kiss_fft.cpp:232-305); ya = tw[192], yb = tw[384] ----------------
    const float2 ya = T.tw[192], yb = T.tw[384];
    for (int u = lane; u < 192; u += 32) {
      float2 z0 = f[fpos(u)];
      float2 z1 = cmul(f[fpos(u + 192)], T.tw5[0][u]);
      float2 z2 = cmul(f[fpos(u + 384)], T.tw5[1][u]);
      float2 z3 = cmul(f[fpos(u + 576)], T.tw5[2][u]);
      float2 z4 = cmul(f[fpos(u + 768)], T.tw5[3][u]);
      float2 s14 = cadd(z1, z4), d14 = csub(z1, z4);
      float2 s23 = cadd(z2, z3), d23 = csub(z2, z3);
      f[fpos(u)] = make_float2(z0.x + (s14.x + s23.x), z0.y + (s14.y + s23.y));
      float2 p = make_float2(z0.x + (s14.x * ya.x + s23.x * yb.x), z0.y + (s14.y * ya.x + s23.y * yb.x));
      float2 q = make_float2(d14.y * ya.y + d23.y * yb.y, -(d14.x * ya.y + d23.x * yb.y));
      f[fpos(u + 192)] = csub(p, q);
      if (kAllOutputs) f[fpos(u + 768)] = cadd(p, q);
      p = make_float2(z0.x + (s14.x * yb.x + s23.x * ya.x), z0.y + (s14.y * yb.x + s23.y * ya.x));
      q = make_float2(d23.y * ya.y - d14.y * yb.y, d14.x * yb.y - d23.x * ya.y);
      if (kAllOutputs || u < 16) f[fpos(u + 384)] = cadd(p, q);
      if (kAllOutputs) f[fpos(u + 576)] = csub(p, q);
    }
  }
  __syncwarp();
}

// ERB band pooling (denoise.cpp:89-123 / 125-160): v[bin] is |X|^2 or Re(X conj P) for bins 0..399.
// Accumulator b receives, in the reference's order, first the frac-weighted bins of band b-1 and then
// the (1-frac)-weighted bins of band b; ends are doubled.
// kDual pools two quantities over the same bands at once (two independent add chains per lane).
template <bool kDual>
__device__ __forceinline__ void band_acc(int b, const float *vf, const float *vo, float *out, const float *vf2,
                                         const float *vo2, float *out2, const short *border) {
  float acc = 0.f, acc2 = 0.f;
  if (b > 0) {
    const int lo = border[b - 1], hi = border[b];
#pragma unroll 4
    for (int k = lo; k < hi; k++) {
      acc = acc + vf[k];
      if (kDual) acc2 = acc2 + vf2[k];
    }
  }
  if (b < kBands - 1) {
    const int lo = border[b], hi = border[b + 1];
#pragma unroll 4
    for (int k = lo; k < hi; k++) {
      acc = acc + vo[k];
      if (kDual) acc2 = acc2 + vo2[k];
    }
  }
  if (b == 0 || b == kBands - 1) { acc *= 2; acc2 *= 2; }
  out[b] = acc;
  if (kDual) out2[b] = acc2;
}
template <bool kDual = false>
__device__ void band_pool_warp(const float *vf, const float *vo, float *out, const short *border, int lane,
                               const float *vf2 = nullptr, const float *vo2 = nullptr, float *out2 = nullptr) {
  // vf[k] = frac[k] * v[k] and vo[k] = (1 - frac[k]) * v[k] were formed by the caller (the very products the
  // reference adds, denoise.cpp:102-103), so the serial part is one load and one add per bin.
  // Accumulators 32 and 33 are the longest chains (96 and 51 adds) and 0 and 1 the shortest (2 and 4): lane j
  // takes accumulator j+2 and lanes 0/1 then add the two short ones, so the critical path is one long chain
  // instead of two.
  static_assert(kBands == 34, "one accumulator per lane plus two short ones on lanes 0 and 1");
  __syncwarp();
  band_acc<kDual>(lane + 2, vf, vo, out, vf2, vo2, out2, border);
  if (lane < 2) band_acc<kDual>(lane, vf, vo, out, vf2, vo2, out2, border);
  __syncwarp();
}

// Sequential dot product s + sum_j a[j] b[j] (ascending j, multiply then add -- the reference's order) with the
// `a` operand fetched four at a time: `a` is the operand that is common to (almost) all lanes, so its 128-bit load
// is a single shared-memory wavefront per four steps.  a must be 16-byte aligned, n a multiple of 4.
__device__ __forceinline__ float seq_dot4(const float *a, const float *b, int n, float s) {
#pragma unroll 2
  for (int j = 0; j < n; j += 4) {
    const float4 av = *reinterpret_cast<const float4 *>(a + j);
    s = s + av.x * b[j];
    s = s + av.y * b[j + 1];
    s = s + av.z * b[j + 2];
    s = s + av.w * b[j + 3];
  }
  return s;
}

// ---- find_best_pitch (pitch.cpp:46-104) with the lags spread over the lanes -------------------------------
// The reference walks the lags in order, keeping the best two by xcorr^2/Syy under a cross-multiplied test whose
// outcome depends on the state left by the earlier lags.  The running energy Syy of every lag does NOT depend on
// that state, so (1) one lane runs the energy recurrence and leaves the energy each lag is tested with in place of
// the deltas, (2) every lane forms its lag's numerator, (3) all lanes test their lag against the current state at
// once; the lowest passing lag is exactly the next lag the sequential walk would have accepted (all lower ones
// fail against the very state they would have met), its update is applied, the higher lags are tested again, and
// so on until none passes.  Same comparisons on the same operands as the reference, a handful of rounds instead
// of one dependent step per lag.
// max(a, b) that returns NaN when a is NaN, like the reference's MAX32(b, a) = (b > a ? b : a) with a constant b:
// one FMNMX instead of a compare and a select
__device__ __forceinline__ float max_nan(float a, float b) {
  float r;
  asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
  return r;
}

struct Best2 {
  float num0, num1, den0, den1;
  int b0, b1;
};
__device__ __forceinline__ Best2 best2_init() { return Best2{-1.f, -1.f, 0.f, 0.f, 0, 1}; }

// in place: d[i] (energy delta of lag i) -> energy lag i is tested with; n4 = number of lags rounded up to 4
__device__ __forceinline__ void energy_chain(float *d, int n4, float syy) {
  for (int i = 0; i < n4; i += 4) {
    const float4 d4 = *reinterpret_cast<const float4 *>(d + i);
    float4 e;
    e.x = syy; syy = max_nan(syy + d4.x, 1.f);
    e.y = syy; syy = max_nan(syy + d4.y, 1.f);
    e.z = syy; syy = max_nan(syy + d4.z, 1.f);
    e.w = syy; syy = max_nan(syy + d4.w, 1.f);
    *reinterpret_cast<float4 *>(d + i) = e;
  }
}

// lanes hold candidates in ascending lag order (lane order)
__device__ __forceinline__ void best2_rounds(Best2 &S, bool alive, float num, float e, int idx, int lane) {
  while (true) {
    const bool pass = alive && (num * S.den1 > S.num1 * e);
    const unsigned m = __ballot_sync(0xffffffffu, pass);
    if (!m) break;
    const int f = __ffs(m) - 1;
    const float nf = __shfl_sync(0xffffffffu, num, f), ef = __shfl_sync(0xffffffffu, e, f);
    const int jf = __shfl_sync(0xffffffffu, idx, f);
    if (nf * S.den0 > S.num0 * ef) {
      S.num1 = S.num0; S.den1 = S.den0; S.b1 = S.b0;
      S.num0 = nf; S.den0 = ef; S.b0 = jf;
    } else {
      S.num1 = nf; S.den1 = ef; S.b1 = jf;
    }
    alive = alive && (lane > f);
  }
}

__device__ __forceinline__ float pitch_gain(float xy, float xx, float yy) {
  return xy / sqrtf(1.f + xx * yy);  // pitch.cpp:417-420 (float sqrt overload)
}

constexpr int kAcHops = 8;  // hops whose pitch_downsample autocorrelations are computed together
struct PitchSmem {
  float lp[kLp];       // decimated, whitened pitch buffer
  float sq[kLp];       // lp[i]^2: the terms of every running energy (find_best_pitch, yy_lookup)
  float yy[392];       // yy_lookup of remove_doubling (385 used); before that the energy deltas of the lag scans
  float cand_xy[32];   // per-candidate cross products of remove_doubling
};
struct WarpSmem {
  union {              // the pitch stage runs strictly between the two transforms of a hop
    float2 fft[kFftLine];  // FFT work line (padded, see fpos)
    PitchSmem p;
  };
  float xc[400];       // xcorr (147 / 294) -- doubles as the per-bin scratch of band pooling (frac-weighted);
                       // the (1-frac)-weighted scratch lives in the tail of the FFT line (bins 0..399 end at slot 447)
  float Ex[kBands], Ep[kBands], Exp[kBands], Ey[kBands];
  float ac_pre[kAcHops * 5];  // autocorrelations of pitch_downsample for a group of hops (see the pre-pass)
};
static_assert(offsetof(WarpSmem, xc) == sizeof(float2) * kFftLine, "the pre-pass treats fft[] + xc[] as one array");
static_assert(kLp + 240 * (kAcHops - 1) + 4 <= 2 * kFftLine + 400, "decimated group does not fit the scratch");

struct BlockSmem {
  FftTw ft;
  float hw[kFrame];
  float frac[kBins];
  float omf[kBins];
  short border[kBands + 2];
  float comb_w[8];
};

// Per-section cycle accounting of the analysis kernel (debug builds only: -DPNB_ANA_TIMING).  Lane 0 of every
// warp samples clock64() at the section boundaries and the deltas are summed into g_ana_cycles.
#ifdef PNB_ANA_TIMING
__device__ unsigned long long g_ana_cycles[16];
#define ANA_TICK(k)                                      \
  do {                                                   \
    long long _now = clock64();                          \
    if (lane == 0) ana_acc[k] += (unsigned long long)(_now - ana_t0); \
    ana_t0 = _now;                                       \
  } while (0)
#else
#define ANA_TICK(k) do { } while (0)
#endif

// ------------------------------------------------------------------------------------------
// The pitch stage of one hop: pitch_downsample (pitch.cpp:148-216) on the 1728-sample pitch buffer `src`,
// pitch_search (pitch.cpp:283-386) and remove_doubling (pitch.cpp:423-527).  `acp` holds the five autocorrelations of
// the decimated signal (celt_lpc.cpp:198-279), computed by the caller.  Shared by the analysis kernel and the
// pitch-only kernel of BASELINE.json config 5.
// ------------------------------------------------------------------------------------------
struct PitchResult {
  int pitch_lag, T;          // lag returned by pitch_search; period after remove_doubling
  float pitch_corr, gain;    // pitch.cpp:385; pitch gain of remove_doubling
};
#ifdef PNB_ANA_TIMING
#define ANA_TIMER_PARAMS , unsigned long long *ana_acc, long long &ana_t0
#define ANA_TIMER_ARGS , ana_acc, ana_t0
#else
#define ANA_TIMER_PARAMS
#define ANA_TIMER_ARGS
#endif
template <bool kInlineAc = false>
__device__ __forceinline__ PitchResult pitch_stage(WarpSmem &W, const float *src, const float *acp, int last_period,
                                                   float last_gain, int lane ANA_TIMER_PARAMS) {
  // ---- pitch_downsample (pitch.cpp:148-216) ----
  {
    for (int i = lane; i < kLp; i += 32) {
      float v;
      if (i == 0) v = .5f * (.5f * src[1] + src[0]);
      else v = .5f * (.5f * (src[2 * i - 1] + src[2 * i + 1]) + src[2 * i]);
      W.p.lp[i] = v;
    }
    __syncwarp();
    ANA_TICK(2);
    // autocorrelation, 5 lags (celt_lpc.cpp:198-279): the analysis kernel computes them for a whole group of hops in
    // its pre-pass; a caller without one (kInlineAc) has lane k run the strictly sequential sum of lag k here
    if (kInlineAc) {
      if (lane < 5) {
        const float *lp = W.p.lp;
        float a = 0.f, d = 0.f;
        for (int j = 0; j < 860; j++) a = a + lp[j] * lp[j + lane];          // fastN = n - lag (celt_lpc.cpp:250-252)
        for (int i = lane + 860; i < kLp; i++) d = d + lp[i] * lp[i - lane];  // the tail, summed apart (:253-256)
        W.ac_pre[lane] = a + d;
      }
      __syncwarp();
      acp = W.ac_pre;
    }
    const float ac0 = acp[0], ac1 = acp[1], ac2 = acp[2], ac3 = acp[3], ac4 = acp[4];
    float fir0 = 0, fir1 = 0, fir2 = 0, fir3 = 0, fir4 = 0;
    ANA_TICK(3);
    if (lane == 0) {
      float a[5] = {ac0, ac1, ac2, ac3, ac4};
      a[0] *= 1.0001f;                                                        // pitch.cpp:190
      for (int i = 1; i <= 4; i++) a[i] -= a[i] * (.008f * i) * (.008f * i);  // :199
      float lpc[4] = {0.f, 0.f, 0.f, 0.f};
      if (a[0] != 0.f) {  // Levinson, celt_lpc.cpp:53-83, the divide in double (:61)
        float err = a[0];
        for (int i = 0; i < 4; i++) {
          float rr = 0.f;
          for (int j = 0; j < i; j++) rr += lpc[j] * a[i - j];
          rr += a[i + 1];
          float r = (float)(-(double)rr / ((double)err + 0.00001));
          lpc[i] = r;
          for (int j = 0; j < (i + 1) >> 1; j++) {
            float t1 = lpc[j], t2 = lpc[i - 1 - j];
            lpc[j] = t1 + r * t2;
            lpc[i - 1 - j] = t2 + r * t1;
          }
          err = err - (r * r) * err;
          if (err < .001f * a[0]) break;
        }
      }
      float tmp = 1.f;
      for (int i = 0; i < 4; i++) { tmp = .9f * tmp; lpc[i] = lpc[i] * tmp; }  // :204-208
      fir0 = lpc[0] + .8f;                                                     // :210-214
      fir1 = lpc[1] + .8f * lpc[0];
      fir2 = lpc[2] + .8f * lpc[1];
      fir3 = lpc[3] + .8f * lpc[2];
      fir4 = .8f * lpc[3];
    }
    fir0 = __shfl_sync(0xffffffffu, fir0, 0);
    fir1 = __shfl_sync(0xffffffffu, fir1, 0);
    fir2 = __shfl_sync(0xffffffffu, fir2, 0);
    fir3 = __shfl_sync(0xffffffffu, fir3, 0);
    fir4 = __shfl_sync(0xffffffffu, fir4, 0);
    ANA_TICK(4);
    // 5-tap FIR in place with zero history (pitch.cpp:106-145,154), walked from the end so the taps
    // still see unfiltered samples
    static_assert(kLp % 32 == 0, "the FIR walk covers [0, kLp) in whole warps");
    for (int base = kLp - 32; base >= 0; base -= 32) {
      int i = base + lane;
      float x0 = W.p.lp[i];
      float m0 = i >= 1 ? W.p.lp[i - 1] : 0.f, m1 = i >= 2 ? W.p.lp[i - 2] : 0.f, m2 = i >= 3 ? W.p.lp[i - 3] : 0.f,
            m3 = i >= 4 ? W.p.lp[i - 4] : 0.f, m4 = i >= 5 ? W.p.lp[i - 5] : 0.f;
      float sum = x0;
      sum = sum + fir0 * m0;
      sum = sum + fir1 * m1;
      sum = sum + fir2 * m2;
      sum = sum + fir3 * m3;
      sum = sum + fir4 * m4;
      __syncwarp();
      W.p.lp[i] = sum;
      W.p.sq[i] = sum * sum;
      __syncwarp();
    }
  }

  ANA_TICK(5);
  // ---- pitch_search (pitch.cpp:283-386): x = lp+384, y = lp, len 960, max_pitch 588 ----
  int pitch_lag, T;
  float pitch_corr, gain;
  {
    int b0, b1;
    // coarse: the 4x-decimated signals are stride-2 views of lp.  A lag lane owns kLagsPerLane adjacent lags and
    // slides a window of y along, so each step costs one new y load; every lag still accumulates in ascending
    // j exactly like the reference (pitch.cpp:218-281).  The lane after the lag lanes accumulates the energy
    // Syy = 1 + sum y4[j]^2 of find_best_pitch (pitch.cpp:54,69-70) through the same code shape (lag 0 of y on y).
    {
      constexpr int NL = 5;          // adjacent lags per lag lane
      constexpr int kLagLanes = 30;  // lanes that own lags
      static_assert(kLagLanes * NL >= 147, "the lag lanes cover every coarse lag");
      static_assert(kLagLanes < 32, "the lane after the lag lanes accumulates Syy");
      const bool syy_lane = (lane == kLagLanes);
      const float *xb = syy_lane ? W.p.lp : W.p.lp + 384;
      const int L0 = (lane < kLagLanes) ? NL * lane : 0;
      const float *yb = W.p.lp + 2 * L0;
      float acc[NL], w[NL];
#pragma unroll
      for (int q = 0; q < NL; q++) { acc[q] = 0.f; w[q] = yb[2 * q]; }
      if (syy_lane) acc[0] = 1.f;
      for (int j = 0; j < 240; j += NL) {
#pragma unroll
        for (int u = 0; u < NL; u++) {
          const float xj = xb[2 * (j + u)];
#pragma unroll
          for (int q = 0; q < NL; q++) acc[q] = acc[q] + xj * w[(u + q) % NL];
          w[u] = yb[2 * (j + u + NL)];
        }
      }
      if (lane < kLagLanes) {
#pragma unroll
        for (int q = 0; q < NL; q++)
          if (L0 + q < 147) W.xc[L0 + q] = acc[q];
      }
      // energy deltas of the coarse scan: y4[i+240]^2 - y4[i]^2 (pitch.cpp:101)
      for (int i = lane; i < 147; i += 32) {
        W.p.yy[i] = W.p.sq[2 * (i + 240)] - W.p.sq[2 * i];
      }
      float syy_c = __shfl_sync(0xffffffffu, acc[0], kLagLanes);
      __syncwarp();
      ANA_TICK(6);
      if (lane == 0) energy_chain(W.p.yy, 148, syy_c);
      __syncwarp();
      {
        Best2 S = best2_init();
        for (int base = 0; base < 147; base += 32) {
          const int i = base + lane;
          const bool valid = i < 147;
          const float xv = valid ? W.xc[i] : 0.f, ev = valid ? W.p.yy[i] : 1.f;
          const float c = xv * 1e-12f;
          best2_rounds(S, valid && xv > 0.f, c * c, ev, i, lane);
        }
        b0 = S.b0; b1 = S.b1;
      }
      __syncwarp();
      ANA_TICK(7);
    }
    // fine: at most ten lags around 2*b0 and 2*b1 (pitch.cpp:344-361); lane 10 accumulates Syy of the
    // second find_best_pitch, lane 11 the xx of remove_doubling (pitch.cpp:448)
    for (int i = lane; i < 294; i += 32) {
      W.xc[i] = 0.f;
      W.p.yy[i] = W.p.sq[i + 480] - W.p.sq[i];  // energy deltas of the fine scan
    }
    __syncwarp();
    int fl = -1;
    if (lane < 5) fl = 2 * b0 - 2 + lane;
    else if (lane < 10) fl = 2 * b1 - 2 + (lane - 5);
    const bool fine_ok = (fl >= 0 && fl < 294);
    float sacc = (lane == 10) ? 1.f : 0.f;
    {
      const float *a, *b;
      int n = 480;
      if (lane < 10) { a = W.p.lp + 384; b = W.p.lp + (fine_ok ? fl : 0); if (!fine_ok) n = 0; }
      else if (lane == 10) { a = W.p.lp; b = W.p.lp; }
      else if (lane == 11) { a = W.p.lp + 384; b = W.p.lp + 384; }
      else { a = W.p.lp; b = W.p.lp; n = 0; }
      if (n) sacc = seq_dot4(a, b, 480, sacc);
    }
    if (fine_ok) W.xc[fl] = (-1.f > sacc) ? -1.f : sacc;
    float syy_f = __shfl_sync(0xffffffffu, sacc, 10);
    float xx = __shfl_sync(0xffffffffu, sacc, 11);
    __syncwarp();
    ANA_TICK(8);
    int off = 0;
    float corr = 0.f;
    pitch_lag = 0;
    // second find_best_pitch (pitch.cpp:362): xcorr is zero outside the two windows and zero entries are never
    // candidates (pitch.cpp:73), so only the (at most ten) window lags are tested; the energy recurrence still
    // runs from lag 0 up to the end of the later window
    int c0;
    {
      const int w0 = 2 * b0 - 2, w1 = 2 * b1 - 2;
      const int lo_a = w0 < w1 ? w0 : w1, lo_b = w0 < w1 ? w1 : w0;
      int loA = lo_a < 0 ? 0 : lo_a;
      loA = loA > 294 ? 294 : loA;
      int hiA = lo_a + 5;
      hiA = hiA < loA ? loA : hiA;
      hiA = hiA > 294 ? 294 : hiA;
      int loB = lo_b < hiA ? hiA : lo_b;
      loB = loB > 294 ? 294 : loB;
      int hiB = lo_b + 5;
      hiB = hiB < loB ? loB : hiB;
      hiB = hiB > 294 ? 294 : hiB;
      if (lane == 0) energy_chain(W.p.yy, (hiB + 3) & ~3, syy_f);
      __syncwarp();
      const int idx = lane < 5 ? loA + lane : loB + (lane - 5);
      const bool valid = lane < 5 ? idx < hiA : (lane < 10 && idx < hiB);
      const float xv = valid ? W.xc[idx] : 0.f, ev = valid ? W.p.yy[idx] : 1.f;
      const float c = xv * 1e-12f;
      Best2 S = best2_init();
      best2_rounds(S, valid && xv > 0.f, c * c, ev, idx, lane);
      c0 = S.b0;
    }
    if (lane == 0) {
      if (c0 > 0 && c0 < 293) {
        float a = W.xc[c0 - 1], b = W.xc[c0], cc = W.xc[c0 + 1];
        if ((cc - a) > .7f * (b - a)) off = 1;
        else if ((a - cc) > .7f * (b - cc)) off = -1;
      }
      pitch_lag = 2 * c0 - off;
      corr = W.xc[c0];
    }
    pitch_lag = __shfl_sync(0xffffffffu, pitch_lag, 0);
    pitch_corr = __shfl_sync(0xffffffffu, corr, 0);
    __syncwarp();  // the scan's energy deltas in W.p.yy are dead; the yy table is built next
    ANA_TICK(9);

    // ---- remove_doubling (pitch.cpp:423-527) with maxperiod 384, minperiod 30, N 480 ----
    const int second_check[16] = {0, 0, 3, 2, 3, 2, 5, 2, 3, 2, 3, 2, 5, 2, 3, 2};
    const float *x = W.p.lp + 384;
    int T0 = (kMaxPeriod - pitch_lag) / 2;
    if (T0 >= 384) T0 = 383;
    const int prev_period = last_period / 2;
    // 32 roles: 0: xy at T0; 1: the yy_lookup recurrence; 2..29: candidate (k, which) = (2 + (role-2)/2, (role-2)&1);
    // 30, 31: xy at T0-1 and T0+1, the neighbours the final refinement needs when no sub-harmonic replaces T0
    // (the usual outcome) -- they ride along in lanes that would idle, and the extra pass below is skipped
    {
      const int role = lane;
      int lag = -1;
      if (role == 0) lag = T0;
      else if (role == 30) lag = T0 - 1;
      else if (role == 31) lag = T0 + 1;
      else if (role >= 2 && role < 30) {
        int k = 2 + ((role - 2) >> 1);
        int T1 = (2 * T0 + k) / (2 * k);
        if (T1 >= 30) {
          if ((role & 1) == 0) lag = T1;
          else if (k == 2) lag = (T1 + T0 > 384) ? T0 : T0 + T1;
          else lag = (2 * second_check[k] * T0 + k) / (2 * k);
        }
      }
      // all lanes meet here before the 480-step loops: without it the lanes whose lag needed no division run the
      // dot loop ahead of the candidate lanes and the loop is executed once per diverged set of lanes
      __syncwarp();
      // the energy table is read only at the lags of roles 0 and 2..29 (T0, T1, T1b): the recurrence stops there
      const int max_lag = __reduce_max_sync(0xffffffffu, role < 30 ? lag : -1);
      if (role == 1) {
        // yy_lookup recurrence (pitch.cpp:449-455), strictly sequential; operands fetched four at a time.
        // Table entry i is stored at W.p.yy[i + 3] so that groups of four are 16-byte aligned.
        float yy = xx;
        W.p.yy[3] = xx;
        for (int i = 1; i <= max_lag; i += 4) {
          const float4 a = *reinterpret_cast<const float4 *>(W.p.sq + 384 - i - 3);  // x[-i-3 .. -i]^2
          const float4 b = *reinterpret_cast<const float4 *>(W.p.sq + 864 - i - 3);  // x[480-i-3 .. 480-i]^2
          float4 o;
          yy = yy + a.w - b.w; o.x = max_nan(yy, 0.f);
          yy = yy + a.z - b.z; o.y = max_nan(yy, 0.f);
          yy = yy + a.y - b.y; o.z = max_nan(yy, 0.f);
          yy = yy + a.x - b.x; o.w = max_nan(yy, 0.f);
          *reinterpret_cast<float4 *>(&W.p.yy[i + 3]) = o;
        }
      } else {
        float d = 0.f;
        if (lag >= 0) d = seq_dot4(x, x - lag, 480, 0.f);
        W.p.cand_xy[role] = d;
      }
    }
    __syncwarp();
    ANA_TICK(10);
    int Tsel = T0;
    float g = 0.f, best_xy = 0.f, best_yy = 0.f;
    if (lane == 0) {
      float xy = W.p.cand_xy[0];
      float yy = W.p.yy[T0 + 3];
      best_xy = xy;
      best_yy = yy;
      float g0 = pitch_gain(xy, xx, yy);
      g = g0;
      for (int k = 2; k <= 15; k++) {
        int T1 = (2 * T0 + k) / (2 * k);
        if (T1 < 30) break;
        int T1b;
        if (k == 2) T1b = (T1 + T0 > 384) ? T0 : T0 + T1;
        else T1b = (2 * second_check[k] * T0 + k) / (2 * k);
        float xy1 = W.p.cand_xy[2 + 2 * (k - 2)], xy2 = W.p.cand_xy[3 + 2 * (k - 2)];
        xy = .5f * (xy1 + xy2);
        yy = .5f * (W.p.yy[T1 + 3] + W.p.yy[T1b + 3]);
        float g1 = pitch_gain(xy, xx, yy);
        float cont;
        int dT = T1 - prev_period;
        dT = dT < 0 ? -dT : dT;
        if (dT <= 1) cont = last_gain;
        else if (dT <= 2 && 5 * k * k < T0) cont = .5f * last_gain;
        else cont = 0.f;
        float th = .7f * g0 - cont;
        float thresh = .3f > th ? .3f : th;
        if (T1 < 90) {
          th = .85f * g0 - cont;
          thresh = .4f > th ? .4f : th;
        }  // the T1 < 2*minperiod branch of the reference is unreachable (SURVEY.md App. C.9)
        if (g1 > thresh) { best_xy = xy; best_yy = yy; Tsel = T1; g = g1; }
      }
    }
    Tsel = __shfl_sync(0xffffffffu, Tsel, 0);
    ANA_TICK(11);
    // final +-1 refinement: three dot products around the selected period (pitch.cpp:512-513)
    {
      float x0, x1, x2;
      if (Tsel == T0) {  // warp-uniform
        x0 = W.p.cand_xy[30]; x1 = W.p.cand_xy[0]; x2 = W.p.cand_xy[31];
      } else {
        float d = 0.f;
        if (lane < 3) d = seq_dot4(x, x - (Tsel + lane - 1), 480, 0.f);
        x0 = __shfl_sync(0xffffffffu, d, 0); x1 = __shfl_sync(0xffffffffu, d, 1); x2 = __shfl_sync(0xffffffffu, d, 2);
      }
      int Tout = 0;
      float pg = 0.f;
      if (lane == 0) {
        best_xy = 0.f > best_xy ? 0.f : best_xy;
        if (best_yy <= best_xy) pg = 1.f;
        else pg = best_xy / (best_yy + 1.f);
        int o2;
        if ((x2 - x0) > .7f * (x1 - x0)) o2 = 1;
        else if ((x0 - x2) > .7f * (x1 - x2)) o2 = -1;
        else o2 = 0;
        if (pg > g) pg = g;
        Tout = 2 * Tsel + o2;
        if (Tout < kMinPeriod) Tout = kMinPeriod;
      }
      T = __shfl_sync(0xffffffffu, Tout, 0);
      gain = __shfl_sync(0xffffffffu, pg, 0);
    }
    ANA_TICK(12);
  }
  PitchResult res;
  res.pitch_lag = pitch_lag; res.T = T; res.pitch_corr = pitch_corr; res.gain = gain;
  return res;
}

constexpr int kAnaWarps = 8;  // one stream per warp

__global__ void __launch_bounds__(kAnaWarps * 32) analysis_kernel(AnalysisArgs A) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  BlockSmem &B = *reinterpret_cast<BlockSmem *>(smem_raw);
  WarpSmem *Wall = reinterpret_cast<WarpSmem *>(smem_raw + ((sizeof(BlockSmem) + 15) / 16) * 16);
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const Tables *T = A.tab;
  for (int i = threadIdx.x; i < kWin; i += blockDim.x) B.ft.tw[i] = T->tw[i];
  for (int i = threadIdx.x; i < 4 * 192; i += blockDim.x) B.ft.tw5[i / 192][i % 192] = T->tw[(i / 192 + 1) * (i % 192)];
  for (int i = threadIdx.x; i < kFrame; i += blockDim.x) B.hw[i] = T->half_window[i];
  for (int i = threadIdx.x; i < kBins; i += blockDim.x) { B.frac[i] = T->frac[i]; B.omf[i] = T->omf[i]; }
  if (threadIdx.x < kBands + 2) B.border[threadIdx.x] = T->border[threadIdx.x];
  if (threadIdx.x < 8) B.comb_w[threadIdx.x] = T->comb_w[threadIdx.x];
  __syncthreads();

  const int s = blockIdx.x * kAnaWarps + wib;
  if (s >= A.n_streams) return;
  WarpSmem &W = Wall[wib];
  float *xo = reinterpret_cast<float *>(&W.fft[448]);
  const float *row = A.pcm + (size_t)s * A.pcm_stride;
  int last_period = A.last_period[s];
  float last_gain = A.last_gain[s];
  // a ragged call's slot walks its own hops: the trip count is uniform across the warp because the warp owns one
  // stream, so every full-warp barrier and shuffle in the hop loop is reached by all 32 lanes
  const int n_frames = A.hops ? A.hops[s] : A.n_frames;

#ifdef PNB_ANA_TIMING
  unsigned long long ana_acc[16];
  for (int i = 0; i < 16; i++) ana_acc[i] = 0;
  long long ana_t0 = clock64();
#endif
  for (int t = 0; t < n_frames; t++) {
    const float *line = row + (size_t)t * kFrame;  // line[j] == reference comb_buf[j] at this hop
    const size_t fs = (size_t)t * A.stride + s;

    // ---- pre-pass, once per group of kAcHops hops: the five autocorrelations pitch_downsample needs
    // (pitch.cpp:182 -> celt_lpc.cpp:198-279).  Inside a hop only five lanes can work on them (one strictly
    // sequential 864-term sum per lag); but the 2:1 decimated signal of hop t+1 is that of hop t advanced by 240
    // samples (only element 0 of each hop's buffer has its own formula, pitch.cpp:165), so the decimated signal
    // of the whole group is laid out once in the scratch line and ONE LANE PER HOP runs the five sums of its hop,
    // sharing every loaded sample between the lags.  Same products, same order of additions as the reference.
    if (t % kAcHops == 0) {
      const int G = (n_frames - t < kAcHops) ? n_frames - t : kAcHops;
      float *D = reinterpret_cast<float *>(W.fft);
      const float *src = line + kOffPitch;
      const int nD = kLp + 240 * (G - 1);
      for (int i = lane; i < nD; i += 32) D[i] = .5f * (.5f * (src[2 * i - 1] + src[2 * i + 1]) + src[2 * i]);
      __syncwarp();
      if (lane < G) {
        const float *Dh = D + 240 * lane, *sh = src + kFrame * lane;
        float4 c = *reinterpret_cast<const float4 *>(Dh), n = *reinterpret_cast<const float4 *>(Dh + 4);
        c.x = .5f * (.5f * sh[1] + sh[0]);  // lp[0] of this hop (pitch.cpp:165)
        float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f, a4 = 0.f;
#define PNB_AC_STEP(X, P1, P2, P3, P4) \
  a0 = a0 + (X) * (X); a1 = a1 + (X) * (P1); a2 = a2 + (X) * (P2); a3 = a3 + (X) * (P3); a4 = a4 + (X) * (P4)
#pragma unroll 1
        for (int m = 0; m < 215; m++) {  // j = 4m .. 4m+3 < 860 (celt_lpc.cpp:250-252: fastN = n - lag)
          PNB_AC_STEP(c.x, c.y, c.z, c.w, n.x);
          PNB_AC_STEP(c.y, c.z, c.w, n.x, n.y);
          PNB_AC_STEP(c.z, c.w, n.x, n.y, n.z);
          PNB_AC_STEP(c.w, n.x, n.y, n.z, n.w);
          c = n;
          if (m < 214) n = *reinterpret_cast<const float4 *>(Dh + 4 * (m + 2));  // up to lp[860..863]
        }
#undef PNB_AC_STEP
        // the tail i = k+860 .. 863 is summed on its own and then added (celt_lpc.cpp:253-256); c = lp[860..863]
        float d0 = 0.f, d1 = 0.f, d2 = 0.f, d3 = 0.f;
        d0 = d0 + c.x * c.x; d0 = d0 + c.y * c.y; d0 = d0 + c.z * c.z; d0 = d0 + c.w * c.w;
        d1 = d1 + c.y * c.x; d1 = d1 + c.z * c.y; d1 = d1 + c.w * c.z;
        d2 = d2 + c.z * c.x; d2 = d2 + c.w * c.y;
        d3 = d3 + c.w * c.x;
        float *o = W.ac_pre + 5 * lane;
        o[0] = a0 + d0; o[1] = a1 + d1; o[2] = a2 + d2; o[3] = a3 + d3; o[4] = a4 + 0.f;
      }
      __syncwarp();
    }

    // ---- one transform per hop.  The look-ahead window of hop c (denoise.cpp:498-506: the newest 960
    // samples) is the very block whose spectrum is the analysis spectrum X five hops later (:402, :333-346:
    // line[2400..3360) at hop c+5 == line[4800..5760) at hop c), so each windowed block is transformed once,
    // kept in a per-stream ring of spectra / band energies, and read back as X and Ex when it comes due.
    const long c = A.hop0 + t;
    const int slot_new = (int)(c % A.ring), slot_x = (int)(((c - 5) % A.ring + A.ring) % A.ring);
    {
      const float *src = line + kOffLook;
      const float *hw = B.hw;
      // window (denoise.cpp:282-289), real -> complex, 1/960 (kiss_fft.cpp:582-583)
      fft960_warp<false>(W.fft, B.ft, lane, [&](int i) {
        float w = hw[i < kFrame ? i : kWin - 1 - i];
        float v = src[i] * w;
        return make_float2((1.f / kWin) * v, 0.f);
      });
    }
    ANA_TICK(0);
    {
      float2 *Zg = A.zring + ((size_t)slot_new * A.stride + s) * kBins;
      for (int k = lane; k < kBins; k += 32) {
        float2 x = W.fft[fpos(k)];
        Zg[k] = x;
        float e = x.x * x.x;
        e += x.y * x.y;
        W.xc[k] = B.frac[k] * e;
        xo[k] = B.omf[k] * e;
      }
      band_pool_warp(W.xc, xo, W.Ey, B.border, lane);
      float *Eg = A.ering + ((size_t)slot_new * A.stride + s) * kBands;
      const float *Eo = A.ering + ((size_t)slot_x * A.stride + s) * kBands;
      for (int b = lane; b < kBands; b += 32) {
        Eg[b] = W.Ey[b];
        W.Ex[b] = Eo[b];  // written five hops ago (by this lane, or by the previous call)
      }
    }
    const float2 *Xg = A.zring + ((size_t)slot_x * A.stride + s) * kBins;
    __syncwarp();
    ANA_TICK(1);

    // ---- pitch_downsample, pitch_search, remove_doubling (pitch.cpp:148-216, 283-386, 423-527) ----
    const PitchResult pr =
        pitch_stage(W, line + kOffPitch, W.ac_pre + 5 * (t % kAcHops), last_period, last_gain, lane ANA_TIMER_ARGS);
    const int pitch_lag = pr.pitch_lag, T = pr.T;
    const float pitch_corr = pr.pitch_corr, gain = pr.gain;
    last_period = T;
    last_gain = gain;

    // ---- comb-filtered block, its spectrum P and the band statistics (denoise.cpp:416-427) ----
    __syncwarp();  // the pitch scratch is dead from here on; its storage becomes the FFT line again
    {
      const float *hw = B.hw;
      const float *cw = B.comb_w;
      const float *ctr = line + kOffAnalysis;
      fft960_warp<false>(W.fft, B.ft, lane, [&](int i) {
        float p = 0.f;
#pragma unroll
        for (int k = -3; k <= 3; k++) p = p + ctr[i - T * k] * cw[k + 3];
        float w = hw[i < kFrame ? i : kWin - 1 - i];
        float v = p * w;
        return make_float2((1.f / kWin) * v, 0.f);
      });
      ANA_TICK(13);
      float2 *Pg = A.P && s < A.P_rows ? A.P + fs * kBins : nullptr;
      for (int k = lane; k < kBins; k += 32) {
        float2 p = W.fft[fpos(k)], x = Xg[k];
        if (Pg) Pg[k] = p;
        float e = p.x * p.x;
        e += p.y * p.y;
        const float fr = B.frac[k], om = B.omf[k];
        W.xc[k] = fr * e;
        xo[k] = om * e;
        float c = x.x * p.x;
        c += x.y * p.y;
        xo[kBins + k] = fr * c;       // the line's tail (fft[448..1080)) holds three 400-float arrays
        xo[2 * kBins + k] = om * c;
      }
      band_pool_warp<true>(W.xc, xo, W.Ep, B.border, lane, xo + kBins, xo + 2 * kBins, W.Exp);
    }

    ANA_TICK(14);
    // ---- features (denoise.cpp:427-433, 487-496, 528-530) ----
    {
      float *F = A.feat + fs * kFeat;
      for (int b = lane; b < kBands; b += 32) {
        float prod = W.Ex[b] * W.Ep[b];                       // float product, then double (H4)
        double v = (double)W.Exp[b] / sqrt(1e-15 + (double)prod);
        v = fmax(0.0, v);
        float coh = (float)fmin(1.0, v);
        F[b] = W.Ey[b] * 30.f;
        F[kBands + b] = coh * 30.f;
        if (A.raw) {
          A.raw[fs * 68 + b] = W.Ey[b];
          A.raw[fs * 68 + kBands + b] = coh;
        }
      }
      if (lane == 0) {
        float E = 0.f;
        for (int b = 0; b < kBands; b++) E += W.Ex[b];
        int silence = ((double)E < 0.1) ? 1 : 0;
        A.silence[fs] = (unsigned char)silence;
        F[68] = (float)T / 588.f;
        F[69] = pitch_corr;
        if (A.tap_pitch) {
          int *tp = A.tap_pitch + fs * 4;
          tp[0] = pitch_lag; tp[1] = T; tp[2] = silence; tp[3] = 0;
          A.tap_pitchf[fs * 2] = pitch_corr;
          A.tap_pitchf[fs * 2 + 1] = gain;
        }
      }
      if (A.Ex) for (int b = lane; b < kBands; b += 32) A.Ex[fs * kBands + b] = W.Ex[b];
    }
    __syncwarp();
    ANA_TICK(15);
  }
#ifdef PNB_ANA_TIMING
  if (lane == 0)
    for (int i = 0; i < 16; i++) atomicAdd(&g_ana_cycles[i], ana_acc[i]);
#endif
  if (lane == 0) {
    A.last_period[s] = last_period;
    A.last_gain[s] = last_gain;
  }
}

// ------------------------------------------------------------------------------------------
// synthesis: per-bin gains from band values, optional comb mix, inverse transform, overlap-add
// ------------------------------------------------------------------------------------------
struct SynWarpSmem {
  float2 fft[kFftLine];
  float g[kBands], r[kBands], ir[kBands], gw[kBands];
};
struct SynBlockSmem {
  FftTw ft;
  float hw[kFrame];
  float frac[kBins];
  float omf[kBins];
  short band_of[kBins];
};
constexpr int kSynWarps = 4;

// kClamp: the int16 conversion of A.clamp16, one instantiation per mode so that each keeps its own code
template <bool kClamp>
__global__ void __launch_bounds__(kSynWarps * 32) synthesis_kernel(SynthesisArgs A) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  SynBlockSmem &B = *reinterpret_cast<SynBlockSmem *>(smem_raw);
  SynWarpSmem *Wall = reinterpret_cast<SynWarpSmem *>(smem_raw + ((sizeof(SynBlockSmem) + 15) / 16) * 16);
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const Tables *T = A.tab;
  for (int i = threadIdx.x; i < kWin; i += blockDim.x) B.ft.tw[i] = T->tw[i];
  for (int i = threadIdx.x; i < 4 * 192; i += blockDim.x) B.ft.tw5[i / 192][i % 192] = T->tw[(i / 192 + 1) * (i % 192)];
  for (int i = threadIdx.x; i < kFrame; i += blockDim.x) B.hw[i] = T->half_window[i];
  for (int i = threadIdx.x; i < kBins; i += blockDim.x) {
    B.frac[i] = T->frac[i];
    B.omf[i] = T->omf[i];
    B.band_of[i] = T->band_of[i];
  }
  __syncthreads();
  const int s = blockIdx.x * kSynWarps + wib;
  if (s >= A.n_streams) return;
  SynWarpSmem &W = Wall[wib];
  const int orow = A.row ? A.row[s] : s;  // output row of slot s

  float mem[15];  // overlap-add memory: samples lane + 32 i  (denoise.cpp:75,357-358)
#pragma unroll
  for (int i = 0; i < 15; i++) mem[i] = A.synth_mem[(size_t)s * kFrame + lane + 32 * i];

  const int n_frames = A.hops ? A.hops[s] : A.n_frames;  // a ragged call's slot: its own hops, zeros after them
  for (int t = 0; t < n_frames; t++) {
    const size_t fs = (size_t)t * A.stride + s;
    const float *gr = A.gr + fs * 68;
    for (int b = lane; b < kBands; b += 32) {
      float g = gr[b], r = gr[kBands + b];
      W.g[b] = g;
      W.r[b] = r;
      W.ir[b] = 1.f - r;
    }
    __syncwarp();
    if (A.postfilter) {  // denoise.cpp:216-250 applied to g (envelope post-filter, beta = 0.02)
      const float *Ey = A.Ex + fs * kBands;
      // sinf of the reference's libm is correctly rounded in all but rare cases; so is the rounded double sine
      for (int b = lane; b < kBands; b += 32) W.gw[b] = W.g[b] * (float)sin((double)(float)(M_PI / 2 * (double)W.g[b]));
      __syncwarp();
      float G = 0.f;
      if (lane == 0) {
        float e0 = 0.f, e1 = 0.f;
        for (int b = 0; b < kBands; b++) e0 += W.g[b] * Ey[b];
        for (int b = 0; b < kBands; b++) e1 += W.gw[b] * Ey[b];
        float q = e0 / (e1 + 1e-6f);
        G = sqrtf(((1.f + 0.02f) * q) / (1.f + 0.02f * (q * q)));
      }
      G = __shfl_sync(0xffffffffu, G, 0);
      __syncwarp();  // lane 0's reads of g are ordered before the overwrite (the shuffle alone is not a memory fence)
      for (int b = lane; b < kBands; b += 32) W.g[b] = G * W.gw[b];
      __syncwarp();
    }
    if (A.tap_g)
      for (int b = lane; b < kBands; b += 32) A.tap_g[fs * kBands + b] = W.g[b];
    const bool silence = A.silence[fs] != 0;
    const long c = A.hop0 + t;
    const int slot_x = (int)(((c - 5) % A.ring + A.ring) % A.ring);
    const float2 *Xg = A.zring + ((size_t)slot_x * A.stride + s) * kBins, *Pg = A.P + fs * kBins;
    // bins 0..399 and their mirror images; everything from 400 to 560 is zero (SURVEY.md App. C.1)
    {
      const float *frac = B.frac, *omf = B.omf;
      const short *band_of = B.band_of;
      const float *gg = W.g, *rr = W.r, *ir = W.ir;
      fft960_warp<true>(W.fft, B.ft, lane, [&](int i) {
        int k = i <= kFrame ? i : kWin - i;
        float2 v = make_float2(0.f, 0.f);
        if (k < kBins) {
          float2 x = Xg[k];
          int b = band_of[k];
          float fr = frac[k], om = omf[k];
          if (!silence) {  // pitch_filter, denoise.cpp:436-485
            float rf = om * ir[b] + fr * ir[b + 1];
            x.x = rf * x.x;
            x.y = rf * x.y;
            rf = om * rr[b] + fr * rr[b + 1];
            float2 p = Pg[k];
            x.x += rf * p.x;
            x.y += rf * p.y;
          }
          float gf = om * gg[b] + fr * gg[b + 1];  // interp_band_gain + gain apply, :539-544
          x.x *= gf;
          x.y *= gf;
          v = (i <= kFrame) ? x : make_float2(x.x, -x.y);  // Hermitian extension, :314-317
        }
        return make_float2((1.f / kWin) * v.x, (1.f / kWin) * v.y);
      });
    }
    // time samples are read back reversed and rescaled (denoise.cpp:318-323), windowed, overlap-added
    float *outp = A.out ? A.out + (size_t)orow * A.out_stride + (size_t)t * kFrame : nullptr;
    short *outs = A.out16 ? A.out16 + (size_t)orow * A.out_stride + (size_t)t * kFrame : nullptr;
#pragma unroll
    for (int i = 0; i < 15; i++) {
      int n = lane + 32 * i;
      float a = (float)kWin * W.fft[fpos((kWin - n) % kWin)].x;
      a = a * B.hw[n];
      float o = a + mem[i];
      if (outp) outp[n] = o;
      if (outs) {
        if (kClamp) outs[n] = (short)fmaxf(-32768.f, fminf(32767.f, o));  // denoise.cpp:756-758: NaN -> 32767
        else outs[n] = (short)(int)(o * 32768.f);                          // main.cpp:36: truncation toward zero
      }
      int n2 = n + kFrame;
      float c = (float)kWin * W.fft[fpos(kWin - n2)].x;
      mem[i] = c * B.hw[kWin - 1 - n2];
    }
    __syncwarp();
  }
  for (int t = n_frames; t < A.n_frames; t++) {
    float *outp = A.out ? A.out + (size_t)orow * A.out_stride + (size_t)t * kFrame : nullptr;
    short *outs = A.out16 ? A.out16 + (size_t)orow * A.out_stride + (size_t)t * kFrame : nullptr;
    for (int n = lane; n < kFrame; n += 32) {
      if (outp) outp[n] = 0.f;
      if (outs) outs[n] = 0;
    }
  }
#pragma unroll
  for (int i = 0; i < 15; i++) A.synth_mem[(size_t)s * kFrame + lane + 32 * i] = mem[i];
}

// ------------------------------------------------------------------------------------------
// the synthesis's gradient with respect to g/r (include/pnb_synth_grad.h), one warp per (row, hop).  Hop t's output
// is out[t][n] = x_t[n] hw[n] + x_{t-1}[480 + n] hw[479 - n], with x_t = Re(sum_i Y'_i e^{2 pi i i n / 960}) the
// inverse transform of the Hermitian extension Y' of the gained spectrum Y (synthesis_kernel).  So, per hop:
//   dx[n] = dout[t][n] hw[n],  dx[480 + m] = dout[t+1][m] hw[479 - m] (0 for the call's last hop: that half goes to
//           the overlap-add memory of the next call)
//   dY_k  = c_k sum_n dx[n] e^{-2 pi i k n / 960}, c_0 = 1, c_k = 2 (bins k and 960 - k fold onto k): one forward
//           transform of the real vector dx
//   Y_k = gf_k Z_k, Z_k = rfx_k X_k + rfp_k P_k (X_k on a silent hop), with gf, rfx, rfp interpolated from the band
//           values g_used, 1 - r, r as interp_band_gain does:
//           dgf_k = Re(conj(dY_k) Z_k),  d(rfp_k) - d(rfx_k) = gf_k Re(conj(dY_k) (P_k - X_k)) =: drf_k
//   band b takes omf_k times the bins of band b and frac_k times the bins of band b - 1
//   post-filter: g_used_b = G gw_b, gw_b = g_b sin(pi g_b / 2), G = sqrt((1 + beta) q / (1 + beta q^2)),
//           q = e0 / (e1 + 1e-6), e0 = sum g_j Ey_j, e1 = sum gw_j Ey_j:
//           dg_b = dgu_b G gw'_b + (sum_j dgu_j gw_j) dG/dq Ey_b (1 - q gw'_b) / (e1 + 1e-6)
//           G = 0 (every g zero): g_used vanishes to second order, and dg is 0.
// ------------------------------------------------------------------------------------------
struct __align__(16) SynGradWarpSmem {  // 16-byte aligned: fft960_warp's first pass stores float4
  float2 fft[kFftLine];  // the transform of dx; then the per-bin products, four arrays of kBins floats
  float g[kBands], r[kBands], ir[kBands], gw[kBands], gu[kBands], dgu[kBands], dr[kBands];
};
struct SynGradBlockSmem {
  FftTw ft;
  float hw[kFrame];
  float frac[kBins];
  float omf[kBins];
  short band_of[kBins];
  short border[kBands + 2];
};
constexpr int kSgWarps = 8;
static_assert(4 * kBins <= 2 * kFftLine, "the per-bin products do not fit the transform's line");
static_assert(sizeof(SynGradWarpSmem) % 16 == 0, "every warp's transform line must start 16-byte aligned");

__global__ void __launch_bounds__(kSgWarps * 32) synthesis_backward_kernel(SynthGradArgs A) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  SynGradBlockSmem &B = *reinterpret_cast<SynGradBlockSmem *>(smem_raw);
  SynGradWarpSmem *Wall = reinterpret_cast<SynGradWarpSmem *>(smem_raw + ((sizeof(SynGradBlockSmem) + 15) / 16) * 16);
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const Tables *T = A.tab;
  for (int i = threadIdx.x; i < kWin; i += blockDim.x) B.ft.tw[i] = T->tw[i];
  for (int i = threadIdx.x; i < 4 * 192; i += blockDim.x) B.ft.tw5[i / 192][i % 192] = T->tw[(i / 192 + 1) * (i % 192)];
  for (int i = threadIdx.x; i < kFrame; i += blockDim.x) B.hw[i] = T->half_window[i];
  for (int i = threadIdx.x; i < kBins; i += blockDim.x) {
    B.frac[i] = T->frac[i];
    B.omf[i] = T->omf[i];
    B.band_of[i] = T->band_of[i];
  }
  for (int i = threadIdx.x; i < kBands + 2; i += blockDim.x) B.border[i] = T->border[i];
  __syncthreads();
  SynGradWarpSmem &W = Wall[wib];
  float *const vgf = reinterpret_cast<float *>(W.fft), *const vgo = vgf + kBins;  // dgf times frac / omf
  float *const vrf = vgf + 2 * kBins, *const vro = vgf + 3 * kBins;               // drf times frac / omf
  const float beta = 0.02f;
  const long long units = A.n_rows * A.n_frames;
  for (long long u = (long long)blockIdx.x * kSgWarps + wib; u < units; u += (long long)gridDim.x * kSgWarps) {
    const long long row = u / A.n_frames;
    const int t = (int)(u % A.n_frames);
    const float *ops = A.ops + (size_t)row * A.ops_stride + (size_t)t * kSynthOps;
    const float *Ey = ops + 4 * kBins;
    const bool silence = ops[4 * kBins + kBands] != 0.f;
    const float *gr = A.gr + (size_t)row * A.gr_stride + (size_t)t * 68;
    const float *d0 = A.dout + (size_t)row * A.dout_stride + (size_t)t * kFrame;
    const float *d1 = t + 1 < A.n_frames ? d0 + kFrame : nullptr;

    // the band gains as the synthesis applied them
    for (int b = lane; b < kBands; b += 32) {
      const float g = gr[b], r = gr[kBands + b];
      W.g[b] = g;
      W.r[b] = r;
      W.ir[b] = 1.f - r;
      W.gw[b] = g * (float)sin((double)(float)(M_PI / 2 * (double)g));
    }
    __syncwarp();
    float G = 0.f, q = 0.f, den = 0.f;
    if (A.postfilter) {
      if (lane == 0) {
        float e0 = 0.f, e1 = 0.f;
        for (int b = 0; b < kBands; b++) e0 += W.g[b] * Ey[b];
        for (int b = 0; b < kBands; b++) e1 += W.gw[b] * Ey[b];
        den = e1 + 1e-6f;
        q = e0 / den;
        G = sqrtf(((1.f + beta) * q) / (1.f + beta * (q * q)));
      }
      G = __shfl_sync(0xffffffffu, G, 0);
      q = __shfl_sync(0xffffffffu, q, 0);
      den = __shfl_sync(0xffffffffu, den, 0);
    }
    for (int b = lane; b < kBands; b += 32) W.gu[b] = A.postfilter ? G * W.gw[b] : W.g[b];

    // dL/dY of bins 0..399: the forward transform of the windowed dL/d(out)
    fft960_warp<false>(W.fft, B.ft, lane, [&](int i) {
      float v;
      if (i < kFrame) v = d0[i] * B.hw[i];
      else v = d1 ? d1[i - kFrame] * B.hw[kWin - 1 - i] : 0.f;
      return make_float2(v, 0.f);
    });
    constexpr int kPer = (kBins + 31) / 32;
    float2 dY[kPer];
#pragma unroll
    for (int j = 0; j < kPer; j++) {
      const int k = lane + 32 * j;
      dY[j] = k < kBins ? W.fft[fpos(k)] : make_float2(0.f, 0.f);
    }
    __syncwarp();  // every lane has read the transform before the products overwrite it
#pragma unroll
    for (int j = 0; j < kPer; j++) {
      const int k = lane + 32 * j;
      if (k >= kBins) continue;
      const float c = k == 0 ? 1.f : 2.f;
      const float2 dy = make_float2(c * dY[j].x, c * dY[j].y);
      const float2 x = make_float2(ops[2 * k], ops[2 * k + 1]);
      const int b = B.band_of[k];
      const float fr = B.frac[k], om = B.omf[k];
      float2 z = x;
      float drf = 0.f;
      const float gf = om * W.gu[b] + fr * W.gu[b + 1];
      if (!silence) {
        const float2 p = make_float2(ops[2 * kBins + 2 * k], ops[2 * kBins + 2 * k + 1]);
        const float rfx = om * W.ir[b] + fr * W.ir[b + 1], rfp = om * W.r[b] + fr * W.r[b + 1];
        z = make_float2(rfx * x.x + rfp * p.x, rfx * x.y + rfp * p.y);
        drf = gf * (dy.x * (p.x - x.x) + dy.y * (p.y - x.y));
      }
      const float dgf = dy.x * z.x + dy.y * z.y;
      vgf[k] = fr * dgf;
      vgo[k] = om * dgf;
      vrf[k] = fr * drf;
      vro[k] = om * drf;
    }
    __syncwarp();
    // band b: omf-weighted bins of band b, frac-weighted bins of band b - 1
    for (int b = lane; b < kBands; b += 32) {
      float ag = 0.f, ar = 0.f;
      if (b > 0)
        for (int k = B.border[b - 1]; k < B.border[b]; k++) { ag += vgf[k]; ar += vrf[k]; }
      if (b < kBands - 1)
        for (int k = B.border[b]; k < B.border[b + 1]; k++) { ag += vgo[k]; ar += vro[k]; }
      W.dgu[b] = ag;
      W.dr[b] = ar;
    }
    __syncwarp();
    float S = 0.f;  // sum_j dgu_j gw_j
    if (A.postfilter) {
      for (int b = lane; b < kBands; b += 32) S += W.dgu[b] * W.gw[b];
      for (int o = 16; o > 0; o >>= 1) S += __shfl_xor_sync(0xffffffffu, S, o);
    }
    float *dgr = A.dgr + (size_t)row * A.dgr_stride + (size_t)t * 68;
    for (int b = lane; b < kBands; b += 32) {
      float dg = W.dgu[b];
      if (A.postfilter) {
        if (G == 0.f) {
          dg = 0.f;
        } else {
          float s, c;
          sincospif(0.5f * W.g[b], &s, &c);
          const float gwp = s + W.g[b] * ((float)(M_PI / 2) * c);
          const float dGdq = ((1.f + beta) * (1.f - beta * (q * q))) / (2.f * G * ((1.f + beta * (q * q)) * (1.f + beta * (q * q))));
          dg = W.dgu[b] * (G * gwp) + S * dGdq * (Ey[b] * (1.f - q * gwp) / den);
        }
      }
      dgr[b] = dg;
      dgr[kBands + b] = silence ? 0.f : W.dr[b];
    }
    __syncwarp();  // the next unit overwrites the band arrays and the line
  }
}

// ------------------------------------------------------------------------------------------
// staging: append the new hops to each stream's PCM line / slide the history forward
// ------------------------------------------------------------------------------------------
__global__ void stage_in_kernel(float *pcm, size_t pcm_stride, const float *in, const short *in16, size_t in_stride,
                                int n_streams, int n_samples, float i16_div, const int *row, const int *hops) {
  const int s = blockIdx.x;  // streams on grid.x (no 65535 limit), chunks of the row on grid.y
  const size_t r = row ? row[s] : s;  // input row of slot s
  const int n = hops ? hops[s] * kFrame : n_samples;  // a ragged call reads only the slot's own hops
  float *dst = pcm + (size_t)s * pcm_stride + kKeep;
  for (int i = blockIdx.y * blockDim.x + threadIdx.x; i < n; i += gridDim.y * blockDim.x) {
    float v;
    if (in) v = in[r * in_stride + i];
    else v = ((float)in16[r * in_stride + i]) / i16_div;  // main.cpp:34 (32768) / denoise.cpp:681 (NORM_RATIO 1)
    dst[i] = v;
  }
}

// keep the last 5280 samples of the line for the next call.  One block per stream; the tail is read
// into registers before anything is overwritten.
__global__ void __launch_bounds__(512) slide_history_kernel(float *pcm, size_t pcm_stride, int n_samples) {
  float *row = pcm + (size_t)blockIdx.x * pcm_stride;
  constexpr int kPer = (kKeep + 511) / 512;
  float keep[kPer];
#pragma unroll
  for (int i = 0; i < kPer; i++) {
    int j = threadIdx.x + 512 * i;
    keep[i] = j < kKeep ? row[n_samples + j] : 0.f;
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < kPer; i++) {
    int j = threadIdx.x + 512 * i;
    if (j < kKeep) row[j] = keep[i];
  }
}

// ------------------------------------------------------------------------------------------
// BASELINE.json config 5: the pitch analysis alone.  One warp per stream-frame: pitch_downsample + pitch_search +
// remove_doubling on a 1728-sample pitch buffer (6 912 B in, 16 B out), the same device code the analysis kernel runs.
// ------------------------------------------------------------------------------------------
constexpr int kPitchWarps = 8;
__global__ void __launch_bounds__(kPitchWarps * 32) pitch_only_kernel(PitchOnlyArgs A) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  WarpSmem *Wall = reinterpret_cast<WarpSmem *>(smem_raw);
  const int lane = threadIdx.x & 31, wib = threadIdx.x >> 5;
  const long s = (long)blockIdx.x * kPitchWarps + wib;
  if (s >= A.n_units) return;
  WarpSmem &W = Wall[wib];
#ifdef PNB_ANA_TIMING
  unsigned long long ana_acc[16];
  long long ana_t0 = clock64();
#endif
  const PitchResult r = pitch_stage<true>(W, A.buf + (size_t)s * A.stride, nullptr, A.prev_period ? A.prev_period[s] : 0,
                                          A.prev_gain ? A.prev_gain[s] : 0.f, lane ANA_TIMER_ARGS);
  if (lane == 0) {
    A.T[s] = r.T;
    A.gain[s] = r.gain;
    A.corr[s] = r.pitch_corr;
    if (A.lag) A.lag[s] = r.pitch_lag;
  }
}

// ---------------------------------------------------------------------------------- launchers
static size_t analysis_smem_bytes() { return ((sizeof(BlockSmem) + 15) / 16) * 16 + kAnaWarps * sizeof(WarpSmem); }
static size_t synthesis_smem_bytes() { return ((sizeof(SynBlockSmem) + 15) / 16) * 16 + kSynWarps * sizeof(SynWarpSmem); }

cudaError_t dsp_configure() {
  cudaError_t e = cudaFuncSetAttribute(analysis_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)analysis_smem_bytes());
  if (e != cudaSuccess) return e;
  e = cudaFuncSetAttribute(synthesis_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                           (int)synthesis_smem_bytes());
  if (e != cudaSuccess) return e;
  return cudaFuncSetAttribute(synthesis_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                              (int)synthesis_smem_bytes());
}

void launch_analysis(const AnalysisArgs &a, cudaStream_t st) {
  dim3 grid((a.n_streams + kAnaWarps - 1) / kAnaWarps);
  analysis_kernel<<<grid, kAnaWarps * 32, analysis_smem_bytes(), st>>>(a);
}
// ------------------------------------------------------------------------------------------
// Training-data labels (SURVEY.md 8 row f1).  One warp per (frame, pair); lane b and b+32 own a band.
// Follows the reference's mixed float/double arithmetic literally (denoise.cpp is C++: sqrt of a float
// expression is sqrtf, of a double expression sqrt); this file is compiled with -fmad=false.
//   calc_ideal_gain :571-577, estimate_phat_corr :549-553, filter_strength_calc :555-569,
//   adjust_gain_strength_by_condition :579-589, post_filtering :216-250 (applied in train() because
//   denoise.cpp:45-46 defines TEST), record layout :761-773.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) train_labels_kernel(LabelArgs A) {
  __shared__ float sh_g[8][kBands], sh_gw[8][kBands];
  const int wib = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const long wid = (long)blockIdx.x * 8 + wib;
  const long total = (long)A.n_frames * A.n_pairs;
  if (wid >= total) return;
  const int t = (int)(wid / A.n_pairs), p = (int)(wid % A.n_pairs);
  const int S = 2 * A.n_pairs;
  const size_t fn = (size_t)t * S + p, fc = fn + A.n_pairs;   // noisy / clean rows of hop t
  float *rec = A.records + (size_t)p * A.pair_stride + (size_t)t * 138;
  const float *Ey = A.Ex + fn * kBands;
  float pna = 0.f;                                            // denoise.cpp:207-210
  for (int i = 0; i < 7; i++) pna += A.tab->comb_w[i] * A.tab->comb_w[i];
  const float n0 = (float)0.03;
  for (int b = lane; b < kBands; b += 32) {
    const float ex = A.Ex[fc * kBands + b], ey = Ey[b];
    const float exp_c = A.raw[fc * 68 + kBands + b], q = A.raw[fn * 68 + kBands + b];
    rec[b] = A.raw[fn * 68 + b];
    rec[kBands + b] = q;
    float g = (float)((double)ex / (.0001 + (double)ey));
    if (g > 1.f) g = 1.f;
    if (g < 0.f) g = 0.f;
    const float ephatp = (float)((double)q / sqrt((double)(1.f - pna) * ((double)q * (double)q) + (double)pna));
    float a = ephatp * ephatp - exp_c * exp_c;
    if (a < 0.f) a = 0.f;
    const float bb = ephatp * q * (1.f - exp_c * exp_c);
    float c = exp_c * exp_c - q * q;
    if (c < 0.f) c = 0.f;
    const float alpha = (float)((double)(sqrtf(bb * bb + a * c) - bb) / ((double)a + 1e-8));
    float r = alpha / (1.f + alpha);
    if (ephatp < exp_c) {
      const float g_att = sqrtf((1.f + n0 - exp_c * exp_c) / (1.f + n0 - ephatp * ephatp));
      r = (float)0.99;
      g *= g_att;
    }
    rec[104 + b] = r;
    if (A.gr) A.gr[fn * 68 + kBands + b] = r;  // the labels again, for the resynthesis of the noisy row (:742-759)
    sh_g[wib][b] = g;
    // sinf of the reference's libm is correctly rounded in all but rare cases; so is the rounded double sine
    sh_gw[wib][b] = g * (float)sin((double)(float)(M_PI / 2 * (double)g));
  }
  __syncwarp();
  float G = 0.f;
  if (lane == 0) {
    float e0 = 0.f, e1 = 0.f;
    for (int b = 0; b < kBands; b++) e0 += sh_g[wib][b] * Ey[b];
    for (int b = 0; b < kBands; b++) e1 += sh_gw[wib][b] * Ey[b];
    const float qq = e0 / (e1 + 1e-6f);
    G = sqrtf(((1.f + 0.02f) * qq) / (1.f + 0.02f * (qq * qq)));
    rec[68] = A.feat[fn * kFeat + 68];
    rec[69] = A.feat[fn * kFeat + 69];
  }
  G = __shfl_sync(0xffffffffu, G, 0);
  for (int b = lane; b < kBands; b += 32) {
    const float g = G * sh_gw[wib][b];
    rec[70 + b] = g;
    if (A.gr) A.gr[fn * 68 + b] = g;
  }
}

#ifdef PNB_ANA_TIMING
extern "C" int pnb_debug_analysis_cycles(unsigned long long *out16, int reset) {
  cudaDeviceSynchronize();
  cudaMemcpyFromSymbol(out16, g_ana_cycles, sizeof(unsigned long long) * 16);
  if (reset) {
    unsigned long long z[16] = {0};
    cudaMemcpyToSymbol(g_ana_cycles, z, sizeof z);
  }
  return 0;
}
#endif

bool launch_pitch_only(const PitchOnlyArgs &a, cudaStream_t st) {
  const size_t smem = kPitchWarps * sizeof(WarpSmem);
  static bool configured = false;
  if (!configured) {
    if (cudaFuncSetAttribute(pitch_only_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess) return false;
    configured = true;
  }
  pitch_only_kernel<<<(unsigned)((a.n_units + kPitchWarps - 1) / kPitchWarps), kPitchWarps * 32, smem, st>>>(a);
  return true;
}

void launch_train_labels(const LabelArgs &a, cudaStream_t st) {
  const long total = (long)a.n_frames * a.n_pairs;
  train_labels_kernel<<<(unsigned)((total + 7) / 8), 256, 0, st>>>(a);
}

// a grid that fills the device once: each warp then walks units (row, hop) at a stride of the grid, so the block's
// tables are staged once per block, not once per eight hops
bool launch_synthesis_backward(const SynthGradArgs &a, cudaStream_t st) {
  const size_t smem = ((sizeof(SynGradBlockSmem) + 15) / 16) * 16 + kSgWarps * sizeof(SynGradWarpSmem);
  int dev = 0, sms = 0, per_sm = 0;
  if (cudaGetDevice(&dev) != cudaSuccess) return false;
  if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess) return false;
  if (cudaFuncSetAttribute(synthesis_backward_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem) != cudaSuccess)
    return false;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, synthesis_backward_kernel, kSgWarps * 32, smem) != cudaSuccess ||
      per_sm < 1)
    return false;
  const long long units = a.n_rows * a.n_frames, need = (units + kSgWarps - 1) / kSgWarps;
  const long long full = (long long)sms * per_sm;
  synthesis_backward_kernel<<<(unsigned)(need < full ? need : full), kSgWarps * 32, smem, st>>>(a);
  return true;
}

void launch_synthesis(const SynthesisArgs &a, cudaStream_t st) {
  dim3 grid((a.n_streams + kSynWarps - 1) / kSynWarps);
  if (a.clamp16) synthesis_kernel<true><<<grid, kSynWarps * 32, synthesis_smem_bytes(), st>>>(a);
  else synthesis_kernel<false><<<grid, kSynWarps * 32, synthesis_smem_bytes(), st>>>(a);
}
void launch_stage_in(float *pcm, size_t pcm_stride, const float *in, const short *in16, size_t in_stride,
                     int n_streams, int n_samples, cudaStream_t st, float i16_div, const int *row, const int *hops) {
  dim3 grid(n_streams, (n_samples + 1023) / 1024 > 8 ? 8 : (n_samples + 1023) / 1024);
  stage_in_kernel<<<grid, 256, 0, st>>>(pcm, pcm_stride, in, in16, in_stride, n_streams, n_samples, i16_div, row, hops);
}
void launch_slide_history(float *pcm, size_t pcm_stride, int n_streams, int n_samples, cudaStream_t st) {
  slide_history_kernel<<<n_streams, 512, 0, st>>>(pcm, pcm_stride, n_samples);
}

}  // namespace pnb
