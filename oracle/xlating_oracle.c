/*
 * oracle/xlating_oracle.c -- CPU restatement of the reference frequency-
 * translating FIR decimator.  TEST INFRASTRUCTURE ONLY (see oracle/oracle.h).
 *
 * What the reference computes (/root/reference/src/xlating.c):
 *   create (:495-582)   w0   = (float)(2*pi*center/fs)                       :524
 *                       bpf[i] = lpf[i] * cexpf(I * (float)i * w0)           :525-528
 *                       rev    = reverse(bpf)  (even lengths keep the middle
 *                                pair un-swapped, a quirk of :530-534)
 *                       incr   = cexpf(I * (-w0 * (float)decimation))        :544
 *                       phase  = 1, history = taps_len-1 zero samples        :543,552
 *   process cf32 (:52-83) work = history ++ convert(input)
 *                       for idx = 0; idx < len(work)-(T-1); idx += D:
 *                           acc  = sum_{j<T} work[idx+j]*rev[j]  (in order, float)
 *                           out  = acc*phase; phase = phase*incr             :70-71
 *                       if any output: phase /= hypotf(re,im)                :73
 *                       history = work[idx..]                                :76-79
 *   process Q15 (:92-140) same walk in int16/int64 with >>15 and saturation.
 *
 * The restatement keeps every float rounding step of the strict build
 * (-std=c11 -O2 -ffp-contract=off; complex multiply = two products and one
 * add/sub per component, as libgcc's __mulsc3 does for finite values) so that it
 * is bit-identical to oracle/_ref/libref_strict.so.  It is written with real
 * arithmetic only (no <complex.h> in the loop) and one shared sample walk for
 * both numeric paths.
 */
#include "oracle.h"

#include <complex.h>
#include <math.h>
#include <stdlib.h>
#include <string.h>

#ifndef M_PI
#define M_PI 3.14159265358979323846
#endif

struct orc_xlating {
  uint32_t decim;
  size_t ntaps;
  float *rev_f32;   /* 2*ntaps: reversed band-pass taps, interleaved re,im */
  int16_t *rev_q15; /* 2*ntaps: same taps in Q15 (:486-487) */

  /* the two numeric paths keep separate sample histories but -- exactly like
   * the reference -- ONE shared history length (struct xlating_t :29) */
  float *work_f32;   /* 2*(max_in/2 + ntaps-1) */
  int16_t *work_q15; /* same count */
  size_t hist;

  float *out_f32;
  int16_t *out_q15;

  float ph_re, ph_im, inc_re, inc_im;     /* :36-37 */
  int16_t qph_re, qph_im, qinc_re, qinc_im; /* :39-42 */
};

void orc_xlating_destroy(orc_xlating *f) {
  if (f == NULL) return;
  free(f->rev_f32);
  free(f->rev_q15);
  free(f->work_f32);
  free(f->work_q15);
  free(f->out_f32);
  free(f->out_q15);
  free(f);
}

int orc_xlating_create(uint32_t decimation, const float *taps, size_t taps_len,
                       int32_t center_freq, uint32_t sampling_freq,
                       uint32_t max_input_len, orc_xlating **out) {
  if (taps_len == 0) return -1; /* :496 */
  orc_xlating *f = (orc_xlating *)calloc(1, sizeof(*f));
  if (f == NULL) return -1;
  f->decim = decimation;
  f->ntaps = taps_len;
  f->rev_f32 = (float *)malloc(sizeof(float) * 2 * taps_len);
  f->rev_q15 = (int16_t *)malloc(sizeof(int16_t) * 2 * taps_len);

  /* :524 -- double expression, rounded once to float */
  const float w0 = (float)(2 * M_PI * (double)center_freq / (double)sampling_freq);
  /* forward band-pass taps, then store them reversed */
  for (size_t i = 0; i < taps_len; i++) {
    const float ang = (float)i * w0;           /* :526 float product */
    const float complex e = cexpf(0.0f + ang * I);
    const size_t dst = taps_len - 1 - i;
    f->rev_f32[2 * dst] = taps[i] * crealf(e); /* :527 real * complex */
    f->rev_f32[2 * dst + 1] = taps[i] * cimagf(e);
  }
  if ((taps_len & 1) == 0) {
    /* :530-534 runs i <= T/2, which re-swaps the middle pair of an even-length
     * vector.  lpf.c only ever produces odd lengths; kept for fidelity. */
    const size_t a = taps_len / 2 - 1, b = taps_len / 2;
    for (int c = 0; c < 2; c++) {
      float t = f->rev_f32[2 * a + c];
      f->rev_f32[2 * a + c] = f->rev_f32[2 * b + c];
      f->rev_f32[2 * b + c] = t;
    }
  }
  for (size_t j = 0; j < 2 * taps_len; j++) {
    f->rev_q15[j] = (int16_t)(f->rev_f32[j] * (1 << 15)); /* :486-487 */
  }

  f->ph_re = 1.0f; /* :543 */
  f->ph_im = 0.0f;
  const float complex inc = cexpf(0.0f + -w0 * decimation * I); /* :544 */
  f->inc_re = crealf(inc);
  f->inc_im = cimagf(inc);
  f->qph_re = INT16_MAX; /* :546-549 */
  f->qph_im = 0;
  f->qinc_re = (int16_t)(f->inc_re * INT16_MAX);
  f->qinc_im = (int16_t)(f->inc_im * INT16_MAX);

  f->hist = taps_len - 1; /* :552 */
  const size_t cap = max_input_len / 2 + f->hist;
  f->work_f32 = (float *)calloc(2 * cap + 2, sizeof(float));
  f->work_q15 = (int16_t *)calloc(2 * cap + 2, sizeof(int16_t));
  const size_t out_cap = max_input_len / 2 / decimation + 1; /* :568 */
  f->out_f32 = (float *)malloc(sizeof(float) * 2 * out_cap);
  f->out_q15 = (int16_t *)malloc(sizeof(int16_t) * 2 * out_cap);
  if (!f->rev_f32 || !f->rev_q15 || !f->work_f32 || !f->work_q15 || !f->out_f32 || !f->out_q15) {
    orc_xlating_destroy(f);
    return -1;
  }
  *out = f;
  return 0;
}

/* scalar converters, src/xlating.c:389-390 / :399-400 / :409-410 (all exact in fp32) */
static inline float to_f32(int fmt, const void *in, size_t i) {
  switch (fmt) {
    case ORC_FMT_CU8: return ((float)((const uint8_t *)in)[i] - 127.5F) / 128.0F;
    case ORC_FMT_CS8: return ((const int8_t *)in)[i] / 128.0F;
    default:          return ((const int16_t *)in)[i] / 32768.0F;
  }
}

/* src/xlating.c:418 / :425 / :432 */
static inline int16_t to_q15(int fmt, const void *in, size_t i) {
  switch (fmt) {
    case ORC_FMT_CU8: return (int16_t)((((int16_t)((const uint8_t *)in)[i]) - 128) << 8);
    case ORC_FMT_CS8: return (int16_t)(((int16_t)((const int8_t *)in)[i]) << 8);
    default:          return ((const int16_t *)in)[i];
  }
}

size_t orc_xlating_process_cf32(orc_xlating *f, int fmt, const void *input,
                                size_t input_len, int renorm, const float **out) {
  const size_t n_in = input_len / 2;
  float *w = f->work_f32;
  for (size_t i = 0; i < 2 * n_in; i++) w[2 * f->hist + i] = to_f32(fmt, input, i);

  const size_t total = f->hist + n_in;
  const size_t T = f->ntaps;
  size_t idx = 0, n_out = 0;
  if (total > T - 1) { /* :58 */
    const size_t limit = total - (T - 1);
    for (; idx < limit; idx += f->decim, n_out++) {
      float acc_re = 0.0f, acc_im = 0.0f;
      const float *x = w + 2 * idx;
      for (size_t j = 0; j < T; j++) { /* :67-69, one complex MAC per tap */
        const float xr = x[2 * j], xi = x[2 * j + 1];
        const float tr = f->rev_f32[2 * j], ti = f->rev_f32[2 * j + 1];
        const float pr = xr * tr - xi * ti;
        const float pi = xr * ti + xi * tr;
        acc_re = acc_re + pr;
        acc_im = acc_im + pi;
      }
      /* :70 derotate, :71 advance the oscillator */
      f->out_f32[2 * n_out] = acc_re * f->ph_re - acc_im * f->ph_im;
      f->out_f32[2 * n_out + 1] = acc_re * f->ph_im + acc_im * f->ph_re;
      const float nr = f->ph_re * f->inc_re - f->ph_im * f->inc_im;
      const float ni = f->ph_re * f->inc_im + f->ph_im * f->inc_re;
      f->ph_re = nr;
      f->ph_im = ni;
    }
    if (renorm) { /* :73 (absent from the AVX variant, :336-339) */
      const float mag = hypotf(f->ph_re, f->ph_im);
      f->ph_re = f->ph_re / mag;
      f->ph_im = f->ph_im / mag;
    }
  }
  f->hist = total - idx; /* :76 */
  if (idx > 0) memmove(w, w + 2 * idx, sizeof(float) * 2 * f->hist);
  *out = f->out_f32;
  return n_out;
}

static inline int16_t sat16(int32_t v) { /* :85-90 */
  if (v > INT16_MAX) return INT16_MAX;
  if (v < INT16_MIN) return INT16_MIN;
  return (int16_t)v;
}

size_t orc_xlating_process_q15(orc_xlating *f, int fmt, const void *input,
                               size_t input_len, const int16_t **out) {
  int16_t *w = f->work_q15;
  for (size_t i = 0; i < input_len; i++) w[2 * f->hist + i] = to_q15(fmt, input, i);
  const size_t n_in = input_len / 2;

  const size_t total = f->hist + n_in;
  const size_t T = f->ntaps;
  size_t idx = 0, n_out = 0;
  if (total > T - 1) { /* :98 */
    const size_t limit = total - (T - 1);
    for (; idx < limit; idx += f->decim, n_out++) {
      int64_t acc_re = 0, acc_im = 0;
      const int16_t *x = w + 2 * idx;
      for (size_t j = 0; j < T; j++) { /* :108-116 */
        const int32_t xr = x[2 * j], xi = x[2 * j + 1];
        const int32_t tr = f->rev_q15[2 * j], ti = f->rev_q15[2 * j + 1];
        /* each pair is summed in 32 bits before it meets the int64 accumulator.  The imaginary pair is
         * 2^31 for x = tap = (-32768, -32768), which the reference's int arithmetic wraps to -2^31: wrap
         * it here with unsigned arithmetic (defined) and gcc's modular conversion back to int32_t.  Each
         * product fits in int32_t. */
        acc_re += (int32_t)((uint32_t)(xr * tr) - (uint32_t)(xi * ti));
        acc_im += (int32_t)((uint32_t)(xr * ti) + (uint32_t)(xi * tr));
      }
      const int16_t ar = sat16((int32_t)(acc_re >> 15)); /* :118-119 */
      const int16_t ai = sat16((int32_t)(acc_im >> 15));
      int64_t rr = ar * f->qph_re - ai * f->qph_im;       /* :121-124 */
      int64_t ri = ar * f->qph_im + ai * f->qph_re;
      f->out_q15[2 * n_out] = sat16((int32_t)(rr >> 15));
      f->out_q15[2 * n_out + 1] = sat16((int32_t)(ri >> 15));
      rr = f->qph_re * f->qinc_re - f->qph_im * f->qinc_im; /* :126-129 */
      ri = f->qph_re * f->qinc_im + f->qph_im * f->qinc_re;
      f->qph_re = sat16((int32_t)(rr >> 15));
      f->qph_im = sat16((int32_t)(ri >> 15));
    }
  }
  f->hist = total - idx; /* :133 */
  if (idx > 0) memmove(w, w + 2 * idx, sizeof(int16_t) * 2 * f->hist);
  *out = f->out_q15;
  return n_out;
}

size_t orc_xlating_history(const orc_xlating *f) { return f->hist; }

size_t orc_xlating_q15_consts(const orc_xlating *f, const int16_t **rev, int16_t *qinc_re, int16_t *qinc_im) {
  *rev = f->rev_q15;
  *qinc_re = f->qinc_re;
  *qinc_im = f->qinc_im;
  return f->ntaps;
}

void orc_xlating_phase(const orc_xlating *f, float *re, float *im) {
  *re = f->ph_re;
  *im = f->ph_im;
}

size_t orc_xlating_taps(const orc_xlating *f, const float **rev) {
  *rev = f->rev_f32;
  return f->ntaps;
}

size_t orc_xlating_get_history(const orc_xlating *f, const float **samples_interleaved) {
  *samples_interleaved = f->work_f32; /* the history sits at the front of the work buffer */
  return f->hist;
}

int orc_xlating_set_state(orc_xlating *f, const float *history_interleaved, size_t hist, float ph_re, float ph_im) {
  if (hist > f->ntaps) return -1;
  memcpy(f->work_f32, history_interleaved, sizeof(float) * 2 * hist);
  f->hist = hist;
  f->ph_re = ph_re;
  f->ph_im = ph_im;
  return 0;
}
