/*
 * csrc/taps_host.c -- per-client filter constants, computed once on the host.
 *
 * The reference turns the real low-pass prototype into a complex band-pass
 * centred on the client's offset and stores it time-reversed so the hot loop is
 * a plain dot product over a sliding window (src/xlating.c:512-534); the
 * translation back to baseband is an oscillator stepped once per OUTPUT sample
 * (:544).  We keep exactly those constants -- including their float rounding --
 * because parity is against the reference's float arithmetic, not exact math:
 *   w0      = (float)(2*pi*center/fs)                     :524
 *   bpf[i]  = lpf[i] * cexpf(j * ((float)i * w0))          :525-528
 *   rev[j]  = bpf[T-1-j]  (even T keeps the middle pair un-swapped, :530-534)
 *   incr    = cexpf(j * (-w0 * (float)D))                  :544
 *   Q15     = (int16)(x * 32768) for taps (:486-487), (int16)(x * 32767) for incr (:548-549)
 * Compiled with -ffp-contract=off.
 */
#include "taps_host.h"

#include <complex.h>
#include <errno.h>
#include <math.h>
#include <stdlib.h>

static const double XL_PI = 3.14159265358979323846;

int xl_client_consts_build(const float *lpf_taps, size_t taps_len, uint32_t decimation,
                           int32_t center_freq, uint32_t sampling_freq, xl_client_consts *out) {
  out->rev_cf32 = (float *)malloc(sizeof(float) * 2 * taps_len);
  out->rev_q15 = (int16_t *)malloc(sizeof(int16_t) * 2 * taps_len);
  if (out->rev_cf32 == NULL || out->rev_q15 == NULL) {
    xl_client_consts_free(out);
    return -ENOMEM;
  }
  const float w0 = (float)(2 * XL_PI * (double)center_freq / (double)sampling_freq);

  for (size_t i = 0; i < taps_len; i++) {
    const float theta = (float)i * w0;
    const float complex rot = cexpf(0.0f + theta * I);
    float *slot = out->rev_cf32 + 2 * (taps_len - 1 - i);
    slot[0] = lpf_taps[i] * crealf(rot);
    slot[1] = lpf_taps[i] * cimagf(rot);
  }
  if (taps_len % 2 == 0) {
    /* the reference's reversal loop runs one step too far and swaps the two
     * middle taps of an even-length filter back; reproduce it */
    float *lo = out->rev_cf32 + 2 * (taps_len / 2 - 1);
    float *hi = out->rev_cf32 + 2 * (taps_len / 2);
    for (int c = 0; c < 2; c++) {
      const float keep = lo[c];
      lo[c] = hi[c];
      hi[c] = keep;
    }
  }
  for (size_t j = 0; j < 2 * taps_len; j++) {
    out->rev_q15[j] = (int16_t)(out->rev_cf32[j] * (1 << 15));
  }

  const float complex step = cexpf(0.0f + -w0 * decimation * I);
  out->incr_re = crealf(step);
  out->incr_im = cimagf(step);
  out->qincr_re = (int16_t)(out->incr_re * INT16_MAX);
  out->qincr_im = (int16_t)(out->incr_im * INT16_MAX);
  return 0;
}

void xl_client_consts_free(xl_client_consts *c) {
  free(c->rev_cf32);
  free(c->rev_q15);
  c->rev_cf32 = NULL;
  c->rev_q15 = NULL;
}

int xl_walk(long long *hist, long long n_in, size_t taps_len, uint32_t decimation, int out_cap) {
  const long long avail = *hist + n_in - (long long)taps_len; /* last admissible window start - first */
  long long n_out = avail >= 0 ? avail / decimation + 1 : 0;
  if (n_out > out_cap) n_out = out_cap;
  *hist += n_in - n_out * (long long)decimation;
  return (int)n_out;
}

void xl_poly_pack(const float *rev_cf32, size_t taps_len, uint32_t interp, float *out) {
  const size_t L = interp, Tb = (taps_len + L - 1) / L;
  for (size_t r = 0; r < L; r++)
    for (size_t t = 0; t < Tb; t++) {
      const size_t j = r + t * L;
      float *slot = out + 2 * (r * Tb + t);
      slot[0] = j < taps_len ? rev_cf32[2 * j] : 0.0f;
      slot[1] = j < taps_len ? rev_cf32[2 * j + 1] : 0.0f;
    }
}

void xl_osc_chain_cf32(float *phase_re, float *phase_im, float incr_re, float incr_im, float *table, int n_out) {
  float pr = *phase_re, pi = *phase_im;
  for (int k = 0; k < n_out; k++) {
    if ((k & 1) == 0) {
      table[k] = pr;
      table[k + 1] = pi;
    }
    /* (pr + j pi)(ir + j ii), every product and sum rounded to float: what __mulsc3
     * computes for finite operands in the reference's strict build (:71) */
    const float nr = pr * incr_re - pi * incr_im;
    const float ni = pr * incr_im + pi * incr_re;
    pr = nr;
    pi = ni;
  }
  if (n_out > 0) {
    const float mag = hypotf(pr, pi); /* :73 */
    pr = pr / mag;
    pi = pi / mag;
  }
  *phase_re = pr;
  *phase_im = pi;
}
