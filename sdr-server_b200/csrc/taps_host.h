/*
 * csrc/taps_host.h -- host-side preparation of a client's filter constants.
 * Stays on the CPU (same libm calls as the reference, so the constants are
 * bit-identical): /root/reference/src/xlating.c:519-549.
 */
#ifndef XLATING_B200_TAPS_HOST_H_
#define XLATING_B200_TAPS_HOST_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct {
  float *rev_cf32;   /* 2*taps_len floats: reversed band-pass taps, (re,im) interleaved */
  int16_t *rev_q15;  /* 2*taps_len int16: the same taps in Q15 */
  float incr_re, incr_im;       /* oscillator step exp(-j*w0*D) */
  int16_t qincr_re, qincr_im;   /* Q15 oscillator step */
} xl_client_consts;

/* Returns 0, or -ENOMEM.  Free with xl_client_consts_free. */
int xl_client_consts_build(const float *lpf_taps, size_t taps_len, uint32_t decimation,
                           int32_t center_freq, uint32_t sampling_freq, xl_client_consts *out);
void xl_client_consts_free(xl_client_consts *c);

/* Polyphase branches of a rational (L/M) client, branch-major: for r < L and t < Tb = ceil(T/L),
 * out[r][t] = rev[r + t*L] ((re, im) interleaved), zero where r + t*L >= T.  Branch r holds the
 * taps that meet the nonzero samples of a zero-stuffed window whose start is -r mod L.
 * `out` has room for 2*L*Tb floats. */
/* The reference's walk over one call (src/xlating.c:58-60, :76): a filter whose next window starts *hist
 * samples (history_offset) before the call's n_in new samples produces the returned number of outputs (at
 * most out_cap) and leaves *hist for the next call.  Stage B of a cascade client walks its stage-A stream
 * with it. */
int xl_walk(long long *hist, long long n_in, size_t taps_len, uint32_t decimation, int out_cap);

void xl_poly_pack(const float *rev_cf32, size_t taps_len, uint32_t interp, float *out);

/* The float oscillator of one call on the host (src/xlating.c:70-73): n_out steps of
 * phase *= incr starting from *phase, the phase of every EVEN output k stored as
 * (re, im) at table[k] / table[k + 1], then -- if n_out > 0 -- the once-per-call
 * renormalisation phase /= hypotf(re, im).  *phase is advanced.  Plain IEEE float
 * arithmetic, unfused, exactly the reference's: a CPU core walks this dependent chain
 * about three times faster than one GPU lane does. */
void xl_osc_chain_cf32(float *phase_re, float *phase_im, float incr_re, float incr_im, float *table, int n_out);

#ifdef __cplusplus
}
#endif
#endif
