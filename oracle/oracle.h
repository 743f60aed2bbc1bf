/*
 * oracle/oracle.h -- CPU restatement of the reference hot path.
 *
 * TEST INFRASTRUCTURE ONLY.  Nothing under oracle/ is part of the product:
 * only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
 * --impl reference legs may load liboracle.so or the oracle/_ref libraries, and there
 * only as the checker / the CPU timing baseline.  The product library
 * (sdr-server_b200/lib/libxlating_b200.so) never links or dlopens this.
 *
 * Parity status: PINNED.  The restatement is checked (tests/test_oracle.py)
 *   - against every golden vector the reference's own tests hold for this path
 *     (test/test_xlating.c:29,35,44,48,55,59,75-80; test/test_lpf.c:30-33;
 *      test/test_tcp_server.c:173-174,208,237) -> tests/golden/reference_fixtures.json
 *   - bit-for-bit against the reference itself compiled from /root/reference
 *     (oracle/_ref/libref_strict.so) when that library is present.
 *
 * All file:line citations are relative to /root/reference.
 */
#ifndef ORACLE_H_
#define ORACLE_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

/* input sample formats, as the three SDR front-ends deliver them
 * (src/xlating.c:384-414): interleaved I,Q scalars. */
enum { ORC_FMT_CU8 = 0, ORC_FMT_CS8 = 1, ORC_FMT_CS16 = 2 };

typedef struct orc_xlating orc_xlating;

/* src/lpf.c:53-99.  Returns 0 and a malloc'd tap vector, or -1 on bad args. */
int orc_lpf_design(float gain, uint32_t sampling_freq, uint32_t cutoff_freq,
                   uint32_t transition_width, float **taps, size_t *len);

/* src/xlating.c:495-582.  Unlike the reference, the taps are COPIED (the
 * oracle never owns caller memory). */
int orc_xlating_create(uint32_t decimation, const float *taps, size_t taps_len,
                       int32_t center_freq, uint32_t sampling_freq,
                       uint32_t max_input_len, orc_xlating **out);
void orc_xlating_destroy(orc_xlating *f);

/* src/xlating.c:52-83 + 384-414.  input_len counts scalar elements (2 per
 * complex sample).  Output is interleaved re,im floats into a filter-owned
 * buffer.  renorm!=0 -> process_native_cf32 behaviour (phase /= hypotf once per
 * call, :73); renorm==0 -> the AVX process_optimized_cf32 behaviour (:336-339,
 * no renormalisation). Returns number of complex outputs. */
size_t orc_xlating_process_cf32(orc_xlating *f, int fmt, const void *input,
                                size_t input_len, int renorm, const float **out);

/* src/xlating.c:92-140 + 416-435 (Q15 integer path). */
size_t orc_xlating_process_q15(orc_xlating *f, int fmt, const void *input,
                               size_t input_len, const int16_t **out);

/* state inspection for tests */
size_t orc_xlating_history(const orc_xlating *f);
void orc_xlating_phase(const orc_xlating *f, float *re, float *im);
size_t orc_xlating_taps(const orc_xlating *f, const float **rev_taps_interleaved);
/* the Q15 path's constants: reversed taps (interleaved re,im) and the oscillator step */
size_t orc_xlating_q15_consts(const orc_xlating *f, const int16_t **rev_q15_interleaved, int16_t *qinc_re,
                              int16_t *qinc_im);

/* State hand-over, for the model check of the drop-in engine's stream overlay
 * (tests/stream_overlay_shim.cpp): the cf32 history the next call will prepend
 * (`hist` complex samples, interleaved; src/xlating.c:76-79) and the oscillator (:36). */
size_t orc_xlating_get_history(const orc_xlating *f, const float **samples_interleaved);
int orc_xlating_set_state(orc_xlating *f, const float *history_interleaved, size_t hist, float ph_re, float ph_im);

#ifdef __cplusplus
}
#endif
#endif
