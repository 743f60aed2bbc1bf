/*
 * include/xlating.h -- drop-in C ABI of the H100 frequency-translating FIR
 * decimator.
 *
 * This header declares the symbols the reference's xlating unit exports
 * (reference: src/xlating.h:8-38, SIMD_STATUS at src/xlating.c:145-156,268), so
 * that the reference's callers -- src/dsp_worker.c:104,110-124,195-197,
 * src/main.c:10,23, test/test_xlating.c, test/perf_xlating.c -- compile and link
 * against libxlating_b200.so unchanged.  Behind them the arithmetic runs in
 * hand-written sm_90a CUDA kernels (sdr-server_b200/csrc/dropin_kernels.cuh, host side
 * in csrc/xlating_dropin.cu: concurrent calls on different filters are combined into
 * shared launches, identical input blocks are transferred once);
 * there is NO CPU fallback: if no CUDA device is usable, create fails with
 * -ENODEV and a "<3>" line on stderr.
 *
 * Contract kept from the reference (file:line in /root/reference):
 *   units      input_len counts scalar elements: bytes for cu8/cs8, int16 count
 *              for cs16 (src/xlating.c:355,375; src/dsp_worker.c:65).  It must not
 *              exceed max_input_buffer_length (also in scalar elements, :553).
 *              *output_len counts complex samples (:82,139).
 *   ownership  `taps` is adopted and free()d by destroy_xlating (:507-508,
 *              :600-602) unless create fails on taps_len==0.  *output points
 *              into filter-owned (pinned) host memory, valid until the next
 *              process_* call on that filter or destroy (:81,138).
 *   errors     create: 0 ok, -1 (taps_len==0), -ENOMEM, and additionally
 *              -ENODEV (no usable GPU) / -EIO (CUDA failure).  process_* are
 *              void: a device failure yields *output_len = 0 and a "<3>" log.
 *   threading  one filter is never used concurrently; different filters are
 *              fully concurrent (one dsp thread per client, src/dsp_worker.c:41-88).
 *   state      history (<= taps_len-1 samples), decimation phase and the
 *              oscillator carry over between calls exactly as
 *              src/xlating.c:52-83 / :92-140 do, including the once-per-call
 *              phase renormalisation (:73).
 *   variants   process_optimized_* == process_native_* (as in the reference's
 *              default x86-64 build where SIMD is "Not detected", :142-153).
 *
 * One extension, marked below, is not a reference symbol:
 * create_rational_frequency_xlating_filter, a filter whose output rate fs * L / M
 * does not divide the band rate.
 *
 * Many clients sharing one wideband input should use the batch extension in
 * include/xlating_group.h: one H2D copy and one fused launch for all clients.
 */
#ifndef XLATING_B200_XLATING_H_
#define XLATING_B200_XLATING_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
/* C++ callers see the interleaved (re, im) float pair layout of C's float complex */
typedef struct { float re, im; } xlating_cf32;
extern "C" {
#else
#include <complex.h>
typedef float complex xlating_cf32;
#endif

typedef struct xlating_t xlating;

/* "CUDA sm_90a" -- printed by the reference's main.c:23 and perf_xlating.c:15 */
extern const char *SIMD_STATUS;

/* replaces src/xlating.c:495-582 */
int create_frequency_xlating_filter(uint32_t decimation, float *taps, size_t taps_len,
                                    int32_t center_freq, uint32_t sampling_freq,
                                    uint32_t max_input_buffer_length, xlating **filter);

/* float path: replaces src/xlating.c:384-414 (native) and :352-382 (optimized) */
void process_native_cu8_cf32(const uint8_t *input, size_t input_len, xlating_cf32 **output, size_t *output_len, xlating *filter);
void process_native_cs8_cf32(const int8_t *input, size_t input_len, xlating_cf32 **output, size_t *output_len, xlating *filter);
void process_native_cs16_cf32(const int16_t *input, size_t input_len, xlating_cf32 **output, size_t *output_len, xlating *filter);
void process_optimized_cu8_cf32(const uint8_t *input, size_t input_len, xlating_cf32 **output, size_t *output_len, xlating *filter);
void process_optimized_cs8_cf32(const int8_t *input, size_t input_len, xlating_cf32 **output, size_t *output_len, xlating *filter);
void process_optimized_cs16_cf32(const int16_t *input, size_t input_len, xlating_cf32 **output, size_t *output_len, xlating *filter);

/* Q15 integer path: replaces src/xlating.c:416-447 (bit-exact) */
void process_native_cu8_cs16(const uint8_t *input, size_t input_len, int16_t **output, size_t *output_len, xlating *filter);
void process_native_cs8_cs16(const int8_t *input, size_t input_len, int16_t **output, size_t *output_len, xlating *filter);
void process_native_cs16_cs16(const int16_t *input, size_t input_len, int16_t **output, size_t *output_len, xlating *filter);
void process_optimized_cu8_cs16(const uint8_t *input, size_t input_len, int16_t **output, size_t *output_len, xlating *filter);
void process_optimized_cs8_cs16(const int8_t *input, size_t input_len, int16_t **output, size_t *output_len, xlating *filter);
void process_optimized_cs16_cs16(const int16_t *input, size_t input_len, int16_t **output, size_t *output_len, xlating *filter);

/* ---- extension (not in the reference) ----
 * A filter at the rational rate sampling_freq * interpolation / decimation.  It is exactly
 * create_frequency_xlating_filter(decimation, taps, taps_len, center_freq,
 * interpolation * sampling_freq, ...) fed the zero-stuffed stream u[interpolation * n] = x[n],
 * zeros elsewhere -- the definition xlg_add_client_rational uses.  Taps are designed at
 * interpolation * sampling_freq (with gain interpolation for unit passband gain); each output sums
 * only the ceil(taps_len / interpolation) taps that meet nonzero samples.  sampling_freq is the band
 * rate; max_input_buffer_length and input_len count scalar elements of the real input, as above.
 * `taps` and the outputs keep create_frequency_xlating_filter's contract.
 * Errors, in this order: -1 for taps_len == 0 (taps not adopted); -EINVAL and a "<3>" line when
 * interpolation == 0, decimation == 0, interpolation * sampling_freq > UINT32_MAX or
 * interpolation * max_input_buffer_length / 2 >= 2^31 (both checked before any CUDA call; taps are
 * freed); then -ENODEV, -EIO, -ENOMEM as create_frequency_xlating_filter.
 * interpolation == 1 is create_frequency_xlating_filter: same kernels, same bits, Q15 included.
 * With interpolation > 1 the process_*_cs16 (Q15) calls are refused: *output_len = 0, one "<3>" line
 * per filter, nothing consumed -- the next cf32 call continues as if the refused one had not been made. */
int create_rational_frequency_xlating_filter(uint32_t interpolation, uint32_t decimation, float *taps,
                                             size_t taps_len, int32_t center_freq, uint32_t sampling_freq,
                                             uint32_t max_input_buffer_length, xlating **filter);

/* replaces src/xlating.c:584-616; NULL is a no-op */
void destroy_xlating(xlating *filter);

#ifdef __cplusplus
}
#endif
#endif /* XLATING_B200_XLATING_H_ */
