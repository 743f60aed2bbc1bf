/*
 * include/xlating_group.h -- batch extension of the xlating C ABI: MANY clients
 * (channels) decimating ONE wideband IQ stream on one GPU.
 *
 * Why it exists.  In the reference every client owns a filter and a dsp thread,
 * and every SDR block is memcpy'd once per client (src/tcp_server.c:262-269 ->
 * src/queue.c:114) and converted + filtered once per client on the CPU
 * (src/dsp_worker.c:49-72 -> src/xlating.c:384-414).  Through the per-filter ABI
 * (include/xlating.h) a GPU library cannot know that C callers hold copies of
 * the SAME block, so this header adds the entry points a maintainer binds in
 * sdr_callback/dsp_worker (see INTEGRATION.md): the block is submitted ONCE,
 * staged into HBM with one pinned async copy, converted once, and all clients'
 * NCO-mix + FIR + decimate run as one fused launch
 * (sdr-server_b200/csrc/xlating_kernels.cuh); each dsp thread then only waits
 * for its ticket and writes its own output.
 *
 * Semantics per client are exactly those of include/xlating.h (history, phase
 * recursion, per-call renormalisation, output counts): a client added at stream
 * position P behaves like a reference filter created at that moment (zero
 * history before P), cf. src/xlating.c:543-565.
 *
 * All functions return 0 (or a non-negative ticket) on success and a negative
 * errno-style code on failure, logging "<3>..." to stderr like the reference
 * (src/dsp_worker.c:17).  A group is NOT thread-safe for submit/add/remove
 * (one producer, like the single SDR thread); xlg_wait/xlg_output may be called
 * concurrently from many consumer threads.
 */
#ifndef XLATING_B200_GROUP_H_
#define XLATING_B200_GROUP_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct xlg_group xlg_group;

/* input sample formats = the three SDR front-ends (src/sdr_device.c; cu8 RTL-SDR,
 * cs8 HackRF, cs16 Airspy), and cf32: interleaved float32 (re, im), the format sdr-server
 * writes for a client and the spectrogram tool reads.  The ring holds cf32 values bit for bit,
 * unconverted, so every client, sub-band, bank and spectrum is defined on the submitted samples
 * exactly as for the other formats; the exact float images of a cu8, cs8 or cs16 block
 * ((u - 127.5) * 2^-7, s * 2^-7, s * 2^-15) give bit-identical outputs and rows.  The Q15 path
 * takes no cf32 (XLG_PATH_Q15 with XLG_FMT_CF32: -EINVAL, logged, nothing enqueued).  A host
 * cf32 block needs staging buffers of 4 bytes per element instead of 2: each slot grows its
 * device buffer on its first host cf32 block and its pinned buffer on its first pageable one
 * (-ENOMEM, logged, no ticket, if that allocation fails). */
enum { XLG_FMT_CU8 = 0, XLG_FMT_CS8 = 1, XLG_FMT_CS16 = 2, XLG_FMT_CF32 = 3 };

/* xlg_create flags */
#define XLG_OUT_DEVICE 0x1u    /* leave outputs in HBM (no D2H); xlg_output returns device pointers */
#define XLG_NO_RENORM 0x2u     /* skip the per-call phase renormalisation (AVX variant, src/xlating.c:336-339) */
#define XLG_FORCE_GENERIC 0x4u /* route every client through the generic kernel (testing) */
#define XLG_SM_PARTITION 0x10u /* reserve 8 SMs (CUDA green context) for the oscillator pre-pass so that it
                                  overlaps the FIR of the previous block without fighting it for issue slots;
                                  meant for throughput-bound deployments with many high-rate clients */
#define XLG_TRACK_STATE 0x20u  /* keep every client's state after each ticket (history_offset, oscillator) readable
                                  with the ticket's results: xlg_copy_output(..., state_after).  Used by the
                                  per-filter drop-in engine, which moves filters in and out of a group. */
/* xlg_submit flags */
#define XLG_INPUT_DEVICE 0x100u /* `input` is a device pointer on the group's GPU (already staged), aligned to one
                                   complex sample: 2 bytes for cu8 and cs8, 4 for cs16, 8 for cf32 (a
                                   torch.complex64 tensor's data_ptr() is).  A misaligned one is
                                   refused (-EINVAL, logged) before anything is enqueued; no ticket is taken.
                                   The block may be overwritten once xlg_input_consumed(ticket) (or xlg_wait)
                                   returns. */
#define XLG_PATH_Q15 0x200u     /* Q15 integer path (src/xlating.c:92-140) instead of cf32 */
#define XLG_INPUT_KEEP 0x400u   /* `input` is page-locked host memory that the caller leaves untouched until
                                   xlg_input_consumed(ticket) (or xlg_wait) returns: xlg_submit then returns
                                   without waiting for the H2D copy.  Without this flag a page-locked input may
                                   be reused as soon as xlg_submit returns, exactly like a pageable one (which
                                   is staged through the group's own pinned buffer with a memcpy). */

/* xlg_add_spectrum flags */
#define XLG_SPECTRUM_POWER 0x1u /* rows of linear power v instead of the reference's 10 * log10f(v) dB */

/* depth of the device pipeline (blocks in flight).  Outputs of ticket t stay valid
 * until ticket t + XLG_SLOTS (or t + host_ring, see xlg_create_ex) is submitted;
 * after that xlg_wait / xlg_output return -ESTALE. */
#ifndef XLG_SLOTS
#define XLG_SLOTS 4
#endif

/* One wideband stream on CUDA device `device`.  max_input_len is the largest
 * block, in scalar elements (like create_frequency_xlating_filter's
 * max_input_buffer_length, src/xlating.c:553). */
int xlg_create(int device, uint32_t sampling_freq, uint32_t max_input_len, uint32_t flags, xlg_group **out);
/* Same, with `host_ring` >= XLG_SLOTS result entries kept in pinned host memory: the
 * outputs of ticket t stay readable until ticket t + host_ring is submitted, so a
 * consumer blocked on a slow socket has the slack the reference gets from its
 * per-client queue of queue_size blocks (src/config.c:183, src/queue.c:42-85). */
int xlg_create_ex(int device, uint32_t sampling_freq, uint32_t max_input_len, uint32_t flags, uint32_t host_ring,
                  xlg_group **out);
void xlg_destroy(xlg_group *g);

/* Attach / detach a client.  Arguments as create_frequency_xlating_filter
 * (src/xlating.c:495); `taps` is copied, not adopted.  *client_id is a small
 * non-negative handle, stable until removed. */
int xlg_add_client(xlg_group *g, uint32_t decimation, const float *taps, size_t taps_len,
                   int32_t center_freq, int *client_id);
/* Dynamic state of one client (what src/xlating.c:29,36 keep between calls). */
typedef struct {
  int64_t valid_history; /* add: how many samples before the current stream position this client has really consumed
                            (older ones read as zero for it); ignored on output */
  int64_t hist;          /* history_offset: samples of the stream already consumed that precede its next window */
  float phase_re, phase_im; /* oscillator */
} xlg_client_state;
/* Attach a client that CONTINUES: it has already consumed the last `valid_history` samples of this stream
 * somewhere else (the per-filter ABI) and carries on here with that decimation phase and oscillator.
 * state == NULL is xlg_add_client (a fresh filter: hist = taps_len-1 zeros, oscillator 1+0i). */
int xlg_add_client_ex(xlg_group *g, uint32_t decimation, const float *taps, size_t taps_len, int32_t center_freq,
                      const xlg_client_state *state, int *client_id);
/* Attach a client at the rational rate fs * interp / decim.  It is exactly the reference filter
 * create_frequency_xlating_filter(decim, taps, taps_len, center_freq, interp * fs, ...) fed the
 * zero-stuffed stream u[interp * n] = x[n], u[m] = 0 for every m not divisible by interp: taps,
 * oscillator increment and renormalisation are those of a filter at interp * fs, and its history,
 * window starts and output counts are in upsampled samples.  Taps are designed at interp * fs with
 * gain interp.  Every output k sums only the ceil(taps_len / interp) taps that meet nonzero samples
 * (one polyphase branch), never a stuffed zero.  interp == 1 is xlg_add_client(g, decim, ...).
 * -EINVAL (logged) unless interp, decim >= 1, interp * fs <= UINT32_MAX and
 * interp * max_input_len / 2 < 2^31.  A group with a rational client refuses XLG_PATH_Q15 submits
 * (-ENOTSUP, nothing enqueued).  With XLG_TRACK_STATE, the hist of a rational client is in
 * upsampled samples. */
int xlg_add_client_rational(xlg_group *g, uint32_t interp, uint32_t decim, const float *taps, size_t taps_len,
                            int32_t center_freq, int *client_id);
/* xlg_add_client_rational for a client that CONTINUES, as xlg_add_client_ex is for xlg_add_client: state->hist
 * is in upsampled samples, state->valid_history in input samples (the stream's ring counts those).
 * state == NULL is a fresh client.  -EINVAL for hist < 0, hist > taps_len or valid_history < 0, besides
 * xlg_add_client_rational's checks; interp == 1 is xlg_add_client_ex. */
int xlg_add_client_rational_ex(xlg_group *g, uint32_t interp, uint32_t decim, const float *taps, size_t taps_len,
                               int32_t center_freq, const xlg_client_state *state, int *client_id);
/* Attach a two-stage client: a wide, short first stage at the band rate, then a narrow second stage at
 * fs / decim1, for the transition band of one long filter at a fraction of its multiply-adds (DESIGN.md
 * section 5, "Cascade clients").  Per submitted block its output is, by definition:
 *   stage A = create_frequency_xlating_filter(decim1, taps1, taps1_len, center_freq, fs, ...), fed the block
 *             exactly as an xlg_add_client client is (same history, zero history before the attach point,
 *             oscillator, renormalisation; XLG_NO_RENORM applies);
 *   stage B = the float path (src/xlating.c:52-83) of create_frequency_xlating_filter(decim2, taps2, taps2_len,
 *             0, fs / decim1, ...), fed the cf32 outputs of stage A for the same block, with taps2_len - 1
 *             zeros of history at the attach point.
 * At centre 0 stage B's rotated taps are (h, 0) (cexpf(0) = 1; the even-length reversal quirk of :530-534
 * applies), its oscillator stays 1 + 0i and renormalisation divides by 1, so stage B is exactly a real-tap
 * complex decimator with history.  The client's output per block is stage B's; *out_len is known when
 * xlg_submit returns, as for every client.  xlg_client_info reports kind 5; xlg_cascade_info tells which
 * kernel serves stage A.  -EINVAL (logged) for decim1, decim2, taps1_len or taps2_len of 0, or a stage B
 * too long for the stage-B kernel's shared memory (about 16000 taps); -ENOTSUP (logged) on an
 * XLG_TRACK_STATE group.  A group with a cascade client refuses XLG_PATH_Q15 submits (-ENOTSUP, nothing
 * enqueued). */
int xlg_add_client_cascade(xlg_group *g, uint32_t decim1, const float *taps1, size_t taps1_len, int32_t center_freq,
                           uint32_t decim2, const float *taps2, size_t taps2_len, int *client_id);
/* A cascade client whose stage B resamples by interp2 / decim2, for client rates that do not divide the band
 * rate (DESIGN.md section 5, "Rational cascade clients").  Stage A is xlg_add_client_cascade's.  Stage B is
 * the float path of create_frequency_xlating_filter(decim2, taps2, taps2_len, 0, interp2 * fs / decim1, ...)
 * fed the zero-stuffed stage-A stream of the same block, u[interp2 * n] = y[n] and u[m] = 0 for every other
 * m (as for xlg_add_client_rational), with taps2_len - 1 upsampled zeros of history at the attach point.
 * Every output sums only the ceil(taps2_len / interp2) taps that meet stage-A samples (one polyphase branch),
 * never a stuffed zero.  Taps2 are designed at interp2 * fs / decim1 with gain interp2.  The output rate is
 * fs * interp2 / (decim1 * decim2).  interp2 == 1 is xlg_add_client_cascade (same kernels, same bits).
 * xlg_client_info reports kind 5, and xlg_cascade_info's stage_b_history is in upsampled samples.
 * -EINVAL (logged) for xlg_add_client_cascade's refusals, interp2 of 0, interp2 * (max_input_len / 2 /
 * decim1 + 2) >= 2^31, or a stage B whose branches and one output's window do not fit the stage-B kernel's
 * shared memory; -ENOTSUP (logged) on an XLG_TRACK_STATE group.  Q15 submits are refused as for every
 * cascade client. */
int xlg_add_client_cascade_rational(xlg_group *g, uint32_t decim1, const float *taps1, size_t taps1_len,
                                    int32_t center_freq, uint32_t interp2, uint32_t decim2,
                                    const float *taps2, size_t taps2_len, int *client_id);
int xlg_remove_client(xlg_group *g, int client_id);
/* Extension: sub-band clients (DESIGN.md section 5, "Sub-band clients").  Many narrow clients near each other
 * share one first stage instead of each running its own (a cascade client's stage A).
 *   A SUB-BAND is create_frequency_xlating_filter(decim1, taps1, taps1_len, center_freq, fs, ...), fed the
 *   group's blocks exactly as an xlg_add_client client is (same history, zero history before its attach
 *   point, oscillator, renormalisation; XLG_NO_RENORM applies).  It has no host-visible output, its id comes
 *   from a small-integer space of its own, and xlg_client_count does not count it.  Taps are copied.
 *   -EINVAL (logged) for decim1 or taps1_len of 0, or fs % decim1 != 0 (a member's centre is in Hz at the
 *   integer rate fs / decim1); -ENOTSUP (logged) on an XLG_TRACK_STATE group.  A group with a sub-band refuses
 *   XLG_PATH_Q15 submits (-ENOTSUP, logged, nothing enqueued). */
int xlg_add_subband(xlg_group *g, uint32_t decim1, const float *taps1, size_t taps1_len, int32_t center_freq,
                    int *subband_id);
/* -EBUSY (logged) while the sub-band still has members; -EINVAL for an unknown id. */
int xlg_remove_subband(xlg_group *g, int subband_id);
/* A MEMBER of a sub-band is the float path (src/xlating.c:52-83) of create_frequency_xlating_filter(decim2,
 * taps2, taps2_len, center_offset, fs / decim1, ...), fed the sub-band's cf32 outputs block by block, with
 * taps2_len - 1 zeros of history at the block it is attached before (sub-band samples from before that block
 * read as zero).  center_offset is its centre relative to the sub-band's, in Hz at fs / decim1; the group's
 * XLG_NO_RENORM applies to it as well.  Its output per block is what xlg_output returns for its client id,
 * and *out_len is known when xlg_submit returns.  *client_id is an ordinary client id: xlg_output,
 * xlg_read_output, xlg_copy_output and xlg_remove_client work on it; xlg_client_info reports kind 6.  Taps
 * are copied.  -EINVAL (logged) for decim2 or taps2_len of 0, an unknown sub-band, or taps and a window too
 * long for the member kernel's shared memory (17 * taps2_len + 63 * decim2 <= about 25600). */
int xlg_add_client_subband(xlg_group *g, int subband_id, uint32_t decim2, const float *taps2, size_t taps2_len,
                           int32_t center_offset, int *client_id);
/* Extension: rational members (DESIGN.md section 5, "Rational sub-band members"), for client rates that do not
 * divide fs / decim1.  A rational member is the float path of create_frequency_xlating_filter(decim2, taps2,
 * taps2_len, center_offset, interp2 * fs / decim1, ...), fed the zero-stuffed sub-band stream
 * (u[interp2 * n] = y[n], 0 elsewhere) from the block it is attached before, with taps2_len - 1 upsampled
 * zeros of history.  Every output sums only the ceil(taps2_len / interp2) taps of one polyphase branch, and
 * the output rate is fs * interp2 / (decim1 * decim2); design the taps at interp2 * fs / decim1 with gain
 * interp2.  xlg_add_client_subband is its interp2 = 1 case.  Kind 6 in xlg_client_info; xlg_subband_info's
 * member history is in upsampled samples.  -EINVAL (logged) for interp2 = 0, interp2 * fs / decim1 above
 * UINT32_MAX, interp2 * (max_input_len / 2 / decim1 + 2) >= 2^31, one branch and a window too long for the
 * member kernel's shared memory (17 * ceil(taps2_len / interp2) + 63 * decim2 <= about 25600), and every
 * refusal of xlg_add_client_subband. */
int xlg_add_client_subband_rational(xlg_group *g, int subband_id, uint32_t interp2, uint32_t decim2,
                                    const float *taps2, size_t taps2_len, int32_t center_offset, int *client_id);
/* A member's sub-band, the kind (0, 1 or 2, as xlg_client_info) of the kernel serving the sub-band, and the
 * member's history_offset in sub-band samples (upsampled samples for a rational member).  -EINVAL for any
 * client that is not a member. */
int xlg_subband_info(const xlg_group *g, int client_id, int *subband_id, int *stage_a_kind, size_t *member_history);
/* Extension: bank sub-bands (DESIGN.md section 5, "Bank sub-bands").  A BANK cuts every sub-band fs / (2 * decim1)
 * apart out of the band with one polyphase filter bank, instead of each sub-band running its own first stage.
 *   A bank of decimation D1 and real taps h (taps1, T1 = taps1_len, copied) attached before the next submitted
 *   block, at stream position P, has K = 2 * D1 channels.  Channel k in [-D1, D1) is centred at k * fs / K and
 *   its output m is
 *     y_k[m] = sum_{j < T1} x[s_m + j] * h[T1-1-j] * e^{-2 pi i k (s_m + j - P) / K},
 *   x read as zero before P, s_m and the outputs per block those of an integer client (D1, T1) attached at P
 *   (xlg_add_client's walk).  For odd T1 this is, in exact arithmetic, xlg_add_subband(g, D1, h, T1,
 *   k * fs / K) attached at P.  Bank ids come from a small-integer space of their own.  -EINVAL (logged) for
 *   decim1 or taps1_len of 0, fs % (2 * decim1) != 0, or taps too long for the bank kernel's shared memory
 *   (about 16000 taps, less at large decim1); -ENOTSUP (logged) on an XLG_TRACK_STATE group.  A group with a
 *   bank refuses XLG_PATH_Q15 submits (-ENOTSUP, logged, nothing enqueued). */
int xlg_add_bank(xlg_group *g, uint32_t decim1, const float *taps1, size_t taps1_len, int *bank_id);
/* Materialise channel `channel` of a bank: an ordinary sub-band id.  xlg_add_client_subband[_rational] and
 * xlg_remove_subband work on it unchanged (-EBUSY while it has members); xlg_subband_info reports
 * stage_a_kind 7 for its members.  Its rows are the bank's from P, whenever it is materialised; its members
 * get zero history at their own attach point.  -EINVAL (logged) for an unknown bank or a channel outside
 * [-D1, D1), -EEXIST (logged) for a channel already materialised. */
int xlg_add_bank_subband(xlg_group *g, int bank_id, int32_t channel, int *subband_id);
/* -EBUSY (logged) while the bank still has channels; -EINVAL for an unknown id. */
int xlg_remove_bank(xlg_group *g, int bank_id);
/* Extension: FFT bank sub-bands (DESIGN.md section 5, "FFT banks").  A bank whose channels are defined exactly as
 * xlg_add_bank's (the same P, s_m, zero history and output counts) and whose channel stage is a K-point FFT of
 * each frame's polyphase sums instead of a direct sum per channel: O(K log K) per frame, whatever the number of
 * channels, which makes wide banks affordable.  Only the rounding differs from xlg_add_bank.  Its id comes from
 * the same space as xlg_add_bank's; xlg_add_bank_subband, xlg_remove_bank, xlg_add_client_subband[_rational]
 * and xlg_remove_subband work on it unchanged, xlg_subband_info reports stage_a_kind 8 for its members and
 * xlg_reserve counts its channels as a bank's.  -EINVAL (logged) for decim1 or taps1_len of 0, K = 2 * decim1
 * not a power of two or above 4096, fs % K != 0, or more than max(16 * K, 16384) taps; -ENOTSUP (logged) on an
 * XLG_TRACK_STATE group.  A group with one refuses XLG_PATH_Q15 submits, as for every bank. */
int xlg_add_bank_fft(xlg_group *g, uint32_t decim1, const float *taps1, size_t taps1_len, int *bank_id);
/* Real FP32 instructions of the butterflies of one K-point FFT bank frame (K a power of two): 28 per radix-4
 * butterfly (16 adds and 3 complex products of 4), 4 per radix-2 butterfly.  The planner costs FFT banks by it. */
uint64_t xlg_bank_fft_flops(uint32_t K);
/* Extension: chirp-z bank sub-bands (DESIGN.md section 5, "Chirp-z banks").  A bank of any even K = 2 * decim1
 * up to 4096 whose channels are defined exactly as xlg_add_bank's; only the rounding differs.  A K that
 * xlg_add_bank_fft takes is served exactly as it serves it (the same kernel and rows, stage_a_kind 8).  Every other
 * K runs the chirp-z stage (stage_a_kind 9): each frame's polyphase sums, placed at (p + r_m) mod K as an FFT bank
 * places them, go through Bluestein's algorithm at M = next_pow2(2K - 1) (16 to 8192) in one kernel:
 *   1. a[n] = u[n] c[n] for n < K, a[n] = 0 for K <= n < M, c[n] = e^{-i pi (n^2 mod 2K) / K} (n^2 in 64 bits);
 *   2. A = the M-point FFT of a (the FFT bank's transform at K = M, in position order bank_fft_pos(k, M));
 *   3. Y = A Bh position by position, Bh the chirp-z spectrum's table at W = K (scaled by 1/M);
 *   4. v = the same M-point FFT of conj(Y) in natural order;
 *   5. y_k = c[k mod K] conj(v[k mod K]).
 * c and Bh are computed in double and rounded once (xlg_bank_any_tables); the order of every rounded operation is
 * stated in xlating_kernels.cuh ("Chirp-z banks").  Ids, xlg_add_bank_subband, xlg_remove_bank, members and
 * xlg_reserve work as for every bank.  -EINVAL (logged, nothing changed) for decim1 or taps1_len of 0, K above
 * 4096, fs % K != 0, or more than max(16 * K, 16384) taps; -ENOTSUP (logged) on an XLG_TRACK_STATE group.  A
 * group with one refuses XLG_PATH_Q15 submits, as for every bank.  Its frames count in xlg_bank_fft_profile. */
int xlg_add_bank_any(xlg_group *g, uint32_t decim1, const float *taps1, size_t taps1_len, int *bank_id);
/* The chirp-z bank stage's tables for K (even, at most 4096, not a power of two; else -EINVAL): *m = M, chirp =
 * c[n] as K (re, im) float pairs and kernel = Bh as M pairs in position order, xlg_spectrum_any_tables' tables at
 * width K.  chirp and kernel may be NULL (then only *m is set).  Needs no group and no device. */
int xlg_bank_any_tables(uint32_t K, float *chirp, float *kernel, uint32_t *m);
/* Extension: spectrum rows (DESIGN.md section 5, "Spectrum rows"): the reference spectrogram tool's rows
 * (src/spectrogram/spectrogram.c) of the band, served beside the clients.
 *   A spectrum of width W, frames_per_row F and skip_per_row S attached before the next submitted block, at
 *   stream position P, has period R = F * W + S.  Row r covers the F frames x[P + r R + f W ... + W), f < F; no
 *   frame reads before P.  For each frame, X = DFT_W(frame), c = X * (1/W) (1/W rounded to float once) and
 *   p = c.re^2 + c.im^2 + 1e-20f; the row's value per bin is the max of p over its F frames.  The row is then
 *   half swapped as spectrogram.c:156-163 does: for j < W/2 (rounded down) out[j] = v[W/2 + j] and
 *   out[W/2 + j] = v[j]; for odd W out[W-1] = v[W-1] (not a true fftshift).  Each value is 10 * log10f(v), the
 *   reference's dB row, or v itself with XLG_SPECTRUM_POWER.  The reference tool's rows are F = fs / W and
 *   S = fs % W; its png_util_set_data turns a dB row into 8-bit grey with (int)(dB + 255) clamped to [0, 255].
 *   A row is returned with the ticket whose block holds the row's last frame sample: a block completes zero,
 *   one or many rows, and a row spans as many blocks as it needs.  Removing a spectrum drops its partial row.
 *   W a power of two from 4 to 4096 runs an FFT per frame; any other W up to 4096 a direct DFT of W complex MACs
 *   per input sample.  W = 8192, 16384, 32768 and 65536 (wide spectra) run the same FFT at K = W in two passes:
 *   the first one or two radix-4 stages over the frame, then the rest on each 2048- or 4096-point chunk.  X and
 *   the rows are exactly those of the FFT at K = W (DESIGN.md section 5).  Besides the hold (cap / R + 2 rows of
 *   W floats, cap as for xlg_add_spectrum_ex), the twiddles (W + C float2, C the chunk), the row map (W ints) and,
 *   for a source, its ring (next_pow2(W - 1 + cap) float2), a wide spectrum keeps a scratch of
 *   ((cap - 1) / min(H, W + S) + 1) x W float2 in HBM (H = W here): the most frames a block completes.  A band
 *   spectrum makes the input ring keep W - 1 samples of history.
 *   Spectrum ids come from a small-integer space of their own; xlg_client_count does not count them.
 *   -EINVAL (logged) for W = 0, W above 65536 or above 4096 and not a power of two, F = 0, R >= 2^31 or an unknown
 *   flag; -ENOTSUP (logged) on an XLG_TRACK_STATE group.  A group with a spectrum refuses XLG_PATH_Q15 submits (-ENOTSUP, logged, nothing
 *   enqueued).  Attaching or removing a spectrum changes no client's output. */
int xlg_add_spectrum(xlg_group *g, uint32_t width, uint32_t frames_per_row, uint32_t skip_per_row, uint32_t flags,
                     int *spectrum_id);
/* Spectrum rows of a source's output instead of the band: defined exactly as xlg_add_spectrum's, with x the
 * source's cf32 output stream and P its output position when the next block is submitted (positions count from
 * there, so a spectrum attached with its client, before the client's first block, covers the client's whole output:
 * the reference tool's rows of the file sdr-server writes for it; spectrogram_params(client_rate, W) gives the tool's
 * F and S).  A client's stream is what xlg_output returns for it, ticket after ticket (a cascade client's final
 * row); a sub-band's or a bank channel's (a sub-band id) is its rows at fs / decim1.  The ids, rows, widths, info,
 * profile and removal are xlg_add_spectrum's, and every refusal of xlg_add_spectrum applies; -EINVAL (logged) for
 * an unknown client or sub-band id.  While a spectrum reads it, xlg_remove_client and xlg_remove_subband return
 * -EBUSY (logged) for its source (and a bank with channels cannot be removed).  Attaching or removing one changes
 * no client's output and no band spectrum's rows. */
int xlg_add_client_spectrum(xlg_group *g, int client_id, uint32_t width, uint32_t frames_per_row,
                            uint32_t skip_per_row, uint32_t flags, int *spectrum_id);
int xlg_add_subband_spectrum(xlg_group *g, int subband_id, uint32_t width, uint32_t frames_per_row,
                             uint32_t skip_per_row, uint32_t flags, int *spectrum_id);
/* Windowed, overlapped and averaged spectra (Welch's method), of the band, a client or a sub-band (source, and
 * source_id as for xlg_add_client_spectrum / xlg_add_subband_spectrum; ignored for the band).  The definition is
 * xlg_add_spectrum's with three more parameters:
 *   hop H >= 1 (0 means W): row period R = (F - 1) * H + W + S; row r covers the frames x[P + r R + f H ... + W),
 *     f < F, so frames overlap by W - H samples when H < W.  With H = W this is xlg_add_spectrum's.
 *   window w[0..W) (copied; NULL: none): each frame is z[n] = (x[n].re * w[n], x[n].im * w[n]), one rounded float
 *     multiply each, before the DFT.  No window is bit for bit a window of ones.
 *   reduce: XLG_SPECTRUM_MAX, the max of p over the row's frames as above, or XLG_SPECTRUM_MEAN: s = +0, then
 *     s = s + p_f for f = 0 .. F - 1 in frame order (one rounded float add each), v = s / float(F) (float(F)
 *     rounded to nearest, the division correctly rounded).
 * p, the half swap, dB or linear power and the ticket a row comes with (the one whose block holds the row's last
 * frame sample, P + r R + (F - 1) H + W - 1) are xlg_add_spectrum's.  With a window w W / sum(w), mean rows are
 * scipy.signal.welch(x, window, nperseg=W, noverlap=W-H, detrend=False, return_onesided=False,
 * scaling="spectrum") + 1e-20, up to float32 rounding and before the half swap.
 * Ids, rows, widths, info, profile, removal and the sources' -EBUSY rules are xlg_add_spectrum's; xlg_reserve
 * counts a spectrum's rows with this R.  A desc with H = W, no window and the max is served exactly as
 * xlg_add_spectrum.  A mean spectrum keeps a frame buffer of ((cap - 1) / min(H, W + S) + 1) x W floats in HBM,
 * cap being max_input_len/2 or the source's row capacity: the most frames a block completes.  A wide spectrum
 * (W from 8192 to 65536, a power of two) keeps its scratch of as many rows of W float2 as well, and a window
 * W floats.
 * -EINVAL (logged, nothing changed) for every refusal of xlg_add_spectrum, a NULL desc, an unknown source, client
 * or sub-band id, 8 H < W (more than 7/8 overlap), R >= 2^31, a window weight that is not finite or an unknown
 * reduce; -ENOTSUP (logged) on an XLG_TRACK_STATE group. */
enum { XLG_SPECTRUM_MAX = 0, XLG_SPECTRUM_MEAN = 1 };                        /* xlg_spectrum_desc.reduce */
enum { XLG_SOURCE_BAND = 0, XLG_SOURCE_CLIENT = 1, XLG_SOURCE_SUBBAND = 2 }; /* xlg_add_spectrum_ex source */
typedef struct {
  uint32_t width, frames_per_row, skip_per_row, flags; /* as xlg_add_spectrum (flags: XLG_SPECTRUM_POWER) */
  uint32_t hop;        /* samples from one frame's start to the next within a row; 0 means width */
  uint32_t reduce;     /* XLG_SPECTRUM_MAX or XLG_SPECTRUM_MEAN */
  const float *window; /* width weights, copied; NULL: none */
} xlg_spectrum_desc;
int xlg_add_spectrum_ex(xlg_group *g, int source, int source_id, const xlg_spectrum_desc *desc, int *spectrum_id);
/* Spectra of any width W from 1 to 65536 (DESIGN.md section 5, "Chirp-z spectra"): the arguments, ids, rows,
 * widths, profile, removal and refusals of xlg_add_spectrum_ex, except its width rule; W = 0 and W above 65536
 * are still refused (-EINVAL, logged, nothing changed).  A width that xlg_add_spectrum_ex serves (W <= 4096, or a
 * power of two up to 65536) is served exactly as xlg_add_spectrum_ex serves it: the same kernels, rows and
 * xlg_spectrum_info kernel.  Every other width runs the chirp-z stage (xlg_spectrum_info kernel 3).  Its rows are
 * xlg_add_spectrum_ex's (frames, hop, window, max or mean, p with its 1/W, hold, half swap, dB or linear) with the
 * W-point DFT X of each windowed frame z computed by Bluestein's algorithm at M = next_pow2(2W - 1):
 *   1. a[n] = z[n] c[n] for n < W, a[n] = 0 for W <= n < M, c[n] = e^{-i pi (n^2 mod 2W) / W} (n^2 in 64 bits);
 *   2. A = the M-point FFT of a (the FFT path's transform at K = M, in position order bank_fft_pos(k, M));
 *   3. Y = A Bh position by position, Bh the M-point DFT of b[m] = e^{+i pi (m^2 mod 2W) / W}, |m| < W, wrapped
 *      mod M and scaled by 1/M;
 *   4. v = the same M-point FFT of conj(Y) in natural order, so X_k = conj(v[k]) c[k] for k < W.
 *   Since |c[k]| = 1, p is defined on v[k] itself, p = (v.re / W)^2 + (v.im / W)^2 + 1e-20f as for every spectrum,
 *   with no final chirp.  c and Bh are computed in double and rounded once to float (xlg_spectrum_any_tables); the
 *   order of every rounded operation is stated in xlating_kernels.cuh ("Chirp-z spectra").
 * Besides what an extended spectrum holds (the hold, the row map of W ints, a source's ring, a window, a mean's
 * frame buffer), a chirp-z spectrum keeps the twiddles, the chirp and Bh ((2 M + C + W) float2, C = M / 16 or
 * M / 4 at M = 16384), the bin of each position (M ints) and two scratches of fb x M float2 in HBM,
 * fb = (cap - 1) / min(H, W + S) + 1 the most frames a block completes: at W = 65535 (M = 131072), 2 MiB per
 * frame.  Its frame costs channel_flops of 2 xlg_bank_fft_flops(M) + 4 W + 4 M + 6 W (the two transforms, the
 * chirp's and Bh's complex products of 4 instructions, the power), plus 2 W windowed and W for a mean. */
int xlg_add_spectrum_any(xlg_group *g, int source, int source_id, const xlg_spectrum_desc *desc, int *spectrum_id);
/* The chirp-z stage's tables for width W (above 4096, at most 65536, not a power of two; else -EINVAL): *m = M,
 * chirp = c[n] as W (re, im) float pairs and kernel = Bh as M pairs in position order (kernel[bank_fft_pos(k, M)]
 * is Bh[k]).  chirp and kernel may be NULL (then only *m is set).  Needs no group and no device. */
int xlg_spectrum_any_tables(uint32_t width, float *chirp, float *kernel, uint32_t *m);
/* Drops its partial row.  -EINVAL for an unknown id. */
int xlg_remove_spectrum(xlg_group *g, int spectrum_id);
/* The rows a spectrum completed in a ticket: *n_rows x W contiguous floats, in pinned host memory, or in HBM for
 * XLG_OUT_DEVICE groups (valid as xlg_output's).  *n_rows is known when xlg_submit returns.  -EINVAL for a
 * spectrum that was not attached when the ticket was submitted. */
int xlg_spectrum_output(xlg_group *g, int64_t ticket, int spectrum_id, const float **rows, size_t *n_rows);
/* The width W of a ticket's rows of a spectrum: the width the id had when the ticket was submitted (an id freed by
 * xlg_remove_spectrum may come back with another width).  -EINVAL as xlg_spectrum_output. */
int xlg_spectrum_width(xlg_group *g, int64_t ticket, int spectrum_id, uint32_t *width);
/* Waits for the ticket and copies at most cap_rows of its rows (xlg_spectrum_width floats each) into dst;
 * *n_rows = rows it has. */
int xlg_read_spectrum(xlg_group *g, int64_t ticket, int spectrum_id, float *dst, size_t cap_rows, size_t *n_rows);
/* The channel stage serving a spectrum (0 = direct DFT, 1 = FFT, 2 = wide FFT, W above 4096, 3 = chirp-z,
 * xlg_add_spectrum_any above 4096 and not a power of two) and the rows completed by the blocks submitted so far. */
int xlg_spectrum_info(const xlg_group *g, int spectrum_id, int *kernel, uint64_t *rows_done);
/* Size the per-ticket result arenas (device and pinned host) for `output_samples_per_block` complex output
 * samples per block summed over all clients (a client at decimation D produces about max_input_len/2/D + 2).
 * A cascade client counts two rows, each rounded up to a multiple of 4 samples: its stage-A row of
 * n1 = max_input_len/2/decim1 + 2 samples, which stays on the device, and its final row of
 * floor(n1 * interp2 / decim2) + 2 (interp2 = 1 for xlg_add_client_cascade).  A sub-band counts one row of
 * n1 = max_input_len/2/decim1 + 2 samples, rounded up to 4, which stays on the device (a bank's channel counts
 * one row like a sub-band); a member counts its
 * final row of floor(n1 * interp2 / decim2) + 2, rounded up to 4 (interp2 = 1 for xlg_add_client_subband).
 * A spectrum counts ceil((max_input_len/2/R + 1) * W / 2) samples, rounded up to 4: room for its rows of W floats.
 * A spectrum of a source (xlg_add_client_spectrum, xlg_add_subband_spectrum) counts the same with max_input_len/2
 * replaced by its source's row capacity: out_cap = max_input_len/2 * L / D + 2 for a client, the final row's
 * floor(out_cap * interp2 / decim2) + 2 for a cascade, n1 for a sub-band or bank channel, a member's final row for
 * a sub-band member.
 * Optional: the arenas grow on demand when clients are added, but a growth re-allocates every ring entry and
 * the results still waiting in the ring are lost (-ESTALE for consumers that had not read them yet, like a
 * block overwritten in the reference's queue).  A server that knows its client limit reserves once, up front. */
int xlg_reserve(xlg_group *g, size_t output_samples_per_block);
int xlg_client_count(const xlg_group *g);

/* Submit one block for ALL clients.  `input_len` in scalar elements.  Returns a
 * ticket (0,1,2,...) immediately; work proceeds asynchronously.  Blocks when
 * XLG_SLOTS tickets are already in flight and the oldest has not completed. */
int64_t xlg_submit(xlg_group *g, int fmt, const void *input, size_t input_len, uint32_t flags);

/* Block until the group has read ticket's input block: its H2D copy for a host block (what XLG_INPUT_KEEP submits
 * wait for), its conversion for an XLG_INPUT_DEVICE block (which may then be reused, also by work on another
 * stream).  Returns at once for a block of no complex sample, and for a ticket whose slot a later ticket already
 * uses (its input was read long ago).  -EINVAL for a ticket not yet submitted. */
int xlg_input_consumed(xlg_group *g, int64_t ticket);

/* Block until ticket's outputs are complete (in pinned host memory, or in HBM
 * with XLG_OUT_DEVICE). */
int xlg_wait(xlg_group *g, int64_t ticket);

/* Output of one client for a completed ticket: cf32 (interleaved float re,im) or,
 * for XLG_PATH_Q15 tickets, int16 re,im pairs.  *out_len counts complex samples
 * and is available right after xlg_submit returns (it is computed on the host). */
int xlg_output(xlg_group *g, int64_t ticket, int client_id, const void **out, size_t *out_len);

/* Copy one client's output of a completed ticket into caller memory (cf32 pairs, or
 * int16 pairs for XLG_PATH_Q15 tickets): waits for the ticket, then copies at most
 * `cap` complex samples from wherever the result lives -- the pinned host arena, or
 * HBM for XLG_OUT_DEVICE groups (a synchronous D2H copy: verification and tools, not
 * the data path).  *out_len = complex samples the client produced. */
int xlg_read_output(xlg_group *g, int64_t ticket, int client_id, void *dst, size_t cap, size_t *out_len);

/* Same copy for a ticket the caller KNOWS to be complete (it, or another thread, returned from xlg_wait):
 * makes no CUDA call, so hundreds of consumer threads can call it per block without queueing on the
 * CUDA context.  Host-output groups only.  With XLG_TRACK_STATE, *state_after (may be NULL) receives the
 * client's history_offset and oscillator after this ticket.  -ESTALE if the ring entry was recycled. */
int xlg_copy_output(xlg_group *g, int64_t ticket, int client_id, void *dst, size_t cap, size_t *out_len,
                    xlg_client_state *state_after);

/* Pinned host memory for input blocks (queue/ingest buffers, SURVEY 8f-2). */
void *xlg_alloc_pinned(size_t bytes);
void xlg_free_pinned(void *p);

/* Make the group's work wait for everything already enqueued on an external
 * CUDA stream (e.g. the torch/NCCL stream that produced a device input).  Every
 * call made since the last xlg_submit is honoured by the next one, so a block
 * produced on several streams takes one call per stream.  Nothing is enqueued
 * on the caller's stream. */
int xlg_wait_stream(xlg_group *g, void *cuda_stream);

/* SMs currently reserved for the oscillator pre-pass (0 = no partition active).  With XLG_SM_PARTITION the group
 * decides per client layout whether the reservation pays (it does when the pre-pass chain would otherwise pace the
 * pipeline); XLATING_B200_PARTITION=0/1 forces the answer. */
int xlg_partition_active(xlg_group *g);

/* Device-side timing of a region of submits: xlg_timer_start drains the group
 * and records a start event; xlg_timer_stop records an end event that depends
 * on all work submitted so far, synchronises and returns elapsed milliseconds. */
int xlg_timer_start(xlg_group *g);
int xlg_timer_stop(xlg_group *g, float *elapsed_ms);

/* Per-kernel profiling (CUDA events around each launch on its own stream).
 * Counters accumulate while enabled and are harvested by xlg_wait. */
typedef struct {
  double fir_tile_ms;    /* tiled multi-client FIR kernel (dominant) */
  double fir_generic_ms; /* generic split-K FIR kernel */
  double phase_ms;       /* oscillator pre-pass */
  double convert_ms;     /* raw -> cf32 ring */
  uint64_t fir_tile_launches, fir_generic_launches, phase_launches, convert_launches;
  uint64_t blocks;       /* submitted blocks accounted */
  uint64_t out_samples;  /* complex outputs produced (all clients) */
  uint64_t in_samples;   /* complex inputs consumed */
  uint64_t tile_macs;    /* complex MACs issued by the tiled kernel incl. padding */
  uint64_t algo_macs;    /* algorithmic complex MACs: sum n_out * taps_len */
  /* host side of xlg_submit (always counted, also with profiling off) */
  double fir_long_ms;    /* split-K long-filter FIR + ordered reduction (both kernels) */
  uint64_t fir_long_launches;
  double host_submit_ms; /* wall time spent inside xlg_submit, including ...          */
  double host_wait_ms;   /* ... the part spent waiting for a free slot (GPU is behind) */
  uint64_t submits;
} xlg_profile;
int xlg_profile_enable(xlg_group *g, int on);
int xlg_profile_read(xlg_group *g, xlg_profile *p, int reset);

/* Kernels of rational clients (xlg_add_client_rational), counted like xlg_profile's while profiling
 * is enabled.  xlg_profile's algo_macs counts n_out * ceil(taps_len / interp) for them. */
typedef struct {
  double fir_poly_tile_ms;    /* tiled classes: the tiled FIR over their polyphase branches + the placement */
  double fir_poly_generic_ms; /* polyphase generic FIR kernel */
  uint64_t fir_poly_tile_launches, fir_poly_generic_launches;
  uint64_t poly_macs;         /* complex MACs of rational clients: sum n_out * ceil(taps_len / interp) */
} xlg_poly_profile;
int xlg_poly_profile_read(xlg_group *g, xlg_poly_profile *p, int reset);

/* Stage B of cascade clients (xlg_add_client_cascade, _rational), counted like xlg_profile's while profiling
 * is enabled.  xlg_profile counts each cascade client's stage A as the integer client it is. */
typedef struct {
  double stage_b_ms;         /* the ring appends + the stage-B kernels (integer and rational) */
  uint64_t stage_b_launches;
  uint64_t stage_b_macs;     /* complex-by-real MACs of stage B: sum n_out * ceil(taps2_len / interp2) */
  uint64_t d2h_bytes;        /* result bytes copied to the host, all clients (stage-A rows are never copied) */
} xlg_cascade_profile;
int xlg_cascade_profile_read(xlg_group *g, xlg_cascade_profile *p, int reset);

/* Sub-band members (xlg_add_client_subband), counted like xlg_profile's while profiling is enabled.
 * xlg_profile counts each sub-band's first stage once, as the integer client it is. */
typedef struct {
  double member_ms;          /* the sub-band ring appends, the member oscillators and the member kernel */
  uint64_t member_launches;
  uint64_t member_macs;      /* complex MACs of the members: sum n2 * ceil(taps2_len / interp2) */
  uint64_t row_samples;      /* sub-band samples produced (and appended to the rings) */
} xlg_subband_profile;
int xlg_subband_profile_read(xlg_group *g, xlg_subband_profile *p, int reset);

/* Banks (xlg_add_bank), counted like xlg_profile's while profiling is enabled.  xlg_profile does not count
 * banks; their channels' ring appends and members are xlg_subband_profile's. */
typedef struct {
  double bank_ms;            /* the bank kernel */
  uint64_t bank_launches;
  uint64_t poly_macs;        /* real-by-complex MACs of the polyphase sums: sum n1 * T1 */
  uint64_t dft_macs;         /* complex MACs of the channel sums: sum n1 * C * K, C materialised channels */
} xlg_bank_profile;
int xlg_bank_profile_read(xlg_group *g, xlg_bank_profile *p, int reset);

/* FFT and chirp-z banks (xlg_add_bank_fft, xlg_add_bank_any), counted like xlg_profile's while profiling is
 * enabled.  xlg_bank_profile counts direct banks only. */
typedef struct {
  double fft_ms;             /* the FFT and chirp-z bank kernels (one span per block) */
  uint64_t fft_launches;
  uint64_t poly_macs;        /* real-by-complex MACs of the polyphase sums: sum n1 * T1 */
  uint64_t butterfly_flops;  /* real FP32 instructions of the butterflies: sum n1 * xlg_bank_fft_flops(K); a
                                chirp-z bank of C materialised channels n1 * (2 xlg_bank_fft_flops(M) + 4 K + 4 M
                                + 4 C) (the two transforms, the chirp's, Bh's and the final chirp's products) */
} xlg_bank_fft_profile;
int xlg_bank_fft_profile_read(xlg_group *g, xlg_bank_fft_profile *p, int reset);

/* Spectra (xlg_add_spectrum), counted like xlg_profile's while profiling is enabled. */
typedef struct {
  double spectrum_ms;        /* the channel stages, the mean's fold and the emit pass */
  uint64_t spectrum_launches;
  uint64_t frames;           /* W-point frames transformed (overlapped frames each count) */
  uint64_t channel_flops;    /* FP32 instructions of the channel stages: per frame xlg_bank_fft_flops(W) + 6 W on
                                the FFT path, 4 W^2 + 6 W on the direct path (an fmaf counts one); 2 W more for a
                                windowed spectrum's frame and W more for a mean spectrum's (the fold's adds); a
                                chirp-z frame 2 xlg_bank_fft_flops(M) + 4 W + 4 M + 6 W (xlg_add_spectrum_any) */
} xlg_spectrum_profile;
int xlg_spectrum_profile_read(xlg_group *g, xlg_spectrum_profile *p, int reset);

/* Introspection for tests: history length (src/xlating.c:29 history_offset; upsampled samples for a
 * rational client, stage A's for a cascade client) and which kernel currently serves the client
 * (0 = generic, 1 = tiled, 2 = long-filter split-K, 3 = rational, polyphase generic, 4 = rational, tiled: at
 * least 8 clients with identical (interp, decim, taps_len, window alignment), gcd(interp, decim) = 1, whose
 * branches fit the tiled kernel's shared memory, 5 = cascade, 6 = sub-band member; 7, as a sub-band's kind in
 * xlg_subband_info only, = a bank's channel, 8 likewise = an FFT bank's channel). */
int xlg_client_info(const xlg_group *g, int client_id, size_t *history, int *kernel_kind);
/* A cascade client's stages: the kind (0, 1 or 2, as xlg_client_info) of the kernel serving stage A, and the
 * history_offset of each stage (stage B's in stage-A samples, upsampled by interp2 for a rational cascade
 * client).  -EINVAL for any other client. */
int xlg_cascade_info(const xlg_group *g, int client_id, int *stage_a_kind, size_t *stage_a_history,
                     size_t *stage_b_history);

/* Counters of the per-filter drop-in ABI (include/xlating.h) on `device`: process_*
 * calls served so far, the number of launches (batches) they were combined into, and
 * how many of them found their input already staged by another filter's call (the
 * reference's per-client copies of one SDR block, src/queue.c:114).  -ENOENT before
 * the first filter was created there. */
int xlg_dropin_stats(int device, uint64_t *batches, uint64_t *calls, uint64_t *shared_inputs);

/* Counters of the drop-in engine's stream overlay on `device` (csrc/stream_overlay.h): stats7[0] process_*
 * calls served by a band's batch group, [1] blocks published (submitted once for all member filters),
 * [2] calls that found their block already published, [3] filters that fell out of step and left a group,
 * [4] filters that joined one, [5] private calls whose block was in the log, [6] filters that are members now. */
int xlg_dropin_stream_stats(int device, uint64_t *stats7);
/* Where the served calls' time went, nanoseconds summed over all calling threads: ns7[0] whole calls served by a
 * group, [1] copying the caller's row out of the result ring, [2] comparing the caller's bytes with the log
 * entry, [3] sleeping until the block's results were readable, and for the publishing callers [4] copying the
 * block into the log, [5] the group submit, [6] waiting for the GPU. */
int xlg_dropin_stream_times(int device, uint64_t *ns7);

#ifdef __cplusplus
}
#endif
#endif /* XLATING_B200_GROUP_H_ */
