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
 * cs8 HackRF, cs16 Airspy) */
enum { XLG_FMT_CU8 = 0, XLG_FMT_CS8 = 1, XLG_FMT_CS16 = 2 };

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
#define XLG_INPUT_DEVICE 0x100u /* `input` is a device pointer on the group's GPU (already staged) */
#define XLG_PATH_Q15 0x200u     /* Q15 integer path (src/xlating.c:92-140) instead of cf32 */
#define XLG_INPUT_KEEP 0x400u   /* `input` is page-locked host memory that the caller leaves untouched until
                                   xlg_input_consumed(ticket) (or xlg_wait) returns: xlg_submit then returns
                                   without waiting for the H2D copy.  Without this flag a page-locked input may
                                   be reused as soon as xlg_submit returns, exactly like a pageable one (which
                                   is staged through the group's own pinned buffer with a memcpy). */

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
int xlg_remove_client(xlg_group *g, int client_id);
/* Size the per-ticket result arenas (device and pinned host) for `output_samples_per_block` complex output
 * samples per block summed over all clients (a client at decimation D produces about max_input_len/2/D + 2).
 * A cascade client counts two rows, each rounded up to a multiple of 4 samples: its stage-A row of
 * n1 = max_input_len/2/decim1 + 2 samples, which stays on the device, and its final row of n1/decim2 + 2.
 * Optional: the arenas grow on demand when clients are added, but a growth re-allocates every ring entry and
 * the results still waiting in the ring are lost (-ESTALE for consumers that had not read them yet, like a
 * block overwritten in the reference's queue).  A server that knows its client limit reserves once, up front. */
int xlg_reserve(xlg_group *g, size_t output_samples_per_block);
int xlg_client_count(const xlg_group *g);

/* Submit one block for ALL clients.  `input_len` in scalar elements.  Returns a
 * ticket (0,1,2,...) immediately; work proceeds asynchronously.  Blocks when
 * XLG_SLOTS tickets are already in flight and the oldest has not completed. */
int64_t xlg_submit(xlg_group *g, int fmt, const void *input, size_t input_len, uint32_t flags);

/* Block until the H2D copy of ticket's input block has completed (XLG_INPUT_KEEP submits). */
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
 * CUDA stream (e.g. the torch/NCCL stream that produced a device input). */
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

/* Stage B of cascade clients (xlg_add_client_cascade), counted like xlg_profile's while profiling is enabled.
 * xlg_profile counts each cascade client's stage A as the integer client it is. */
typedef struct {
  double stage_b_ms;         /* the ring appends + the stage-B kernel */
  uint64_t stage_b_launches;
  uint64_t stage_b_macs;     /* complex-by-real MACs of stage B: sum n_out * taps2_len */
  uint64_t d2h_bytes;        /* result bytes copied to the host, all clients (stage-A rows are never copied) */
} xlg_cascade_profile;
int xlg_cascade_profile_read(xlg_group *g, xlg_cascade_profile *p, int reset);

/* Introspection for tests: history length (src/xlating.c:29 history_offset; upsampled samples for a
 * rational client, stage A's for a cascade client) and which kernel currently serves the client
 * (0 = generic, 1 = tiled, 2 = long-filter split-K, 3 = rational, polyphase generic, 4 = rational, tiled: at
 * least 8 clients with identical (interp, decim, taps_len, window alignment), gcd(interp, decim) = 1, whose
 * branches fit the tiled kernel's shared memory, 5 = cascade). */
int xlg_client_info(const xlg_group *g, int client_id, size_t *history, int *kernel_kind);
/* A cascade client's stages: the kind (0, 1 or 2, as xlg_client_info) of the kernel serving stage A, and the
 * history_offset of each stage (stage B's in stage-A samples).  -EINVAL for any other client. */
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
