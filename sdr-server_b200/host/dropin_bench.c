/*
 * host/dropin_bench.c -- the UNMODIFIED reference threading model on the drop-in ABI:
 * one filter and one dsp thread per client (src/dsp_worker.c:41-88), every thread
 * processing its own private copy of the same block sequence (src/queue.c:114), no
 * batch binding.  Measures what sdr-server gets by only re-linking against
 * libxlating_b200.so (INTEGRATION.md section 1).
 *
 * usage: dropin_bench <clients> <blocks> [window [warmup_blocks [rational]]]
 *
 * Default workload: 2.016 Msps cu8, 48/96 ksps clients mixed.  With `rational` as the fifth argument:
 * 48 ksps clients of a 2.048 Msps cu8 stream, each a rational 3/128 filter
 * (create_rational_frequency_xlating_filter) with taps designed at 3 x 2.048 MHz with gain 3.
 *
 * The timed region starts after `warmup_blocks` (default 16) blocks have gone through the same
 * threads: a server's one-time start-up work -- the first CUDA call of every dsp thread, the
 * page-locked result ring of the band's batch group (hundreds of MB for hundreds of clients),
 * filters joining the group -- is not what this measures.
 *
 * window = 0: every dsp thread free-runs through its blocks (pure throughput).
 * window = W > 0: an SDR thread delivers block b to all clients at once, and only after
 * every client has finished block b - W: per-client queues of W blocks with
 * back-pressure instead of the reference's drop-newest (src/queue.c:90-94).
 */
#include <pthread.h>
#include <semaphore.h>
#include <stdatomic.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <time.h>

#include "lpf.h"
#include "xlating.h"
#include "xlating_group.h"

#define BLOCK 262144

static int g_window = 0, g_clients = 0, g_blocks = 0, g_warmup = 16;
static pthread_barrier_t g_warm_barrier; /* all dsp threads + main: end of warm-up = start of the timed region */
/* the SDR thread: block p is delivered to every client queue (one semaphore per
 * client, like the reference's one mutex + condition per queue, src/queue.c:87-112) once
 * all clients have finished block p - window */
static sem_t *g_queue;      /* per client: blocks delivered and not yet taken */
static sem_t g_sdr;         /* posted when some block has been finished by every client */
static atomic_int *g_finished; /* per block: clients that are done with it */

static void *sdr_thread(void *arg) {
  (void)arg;
  for (int p = 0; p < g_blocks; p++) {
    if (p >= g_window) sem_wait(&g_sdr); /* block p - window is complete (they complete in order) */
    for (int c = 0; c < g_clients; c++) sem_post(&g_queue[c]);
  }
  return NULL;
}

static void wait_for_block(int id) { sem_wait(&g_queue[id]); }

static void finished_block(int b) {
  if (atomic_fetch_add(&g_finished[b], 1) + 1 == g_clients) sem_post(&g_sdr);
}

typedef struct {
  int id;
  xlating *filter;
  uint8_t *blocks[4]; /* private copies, like the per-client queue nodes */
  int n_blocks;
  uint64_t outputs;
} client_t;

static void *dsp_thread(void *arg) {
  client_t *c = (client_t *)arg;
  xlating_cf32 *out = NULL;
  size_t n = 0;
  for (int b = 0; b < c->n_blocks; b++) {
    if (b == g_warmup) {
      pthread_barrier_wait(&g_warm_barrier); /* everybody has finished the warm-up blocks */
      pthread_barrier_wait(&g_warm_barrier); /* main has taken t0 */
      c->outputs = 0;
    }
    if (g_window > 0) wait_for_block(c->id);
    /* every SDR block is new data, and every client holds the same bytes of it */
    memcpy(c->blocks[b % 4] + 64, &b, sizeof(b));
    process_native_cu8_cf32(c->blocks[b % 4], BLOCK, &out, &n, c->filter);
    c->outputs += n;
    if (g_window > 0) finished_block(b);
  }
  return NULL;
}

int main(int argc, char **argv) {
  const int n_clients = argc > 1 ? atoi(argv[1]) : 64;
  const int n_blocks = argc > 2 ? atoi(argv[2]) : 50;
  g_window = argc > 3 ? atoi(argv[3]) : 0;
  g_warmup = argc > 4 ? atoi(argv[4]) : 16;
  if (g_warmup < 1) g_warmup = 1;
  const int rational = argc > 5 && strcmp(argv[5], "rational") == 0;
  g_clients = n_clients;
  g_blocks = n_blocks + g_warmup; /* warm-up blocks first, then the timed ones */
  pthread_barrier_init(&g_warm_barrier, NULL, (unsigned)n_clients + 1);
  g_finished = (atomic_int *)calloc((size_t)g_blocks, sizeof(atomic_int));
  g_queue = (sem_t *)calloc((size_t)n_clients, sizeof(sem_t));
  for (int c = 0; c < n_clients; c++) sem_init(&g_queue[c], 0, 0);
  sem_init(&g_sdr, 0, 0);
  const uint32_t fs = rational ? 2048000 : 2016000;
  const uint32_t interp = 3, decim = 128; /* rational: 2.048 MHz * 3 / 128 = 48 kHz */
  uint8_t *master[4];
  uint64_t s = 0x9E3779B97F4A7C15ull;
  for (int i = 0; i < 4; i++) {
    master[i] = (uint8_t *)malloc(BLOCK);
    for (int j = 0; j < BLOCK; j++) {
      s ^= s << 13;
      s ^= s >> 7;
      s ^= s << 17;
      master[i][j] = (uint8_t)s;
    }
  }
  client_t *clients = (client_t *)calloc((size_t)n_clients, sizeof(client_t));
  for (int c = 0; c < n_clients; c++) {
    const uint32_t rate = (rational || c % 2 == 0) ? 48000 : 96000;
    float *taps = NULL;
    size_t len = 0;
    const int32_t center = (int32_t)(-(int32_t)fs / 2 + (int32_t)rate / 2 +
                                     (int64_t)c * (fs - rate) / (n_clients > 1 ? n_clients - 1 : 1));
    int rc;
    if (rational) {
      if (create_low_pass_filter((float)interp, interp * fs, rate / 2, rate / 5, &taps, &len) != 0) return 1;
      rc = create_rational_frequency_xlating_filter(interp, decim, taps, len, center, fs, BLOCK, &clients[c].filter);
    } else {
      if (create_low_pass_filter(1.0f, fs, rate / 2, rate / 5, &taps, &len) != 0) return 1;
      rc = create_frequency_xlating_filter(fs / rate, taps, len, center, fs, BLOCK, &clients[c].filter);
    }
    if (rc != 0) {
      fprintf(stderr, "create failed for client %d\n", c);
      return 1;
    }
    for (int i = 0; i < 4; i++) {
      clients[c].blocks[i] = (uint8_t *)malloc(BLOCK);
      memcpy(clients[c].blocks[i], master[i], BLOCK);
    }
    clients[c].n_blocks = g_blocks;
    clients[c].id = c;
  }
  /* warm-up: one block each, sequentially */
  for (int c = 0; c < n_clients; c++) {
    xlating_cf32 *out = NULL;
    size_t n = 0;
    process_native_cu8_cf32(clients[c].blocks[0], BLOCK, &out, &n, clients[c].filter);
  }
  pthread_t *threads = (pthread_t *)malloc(sizeof(pthread_t) * (size_t)n_clients);
  struct timespec t0, t1;
  pthread_t sdr;
  for (int c = 0; c < n_clients; c++) pthread_create(&threads[c], NULL, dsp_thread, &clients[c]);
  if (g_window > 0) pthread_create(&sdr, NULL, sdr_thread, NULL);
  pthread_barrier_wait(&g_warm_barrier);
  uint64_t st0[7] = {0, 0, 0, 0, 0, 0, 0}, ns0[7] = {0, 0, 0, 0, 0, 0, 0}, batches0 = 0, calls0 = 0, shared0 = 0;
  xlg_dropin_stats(0, &batches0, &calls0, &shared0);
  xlg_dropin_stream_stats(0, st0);
  xlg_dropin_stream_times(0, ns0);
  clock_gettime(CLOCK_MONOTONIC, &t0);
  pthread_barrier_wait(&g_warm_barrier);
  for (int c = 0; c < n_clients; c++) pthread_join(threads[c], NULL);
  if (g_window > 0) pthread_join(sdr, NULL);
  clock_gettime(CLOCK_MONOTONIC, &t1);
  const double dt = (double)(t1.tv_sec - t0.tv_sec) + 1e-9 * (double)(t1.tv_nsec - t0.tv_nsec);
  uint64_t outputs = 0;
  for (int c = 0; c < n_clients; c++) outputs += clients[c].outputs;
  uint64_t batches = 0, calls = 0, shared = 0;
  xlg_dropin_stats(0, &batches, &calls, &shared); /* stays 0 with XLATING_B200_DROPIN=group */
  batches -= batches0;
  calls -= calls0;
  shared -= shared0;
  uint64_t st[7] = {0, 0, 0, 0, 0, 0, 0};
  xlg_dropin_stream_stats(0, st); /* the band's stream overlay (csrc/stream_overlay.h) */
  uint64_t ns[7] = {0, 0, 0, 0, 0, 0, 0};
  xlg_dropin_stream_times(0, ns);
  for (int i = 0; i < 6; i++) st[i] -= st0[i]; /* st[6] = members now */
  for (int i = 0; i < 7; i++) ns[i] -= ns0[i];
  if (st[0] > 0 && st[1] > 0)
    fprintf(stderr, "overlay: per served call %.1f us (compare %.1f, wait for the block %.1f, copy out %.1f); per published "
                    "block: copy %.1f us, submit %.1f us, wait GPU %.1f us\n",
            ns[0] / 1e3 / st[0], ns[2] / 1e3 / st[0], ns[3] / 1e3 / st[0], ns[1] / 1e3 / st[0], ns[4] / 1e3 / st[1],
            ns[5] / 1e3 / st[1], ns[6] / 1e3 / st[1]);
  printf("{\"bench\": \"dropin_thread_per_client\", \"workload\": \"%s\", \"simd_status\": \"%s\", \"clients\": %d, \"blocks\": %d, \"window\": %d, "
         "\"seconds\": %.4f, \"input_msps\": %.2f, \"calls_per_s\": %.0f, \"us_per_call_per_thread\": %.1f, "
         "\"outputs\": %llu, \"launch_batches\": %llu, \"engine_calls\": %llu, \"shared_inputs\": %llu, "
         "\"stream_served\": %llu, \"stream_blocks\": %llu, \"stream_hits\": %llu, \"stream_desyncs\": %llu, "
         "\"stream_joins\": %llu, \"stream_members\": %llu}\n",
         rational ? "rational_3_128_of_2048k" : "integer_48k_96k_of_2016k", SIMD_STATUS, n_clients, n_blocks, g_window, dt, n_blocks * (BLOCK / 2) / dt / 1e6, (double)n_clients * n_blocks / dt,
         dt / n_blocks * 1e6, (unsigned long long)outputs, (unsigned long long)batches, (unsigned long long)calls,
         (unsigned long long)shared, (unsigned long long)st[0], (unsigned long long)st[1], (unsigned long long)st[2],
         (unsigned long long)st[3], (unsigned long long)st[4], (unsigned long long)st[6]);
  for (int c = 0; c < n_clients; c++) destroy_xlating(clients[c].filter);
  return 0;
}
