/*
 * csrc/xlating_dropin.cu -- the reference's per-filter C ABI (include/xlating.h).
 *
 * Replaces, symbol for symbol: src/xlating.c:495-582 (create), :384-447 and
 * :352-382 (the twelve process_* entry points), :584-616 (destroy) and the
 * SIMD_STATUS string (:145-156, :268).  There is no CPU implementation behind
 * these symbols.
 *
 * Model.  The reference gives every client a filter and a dsp thread
 * (src/dsp_worker.c:41-88), and all those threads call process_* at about the
 * same time, each on a private copy of the same SDR block (src/queue.c:114).  A
 * GPU pipeline per filter would make that C x (copies + launches + syncs) per
 * block, all serialised on the CUDA context lock: measured 13 k calls/s however
 * many threads.  So the calls are COMBINED, per device:
 *
 *   - the calling thread stages its input into the filter's pinned buffer
 *     (the only per-call memcpy, done in parallel by the callers) and queues a
 *     request;
 *   - the first caller that finds a free launch lane becomes the leader
 *     (call_combiner.h): it takes every queued request (its own included), writes
 *     the request table, launches dropin_front_kernel + dropin_fir_kernel for the
 *     whole batch (dropin_kernels.cuh) and synchronises once; the others sleep, each
 *     on its own condition variable, until their request is marked done.  A lone
 *     caller is always its own leader, so the single-filter latency has no thread
 *     hand-off in it.
 *
 * Inputs are read and outputs are written by the kernels directly in pinned host
 * memory (zero-copy over PCIe; outputs as full 256-byte lines), so a batch is two
 * launches and one synchronise.  (Copy-engine staging was measured and dropped: one
 * cudaMemcpyAsync per request, or one cudaMemcpyBatchAsync per batch, cost ~37 us per
 * request and ran 2.6x slower than SM loads over PCIe at 19 GB/s.)
 *
 * Identical inputs.  The dsp threads of the reference all hold copies of the SAME
 * block.  With two or more filters alive a caller therefore first looks its input up
 * in a small content-addressed cache (block_cache.h: a sampled key, then memcmp against
 * the published copies with that key -- never trusting the key): the first caller publishes the block
 * (pinned copy + one async H2D), the others share its HBM copy, so the block crosses
 * PCIe once per SDR block instead of once per client.  Callers with unique data, or
 * arriving when every cache entry is in use, take the private zero-copy path.
 * Filters keep private state (ring, oscillator, history) on the device; results
 * are independent of how calls happen to be batched.
 *
 * One stream, one batch (stream_overlay.h).  When several filters of one band
 * (same device, sampling rate and block size) are alive, their calls are first matched
 * against a log of "the stream": the dsp threads of the reference all consume the same
 * block sequence, so the first thread that brings a block submits it ONCE to a batch group
 * (include/xlating_group.h: one H2D copy, one fused tiled launch for all member filters)
 * and every other thread only compares its bytes with the log entry (memcmp, always),
 * sleeps until the GPU is done and copies its own row of the result.  A filter whose
 * input is not the stream's next block (its queue dropped one, it lags a whole ring, it
 * is fed by another source) leaves the group and is served by the combined per-filter
 * engine below from its own mirror of the state; it rejoins when it is in step again.
 * XLATING_B200_STREAM=0 turns this off, XLATING_B200_STREAM_RING=<blocks> sizes the log
 * and the group's result ring (default 64 = the reference's queue_size, src/config.c:183).
 *
 * XLATING_B200_DROPIN=group selects the older model instead (each filter a private
 * one-client batch group with its own streams), kept for A/B measurements.
 *
 * Rational filters (create_rational_frequency_xlating_filter, interpolation L > 1) are the
 * filter with decimation M at L * fs fed the zero-stuffed stream, as the batch group's
 * rational clients are: history and output counts in upsampled samples, polyphase taps, no
 * Q15 path.  They share their band's group with the integer filters.
 */
#include <cuda_runtime.h>
#include <errno.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <atomic>
#include <condition_variable>
#include <map>
#include <mutex>
#include <new>
#include <vector>

#include "block_cache.h"
#include "call_combiner.h"
#include "dropin_kernels.cuh"
#include "stream_overlay.h"
#include "taps_host.h"
#include "xl_log.h"
#include "xlating.h"
#include "xlating_group.h"

using namespace xl;


#define CU_TRY(expr)                                                                      \
  do {                                                                                    \
    cudaError_t e_ = (expr);                                                              \
    if (e_ != cudaSuccess) {                                                              \
      XL_LOG("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e_), __FILE__, __LINE__); \
      rc = -EIO;                                                                          \
      goto fail;                                                                          \
    }                                                                                     \
  } while (0)

namespace {

constexpr int kMaxFilters = 4096;  // FilterDev table entries per device
constexpr int kMaxLanes = CallCombiner::kMaxLanes;
constexpr int kMaxBatch = 1024;    // requests per launch

// The cf32 oscillator of a call is a dependent chain of n_out steps.  A CPU core walks
// it faster than a GPU lane, so it can run on the calling thread (taps_host.c:
// xl_osc_chain_cf32, bit-identical arithmetic) into a pinned table the FIR kernel reads;
// a lone filter's chain runs while the front kernel converts, which shortens a lone call.
// XLATING_B200_OSC=device|lanes|host.
constexpr bool kOscHostDefault = true;

struct Lane {
  cudaStream_t stream = nullptr;
  DropinReq *h_req = nullptr;        // pinned, read by the front kernel over PCIe
  const DropinReq *d_req = nullptr;  // its device address
  int2 *d_batch = nullptr;           // (filter, q15) per request, written by the front kernel
};

struct Engine;

// One SDR band as the overlay sees it: filters created with the same sampling rate and
// block size on one device.  The batch group and the stream log exist only while at least
// two such filters are alive (a lone filter keeps its 46 us private path).
struct StreamHost {
  Engine *e = nullptr;
  uint32_t fs = 0, max_in = 0;
  int refs = 0;                          // filters with this key (guarded by Engine::mu)
  xlg_group *g = nullptr;
  std::atomic<AutoStream *> as{nullptr};
};

struct Engine {
  int device = 0;
  CallCombiner *combiner = nullptr;
  Lane lanes[kMaxLanes];
  int n_lanes = 4;
  FilterDev *d_filters = nullptr;
  std::mutex mu;  // guards free_slots
  std::vector<int> free_slots;
  // identical-input sharing
  BlockCache *cache = nullptr;
  cudaStream_t s_upload = nullptr;             // H2D of published blocks
  cudaEvent_t ev_slot[BlockCache::kSlots] = {};  // "entry is in HBM", recorded at each publish
  std::atomic<int> live_filters{0};
  bool share_inputs = true;                    // XLATING_B200_SHARE=0 turns the cache off
  bool osc_lanes = false;                      // XLATING_B200_OSC=lanes: oscillator chains share one warp (A/B)
  bool osc_host = kOscHostDefault;             // XLATING_B200_OSC=host|device: who walks the cf32 oscillator
  // Memory of destroyed filters, kept for the next create: destroy_xlating is then a few
  // microseconds like the reference's free() (src/xlating.c:584-616) instead of two
  // synchronising CUDA frees.  The reference's tcp threads tear a client down while
  // holding the server mutex (src/tcp_server.c:231-254) and its server test relies on
  // that being quick (test/test_tcp_server.c:43-63: a late close() of an already closed
  // descriptor must not land after the descriptor number has been reused).
  struct Pooled {
    void *d_mem, *h_mem;
    size_t d_bytes, h_bytes;
  };
  std::vector<Pooled> pool;  // guarded by mu
  size_t pool_bytes = 0;
  // stream overlay (stream_overlay.h)
  bool overlay = true;       // XLATING_B200_STREAM=0 turns it off
  int stream_ring = 64;      // XLATING_B200_STREAM_RING
  std::vector<StreamHost *> streams;  // guarded by mu
  // served calls, time in xlg_copy_output / in whole served calls -- sharded like the overlay's counters
  struct alignas(64) ServedShard {
    std::atomic<uint64_t> served{0}, copy_ns{0}, call_ns{0};
  };
  ServedShard served[AutoStream::kLanes];
};
constexpr size_t kPoolMaxBytes = (size_t)2 << 30;  // device + pinned bytes kept for reuse

constexpr size_t kShareMinBytes = 4096;  // smaller inputs are not worth hashing
static_assert(BlockCache::kSlots <= 32, "run_batch keeps the referenced entries in a 32-bit mask");

int cache_alloc(void *ctx, size_t bytes, void **host, void **dev) {
  Engine *e = (Engine *)ctx;
  *host = *dev = nullptr;
  if (cudaSetDevice(e->device) != cudaSuccess) return -1;
  if (cudaHostAlloc(host, bytes, cudaHostAllocDefault) != cudaSuccess) return -1;
  if (cudaMalloc(dev, bytes) != cudaSuccess) {
    cudaFreeHost(*host);
    *host = nullptr;
    cudaGetLastError();
    return -1;
  }
  return 0;
}

void cache_release(void *ctx, void *host, void *dev) {
  cudaSetDevice(((Engine *)ctx)->device);
  cudaFreeHost(host);
  cudaFree(dev);
}

int cache_upload(void *ctx, int slot, const void *host, void *dev, size_t bytes) {
  Engine *e = (Engine *)ctx;
  if (cudaSetDevice(e->device) != cudaSuccess) return -1;
  if (cudaMemcpyAsync(dev, host, bytes, cudaMemcpyHostToDevice, e->s_upload) != cudaSuccess ||
      cudaEventRecord(e->ev_slot[slot], e->s_upload) != cudaSuccess) {
    cudaGetLastError();
    return -1;
  }
  return 0;
}



std::mutex g_engines_mu;
std::map<int, Engine *> g_engines;  // one per device, for the life of the process

}  // namespace

struct xlating_t {
  float *adopted_taps = nullptr;  // freed on destroy, like src/xlating.c:600-602
  // --- XLATING_B200_DROPIN=group ---
  xlg_group *group = nullptr;
  int client = -1;
  // --- combined engine ---
  Engine *e = nullptr;
  int slot = -1;
  bool counted = false;  // in Engine::live_filters
  uint32_t D = 0, max_in = 0;
  uint32_t L = 1;           // interpolation (create_rational_frequency_xlating_filter); 1 = integer filter
  long long T = 0;
  int out_cap = 0;
  long long hist = 0;       // host mirror of FilterDev::hist (same integer formula; upsampled samples)
  long long S = 0, qS = 0;  // samples consumed so far by the cf32 / Q15 path
  void *d_mem = nullptr;    // ring | qring | taps | qtaps | phases | qphases
  void *h_mem = nullptr;    // pinned: staged input | cf32 output | Q15 output
  size_t d_bytes = 0, h_bytes = 0;
  void *h_in = nullptr;
  const void *d_in = nullptr;  // device address of h_in (zero-copy)
  float2 *h_out = nullptr;
  short2 *h_qout = nullptr;
  float *h_phases = nullptr;  // pinned oscillator table (host-walked chain), read by the FIR kernel
  float ph_re = 1.0f, ph_im = 0.0f, inc_re = 0.0f, inc_im = 0.0f;  // host oscillator (src/xlating.c:543-544)
  bool osc_deferred = false;  // this call's chain is still to be walked (by the batch leader)
  // --- stream overlay: membership in the band's batch group, and the mirror of the state
  // after the last block this filter really consumed (hist, ph_re/ph_im above, tail below),
  // from which either engine can carry on
  StreamHost *sh = nullptr;
  AutoStream::Member as_m;
  int32_t center_freq = 0;
  uint32_t fs = 0;
  bool as_disabled = false;   // a Q15 call was made: the two paths share history_offset, stay private
  bool q15_refused = false;   // a Q15 call on a rational filter was refused (and logged, once)
  bool dev_stale = false;     // the private device state is behind the mirror (group served the last blocks)
  std::vector<float2> tail;   // the last floor((T-1)/L) samples consumed (cf32), oldest first, zeros before
                              // the first: all that the next window can reach
  float2 *d_ring = nullptr;   // the filter's private cf32 ring (inside d_mem) and its size
  size_t ring_cap = 0;
  // the call in flight
  DropinReq req;
  int req_out = 0;
  int req_slot = -1;  // block-cache entry the input is shared through, or -1 (private staging)
  CombinerCall call;  // user = this filter
};

namespace {

size_t align_up(size_t v, size_t a) { return (v + a - 1) / a * a; }

// ---- stream overlay: group operations (StreamOps) ----
void *stream_alloc(void *ctx, size_t bytes) {
  StreamHost *sh = (StreamHost *)ctx;
  void *p = nullptr;
  if (cudaSetDevice(sh->e->device) != cudaSuccess || cudaHostAlloc(&p, bytes, cudaHostAllocDefault) != cudaSuccess) {
    cudaGetLastError();
    return nullptr;
  }
  return p;
}
void stream_free(void *ctx, void *p) {
  cudaSetDevice(((StreamHost *)ctx)->e->device);
  cudaFreeHost(p);
}
int stream_submit(void *ctx, int fmt, const void *block, size_t elems, int64_t *ticket) {
  StreamHost *sh = (StreamHost *)ctx;
  // the log entry is page-locked and stays untouched for a whole ring of blocks
  const int64_t t = xlg_submit(sh->g, fmt, block, elems, XLG_INPUT_KEEP);
  if (t < 0) return (int)t;
  *ticket = t;
  return 0;
}
int stream_wait(void *ctx, int64_t ticket) { return xlg_wait(((StreamHost *)ctx)->g, ticket); }
int stream_add(void *ctx, void *filter, int64_t valid_history, int *client) {
  StreamHost *sh = (StreamHost *)ctx;
  const xlating *f = (const xlating *)filter;
  xlg_client_state st;
  st.valid_history = valid_history;
  st.hist = f->hist;
  st.phase_re = f->ph_re;
  st.phase_im = f->ph_im;
  if (f->L > 1)
    return xlg_add_client_rational_ex(sh->g, f->L, f->D, f->adopted_taps, (size_t)f->T, f->center_freq, &st, client);
  return xlg_add_client_ex(sh->g, f->D, f->adopted_taps, (size_t)f->T, f->center_freq, &st, client);
}
int stream_remove(void *ctx, int client) { return xlg_remove_client(((StreamHost *)ctx)->g, client); }

// host twins of the device conversions (xlating_common.cuh: all exact)
inline float2 host_sample(int fmt, const void *input, size_t i) {
  if (fmt == XLG_FMT_CU8) {
    const uint8_t *u = (const uint8_t *)input + 2 * i;
    return make_float2(((float)u[0] - 127.5f) * 0.0078125f, ((float)u[1] - 127.5f) * 0.0078125f);
  }
  if (fmt == XLG_FMT_CS8) {
    const int8_t *u = (const int8_t *)input + 2 * i;
    return make_float2((float)u[0] * 0.0078125f, (float)u[1] * 0.0078125f);
  }
  const int16_t *u = (const int16_t *)input + 2 * i;
  return make_float2((float)u[0] * (1.0f / 32768.0f), (float)u[1] * (1.0f / 32768.0f));
}

// the last T-1 samples of (tail ++ block)
void tail_push(xlating *f, int fmt, const void *input, size_t n) {
  const size_t keep = f->tail.size();
  if (keep == 0) return;
  if (n >= keep) {
    for (size_t i = 0; i < keep; i++) f->tail[i] = host_sample(fmt, input, n - keep + i);
  } else {
    memmove(f->tail.data(), f->tail.data() + n, sizeof(float2) * (keep - n));
    for (size_t i = 0; i < n; i++) f->tail[keep - n + i] = host_sample(fmt, input, i);
  }
}

// The group served this filter's last blocks: bring the PRIVATE device state up to the
// mirror before the per-filter engine runs again (history into the private ring at the
// positions the next call's window reads, history_offset, oscillator).
int sync_device_state(xlating *f) {
  cudaError_t err = cudaSetDevice(f->e->device);
  const size_t keep = f->tail.size();
  const unsigned mask = (unsigned)(f->ring_cap - 1);
  for (size_t done = 0; done < keep && err == cudaSuccess;) {
    const unsigned idx = (unsigned)((unsigned long long)(f->S - (long long)keep + (long long)done)) & mask;
    const size_t run = std::min(keep - done, (size_t)(mask + 1u - idx));
    err = cudaMemcpy(f->d_ring + idx, f->tail.data() + done, run * sizeof(float2), cudaMemcpyHostToDevice);
    done += run;
  }
  FilterDev *d = f->e->d_filters + f->slot;
  const long long hist = f->hist;
  const float2 ph = make_float2(f->ph_re, f->ph_im);
  if (err == cudaSuccess)
    err = cudaMemcpy((char *)d + offsetof(FilterDev, hist), &hist, sizeof(hist), cudaMemcpyHostToDevice);
  if (err == cudaSuccess)
    err = cudaMemcpy((char *)d + offsetof(FilterDev, phase), &ph, sizeof(ph), cudaMemcpyHostToDevice);
  if (err != cudaSuccess) {
    XL_LOG("could not restore a filter's private state: %s", cudaGetErrorString(err));
    return -EIO;
  }
  f->dev_stale = false;
  return 0;
}

// Launch one batch on lane `lane` and wait for it (CallCombiner::RunBatch; called by the
// batch's leader thread).
int run_batch(void *ctx, int lane, CombinerCall *const *batch, int n_req) {
  Engine *e = (Engine *)ctx;
  Lane &L = e->lanes[lane];
  cudaError_t err = cudaSetDevice(e->device);
  if (err == cudaSuccess) {
    int max_n = 0, max_out = 0, max_poly_ctas = 0;
    unsigned slots = 0;  // shared inputs this batch reads: wait for their H2D
    for (int i = 0; i < n_req; i++) {
      const xlating *b = (const xlating *)batch[i]->user;
      L.h_req[i] = b->req;
      if (b->req.n > max_n) max_n = b->req.n;
      if (b->L > 1) {
        const int span = dropin_fir_span((int)b->L);
        max_poly_ctas = std::max(max_poly_ctas, (b->req_out + span - 1) / span);
      } else if (b->req_out > max_out) {
        max_out = b->req_out;
      }
      if (b->req_slot >= 0) slots |= 1u << b->req_slot;
    }
    for (int sl = 0; sl < BlockCache::kSlots && err == cudaSuccess; sl++)
      if (slots & (1u << sl)) err = cudaStreamWaitEvent(L.stream, e->ev_slot[sl], 0);
    const int osc_per_block = e->osc_lanes ? 32 : DF_OSC_PER_BLOCK;
    const int n_osc = (n_req + osc_per_block - 1) / osc_per_block;
    const int cpr = (max_n + DF_SPB - 1) / DF_SPB;
    if (err == cudaSuccess) {
      dropin_front_kernel<<<n_osc + n_req * cpr, DF_THREADS, 0, L.stream>>>(e->d_filters, L.d_req, L.d_batch, n_req,
                                                                            n_osc, cpr, e->osc_lanes ? 1 : 0);
      for (int i = 0; i < n_req; i++) {
        xlating *b = (xlating *)batch[i]->user;  // its owner is asleep (or is this thread)
        if (b->osc_deferred) {
          xl_osc_chain_cf32(&b->ph_re, &b->ph_im, b->inc_re, b->inc_im, b->h_phases, b->req_out);
          b->osc_deferred = false;
        }
      }
      if (max_out > 0)
        dropin_fir_kernel<<<dim3((max_out + G_OPC - 1) / G_OPC, n_req), G_THREADS, 0, L.stream>>>(e->d_filters,
                                                                                                  L.d_batch);
      if (max_poly_ctas > 0)
        dropin_fir_poly_kernel<<<dim3(max_poly_ctas, n_req), G_THREADS, 0, L.stream>>>(e->d_filters, L.d_batch);
      err = cudaGetLastError();
    }
    if (err == cudaSuccess) err = cudaStreamSynchronize(L.stream);
  }
  if (err != cudaSuccess) {
    XL_LOG("drop-in batch of %d calls failed: %s", n_req, cudaGetErrorString(err));
    return -EIO;
  }
  return 0;
}

int engine_get(int device, Engine **out) {
  std::lock_guard<std::mutex> lk(g_engines_mu);
  auto it = g_engines.find(device);
  if (it != g_engines.end()) {
    *out = it->second;
    return 0;
  }
  int ndev = 0;
  cudaError_t err = cudaGetDeviceCount(&ndev);
  if (err != cudaSuccess || ndev == 0) {
    XL_LOG("no usable CUDA device (%s); this library has no CPU fallback",
           err == cudaSuccess ? "device count is 0" : cudaGetErrorString(err));
    return -ENODEV;
  }
  if (device < 0 || device >= ndev) {
    XL_LOG("device %d out of range (%d present)", device, ndev);
    return -ENODEV;
  }
  int rc = 0;
  Engine *e = nullptr;
  cudaDeviceProp prop;
  CU_TRY(cudaSetDevice(device));
  CU_TRY(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) {
    XL_LOG("device %d is sm_%d%d; this library is built for sm_90a only", device, prop.major, prop.minor);
    return -ENODEV;
  }
  e = new (std::nothrow) Engine();
  if (e == nullptr) return -ENOMEM;
  e->device = device;
  {
    const char *env = getenv("XLATING_B200_LANES");
    if (env != nullptr) e->n_lanes = atoi(env);
    if (e->n_lanes < 1) e->n_lanes = 1;
    if (e->n_lanes > kMaxLanes) e->n_lanes = kMaxLanes;
    env = getenv("XLATING_B200_SHARE");
    e->share_inputs = !(env != nullptr && strcmp(env, "0") == 0);
    env = getenv("XLATING_B200_STREAM");
    e->overlay = !(env != nullptr && strcmp(env, "0") == 0);
    env = getenv("XLATING_B200_STREAM_RING");
    if (env != nullptr) e->stream_ring = std::min(std::max(atoi(env), 4), 1024);
    env = getenv("XLATING_B200_OSC");
    e->osc_lanes = env != nullptr && strcmp(env, "lanes") == 0;
    if (env != nullptr && strcmp(env, "host") == 0) e->osc_host = true;
    if (env != nullptr && (strcmp(env, "device") == 0 || strcmp(env, "lanes") == 0)) e->osc_host = false;
  }
  {
    CU_TRY(cudaStreamCreateWithFlags(&e->s_upload, cudaStreamNonBlocking));
    for (int i = 0; i < BlockCache::kSlots; i++)
      CU_TRY(cudaEventCreateWithFlags(&e->ev_slot[i], cudaEventDisableTiming));
    const BlockCacheOps ops = {cache_alloc, cache_release, cache_upload, e};
    e->cache = new (std::nothrow) BlockCache(ops);
    if (e->cache == nullptr) return -ENOMEM;
  }
  CU_TRY(cudaMalloc(&e->d_filters, sizeof(FilterDev) * kMaxFilters));
  CU_TRY(cudaMemset(e->d_filters, 0, sizeof(FilterDev) * kMaxFilters));
  for (int i = 0; i < e->n_lanes; i++) {
    Lane &L = e->lanes[i];
    CU_TRY(cudaStreamCreateWithFlags(&L.stream, cudaStreamNonBlocking));
    CU_TRY(cudaHostAlloc((void **)&L.h_req, sizeof(DropinReq) * kMaxBatch, cudaHostAllocMapped));
    CU_TRY(cudaHostGetDevicePointer((void **)&L.d_req, L.h_req, 0));
    CU_TRY(cudaMalloc(&L.d_batch, sizeof(int2) * kMaxBatch));
  }
  for (int i = kMaxFilters - 1; i >= 0; i--) e->free_slots.push_back(i);
  e->combiner = new (std::nothrow) CallCombiner(e->n_lanes, kMaxBatch, run_batch, e);
  if (e->combiner == nullptr) return -ENOMEM;
  g_engines[device] = e;
  *out = e;
  return 0;
fail:
  // partially built engine: leave the (few) allocations to process teardown
  return rc;
}

void stream_detach(xlating *f) {
  StreamHost *sh = f->sh;
  if (sh == nullptr) return;
  AutoStream *as = sh->as.load();
  if (as != nullptr) as->leave(f->as_m);
  f->sh = nullptr;
  Engine *e = sh->e;
  AutoStream *dead_as = nullptr;
  xlg_group *dead_g = nullptr;
  bool last = false;
  {
    std::lock_guard<std::mutex> lk(e->mu);
    if (--sh->refs == 0) {
      last = true;
      // nobody can reach the stream any more: filters find it only through their own sh
      dead_as = sh->as.exchange(nullptr);
      dead_g = sh->g;
      for (size_t i = 0; i < e->streams.size(); i++)
        if (e->streams[i] == sh) {
          e->streams.erase(e->streams.begin() + (long)i);
          break;
        }
    }
  }
  if (last) {
    delete dead_as;  // frees the log's pinned blocks (before the group: its callbacks use sh)
    if (dead_g != nullptr) xlg_destroy(dead_g);
    delete sh;
  }
}

// The band's stream: found or created when a filter is built; the batch group and the log
// come to life with the second filter of the band.
void stream_attach(xlating *f, uint32_t fs, uint32_t max_in) {
  Engine *e = f->e;
  if (!e->overlay || !e->osc_host) return;  // the mirror needs the host-walked oscillator
  StreamHost *sh = nullptr;
  bool start = false;
  {
    std::lock_guard<std::mutex> lk(e->mu);
    for (StreamHost *c : e->streams)
      if (c->fs == fs && c->max_in == max_in) sh = c;
    if (sh == nullptr) {
      sh = new (std::nothrow) StreamHost();
      if (sh == nullptr) return;
      sh->e = e;
      sh->fs = fs;
      sh->max_in = max_in;
      e->streams.push_back(sh);
    }
    sh->refs++;
    start = sh->refs >= 2 && sh->as.load() == nullptr && sh->g == nullptr;
    if (start) {
      // still under e->mu: one creator.  (xlg_create_ex is slow -- pinned staging, streams --
      // but it happens once per band.)
      if (xlg_create_ex(e->device, fs, max_in, XLG_TRACK_STATE, (uint32_t)e->stream_ring, &sh->g) == 0) {
        const StreamOps ops = {sh, stream_alloc, stream_free, stream_submit, stream_wait, stream_add, stream_remove};
        AutoStream *as = new (std::nothrow) AutoStream(ops, e->stream_ring, (size_t)max_in * sizeof(int16_t));
        if (as != nullptr) {
          sh->as.store(as);
        } else {
          xlg_destroy(sh->g);
          sh->g = nullptr;
        }
      } else {
        sh->g = nullptr;
      }
    }
  }
  f->sh = sh;
}

void filter_release(xlating *f) {
  stream_detach(f);
  if (f->e != nullptr) {
    bool pooled = false;
    {
      std::lock_guard<std::mutex> lk(f->e->mu);
      if (f->slot >= 0) f->e->free_slots.push_back(f->slot);
      if (f->d_mem != nullptr && f->h_mem != nullptr &&
          f->e->pool_bytes + f->d_bytes + f->h_bytes <= kPoolMaxBytes) {
        f->e->pool.push_back({f->d_mem, f->h_mem, f->d_bytes, f->h_bytes});
        f->e->pool_bytes += f->d_bytes + f->h_bytes;
        pooled = true;
      }
    }
    if (!pooled) {
      cudaSetDevice(f->e->device);
      if (f->d_mem != nullptr) cudaFree(f->d_mem);
      if (f->h_mem != nullptr) cudaFreeHost(f->h_mem);
    }
    if (f->counted) f->e->live_filters--;
  }
  if (f->group != nullptr) xlg_destroy(f->group);
  if (f->adopted_taps != nullptr) free(f->adopted_taps);
  delete f;
}

// A filter with interpolation L > 1 is the filter with decimation M = `decimation` at L * fs fed the
// zero-stuffed stream (create_rational_frequency_xlating_filter): its constants are built at L * fs, its
// taps are kept as polyphase branches and it has no Q15 ring or taps.  L = 1 is the integer filter.
int filter_build(xlating *f, int device, uint32_t interp, uint32_t decimation, const float *taps, size_t taps_len,
                 int32_t center_freq, uint32_t sampling_freq, uint32_t max_in) {
  if (decimation == 0 || sampling_freq == 0) return -EINVAL;
  int rc = engine_get(device, &f->e);
  if (rc != 0) {
    f->e = nullptr;
    return rc;
  }
  xl_client_consts k;
  rc = xl_client_consts_build(taps, taps_len, decimation, center_freq, interp * sampling_freq, &k);
  if (rc != 0) return rc;
  const bool q15 = interp == 1;  // rational filters refuse the Q15 path
  const size_t Tb = (taps_len + interp - 1) / interp;  // taps per polyphase branch (T for L = 1)
  std::vector<float> branches;
  if (!q15) {
    branches.resize(2 * (size_t)interp * Tb);
    xl_poly_pack(k.rev_cf32, taps_len, interp, branches.data());
  }
  f->D = decimation;
  f->L = interp;
  f->T = (long long)taps_len;
  f->max_in = max_in;
  f->hist = (long long)taps_len - 1;  // src/xlating.c:552 (upsampled samples)
  // >= any call's output count (hist <= T-1)
  f->out_cap = (int)((uint64_t)(max_in / 2) * interp / decimation + 2);
  const size_t max_n = max_in / 2;
  const size_t hist_in = (taps_len - 1) / interp + 1;  // input samples the oldest window can reach
  size_t cap = 1024;
  while (cap < hist_in + max_n + 64) cap <<= 1;      // history + one block, power of two
  FilterDev d;
  memset(&d, 0, sizeof(d));
  // device arena
  const size_t o_ring = 0;
  const size_t o_qring = align_up(o_ring + cap * sizeof(float2), 256);
  const size_t o_taps = align_up(o_qring + (q15 ? cap * sizeof(short2) : 0), 256);
  const size_t o_qtaps = align_up(o_taps + interp * Tb * sizeof(float2), 256);
  const size_t o_ph = align_up(o_qtaps + (q15 ? taps_len * sizeof(short2) : 0), 256);
  const size_t o_qph = align_up(o_ph + ((size_t)f->out_cap / 2 + 2) * sizeof(float2), 256);
  const size_t d_bytes = align_up(o_qph + (q15 ? ((size_t)f->out_cap + 2) * sizeof(short2) : 0), 256);
  // pinned host arena
  const size_t h_in_bytes = align_up((size_t)max_in * sizeof(int16_t), 256);  // cs16 is the widest input
  const size_t h_out_bytes = align_up((size_t)f->out_cap * sizeof(float2), 256);
  const size_t h_qout_bytes = align_up((size_t)f->out_cap * sizeof(short2), 256);
  const size_t h_ph_bytes = align_up(((size_t)f->out_cap / 2 + 2) * sizeof(float2), 256);
  char *dm = nullptr, *hm = nullptr, *hm_dev = nullptr;
  CU_TRY(cudaSetDevice(device));
  {
    // memory of a destroyed filter of the same shape, if any
    std::lock_guard<std::mutex> lk(f->e->mu);
    const size_t h_need = h_in_bytes + h_out_bytes + h_qout_bytes + h_ph_bytes;
    for (size_t i = 0; i < f->e->pool.size(); i++) {
      const Engine::Pooled &p = f->e->pool[i];
      if (p.d_bytes >= d_bytes && p.h_bytes >= h_need && p.d_bytes <= 2 * d_bytes && p.h_bytes <= 2 * h_need) {
        f->d_mem = p.d_mem;
        f->h_mem = p.h_mem;
        f->d_bytes = p.d_bytes;
        f->h_bytes = p.h_bytes;
        f->e->pool_bytes -= p.d_bytes + p.h_bytes;
        f->e->pool.erase(f->e->pool.begin() + (long)i);
        break;
      }
    }
  }
  if (f->d_mem == nullptr) {
    CU_TRY(cudaMalloc(&f->d_mem, d_bytes));
    f->d_bytes = d_bytes;
  }
  dm = (char *)f->d_mem;
  CU_TRY(cudaMemset(dm, 0, o_taps));  // both rings start as the reference's zeroed working buffers (:556-565)
  if (q15) {
    CU_TRY(cudaMemcpy(dm + o_taps, k.rev_cf32, taps_len * sizeof(float2), cudaMemcpyHostToDevice));
    CU_TRY(cudaMemcpy(dm + o_qtaps, k.rev_q15, taps_len * sizeof(short2), cudaMemcpyHostToDevice));
  } else {
    CU_TRY(cudaMemcpy(dm + o_taps, branches.data(), branches.size() * sizeof(float), cudaMemcpyHostToDevice));
  }
  if (f->h_mem == nullptr) {
    f->h_bytes = h_in_bytes + h_out_bytes + h_qout_bytes + h_ph_bytes;
    CU_TRY(cudaHostAlloc(&f->h_mem, f->h_bytes, cudaHostAllocMapped));
  }
  hm = (char *)f->h_mem;
  CU_TRY(cudaHostGetDevicePointer((void **)&hm_dev, f->h_mem, 0));
  f->h_in = hm;
  f->d_in = hm_dev;
  f->h_out = (float2 *)(hm + h_in_bytes);
  f->h_qout = (short2 *)(hm + h_in_bytes + h_out_bytes);
  f->h_phases = (float *)(hm + h_in_bytes + h_out_bytes + h_qout_bytes);
  f->inc_re = k.incr_re;
  f->inc_im = k.incr_im;
  f->center_freq = center_freq;
  f->fs = sampling_freq;
  f->tail.assign((taps_len - 1) / interp, make_float2(0.f, 0.f));  // src/xlating.c:552-565: zero history
  f->d_ring = (float2 *)(dm + o_ring);
  f->ring_cap = cap;
  d.ring = (float2 *)(dm + o_ring);
  d.qring = q15 ? (short2 *)(dm + o_qring) : nullptr;
  d.taps = (const float2 *)(dm + o_taps);
  d.qtaps = q15 ? (const short2 *)(dm + o_qtaps) : nullptr;
  d.phases = (float2 *)(dm + o_ph);
  d.phases_host = (const float2 *)(hm_dev + h_in_bytes + h_out_bytes + h_qout_bytes);
  d.qphases = q15 ? (short2 *)(dm + o_qph) : nullptr;
  d.out = (float2 *)(hm_dev + h_in_bytes);
  d.qout = (short2 *)(hm_dev + h_in_bytes + h_out_bytes);
  d.hist = f->hist;
  d.phase = make_float2(1.0f, 0.0f);  // src/xlating.c:543
  d.incr = make_float2(k.incr_re, k.incr_im);
  d.qphase = make_short2(INT16_MAX, 0);  // :546-547
  d.qincr = make_short2(k.qincr_re, k.qincr_im);
  d.mask = (unsigned)(cap - 1);
  d.D = (int)decimation;
  d.T = (int)taps_len;
  d.out_cap = f->out_cap;
  d.L = (int)interp;
  {
    std::lock_guard<std::mutex> lk(f->e->mu);
    if (f->e->free_slots.empty()) {
      XL_LOG("more than %d filters on device %d", kMaxFilters, device);
      rc = -ENOMEM;
      goto fail;
    }
    f->slot = f->e->free_slots.back();
    f->e->free_slots.pop_back();
  }
  CU_TRY(cudaMemcpy(f->e->d_filters + f->slot, &d, sizeof(d), cudaMemcpyHostToDevice));
  f->e->live_filters++;
  f->counted = true;
  xl_client_consts_free(&k);
  stream_attach(f, sampling_freq, max_in);
  return 0;
fail:
  xl_client_consts_free(&k);
  return rc;
}

bool use_group_model() {
  const char *env = getenv("XLATING_B200_DROPIN");
  return env != nullptr && strcmp(env, "group") == 0;
}

void run_block_group(xlating *f, int fmt, const void *input, size_t input_len, uint32_t path, void **output,
                     size_t *output_len) {
  const int64_t ticket = xlg_submit(f->group, fmt, input, input_len, path);
  if (ticket < 0) {
    XL_LOG("block dropped (submit -> %lld)", (long long)ticket);
    return;
  }
  int rc = xlg_wait(f->group, ticket);
  if (rc != 0) {
    XL_LOG("block dropped (wait -> %d)", rc);
    return;
  }
  const void *out = NULL;
  size_t n = 0;
  rc = xlg_output(f->group, ticket, f->client, &out, &n);
  if (rc != 0) {
    XL_LOG("block dropped (output -> %d)", rc);
    return;
  }
  *output = (void *)out;
  *output_len = n;
}

void run_block(xlating *f, int fmt, const void *input, size_t input_len, bool q15, void **output,
               size_t *output_len) {
  *output_len = 0;
  if (q15 && f->L > 1) {
    // the Q15 path serves integer filters only: refuse before anything is consumed, so that the
    // filter's cf32 stream (and its place in the band's group) carries on as if this call never happened
    if (!f->q15_refused) XL_LOG("Q15 output is not available for a rational (L = %u) filter; use process_*_cf32", f->L);
    f->q15_refused = true;
    *output = (void *)f->h_qout;
    return;
  }
  if (f->group != nullptr) {
    run_block_group(f, fmt, input, input_len, q15 ? XLG_PATH_Q15 : 0, output, output_len);
    return;
  }
  *output = q15 ? (void *)f->h_qout : (void *)f->h_out;
  if (input_len > f->max_in) {
    // the reference would overrun its working buffer here (src/xlating.c:553)
    XL_LOG("block of %zu elements exceeds max_input_buffer_length %u", input_len, f->max_in);
    return;
  }
  const int n = (int)(input_len / 2);  // complex samples (src/xlating.c:387)
  if (n == 0) return;
  const size_t bytes = (size_t)n * 2 * (fmt == XLG_FMT_CS16 ? sizeof(int16_t) : 1);
  Engine *e = f->e;
  // ---- one stream, one batch: is this the band's next block? (stream_overlay.h) ----
  AutoStream *as = (f->sh != nullptr && !f->as_disabled) ? f->sh->as.load(std::memory_order_acquire) : nullptr;
  bool observed = false;
  if (as != nullptr && q15) {
    as->leave(f->as_m);  // the Q15 path shares history_offset with this one (src/xlating.c:29): stay private
    f->as_disabled = true;
    as = nullptr;
  }
  if (as != nullptr) {
    const size_t elems = (size_t)n * 2;
    AutoStream::Served sv;
    const uint64_t t_call = AutoStream::now_ns();
    if (f->as_m.member && as->member_call(f->as_m, input, bytes, fmt, elems, &sv) == 1) {
      // the group computed this block for every member; take this filter's row and state
      const long long first = f->S * f->L - f->hist;
      const long long last_ok = (f->S + n) * f->L - f->T;
      size_t want = 0, got = 0;
      if (last_ok >= first) want = (size_t)((last_ok - first) / (long long)f->D) + 1;
      xlg_client_state st;
      const uint64_t t_copy = AutoStream::now_ns();
      const int rc = xlg_copy_output(f->sh->g, sv.ticket, sv.client, f->h_out, (size_t)f->out_cap, &got, &st);
      Engine::ServedShard &shard = e->served[(size_t)(f->as_m.lane >= 0 ? f->as_m.lane : 0)];
      shard.copy_ns.fetch_add(AutoStream::now_ns() - t_copy, std::memory_order_relaxed);
      if (rc == 0 && got == want) {
        f->hist = st.hist;
        f->ph_re = st.phase_re;
        f->ph_im = st.phase_im;
        tail_push(f, fmt, input, (size_t)n);
        f->S += n;
        f->dev_stale = true;
        shard.served.fetch_add(1, std::memory_order_relaxed);
        shard.call_ns.fetch_add(AutoStream::now_ns() - t_call, std::memory_order_relaxed);
        *output_len = got;
        return;
      }
      // the result ring was recycled under this (slow) caller, or the group disagrees about the
      // output count: the mirror is untouched, serve the block privately
      if (rc == 0) XL_LOG("stream group produced %zu outputs where %zu were expected; filter leaves the group", got, want);
      as->leave(f->as_m);
    }
    observed = as->private_observe(f->as_m, input, bytes, fmt, elems);
  }
  if (f->dev_stale && sync_device_state(f) != 0) return;
  // other filters exist: they are probably being handed the same bytes (src/queue.c:114)
  int slot = BlockCache::kPrivate;
  if (e->share_inputs && bytes >= kShareMinBytes && e->live_filters.load() >= 2) slot = e->cache->acquire(input, bytes);
  if (slot < 0) memcpy(f->h_in, input, bytes);
  const long long S = q15 ? f->qS : f->S;
  // host mirror of the output count (the oscillator lane uses the same integers, in upsampled
  // samples: L = 1 for the Q15 path)
  const long long first = S * f->L - f->hist;
  const long long last_ok = (S + n) * f->L - f->T;
  int n_out = 0;
  if (last_ok >= first) n_out = (int)((last_ok - first) / (long long)f->D) + 1;
  if (n_out > f->out_cap) n_out = f->out_cap;
  f->req.raw = slot >= 0 ? e->cache->device_ptr(slot) : f->d_in;
  f->req_slot = slot;
  f->req.S = S;
  f->req.filter = f->slot;
  f->req.n = n;
  f->req.fmt = fmt;
  f->req.q15 = q15 ? 1 : 0;
  f->req.osc_host = 0;
  f->req.n_out = n_out;
  f->req_out = n_out;
  f->osc_deferred = false;
  if (e->osc_host && !q15) {
    if (e->live_filters.load() >= 2) {
      // many callers: each walks its own chain, in parallel, before queueing
      xl_osc_chain_cf32(&f->ph_re, &f->ph_im, f->inc_re, f->inc_im, f->h_phases, n_out);
      f->req.osc_host = 1;
    } else {
      // a lone filter: the chain is walked while the front kernel converts (run_batch)
      f->osc_deferred = true;
      f->req.osc_host = 2;
    }
  }
  const int rc = e->combiner->run(&f->call);
  if (slot >= 0) e->cache->release(slot);
  // the samples are consumed whatever happened to the launch
  f->hist = (S + n) * f->L - (first + (long long)n_out * (long long)f->D);
  if (q15)
    f->qS += n;
  else
    f->S += n;
  if (!q15) {
    tail_push(f, fmt, input, (size_t)n);
    if (as != nullptr && rc == 0) {
      if (!observed) as->private_observe(f->as_m, input, bytes, fmt, (size_t)n * 2, /*retry=*/true);
      as->try_join(f->as_m, ((int64_t)f->T - 1) / f->L, (int64_t)f->S, f);  // the mirror's tail
    }
  }
  if (rc != 0) {
    XL_LOG("block dropped (%d)", rc);
    return;
  }
  *output_len = (size_t)n_out;
}

// Both constructors after their argument checks: adopts `taps`.
int create_filter(uint32_t interp, uint32_t decimation, float *taps, size_t taps_len, int32_t center_freq,
                  uint32_t sampling_freq, uint32_t max_input_buffer_length, xlating **filter) {
  xlating *f = new (std::nothrow) xlating_t();
  if (f == NULL) {
    return -ENOMEM;
  }
  f->adopted_taps = taps;
  f->call.user = f;
  f->L = interp;
  int device = 0;
  const char *env = getenv("XLATING_B200_DEVICE");
  if (env != NULL) {
    device = atoi(env);
  }
  const uint32_t max_in = max_input_buffer_length < 2 ? 2 : max_input_buffer_length;
  int rc;
  if (use_group_model()) {
    rc = xlg_create(device, sampling_freq, max_in, 0, &f->group);
    if (rc == 0)
      rc = interp == 1 ? xlg_add_client(f->group, decimation, taps, taps_len, center_freq, &f->client)
                       : xlg_add_client_rational(f->group, interp, decimation, taps, taps_len, center_freq, &f->client);
  } else {
    rc = filter_build(f, device, interp, decimation, taps, taps_len, center_freq, sampling_freq, max_in);
  }
  if (rc != 0) {
    filter_release(f);
    return rc;
  }
  *filter = f;
  return 0;
}

}  // namespace

extern "C" {

const char *SIMD_STATUS = "CUDA sm_90a";

int create_frequency_xlating_filter(uint32_t decimation, float *taps, size_t taps_len, int32_t center_freq,
                                    uint32_t sampling_freq, uint32_t max_input_buffer_length, xlating **filter) {
  if (taps_len == 0) {
    return -1;  // src/xlating.c:496-498 (taps NOT adopted on this path)
  }
  if (filter == NULL || taps == NULL) {
    return -EINVAL;
  }
  return create_filter(1, decimation, taps, taps_len, center_freq, sampling_freq, max_input_buffer_length, filter);
}

int create_rational_frequency_xlating_filter(uint32_t interpolation, uint32_t decimation, float *taps,
                                             size_t taps_len, int32_t center_freq, uint32_t sampling_freq,
                                             uint32_t max_input_buffer_length, xlating **filter) {
  if (taps_len == 0) {
    return -1;  // as create_frequency_xlating_filter (taps NOT adopted on this path)
  }
  if (filter == NULL || taps == NULL) {
    return -EINVAL;
  }
  // the batch group's rules (xlg_add_client_rational), checked before any CUDA call
  const uint32_t max_in = max_input_buffer_length < 2 ? 2 : max_input_buffer_length;
  const char *why = NULL;
  if (interpolation == 0 || decimation == 0)
    why = "interpolation and decimation must both be at least 1";
  else if ((uint64_t)interpolation * sampling_freq > UINT32_MAX)
    why = "the upsampled rate interpolation x sampling_freq exceeds UINT32_MAX";
  else if ((uint64_t)interpolation * (max_in / 2) >= (1ull << 31))
    why = "interpolation x max_input_buffer_length / 2 upsampled samples per call reach 2^31";
  if (why != NULL) {
    XL_LOG("rational filter %u/%u at %u Hz, blocks of %u: %s", interpolation, decimation, sampling_freq, max_in, why);
    free(taps);  // adopted, as on every other failure but taps_len == 0
    return -EINVAL;
  }
  return create_filter(interpolation, decimation, taps, taps_len, center_freq, sampling_freq,
                       max_input_buffer_length, filter);
}

void destroy_xlating(xlating *filter) {
  if (filter == NULL) {
    return;
  }
  filter_release(filter);
}

int xlg_dropin_stats(int device, uint64_t *batches, uint64_t *calls, uint64_t *shared_inputs) {
  std::lock_guard<std::mutex> lk(g_engines_mu);
  auto it = g_engines.find(device);
  if (it == g_engines.end()) return -ENOENT;
  uint64_t b = 0, c = 0;
  it->second->combiner->stats(&b, &c);
  if (batches != NULL) *batches = b;
  if (calls != NULL) *calls = c;
  uint64_t hits = 0, publishes = 0;
  it->second->cache->stats(&hits, &publishes);
  if (shared_inputs != NULL) *shared_inputs = hits;
  return 0;
}

int xlg_dropin_stream_times(int device, uint64_t *ns7) {
  std::lock_guard<std::mutex> lk(g_engines_mu);
  auto it = g_engines.find(device);
  if (it == g_engines.end() || ns7 == NULL) return -ENOENT;
  Engine *e = it->second;
  memset(ns7, 0, 7 * sizeof(uint64_t));
  for (const Engine::ServedShard &sh : e->served) {
    ns7[0] += sh.call_ns.load();
    ns7[1] += sh.copy_ns.load();
  }
  std::lock_guard<std::mutex> lk2(e->mu);
  for (StreamHost *sh : e->streams) {
    AutoStream *as = sh->as.load();
    if (as == nullptr) continue;
    const AutoStream::Stats st = as->stats();
    ns7[2] += st.ns_compare;
    ns7[3] += st.ns_wait;
    ns7[4] += st.ns_pub_copy;
    ns7[5] += st.ns_pub_submit;
    ns7[6] += st.ns_pub_wait;
  }
  return 0;
}

int xlg_dropin_stream_stats(int device, uint64_t *stats7) {
  std::lock_guard<std::mutex> lk(g_engines_mu);
  auto it = g_engines.find(device);
  if (it == g_engines.end() || stats7 == NULL) return -ENOENT;
  Engine *e = it->second;
  memset(stats7, 0, 7 * sizeof(uint64_t));
  for (const Engine::ServedShard &sh : e->served) stats7[0] += sh.served.load();
  std::lock_guard<std::mutex> lk2(e->mu);
  for (StreamHost *sh : e->streams) {
    AutoStream *as = sh->as.load();
    if (as == nullptr) continue;
    const AutoStream::Stats st = as->stats();
    stats7[1] += st.published;
    stats7[2] += st.hits;
    stats7[3] += st.desyncs;
    stats7[4] += st.joins;
    stats7[5] += st.private_matches;
    stats7[6] += (uint64_t)as->members();
  }
  return 0;
}

#define XL_DEFINE_CF32(variant, name, ctype, fmt)                                                     \
  void process_##variant##_##name##_cf32(const ctype *input, size_t input_len, xlating_cf32 **output, \
                                         size_t *output_len, xlating *filter) {                       \
    run_block(filter, fmt, input, input_len, false, (void **)output, output_len);                     \
  }
#define XL_DEFINE_Q15(variant, name, ctype, fmt)                                                 \
  void process_##variant##_##name##_cs16(const ctype *input, size_t input_len, int16_t **output, \
                                         size_t *output_len, xlating *filter) {                  \
    run_block(filter, fmt, input, input_len, true, (void **)output, output_len);                 \
  }

XL_DEFINE_CF32(native, cu8, uint8_t, XLG_FMT_CU8)
XL_DEFINE_CF32(native, cs8, int8_t, XLG_FMT_CS8)
XL_DEFINE_CF32(native, cs16, int16_t, XLG_FMT_CS16)
XL_DEFINE_CF32(optimized, cu8, uint8_t, XLG_FMT_CU8)
XL_DEFINE_CF32(optimized, cs8, int8_t, XLG_FMT_CS8)
XL_DEFINE_CF32(optimized, cs16, int16_t, XLG_FMT_CS16)
XL_DEFINE_Q15(native, cu8, uint8_t, XLG_FMT_CU8)
XL_DEFINE_Q15(native, cs8, int8_t, XLG_FMT_CS8)
XL_DEFINE_Q15(native, cs16, int16_t, XLG_FMT_CS16)
XL_DEFINE_Q15(optimized, cu8, uint8_t, XLG_FMT_CU8)
XL_DEFINE_Q15(optimized, cs8, int8_t, XLG_FMT_CS8)
XL_DEFINE_Q15(optimized, cs16, int16_t, XLG_FMT_CS16)

}  // extern "C"
