/*
 * csrc/xlating_group.cu -- host side of the batch C ABI (include/xlating_group.h):
 * one wideband stream, many clients, one GPU.
 *
 * Data layout in HBM (per group):
 *   ring / qring     power-of-two ring of converted samples (float2 / short2); the
 *                    absolute stream index s lives at ring[s & mask].  Holds the
 *                    in-flight blocks plus the longest history (T-1 samples), so
 *                    history never has to be moved (the reference memmoves it
 *                    every call, src/xlating.c:76-79).
 *   clients          ClientDev table: decimation phase (hist), oscillator, offsets
 *   taps / qtaps     reversed band-pass taps per client, natural order
 *   tile_taps        the same taps re-packed [class][group of 32][flat tap][32]
 *                    for the tiled kernel's TMA chunks
 *   per slot (XLG_SLOTS in flight): raw input staging, BlkInfo, per-output
 *                    oscillator table, output arena (+ pinned host mirrors)
 *   cascade clients  a stage-A history ring each (HostClient::d_cring), their stage-B taps
 *                    (d_taps2); stage-A rows follow the host-visible rows of the arena
 *   sub-bands        a history ring each (HostClient::d_cring), rows after the host-visible ones;
 *                    their members' taps packed per group of SB_MG (d_sbtaps, SbGroup; branch-major
 *                    for rational members), and per slot the members' oscillator table (d_sbph)
 *
 * Streams: s_in (H2D), s_ph (oscillator pre-pass chain), s_cs[0..n_cs) (convert + FIR,
 * round-robin by block; 3 by default, XLATING_B200_CSTREAMS=1..4), s_out (D2H); events order them per block so block b+1's
 * copy and pre-pass overlap block b's FIR and consecutive FIRs overlap each other.
 * With XLG_SM_PARTITION s_ph lives in an 8-SM green context and the compute streams in the rest.
 *
 * The reference's per-client dsp loop this replaces: src/dsp_worker.c:41-88 calling
 * src/xlating.c:384-414 -> :52-83 once per client per block.
 */
#include <cuda.h>
#include <cuda_runtime.h>
#include <errno.h>
#include <limits.h>
#include <sched.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <chrono>
#include <map>
#include <mutex>
#include <numeric>
#include <tuple>
#include <array>
#include <cstdint>
#include <vector>

#include "taps_host.h"
#include "xl_log.h"
#include "xlating_group.h"
#include "xlating_kernels.cuh"

using namespace xl;


#define CU_OK(expr)                                                                      \
  do {                                                                                   \
    cudaError_t e_ = (expr);                                                             \
    if (e_ != cudaSuccess) {                                                             \
      XL_LOG("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e_), __FILE__, __LINE__); \
      return -EIO;                                                                       \
    }                                                                                    \
  } while (0)

namespace {

constexpr int kTileMinClients = 8;     // smaller aligned classes go to the generic kernel
constexpr int kTileMinOutputs = 12;    // per block; below this even a 16-output tile is mostly idle
// shared memory of an SM (CTAs get kSmSmem / n - 1 KiB each at n per SM)
constexpr int kSmSmem = 228 * 1024;

// The tiled FIR's shapes, largest tile first.  min_ctas = CTAs per SM whose shared memory the
// shape needs (0: any); code = LO*100 + RK*10 + OS, the value XLATING_B200_TILE pins it by.
struct TileShapeHost {
  int lo, rk, os, min_ctas;
  decltype(&fir_tile_cf32_kernel<16, 1, 1>) kernel;
  int threads;
  int kt() const { return lo * rk * os; }
  int code() const { return lo * 100 + rk * 10 + os; }
};
#define XL_TILE_SHAPE(LO_, RK_, OS_, MIN_CTAS_) \
  {LO_, RK_, OS_, MIN_CTAS_, fir_tile_cf32_kernel<LO_, RK_, OS_>, TileShape<LO_, RK_, OS_>::kThreads}
const TileShapeHost kTileShapes[] = {XL_TILE_SHAPE(16, 4, 2, 3), XL_TILE_SHAPE(16, 4, 1, 0), XL_TILE_SHAPE(16, 2, 1, 0),
                                     XL_TILE_SHAPE(16, 1, 1, 0)};
#undef XL_TILE_SHAPE
constexpr int kTileSmallest = sizeof(kTileShapes) / sizeof(kTileShapes[0]) - 1;

// index into kTileShapes of the shape with this code, -1 if none has it
int tile_shape_index(int code) {
  for (int i = 0; i <= kTileSmallest; i++)
    if (kTileShapes[i].code() == code) return i;
  return -1;
}

struct HostClient {
  bool active = false;
  uint32_t D = 0;
  uint32_t L = 1;                // interpolation of a rational client (xlg_add_client_rational)
  size_t T = 0;
  std::vector<float> rev;        // 2*T; a rational client's polyphase branches, 2*L*ceil(T/L)
  std::vector<int16_t> rev_q15;  // 2*T
  float incr_re = 0, incr_im = 0;
  int16_t qincr_re = 0, qincr_im = 0;
  long long hist = 0;            // mirror of ClientDev::hist (upsampled samples for L > 1)
  long long zero_before = 0, qzero_before = 0;
  bool is_new = true;            // dynamic state not yet on the device
  float init_ph_re = 1.0f, init_ph_im = 0.0f;  // oscillator at attach (src/xlating.c:543, or xlg_add_client_ex)
  int kind = 0;
  int out_off = 0, out_cap = 0;
  int taps_off = 0;
  int ph_off = 0;
  bool tile_ineligible = false;  // its class cannot use the tiled kernel (shared memory, too few outputs)
  bool pending_settle = false;   // still inside its zero-history window at the last layout rebuild
  int poly_off = 0, poly_rowcap = 0;  // kind 4: its branches' rows in the slot's polyphase scratch
  // cascade client (xlg_add_client_cascade): everything above describes its stage A, an integer client
  // whose out_off row lies after every host-visible row; stage B is described here
  bool casc = false;
  uint32_t L2 = 1, D2 = 0;       // stage B's interpolation (> 1: xlg_add_client_cascade_rational) and decimation
  size_t T2 = 0;
  int Tb2 = 0, ko2 = 0;          // L2 > 1: taps per branch, outputs per CTA of cascade_fir_poly_cf32_kernel
  std::vector<float> rev2;       // stage B's reversed taps (the real parts of its rotated taps at centre 0),
                                 // packed branch-major (xl_poly_pack) when L2 > 1
  long long hist2 = 0;           // stage B's history_offset, in stage-A samples (upsampled when L2 > 1)
  long long a_pos = 0;           // stage-A outputs produced since the attach: the ring's stream position
  float2 *d_cring = nullptr;     // stage-A history ring, cring_cap samples (a power of two)
  size_t cring_cap = 0;
  int fin_off = 0, fin_cap = 0;  // final row of the slot's output arena
  int taps2_off = 0;             // rev2 in the real tap arena
  int last_n2 = 0;               // stage-B outputs of the block being submitted
  // sub-band (xlg_add_subband): an integer client, not visible to the caller, whose row lies after every
  // host-visible row; d_cring, cring_cap and a_pos above are its history ring
  bool sb = false;
  int sb_id = -1;
  // sub-band member (xlg_add_client_subband[_rational]): not an integer client -- its ClientDev only carries
  // its oscillator; L2, D2, T2, Tb2, hist2 (in sub-band samples, upsampled when L2 > 1) and last_n2 above are
  // its own, rev2 holds its rotated reversed taps (2 * T2 floats; branch-major, 2 * L2 * Tb2, when L2 > 1),
  // out_off / out_cap its final row
  bool mem = false;
  int sb_cid = -1;               // its sub-band's client index
  long long zb2 = 0;             // sub-band position of its attach point: earlier samples read as zero
  int ph_row = 0;                // its rows of the slot's member oscillator table
};

// members of one sub-band that read the same windows: equal (L2, D2, T2, hist2) and, until their windows have
// passed it, the same attach point
struct SbClassHost {
  int sb_cid;
  int L2, Tb;    // Tb: taps per branch (T2 when L2 = 1)
  std::vector<int> members;
  long long zb;  // the largest attach point of its members
};

struct Slot {
  void *d_raw = nullptr, *h_raw = nullptr;
  float2 *d_out = nullptr;
  short2 *d_qout = nullptr;
  float2 *d_phases = nullptr;
  float2 *d_partial = nullptr;  // split-K partial sums of the long-filter classes
  short2 *d_qphases = nullptr;
  BlkInfo *d_blk = nullptr;
  float2 *d_endph = nullptr;  // XLG_TRACK_STATE: every client's oscillator after this block (same capacity as d_blk)
  size_t blk_cap = 0;
  cudaEvent_t ev_h2d = nullptr, ev_conv = nullptr, ev_phase = nullptr, ev_fir = nullptr, ev_done = nullptr;
  cudaEvent_t pf[10] = {nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr, nullptr};
  cudaEvent_t tl_ph[2][2] = {{nullptr, nullptr}, {nullptr, nullptr}};  // timeline: pre-pass stamps, by occupancy parity (it runs a block ahead)
  bool pf_conv = false, pf_phase = false, pf_tile = false, pf_gen = false, pf_long = false;
  cudaEvent_t pf_poly[4] = {nullptr, nullptr, nullptr, nullptr};  // around the polyphase generic / tiled kernels
  bool pf_pg = false, pf_pt = false;
  float2 *d_pscratch = nullptr;  // kind 4: unrotated outputs per branch (ClientDev::poly_off)
  BlkInfo *d_vblk = nullptr, *h_vblk = nullptr;  // kind 4: per branch class, this block's window start and count
  uint64_t poly_macs = 0;
  CascBlk *d_cblk = nullptr, *h_cblk = nullptr;  // cascade clients: this block's ring positions, windows and counts
  size_t cblk_cap = 0;                           // (integer stage B first, then the rational ones)
  CascPolyBlk *d_pblk = nullptr, *h_pblk = nullptr;  // rational cascade clients: this block's stage B
  size_t pblk_cap = 0;
  cudaEvent_t ev_casc = nullptr;                 // stage B of this block done (its rings' appends are ordered on it)
  cudaEvent_t pf_casc[2] = {nullptr, nullptr};
  bool pf_cb = false;
  uint64_t casc_macs = 0, d2h_bytes = 0;
  CascBlk *d_sbcb = nullptr, *h_sbcb = nullptr;  // sub-bands: this block's ring appends
  size_t sbcb_cap = 0;
  SbBlk *d_sbblk = nullptr, *h_sbblk = nullptr;  // member classes: this block's windows and counts
  size_t sbblk_cap = 0;
  float2 *d_sbph = nullptr;                      // member oscillator table (HostClient::ph_row)
  cudaEvent_t pf_sb[2] = {nullptr, nullptr};
  bool pf_sbk = false;
  uint64_t sb_macs = 0, sb_rows = 0;
  std::atomic<int64_t> ticket{-1};
  bool q15 = false;
  bool harvested = true;
  uint64_t tile_macs = 0, algo_macs = 0, out_samples = 0, in_samples = 0;
};

// Optional spatial partition of the GPU (CUDA green contexts): the oscillator
// pre-pass is a latency-bound dependent chain (8-14 cycles per output, one lane
// per client); when it shares an SM sub-partition with FIR warps that can issue an
// FMA every cycle it loses the issue arbitration and runs 3x slower, which then
// bounds the whole pipeline.  Giving it 8 SMs of its own (the minimum partition on
// sm_90) and the FIR the other 124 of an H100's 132 removes that stall for a few
// percent of the FIR's SMs.
// The driver entry points are resolved at run time (cudaGetDriverEntryPoint) so
// the library has no link-time dependency on libcuda.
struct SmPartition {
  CUgreenCtx small_ctx = nullptr, big_ctx = nullptr;
  int small_sms = 0, big_sms = 0;
  bool ok = false;
};

typedef CUresult (*pfn_cuDeviceGet)(CUdevice *, int);
typedef CUresult (*pfn_cuDeviceGetDevResource)(CUdevice, CUdevResource *, CUdevResourceType);
typedef CUresult (*pfn_cuDevSmResourceSplitByCount)(CUdevResource *, unsigned int *, const CUdevResource *,
                                                    CUdevResource *, unsigned int, unsigned int);
typedef CUresult (*pfn_cuDevResourceGenerateDesc)(CUdevResourceDesc *, CUdevResource *, unsigned int);
typedef CUresult (*pfn_cuGreenCtxCreate)(CUgreenCtx *, CUdevResourceDesc, CUdevice, unsigned int);
typedef CUresult (*pfn_cuGreenCtxDestroy)(CUgreenCtx);
typedef CUresult (*pfn_cuGreenCtxStreamCreate)(CUstream *, CUgreenCtx, unsigned int, int);

template <typename F>
static bool drv(const char *name, F *fn) {
  void *p = nullptr;
  cudaDriverEntryPointQueryResult q;
  if (cudaGetDriverEntryPoint(name, &p, cudaEnableDefault, &q) != cudaSuccess || q != cudaDriverEntryPointSuccess ||
      p == nullptr) {
    cudaGetLastError();
    return false;
  }
  *fn = reinterpret_cast<F>(p);
  return true;
}

// Host-visible results of one ticket.  There are `host_ring` of these (>= XLG_SLOTS):
// the device pipeline is XLG_SLOTS deep, but results stay readable for host_ring
// tickets so that a consumer thread blocked on a slow socket does not lose data
// (the reference absorbs that with a 64-block queue per client, src/config.c:183).
// Per-ticket metadata array that consumer threads read WITHOUT a lock (xlg_copy_output: the
// entry's ticket is the sequence number of a seqlock -- xlg_submit sets it to -1 before it
// touches the array and to the new ticket afterwards).  The storage only ever grows; an
// outgrown array is retired, never freed while the group lives, so a reader that raced with
// the growth still reads valid memory (and is then rejected by the ticket check).
template <typename T>
struct MetaArr {
  std::atomic<T *> p{nullptr};
  size_t cap = 0;
  std::atomic<size_t> n{0};
  std::vector<T *> *retired = nullptr;
  MetaArr() = default;
  MetaArr(const MetaArr &) : p(nullptr), cap(0), n(0), retired(nullptr) {}  // (vector<HostOut> construction only)
  size_t size() const { return n.load(std::memory_order_relaxed); }
  T &operator[](size_t i) { return p.load(std::memory_order_relaxed)[i]; }
  T get(size_t i) const { return p.load(std::memory_order_acquire)[i]; }
  void assign(size_t count, T value) {
    if (count > cap) {
      const size_t ncap = std::max<size_t>(count * 2, 64);
      T *fresh = new T[ncap];
      T *old = p.load();
      if (old != nullptr && retired != nullptr) retired->push_back(old);
      p.store(fresh, std::memory_order_release);
      cap = ncap;
    }
    T *a = p.load();
    for (size_t i = 0; i < count; i++) a[i] = value;
    n.store(count, std::memory_order_release);
  }
  void release() {
    delete[] p.load();
    p.store(nullptr);
    cap = 0;
  }
};

struct HostOut {
  std::atomic<int64_t> ticket{-1};
  bool q15 = false;
  float2 *h_out = nullptr;   // pinned; nullptr for XLG_OUT_DEVICE groups
  short2 *h_qout = nullptr;
  MetaArr<int> n_out;    // per client id
  MetaArr<int> out_off;  // per client id
  MetaArr<long long> hist_after;  // XLG_TRACK_STATE: per client id, history_offset after this ticket
  float2 *h_endph = nullptr;          // XLG_TRACK_STATE: pinned, oscillator after this ticket, per client id
  size_t endph_cap = 0;
};

struct TileClassHost {
  TileClass k;
  std::vector<int> members;  // client id per member slot, -1 = padding; 32 slots per group
  std::vector<int> real;     // the real client ids
  size_t T;
  bool merged = false;       // members may have different window alignments (natural layout only)
  int branch = -1;           // rational (kind 4) classes: the polyphase branch r this class computes
  uint32_t interp = 1;
  long long minv = 0;        // decimation^-1 mod interp
};

}  // namespace

struct xlg_group {
  int device = 0;
  uint32_t fs = 0;
  uint32_t max_input_len = 0;  // scalar elements
  uint32_t flags = 0;
  cudaStream_t s_in = nullptr, s_ph = nullptr, s_out = nullptr;
  // raw -> ring conversion: its own stream, in the oscillator partition (or at high priority without one), so
  // that block b+1's conversion never queues behind the CTAs of block b's FIR that are still waiting for an SM
  cudaEvent_t ev_user = nullptr;  // xlg_wait_stream: recorded on the caller's stream, waited for by the next submit's first reader
  bool user_wait_pending = false;
  cudaStream_t s_cv = nullptr;
  bool conv_own_stream = true;  // XLATING_B200_CONV_STREAM=0: convert on the block's compute stream (the old order)
  static constexpr int kMaxCs = 4;
  cudaStream_t s_cs[kMaxCs] = {nullptr, nullptr, nullptr, nullptr};  // compute streams, round-robin by block
  int n_cs = 3;  // compute streams used round-robin (XLATING_B200_CSTREAMS)
  SmPartition part;
  // Two complete sets of pre-pass / conversion / compute streams: inside the green contexts (8 SMs + the rest) and
  // ordinary ones (all SMs).  s_ph / s_cv / s_cs alias the ACTIVE set; with XLG_SM_PARTITION the choice is made
  // per layout (rebuild_layout: the partition pays only where the oscillator chain, ~5x slower when it shares SMs
  // with FIR warps, would otherwise pace the pipeline), XLATING_B200_PARTITION=0/1 forces it.
  struct StreamSet {
    cudaStream_t ph = nullptr, cv = nullptr, cs[4] = {nullptr, nullptr, nullptr, nullptr};
  } set_part, set_plain;
  bool part_active = false;
  int part_force = -1;    // -1 = automatic
  int total_sms = 0;
  double sm_mhz = 0;      // SM clock the device reports (the partition's cost model is in cycles)

  float2 *ring = nullptr;
  short2 *qring = nullptr;
  size_t ring_cap = 0;    // samples, power of two
  size_t hist_cap = 0;    // longest T-1 the ring was sized for
  long long S = 0, qS = 0;  // absolute stream positions of the two paths

  std::vector<HostClient> clients;
  ClientDev *d_clients = nullptr;
  size_t d_clients_cap = 0;
  // Speculative oscillator pre-pass.  The pre-pass of a block depends on its LENGTH only, and
  // SDR blocks all have the same length: right after block t's pre-pass the one of block t+1
  // is launched for "the same length again" (after saving the client table).  If the next
  // submit is what was guessed, its pre-pass is already done -- a lone block then takes
  // convert + FIR instead of 49 us of dependent chain + FIR; otherwise the table is restored
  // and the pre-pass runs as before.  XLATING_B200_SPECULATE=0 turns it off.
  SpecSave *d_clients_backup = nullptr;  // (hist, oscillator) of every client before the speculative pre-pass
  bool speculate = true;
  bool spec_valid = false;
  long long spec_S = 0;
  int spec_n = 0;
  int64_t spec_ticket = -1;
  uint64_t spec_hits = 0, spec_misses = 0;
  float2 *d_taps = nullptr;
  short2 *d_qtaps = nullptr;
  void *d_tile_taps = nullptr;
  std::vector<float2> h_taps, h_tile_taps;  // host staging of the tap arenas, kept between re-layouts (no fresh pages)
  std::vector<short2> h_qtaps;
  size_t cap_taps = 0, cap_qtaps = 0, cap_tile_taps = 0, cap_members = 0, cap_member_cid = 0, cap_member_incr = 0;
  int tile_force = 0;     // XLATING_B200_TILE=<LO*100+RK*10+OS> pins the tile shape (1642, 1641, 1621 or 1611)
  // long4's input strips through a TMA tensor map over the ring (XLATING_B200_LONG_TMAP=0: 28 bulk copies per stage)
  bool long_tmap = true;
  CUtensorMap strip_map;          // valid for (strip_ring, strip_cap, strip_D)
  const void *strip_ring = nullptr;
  size_t strip_cap = 0;
  int strip_D = 0, strip_w = 0;   // strip_w: inner width of the map in samples (0 = could not be encoded)
  int fir_sms = 0;        // SMs the FIR kernels can use (all, or all minus the reserved partition)
  int *d_members = nullptr;
  int *d_member_cid = nullptr;      // client id per member slot (-1 = padding)
  float2 *d_member_incr = nullptr;  // oscillator step per member slot (same indexing as d_members)
  int *d_order = nullptr;   // clients in oscillator-table order, 32 per group, -1 = padding
  int n_order = 0;
  size_t phase_cap = 0;     // float2 per slot oscillator table
  size_t arena_cap = 0;   // complex samples per slot arena
  bool q_alloc = false;

  std::vector<TileClassHost> classes;
  std::vector<TileClassHost> long_classes;  // split-K long-filter classes (fir_long4 / fir_long2)
  std::vector<TileClassHost> poly_classes;  // kind 4: one class per (rational class, polyphase branch)
  bool poly_tile = true;                    // XLATING_B200_POLY_TILE=0: every rational client on the generic kernel
  int *d_poly3 = nullptr, *d_poly4 = nullptr;  // ids of the kind-3 / kind-4 clients
  size_t cap_poly3 = 0, cap_poly4 = 0;
  int n_poly3 = 0, n_poly4 = 0;
  float2 *d_ones = nullptr;                 // phase 1 + 0i for the kind-4 classes' tiled launch
  size_t ones_cap = 0, pscratch_cap = 0;
  size_t partial_cap = 0;                   // float2 per slot partial-sum buffer
  float *d_taps2 = nullptr;                 // cascade clients' stage-B taps (HostClient::taps2_off)
  size_t cap_taps2 = 0;
  int n_casc = 0;                           // active cascade clients
  int n_casc_int = 0;                       // of which integer stage B (their CascBlk entries come first)
  std::vector<float2 *> dead_rings;         // rings of removed cascade clients, freed once the pipeline is drained
  cudaEvent_t ev_last_casc = nullptr;       // ev_casc of the last block with cascade clients or sub-bands
  bool have_last_casc = false;
  std::vector<int> subbands;                // sub-band id -> client index (-1 = free)
  std::vector<int> sb_list;                 // active sub-bands' client indices (their appends, in this order)
  std::vector<SbClassHost> sb_classes;
  int n_sb_mem = 0, n_sb_groups = 0;
  int n_sb_groups_int = 0;                  // of which integer classes' (their SbGroup entries come first)
  SbGroup *d_sbgrp = nullptr;
  SbMem *d_sbmem = nullptr;
  float2 *d_sbtaps = nullptr;
  size_t cap_sbgrp = 0, cap_sbmem = 0, cap_sbtaps = 0, sbph_cap = 0;
  xlg_subband_profile sb_prof;
  int n_generic = 0;
  int max_client = 0;     // highest active id + 1
  bool dirty = true;

  Slot slots[XLG_SLOTS];
  std::vector<HostOut> ring_out;  // indexed by ticket % ring_out.size()
  std::vector<void *> retired_host;
  std::vector<int *> retired_meta_i;        // outgrown MetaArr storage (see MetaArr)
  std::vector<long long *> retired_meta_ll;
  long long *d_trace = nullptr;  // XLATING_B200_TRACE=1: per-CTA timeline of the tiled kernel
  int trace_ctas = 0;
  // XLATING_B200_TIMELINE=path: GPU timestamps (ms since the first submit) of every block's kernels in the
  // REAL pipeline (all streams, speculation on): conv ready/done, phase start/done, FIR ready/done
  bool timeline = false;
  cudaEvent_t ev_base = nullptr;
  bool base_recorded = false;
  std::vector<std::array<float, 7>> tl;
  long long trace_launches = 0;  // tiled launches so far (the timeline keeps the last T_TRACE_LAUNCHES)
  int trace_n[T_TRACE_LAUNCHES] = {0};
  std::atomic<int64_t> next_ticket{0};
  cudaEvent_t ev_last_conv_ref = nullptr;  // ev_conv of the previous block's slot (history dependency)
  bool have_last_conv = false;
  cudaEvent_t ev_t0 = nullptr, ev_t1 = nullptr;

  bool profiling = false;
  xlg_profile prof;
  xlg_poly_profile poly_prof;
  xlg_cascade_profile casc_prof;
  uint64_t host_submit_ns = 0, host_wait_ns = 0, host_count_base = 0;
  std::mutex mu;  // guards slots' harvest + profile
};

// ---------------------------------------------------------------------------
// helpers
// ---------------------------------------------------------------------------

static size_t next_pow2(size_t v) {
  size_t p = 1;
  while (p < v) p <<= 1;
  return p;
}

static int elem_bytes(int fmt) { return fmt == XLG_FMT_CS16 ? 2 : 1; }

static void slot_free(Slot &s) {
  if (s.d_raw) cudaFree(s.d_raw);
  if (s.h_raw) cudaFreeHost(s.h_raw);
  if (s.d_out) cudaFree(s.d_out);
  if (s.d_qout) cudaFree(s.d_qout);
  if (s.d_phases) cudaFree(s.d_phases);
  if (s.d_partial) cudaFree(s.d_partial);
  if (s.d_qphases) cudaFree(s.d_qphases);
  if (s.d_blk) cudaFree(s.d_blk);
  if (s.d_endph) cudaFree(s.d_endph);
  if (s.d_pscratch) cudaFree(s.d_pscratch);
  if (s.d_vblk) cudaFree(s.d_vblk);
  if (s.h_vblk) cudaFreeHost(s.h_vblk);
  if (s.d_cblk) cudaFree(s.d_cblk);
  if (s.h_cblk) cudaFreeHost(s.h_cblk);
  s.d_cblk = s.h_cblk = nullptr;
  s.cblk_cap = 0;
  if (s.d_pblk) cudaFree(s.d_pblk);
  if (s.h_pblk) cudaFreeHost(s.h_pblk);
  s.d_pblk = s.h_pblk = nullptr;
  s.pblk_cap = 0;
  if (s.d_sbcb) cudaFree(s.d_sbcb);
  if (s.h_sbcb) cudaFreeHost(s.h_sbcb);
  if (s.d_sbblk) cudaFree(s.d_sbblk);
  if (s.h_sbblk) cudaFreeHost(s.h_sbblk);
  if (s.d_sbph) cudaFree(s.d_sbph);
  s.d_sbcb = s.h_sbcb = nullptr;
  s.d_sbblk = s.h_sbblk = nullptr;
  s.d_sbph = nullptr;
  s.sbcb_cap = s.sbblk_cap = 0;
  s.d_pscratch = nullptr;
  s.d_vblk = s.h_vblk = nullptr;
  s.d_endph = nullptr;
  s.d_raw = s.h_raw = nullptr;
  s.d_out = nullptr;
  s.d_qout = nullptr;
  s.d_phases = nullptr;
  s.d_partial = nullptr;
  s.d_qphases = nullptr;
  s.d_blk = nullptr;
}

static int drain(xlg_group *g) {
  CU_OK(cudaStreamSynchronize(g->s_in));
  for (const xlg_group::StreamSet *ss : {&g->set_part, &g->set_plain}) {
    if (ss->ph) CU_OK(cudaStreamSynchronize(ss->ph));
    if (ss->cv) CU_OK(cudaStreamSynchronize(ss->cv));
    for (cudaStream_t st : ss->cs)
      if (st) CU_OK(cudaStreamSynchronize(st));
  }
  CU_OK(cudaStreamSynchronize(g->s_out));
  return 0;
}

static void harvest_locked(xlg_group *g, Slot &s) {
  if (s.harvested) return;
  s.harvested = true;
  if (g->timeline && g->base_recorded && s.pf_conv && s.pf_phase && s.pf_tile) {
    std::array<float, 7> r;
    r[0] = (float)s.ticket.load();
    const int par = (int)((s.ticket.load() / XLG_SLOTS) & 1);
    for (int i = 0; i < 6; i++) {
      cudaEvent_t e = (i == 2 || i == 3) ? s.tl_ph[par][i - 2] : s.pf[i];
      if (cudaEventElapsedTime(&r[1 + i], g->ev_base, e) != cudaSuccess) r[1 + i] = -1.f;
    }
    g->tl.push_back(r);
    cudaGetLastError();
  }
  if (!g->profiling) return;
  float ms = 0;
  if (s.pf_conv && cudaEventElapsedTime(&ms, s.pf[0], s.pf[1]) == cudaSuccess) {
    g->prof.convert_ms += ms;
    g->prof.convert_launches++;
  }
  if (s.pf_phase && cudaEventElapsedTime(&ms, s.pf[2], s.pf[3]) == cudaSuccess) {
    g->prof.phase_ms += ms;
    g->prof.phase_launches++;
  }
  if (s.pf_tile && cudaEventElapsedTime(&ms, s.pf[4], s.pf[5]) == cudaSuccess) {
    g->prof.fir_tile_ms += ms;
    g->prof.fir_tile_launches++;
  }
  if (s.pf_gen && cudaEventElapsedTime(&ms, s.pf[6], s.pf[7]) == cudaSuccess) {
    g->prof.fir_generic_ms += ms;
    g->prof.fir_generic_launches++;
  }
  if (s.pf_long && cudaEventElapsedTime(&ms, s.pf[8], s.pf[9]) == cudaSuccess) {
    g->prof.fir_long_ms += ms;
    g->prof.fir_long_launches++;
  }
  if (s.pf_pg && cudaEventElapsedTime(&ms, s.pf_poly[0], s.pf_poly[1]) == cudaSuccess) {
    g->poly_prof.fir_poly_generic_ms += ms;
    g->poly_prof.fir_poly_generic_launches++;
  }
  if (s.pf_pt && cudaEventElapsedTime(&ms, s.pf_poly[2], s.pf_poly[3]) == cudaSuccess) {
    g->poly_prof.fir_poly_tile_ms += ms;
    g->poly_prof.fir_poly_tile_launches++;
  }
  g->poly_prof.poly_macs += s.poly_macs;
  if (s.pf_cb && cudaEventElapsedTime(&ms, s.pf_casc[0], s.pf_casc[1]) == cudaSuccess) {
    g->casc_prof.stage_b_ms += ms;
    g->casc_prof.stage_b_launches++;
  }
  g->casc_prof.stage_b_macs += s.casc_macs;
  g->casc_prof.d2h_bytes += s.d2h_bytes;
  if (s.pf_sbk && cudaEventElapsedTime(&ms, s.pf_sb[0], s.pf_sb[1]) == cudaSuccess) {
    g->sb_prof.member_ms += ms;
    g->sb_prof.member_launches++;
  }
  g->sb_prof.member_macs += s.sb_macs;
  g->sb_prof.row_samples += s.sb_rows;
  g->prof.blocks++;
  g->prof.out_samples += s.out_samples;
  g->prof.in_samples += s.in_samples;
  g->prof.tile_macs += s.tile_macs;
  g->prof.algo_macs += s.algo_macs;
}

// (re)allocate the sample rings so that they hold XLG_SLOTS blocks + history
static int ensure_ring(xlg_group *g, size_t need_hist, bool need_q) {
  const size_t max_n = g->max_input_len / 2;
  if (g->ring && need_hist <= g->hist_cap && (!need_q || g->qring)) return 0;
  const size_t hist_cap = std::max<size_t>(std::max(need_hist, g->hist_cap), 4096);
  const size_t cap = next_pow2((XLG_SLOTS + 1) * max_n + hist_cap + 64);
  if (drain(g)) return -EIO;
  if (!g->ring || cap != g->ring_cap) {
    float2 *nr = nullptr;
    CU_OK(cudaMalloc(&nr, cap * sizeof(float2)));
    CU_OK(cudaMemset(nr, 0, cap * sizeof(float2)));
    if (g->ring) {
      // keep the most recent samples at their new ring positions
      const size_t keep = std::min<size_t>(g->ring_cap, (size_t)std::max<long long>(g->S, 0));
      std::vector<float2> tmp(g->ring_cap);
      CU_OK(cudaMemcpy(tmp.data(), g->ring, g->ring_cap * sizeof(float2), cudaMemcpyDeviceToHost));
      std::vector<float2> fresh(cap, make_float2(0.f, 0.f));
      for (size_t i = 1; i <= keep; i++) {
        const unsigned long long ab = (unsigned long long)(g->S - (long long)i);
        fresh[ab & (cap - 1)] = tmp[ab & (g->ring_cap - 1)];
      }
      CU_OK(cudaMemcpy(nr, fresh.data(), cap * sizeof(float2), cudaMemcpyHostToDevice));
      cudaFree(g->ring);
    }
    g->ring = nr;
    if (g->qring) {
      short2 *nq = nullptr;
      CU_OK(cudaMalloc(&nq, cap * sizeof(short2)));
      const size_t keep = std::min<size_t>(g->ring_cap, (size_t)std::max<long long>(g->qS, 0));
      std::vector<short2> tmp(g->ring_cap);
      CU_OK(cudaMemcpy(tmp.data(), g->qring, g->ring_cap * sizeof(short2), cudaMemcpyDeviceToHost));
      std::vector<short2> fresh(cap, make_short2(0, 0));
      for (size_t i = 1; i <= keep; i++) {
        const unsigned long long ab = (unsigned long long)(g->qS - (long long)i);
        fresh[ab & (cap - 1)] = tmp[ab & (g->ring_cap - 1)];
      }
      CU_OK(cudaMemcpy(nq, fresh.data(), cap * sizeof(short2), cudaMemcpyHostToDevice));
      cudaFree(g->qring);
      g->qring = nq;
    }
    g->ring_cap = cap;
  }
  if (need_q && !g->qring) {
    CU_OK(cudaMalloc(&g->qring, g->ring_cap * sizeof(short2)));
    CU_OK(cudaMemset(g->qring, 0, g->ring_cap * sizeof(short2)));
  }
  g->hist_cap = hist_cap;
  return 0;
}

static int ensure_arenas(xlg_group *g, size_t need, bool need_q) {
  const bool dev_out = (g->flags & XLG_OUT_DEVICE) != 0;
  if (need > g->arena_cap) {
    const size_t cap = std::max<size_t>(need + need / 4, 1024);
    for (Slot &s : g->slots) {
      if (s.d_out) cudaFree(s.d_out);
      s.d_out = nullptr;
      CU_OK(cudaMalloc(&s.d_out, cap * sizeof(float2)));
      if (g->q_alloc) {
        if (s.d_qout) cudaFree(s.d_qout);
        if (s.d_qphases) cudaFree(s.d_qphases);
        s.d_qout = nullptr;
        s.d_qphases = nullptr;
        CU_OK(cudaMalloc(&s.d_qout, cap * sizeof(short2)));
        CU_OK(cudaMalloc(&s.d_qphases, cap * sizeof(short2)));
      }
    }
    for (HostOut &h : g->ring_out) {
      float2 *n_out = nullptr;
      short2 *n_qout = nullptr;
      if (!dev_out) {
        CU_OK(cudaHostAlloc(&n_out, cap * sizeof(float2), cudaHostAllocDefault));
        if (g->q_alloc) CU_OK(cudaHostAlloc(&n_qout, cap * sizeof(short2), cudaHostAllocDefault));
      }
      std::lock_guard<std::mutex> lk(g->mu);
      h.ticket.store(-1);  // resized: older results are gone
      // a consumer thread may still be writing an old result to its socket: the old
      // pinned arenas are retired, not freed, until the group is destroyed
      if (h.h_out) g->retired_host.push_back(h.h_out);
      if (h.h_qout) g->retired_host.push_back(h.h_qout);
      h.h_out = n_out;
      h.h_qout = n_qout;
    }
    g->arena_cap = cap;
  }
  if (need_q && !g->q_alloc) {
    for (Slot &s : g->slots) {
      CU_OK(cudaMalloc(&s.d_qout, std::max<size_t>(g->arena_cap, 1) * sizeof(short2)));
      CU_OK(cudaMalloc(&s.d_qphases, std::max<size_t>(g->arena_cap, 1) * sizeof(short2)));
    }
    if (!dev_out)
      for (HostOut &h : g->ring_out)
        CU_OK(cudaHostAlloc(&h.h_qout, std::max<size_t>(g->arena_cap, 1) * sizeof(short2), cudaHostAllocDefault));
    g->q_alloc = true;
  }
  return 0;
}

// Re-derive everything that depends on the client set: output offsets, tap
// arenas, kernel classes.  Dynamic per-client state (hist, phase) lives on the
// device and is preserved.
static void choose_partition(xlg_group *g);
// (re)fill a device array; the allocation is reused while it is large enough (a re-layout per attach must not
// pay a cudaFree + cudaMalloc -- each an implicit device synchronisation -- for every table)
template <typename T>
static int dev_assign(T **dptr, size_t *cap_bytes, const void *src, size_t bytes) {
  if (bytes == 0) return 0;
  if (*dptr == nullptr || *cap_bytes < bytes) {
    if (*dptr) cudaFree(*dptr);
    *dptr = nullptr;
    const size_t want = bytes + bytes / 4 + 4096;
    CU_OK(cudaMalloc(dptr, want));
    *cap_bytes = want;
  }
  CU_OK(cudaMemcpy(*dptr, src, bytes, cudaMemcpyHostToDevice));
  return 0;
}
// first input sample a client's next window reads: floor((L*S - hist) / L)  (S - hist for integer clients)
static long long first_input(const HostClient &h, long long S) {
  const long long fu = S * h.L - h.hist;
  return fu >= 0 ? fu / h.L : -((-fu + h.L - 1) / h.L);
}
// its zero-history window has passed (or the ring itself is still zero there): it may join a tiled class
static bool poly_settled(const xlg_group *g, const HostClient &h) {
  return (h.zero_before == 0 && g->S < (long long)g->ring_cap / 2) || h.zero_before <= first_input(h, g->S);
}
// Sub-bands and their members (the pipeline is drained): sub-band rows after every host-visible row (the
// D2H copy ends before them), one zeroed history ring per sub-band, grown when a longer member attaches,
// the member classes, their groups of SB_MG members with packed taps, and the per-slot tables.
static int rebuild_subbands(xlg_group *g, size_t &out_total) {
  g->sb_list.clear();
  g->sb_classes.clear();
  g->n_sb_mem = g->n_sb_groups = g->n_sb_groups_int = 0;
  const int nc = (int)g->clients.size();
  for (int i = 0; i < nc; i++)
    if (g->clients[i].active && g->clients[i].sb) g->sb_list.push_back(i);
  if (g->sb_list.empty()) return 0;
  CU_OK(cudaFuncSetAttribute(subband_fir_cf32_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kTileMaxSmem));
  std::vector<size_t> back(nc, 0);  // longest member history per sub-band
  // integer classes (L2 = 1) and rational ones apart: the integer classes' groups come first
  std::map<std::tuple<int, uint32_t, size_t, long long, long long>, std::vector<int>> keyed;
  std::map<std::tuple<int, uint32_t, uint32_t, size_t, long long, long long>, std::vector<int>> keyed_rat;
  bool any_rat = false;
  for (int i = 0; i < nc; i++) {
    const HostClient &h = g->clients[i];
    if (!h.active || !h.mem) continue;
    // a rational member's history of at most T2 - 1 upsampled samples reaches back ceil((T2 - 1) / L2)
    // sub-band samples, and its last branch may read one zero-weighted sample past the block
    back[h.sb_cid] = std::max(back[h.sb_cid], h.L2 == 1 ? h.T2 - 1 : (h.T2 - 1 + h.L2 - 1) / h.L2 + 1);
    // its window has passed its attach point: it reads what every settled member of the class reads
    const bool settled = h.zb2 * (long long)h.L2 <= (long long)h.L2 * g->clients[h.sb_cid].a_pos - h.hist2;
    if (h.L2 == 1) {
      keyed[std::make_tuple(h.sb_cid, h.D2, h.T2, h.hist2, settled ? LLONG_MIN : h.zb2)].push_back(i);
    } else {
      keyed_rat[std::make_tuple(h.sb_cid, h.L2, h.D2, h.T2, h.hist2, settled ? LLONG_MIN : h.zb2)].push_back(i);
      any_rat = true;
    }
  }
  if (any_rat)
    CU_OK(cudaFuncSetAttribute(subband_fir_poly_cf32_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                               kTileMaxSmem));
  for (int i : g->sb_list) {
    HostClient &h = g->clients[i];
    h.out_off = (int)out_total;
    out_total += (size_t)h.out_cap;
    out_total = (out_total + 3) & ~(size_t)3;
    // a member of block b reads sub-band samples of earlier blocks; the submit of block b + XLG_SLOTS waits
    // for ticket b, so its history (above) + (XLG_SLOTS + 1) * max n1 samples are never overwritten while
    // still needed
    const size_t cap = next_pow2(back[i] + (size_t)(XLG_SLOTS + 1) * (size_t)h.out_cap);
    if (h.d_cring != nullptr && cap <= h.cring_cap) continue;
    float2 *ring = nullptr;
    CU_OK(cudaMalloc(&ring, cap * sizeof(float2)));
    std::vector<float2> fresh(cap, make_float2(0.f, 0.f));
    if (h.d_cring != nullptr) {
      // grow: the last cring_cap positions keep their samples at their new places
      std::vector<float2> old(h.cring_cap);
      CU_OK(cudaMemcpy(old.data(), h.d_cring, h.cring_cap * sizeof(float2), cudaMemcpyDeviceToHost));
      for (size_t k = 1; k <= h.cring_cap; k++) {
        const unsigned long long p = (unsigned long long)(h.a_pos - (long long)k);
        fresh[p & (cap - 1)] = old[p & (h.cring_cap - 1)];
      }
      cudaFree(h.d_cring);
    }
    CU_OK(cudaMemcpy(ring, fresh.data(), cap * sizeof(float2), cudaMemcpyHostToDevice));
    h.d_cring = ring;
    h.cring_cap = cap;
  }
  std::vector<SbGroup> groups;
  std::vector<SbMem> mems;
  std::vector<float2> taps;
  // one class: its groups of SB_MG members, taps [branch][SB_MG][tpad] per group, so that one bulk copy
  // stages one branch for the group (a single branch, the reversed taps themselves, when L2 = 1)
  auto add_class = [&](int sb_cid, const std::vector<int> &members) {
    const int cls = (int)g->sb_classes.size();
    SbClassHost ch;
    ch.sb_cid = sb_cid;
    ch.members = members;
    ch.zb = LLONG_MIN;
    const HostClient &h0 = g->clients[members[0]];
    ch.L2 = (int)h0.L2;
    ch.Tb = h0.L2 == 1 ? (int)h0.T2 : h0.Tb2;
    const int tpad = sb_tpad(ch.Tb);
    for (size_t m0 = 0; m0 < ch.members.size(); m0 += SB_MG) {
      SbGroup gp;
      memset(&gp, 0, sizeof(gp));
      gp.cls = cls;
      gp.n_mem = (int)std::min<size_t>(SB_MG, ch.members.size() - m0);
      gp.taps_off = (int)taps.size();
      gp.l2 = ch.L2;
      taps.resize(taps.size() + (size_t)ch.L2 * SB_MG * tpad, make_float2(0.f, 0.f));
      for (int m = 0; m < gp.n_mem; m++) {
        HostClient &h = g->clients[ch.members[m0 + m]];
        for (int r = 0; r < ch.L2; r++)
          memcpy(&taps[gp.taps_off + ((size_t)r * SB_MG + m) * tpad], h.rev2.data() + 2 * (size_t)r * ch.Tb,
                 2 * (size_t)ch.Tb * sizeof(float));
        mems.push_back(SbMem{ch.members[m0 + m], cls, 0});
        ch.zb = std::max(ch.zb, h.zb2);
      }
      groups.push_back(gp);
    }
    g->sb_classes.push_back(ch);
  };
  for (auto &kv : keyed) add_class(std::get<0>(kv.first), kv.second);
  g->n_sb_groups_int = (int)groups.size();
  for (auto &kv : keyed_rat) add_class(std::get<0>(kv.first), kv.second);
  // oscillator table: groups of 32 members in SbMem order, phase of even output k of slot l at
  // base + 32 * (k / 2) + l
  size_t rows = 0;
  for (size_t base = 0; base < mems.size(); base += 32) {
    int cap = 0;
    for (size_t i = base; i < std::min(base + 32, mems.size()); i++) cap = std::max(cap, g->clients[mems[i].cid].out_cap);
    for (size_t i = base; i < std::min(base + 32, mems.size()); i++) {
      mems[i].ph_off = (int)(rows + (i - base));
      g->clients[mems[i].cid].ph_row = mems[i].ph_off;
    }
    rows += (size_t)(cap / 2 + 1) * 32;
  }
  {
    size_t i = 0;
    for (SbGroup &gp : groups)
      for (int m = 0; m < gp.n_mem; m++, i++) {
        const HostClient &h = g->clients[mems[i].cid];
        gp.out_off[m] = h.out_off;
        gp.ph_off[m] = h.ph_row;
        gp.incr[m] = make_float2(h.incr_re, h.incr_im);
      }
  }
  g->n_sb_mem = (int)mems.size();
  while (mems.size() % 32 != 0) mems.push_back(SbMem{-1, 0, 0});
  g->n_sb_groups = (int)groups.size();
  if (dev_assign(&g->d_sbgrp, &g->cap_sbgrp, groups.data(), groups.size() * sizeof(SbGroup)) ||
      dev_assign(&g->d_sbmem, &g->cap_sbmem, mems.data(), mems.size() * sizeof(SbMem)) ||
      dev_assign(&g->d_sbtaps, &g->cap_sbtaps, taps.data(), taps.size() * sizeof(float2)))
    return -EIO;
  const size_t n_sb = g->sb_list.size(), n_cls = g->sb_classes.size();
  const bool grow_ph = rows > g->sbph_cap;
  if (grow_ph) g->sbph_cap = rows + rows / 4 + 1024;
  for (Slot &s : g->slots) {
    if (s.pf_sb[0] == nullptr)
      for (cudaEvent_t &ev : s.pf_sb) CU_OK(cudaEventCreate(&ev));
    if (s.sbcb_cap < n_sb) {
      if (s.d_sbcb) cudaFree(s.d_sbcb);
      if (s.h_sbcb) cudaFreeHost(s.h_sbcb);
      s.d_sbcb = s.h_sbcb = nullptr;
      s.sbcb_cap = std::max<size_t>(n_sb * 2, 16);
      CU_OK(cudaMalloc(&s.d_sbcb, s.sbcb_cap * sizeof(CascBlk)));
      CU_OK(cudaHostAlloc(&s.h_sbcb, s.sbcb_cap * sizeof(CascBlk), cudaHostAllocDefault));
    }
    if (s.sbblk_cap < n_cls) {
      if (s.d_sbblk) cudaFree(s.d_sbblk);
      if (s.h_sbblk) cudaFreeHost(s.h_sbblk);
      s.d_sbblk = s.h_sbblk = nullptr;
      s.sbblk_cap = std::max<size_t>(n_cls * 2, 16);
      CU_OK(cudaMalloc(&s.d_sbblk, s.sbblk_cap * sizeof(SbBlk)));
      CU_OK(cudaHostAlloc(&s.h_sbblk, s.sbblk_cap * sizeof(SbBlk), cudaHostAllocDefault));
    }
    if ((grow_ph || s.d_sbph == nullptr) && g->sbph_cap > 0) {
      if (s.d_sbph) cudaFree(s.d_sbph);
      s.d_sbph = nullptr;
      CU_OK(cudaMalloc(&s.d_sbph, g->sbph_cap * sizeof(float2)));
    }
  }
  return 0;
}

static int rebuild_layout(xlg_group *g) {
  // XLATING_B200_REBUILD_TIMING=1: where a re-layout spends its time (logged per call)
  static const bool timing = getenv("XLATING_B200_REBUILD_TIMING") != nullptr;
  auto t_prev = std::chrono::steady_clock::now();
  double t_stage[6] = {0, 0, 0, 0, 0, 0};
  auto tick = [&](int i) {
    const auto now = std::chrono::steady_clock::now();
    t_stage[i] += std::chrono::duration<double, std::micro>(now - t_prev).count();
    t_prev = now;
  };
  if (drain(g)) return -EIO;
  tick(0);
  const bool env_skewed = getenv("XLATING_B200_SKEWED") != nullptr, env_no_long = getenv("XLATING_B200_NO_LONG") != nullptr,
             env_no_merge = getenv("XLATING_B200_NO_MERGE") != nullptr;
  const int nc = (int)g->clients.size();
  g->max_client = 0;
  for (int i = 0; i < nc; i++)
    if (g->clients[i].active) g->max_client = i + 1;

  // 1. current device state
  std::vector<ClientDev> tab(std::max(nc, 1));
  memset(tab.data(), 0, tab.size() * sizeof(ClientDev));
  if (g->d_clients && g->d_clients_cap > 0) {
    const size_t n = std::min<size_t>(g->d_clients_cap, tab.size());
    CU_OK(cudaMemcpy(tab.data(), g->d_clients, n * sizeof(ClientDev), cudaMemcpyDeviceToHost));
  }

  // 2. offsets + natural tap arenas
  size_t out_total = 0, taps_total = 0, max_hist = 0;
  for (int i = 0; i < nc; i++) {
    HostClient &h = g->clients[i];
    if (!h.active) continue;
    if (h.mem) {
      // n2 <= (L2 * n1 - 1) / D2 + 1 for any history, n1 at most its sub-band's row
      h.out_cap = (int)(((uint64_t)g->max_input_len / 2 / g->clients[h.sb_cid].D + 2) * h.L2 / h.D2 + 2);
      h.out_off = (int)out_total;
      out_total += (size_t)h.out_cap;
      out_total = (out_total + 3) & ~(size_t)3;
      continue;
    }
    h.out_cap = (int)((uint64_t)g->max_input_len / 2 * h.L / h.D + 2);
    if (h.casc) {
      // n2 <= (L2 * n1 - 1) / D2 + 1 for any history
      h.fin_cap = (int)((uint64_t)h.out_cap * h.L2 / h.D2 + 2);
      h.fin_off = (int)out_total;
      out_total += (size_t)h.fin_cap;
    } else if (!h.sb) {
      h.out_off = (int)out_total;
      out_total += (size_t)h.out_cap;
    }
    out_total = (out_total + 3) & ~(size_t)3;  // keep rows 32-byte aligned
    h.taps_off = (int)taps_total;
    taps_total += h.rev.size() / 2;
    // a rational client's history of at most T - 1 upsampled samples reaches back ceil((T-1)/L) + 1 inputs
    max_hist = std::max(max_hist, h.L == 1 ? h.T - 1 : (h.T - 1 + h.L - 1) / h.L + 1);
  }
  // cascade clients: stage-A rows after every host-visible row (the D2H copy ends before them), stage-B taps,
  // and a zeroed history ring for each new client (its positions before the attach read as zero)
  {
    std::vector<float> taps2;
    g->n_casc = g->n_casc_int = 0;
    for (int i = 0; i < nc; i++) {
      HostClient &h = g->clients[i];
      if (!h.active || !h.casc) continue;
      h.out_off = (int)out_total;
      out_total += (size_t)h.out_cap;
      out_total = (out_total + 3) & ~(size_t)3;
      h.taps2_off = (int)taps2.size();
      taps2.insert(taps2.end(), h.rev2.begin(), h.rev2.end());
      taps2.resize((taps2.size() + 3) & ~(size_t)3, 0.f);  // 16-byte aligned bulk copies of whole float4s
      if (h.d_cring == nullptr) {
        // stage B of block b reads stage-A outputs of earlier blocks; the submit of block b + XLG_SLOTS waits
        // for ticket b, so T2 - 1 + (XLG_SLOTS + 1) * max n1 samples are never overwritten while still needed;
        // a rational stage B's history of at most T2 - 1 upsampled samples reaches back ceil((T2 - 1) / L2)
        // stage-A samples, and its last branch may read one zero-weighted sample past the block
        const size_t back = h.L2 == 1 ? h.T2 - 1 : (h.T2 - 1 + h.L2 - 1) / h.L2 + 1;
        h.cring_cap = next_pow2(back + (size_t)(XLG_SLOTS + 1) * (size_t)h.out_cap);
        CU_OK(cudaMalloc(&h.d_cring, h.cring_cap * sizeof(float2)));
        CU_OK(cudaMemset(h.d_cring, 0, h.cring_cap * sizeof(float2)));
      }
      g->n_casc++;
      if (h.L2 == 1) g->n_casc_int++;
    }
    if (dev_assign(&g->d_taps2, &g->cap_taps2, taps2.data(), taps2.size() * sizeof(float))) return -EIO;
    for (float2 *p : g->dead_rings) cudaFree(p);
    g->dead_rings.clear();
    for (Slot &s : g->slots) {
      if (s.cblk_cap >= (size_t)g->n_casc) continue;
      if (s.d_cblk) cudaFree(s.d_cblk);
      if (s.h_cblk) cudaFreeHost(s.h_cblk);
      s.d_cblk = s.h_cblk = nullptr;
      s.cblk_cap = std::max<size_t>((size_t)g->n_casc * 2, 16);
      CU_OK(cudaMalloc(&s.d_cblk, s.cblk_cap * sizeof(CascBlk)));
      CU_OK(cudaHostAlloc(&s.h_cblk, s.cblk_cap * sizeof(CascBlk), cudaHostAllocDefault));
    }
    const int n_rat = g->n_casc - g->n_casc_int;
    for (Slot &s : g->slots) {
      if (s.pblk_cap >= (size_t)n_rat) continue;
      if (s.d_pblk) cudaFree(s.d_pblk);
      if (s.h_pblk) cudaFreeHost(s.h_pblk);
      s.d_pblk = s.h_pblk = nullptr;
      s.pblk_cap = std::max<size_t>((size_t)n_rat * 2, 16);
      CU_OK(cudaMalloc(&s.d_pblk, s.pblk_cap * sizeof(CascPolyBlk)));
      CU_OK(cudaHostAlloc(&s.h_pblk, s.pblk_cap * sizeof(CascPolyBlk), cudaHostAllocDefault));
    }
  }
  if (rebuild_subbands(g, out_total)) return -EIO;
  if (ensure_ring(g, max_hist, g->qring != nullptr)) return -EIO;
  if (ensure_arenas(g, out_total, g->q_alloc)) return -EIO;

  std::vector<float2> &taps = g->h_taps;
  std::vector<short2> &qtaps = g->h_qtaps;
  taps.resize(std::max<size_t>(taps_total, 1));
  qtaps.resize(std::max<size_t>(taps_total, 1));
  for (int i = 0; i < nc; i++) {
    const HostClient &h = g->clients[i];
    if (!h.active) continue;
    memcpy(&taps[h.taps_off], h.rev.data(), h.rev.size() * sizeof(float));  // both interleaved (re, im)
    memcpy(&qtaps[h.taps_off], h.rev_q15.data(), h.rev_q15.size() * sizeof(int16_t));
  }
  if (dev_assign(&g->d_taps, &g->cap_taps, taps.data(), taps.size() * sizeof(float2)) ||
      dev_assign(&g->d_qtaps, &g->cap_qtaps, qtaps.data(), qtaps.size() * sizeof(short2)))
    return -EIO;

  tick(1);
  // 3. classes for the tiled / long-filter kernels.  A class is a set of clients with
  //    the same (D, T) whose zero-history window has passed (zero_before behind the
  //    next window start, or the stream origin where the ring itself is still zero).
  //    With the natural input layout the members may have different window alignments
  //    (they attached at different stream positions): the kernel shifts each 8-client
  //    subgroup by its own delta, so members are packed into subgroups of 8 with equal
  //    alignment.  The skewed layout and the long-filter kernel need identical
  //    alignment (hist) across the class.
  g->classes.clear();
  g->long_classes.clear();
  g->n_generic = 0;
  // tile of RK = 4: decides eligibility (smaller shapes need less; RK = 5 is used only where its tile fits)
  const int KT = 64;
  const size_t smem_fixed = (size_t)T_SMEM_FIXED;
  struct Mode {
    bool natural, as_long, eligible;
    int Dp, L;
  };
  auto mode_of = [&](uint32_t D, size_t T) {
    Mode m;
    const unsigned g16 = (D % 16 == 0) ? 16u : (D % 8 == 0) ? 8u : (D % 4 == 0) ? 4u : (D % 2 == 0) ? 2u : 1u;
    m.natural = g16 <= 2 && !env_skewed;
    m.Dp = m.natural ? (int)D : (int)(D | 1u);
    const size_t q_last = (T - 1) / D, r_last = (T - 1) % D;
    m.L = (int)(((q_last * m.Dp + r_last + 1) + 7) / 8 * 8);
    const size_t smem = smem_fixed + ((size_t)(KT - 1) * m.Dp + m.L + D + 10) * sizeof(float2);
    const size_t typical_out = g->max_input_len / 2 / D;
    // too long for a shared-memory tile -> split-K long-filter class (natural layout)
    m.as_long = smem > (size_t)kTileMaxSmem && typical_out >= 1 && !env_no_long;
    m.eligible = m.as_long || (smem <= (size_t)kTileMaxSmem && typical_out >= (size_t)kTileMinOutputs);
    if (m.as_long) {
      m.natural = true;
      m.Dp = (int)D;
      m.L = (int)((T + 7) / 8 * 8);
    }
    return m;
  };
  std::map<std::tuple<uint32_t, size_t, long long>, std::vector<int>> buckets;
  std::map<std::tuple<uint32_t, uint32_t, size_t, long long>, std::vector<int>> pbuckets;  // (L, M, T, hist)
  g->poly_classes.clear();
  for (int i = 0; i < nc; i++) {
    HostClient &h = g->clients[i];
    if (!h.active) continue;
    if (h.mem) {
      h.kind = 6;  // served by subband_fir_cf32_kernel (subband_fir_poly_cf32_kernel when L2 > 1)
      continue;
    }
    h.kind = h.L > 1 ? 3 : 0;
    h.tile_ineligible = false;
    h.pending_settle = false;
    if (h.L > 1) {
      // rational: a tiled class per (L, M, T, alignment) where every branch is an integer class the tiled
      // kernel takes (gcd(L, M) = 1: each block uses every branch, outputs L apart)
      const size_t Tb = (h.T + h.L - 1) / h.L;
      const Mode m = mode_of(h.D, Tb);
      if ((g->flags & XLG_FORCE_GENERIC) || !g->poly_tile || std::gcd(h.L, h.D) != 1 || !m.eligible || m.as_long)
        continue;
      if (!poly_settled(g, h)) {
        h.pending_settle = true;
        continue;
      }
      pbuckets[std::make_tuple(h.L, h.D, h.T, h.hist)].push_back(i);
      continue;
    }
    const long long first = g->S - h.hist;
    const bool settled = (h.zero_before == 0 && g->S < (long long)g->ring_cap / 2) || h.zero_before <= first;
    if (g->flags & XLG_FORCE_GENERIC) continue;
    const Mode m = mode_of(h.D, h.T);
    if (!m.eligible) {
      h.tile_ineligible = true;
      continue;
    }
    if (!settled) {
      h.pending_settle = true;  // re-derive the layout once its window has passed
      continue;
    }
    const bool merge = m.natural && !m.as_long && !env_no_merge;
    buckets[std::make_tuple(h.D, h.T, merge ? -1ll : h.hist)].push_back(i);
  }
  std::vector<int> members;       // output row offset per member slot
  std::vector<int> member_cid;    // client id per member slot
  std::vector<float2> member_incr;
  std::vector<float2> &tile_taps = g->h_tile_taps;
  tile_taps.clear();
  for (auto &kv : buckets) {
    const uint32_t D = std::get<0>(kv.first);
    const size_t T = std::get<1>(kv.first);
    const bool merged = std::get<2>(kv.first) < 0;
    const Mode m = mode_of(D, T);
    // subgroups of 8 slots with one window alignment each
    std::map<long long, std::vector<int>> by_align;
    for (int id : kv.second) by_align[merged ? (long long)(T - 1) - g->clients[id].hist : 0].push_back(id);
    std::vector<int> slots;
    std::vector<int> real;
    for (auto &al : by_align) {
      if (merged && al.second.size() < 2) {
        // a lone alignment would occupy an 8-slot subgroup by itself: generic kernel
        g->clients[al.second[0]].tile_ineligible = true;
        continue;
      }
      for (size_t i = 0; i < al.second.size(); i++) {
        slots.push_back(al.second[i]);
        real.push_back(al.second[i]);
      }
      while (slots.size() % T_RC != 0) slots.push_back(-1);
    }
    std::vector<TileClassHost> &dest = m.as_long ? g->long_classes : g->classes;
    if ((int)real.size() < kTileMinClients || (int)dest.size() >= T_MAX_CLASSES) {
      if ((int)dest.size() >= T_MAX_CLASSES)
        for (int id : real) g->clients[id].tile_ineligible = true;
      continue;
    }
    while (slots.size() % T_CG != 0) slots.push_back(-1);
    TileClassHost ch;
    memset(&ch.k, 0, sizeof(ch.k));
    ch.T = T;
    ch.members = slots;
    ch.real = real;
    ch.merged = merged;
    ch.k.D = (int)D;
    ch.k.Dp = m.Dp;
    ch.k.L = m.L;
    ch.k.n_groups = (int)(slots.size() / T_CG);
    ch.k.n_members = (int)real.size();
    ch.k.natural = m.natural ? 1 : 0;
    ch.k.nseg = m.as_long ? (ch.k.L + W_JS - 1) / W_JS : 0;
    ch.k.members_off = (int)members.size();
    ch.k.taps_off = (long long)tile_taps.size();
    const size_t base = tile_taps.size();
    tile_taps.resize(base + slots.size() * (size_t)m.L, make_float2(0.f, 0.f));
    for (size_t sl = 0; sl < slots.size(); sl++) {
      const int id = slots[sl];
      member_cid.push_back(id);
      if (id < 0) {
        members.push_back(-1);
        member_incr.push_back(make_float2(1.f, 0.f));
        continue;
      }
      HostClient &h = g->clients[id];
      members.push_back(h.out_off);
      member_incr.push_back(make_float2(h.incr_re, h.incr_im));
      h.kind = m.as_long ? 2 : 1;
    }
    // taps into [group][flat tap f][32 slots]: one 256-byte line (all 32 slots of a tap) at a time -- slot-major
    // packing touched a new cache line for every tap of every client (1.5 ms per re-layout at 1000 clients)
    for (size_t gi = 0; gi < slots.size() / T_CG; gi++) {
      float2 *dst = tile_taps.data() + base + gi * (size_t)m.L * T_CG;
      const float *src[T_CG];
      for (int sl = 0; sl < T_CG; sl++) {
        const int id = slots[gi * T_CG + sl];
        src[sl] = id < 0 ? nullptr : g->clients[id].rev.data();
      }
      size_t q = 0, r = 0;  // j = q * D + r
      for (size_t j = 0; j < T; j++) {
        const size_t f = q * m.Dp + r;
        if (++r == D) {
          r = 0;
          q++;
        }
        float2 *row = dst + f * T_CG;
        for (int sl = 0; sl < T_CG; sl++)
          if (src[sl]) row[sl] = make_float2(src[sl][2 * j], src[sl][2 * j + 1]);
      }
    }
    dest.push_back(ch);
  }
  // rational tiled classes: one tiled class per polyphase branch r, members in the same slots of every branch
  size_t pscratch = 0;
  int max_rowcap = 0;
  for (auto &kv : pbuckets) {
    const uint32_t L = std::get<0>(kv.first), M = std::get<1>(kv.first);
    const size_t T = std::get<2>(kv.first), Tb = (T + L - 1) / L;
    std::vector<int> &real = kv.second;
    if ((int)real.size() < kTileMinClients || g->poly_classes.size() + L > (size_t)T_MAX_CLASSES) continue;
    const Mode m = mode_of(M, Tb);
    std::vector<int> slots(real);
    while (slots.size() % T_CG != 0) slots.push_back(-1);
    long long minv = 0;  // M^-1 mod L (extended Euclid)
    {
      long long a = M % L, b = L, x0 = 1, x1 = 0;
      while (b != 0) {
        const long long q = a / b, t = a - q * b, tx = x0 - q * x1;
        a = b;
        b = t;
        x0 = x1;
        x1 = tx;
      }
      minv = ((x0 % (long long)L) + L) % L;
    }
    for (int id : real) {
      HostClient &h = g->clients[id];
      h.kind = 4;
      h.poly_rowcap = (h.out_cap + (int)L - 1) / (int)L + 1;
      h.poly_off = (int)pscratch;
      pscratch += (size_t)L * h.poly_rowcap;
      max_rowcap = std::max(max_rowcap, h.poly_rowcap);
    }
    for (uint32_t r = 0; r < L; r++) {
      TileClassHost ch;
      memset(&ch.k, 0, sizeof(ch.k));
      ch.T = Tb;
      ch.members = slots;
      ch.real = real;
      ch.branch = (int)r;
      ch.interp = L;
      ch.minv = minv;
      ch.k.D = (int)M;
      ch.k.Dp = m.Dp;
      ch.k.L = m.L;
      ch.k.n_groups = (int)(slots.size() / T_CG);
      ch.k.n_members = (int)real.size();
      ch.k.natural = m.natural ? 1 : 0;
      ch.k.members_off = (int)members.size();
      ch.k.taps_off = (long long)tile_taps.size();
      const int v = (int)g->poly_classes.size();  // the tiled kernel reads this class's BlkInfo at d_vblk[v]
      for (int id : slots) {
        member_cid.push_back(id < 0 ? -1 : v);
        members.push_back(id < 0 ? -1 : g->clients[id].poly_off + (int)r * g->clients[id].poly_rowcap);
        member_incr.push_back(make_float2(1.f, 0.f));
      }
      const size_t base = tile_taps.size();
      tile_taps.resize(base + slots.size() * (size_t)m.L, make_float2(0.f, 0.f));
      for (size_t gi = 0; gi < slots.size() / T_CG; gi++) {
        float2 *dst = tile_taps.data() + base + gi * (size_t)m.L * T_CG;
        for (int sl = 0; sl < T_CG; sl++) {
          const int id = slots[gi * T_CG + sl];
          if (id < 0) continue;
          const float *src = g->clients[id].rev.data() + 2 * (size_t)r * Tb;  // branch r (xl_poly_pack)
          for (size_t t = 0; t < Tb; t++)
            dst[((t / M) * m.Dp + t % M) * T_CG + sl] = make_float2(src[2 * t], src[2 * t + 1]);
        }
      }
      g->poly_classes.push_back(ch);
    }
  }
  tick(2);
  // heaviest classes first: their CTAs are scheduled first and the lighter ones
  // fill the tail of the launch
  std::sort(g->classes.begin(), g->classes.end(), [](const TileClassHost &a, const TileClassHost &b) {
    return a.k.L > b.k.L;
  });
  if (!tile_taps.empty()) {
    void *tt = g->d_tile_taps;
    if (dev_assign(&tt, &g->cap_tile_taps, tile_taps.data(), tile_taps.size() * sizeof(float2)) ||
        dev_assign(&g->d_members, &g->cap_members, members.data(), members.size() * sizeof(int)) ||
        dev_assign(&g->d_member_cid, &g->cap_member_cid, member_cid.data(), member_cid.size() * sizeof(int)) ||
        dev_assign(&g->d_member_incr, &g->cap_member_incr, member_incr.data(), member_incr.size() * sizeof(float2))) {
      g->d_tile_taps = tt;
      return -EIO;
    }
    g->d_tile_taps = tt;
  }

  // 3a. long filters: every 256 KiB block streams ALL their taps once (each tap serves only ~52
  //     outputs of a block), 63 MB for BASELINE configs[4]'s 512 clients per GPU -- more than an
  //     H100's 50 MB L2, and the partial sums and the ring evict them between launches.  Pin what
  //     the persisting carve-out holds: a persisting access-policy window over the packed taps on
  //     the compute streams (hitRatio = carve-out / window when the taps exceed it).
  if (!g->long_classes.empty() && !tile_taps.empty() && getenv("XLATING_B200_NO_L2PIN") == nullptr) {
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, g->device) == cudaSuccess && prop.persistingL2CacheMaxSize > 0 &&
        prop.accessPolicyMaxWindowSize > 0) {
      const size_t bytes = tile_taps.size() * sizeof(float2);
      const size_t carve = std::min(bytes, (size_t)prop.persistingL2CacheMaxSize);
      const size_t window = std::min(bytes, (size_t)prop.accessPolicyMaxWindowSize);
      cudaStreamAttrValue attr;
      memset(&attr, 0, sizeof(attr));
      attr.accessPolicyWindow.base_ptr = g->d_tile_taps;
      attr.accessPolicyWindow.num_bytes = window;
      attr.accessPolicyWindow.hitRatio = (float)std::min(1.0, (double)carve / (double)window);
      attr.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
      attr.accessPolicyWindow.missProp = cudaAccessPropertyStreaming;
      bool ok = cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, carve) == cudaSuccess;
      for (int i = 0; i < xlg_group::kMaxCs && ok; i++)
        ok = cudaStreamSetAttribute(g->s_cs[i], cudaStreamAttributeAccessPolicyWindow, &attr) == cudaSuccess;
      if (!ok) {
        cudaGetLastError();
        XL_LOG("could not pin the long filters' taps in L2 (continuing without)");
      }
    }
  }

  tick(3);
  // 3b. oscillator-table order: tile classes (the order the tiled kernel walks them),
  //     then generic clients; 32 clients per table group
  {
    std::vector<int> order;
    size_t table = 0;
    std::vector<TileClassHost *> tabled;
    for (TileClassHost &ch : g->classes) tabled.push_back(&ch);
    for (TileClassHost &ch : g->long_classes) tabled.push_back(&ch);
    for (TileClassHost *chp : tabled) {
      TileClassHost &ch = *chp;
      int cap = 0;
      for (int id : ch.real) cap = std::max(cap, g->clients[id].out_cap);
      cap = cap / 2 + 1;  // only even outputs are tabulated
      ch.k.ph_base = (long long)table;
      ch.k.ph_stride = cap * 32;
      for (int gi = 0; gi < ch.k.n_groups; gi++) {
        for (int m = 0; m < T_CG; m++) {
          const size_t idx = (size_t)gi * T_CG + m;
          if (idx < ch.members.size() && ch.members[idx] >= 0) {
            g->clients[ch.members[idx]].ph_off = (int)(table + m);
            order.push_back(ch.members[idx]);
          } else {
            order.push_back(-1);
          }
        }
        table += (size_t)cap * 32;
      }
    }
    std::vector<int> loose;
    for (int i = 0; i < nc; i++)
      if (g->clients[i].active && !g->clients[i].mem && (g->clients[i].kind == 0 || g->clients[i].kind >= 3))
        loose.push_back(i);
    for (size_t base = 0; base < loose.size(); base += 32) {
      int cap = 0;
      for (size_t m = base; m < std::min(base + 32, loose.size()); m++) cap = std::max(cap, g->clients[loose[m]].out_cap);
      cap = cap / 2 + 1;
      for (size_t m = 0; m < 32; m++) {
        if (base + m < loose.size()) {
          g->clients[loose[base + m]].ph_off = (int)(table + m);
          order.push_back(loose[base + m]);
        } else {
          order.push_back(-1);
        }
      }
      table += (size_t)cap * 32;
    }
    if (g->d_order) cudaFree(g->d_order);
    g->d_order = nullptr;
    g->n_order = (int)order.size();
    if (!order.empty()) {
      CU_OK(cudaMalloc(&g->d_order, order.size() * sizeof(int)));
      CU_OK(cudaMemcpy(g->d_order, order.data(), order.size() * sizeof(int), cudaMemcpyHostToDevice));
    }
    {
      size_t part = 0;
      for (TileClassHost &ch : g->long_classes) {
        int cap = 0;
        for (int id : ch.real) cap = std::max(cap, g->clients[id].out_cap);
        const size_t kt = (size_t)W2_KT;
        const size_t kpad_max = ((size_t)cap + kt - 1) / kt * kt;
        ch.k.part_off = (long long)part;
        ch.k.kpad = (int)kpad_max;
        part += (size_t)ch.k.nseg * ch.k.n_groups * kpad_max * T_CG;  // (the pipelined kernel uses ksplit <= nseg slabs of it)
      }
      if (part > g->partial_cap) {
        g->partial_cap = part;
        for (Slot &sl : g->slots) {
          if (sl.d_partial) cudaFree(sl.d_partial);
          sl.d_partial = nullptr;
          CU_OK(cudaMalloc(&sl.d_partial, g->partial_cap * sizeof(float2)));
        }
      }
    }
    if (pscratch > g->pscratch_cap) {
      g->pscratch_cap = pscratch + pscratch / 4 + 1024;
      for (Slot &sl : g->slots) {
        if (sl.d_pscratch) cudaFree(sl.d_pscratch);
        sl.d_pscratch = nullptr;
        CU_OK(cudaMalloc(&sl.d_pscratch, g->pscratch_cap * sizeof(float2)));
      }
    }
    // the tiled kernel reads the phase of output j at [32 * (j / 2) + client slot]: a table of ones that long
    const size_t ones = ((size_t)max_rowcap / 2 + 2) * 32;
    if (!g->poly_classes.empty() && ones > g->ones_cap) {
      if (g->d_ones) cudaFree(g->d_ones);
      g->d_ones = nullptr;
      g->ones_cap = ones;
      std::vector<float2> one(ones, make_float2(1.f, 0.f));
      CU_OK(cudaMalloc(&g->d_ones, ones * sizeof(float2)));
      CU_OK(cudaMemcpy(g->d_ones, one.data(), ones * sizeof(float2), cudaMemcpyHostToDevice));
    }
    if (table > g->phase_cap) {
      g->phase_cap = table + table / 4 + 1024;
      for (Slot &sl : g->slots) {
        if (sl.d_phases) cudaFree(sl.d_phases);
        sl.d_phases = nullptr;
        CU_OK(cudaMalloc(&sl.d_phases, g->phase_cap * sizeof(float2)));
      }
    }
  }

  // 4. device client table
  for (int i = 0; i < nc; i++) {
    HostClient &h = g->clients[i];
    ClientDev &d = tab[i];
    if (!h.active) {
      d.active = 0;
      continue;
    }
    if (h.is_new) {
      memset(&d, 0, sizeof(d));
      d.hist = h.hist;
      d.zero_before = h.zero_before;
      d.qzero_before = h.qzero_before;
      d.phase = make_float2(h.init_ph_re, h.init_ph_im);  // (1, 0): src/xlating.c:543
      d.incr = make_float2(h.incr_re, h.incr_im);
      d.qph_re = INT16_MAX;  // src/xlating.c:546-547
      d.qph_im = 0;
      d.qinc_re = h.qincr_re;
      d.qinc_im = h.qincr_im;
      h.is_new = false;
    }
    d.D = (int)h.D;
    d.L = (int)h.L;
    d.T = (int)h.T;
    d.taps_off = h.taps_off;
    d.qtaps_off = h.taps_off;
    d.out_off = h.out_off;
    d.out_cap = h.out_cap;
    d.active = h.mem ? 0 : 1;  // a member's entry only carries its oscillator (subband_phase_kernel)
    d.kind = h.kind;
    d.renorm = (g->flags & XLG_NO_RENORM) ? 0 : 1;
    d.ph_off = h.ph_off;
    d.poly_off = h.poly_off;
    d.poly_rowcap = h.poly_rowcap;
    if (h.kind == 0) g->n_generic++;
  }
  {
    std::vector<int> p3, p4;
    for (int i = 0; i < nc; i++)
      if (g->clients[i].active && g->clients[i].kind == 3) p3.push_back(i);
      else if (g->clients[i].active && g->clients[i].kind == 4) p4.push_back(i);
    g->n_poly3 = (int)p3.size();
    g->n_poly4 = (int)p4.size();
    if (dev_assign(&g->d_poly3, &g->cap_poly3, p3.data(), p3.size() * sizeof(int)) ||
        dev_assign(&g->d_poly4, &g->cap_poly4, p4.data(), p4.size() * sizeof(int)))
      return -EIO;
  }
  if ((size_t)nc > g->d_clients_cap) {
    if (g->d_clients) cudaFree(g->d_clients);
    g->d_clients = nullptr;
    g->d_clients_cap = std::max<size_t>((size_t)nc * 2, 64);
    CU_OK(cudaMalloc(&g->d_clients, g->d_clients_cap * sizeof(ClientDev)));
    CU_OK(cudaMemset(g->d_clients, 0, g->d_clients_cap * sizeof(ClientDev)));
    if (g->d_clients_backup) cudaFree(g->d_clients_backup);
    g->d_clients_backup = nullptr;
    CU_OK(cudaMalloc(&g->d_clients_backup, g->d_clients_cap * sizeof(SpecSave)));
  }
  if (nc > 0) CU_OK(cudaMemcpy(g->d_clients, tab.data(), (size_t)nc * sizeof(ClientDev), cudaMemcpyHostToDevice));

  for (Slot &s : g->slots) {
    if (s.blk_cap < (size_t)std::max(nc, 1)) {
      if (s.d_blk) cudaFree(s.d_blk);
      s.d_blk = nullptr;
      s.blk_cap = std::max<size_t>((size_t)nc * 2, 64);
      CU_OK(cudaMalloc(&s.d_blk, s.blk_cap * sizeof(BlkInfo)));
      if (s.d_endph) cudaFree(s.d_endph);
      s.d_endph = nullptr;
      if (g->flags & XLG_TRACK_STATE) CU_OK(cudaMalloc(&s.d_endph, s.blk_cap * sizeof(float2)));
    }
  }
  if (g->flags & XLG_TRACK_STATE) {
    const size_t want = std::max<size_t>((size_t)nc * 2, 64);
    for (HostOut &h : g->ring_out) {
      if (h.endph_cap >= (size_t)std::max(nc, 1)) continue;
      float2 *fresh = nullptr;
      CU_OK(cudaHostAlloc(&fresh, want * sizeof(float2), cudaHostAllocDefault));
      if (h.h_endph != nullptr) memcpy(fresh, h.h_endph, h.endph_cap * sizeof(float2));  // tickets in the ring stay readable
      std::lock_guard<std::mutex> lk(g->mu);
      if (h.h_endph) g->retired_host.push_back(h.h_endph);  // a reader may still hold the old array
      h.h_endph = fresh;
      h.endph_cap = want;
    }
  }
  choose_partition(g);
  g->dirty = false;
  tick(4);
  if (timing)
    XL_LOG("re-layout of %d clients: drain %.0f us, state + natural taps %.0f, classes + packing %.0f, tile uploads %.0f, "
           "tables + arenas %.0f", nc, t_stage[0], t_stage[1], t_stage[2], t_stage[3], t_stage[4]);
  return 0;
}

static void activate_streams(xlg_group *g, bool part) {
  const xlg_group::StreamSet &ss = part ? g->set_part : g->set_plain;
  g->s_ph = ss.ph;
  g->s_cv = ss.cv;
  for (int i = 0; i < xlg_group::kMaxCs; i++) g->s_cs[i] = ss.cs[i];
  g->part_active = part;
  g->fir_sms = part ? g->part.big_sms : g->total_sms;
}

// Partition or not, for the layout just built (the pipeline is drained).  Estimates per full-size block: the
// oscillator chain alone (~6 us + ~10.75 cycles per output of the fastest client) and the FIR at about three
// quarters of the FP32 FMA peak (128 FMA per clock per SM).  Sharing SMs with FIR warps the chain runs about
// 5x slower: if that still fits inside the FIR time the 8 SMs are worth more as FIR SMs, otherwise the chain
// would pace the pipeline and the partition wins.
static void choose_partition(xlg_group *g) {
  if (!g->part.ok) return;
  bool want = true;
  if (g->part_force >= 0) {
    want = g->part_force != 0;
  } else {
    const double n = (double)(g->max_input_len / 2);
    double steps = 0, fma = 0;
    for (const HostClient &h : g->clients) {
      if (!h.active || h.mem) continue;
      const double n_out = n * h.L / (double)h.D;
      steps = std::max(steps, n_out);
      fma += 4.0 * n_out * (double)((h.T + h.L - 1) / h.L);
    }
    const double t_chain_us = 6.0 + steps * 10.75 / g->sm_mhz * 1.15;
    const double fma_per_us = 128.0 * g->sm_mhz * (double)g->part.big_sms;
    const double t_fir_us = fma / (0.76 * fma_per_us);
    want = t_chain_us * 5.0 > t_fir_us;
  }
  if (want != g->part_active) activate_streams(g, want);
}

// Split the device into an 8-SM partition (oscillator pre-pass) and the rest (FIR)
// and create the compute streams inside them.  Any failure leaves part.ok false
// and the group falls back to ordinary streams.
static void partition_create(xlg_group *g, int device) {
  pfn_cuDeviceGet p_devget;
  pfn_cuDeviceGetDevResource p_getres;
  pfn_cuDevSmResourceSplitByCount p_split;
  pfn_cuDevResourceGenerateDesc p_desc;
  pfn_cuGreenCtxCreate p_create;
  pfn_cuGreenCtxStreamCreate p_stream;
  if (!drv("cuDeviceGet", &p_devget) || !drv("cuDeviceGetDevResource", &p_getres) ||
      !drv("cuDevSmResourceSplitByCount", &p_split) || !drv("cuDevResourceGenerateDesc", &p_desc) ||
      !drv("cuGreenCtxCreate", &p_create) || !drv("cuGreenCtxStreamCreate", &p_stream)) {
    XL_LOG("green contexts unavailable in this driver; SM partition disabled");
    return;
  }
  cudaFree(0);  // make sure the primary context exists
  // SMs asked for the oscillator partition: the driver rounds up to its granularity (8 on
  // sm_90); XLATING_B200_PART_SMS asks for another count (measurement switch)
  int want_sms = 8;
  if (getenv("XLATING_B200_PART_SMS") != nullptr) want_sms = std::min(std::max(atoi(getenv("XLATING_B200_PART_SMS")), 1), 64);
  CUdevice dev;
  CUdevResource all, small, rest;
  unsigned int groups = 1;
  CUdevResourceDesc d_small = nullptr, d_rest = nullptr;
  CUstream st_ph = nullptr, st_cv = nullptr, st_c[xlg_group::kMaxCs] = {nullptr, nullptr, nullptr, nullptr};
  if (p_devget(&dev, device) != CUDA_SUCCESS || p_getres(dev, &all, CU_DEV_RESOURCE_TYPE_SM) != CUDA_SUCCESS ||
      p_split(&small, &groups, &all, &rest, 0, (unsigned)want_sms) != CUDA_SUCCESS || groups != 1 ||
      p_desc(&d_small, &small, 1) != CUDA_SUCCESS || p_desc(&d_rest, &rest, 1) != CUDA_SUCCESS ||
      p_create(&g->part.small_ctx, d_small, dev, CU_GREEN_CTX_DEFAULT_STREAM) != CUDA_SUCCESS ||
      p_create(&g->part.big_ctx, d_rest, dev, CU_GREEN_CTX_DEFAULT_STREAM) != CUDA_SUCCESS ||
      p_stream(&st_ph, g->part.small_ctx, CU_STREAM_NON_BLOCKING, 0) != CUDA_SUCCESS ||
      p_stream(&st_cv, g->part.small_ctx, CU_STREAM_NON_BLOCKING, 0) != CUDA_SUCCESS ||
      p_stream(&st_c[0], g->part.big_ctx, CU_STREAM_NON_BLOCKING, 0) != CUDA_SUCCESS ||
      p_stream(&st_c[1], g->part.big_ctx, CU_STREAM_NON_BLOCKING, 0) != CUDA_SUCCESS ||
      p_stream(&st_c[2], g->part.big_ctx, CU_STREAM_NON_BLOCKING, 0) != CUDA_SUCCESS ||
      p_stream(&st_c[3], g->part.big_ctx, CU_STREAM_NON_BLOCKING, 0) != CUDA_SUCCESS) {
    XL_LOG("could not create the SM partition (green contexts); continuing without it");
    cudaGetLastError();
    return;
  }
  g->part.small_sms = (int)small.sm.smCount;
  g->part.big_sms = (int)rest.sm.smCount;
  g->set_part.ph = (cudaStream_t)st_ph;
  g->set_part.cv = (cudaStream_t)st_cv;
  for (int i = 0; i < xlg_group::kMaxCs; i++) g->set_part.cs[i] = (cudaStream_t)st_c[i];
  g->part.ok = true;
}

// Tensor map of the sample ring as rows of pitch D: element (c, r) = ring[r * D + c], 8-byte elements, box =
// W_JSP x W4_KT (one stage's strips).  Rows overlap in memory when the inner width exceeds D; if the driver
// refuses that, the map is D wide and boxes that would cross a row end fall back to per-strip copies.
typedef CUresult (*pfn_cuTensorMapEncodeTiled)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                               const cuuint64_t *, const cuuint32_t *, const cuuint32_t *,
                                               CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                               CUtensorMapFloatOOBfill);
static void strip_map_update(xlg_group *g, int D) {
  if (g->strip_ring == g->ring && g->strip_cap == g->ring_cap && g->strip_D == D) return;
  g->strip_ring = g->ring;
  g->strip_cap = g->ring_cap;
  g->strip_D = D;
  g->strip_w = 0;
  pfn_cuTensorMapEncodeTiled enc;
  if (!g->long_tmap || (D & 1) != 0 || (size_t)D + W_JSP >= g->ring_cap || !drv("cuTensorMapEncodeTiled", &enc)) return;
  const cuuint32_t box[2] = {(cuuint32_t)W_JSP, (cuuint32_t)W4_KT}, estr[2] = {1, 1};
  const cuuint64_t gstride[1] = {(cuuint64_t)D * 8};
  for (int width : {D + W_JSP, D}) {
    if (width < W_JSP) continue;
    // rows up to the ring's end: the kernel only issues boxes that lie inside the ring (its own bound check),
    // so the last rows' columns beyond the allocation are never touched
    const cuuint64_t gdim[2] = {(cuuint64_t)width, (cuuint64_t)(g->ring_cap / (size_t)D + 1)};
    if (gdim[1] < (cuuint64_t)W4_KT) continue;
    if (enc(&g->strip_map, CU_TENSOR_MAP_DATA_TYPE_UINT64, 2, g->ring, gdim, gstride, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
            CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS) {
      g->strip_w = width;
      break;
    }
  }
  if (g->strip_w == 0) XL_LOG("cuTensorMapEncodeTiled refused the strip map (D = %d); long filters use per-strip copies", D);
}

// ---------------------------------------------------------------------------
// public API
// ---------------------------------------------------------------------------
extern "C" int xlg_create(int device, uint32_t sampling_freq, uint32_t max_input_len, uint32_t flags,
                          xlg_group **out) {
  return xlg_create_ex(device, sampling_freq, max_input_len, flags, XLG_SLOTS, out);
}

extern "C" int xlg_create_ex(int device, uint32_t sampling_freq, uint32_t max_input_len, uint32_t flags,
                             uint32_t host_ring, xlg_group **out) {
  if (out == nullptr || max_input_len < 2 || sampling_freq == 0) return -EINVAL;
  if (host_ring < XLG_SLOTS) host_ring = XLG_SLOTS;
  if (host_ring > 1024) return -EINVAL;
  int ndev = 0;
  cudaError_t e = cudaGetDeviceCount(&ndev);
  if (e != cudaSuccess || ndev == 0) {
    XL_LOG("no usable CUDA device (%s); this library has no CPU fallback",
           e == cudaSuccess ? "device count is 0" : cudaGetErrorString(e));
    return -ENODEV;
  }
  if (device < 0 || device >= ndev) {
    XL_LOG("device %d out of range (%d present)", device, ndev);
    return -ENODEV;
  }
  CU_OK(cudaSetDevice(device));
  cudaDeviceProp prop;
  CU_OK(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) {
    XL_LOG("device %d is sm_%d%d; this library is built for sm_90a only", device, prop.major, prop.minor);
    return -ENODEV;
  }
  xlg_group *g = new (std::nothrow) xlg_group();
  if (g == nullptr) return -ENOMEM;
  memset(&g->prof, 0, sizeof(g->prof));
  memset(&g->poly_prof, 0, sizeof(g->poly_prof));
  memset(&g->casc_prof, 0, sizeof(g->casc_prof));
  memset(&g->sb_prof, 0, sizeof(g->sb_prof));
  g->device = device;
  g->fs = sampling_freq;
  g->max_input_len = max_input_len;
  g->flags = flags;
  g->ring_out = std::vector<HostOut>(host_ring);
  for (HostOut &h : g->ring_out) {
    h.n_out.retired = &g->retired_meta_i;
    h.out_off.retired = &g->retired_meta_i;
    h.hist_after.retired = &g->retired_meta_ll;
  }
  int rc = 0;
  auto fail = [&](int code) {
    xlg_destroy(g);
    return code;
  };
  g->total_sms = prop.multiProcessorCount;
  {
    int khz = 0;
    if (cudaDeviceGetAttribute(&khz, cudaDevAttrClockRate, device) != cudaSuccess || khz <= 0) return fail(-EIO);
    g->sm_mhz = khz / 1000.0;
  }
  {
    bool want = (flags & XLG_SM_PARTITION) != 0;
    const char *pe = getenv("XLATING_B200_PARTITION");
    if (pe != nullptr) {
      want = atoi(pe) != 0;
      g->part_force = want ? 1 : 0;
    }
    if (getenv("XLATING_B200_PARTITION_AUTO") != nullptr && atoi(getenv("XLATING_B200_PARTITION_AUTO")) == 0 && g->part_force < 0)
      g->part_force = want ? 1 : 0;  // the flag means "always", as in round 1
    if (want) partition_create(g, device);
  }
  if (cudaStreamCreateWithFlags(&g->s_in, cudaStreamNonBlocking) != cudaSuccess ||
      cudaStreamCreateWithFlags(&g->s_out, cudaStreamNonBlocking) != cudaSuccess)
    return fail(-EIO);
  {
    if (cudaStreamCreateWithFlags(&g->set_plain.ph, cudaStreamNonBlocking) != cudaSuccess) return fail(-EIO);
    int prio_lo = 0, prio_hi = 0;  // "greatest" priority is the numerically lowest
    if (cudaDeviceGetStreamPriorityRange(&prio_lo, &prio_hi) != cudaSuccess) prio_lo = prio_hi = 0;
    if (cudaStreamCreateWithPriority(&g->set_plain.cv, cudaStreamNonBlocking, prio_hi) != cudaSuccess) return fail(-EIO);
    for (int i = 0; i < xlg_group::kMaxCs; i++)
      if (cudaStreamCreateWithFlags(&g->set_plain.cs[i], cudaStreamNonBlocking) != cudaSuccess) return fail(-EIO);
  }
  activate_streams(g, g->part.ok);
  const size_t raw_bytes = (size_t)max_input_len * 2;  // cs16 worst case
  for (Slot &s : g->slots) {
    if (cudaMalloc(&s.d_raw, raw_bytes) != cudaSuccess) return fail(-ENOMEM);
    if (cudaHostAlloc(&s.h_raw, raw_bytes, cudaHostAllocDefault) != cudaSuccess) return fail(-ENOMEM);
    cudaEvent_t *evs[] = {&s.ev_h2d, &s.ev_conv, &s.ev_phase, &s.ev_fir, &s.ev_done};
    for (cudaEvent_t *ev : evs)
      if (cudaEventCreateWithFlags(ev, cudaEventDisableTiming) != cudaSuccess) return fail(-EIO);
    for (int i = 0; i < 10; i++)
      if (cudaEventCreate(&s.pf[i]) != cudaSuccess) return fail(-EIO);
    for (cudaEvent_t &ev : s.pf_poly)
      if (cudaEventCreate(&ev) != cudaSuccess) return fail(-EIO);
    for (cudaEvent_t &ev : s.pf_casc)
      if (cudaEventCreate(&ev) != cudaSuccess) return fail(-EIO);
    if (cudaEventCreateWithFlags(&s.ev_casc, cudaEventDisableTiming) != cudaSuccess) return fail(-EIO);
    if (cudaMalloc(&s.d_vblk, T_MAX_CLASSES * sizeof(BlkInfo)) != cudaSuccess ||
        cudaHostAlloc(&s.h_vblk, T_MAX_CLASSES * sizeof(BlkInfo), cudaHostAllocDefault) != cudaSuccess)
      return fail(-ENOMEM);
  }
  if (cudaEventCreate(&g->ev_t0) != cudaSuccess || cudaEventCreate(&g->ev_t1) != cudaSuccess) return fail(-EIO);
  // the tiled kernel needs > 48 KiB of dynamic shared memory
  {
    const char *tv = getenv("XLATING_B200_TILE");
    if (tv != nullptr) {
      g->tile_force = atoi(tv);
      if (tile_shape_index(g->tile_force) < 0) {
        XL_LOG("XLATING_B200_TILE=%s is not a tile shape (1642, 1641, 1621 or 1611); choosing automatically", tv);
        g->tile_force = 0;
      }
    }
    const char *cvs = getenv("XLATING_B200_CONV_STREAM");
    if (cvs != nullptr) g->conv_own_stream = atoi(cvs) != 0;
    const char *tm = getenv("XLATING_B200_LONG_TMAP");
    if (tm != nullptr) g->long_tmap = atoi(tm) != 0;
    const char *sv = getenv("XLATING_B200_SPECULATE");
    if (sv != nullptr) g->speculate = atoi(sv) != 0;
    const char *pt = getenv("XLATING_B200_POLY_TILE");
    if (pt != nullptr) g->poly_tile = atoi(pt) != 0;
    const char *cv = getenv("XLATING_B200_CSTREAMS");
    if (cv != nullptr) g->n_cs = std::min(std::max(atoi(cv), 1), (int)xlg_group::kMaxCs);
  }
  for (const TileShapeHost &sh : kTileShapes)
    if (cudaFuncSetAttribute(sh.kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kTileMaxSmem) != cudaSuccess) {
      XL_LOG("cannot raise dynamic shared memory to %d bytes", kTileMaxSmem);
      return fail(-EIO);
    }
  if (cudaFuncSetAttribute(fir_long2_cf32_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, W2_SMEM) != cudaSuccess ||
      cudaFuncSetAttribute(fir_long4_cf32_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, W4_SMEM) != cudaSuccess ||
      cudaFuncSetAttribute(cascade_fir_cf32_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kTileMaxSmem) != cudaSuccess ||
      cudaFuncSetAttribute(cascade_fir_poly_cf32_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kTileMaxSmem) != cudaSuccess) {
    XL_LOG("cannot raise dynamic shared memory to %d bytes", kTileMaxSmem);
    return fail(-EIO);
  }
  if (getenv("XLATING_B200_TIMELINE") != nullptr && cudaEventCreate(&g->ev_base) == cudaSuccess) {
    g->timeline = true;
    for (Slot &sl : g->slots)
      for (int a = 0; a < 2; a++)
        for (int b = 0; b < 2; b++)
          if (cudaEventCreate(&sl.tl_ph[a][b]) != cudaSuccess) g->timeline = false;
  }
  if (getenv("XLATING_B200_TRACE") != nullptr && atoi(getenv("XLATING_B200_TRACE")) != 0) {
    if (cudaMalloc(&g->d_trace, sizeof(long long) * T_TRACE_REC * T_TRACE_CTAS * T_TRACE_LAUNCHES) != cudaSuccess) g->d_trace = nullptr;
  }
  rc = ensure_ring(g, 4096, false);
  if (rc) return fail(rc);
  *out = g;
  return 0;
}

extern "C" void xlg_destroy(xlg_group *g) {
  if (g == nullptr) return;
  cudaSetDevice(g->device);
  if (g->s_in) cudaStreamSynchronize(g->s_in);
  for (const xlg_group::StreamSet *ss : {&g->set_part, &g->set_plain}) {
    if (ss->ph) cudaStreamSynchronize(ss->ph);
    if (ss->cv) cudaStreamSynchronize(ss->cv);
    for (cudaStream_t st : ss->cs)
      if (st) cudaStreamSynchronize(st);
  }
  if (g->s_out) cudaStreamSynchronize(g->s_out);
  if (g->timeline) {
    for (Slot &sl : g->slots)
      if (sl.ticket.load() >= 0) harvest_locked(g, sl);
    FILE *f = fopen(getenv("XLATING_B200_TIMELINE") ? getenv("XLATING_B200_TIMELINE") : "/dev/null", "w");
    if (f != nullptr) {
      fprintf(f, "# ticket conv_ready conv_done phase_start phase_done fir_ready fir_done   (ms since the first submit)\n");
      for (const auto &r : g->tl)
        fprintf(f, "%.0f %.4f %.4f %.4f %.4f %.4f %.4f\n", r[0], r[1], r[2], r[3], r[4], r[5], r[6]);
      fclose(f);
    }
    cudaEventDestroy(g->ev_base);
  }
  if (g->d_trace != nullptr && g->trace_ctas <= 0) cudaFree(g->d_trace);
  if (g->d_trace != nullptr && g->trace_ctas > 0) {
    // timeline of the last T_TRACE_LAUNCHES tiled launches; the summary line is about the newest one
    std::vector<long long> t((size_t)T_TRACE_REC * T_TRACE_CTAS * T_TRACE_LAUNCHES);
    if (cudaMemcpy(t.data(), g->d_trace, t.size() * sizeof(long long), cudaMemcpyDeviceToHost) == cudaSuccess) {
      const int slot = (int)((g->trace_launches - 1) % T_TRACE_LAUNCHES);
      const long long *r = t.data() + (size_t)slot * T_TRACE_REC * T_TRACE_CTAS;
      double stage = 0, loop = 0, epi = 0;
      for (int i = 0; i < g->trace_ctas; i++) {
        const long long *e = r + (size_t)T_TRACE_REC * i;
        const long long t2 = (e[2] & 0x0000ffffffffffffll) | (e[1] & ~0x0000ffffffffffffll);
        stage += (double)(e[1] - e[0]);
        loop += (double)(t2 - e[1]);
        epi += (double)(e[3] - t2);
      }
      const double n = g->trace_ctas;
      fprintf(stderr, "xlating_b200 trace: %d CTAs, mean cycles stage %.0f loop %.0f epilogue %.0f (%.1f%% / %.1f%% / %.1f%%)\n",
              g->trace_ctas, stage / n, loop / n, epi / n, 100 * stage / (stage + loop + epi),
              100 * loop / (stage + loop + epi), 100 * epi / (stage + loop + epi));
      const char *path = getenv("XLATING_B200_TRACE_FILE");
      if (path != nullptr) {
        // header: record length, CTAs per launch slot, launch slots, launches so far, CTAs of each slot
        FILE *f = fopen(path, "wb");
        if (f != nullptr) {
          long long hdr[4 + T_TRACE_LAUNCHES] = {T_TRACE_REC, T_TRACE_CTAS, T_TRACE_LAUNCHES, g->trace_launches};
          for (int i = 0; i < T_TRACE_LAUNCHES; i++) hdr[4 + i] = g->trace_n[i];
          fwrite(hdr, sizeof(long long), 4 + T_TRACE_LAUNCHES, f);
          fwrite(t.data(), sizeof(long long), t.size(), f);
          fclose(f);
        }
      }
    }
    cudaFree(g->d_trace);
  }
  for (Slot &s : g->slots) {
    slot_free(s);
    cudaEvent_t evs[] = {s.ev_h2d, s.ev_conv, s.ev_phase, s.ev_fir, s.ev_done};
    for (cudaEvent_t ev : evs)
      if (ev) cudaEventDestroy(ev);
    for (int i = 0; i < 10; i++)
      if (s.pf[i]) cudaEventDestroy(s.pf[i]);
    for (cudaEvent_t ev : s.pf_poly)
      if (ev) cudaEventDestroy(ev);
    for (cudaEvent_t ev : s.pf_casc)
      if (ev) cudaEventDestroy(ev);
    if (s.ev_casc) cudaEventDestroy(s.ev_casc);
    for (cudaEvent_t ev : s.pf_sb)
      if (ev) cudaEventDestroy(ev);
  }
  for (HostOut &h : g->ring_out) {
    if (h.h_out) cudaFreeHost(h.h_out);
    if (h.h_qout) cudaFreeHost(h.h_qout);
    if (h.h_endph) cudaFreeHost(h.h_endph);
    h.n_out.release();
    h.out_off.release();
    h.hist_after.release();
  }
  for (int *p : g->retired_meta_i) delete[] p;
  for (long long *p : g->retired_meta_ll) delete[] p;
  for (void *p : g->retired_host) cudaFreeHost(p);
  if (g->ev_t0) cudaEventDestroy(g->ev_t0);
  if (g->ev_t1) cudaEventDestroy(g->ev_t1);
  if (g->ring) cudaFree(g->ring);
  if (g->qring) cudaFree(g->qring);
  if (g->d_clients) cudaFree(g->d_clients);
  if (g->d_clients_backup) cudaFree(g->d_clients_backup);
  if (g->d_taps) cudaFree(g->d_taps);
  if (g->d_qtaps) cudaFree(g->d_qtaps);
  if (g->d_tile_taps) cudaFree(g->d_tile_taps);
  if (g->d_members) cudaFree(g->d_members);
  if (g->d_member_incr) cudaFree(g->d_member_incr);
  if (g->d_member_cid) cudaFree(g->d_member_cid);
  if (g->d_order) cudaFree(g->d_order);
  if (g->d_poly3) cudaFree(g->d_poly3);
  if (g->d_poly4) cudaFree(g->d_poly4);
  if (g->d_ones) cudaFree(g->d_ones);
  if (g->d_taps2) cudaFree(g->d_taps2);
  if (g->d_sbgrp) cudaFree(g->d_sbgrp);
  if (g->d_sbmem) cudaFree(g->d_sbmem);
  if (g->d_sbtaps) cudaFree(g->d_sbtaps);
  for (HostClient &h : g->clients)
    if (h.d_cring) cudaFree(h.d_cring);
  for (float2 *p : g->dead_rings) cudaFree(p);
  if (g->ev_user) cudaEventDestroy(g->ev_user);
  if (g->s_in) cudaStreamDestroy(g->s_in);
  for (const xlg_group::StreamSet *ss : {&g->set_part, &g->set_plain}) {
    if (ss->ph) cudaStreamDestroy(ss->ph);
    if (ss->cv) cudaStreamDestroy(ss->cv);
    for (cudaStream_t st : ss->cs)
      if (st) cudaStreamDestroy(st);
  }
  if (g->s_out) cudaStreamDestroy(g->s_out);
  if (g->part.small_ctx || g->part.big_ctx) {
    pfn_cuGreenCtxDestroy p_destroy;
    if (drv("cuGreenCtxDestroy", &p_destroy)) {
      if (g->part.small_ctx) p_destroy(g->part.small_ctx);
      if (g->part.big_ctx) p_destroy(g->part.big_ctx);
    }
  }
  delete g;
}

extern "C" int xlg_add_client(xlg_group *g, uint32_t decimation, const float *taps, size_t taps_len,
                              int32_t center_freq, int *client_id) {
  return xlg_add_client_ex(g, decimation, taps, taps_len, center_freq, nullptr, client_id);
}

// Attach a client: the reference filter with `decimation` at `rate` (fs, or interp * fs for a rational client,
// whose taps are kept as polyphase branches).  The callers have validated their arguments.
static int attach_client(xlg_group *g, uint32_t interp, uint32_t decimation, uint32_t rate, const float *taps,
                         size_t taps_len, int32_t center_freq, const xlg_client_state *state, int *client_id) {
  xl_client_consts k;
  int rc = xl_client_consts_build(taps, taps_len, decimation, center_freq, rate, &k);
  if (rc) return rc;
  int id = -1;
  for (size_t i = 0; i < g->clients.size(); i++)
    if (!g->clients[i].active) {
      id = (int)i;
      break;
    }
  if (id < 0) {
    g->clients.emplace_back();
    id = (int)g->clients.size() - 1;
  }
  HostClient &h = g->clients[id];
  h = HostClient();
  h.active = true;
  h.D = decimation;
  h.L = interp;
  h.T = taps_len;
  if (interp == 1) {
    h.rev.assign(k.rev_cf32, k.rev_cf32 + 2 * taps_len);
    h.rev_q15.assign(k.rev_q15, k.rev_q15 + 2 * taps_len);
  } else {
    h.rev.resize(2 * (size_t)interp * ((taps_len + interp - 1) / interp));  // no Q15 path for rational clients
    xl_poly_pack(k.rev_cf32, taps_len, interp, h.rev.data());
  }
  h.incr_re = k.incr_re;
  h.incr_im = k.incr_im;
  h.qincr_re = k.qincr_re;
  h.qincr_im = k.qincr_im;
  h.hist = (long long)taps_len - 1;  // src/xlating.c:552 (upsampled samples for a rational client)
  h.zero_before = g->S;
  h.qzero_before = g->qS;
  if (state != nullptr) {
    // a filter that already consumed the last `valid_history` samples of this stream elsewhere
    // (the per-filter drop-in engine) continues here: same decimation phase, same oscillator;
    // samples further back read as zero, as they did for it
    h.hist = state->hist;
    h.zero_before = g->S - state->valid_history;
    h.init_ph_re = state->phase_re;
    h.init_ph_im = state->phase_im;
  }
  h.is_new = true;
  xl_client_consts_free(&k);
  g->dirty = true;
  *client_id = id;
  return 0;
}

extern "C" int xlg_add_client_ex(xlg_group *g, uint32_t decimation, const float *taps, size_t taps_len,
                                 int32_t center_freq, const xlg_client_state *state, int *client_id) {
  if (g == nullptr || client_id == nullptr) return -EINVAL;
  if (state != nullptr && (state->hist < 0 || state->valid_history < 0 || (size_t)state->hist > taps_len)) return -EINVAL;
  if (taps_len == 0 || taps == nullptr) return -1;  // src/xlating.c:496
  if (decimation == 0) return -EINVAL;
  return attach_client(g, 1, decimation, g->fs, taps, taps_len, center_freq, state, client_id);
}

extern "C" int xlg_add_client_rational(xlg_group *g, uint32_t interp, uint32_t decim, const float *taps,
                                       size_t taps_len, int32_t center_freq, int *client_id) {
  return xlg_add_client_rational_ex(g, interp, decim, taps, taps_len, center_freq, nullptr, client_id);
}

extern "C" int xlg_add_client_rational_ex(xlg_group *g, uint32_t interp, uint32_t decim, const float *taps,
                                          size_t taps_len, int32_t center_freq, const xlg_client_state *state,
                                          int *client_id) {
  if (g == nullptr || client_id == nullptr) return -EINVAL;
  if (interp == 0 || decim == 0) {
    XL_LOG("rational client: interpolation %u and decimation %u must both be at least 1", interp, decim);
    return -EINVAL;
  }
  if ((uint64_t)interp * g->fs > UINT32_MAX) {
    XL_LOG("rational client: %u x %u Hz upsampled rate exceeds UINT32_MAX", interp, g->fs);
    return -EINVAL;
  }
  if ((uint64_t)interp * (g->max_input_len / 2) >= (1ull << 31)) {
    XL_LOG("rational client: %u x %u samples per block upsampled exceed 2^31", interp, g->max_input_len / 2);
    return -EINVAL;
  }
  if (interp == 1) return xlg_add_client_ex(g, decim, taps, taps_len, center_freq, state, client_id);
  // state->hist is in upsampled samples, state->valid_history in input samples (the ring's unit)
  if (state != nullptr && (state->hist < 0 || state->valid_history < 0 || (size_t)state->hist > taps_len)) return -EINVAL;
  if (taps_len == 0 || taps == nullptr) return -1;  // as xlg_add_client (src/xlating.c:496)
  if (taps_len > (size_t)INT32_MAX) return -EINVAL;
  return attach_client(g, interp, decim, interp * g->fs, taps, taps_len, center_freq, state, client_id);
}

extern "C" int xlg_add_client_cascade(xlg_group *g, uint32_t decim1, const float *taps1, size_t taps1_len,
                                      int32_t center_freq, uint32_t decim2, const float *taps2, size_t taps2_len,
                                      int *client_id) {
  return xlg_add_client_cascade_rational(g, decim1, taps1, taps1_len, center_freq, 1, decim2, taps2, taps2_len,
                                         client_id);
}

extern "C" int xlg_add_client_cascade_rational(xlg_group *g, uint32_t decim1, const float *taps1, size_t taps1_len,
                                               int32_t center_freq, uint32_t interp2, uint32_t decim2,
                                               const float *taps2, size_t taps2_len, int *client_id) {
  if (g == nullptr || client_id == nullptr) return -EINVAL;
  if (decim1 == 0 || decim2 == 0 || taps1_len == 0 || taps2_len == 0 || taps1 == nullptr || taps2 == nullptr) {
    XL_LOG("cascade client: decimations (%u, %u) and tap counts (%zu, %zu) must all be at least 1", decim1, decim2,
           taps1_len, taps2_len);
    return -EINVAL;
  }
  if (interp2 == 0) {
    XL_LOG("cascade client: stage-B interpolation must be at least 1");
    return -EINVAL;
  }
  if (interp2 > 1 && (uint64_t)interp2 * ((uint64_t)g->max_input_len / 2 / decim1 + 2) >= (1ull << 31)) {
    XL_LOG("cascade client: %u x %u stage-A samples per block upsampled exceed 2^31", interp2,
           g->max_input_len / 2 / decim1 + 2);
    return -EINVAL;
  }
  if (g->flags & XLG_TRACK_STATE) {
    XL_LOG("cascade client: an XLG_TRACK_STATE group cannot carry the state of two stages");
    return -ENOTSUP;
  }
  const size_t Tb2 = (taps2_len + interp2 - 1) / interp2;
  if (taps2_len > (size_t)INT32_MAX ||
      (interp2 == 1 ? cascade_smem(1, (int)decim2, (int)taps2_len)
                    : cascade_poly_smem(1, (int)interp2, (int)decim2, (int)Tb2)) > (size_t)kTileMaxSmem) {
    XL_LOG("cascade client: %zu stage-B taps (interpolation %u) exceed the stage-B kernel's shared memory", taps2_len,
           interp2);
    return -EINVAL;
  }
  // stage B: the reference filter at interp2 * fs / D1 with centre 0 -- its rotated taps are (h, +-0), so the
  // real parts of the reversed taps (the even-length quirk included) are all it needs; at centre 0 the rate
  // only enters the rotation, so clamping it changes nothing
  const uint64_t rate2 = (uint64_t)interp2 * std::max<uint32_t>(g->fs / decim1, 1);
  xl_client_consts k2;
  int rc = xl_client_consts_build(taps2, taps2_len, decim2, 0, (uint32_t)std::min<uint64_t>(rate2, UINT32_MAX), &k2);
  if (rc) return rc;
  std::vector<float> rev2(taps2_len);
  if (interp2 == 1) {
    for (size_t j = 0; j < taps2_len; j++) rev2[j] = k2.rev_cf32[2 * j];
  } else {
    // branch-major P[r][t] = rev2[r + t * L2], zero-padded to Tb2 taps per branch
    std::vector<float> packed(2 * (size_t)interp2 * Tb2);
    xl_poly_pack(k2.rev_cf32, taps2_len, interp2, packed.data());
    rev2.resize((size_t)interp2 * Tb2);
    for (size_t j = 0; j < rev2.size(); j++) rev2[j] = packed[2 * j];
  }
  xl_client_consts_free(&k2);
  int id = -1;
  rc = attach_client(g, 1, decim1, g->fs, taps1, taps1_len, center_freq, nullptr, &id);
  if (rc) return rc;
  HostClient &h = g->clients[id];
  h.casc = true;
  h.L2 = interp2;
  h.D2 = decim2;
  h.T2 = taps2_len;
  h.rev2.swap(rev2);
  h.hist2 = (long long)taps2_len - 1;  // src/xlating.c:552 (upsampled samples when L2 > 1)
  if (interp2 > 1) {
    h.Tb2 = (int)Tb2;
    h.ko2 = cascade_poly_ko((int)interp2, (int)decim2, h.Tb2);
  }
  *client_id = id;
  return 0;
}

extern "C" int xlg_reserve(xlg_group *g, size_t output_samples_per_block) {
  if (g == nullptr) return -EINVAL;
  CU_OK(cudaSetDevice(g->device));
  if (output_samples_per_block <= g->arena_cap) return 0;
  if (drain(g)) return -EIO;
  // ensure_arenas adds 25 % on top: ask for exactly what was requested
  return ensure_arenas(g, output_samples_per_block - output_samples_per_block / 5, g->q_alloc);
}

extern "C" int xlg_remove_client(xlg_group *g, int client_id) {
  if (g == nullptr || client_id < 0 || client_id >= (int)g->clients.size() || !g->clients[client_id].active ||
      g->clients[client_id].sb)
    return -EINVAL;
  g->clients[client_id].active = false;
  if (g->clients[client_id].d_cring) g->dead_rings.push_back(g->clients[client_id].d_cring);  // in-flight tickets read it
  g->clients[client_id].d_cring = nullptr;
  g->clients[client_id].rev2.clear();
  g->clients[client_id].rev.clear();
  g->clients[client_id].rev_q15.clear();
  g->dirty = true;
  return 0;
}

extern "C" int xlg_client_count(const xlg_group *g) {
  if (g == nullptr) return -EINVAL;
  int n = 0;
  for (const HostClient &h : g->clients) n += h.active && !h.sb ? 1 : 0;
  return n;
}

extern "C" int xlg_client_info(const xlg_group *g, int client_id, size_t *history, int *kernel_kind) {
  if (g == nullptr || client_id < 0 || client_id >= (int)g->clients.size() || !g->clients[client_id].active ||
      g->clients[client_id].sb)
    return -EINVAL;
  if (history) *history = (size_t)(g->clients[client_id].mem ? g->clients[client_id].hist2 : g->clients[client_id].hist);
  if (kernel_kind) *kernel_kind = g->clients[client_id].casc ? 5 : g->clients[client_id].kind;
  return 0;
}

extern "C" int xlg_cascade_info(const xlg_group *g, int client_id, int *stage_a_kind, size_t *stage_a_history,
                                size_t *stage_b_history) {
  if (g == nullptr || client_id < 0 || client_id >= (int)g->clients.size() || !g->clients[client_id].active ||
      !g->clients[client_id].casc)
    return -EINVAL;
  const HostClient &h = g->clients[client_id];
  if (stage_a_kind) *stage_a_kind = h.kind;
  if (stage_a_history) *stage_a_history = (size_t)h.hist;
  if (stage_b_history) *stage_b_history = (size_t)h.hist2;
  return 0;
}

extern "C" int xlg_add_subband(xlg_group *g, uint32_t decim1, const float *taps1, size_t taps1_len,
                               int32_t center_freq, int *subband_id) {
  if (g == nullptr || subband_id == nullptr) return -EINVAL;
  if (decim1 == 0 || taps1_len == 0 || taps1 == nullptr) {
    XL_LOG("sub-band: decimation %u and tap count %zu must both be at least 1", decim1, taps1_len);
    return -EINVAL;
  }
  if (g->fs % decim1 != 0) {
    XL_LOG("sub-band: decimation %u does not divide the band rate %u (members are centred in Hz at fs / decim1)",
           decim1, g->fs);
    return -EINVAL;
  }
  if (g->flags & XLG_TRACK_STATE) {
    XL_LOG("sub-band: an XLG_TRACK_STATE group cannot carry the state of two stages");
    return -ENOTSUP;
  }
  int cid = -1;
  const int rc = attach_client(g, 1, decim1, g->fs, taps1, taps1_len, center_freq, nullptr, &cid);
  if (rc) return rc;
  int id = 0;
  while (id < (int)g->subbands.size() && g->subbands[id] >= 0) id++;
  if (id == (int)g->subbands.size()) g->subbands.push_back(-1);
  g->subbands[id] = cid;
  g->clients[cid].sb = true;
  g->clients[cid].sb_id = id;
  *subband_id = id;
  return 0;
}

static int subband_client(const xlg_group *g, int subband_id) {
  if (subband_id < 0 || subband_id >= (int)g->subbands.size()) return -1;
  return g->subbands[subband_id];
}

extern "C" int xlg_remove_subband(xlg_group *g, int subband_id) {
  if (g == nullptr) return -EINVAL;
  const int cid = subband_client(g, subband_id);
  if (cid < 0) {
    XL_LOG("sub-band %d does not exist", subband_id);
    return -EINVAL;
  }
  int members = 0;
  for (const HostClient &h : g->clients) members += h.active && h.mem && h.sb_cid == cid ? 1 : 0;
  if (members > 0) {
    XL_LOG("sub-band %d still has %d members; remove them first", subband_id, members);
    return -EBUSY;
  }
  g->clients[cid].sb = false;
  g->subbands[subband_id] = -1;
  return xlg_remove_client(g, cid);
}

extern "C" int xlg_add_client_subband(xlg_group *g, int subband_id, uint32_t decim2, const float *taps2,
                                      size_t taps2_len, int32_t center_offset, int *client_id) {
  return xlg_add_client_subband_rational(g, subband_id, 1, decim2, taps2, taps2_len, center_offset, client_id);
}

extern "C" int xlg_add_client_subband_rational(xlg_group *g, int subband_id, uint32_t interp2, uint32_t decim2,
                                               const float *taps2, size_t taps2_len, int32_t center_offset,
                                               int *client_id) {
  if (g == nullptr || client_id == nullptr) return -EINVAL;
  const int sb = subband_client(g, subband_id);
  if (sb < 0) {
    XL_LOG("sub-band member: sub-band %d does not exist", subband_id);
    return -EINVAL;
  }
  if (decim2 == 0 || taps2_len == 0 || taps2 == nullptr) {
    XL_LOG("sub-band member: decimation %u and tap count %zu must both be at least 1", decim2, taps2_len);
    return -EINVAL;
  }
  if (interp2 == 0) {
    XL_LOG("sub-band member: interpolation must be at least 1");
    return -EINVAL;
  }
  const uint32_t decim1 = g->clients[sb].D;
  if ((uint64_t)interp2 * (g->fs / decim1) > UINT32_MAX) {
    XL_LOG("sub-band member: %u x %u Hz upsampled rate exceeds UINT32_MAX", interp2, g->fs / decim1);
    return -EINVAL;
  }
  if ((uint64_t)interp2 * ((uint64_t)g->max_input_len / 2 / decim1 + 2) >= (1ull << 31)) {
    XL_LOG("sub-band member: %u x %u sub-band samples per block upsampled exceed 2^31", interp2,
           g->max_input_len / 2 / decim1 + 2);
    return -EINVAL;
  }
  // one branch's taps for a group and the window of SB_KO outputs (of one residue) in shared memory
  const size_t Tb2 = (taps2_len + interp2 - 1) / interp2;
  if (taps2_len > (size_t)INT32_MAX || decim2 > (uint32_t)INT32_MAX ||
      subband_smem((int)decim2, (int)Tb2) > (size_t)kTileMaxSmem) {
    XL_LOG("sub-band member: %zu taps at interpolation %u, decimation %u exceed the member kernel's shared memory",
           taps2_len, interp2, decim2);
    return -EINVAL;
  }
  // the reference filter at interp2 * fs / D1 centred center_offset from the sub-band: rotated reversed taps
  // (the even-length reversal quirk included) and oscillator step
  xl_client_consts k;
  int rc = xl_client_consts_build(taps2, taps2_len, decim2, center_offset, interp2 * (g->fs / decim1), &k);
  if (rc) return rc;
  int id = -1;
  for (size_t i = 0; i < g->clients.size(); i++)
    if (!g->clients[i].active) {
      id = (int)i;
      break;
    }
  if (id < 0) {
    g->clients.emplace_back();
    id = (int)g->clients.size() - 1;
  }
  HostClient &h = g->clients[id];
  h = HostClient();
  h.active = true;
  h.mem = true;
  h.sb_cid = sb;
  h.D = 0;
  h.L2 = interp2;
  h.D2 = decim2;
  h.T2 = taps2_len;
  h.Tb2 = (int)Tb2;
  if (interp2 == 1) {
    h.rev2.assign(k.rev_cf32, k.rev_cf32 + 2 * taps2_len);
  } else {
    h.rev2.resize(2 * (size_t)interp2 * Tb2);  // branch-major P[r][t] = rev[r + t * L2], zero-padded
    xl_poly_pack(k.rev_cf32, taps2_len, interp2, h.rev2.data());
  }
  h.incr_re = k.incr_re;
  h.incr_im = k.incr_im;
  h.hist2 = (long long)taps2_len - 1;  // src/xlating.c:552 (upsampled samples when L2 > 1)
  h.zb2 = g->clients[sb].a_pos;
  h.is_new = true;
  xl_client_consts_free(&k);
  g->dirty = true;
  *client_id = id;
  return 0;
}

extern "C" int xlg_subband_info(const xlg_group *g, int client_id, int *subband_id, int *stage_a_kind,
                                size_t *member_history) {
  if (g == nullptr || client_id < 0 || client_id >= (int)g->clients.size() || !g->clients[client_id].active ||
      !g->clients[client_id].mem)
    return -EINVAL;
  const HostClient &h = g->clients[client_id];
  if (subband_id) *subband_id = g->clients[h.sb_cid].sb_id;
  if (stage_a_kind) *stage_a_kind = g->clients[h.sb_cid].kind;
  if (member_history) *member_history = (size_t)h.hist2;
  return 0;
}

template <int FMT>
static void launch_convert(bool q15, const void *raw, xlg_group *g, long long S, int n, cudaStream_t st) {
  const int threads = 256, blocks = (n + threads - 1) / threads;
  const unsigned mask = (unsigned)(g->ring_cap - 1);
  const size_t pair_bytes = FMT == 2 ? 8 : 4;
  if (q15) {
    convert_q15_kernel<FMT><<<blocks, threads, 0, st>>>(raw, g->qring, mask, S, n);
  } else if ((n & 1) == 0 && (S & 1) == 0 && ((uintptr_t)raw % pair_bytes) == 0) {
    const int per_cta = threads * CV_STEPS * 2;
    convert_cf32_vec_kernel<FMT><<<(n + per_cta - 1) / per_cta, threads, 0, st>>>(raw, g->ring, mask, S, n);
  } else {
    convert_cf32_kernel<FMT><<<blocks, threads, 0, st>>>(raw, g->ring, mask, S, n);
  }
}

extern "C" int64_t xlg_submit(xlg_group *g, int fmt, const void *input, size_t input_len, uint32_t flags) {
  if (g == nullptr || (input == nullptr && input_len > 0)) return -EINVAL;
  if (fmt < XLG_FMT_CU8 || fmt > XLG_FMT_CS16) return -EINVAL;
  if (input_len > g->max_input_len) {
    XL_LOG("block of %zu elements exceeds max_input_len %u", input_len, g->max_input_len);
    return -EINVAL;
  }
  const bool q15 = (flags & XLG_PATH_Q15) != 0;
  if (q15)
    for (const HostClient &h : g->clients)
      if (h.active && (h.L > 1 || h.casc)) {
        XL_LOG("the Q15 path does not serve rational or cascade clients; submit without XLG_PATH_Q15");
        return -ENOTSUP;
      } else if (h.active && h.sb) {
        XL_LOG("the Q15 path does not serve sub-bands; submit without XLG_PATH_Q15");
        return -ENOTSUP;
      }
  CU_OK(cudaSetDevice(g->device));
  const bool dev_in = (flags & XLG_INPUT_DEVICE) != 0;
  const bool dev_out = (g->flags & XLG_OUT_DEVICE) != 0;

  // clients whose zero-history window has passed may move to a tiled / long class
  if (!g->dirty && !q15) {
    for (const HostClient &h : g->clients)
      if (h.active && h.pending_settle && h.zero_before <= first_input(h, g->S)) {
        g->dirty = true;
        break;
      }
  }
  // a speculative pre-pass that guessed wrong (another length, the Q15 path, a changed client
  // set) is undone BEFORE anything reads the client table again
  {
    const int64_t t_next = g->next_ticket.load();
    const bool hit = g->spec_valid && !q15 && !g->dirty && !g->profiling && g->spec_ticket == t_next &&
                     g->spec_S == g->S && g->spec_n == (int)(input_len / 2);
    if (g->spec_valid && !hit) {
      restore_clients_kernel<<<(g->max_client + 127) / 128, 128, 0, g->s_ph>>>(g->d_clients, g->d_clients_backup,
                                                                              g->max_client);
      g->spec_valid = false;
      g->spec_misses++;
    }
  }
  if (q15 && (!g->qring || !g->q_alloc)) {
    if (drain(g)) return -EIO;
    int rc = ensure_ring(g, g->hist_cap, true);
    if (rc) return rc;
    rc = ensure_arenas(g, g->arena_cap, true);
    if (rc) return rc;
  }
  if (g->dirty) {
    int rc = rebuild_layout(g);
    if (rc) return rc;
  }

  const int64_t ticket = g->next_ticket.load();
  Slot &s = g->slots[ticket % XLG_SLOTS];
  HostOut &ho = g->ring_out[ticket % (int64_t)g->ring_out.size()];
  const auto t_enter = std::chrono::steady_clock::now();
  if (s.ticket.load() >= 0) {
    CU_OK(cudaEventSynchronize(s.ev_done));
    g->host_wait_ns += (uint64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(
                           std::chrono::steady_clock::now() - t_enter).count();
    std::lock_guard<std::mutex> lk(g->mu);
    harvest_locked(g, s);
  }
  const int n = (int)(input_len / 2);  // complex samples (src/xlating.c:387)
  const long long S = q15 ? g->qS : g->S;
  const int nc = g->max_client;
  const unsigned mask = (unsigned)(g->ring_cap - 1);

  // host mirror of the per-client output counts (same integer formula as the
  // oscillator pre-pass kernel)
  {
    // consumers read this entry's metadata under the same mutex (xlg_output) / spinlock (xlg_copy_output)
    std::lock_guard<std::mutex> lk(g->mu);
    ho.ticket.store(-1);  // the entry is being recycled (seqlock write-begin for lock-free readers)
    std::atomic_thread_fence(std::memory_order_seq_cst);
    ho.n_out.assign(g->clients.size(), 0);
    ho.out_off.assign(g->clients.size(), 0);
    if (g->flags & XLG_TRACK_STATE) ho.hist_after.assign(g->clients.size(), 0);
    ho.q15 = q15;
  }
  s.q15 = q15;
  s.tile_macs = s.algo_macs = s.out_samples = s.poly_macs = s.casc_macs = s.d2h_bytes = 0;
  s.in_samples = (uint64_t)n;
  int max_generic_out = 0, poly_warps = 0, max_poly4_out = 0, n_casc = 0, max_n1 = 0, max_n2 = 0;
  int n_cint = 0, n_crat = 0, max_rat_ctas = 0;  // integer / rational stage B; CTAs per rational client
  size_t casc_smem = 0, casc_poly_smem = 0;
  for (size_t i = 0; i < g->clients.size(); i++) {
    HostClient &h = g->clients[i];
    if (!h.active || h.mem) continue;
    // upsampled coordinates (the same integers for L = 1)
    const long long Su = S * h.L, Eu = (S + n) * h.L;
    const long long first = Su - h.hist;
    const long long last_ok = Eu - (long long)h.T;
    int n_out = 0;
    if (last_ok >= first) n_out = (int)((last_ok - first) / (long long)h.D) + 1;
    if (n_out > h.out_cap) n_out = h.out_cap;
    ho.n_out[i] = n_out;
    ho.out_off[i] = h.out_off;
    h.hist = Eu - (first + (long long)n_out * (long long)h.D);
    if (g->flags & XLG_TRACK_STATE) ho.hist_after[i] = h.hist;
    s.out_samples += (uint64_t)n_out;
    const uint64_t macs = (uint64_t)n_out * ((h.T + h.L - 1) / h.L);
    s.algo_macs += macs;
    if (h.kind >= 3) s.poly_macs += macs;
    if (h.kind == 4) max_poly4_out = std::max(max_poly4_out, n_out);
    if (h.kind == 3) {
      // warps of fir_poly_generic_cf32_kernel: min(L, n_out) residues x groups of G_OPW outputs
      const int per = (int)((n_out + (long long)h.L - 1) / h.L);
      poly_warps = std::max(poly_warps, (int)std::min<long long>(h.L, n_out) * ((per + G_OPW - 1) / G_OPW));
    }
    if (q15 || h.kind == 0) max_generic_out = std::max(max_generic_out, n_out);
    if (h.casc) {
      // stage B: the reference's walk over this block's n_out stage-A samples, upsampled by L2 (the
      // zero-stuffed stream u[L2 * n] = y[n]; the same integers for L2 = 1)
      const long long first2 = (long long)h.L2 * h.a_pos - h.hist2;
      const int n2 = xl_walk(&h.hist2, (long long)h.L2 * n_out, h.T2, h.D2, h.fin_cap);
      CascBlk &cb = s.h_cblk[h.L2 == 1 ? n_cint++ : g->n_casc_int + n_crat];
      cb.ring = h.d_cring;
      cb.a_pos = h.a_pos;
      cb.first = first2;
      cb.mask = (unsigned)(h.cring_cap - 1);
      cb.a_off = h.out_off;
      cb.n1 = n_out;
      cb.n2 = n2;
      cb.D2 = (int)h.D2;
      cb.T2 = (int)h.T2;
      cb.taps_off = h.taps2_off;
      cb.out_off = h.fin_off;
      if (h.L2 == 1) {
        max_n2 = std::max(max_n2, n2);
        casc_smem = std::max(casc_smem, cascade_smem(C_KO, cb.D2, cb.T2));
        s.casc_macs += (uint64_t)n2 * h.T2;
      } else {
        // only the appends read this client's CascBlk; cascade_fir_poly_cf32_kernel reads its CascPolyBlk
        CascPolyBlk &pb = s.h_pblk[n_crat++];
        pb.ring = h.d_cring;
        pb.first = first2;
        pb.mask = cb.mask;
        pb.n2 = n2;
        pb.L2 = (int)h.L2;
        pb.M2 = (int)h.D2;
        pb.Tb2 = h.Tb2;
        pb.ko = h.ko2;
        pb.taps_off = h.taps2_off;
        pb.out_off = h.fin_off;
        max_rat_ctas = std::max(max_rat_ctas, (n2 + h.ko2 - 1) / h.ko2);
        casc_poly_smem = std::max(casc_poly_smem, cascade_poly_smem(h.ko2, pb.L2, pb.M2, pb.Tb2));
        s.casc_macs += (uint64_t)n2 * (uint64_t)h.Tb2;
      }
      n_casc++;
      h.a_pos += n_out;
      h.last_n2 = n2;
      max_n1 = std::max(max_n1, n_out);
    }
  }

  // sub-band members: each class walks its sub-band's n1 new samples with the reference's count formula, in
  // sub-band coordinates (the sub-band's a_pos before this block's samples), upsampled by L2 for a rational
  // class
  const int n_sb = (int)g->sb_list.size();
  int max_sb_n1 = 0, max_sb_n2 = 0;
  int max_sbr_ctas = 0, max_sbr_l2 = 0;  // rational classes: output tiles of the longest residue, largest L2
  size_t sb_smem = 0, sbr_smem = 0;
  s.sb_macs = s.sb_rows = 0;
  if (n_sb > 0) {
    for (size_t c = 0; c < g->sb_classes.size(); c++) {
      const SbClassHost &ch = g->sb_classes[c];
      const HostClient &a = g->clients[ch.sb_cid];
      const HostClient &m0 = g->clients[ch.members[0]];
      long long hist2 = m0.hist2;
      const long long first2 = (long long)ch.L2 * a.a_pos - hist2;
      const int n2 = xl_walk(&hist2, (long long)ch.L2 * ho.n_out[ch.sb_cid], m0.T2, m0.D2, m0.out_cap);
      SbBlk &b = s.h_sbblk[c];
      b.ring = a.d_cring;
      b.first = first2;
      b.zb = ch.zb;
      b.mask = (unsigned)(a.cring_cap - 1);
      b.n2 = n2;
      b.D2 = (int)m0.D2;
      b.T2 = ch.Tb;
      for (int id : ch.members) {
        g->clients[id].hist2 = hist2;
        ho.n_out[id] = n2;
        ho.out_off[id] = g->clients[id].out_off;
      }
      s.sb_macs += (uint64_t)n2 * ch.Tb * ch.members.size();
      if (ch.L2 == 1) {
        max_sb_n2 = std::max(max_sb_n2, n2);
        sb_smem = std::max(sb_smem, subband_smem(b.D2, b.T2));
      } else if (n2 > 0) {
        max_sbr_ctas = std::max(max_sbr_ctas, ((n2 + ch.L2 - 1) / ch.L2 + SB_KO - 1) / SB_KO);
        max_sbr_l2 = std::max(max_sbr_l2, ch.L2);
        sbr_smem = std::max(sbr_smem, subband_smem(b.D2, b.T2));
      }
    }
    for (int k = 0; k < n_sb; k++) {
      const int i = g->sb_list[k];
      HostClient &a = g->clients[i];
      const int n1 = ho.n_out[i];
      CascBlk &cb = s.h_sbcb[k];
      memset(&cb, 0, sizeof(cb));
      cb.ring = a.d_cring;
      cb.a_pos = a.a_pos;
      cb.mask = (unsigned)(a.cring_cap - 1);
      cb.a_off = a.out_off;
      cb.n1 = n1;
      a.a_pos += n1;
      s.sb_rows += (uint64_t)n1;
      max_sb_n1 = std::max(max_sb_n1, n1);
    }
  }

  // consecutive blocks alternate between two compute streams so that the tail of
  // one block's FIR overlaps the head of the next (each block's launch alone
  // cannot fill 132 SMs evenly); per-kernel profiling keeps a single stream so
  // that event-timed durations are not inflated by the overlap
  cudaStream_t cs = g->profiling ? g->s_cs[0] : g->s_cs[ticket % g->n_cs];
  cudaStream_t cvs = g->conv_own_stream ? g->s_cv : cs;  // stream of the raw -> ring conversion

  // ---- input staging ----
  const void *d_in = input;
  if (!dev_in && n > 0) {
    const size_t bytes = (size_t)n * 2 * elem_bytes(fmt);
    cudaPointerAttributes attr;
    bool pinned = false;
    if (cudaPointerGetAttributes(&attr, input) == cudaSuccess)
      pinned = attr.type == cudaMemoryTypeHost;
    else
      cudaGetLastError();
    const void *src = input;
    if (!pinned) {
      memcpy(s.h_raw, input, bytes);
      src = s.h_raw;
    }
    CU_OK(cudaMemcpyAsync(s.d_raw, src, bytes, cudaMemcpyHostToDevice, g->s_in));
    CU_OK(cudaEventRecord(s.ev_h2d, g->s_in));
    CU_OK(cudaStreamWaitEvent(cvs, s.ev_h2d, 0));
    // caller-owned pinned memory is read by the copy engine AFTER this call returns: unless
    // the caller promised to leave it alone (XLG_INPUT_KEEP), wait for the copy (a 256 KiB
    // block is ~10 us) so that the buffer may be reused at once, like a pageable one
    if (pinned && !(flags & XLG_INPUT_KEEP)) CU_OK(cudaEventSynchronize(s.ev_h2d));
    d_in = s.d_raw;
  }

  if (g->user_wait_pending) {
    // (in-order streams: later submits' conversions queue behind this one's, so one wait is enough)
    CU_OK(cudaStreamWaitEvent(cvs, g->ev_user, 0));
    CU_OK(cudaStreamWaitEvent(g->s_in, g->ev_user, 0));
    if (!g->conv_own_stream)
      for (int i = 0; i < g->n_cs; i++) CU_OK(cudaStreamWaitEvent(g->s_cs[i], g->ev_user, 0));
    g->user_wait_pending = false;
  }
  // ---- convert (its own stream: never behind the FIR CTAs of earlier blocks that still wait for an SM) ----
  s.pf_conv = s.pf_phase = s.pf_tile = s.pf_gen = false;
  if (n > 0) {
    if (g->timeline && !g->base_recorded) {
      CU_OK(cudaEventRecord(g->ev_base, cvs));
      g->base_recorded = true;
    }
    if (g->profiling || g->timeline) {
      CU_OK(cudaEventRecord(s.pf[0], cvs));
      s.pf_conv = true;
    }
    if (fmt == XLG_FMT_CU8)
      launch_convert<0>(q15, d_in, g, S, n, cvs);
    else if (fmt == XLG_FMT_CS8)
      launch_convert<1>(q15, d_in, g, S, n, cvs);
    else
      launch_convert<2>(q15, d_in, g, S, n, cvs);
    if (g->profiling || g->timeline) CU_OK(cudaEventRecord(s.pf[1], cvs));
    CU_OK(cudaEventRecord(s.ev_conv, cvs));
  }
  // the FIR reads this block's samples and, as history, the previous blocks'
  // (s_cv is in order: waiting for THIS block's conversion covers the earlier ones -- one driver call less)
  if (g->have_last_conv && (cvs == cs || n == 0)) CU_OK(cudaStreamWaitEvent(cs, g->ev_last_conv_ref, 0));
  if (n > 0) {
    if (cvs != cs) CU_OK(cudaStreamWaitEvent(cs, s.ev_conv, 0));
    g->ev_last_conv_ref = s.ev_conv;
    g->have_last_conv = true;
  }

  // ---- oscillator pre-pass (own stream: chains only on the previous pre-pass) ----
  if (nc > 0) {
    const bool tl_phase = g->timeline && !(g->spec_valid && !q15);  // a pre-pass that ran ahead was stamped then
    if (g->profiling) CU_OK(cudaEventRecord(s.pf[2], g->s_ph));
    if (tl_phase) CU_OK(cudaEventRecord(s.tl_ph[(ticket / XLG_SLOTS) & 1][0], g->s_ph));
    if (g->profiling || g->timeline) s.pf_phase = true;
    bool ran_ahead = false;
    if (q15) {
      phase_q15_kernel<<<(nc + P_QTHREADS - 1) / P_QTHREADS, P_QTHREADS, 0, g->s_ph>>>(g->d_clients, nc, s.d_blk,
                                                                                      s.d_qphases, S, n);
    } else if (g->spec_valid) {
      // guessed right (checked on entry): this block's pre-pass was launched with the previous
      // block and s.ev_phase was recorded then
      ran_ahead = true;
      g->spec_valid = false;
      g->spec_hits++;
    } else {
      phase_cf32_kernel<<<g->n_order / 32, P_THREADS, 0, g->s_ph>>>(g->d_clients, g->d_order, s.d_blk, s.d_phases,
                                                                   s.d_endph, nullptr, S, n);
    }
    if (g->profiling) CU_OK(cudaEventRecord(s.pf[3], g->s_ph));
    if (tl_phase) CU_OK(cudaEventRecord(s.tl_ph[(ticket / XLG_SLOTS) & 1][1], g->s_ph));
    if (!ran_ahead) CU_OK(cudaEventRecord(s.ev_phase, g->s_ph));
    CU_OK(cudaStreamWaitEvent(cs, s.ev_phase, 0));
    // ... and the NEXT block's pre-pass, assuming it is as long as this one
    if (!q15 && g->speculate && !g->profiling && n > 0 && g->n_order > 0 && g->d_clients_backup != nullptr) {
      Slot &ns = g->slots[(ticket + 1) % XLG_SLOTS];
      if (ns.ticket.load() >= 0) CU_OK(cudaStreamWaitEvent(g->s_ph, ns.ev_done, 0));  // its tables are still in use
      // (the kernel itself saves every client's state before it advances it: no copy on the critical path)
      if (g->timeline) CU_OK(cudaEventRecord(ns.tl_ph[((ticket + 1) / XLG_SLOTS) & 1][0], g->s_ph));
      phase_cf32_kernel<<<g->n_order / 32, P_THREADS, 0, g->s_ph>>>(g->d_clients, g->d_order, ns.d_blk, ns.d_phases,
                                                                   ns.d_endph, g->d_clients_backup, S + n, n);
      if (g->timeline) CU_OK(cudaEventRecord(ns.tl_ph[((ticket + 1) / XLG_SLOTS) & 1][1], g->s_ph));
      CU_OK(cudaEventRecord(ns.ev_phase, g->s_ph));
      g->spec_valid = true;
      g->spec_S = S + n;
      g->spec_n = n;
      g->spec_ticket = ticket + 1;
    }
  }

  // ---- FIR ----
  if (!q15 && !g->classes.empty()) {
    // Tile shape for this launch: the largest thread tile (best FMA : load ratio) that
    // still yields about two CTAs per SM; fewer clients / outputs -> smaller tiles.
    // (The natural input layout is 2-way bank conflicting for even D, which 16 output
    // lanes absorb and 32 would not, so the production shapes all have LO = 16.
    // Measured on cfg2: an isolated launch takes ~94 us with every shape -- finer tiles
    // balance better but pay more shared loads per FMA -- while in steady state, where
    // consecutive blocks overlap, RK = 4 is 25 % faster than RK = 1.)
    // The 128-output tile of 4 warps (two output sets) must fit 3 CTAs per SM, and it is taken only
    // when its waves are at least 70 % full: its CTAs are twice as long, so a thin last wave idles SMs
    // for longer (measured on H100: cfg2 at 0.80 and c1000 at 0.72 run faster with it, c512 at 0.54
    // ran 4 % slower).
    // input tile + tap stages of a class at KT outputs per CTA (the merged layout reads D more samples)
    auto tile_smem = [](const TileClassHost &ch, int KT) {
      return (size_t)T_SMEM_FIXED + ((size_t)(KT - 1) * ch.k.Dp + ch.k.L + ch.k.D + 10) * sizeof(float2);
    };
    int si = kTileSmallest;
    for (int i = 0; i <= kTileSmallest; i++) {
      const TileShapeHost &sh = kTileShapes[i];
      const int kt = sh.kt();
      int ctas = 0;
      bool fits = true;
      for (TileClassHost &ch : g->classes) {
        int n_out = 0;
        for (int id : ch.real) n_out = std::max(n_out, ho.n_out[id]);
        if (n_out > 0) ctas += ((n_out + kt - 1) / kt) * ch.k.n_groups;
        if (sh.min_ctas > 0 && tile_smem(ch, kt) > (size_t)(kSmSmem / sh.min_ctas - 1024)) fits = false;
      }
      const int slots = sh.min_ctas * g->fir_sms;  // resident CTAs per wave
      if (sh.min_ctas > 0 && ctas > 0 && 10 * ctas < 7 * ((ctas + slots - 1) / slots) * slots) fits = false;
      if (fits && ctas >= 2 * g->fir_sms) {
        si = i;
        break;
      }
    }
    if (g->tile_force > 0) {  // a shape of kTileShapes (checked in xlg_create_ex)
      si = tile_shape_index(g->tile_force);
      for (TileClassHost &ch : g->classes)  // an experiment must not overflow shared memory
        if (tile_smem(ch, kTileShapes[si].kt()) > (size_t)kTileMaxSmem) si = kTileSmallest;
    }
    const TileShapeHost &shape = kTileShapes[si];
    const int KT = shape.kt();
    TileLaunch P;
    memset(&P, 0, sizeof(P));
    int ctas = 0;
    size_t smem = 0;
    for (TileClassHost &ch : g->classes) {
      int n_out = 0;
      for (int id : ch.real) n_out = std::max(n_out, ho.n_out[id]);
      if (n_out <= 0) continue;
      TileClass k = ch.k;
      if (ch.merged) {
        // earliest possible window start of this block (history = T-1); every member's
        // window starts delta in [0, D) samples later, read on the device from BlkInfo
        k.first = S - (long long)(ch.T - 1);
      } else {
        // identical alignment: hist was already advanced above; recover this block's start
        const HostClient &h0 = g->clients[ch.real[0]];
        k.first = (S + n) - h0.hist - (long long)ho.n_out[ch.real[0]] * (long long)h0.D;
      }
      k.n_out = n_out;
      k.tiles = (n_out + KT - 1) / KT;
      k.xs_len = (KT - 1) * k.Dp + k.L + (ch.merged ? k.D : 0);
      k.cta_begin = ctas;
      ctas += k.tiles * k.n_groups;
      smem = std::max(smem, (size_t)T_SMEM_FIXED + ((size_t)k.xs_len + 10) * sizeof(float2));
      P.cls[P.n_classes++] = k;
      s.tile_macs += (uint64_t)k.tiles * KT * (uint64_t)k.L * (uint64_t)ch.members.size();
    }
    if (ctas > 0) {
      if (g->profiling || g->timeline) {
        CU_OK(cudaEventRecord(s.pf[4], cs));
        s.pf_tile = true;
      }
      const float2 *tt = (const float2 *)g->d_tile_taps;
      long long *trace_ptr = nullptr;
      if (g->d_trace != nullptr && ctas <= T_TRACE_CTAS) {
        const int tslot = (int)(g->trace_launches % T_TRACE_LAUNCHES);
        trace_ptr = g->d_trace + (size_t)tslot * T_TRACE_REC * T_TRACE_CTAS;
        g->trace_n[tslot] = ctas;
        g->trace_launches++;
        g->trace_ctas = ctas;
      }
      shape.kernel<<<ctas, shape.threads, smem, cs>>>(P, g->ring, mask, tt, g->d_members, g->d_member_cid,
                                                      g->d_member_incr, s.d_blk, s.d_phases, s.d_out, trace_ptr);
      if (g->profiling || g->timeline) CU_OK(cudaEventRecord(s.pf[5], cs));
    }
  }
  // ---- long filters: split-K partial sums, then the ordered reduction ----
  s.pf_long = false;
  if (!q15 && !g->long_classes.empty()) {
    TileLaunch P;
    memset(&P, 0, sizeof(P));
    int ctas = 0, max_out = 0, max_groups = 0;
    // fir_long4's TMA bulk copies need 16-byte aligned strips: with even D every strip has the parity of
    // the window start, and an odd start is fetched from one sample earlier.  One odd-D class sends the
    // whole launch to fir_long2, which falls back to 8-byte cp.async for unaligned strips.
    bool pipelined = true;
    for (TileClassHost &ch : g->long_classes)
      if (ho.n_out[ch.real[0]] > 0 && (g->clients[ch.real[0]].D & 1) != 0) pipelined = false;
    int n_live = 0;
    for (TileClassHost &ch : g->long_classes) n_live += ho.n_out[ch.real[0]] > 0 ? 1 : 0;
    for (TileClassHost &ch : g->long_classes) {
      const HostClient &h0 = g->clients[ch.real[0]];
      const int n_out = ho.n_out[ch.real[0]];
      if (n_out <= 0) continue;
      TileClass k = ch.k;
      k.first = (S + n) - h0.hist - (long long)n_out * (long long)h0.D;
      k.n_out = n_out;
      k.tiles = (n_out + W2_KT - 1) / W2_KT;
      k.cta_begin = ctas;
      k.nslab = k.nseg;
      k.ksplit = k.nseg;
      k.seg_per = 1;
      if (pipelined) {
        // one resident CTA per SM: as many CTAs along the tap axis as fill one wave of this class's share
        const int units = ((n_out + W4_KT - 1) / W4_KT) * ((k.n_groups + W4_GROUPS - 1) / W4_GROUPS);
        k.tiles = (n_out + W4_KT - 1) / W4_KT;  // (kpad, a multiple of 56, covers 2 x 28 too)
        const int share = std::max(1, g->fir_sms / std::max(n_live, 1));
        const int want = std::max(1, share / std::max(1, units));
        k.seg_per = (k.nseg + std::min(want, k.nseg) - 1) / std::min(want, k.nseg);
        k.ksplit = (k.nseg + k.seg_per - 1) / k.seg_per;
        k.nslab = k.ksplit;
        ctas += k.ksplit * units;
      } else {
        ctas += k.nseg * k.tiles * k.n_groups;
      }
      max_out = std::max(max_out, n_out);
      max_groups = std::max(max_groups, k.n_groups);
      P.cls[P.n_classes++] = k;
      s.tile_macs += (uint64_t)k.tiles * W2_KT * (uint64_t)k.L * (uint64_t)ch.members.size();
    }
    if (ctas > 0) {
      if (g->profiling) {
        CU_OK(cudaEventRecord(s.pf[8], cs));
        s.pf_long = true;
      }
      if (pipelined) {
        // the first class gets the tensor map for its strips (all long clients of a stream normally share one D);
        // tmap_w = 0 (no map) sends every stage down the per-strip bulk copies
        strip_map_update(g, P.cls[0].D);
        P.cls[0].tmap_w = g->strip_w;
        fir_long4_cf32_kernel<<<ctas, W4_THREADS, W4_SMEM, cs>>>(P, g->ring, mask, (const float2 *)g->d_tile_taps,
                                                                s.d_partial, g->strip_map);
      } else {
        fir_long2_cf32_kernel<<<ctas, W2_THREADS, W2_SMEM, cs>>>(P, g->ring, mask, (const float2 *)g->d_tile_taps,
                                                                s.d_partial);
      }
      dim3 rgrid((max_out + 7) / 8, max_groups, P.n_classes);
      fir_long_reduce_kernel<<<rgrid, 256, 0, cs>>>(P, s.d_partial, g->d_members, g->d_member_incr, s.d_phases,
                                                    s.d_out);
      if (g->profiling) CU_OK(cudaEventRecord(s.pf[9], cs));
    }
  }
  if (nc > 0 && max_generic_out > 0) {
    dim3 grid((max_generic_out + G_OPC - 1) / G_OPC, nc);
    if (g->profiling) {
      CU_OK(cudaEventRecord(s.pf[6], cs));
      s.pf_gen = true;
    }
    if (q15)
      fir_generic_q15_kernel<<<grid, G_THREADS, 0, cs>>>(g->d_clients, s.d_blk, g->qring, mask, g->d_qtaps,
                                                             s.d_qphases, s.d_qout);
    else
      fir_generic_cf32_kernel<<<grid, G_THREADS, 0, cs>>>(g->d_clients, s.d_blk, g->ring, mask, g->d_taps,
                                                              s.d_phases, s.d_out);
    if (g->profiling) CU_OK(cudaEventRecord(s.pf[7], cs));
  }
  // ---- rational tiled classes: the tiled kernel over one class per polyphase branch, then the placement ----
  s.pf_pt = false;
  if (!q15 && !g->poly_classes.empty() && max_poly4_out > 0) {
    TileLaunch P;
    memset(&P, 0, sizeof(P));
    // largest tile that still gives about two CTAs per SM (every shape fits: eligibility was checked at 64)
    static const int kPolyShapes[][2] = {{16, 4}, {16, 2}, {16, 1}};
    int lo = 16, rk = 1;
    for (const auto &sh : kPolyShapes) {
      int ctas = 0;
      for (const TileClassHost &ch : g->poly_classes)
        ctas += ((ho.n_out[ch.real[0]] / (int)ch.interp + 1 + sh[0] * sh[1] - 1) / (sh[0] * sh[1])) * ch.k.n_groups;
      if (ctas >= 2 * g->fir_sms) {
        lo = sh[0];
        rk = sh[1];
        break;
      }
    }
    const int KT = lo * rk;
    int ctas = 0;
    size_t smem = 0;
    for (size_t v = 0; v < g->poly_classes.size(); v++) {
      const TileClassHost &ch = g->poly_classes[v];
      const HostClient &h0 = g->clients[ch.real[0]];
      const int n_out = ho.n_out[ch.real[0]];
      const long long L = ch.interp, M = h0.D;
      // this block's first upsampled window (hist was advanced above); branch r serves k = rho + j*L
      const long long first_u = (S + n) * L - h0.hist - (long long)n_out * M;
      const long long a = (((-(first_u + ch.branch)) % L) + L) % L;
      const long long rho = (a * ch.minv) % L;
      const int nv = rho < n_out ? (int)((n_out - 1 - rho) / L) + 1 : 0;
      s.h_vblk[v].first = (first_u + rho * M + ch.branch) / L;  // exact: the window start is -r mod L
      s.h_vblk[v].n_out = nv;
      s.h_vblk[v].pad_ = 0;
      if (nv <= 0) continue;
      TileClass k = ch.k;
      k.first = s.h_vblk[v].first;
      k.n_out = nv;
      k.tiles = (nv + KT - 1) / KT;
      k.xs_len = (KT - 1) * k.Dp + k.L;
      k.cta_begin = ctas;
      ctas += k.tiles * k.n_groups;
      smem = std::max(smem, (size_t)T_SMEM_FIXED + ((size_t)k.xs_len + 10) * sizeof(float2));
      P.cls[P.n_classes++] = k;
      s.tile_macs += (uint64_t)k.tiles * KT * (uint64_t)k.L * (uint64_t)ch.members.size();
    }
    if (ctas > 0) {
      if (g->profiling) {
        CU_OK(cudaEventRecord(s.pf_poly[2], cs));
        s.pf_pt = true;
      }
      CU_OK(cudaMemcpyAsync(s.d_vblk, s.h_vblk, g->poly_classes.size() * sizeof(BlkInfo), cudaMemcpyHostToDevice, cs));
      const float2 *tt = (const float2 *)g->d_tile_taps;
#define XL_LAUNCH_PTILE(RK_)                                                                                     \
  fir_tile_cf32_kernel<16, RK_, 1><<<ctas, TileShape<16, RK_, 1>::kThreads, smem, cs>>>(                          \
      P, g->ring, mask, tt, g->d_members, g->d_member_cid, g->d_member_incr, s.d_vblk, g->d_ones, s.d_pscratch, nullptr)
      if (rk == 4)
        XL_LAUNCH_PTILE(4);
      else if (rk == 2)
        XL_LAUNCH_PTILE(2);
      else
        XL_LAUNCH_PTILE(1);
#undef XL_LAUNCH_PTILE
      dim3 pgrid((max_poly4_out + 255) / 256, g->n_poly4);
      poly_tile_place_cf32_kernel<<<pgrid, 256, 0, cs>>>(g->d_clients, g->d_poly4, s.d_blk, s.d_pscratch, s.d_phases,
                                                         s.d_out);
      if (g->profiling) CU_OK(cudaEventRecord(s.pf_poly[3], cs));
    }
  }
  s.pf_pg = false;
  if (!q15 && g->n_poly3 > 0 && poly_warps > 0) {
    constexpr int warps_per_cta = G_THREADS / 32;
    dim3 grid((poly_warps + warps_per_cta - 1) / warps_per_cta, g->n_poly3);
    if (g->profiling) {
      CU_OK(cudaEventRecord(s.pf_poly[0], cs));
      s.pf_pg = true;
    }
    fir_poly_generic_cf32_kernel<<<grid, G_THREADS, 0, cs>>>(g->d_clients, g->d_poly3, s.d_blk, g->ring, mask, g->d_taps,
                                                             s.d_phases, s.d_out);
    if (g->profiling) CU_OK(cudaEventRecord(s.pf_poly[1], cs));
  }
  // ---- cascade clients: append the stage-A outputs to their rings, then stage B ----
  s.pf_cb = false;
  if (!q15 && n_casc > 0) {
    // the rings are appended in block order: after the previous block's stage B, whichever stream ran it
    if (g->have_last_casc) CU_OK(cudaStreamWaitEvent(cs, g->ev_last_casc, 0));
    if (g->profiling) {
      CU_OK(cudaEventRecord(s.pf_casc[0], cs));
      s.pf_cb = true;
    }
    CU_OK(cudaMemcpyAsync(s.d_cblk, s.h_cblk, (size_t)n_casc * sizeof(CascBlk), cudaMemcpyHostToDevice, cs));
    if (n_crat > 0)
      CU_OK(cudaMemcpyAsync(s.d_pblk, s.h_pblk, (size_t)n_crat * sizeof(CascPolyBlk), cudaMemcpyHostToDevice, cs));
    if (max_n1 > 0) cascade_append_kernel<<<dim3((max_n1 + 255) / 256, n_casc), 256, 0, cs>>>(s.d_cblk, s.d_out);
    if (max_n2 > 0) {
      // fewer outputs per CTA where a long stage-B window would not fit (attach checked that one output fits)
      int ko = C_KO;
      while (ko > 1 && casc_smem > (size_t)kTileMaxSmem) {
        ko /= 2;
        casc_smem = 0;
        for (int c = 0; c < n_cint; c++)
          casc_smem = std::max(casc_smem, cascade_smem(ko, s.h_cblk[c].D2, s.h_cblk[c].T2));
      }
      cascade_fir_cf32_kernel<<<dim3((max_n2 + ko - 1) / ko, n_cint), C_THREADS, casc_smem, cs>>>(s.d_cblk, g->d_taps2,
                                                                                                s.d_out, ko);
    }
    // rational stage B: each client's CTA size was fixed at attach to fit the shared memory
    if (max_rat_ctas > 0)
      cascade_fir_poly_cf32_kernel<<<dim3(max_rat_ctas, n_crat), C_THREADS, casc_poly_smem, cs>>>(s.d_pblk, g->d_taps2,
                                                                                                s.d_out);
    if (g->profiling) CU_OK(cudaEventRecord(s.pf_casc[1], cs));
    CU_OK(cudaEventRecord(s.ev_casc, cs));
    g->ev_last_casc = s.ev_casc;
    g->have_last_casc = true;
    // from here on the client's results are its final row
    for (size_t i = 0; i < g->clients.size(); i++)
      if (g->clients[i].active && g->clients[i].casc) {
        ho.n_out[i] = g->clients[i].last_n2;
        ho.out_off[i] = g->clients[i].fin_off;
      }
  }
  // ---- sub-bands: append their outputs to their rings, then the members' oscillators and FIR ----
  s.pf_sbk = false;
  if (n_sb > 0) {
    // the rings are appended in block order (the cascades' event orders both)
    if (g->have_last_casc) CU_OK(cudaStreamWaitEvent(cs, g->ev_last_casc, 0));
    if (g->profiling) {
      CU_OK(cudaEventRecord(s.pf_sb[0], cs));
      s.pf_sbk = true;
    }
    CU_OK(cudaMemcpyAsync(s.d_sbcb, s.h_sbcb, (size_t)n_sb * sizeof(CascBlk), cudaMemcpyHostToDevice, cs));
    if (max_sb_n1 > 0) cascade_append_kernel<<<dim3((max_sb_n1 + 255) / 256, n_sb), 256, 0, cs>>>(s.d_sbcb, s.d_out);
    if (max_sb_n2 > 0 || max_sbr_ctas > 0) {
      CU_OK(cudaMemcpyAsync(s.d_sbblk, s.h_sbblk, g->sb_classes.size() * sizeof(SbBlk), cudaMemcpyHostToDevice, cs));
      subband_phase_kernel<<<(g->n_sb_mem + 31) / 32, 32, 0, cs>>>(g->d_clients, g->d_sbmem, s.d_sbblk, s.d_sbph);
      if (max_sb_n2 > 0)
        subband_fir_cf32_kernel<<<dim3((max_sb_n2 + SB_KO - 1) / SB_KO, g->n_sb_groups_int), SB_THREADS, sb_smem,
                                  cs>>>(s.d_sbblk, g->d_sbgrp, g->d_sbtaps, s.d_sbph, s.d_out);
      // rational classes: their groups follow the integer ones, one CTA layer per residue
      if (max_sbr_ctas > 0)
        subband_fir_poly_cf32_kernel<<<dim3(max_sbr_ctas, g->n_sb_groups - g->n_sb_groups_int, max_sbr_l2), SB_THREADS,
                                       sbr_smem, cs>>>(s.d_sbblk, g->d_sbgrp + g->n_sb_groups_int, g->d_sbtaps,
                                                       s.d_sbph, s.d_out);
    }
    if (g->profiling) CU_OK(cudaEventRecord(s.pf_sb[1], cs));
    CU_OK(cudaEventRecord(s.ev_casc, cs));
    g->ev_last_casc = s.ev_casc;
    g->have_last_casc = true;
    // (the FIR launches above sized themselves by these counts) a sub-band is not a client: nothing to
    // read, and the D2H copy ends before its row
    for (int i : g->sb_list) {
      ho.n_out[i] = 0;
      ho.out_off[i] = 0;
    }
  }
  CU_OK(cudaGetLastError());
  CU_OK(cudaEventRecord(s.ev_fir, cs));

  // ---- results back to the host ----
  if (!dev_out && g->arena_cap > 0 && nc > 0) {
    size_t used = 0;
    for (size_t i = 0; i < g->clients.size(); i++)
      if (g->clients[i].active) used = std::max(used, (size_t)ho.out_off[i] + (size_t)ho.n_out[i]);  // final rows
    CU_OK(cudaStreamWaitEvent(g->s_out, s.ev_fir, 0));
    if (used > 0) {
      if (q15)
        CU_OK(cudaMemcpyAsync(ho.h_qout, s.d_qout, used * sizeof(short2), cudaMemcpyDeviceToHost, g->s_out));
      else
        CU_OK(cudaMemcpyAsync(ho.h_out, s.d_out, used * sizeof(float2), cudaMemcpyDeviceToHost, g->s_out));
      s.d2h_bytes = used * (q15 ? sizeof(short2) : sizeof(float2));
    }
    if ((g->flags & XLG_TRACK_STATE) && !q15 && s.d_endph != nullptr && ho.h_endph != nullptr)
      CU_OK(cudaMemcpyAsync(ho.h_endph, s.d_endph, (size_t)nc * sizeof(float2), cudaMemcpyDeviceToHost, g->s_out));
    CU_OK(cudaEventRecord(s.ev_done, g->s_out));
  } else {
    CU_OK(cudaEventRecord(s.ev_done, cs));  // results stay on the device: done = FIR done, no hop through s_out
  }

  if (q15)
    g->qS += n;
  else
    g->S += n;
  s.ticket.store(ticket);
  ho.ticket.store(ticket);
  s.harvested = false;
  g->next_ticket.store(ticket + 1);
  g->host_submit_ns += (uint64_t)std::chrono::duration_cast<std::chrono::nanoseconds>(
                           std::chrono::steady_clock::now() - t_enter).count();
  return ticket;
}

extern "C" int xlg_wait(xlg_group *g, int64_t ticket) {
  if (g == nullptr || ticket < 0 || ticket >= g->next_ticket.load()) return -EINVAL;
  HostOut &ho = g->ring_out[ticket % (int64_t)g->ring_out.size()];
  if (ho.ticket.load() != ticket) return -ESTALE;  // overwritten: the consumer fell too far behind
  Slot &s = g->slots[ticket % XLG_SLOTS];
  if (s.ticket.load() == ticket) {
    cudaSetDevice(g->device);
    CU_OK(cudaEventSynchronize(s.ev_done));
    std::lock_guard<std::mutex> lk(g->mu);
    if (s.ticket.load() == ticket) harvest_locked(g, s);
  }
  // else: the device slot already serves a later ticket, which xlg_submit only allows
  // after this ticket's copy-out completed
  return ho.ticket.load() == ticket ? 0 : -ESTALE;
}

extern "C" int xlg_output(xlg_group *g, int64_t ticket, int client_id, const void **out, size_t *out_len) {
  if (g == nullptr || ticket < 0 || ticket >= g->next_ticket.load()) return -EINVAL;
  HostOut &ho = g->ring_out[ticket % (int64_t)g->ring_out.size()];
  std::lock_guard<std::mutex> lk(g->mu);
  if (ho.ticket.load() != ticket) return -ESTALE;
  if (client_id < 0 || client_id >= (int)ho.n_out.size()) return -EINVAL;
  const bool dev_out = (g->flags & XLG_OUT_DEVICE) != 0;
  if (out_len) *out_len = (size_t)ho.n_out[client_id];
  if (out) {
    if (dev_out) {
      Slot &s = g->slots[ticket % XLG_SLOTS];
      if (s.ticket.load() != ticket) return -ESTALE;  // device arenas live XLG_SLOTS tickets
      *out = ho.q15 ? (const void *)(s.d_qout + ho.out_off[client_id]) : (const void *)(s.d_out + ho.out_off[client_id]);
    } else {
      *out = ho.q15 ? (const void *)(ho.h_qout + ho.out_off[client_id]) : (const void *)(ho.h_out + ho.out_off[client_id]);
    }
  }
  return 0;
}

extern "C" int xlg_read_output(xlg_group *g, int64_t ticket, int client_id, void *dst, size_t cap, size_t *out_len) {
  if (g == nullptr || dst == nullptr) return -EINVAL;
  int rc = xlg_wait(g, ticket);
  if (rc != 0) return rc;
  const void *src = nullptr;
  size_t n = 0;
  rc = xlg_output(g, ticket, client_id, &src, &n);
  if (rc != 0) return rc;
  if (out_len) *out_len = n;
  const HostOut &ho = g->ring_out[ticket % (int64_t)g->ring_out.size()];
  const size_t bytes = std::min(n, cap) * (ho.q15 ? sizeof(short2) : sizeof(float2));
  if (bytes == 0) return 0;
  if (g->flags & XLG_OUT_DEVICE) {
    cudaSetDevice(g->device);
    CU_OK(cudaMemcpy(dst, src, bytes, cudaMemcpyDeviceToHost));
    // the device arena may have been recycled while we copied
    if (g->slots[ticket % XLG_SLOTS].ticket.load() != ticket) return -ESTALE;
  } else {
    memcpy(dst, src, bytes);
    // seqlock-style validation: xlg_submit marks the entry (ticket = -1) BEFORE it enqueues the
    // copy that overwrites it, so an unchanged ticket after our reads means they saw this ticket's data
    std::atomic_thread_fence(std::memory_order_acquire);
    if (ho.ticket.load() != ticket) return -ESTALE;
  }
  return 0;
}

extern "C" int xlg_copy_output(xlg_group *g, int64_t ticket, int client_id, void *dst, size_t cap, size_t *out_len,
                               xlg_client_state *state_after) {
  // No CUDA call in here: the caller knows the ticket is complete (it, or the thread that
  // published the block, returned from xlg_wait); hundreds of consumer threads call this
  // per block and must not queue up on the CUDA context lock.
  if (g == nullptr || dst == nullptr || (g->flags & XLG_OUT_DEVICE)) return -EINVAL;
  if (ticket < 0 || ticket >= g->next_ticket.load()) return -EINVAL;
  HostOut &ho = g->ring_out[ticket % (int64_t)g->ring_out.size()];
  const void *src = nullptr;
  size_t n = 0;
  long long hist_after = 0;
  const float2 *endph = nullptr;
  bool q15 = false;
  {
    // lock-free: every consumer thread of a block arrives here at the same moment
    if (ho.ticket.load(std::memory_order_acquire) != ticket) return -ESTALE;
    if (client_id < 0 || client_id >= (int)ho.n_out.size()) return -EINVAL;
    n = (size_t)ho.n_out.get((size_t)client_id);
    q15 = ho.q15;
    const int off = ho.out_off.get((size_t)client_id);
    float2 *const h_out = *(float2 *volatile *)&ho.h_out;
    short2 *const h_qout = *(short2 *volatile *)&ho.h_qout;
    src = q15 ? (const void *)(h_qout + off) : (const void *)(h_out + off);
    if (state_after != nullptr) {
      float2 *const h_endph = *(float2 *volatile *)&ho.h_endph;
      if (!(g->flags & XLG_TRACK_STATE) || q15 || h_endph == nullptr || client_id >= (int)ho.hist_after.size())
        return -EINVAL;
      hist_after = ho.hist_after.get((size_t)client_id);
      endph = h_endph + client_id;
    }
    std::atomic_thread_fence(std::memory_order_acquire);
    if (ho.ticket.load() != ticket) return -ESTALE;  // recycled while we looked: nothing above can be trusted
    if (src == nullptr || n > g->arena_cap) return -ESTALE;
  }
  if (out_len) *out_len = n;
  memcpy(dst, src, std::min(n, cap) * (q15 ? sizeof(short2) : sizeof(float2)));
  if (state_after != nullptr) {
    state_after->hist = hist_after;
    state_after->valid_history = 0;
    state_after->phase_re = endph->x;
    state_after->phase_im = endph->y;
  }
  std::atomic_thread_fence(std::memory_order_acquire);
  return ho.ticket.load() == ticket ? 0 : -ESTALE;
}

extern "C" int xlg_input_consumed(xlg_group *g, int64_t ticket) {
  if (g == nullptr || ticket < 0 || ticket >= g->next_ticket.load()) return -EINVAL;
  Slot &s = g->slots[ticket % XLG_SLOTS];
  if (s.ticket.load() != ticket) return 0;  // the slot serves a later ticket: this one's copy finished long ago
  cudaSetDevice(g->device);
  CU_OK(cudaEventSynchronize(s.ev_h2d));
  return 0;
}

extern "C" void *xlg_alloc_pinned(size_t bytes) {
  void *p = nullptr;
  if (cudaHostAlloc(&p, bytes, cudaHostAllocDefault) != cudaSuccess) {
    XL_LOG("cudaHostAlloc(%zu) failed", bytes);
    return nullptr;
  }
  return p;
}

extern "C" void xlg_free_pinned(void *p) {
  if (p) cudaFreeHost(p);
}

extern "C" int xlg_wait_stream(xlg_group *g, void *cuda_stream) {
  if (g == nullptr) return -EINVAL;
  cudaSetDevice(g->device);
  // Only the first reader of a device-resident input has to wait: the conversion (and the H2D stream, for
  // symmetry with host inputs).  The event is recorded now and attached to the consuming stream by the next
  // xlg_submit -- which knows the stream (a re-layout in between may switch stream sets) -- so a call costs one
  // record here and one wait there instead of a wait on every stream of the group.
  if (g->ev_user == nullptr) CU_OK(cudaEventCreateWithFlags(&g->ev_user, cudaEventDisableTiming));
  CU_OK(cudaEventRecord(g->ev_user, (cudaStream_t)cuda_stream));
  g->user_wait_pending = true;
  return 0;
}

extern "C" int xlg_partition_active(xlg_group *g) {
  if (g == nullptr) return -EINVAL;
  return g->part_active ? g->part.small_sms : 0;
}

extern "C" int xlg_timer_start(xlg_group *g) {
  if (g == nullptr) return -EINVAL;
  cudaSetDevice(g->device);
  if (drain(g)) return -EIO;
  CU_OK(cudaEventRecord(g->ev_t0, g->s_cs[0]));
  // every stream starts after t0
  CU_OK(cudaStreamWaitEvent(g->s_in, g->ev_t0, 0));
  for (int i = 1; i < g->n_cs; i++) CU_OK(cudaStreamWaitEvent(g->s_cs[i], g->ev_t0, 0));
  CU_OK(cudaStreamWaitEvent(g->s_ph, g->ev_t0, 0));
  CU_OK(cudaStreamWaitEvent(g->s_cv, g->ev_t0, 0));
  CU_OK(cudaStreamWaitEvent(g->s_out, g->ev_t0, 0));
  return 0;
}

extern "C" int xlg_timer_stop(xlg_group *g, float *elapsed_ms) {
  if (g == nullptr || elapsed_ms == nullptr) return -EINVAL;
  cudaSetDevice(g->device);
  // s_out's last event already depends on the FIR of the last block; add the others
  cudaEvent_t ev;
  CU_OK(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
  cudaStream_t others[3 + xlg_group::kMaxCs] = {g->s_in, g->s_ph, g->s_cv};
  for (int i = 0; i < g->n_cs; i++) others[3 + i] = g->s_cs[i];
  for (int oi = 0; oi < 3 + g->n_cs; oi++) {
    cudaStream_t st = others[oi];
    CU_OK(cudaEventRecord(ev, st));
    CU_OK(cudaStreamWaitEvent(g->s_out, ev, 0));
  }
  CU_OK(cudaEventRecord(g->ev_t1, g->s_out));
  CU_OK(cudaEventSynchronize(g->ev_t1));
  CU_OK(cudaEventDestroy(ev));
  CU_OK(cudaEventElapsedTime(elapsed_ms, g->ev_t0, g->ev_t1));
  return 0;
}

extern "C" int xlg_profile_enable(xlg_group *g, int on) {
  if (g == nullptr) return -EINVAL;
  cudaSetDevice(g->device);
  if (drain(g)) return -EIO;
  std::lock_guard<std::mutex> lk(g->mu);
  for (Slot &s : g->slots) harvest_locked(g, s);
  g->profiling = on != 0;
  return 0;
}

extern "C" int xlg_poly_profile_read(xlg_group *g, xlg_poly_profile *p, int reset) {
  if (g == nullptr || p == nullptr) return -EINVAL;
  std::lock_guard<std::mutex> lk(g->mu);
  *p = g->poly_prof;
  if (reset) memset(&g->poly_prof, 0, sizeof(g->poly_prof));
  return 0;
}

extern "C" int xlg_cascade_profile_read(xlg_group *g, xlg_cascade_profile *p, int reset) {
  if (g == nullptr || p == nullptr) return -EINVAL;
  std::lock_guard<std::mutex> lk(g->mu);
  *p = g->casc_prof;
  if (reset) memset(&g->casc_prof, 0, sizeof(g->casc_prof));
  return 0;
}

extern "C" int xlg_subband_profile_read(xlg_group *g, xlg_subband_profile *p, int reset) {
  if (g == nullptr || p == nullptr) return -EINVAL;
  std::lock_guard<std::mutex> lk(g->mu);
  *p = g->sb_prof;
  if (reset) memset(&g->sb_prof, 0, sizeof(g->sb_prof));
  return 0;
}

extern "C" int xlg_profile_read(xlg_group *g, xlg_profile *p, int reset) {
  if (g == nullptr || p == nullptr) return -EINVAL;
  std::lock_guard<std::mutex> lk(g->mu);
  *p = g->prof;
  p->host_submit_ms = (double)g->host_submit_ns * 1e-6;
  p->host_wait_ms = (double)g->host_wait_ns * 1e-6;
  p->submits = (uint64_t)g->next_ticket.load() - g->host_count_base;
  if (reset) {
    memset(&g->prof, 0, sizeof(g->prof));
    g->host_submit_ns = g->host_wait_ns = 0;
    g->host_count_base = (uint64_t)g->next_ticket.load();
  }
  return 0;
}

// ---- stage-B launchers for the per-filter engine (cascade_stage_b.cuh) ----
namespace xl {

cudaError_t cascade_stage_b_init() {
  cudaError_t err = cudaFuncSetAttribute(cascade_fir_cf32_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kTileMaxSmem);
  if (err == cudaSuccess)
    err = cudaFuncSetAttribute(cascade_fir_poly_cf32_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kTileMaxSmem);
  return err;
}

void cascade_launch_append(const CascBlk *cb, int n, int max_n1, const float2 *a_rows, cudaStream_t s) {
  cascade_append_kernel<<<dim3((max_n1 + 255) / 256, n), 256, 0, s>>>(cb, a_rows);
}

void cascade_launch_fir(const CascBlk *cb, int n, int max_n2, int ko, size_t smem, const float *taps2, float2 *out,
                        cudaStream_t s) {
  cascade_fir_cf32_kernel<<<dim3((max_n2 + ko - 1) / ko, n), C_THREADS, smem, s>>>(cb, taps2, out, ko);
}

void cascade_launch_fir_poly(const CascPolyBlk *pb, int n, int max_ctas, size_t smem, const float *taps2,
                             float2 *out, cudaStream_t s) {
  cascade_fir_poly_cf32_kernel<<<dim3(max_ctas, n), C_THREADS, smem, s>>>(pb, taps2, out);
}

}  // namespace xl
