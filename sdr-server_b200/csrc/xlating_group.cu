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
 *   cascade clients  a stage-A history ring each (HostClient::b2.ring), their stage-B taps
 *                    (d_taps2); stage-A rows follow the host-visible rows of the arena
 *   sub-bands        a history ring each (HostClient::b2.ring), rows after the host-visible ones;
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
#include <cmath>
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
  // whose out_off row lies after every host-visible row; stage B is described in b2
  bool casc = false;
  StageB b2;                     // (its fin_off / fin_cap: the final row of the slot's output arena)
  int last_n2 = 0;               // stage-B outputs of the block being submitted
  int cblk = 0;                  // integer stage B: its entry in the per-slot CascBlk table
  // sub-band (xlg_add_subband): an integer client, not visible to the caller, whose row lies after every
  // host-visible row; b2.ring is its history ring
  bool sb = false;
  int sb_id = -1;
  // sub-band member (xlg_add_client_subband[_rational]): not an integer client -- its ClientDev only carries
  // its oscillator; b2.geo is its filter (in sub-band samples), mtaps its rotated reversed taps (2 * T2 floats;
  // branch-major, 2 * L2 * Tb2, when L2 > 1), out_off / out_cap its final row
  bool mem = false;
  std::vector<float> mtaps;
  int sb_cid = -1;               // its sub-band's client index
  long long zb2 = 0;             // sub-band position of its attach point: earlier samples read as zero
  int ph_row = 0;                // its rows of the slot's member oscillator table
  // bank channel (xlg_add_bank_subband): a sub-band (sb) whose row its bank's kernel writes; D and T are its
  // bank's, and it is not an integer client (inactive ClientDev, no oscillator, no tap row)
  int bank = -1;                 // its bank's id
  int chan = 0;                  // its channel k in [-D1, D1)
};

// which kernel serves a bank's channel stage; also its per-block table (Slot::bkblk, bfblk, bzblk)
enum BankKind {
  BANK_DIRECT,  // xlg_add_bank: bank_cf32_kernel
  BANK_FFT,     // xlg_add_bank_fft, and xlg_add_bank_any at a power-of-two K: bank_fft_cf32_kernel
  BANK_CZT,     // xlg_add_bank_any at every other K: bank_czt_cf32_kernel
};

// a channel bank (xlg_add_bank, xlg_add_bank_fft, xlg_add_bank_any): reversed padded taps, twiddles, and the
// walk of an integer client (D1, T1) attached at P
struct BankHost {
  bool active = false;
  BankKind kind = BANK_DIRECT;
  uint32_t D1 = 0;
  size_t T1 = 0;
  int K = 0, tpad = 0;
  std::vector<float> taps;   // h[T1-1-j] at j, zero to tpad
  std::vector<float2> tw;    // e^{-2 pi i j / K}; BANK_CZT: e^{-2 pi i j / M}, then c (K) and Bh (M)
  long long P = 0, hist = 0;
  std::vector<int> cids;     // its materialised channels' client indices (the layout's)
  int taps_off = 0, tw_off = 0, ch_off = 0;
};

// which channel stages serve a spectrum; also its segment of the per-block tables, in this order:
// [plain | extended | wide | chirp-z]
enum SpecKind {
  SPEC_PLAIN,  // hop W, no window, the max, W <= 4096: spectrum_fft_kernel or spectrum_direct_kernel
  SPEC_EXT,    // a hop other than W, a window or the mean, W <= 4096: their _ext twins
  SPEC_WIDE,   // W a power of two above 4096: the two wide passes, plain or extended
  SPEC_CZT,    // every other W above 4096 (xlg_add_spectrum_any): the chirp-z passes, plain or extended
};

// a spectrum (xlg_add_spectrum, xlg_add_client_spectrum, xlg_add_subband_spectrum): its device tables and hold
// rows, and its walk from P in 64-bit stream positions -- the band's, or its source's own, counted from the attach
struct SpectrumHost {
  bool active = false;
  SpecKind kind = SPEC_PLAIN;
  bool power = false;        // XLG_SPECTRUM_POWER
  int W = 0, F = 0, S = 0, R = 0;
  long long P = 0;
  int src = -1;              // its source's client index (a client, a cascade's final row, a sub-band or bank
                             // channel); -1: the band
  long long pos = 0;         // source samples appended to d_ring so far (P = 0)
  float2 *d_ring = nullptr;  // the source's samples at pos & ring_mask
  unsigned ring_mask = 0;
  uint64_t rows_done = 0;    // rows completed by the blocks submitted so far
  int fir = 0;               // frames of the current row completed so far
  int rows_cap = 0, NR = 0;  // rows a block can complete; hold rows (rows_cap + 1: all that a block touches)
  float2 *d_tw = nullptr;
  int *d_map = nullptr;
  unsigned *d_hold = nullptr;
  int out_off = 0;           // its rows in the slot's arena, in complex samples
  // xlg_add_spectrum_ex
  bool mean = false;
  int H = 0;                 // hop (W for today's spectra)
  float *d_win = nullptr;    // W weights, or none
  float *d_fbuf = nullptr;   // mean: fb_frames rows of W, the powers of the frames a block completes
  int fb_frames = 0;         // the most frames a block completes (kept for a mean or a wide spectrum)
  // SPEC_WIDE: d_tw holds the W-point table, then the C-point one
  float2 *d_scratch = nullptr;  // fb_frames rows of W: pass A's output
  // SPEC_CZT, at M = next_pow2(2W - 1): d_tw holds the M-point table, the C-point one, the chirp (W) and Bh (M),
  // d_map the half swap alone (the hold is in natural bin order), d_scratch two sets of fb_frames rows of M
  int M = 0;
  int *d_bin = nullptr;  // the bin of each of the M positions

  // every device buffer it holds (null where it has none)
  std::array<void *, 8> buffers() const { return {d_tw, d_map, d_hold, d_ring, d_win, d_fbuf, d_scratch, d_bin}; }
};

// members of one sub-band that read the same windows: equal (L2, D2, T2, hist2) and, until their windows have
// passed it, the same attach point
struct SbClassHost {
  int sb_cid;
  int L2, Tb;    // Tb: taps per branch (T2 when L2 = 1)
  std::vector<int> members;
  long long zb;  // the largest attach point of its members
};

// A per-slot table the host fills each block and the kernels read: pinned entries and their device copy.
template <typename T>
struct BlkTable {
  T *h = nullptr, *d = nullptr;
  size_t cap = 0;
  // room for n entries (the pipeline is drained); a table grows to max(2n, 16)
  int reserve(size_t n) {
    if (cap >= n) return 0;
    release();
    const size_t want = std::max<size_t>(n * 2, 16);
    CU_OK(cudaMalloc(&d, want * sizeof(T)));
    CU_OK(cudaHostAlloc(&h, want * sizeof(T), cudaHostAllocDefault));
    cap = want;
    return 0;
  }
  cudaError_t upload(size_t n, cudaStream_t s) const {
    return cudaMemcpyAsync(d, h, n * sizeof(T), cudaMemcpyHostToDevice, s);
  }
  void release() {
    if (d) cudaFree(d);
    if (h) cudaFreeHost(h);
    d = h = nullptr;
    cap = 0;
  }
};

// Timed spans of a block: each has a begin and an end event per slot.  Profiling records every span; the
// timeline (XLATING_B200_TIMELINE) records the convert and tile spans too.
enum Span {
  SP_CONV, SP_PHASE, SP_TILE, SP_GEN, SP_LONG, SP_POLY_GEN, SP_POLY_TILE, SP_STAGE_B, SP_SB, SP_BANK, SP_BANK_FFT, SP_SPEC,
  SP_N
};

struct Slot {
  void *d_raw = nullptr, *h_raw = nullptr;
  size_t d_raw_bytes = 0, h_raw_bytes = 0;
  float2 *d_out = nullptr;
  short2 *d_qout = nullptr;
  float2 *d_phases = nullptr;
  float2 *d_partial = nullptr;  // split-K partial sums of the long-filter classes
  short2 *d_qphases = nullptr;
  BlkInfo *d_blk = nullptr;
  float2 *d_endph = nullptr;  // XLG_TRACK_STATE: every client's oscillator after this block (same capacity as d_blk)
  size_t blk_cap = 0;
  cudaEvent_t ev_h2d = nullptr, ev_conv = nullptr, ev_phase = nullptr, ev_fir = nullptr, ev_done = nullptr;
  cudaEvent_t ev_input = nullptr;  // the last reader of this ticket's input: ev_h2d, ev_conv, or none for n = 0
  cudaEvent_t pf[SP_N][2] = {};  // begin / end of each span
  bool pf_on[SP_N] = {};         // the span ran in this block (its events are recorded, or, for the pre-pass, stamped)
  cudaEvent_t tl_ph[2][2] = {{nullptr, nullptr}, {nullptr, nullptr}};  // timeline: pre-pass stamps, by occupancy parity (it runs a block ahead)
  float2 *d_pscratch = nullptr;  // kind 4: unrotated outputs per branch (ClientDev::poly_off)
  BlkInfo *d_vblk = nullptr, *h_vblk = nullptr;  // kind 4: per branch class, this block's window start and count
  uint64_t poly_macs = 0;
  BlkTable<CascBlk> cblk;        // cascade clients: this block's ring positions, windows and counts
                                 // (integer stage B first, then the rational ones)
  BlkTable<CascPolyBlk> pblk;    // rational cascade clients: this block's stage B
  cudaEvent_t ev_casc = nullptr;                 // stage B of this block done (its rings' appends are ordered on it)
  uint64_t casc_macs = 0, d2h_bytes = 0;
  BlkTable<CascBlk> sbcb;        // sub-bands: this block's ring appends
  BlkTable<SbBlk> sbblk;         // member classes: this block's windows and counts
  float2 *d_sbph = nullptr;                      // member oscillator table (HostClient::ph_row)
  uint64_t sb_macs = 0, sb_rows = 0;
  BlkTable<BankBlk> bkblk;       // banks with channels: this block's windows, counts and channel tables
  uint64_t bk_poly = 0, bk_dft = 0;
  BlkTable<BankBlk> bfblk;       // the same for the FFT banks
  BlkTable<BankBlk> bzblk;       // and for the chirp-z banks
  uint64_t bf_poly = 0, bf_flops = 0;  // FFT and chirp-z banks
  BlkTable<SpecBlk> spblk;       // spectra with work in this block
  BlkTable<const float2 *> spring;  // the ring each spblk entry reads
  BlkTable<SpecExt> spext;       // the extended and wide entries' hop, window and frame buffer (the tail of spblk)
  BlkTable<SpecWide> spwide;     // the wide entries' scratch and chunk table (the tail of spext)
  BlkTable<SpecCzt> spczt;       // the chirp-z entries' scratches and tables (after the wide ones in spext)
  BlkTable<CascBlk> spcb;        // spectra of a source: this block's appends to their rings
  uint64_t sp_frames = 0, sp_flops = 0;
  cudaEvent_t ev_spec = nullptr;  // this block's spectra done (the hold rows are updated in block order on it)
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
  MetaArr<int> sp_rows, sp_off, sp_w;  // per spectrum id: rows, their offset in floats, width (0: not attached)
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

// A tiled launch at KT outputs per CTA being assembled: its classes, CTAs and shared memory
struct TileBatch {
  TileLaunch P;
  int KT, ctas = 0;
  size_t smem = 0;
  explicit TileBatch(int kt) : KT(kt) { memset(&P, 0, sizeof(P)); }
  // n_out outputs of class ch, output 0 reading the window at first; returns the MACs its CTAs issue
  uint64_t add(const TileClassHost &ch, long long first, int n_out) {
    TileClass k = ch.k;
    k.first = first;
    k.n_out = n_out;
    k.tiles = (n_out + KT - 1) / KT;
    k.xs_len = (KT - 1) * k.Dp + k.L + (ch.merged ? k.D : 0);
    k.cta_begin = ctas;
    ctas += k.tiles * k.n_groups;
    smem = std::max(smem, (size_t)T_SMEM_FIXED + ((size_t)k.xs_len + 10) * sizeof(float2));
    P.cls[P.n_classes++] = k;
    return (uint64_t)k.tiles * KT * (uint64_t)k.L * (uint64_t)ch.members.size();
  }
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
  // xlg_wait_stream: one event per call since the last submit, each recorded on the caller's stream and waited for
  // by the next submit's first reader; the pool is reused, n_user_waits of it are pending
  std::vector<cudaEvent_t> ev_user;
  size_t n_user_waits = 0;
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
  size_t cap_order = 0;
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
  struct CascRun {
    int ko, c0, c1;                         // the integer CascBlk entries [c0, c1) have outputs per CTA ko
  };
  std::vector<CascRun> casc_runs;           // integer stage B by ko, largest first: one launch each
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
  std::vector<BankHost> banks;              // bank id -> bank (inactive = free)
  std::vector<int> bank_live;               // banks with channels, in BankBlk order
  float *d_bktaps = nullptr;
  float2 *d_bktw = nullptr;
  int2 *d_bkch = nullptr;
  size_t cap_bktaps = 0, cap_bktw = 0, cap_bkch = 0;
  xlg_bank_profile bank_prof;
  xlg_bank_fft_profile bank_fft_prof;
  std::vector<SpectrumHost> spectra;        // spectrum id -> spectrum (inactive = free)
  std::vector<void *> dead_spec;            // tables and holds of removed spectra, freed once the pipeline is drained
  cudaEvent_t ev_last_spec = nullptr;       // ev_spec of the last block with spectrum work
  bool have_last_spec = false;
  xlg_spectrum_profile spec_prof;
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

static int elem_bytes(int fmt) { return fmt == XLG_FMT_CF32 ? 4 : fmt == XLG_FMT_CS16 ? 2 : 1; }

static bool page_locked(const void *p) {
  cudaPointerAttributes attr;
  if (cudaPointerGetAttributes(&attr, p) == cudaSuccess) return attr.type == cudaMemoryTypeHost;
  cudaGetLastError();
  return false;
}

// A slot's staging buffers hold max_input_len elements of 2 bytes (cs16) from xlg_create on.  A host cf32 block
// needs 4: the device buffer grows on the slot's first one, the pinned buffer on its first pageable one, so a group
// that never receives cf32 from the host keeps its footprint.  The slot is idle here (xlg_submit waited for it).
static int grow_raw_cf32(xlg_group *g, Slot &s, bool pageable) {
  const size_t bytes = (size_t)g->max_input_len * 4;
  if (s.d_raw_bytes < bytes) {
    void *d = nullptr;
    if (cudaMalloc(&d, bytes) != cudaSuccess) {
      cudaGetLastError();
      XL_LOG("no device memory for a %zu-byte cf32 staging buffer", bytes);
      return -ENOMEM;
    }
    cudaFree(s.d_raw);
    s.d_raw = d;
    s.d_raw_bytes = bytes;
  }
  if (pageable && s.h_raw_bytes < bytes) {
    void *h = nullptr;
    if (cudaHostAlloc(&h, bytes, cudaHostAllocDefault) != cudaSuccess) {
      cudaGetLastError();
      XL_LOG("no pinned memory for a %zu-byte cf32 staging buffer", bytes);
      return -ENOMEM;
    }
    cudaFreeHost(s.h_raw);
    s.h_raw = h;
    s.h_raw_bytes = bytes;
  }
  return 0;
}

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

// replace a device buffer whose contents need not survive by an uninitialised one of `bytes` (its caller has
// decided that it grows)
template <typename T>
static int dev_grow(T **dptr, size_t bytes) {
  if (*dptr) cudaFree(*dptr);
  *dptr = nullptr;
  CU_OK(cudaMalloc(dptr, bytes));
  return 0;
}

// Move a power-of-two ring of cap samples into a new one of ncap (the pipeline is drained): the `keep` samples
// before stream position pos stay at their positions mod ncap, all others read zero.  A ring that does not exist
// yet (*ring == nullptr) becomes a zeroed one.
template <typename T>
static int ring_rehome(T **ring, size_t cap, size_t ncap, long long pos, size_t keep) {
  T *fresh = nullptr;
  CU_OK(cudaMalloc(&fresh, ncap * sizeof(T)));
  if (*ring == nullptr) {
    CU_OK(cudaMemset(fresh, 0, ncap * sizeof(T)));
  } else {
    std::vector<T> old(cap), h(ncap, T{});
    CU_OK(cudaMemcpy(old.data(), *ring, cap * sizeof(T), cudaMemcpyDeviceToHost));
    for (size_t k = 1; k <= keep; k++) {
      const unsigned long long ab = (unsigned long long)(pos - (long long)k);
      h[ab & (ncap - 1)] = old[ab & (cap - 1)];
    }
    CU_OK(cudaMemcpy(fresh, h.data(), ncap * sizeof(T), cudaMemcpyHostToDevice));
    cudaFree(*ring);
  }
  *ring = fresh;
  return 0;
}

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
  s.cblk.release();
  s.pblk.release();
  s.sbcb.release();
  s.sbblk.release();
  s.bkblk.release();
  s.bfblk.release();
  s.bzblk.release();
  s.spblk.release();
  s.spcb.release();
  s.spring.release();
  s.spext.release();
  s.spwide.release();
  s.spczt.release();
  if (s.d_sbph) cudaFree(s.d_sbph);
  s.d_sbph = nullptr;
  s.d_pscratch = nullptr;
  s.d_vblk = s.h_vblk = nullptr;
  s.d_endph = nullptr;
  s.d_raw = s.h_raw = nullptr;
  s.d_raw_bytes = s.h_raw_bytes = 0;
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

// a span's events are recorded while profiling, the convert and tile spans also for the timeline
static bool span_timed(const xlg_group *g, Span sp) {
  return g->profiling || (g->timeline && (sp == SP_CONV || sp == SP_TILE));
}

static int span_begin(xlg_group *g, Slot &s, Span sp, cudaStream_t st) {
  if (!span_timed(g, sp)) return 0;
  CU_OK(cudaEventRecord(s.pf[sp][0], st));
  s.pf_on[sp] = true;
  return 0;
}

static int span_end(xlg_group *g, Slot &s, Span sp, cudaStream_t st) {
  if (span_timed(g, sp)) CU_OK(cudaEventRecord(s.pf[sp][1], st));
  return 0;
}

static void harvest_locked(xlg_group *g, Slot &s) {
  if (s.harvested) return;
  s.harvested = true;
  if (g->timeline && g->base_recorded && s.pf_on[SP_CONV] && s.pf_on[SP_PHASE] && s.pf_on[SP_TILE]) {
    const int par = (int)((s.ticket.load() / XLG_SLOTS) & 1);
    const cudaEvent_t e[6] = {s.pf[SP_CONV][0], s.pf[SP_CONV][1], s.tl_ph[par][0], s.tl_ph[par][1], s.pf[SP_TILE][0],
                              s.pf[SP_TILE][1]};
    std::array<float, 7> r;
    r[0] = (float)s.ticket.load();
    for (int i = 0; i < 6; i++)
      if (cudaEventElapsedTime(&r[1 + i], g->ev_base, e[i]) != cudaSuccess) r[1 + i] = -1.f;
    g->tl.push_back(r);
    cudaGetLastError();
  }
  if (!g->profiling) return;
  // where each span's time and launch count go, in Span order
  const std::pair<double *, uint64_t *> sink[SP_N] = {
      {&g->prof.convert_ms, &g->prof.convert_launches},
      {&g->prof.phase_ms, &g->prof.phase_launches},
      {&g->prof.fir_tile_ms, &g->prof.fir_tile_launches},
      {&g->prof.fir_generic_ms, &g->prof.fir_generic_launches},
      {&g->prof.fir_long_ms, &g->prof.fir_long_launches},
      {&g->poly_prof.fir_poly_generic_ms, &g->poly_prof.fir_poly_generic_launches},
      {&g->poly_prof.fir_poly_tile_ms, &g->poly_prof.fir_poly_tile_launches},
      {&g->casc_prof.stage_b_ms, &g->casc_prof.stage_b_launches},
      {&g->sb_prof.member_ms, &g->sb_prof.member_launches},
      {&g->bank_prof.bank_ms, &g->bank_prof.bank_launches},
      {&g->bank_fft_prof.fft_ms, &g->bank_fft_prof.fft_launches},
      {&g->spec_prof.spectrum_ms, &g->spec_prof.spectrum_launches}};
  for (int sp = 0; sp < SP_N; sp++) {
    float ms = 0;
    if (s.pf_on[sp] && cudaEventElapsedTime(&ms, s.pf[sp][0], s.pf[sp][1]) == cudaSuccess) {
      *sink[sp].first += ms;
      (*sink[sp].second)++;
    }
  }
  g->poly_prof.poly_macs += s.poly_macs;
  g->casc_prof.stage_b_macs += s.casc_macs;
  g->casc_prof.d2h_bytes += s.d2h_bytes;
  g->sb_prof.member_macs += s.sb_macs;
  g->sb_prof.row_samples += s.sb_rows;
  g->bank_prof.poly_macs += s.bk_poly;
  g->bank_prof.dft_macs += s.bk_dft;
  g->bank_fft_prof.poly_macs += s.bf_poly;
  g->bank_fft_prof.butterfly_flops += s.bf_flops;
  g->spec_prof.frames += s.sp_frames;
  g->spec_prof.channel_flops += s.sp_flops;
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
    // keep the most recent samples at their new ring positions
    auto keep = [g](long long pos) { return std::min<size_t>(g->ring_cap, (size_t)std::max<long long>(pos, 0)); };
    if (ring_rehome(&g->ring, g->ring_cap, cap, g->S, keep(g->S)) ||
        (g->qring && ring_rehome(&g->qring, g->ring_cap, cap, g->qS, keep(g->qS))))
      return -EIO;
    g->ring_cap = cap;
  }
  if (need_q && !g->qring && ring_rehome(&g->qring, 0, g->ring_cap, 0, 0)) return -EIO;
  g->hist_cap = hist_cap;
  return 0;
}

static int ensure_arenas(xlg_group *g, size_t need, bool need_q) {
  const bool dev_out = (g->flags & XLG_OUT_DEVICE) != 0;
  if (need > g->arena_cap) {
    const size_t cap = std::max<size_t>(need + need / 4, 1024);
    for (Slot &s : g->slots)
      if (dev_grow(&s.d_out, cap * sizeof(float2)) ||
          (g->q_alloc && (dev_grow(&s.d_qout, cap * sizeof(short2)) || dev_grow(&s.d_qphases, cap * sizeof(short2)))))
        return -EIO;
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
    for (Slot &s : g->slots)
      if (dev_grow(&s.d_qout, std::max<size_t>(g->arena_cap, 1) * sizeof(short2)) ||
          dev_grow(&s.d_qphases, std::max<size_t>(g->arena_cap, 1) * sizeof(short2)))
        return -EIO;
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
// Give a cascade's or a sub-band's history ring room for cap samples (a power of two; the pipeline is drained):
// a new ring is zero, which its positions before the attach read, and a grown one keeps its last samples at
// their new places.
static int ring_ensure(HistRing &r, size_t cap) {
  if (r.p != nullptr && cap <= r.cap) return 0;
  if (ring_rehome(&r.p, r.cap, cap, r.pos, r.cap)) return -EIO;
  r.cap = cap;
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
    const StageBGeom &b = h.b2.geo;
    back[h.sb_cid] = std::max(back[h.sb_cid], history_reach(b.T2, b.L2));
    // its window has passed its attach point: it reads what every settled member of the class reads
    const bool settled = h.zb2 * (long long)b.L2 <= (long long)b.L2 * g->clients[h.sb_cid].b2.ring.pos - b.hist2;
    if (b.L2 == 1) {
      keyed[std::make_tuple(h.sb_cid, b.D2, b.T2, b.hist2, settled ? LLONG_MIN : h.zb2)].push_back(i);
    } else {
      keyed_rat[std::make_tuple(h.sb_cid, b.L2, b.D2, b.T2, b.hist2, settled ? LLONG_MIN : h.zb2)].push_back(i);
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
    if (ring_ensure(h.b2.ring, next_pow2(back[i] + (size_t)(XLG_SLOTS + 1) * (size_t)h.out_cap))) return -EIO;
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
    ch.L2 = (int)h0.b2.geo.L2;
    ch.Tb = h0.b2.geo.Tb2;
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
          memcpy(&taps[gp.taps_off + ((size_t)r * SB_MG + m) * tpad], h.mtaps.data() + 2 * (size_t)r * ch.Tb,
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
  for (Slot &s : g->slots)
    if (s.sbcb.reserve(n_sb) || s.sbblk.reserve(n_cls) ||
        ((grow_ph || s.d_sbph == nullptr) && g->sbph_cap > 0 && dev_grow(&s.d_sbph, g->sbph_cap * sizeof(float2))))
      return -EIO;
  return 0;
}

// Where channel k of an FFT bank lies in its transformed row (bank_fft_cf32_kernel): the digit reversal of
// k mod K, one base-4 digit per radix-4 stage (the first stage's digit is the most significant), then the radix-2
// stage's bit
static int bank_fft_pos(int k, int K) {
  int pos = 0, L = K;
  k = (k % K + K) % K;
  for (; L >= 4; L >>= 2, k >>= 2) pos += (k & 3) * (L >> 2);
  return L == 2 ? pos + (k & 1) : pos;
}

// Banks (the pipeline is drained, the channels' rows are placed): one arena each for the taps, the twiddles and
// the channel tables of the banks that have channels, and the per-slot tables.
static int rebuild_banks(xlg_group *g) {
  g->bank_live.clear();
  size_t n_fft = 0, n_czt = 0;
  std::vector<float> taps;
  std::vector<float2> tw;
  std::vector<int2> chans;
  for (int b = 0; b < (int)g->banks.size(); b++) {
    BankHost &k = g->banks[b];
    k.cids.clear();
    if (!k.active) continue;
    for (int i = 0; i < (int)g->clients.size(); i++)
      if (g->clients[i].active && g->clients[i].bank == b) k.cids.push_back(i);
    if (k.cids.empty()) continue;
    k.ch_off = (int)chans.size();
    for (int i : k.cids) {
      const int c = g->clients[i].chan, kk = (c + k.K) % k.K;
      const int x = k.kind == BANK_FFT ? bank_fft_pos(c, k.K)
                    : k.kind == BANK_CZT ? bank_fft_pos(kk, bank_czt_m(k.K)) | kk << 16  // (position, k mod K)
                                         : kk;
      chans.push_back(make_int2(x, g->clients[i].out_off));
    }
    n_fft += k.kind == BANK_FFT ? 1 : 0;
    n_czt += k.kind == BANK_CZT ? 1 : 0;
    k.taps_off = (int)taps.size();
    taps.insert(taps.end(), k.taps.begin(), k.taps.end());
    k.tw_off = (int)tw.size();
    tw.insert(tw.end(), k.tw.begin(), k.tw.end());
    g->bank_live.push_back(b);
  }
  if (g->bank_live.empty()) return 0;
  CU_OK(cudaFuncSetAttribute(bank_cf32_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kTileMaxSmem));
  if (n_czt > 0)
    CU_OK(cudaFuncSetAttribute(bank_czt_cf32_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                               (int)bank_czt_smem(BZ_N)));
  if (dev_assign(&g->d_bktaps, &g->cap_bktaps, taps.data(), taps.size() * sizeof(float)) ||
      dev_assign(&g->d_bktw, &g->cap_bktw, tw.data(), tw.size() * sizeof(float2)) ||
      dev_assign(&g->d_bkch, &g->cap_bkch, chans.data(), chans.size() * sizeof(int2)))
    return -EIO;
  for (Slot &s : g->slots)
    if (s.bkblk.reserve(g->bank_live.size() - n_fft - n_czt) || s.bfblk.reserve(n_fft) || s.bzblk.reserve(n_czt))
      return -EIO;
  return 0;
}

// Spectra (the pipeline is drained): their rows after the clients' final rows, inside the D2H copy; a frame reads
// at most W - 1 samples of earlier blocks
static int rebuild_spectra(xlg_group *g, size_t &out_total, size_t &max_hist) {
  for (void *p : g->dead_spec) cudaFree(p);
  g->dead_spec.clear();
  size_t n = 0, n_src = 0, n_ext = 0, n_wide = 0, n_czt = 0;
  for (SpectrumHost &p : g->spectra) {
    if (!p.active) continue;
    n_ext += p.kind != SPEC_PLAIN ? 1 : 0;
    n_wide += p.kind == SPEC_WIDE ? 1 : 0;
    n_czt += p.kind == SPEC_CZT ? 1 : 0;
    p.out_off = (int)out_total;
    out_total += ((size_t)p.rows_cap * p.W + 1) / 2;
    out_total = (out_total + 3) & ~(size_t)3;
    if (p.src < 0)
      max_hist = std::max(max_hist, (size_t)p.W - 1);
    else
      n_src++;  // (its frames read its own ring)
    n++;
  }
  if (n == 0) return 0;
  CU_OK(cudaFuncSetAttribute(spectrum_direct_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             (int)spec_direct_smem(SPEC_MAX_W - 1)));
  CU_OK(cudaFuncSetAttribute(spectrum_direct_ext_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                             (int)spec_direct_smem(SPEC_MAX_W - 1)));
  if (n_czt > 0) {
    CU_OK(cudaFuncSetAttribute(spectrum_czt_b_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                               (int)SPEC_CZT_SMEM));
    CU_OK(cudaFuncSetAttribute(spectrum_czt_d_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                               (int)SPEC_CZT_SMEM));
  }
  for (Slot &s : g->slots)
    if (s.spblk.reserve(n) || s.spring.reserve(n) || s.spcb.reserve(n_src) || s.spext.reserve(n_ext) ||
        s.spwide.reserve(n_wide) || s.spczt.reserve(n_czt))
      return -EIO;
  return 0;
}

// Cascade clients (the pipeline is drained): stage-A rows after every host-visible row (the D2H copy ends before
// them), stage-B taps, and a zeroed history ring for each new client (its positions before the attach read as
// zero)
static int rebuild_cascades(xlg_group *g, size_t &out_total) {
  const int nc = (int)g->clients.size();
  std::vector<float> taps2;
  g->n_casc = g->n_casc_int = 0;
  for (int i = 0; i < nc; i++) {
    HostClient &h = g->clients[i];
    if (!h.active || !h.casc) continue;
    h.out_off = (int)out_total;
    out_total += (size_t)h.out_cap;
    out_total = (out_total + 3) & ~(size_t)3;
    h.b2.taps_off = (int)taps2.size();
    taps2.insert(taps2.end(), h.b2.taps.begin(), h.b2.taps.end());
    // stage B of block b reads stage-A outputs of earlier blocks; the submit of block b + XLG_SLOTS waits
    // for ticket b, so its history + (XLG_SLOTS + 1) * max n1 samples are never overwritten while still needed
    if (ring_ensure(h.b2.ring, next_pow2(history_reach(h.b2.geo.T2, h.b2.geo.L2) +
                                         (size_t)(XLG_SLOTS + 1) * (size_t)h.out_cap)))
      return -EIO;
    g->n_casc++;
    if (h.b2.geo.L2 == 1) g->n_casc_int++;
  }
  // integer entries ordered by ko, one stage-B launch per distinct ko: a client's lanes walk its taps as they
  // would in a group of its own, whatever ko its neighbours have
  std::vector<int> ints;
  for (int i = 0; i < nc; i++)
    if (g->clients[i].active && g->clients[i].casc && g->clients[i].b2.geo.L2 == 1) ints.push_back(i);
  std::stable_sort(ints.begin(), ints.end(),
                   [g](int a, int b) { return g->clients[a].b2.ko > g->clients[b].b2.ko; });
  g->casc_runs.clear();
  for (int e = 0; e < (int)ints.size(); e++) {
    HostClient &h = g->clients[ints[e]];
    h.cblk = e;
    if (g->casc_runs.empty() || g->casc_runs.back().ko != h.b2.ko) g->casc_runs.push_back({h.b2.ko, e, e});
    g->casc_runs.back().c1 = e + 1;
  }
  if (dev_assign(&g->d_taps2, &g->cap_taps2, taps2.data(), taps2.size() * sizeof(float))) return -EIO;
  for (float2 *p : g->dead_rings) cudaFree(p);
  g->dead_rings.clear();
  for (Slot &s : g->slots)
    if (s.cblk.reserve((size_t)g->n_casc) || s.pblk.reserve((size_t)(g->n_casc - g->n_casc_int))) return -EIO;
  return 0;
}

// How the tiled kernels read a class of (D, T): natural or skewed input layout at pitch Dp, L flat taps per slot,
// and whether it is a split-K long-filter class and can be tiled at all
struct TileMode {
  bool natural, as_long, eligible;
  int Dp, L;
};

// A tiled class over `slots` (T_CG per group, -1 = padding) of clients with T taps at decimation D: its kernel
// entry (the caller adds what is particular to its family) and its taps, appended to tile_taps as
// [group][flat tap f][T_CG slots] with tap j = q * D + r at f = q * Dp + r.  taps(id) is a member's T reversed
// taps (re, im interleaved).
template <typename Taps>
static TileClassHost tile_class(const std::vector<int> &slots, const std::vector<int> &real, uint32_t D, size_t T,
                                const TileMode &m, int members_off, std::vector<float2> &tile_taps, Taps taps) {
  TileClassHost ch;
  memset(&ch.k, 0, sizeof(ch.k));
  ch.T = T;
  ch.members = slots;
  ch.real = real;
  ch.k.D = (int)D;
  ch.k.Dp = m.Dp;
  ch.k.L = m.L;
  ch.k.n_groups = (int)(slots.size() / T_CG);
  ch.k.n_members = (int)real.size();
  ch.k.natural = m.natural ? 1 : 0;
  ch.k.members_off = members_off;
  ch.k.taps_off = (long long)tile_taps.size();
  const size_t base = tile_taps.size();
  tile_taps.resize(base + slots.size() * (size_t)m.L, make_float2(0.f, 0.f));
  // one 256-byte line (all 32 slots of a tap) at a time -- slot-major packing touched a new cache line for every
  // tap of every client (1.5 ms per re-layout at 1000 clients)
  for (size_t gi = 0; gi < slots.size() / T_CG; gi++) {
    float2 *dst = tile_taps.data() + base + gi * (size_t)m.L * T_CG;
    const float *src[T_CG];
    for (int sl = 0; sl < T_CG; sl++) {
      const int id = slots[gi * T_CG + sl];
      src[sl] = id < 0 ? nullptr : taps(id);
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
  return ch;
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
      // n1 at most its sub-band's row
      h.out_cap = stage_b_rows((uint64_t)g->max_input_len / 2 / g->clients[h.sb_cid].D + 2, h.b2.geo.L2, h.b2.geo.D2);
      h.out_off = (int)out_total;
      out_total += (size_t)h.out_cap;
      out_total = (out_total + 3) & ~(size_t)3;
      continue;
    }
    h.out_cap = (int)((uint64_t)g->max_input_len / 2 * h.L / h.D + 2);
    if (h.casc) {
      h.b2.fin_cap = stage_b_rows((uint64_t)h.out_cap, h.b2.geo.L2, h.b2.geo.D2);
      h.b2.fin_off = (int)out_total;
      out_total += (size_t)h.b2.fin_cap;
    } else if (!h.sb) {
      h.out_off = (int)out_total;
      out_total += (size_t)h.out_cap;
    }
    out_total = (out_total + 3) & ~(size_t)3;  // keep rows 32-byte aligned
    h.taps_off = (int)taps_total;
    taps_total += h.rev.size() / 2;
    max_hist = std::max(max_hist, history_reach(h.T, h.L));
  }
  for (const BankHost &k : g->banks)  // a bank walks (and its channels read history) without channels too
    if (k.active) max_hist = std::max(max_hist, k.T1 - 1);
  if (rebuild_spectra(g, out_total, max_hist)) return -EIO;
  if (rebuild_cascades(g, out_total)) return -EIO;
  if (rebuild_subbands(g, out_total)) return -EIO;
  if (rebuild_banks(g)) return -EIO;
  if (ensure_ring(g, max_hist, g->qring != nullptr)) return -EIO;
  if (ensure_arenas(g, out_total, g->q_alloc)) return -EIO;

  std::vector<float2> &taps = g->h_taps;
  std::vector<short2> &qtaps = g->h_qtaps;
  taps.resize(std::max<size_t>(taps_total, 1));
  qtaps.resize(std::max<size_t>(taps_total, 1));
  for (int i = 0; i < nc; i++) {
    const HostClient &h = g->clients[i];
    if (!h.active || h.bank >= 0) continue;  // (a bank channel has no taps of its own)
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
  auto mode_of = [&](uint32_t D, size_t T) {
    TileMode m;
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
    if (h.bank >= 0) {
      // a bank channel: bank_cf32_kernel writes it (8: bank_fft_cf32_kernel, 9: bank_czt_cf32_kernel)
      h.kind = g->banks[h.bank].kind == BANK_CZT ? 9 : g->banks[h.bank].kind == BANK_FFT ? 8 : 7;
      continue;
    }
    h.kind = h.L > 1 ? 3 : 0;
    h.tile_ineligible = false;
    h.pending_settle = false;
    if (h.L > 1) {
      // rational: a tiled class per (L, M, T, alignment) where every branch is an integer class the tiled
      // kernel takes (gcd(L, M) = 1: each block uses every branch, outputs L apart)
      const size_t Tb = (h.T + h.L - 1) / h.L;
      const TileMode m = mode_of(h.D, Tb);
      if ((g->flags & XLG_FORCE_GENERIC) || !g->poly_tile || std::gcd(h.L, h.D) != 1 || !m.eligible || m.as_long)
        continue;
      if (!poly_settled(g, h)) {
        h.pending_settle = true;
        continue;
      }
      pbuckets[std::make_tuple(h.L, h.D, h.T, h.hist)].push_back(i);
      continue;
    }
    if (g->flags & XLG_FORCE_GENERIC) continue;
    const TileMode m = mode_of(h.D, h.T);
    if (!m.eligible) {
      h.tile_ineligible = true;
      continue;
    }
    if (!poly_settled(g, h)) {
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
    const TileMode m = mode_of(D, T);
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
    const int members_off = (int)members.size();
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
    TileClassHost ch = tile_class(slots, real, D, T, m, members_off, tile_taps,
                                  [g](int id) { return g->clients[id].rev.data(); });
    ch.merged = merged;
    ch.k.nseg = m.as_long ? (ch.k.L + W_JS - 1) / W_JS : 0;
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
    const TileMode m = mode_of(M, Tb);
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
      const int members_off = (int)members.size();
      const int v = (int)g->poly_classes.size();  // the tiled kernel reads this class's BlkInfo at d_vblk[v]
      for (int id : slots) {
        member_cid.push_back(id < 0 ? -1 : v);
        members.push_back(id < 0 ? -1 : g->clients[id].poly_off + (int)r * g->clients[id].poly_rowcap);
        member_incr.push_back(make_float2(1.f, 0.f));
      }
      // branch r of every member (xl_poly_pack)
      TileClassHost ch = tile_class(slots, real, M, Tb, m, members_off, tile_taps,
                                    [g, r, Tb](int id) { return g->clients[id].rev.data() + 2 * (size_t)r * Tb; });
      ch.branch = (int)r;
      ch.interp = L;
      ch.minv = minv;
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
      if (g->clients[i].active && !g->clients[i].mem && g->clients[i].bank < 0 &&
          (g->clients[i].kind == 0 || g->clients[i].kind >= 3))
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
    g->n_order = (int)order.size();
    if (dev_assign(&g->d_order, &g->cap_order, order.data(), order.size() * sizeof(int))) return -EIO;
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
        for (Slot &sl : g->slots)
          if (dev_grow(&sl.d_partial, g->partial_cap * sizeof(float2))) return -EIO;
      }
    }
    if (pscratch > g->pscratch_cap) {
      g->pscratch_cap = pscratch + pscratch / 4 + 1024;
      for (Slot &sl : g->slots)
        if (dev_grow(&sl.d_pscratch, g->pscratch_cap * sizeof(float2))) return -EIO;
    }
    // the tiled kernel reads the phase of output j at [32 * (j / 2) + client slot]: a table of ones that long
    const size_t ones = ((size_t)max_rowcap / 2 + 2) * 32;
    if (!g->poly_classes.empty() && ones > g->ones_cap) {
      g->ones_cap = ones;
      std::vector<float2> one(ones, make_float2(1.f, 0.f));
      if (dev_grow(&g->d_ones, ones * sizeof(float2))) return -EIO;
      CU_OK(cudaMemcpy(g->d_ones, one.data(), ones * sizeof(float2), cudaMemcpyHostToDevice));
    }
    if (table > g->phase_cap) {
      g->phase_cap = table + table / 4 + 1024;
      for (Slot &sl : g->slots)
        if (dev_grow(&sl.d_phases, g->phase_cap * sizeof(float2))) return -EIO;
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
    d.active = h.mem || h.bank >= 0 ? 0 : 1;  // a member's entry only carries its oscillator (subband_phase_kernel)
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
    g->d_clients_cap = std::max<size_t>((size_t)nc * 2, 64);
    if (dev_grow(&g->d_clients, g->d_clients_cap * sizeof(ClientDev))) return -EIO;
    CU_OK(cudaMemset(g->d_clients, 0, g->d_clients_cap * sizeof(ClientDev)));
    if (dev_grow(&g->d_clients_backup, g->d_clients_cap * sizeof(SpecSave))) return -EIO;
  }
  if (nc > 0) CU_OK(cudaMemcpy(g->d_clients, tab.data(), (size_t)nc * sizeof(ClientDev), cudaMemcpyHostToDevice));

  for (Slot &s : g->slots) {
    if (s.blk_cap < (size_t)std::max(nc, 1)) {
      s.blk_cap = std::max<size_t>((size_t)nc * 2, 64);
      // (d_endph exists in XLG_TRACK_STATE groups only)
      if (dev_grow(&s.d_blk, s.blk_cap * sizeof(BlkInfo)) ||
          ((g->flags & XLG_TRACK_STATE) && dev_grow(&s.d_endph, s.blk_cap * sizeof(float2))))
        return -EIO;
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
      if (!h.active || h.mem || h.bank >= 0) continue;  // (no oscillator chain, no FIR of their own)
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
  memset(&g->bank_prof, 0, sizeof(g->bank_prof));
  memset(&g->bank_fft_prof, 0, sizeof(g->bank_fft_prof));
  memset(&g->spec_prof, 0, sizeof(g->spec_prof));
  g->device = device;
  g->fs = sampling_freq;
  g->max_input_len = max_input_len;
  g->flags = flags;
  g->ring_out = std::vector<HostOut>(host_ring);
  for (HostOut &h : g->ring_out) {
    h.n_out.retired = &g->retired_meta_i;
    h.out_off.retired = &g->retired_meta_i;
    h.hist_after.retired = &g->retired_meta_ll;
    h.sp_rows.retired = h.sp_off.retired = h.sp_w.retired = &g->retired_meta_i;
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
    s.d_raw_bytes = s.h_raw_bytes = raw_bytes;
    cudaEvent_t *evs[] = {&s.ev_h2d, &s.ev_conv, &s.ev_phase, &s.ev_fir, &s.ev_done};
    for (cudaEvent_t *ev : evs)
      if (cudaEventCreateWithFlags(ev, cudaEventDisableTiming) != cudaSuccess) return fail(-EIO);
    for (auto &span : s.pf)
      for (cudaEvent_t &ev : span)
        if (cudaEventCreate(&ev) != cudaSuccess) return fail(-EIO);
    if (cudaEventCreateWithFlags(&s.ev_casc, cudaEventDisableTiming) != cudaSuccess) return fail(-EIO);
    if (cudaEventCreateWithFlags(&s.ev_spec, cudaEventDisableTiming) != cudaSuccess) return fail(-EIO);
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
      cascade_stage_b_init() != cudaSuccess) {
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
    for (auto &span : s.pf)
      for (cudaEvent_t ev : span)
        if (ev) cudaEventDestroy(ev);
    if (s.ev_casc) cudaEventDestroy(s.ev_casc);
    if (s.ev_spec) cudaEventDestroy(s.ev_spec);
  }
  for (HostOut &h : g->ring_out) {
    if (h.h_out) cudaFreeHost(h.h_out);
    if (h.h_qout) cudaFreeHost(h.h_qout);
    if (h.h_endph) cudaFreeHost(h.h_endph);
    h.n_out.release();
    h.out_off.release();
    h.hist_after.release();
    h.sp_rows.release();
    h.sp_off.release();
    h.sp_w.release();
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
  if (g->d_bktaps) cudaFree(g->d_bktaps);
  if (g->d_bktw) cudaFree(g->d_bktw);
  if (g->d_bkch) cudaFree(g->d_bkch);
  for (HostClient &h : g->clients)
    if (h.b2.ring.p) cudaFree(h.b2.ring.p);
  for (float2 *p : g->dead_rings) cudaFree(p);
  for (const SpectrumHost &p : g->spectra)
    for (void *d : p.buffers())
      if (d) cudaFree(d);
  for (void *p : g->dead_spec) cudaFree(p);
  for (cudaEvent_t e : g->ev_user) cudaEventDestroy(e);
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
  const char *why = rational_refusal(g->fs, g->max_input_len, interp, decim);
  if (why != nullptr) {
    XL_LOG("rational client %u/%u at %u Hz, blocks of %u: %s", interp, decim, g->fs, g->max_input_len, why);
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
  if (taps1_len == 0 || taps2_len == 0 || taps1 == nullptr || taps2 == nullptr) {
    XL_LOG("cascade client: tap counts (%zu, %zu) must both be at least 1", taps1_len, taps2_len);
    return -EINVAL;
  }
  const char *why = cascade_refusal(g->max_input_len, decim1, interp2, decim2, taps2_len);
  if (why != nullptr) {
    XL_LOG("cascade client %u x %u/%u with %zu + %zu taps, blocks of %u: %s", decim1, interp2, decim2, taps1_len,
           taps2_len, g->max_input_len, why);
    return -EINVAL;
  }
  if (g->flags & XLG_TRACK_STATE) {
    XL_LOG("cascade client: an XLG_TRACK_STATE group cannot carry the state of two stages");
    return -ENOTSUP;
  }
  StageB b2;
  int rc = stage_b_init(&b2, taps2, taps2_len, interp2, decim2, g->fs / decim1);
  if (rc) return rc;
  int id = -1;
  rc = attach_client(g, 1, decim1, g->fs, taps1, taps1_len, center_freq, nullptr, &id);
  if (rc) return rc;
  HostClient &h = g->clients[id];
  h.casc = true;
  h.b2 = std::move(b2);
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

// the id of a spectrum whose source is client index cid, -1 if none reads it
static int spectrum_reading(const xlg_group *g, int cid) {
  for (int id = 0; id < (int)g->spectra.size(); id++)
    if (g->spectra[id].active && g->spectra[id].src == cid) return id;
  return -1;
}

extern "C" int xlg_remove_client(xlg_group *g, int client_id) {
  if (g == nullptr || client_id < 0 || client_id >= (int)g->clients.size() || !g->clients[client_id].active ||
      g->clients[client_id].sb)
    return -EINVAL;
  if (spectrum_reading(g, client_id) >= 0) {
    XL_LOG("client %d is the source of spectrum %d; remove the spectrum first", client_id,
           spectrum_reading(g, client_id));
    return -EBUSY;
  }
  g->clients[client_id].active = false;
  if (g->clients[client_id].b2.ring.p) g->dead_rings.push_back(g->clients[client_id].b2.ring.p);  // in-flight tickets read it
  g->clients[client_id].b2 = StageB();
  g->clients[client_id].mtaps.clear();
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
  if (history) *history = (size_t)(g->clients[client_id].mem ? g->clients[client_id].b2.geo.hist2 : g->clients[client_id].hist);
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
  if (stage_b_history) *stage_b_history = (size_t)h.b2.geo.hist2;
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
  if (spectrum_reading(g, cid) >= 0) {
    XL_LOG("sub-band %d is the source of spectrum %d; remove the spectrum first", subband_id, spectrum_reading(g, cid));
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
  h.b2.geo = stage_b_geom(interp2, decim2, taps2_len);
  if (interp2 == 1) {
    h.mtaps.assign(k.rev_cf32, k.rev_cf32 + 2 * taps2_len);
  } else {
    h.mtaps.resize(2 * (size_t)interp2 * Tb2);  // branch-major P[r][t] = rev[r + t * L2], zero-padded
    xl_poly_pack(k.rev_cf32, taps2_len, interp2, h.mtaps.data());
  }
  h.incr_re = k.incr_re;
  h.incr_im = k.incr_im;
  h.zb2 = g->clients[sb].b2.ring.pos;
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
  if (member_history) *member_history = (size_t)h.b2.geo.hist2;
  return 0;
}

// e^{-2 pi i j / K}, j < K, of the banks and spectra: (-i)^q e^{-i t}, 4j = qK + rem, t = 2 pi rem / 4K in
// [0, pi/2), in double, rounded once: quarter turns are exact (W = 1, -i, -1, i where 4j % K == 0)
static std::vector<float2> twiddle_table(int K) {
  std::vector<float2> tw((size_t)K);
  for (int j = 0; j < K; j++) {
    const int q = (int)(4LL * j / K), rem = (int)(4LL * j - (long long)q * K);
    const double t = 2.0 * 3.14159265358979323846 * (double)rem / (4.0 * (double)K);
    const float c = (float)cos(t), sn = (float)sin(t);
    tw[j] = q == 0 ? make_float2(c, -sn) : q == 1 ? make_float2(-sn, -c) : q == 2 ? make_float2(-c, sn) : make_float2(sn, c);
  }
  return tw;
}

static void czt_tables(int W, std::vector<float2> &chirp, std::vector<float2> &kern, std::vector<int> &bin);

// A bank whose channel stage is `kind`'s kernel, after the checks of that kernel
static int add_bank(xlg_group *g, uint32_t decim1, const float *taps1, size_t taps1_len, BankKind kind,
                    int *bank_id) {
  const bool fft = kind != BANK_DIRECT;
  const char *what = kind == BANK_CZT ? "chirp-z bank" : fft ? "FFT bank" : "bank";
  if (g == nullptr || bank_id == nullptr) return -EINVAL;
  if (decim1 == 0 || taps1_len == 0 || taps1 == nullptr) {
    XL_LOG("%s: decimation %u and tap count %zu must both be at least 1", what, decim1, taps1_len);
    return -EINVAL;
  }
  if (decim1 > (uint32_t)(INT32_MAX / 2) || g->fs % (2 * decim1) != 0) {
    XL_LOG("%s: 2 x decimation %u does not divide the band rate %u (channel centres are in Hz at fs / %u)", what,
           decim1, g->fs, 2 * decim1);
    return -EINVAL;
  }
  if (fft) {
    const uint32_t K = 2 * decim1;
    if (kind == BANK_FFT && ((K & (K - 1)) != 0 || K > 4096)) {
      XL_LOG("FFT bank: K = 2 x decimation %u = %u is not a power of two up to 4096", decim1, K);
      return -EINVAL;
    }
    if (K > 4096) {
      XL_LOG("chirp-z bank: K = 2 x decimation %u = %u exceeds 4096", decim1, K);
      return -EINVAL;
    }
    if (taps1_len > (size_t)bank_fft_max_taps((int)K)) {
      XL_LOG("%s: %zu taps at decimation %u exceed the kernel's bound of %lld", what, taps1_len, decim1,
             bank_fft_max_taps((int)K));
      return -EINVAL;
    }
  } else if (taps1_len > (size_t)INT32_MAX / 8 || bank_smem((int)decim1, (int)taps1_len) > (size_t)kTileMaxSmem) {
    XL_LOG("bank: %zu taps at decimation %u exceed the bank kernel's shared memory", taps1_len, decim1);
    return -EINVAL;
  }
  if (g->flags & XLG_TRACK_STATE) {
    XL_LOG("%s: an XLG_TRACK_STATE group cannot carry the state of two stages", what);
    return -ENOTSUP;
  }
  BankHost k;
  k.active = true;
  k.kind = kind;
  k.D1 = decim1;
  k.T1 = taps1_len;
  k.K = 2 * (int)decim1;
  k.tpad = bank_tpad(k.K, (int)taps1_len);
  k.taps.assign((size_t)k.tpad, 0.f);
  for (size_t j = 0; j < taps1_len; j++) k.taps[j] = taps1[taps1_len - 1 - j];
  if (kind == BANK_CZT) {  // the M-point table, then c and Bh
    std::vector<float2> chirp, kern;
    std::vector<int> bin;
    czt_tables(k.K, chirp, kern, bin);
    k.tw = twiddle_table(bank_czt_m(k.K));
    k.tw.insert(k.tw.end(), chirp.begin(), chirp.end());
    k.tw.insert(k.tw.end(), kern.begin(), kern.end());
  } else {
    k.tw = twiddle_table(k.K);
  }
  k.P = g->S;
  k.hist = (long long)taps1_len - 1;  // a fresh filter's history: T1 - 1 samples, zero before P
  int id = 0;
  while (id < (int)g->banks.size() && g->banks[id].active) id++;
  if (id == (int)g->banks.size()) g->banks.emplace_back();
  g->banks[id] = std::move(k);
  g->dirty = true;  // the input ring's history bound
  *bank_id = id;
  return 0;
}

extern "C" int xlg_add_bank(xlg_group *g, uint32_t decim1, const float *taps1, size_t taps1_len, int *bank_id) {
  return add_bank(g, decim1, taps1, taps1_len, BANK_DIRECT, bank_id);
}

extern "C" int xlg_add_bank_fft(xlg_group *g, uint32_t decim1, const float *taps1, size_t taps1_len, int *bank_id) {
  return add_bank(g, decim1, taps1, taps1_len, BANK_FFT, bank_id);
}

extern "C" int xlg_add_bank_any(xlg_group *g, uint32_t decim1, const float *taps1, size_t taps1_len, int *bank_id) {
  const uint32_t K = 2 * decim1;
  const bool fft = decim1 <= 2048 && (K & (K - 1)) == 0;  // a K that xlg_add_bank_fft takes
  return add_bank(g, decim1, taps1, taps1_len, fft ? BANK_FFT : BANK_CZT, bank_id);
}

extern "C" uint64_t xlg_bank_fft_flops(uint32_t K) {
  uint64_t n = 0, L = K;
  for (; L >= 4; L >>= 2) n += (uint64_t)K / 4 * 28;  // radix 4: 16 adds, 3 products of 4 instructions
  return L == 2 ? n + (uint64_t)K / 2 * 4 : n;        // radix 2: 4 adds
}

static BankHost *bank_of(xlg_group *g, int bank_id) {
  if (bank_id < 0 || bank_id >= (int)g->banks.size() || !g->banks[bank_id].active) return nullptr;
  return &g->banks[bank_id];
}

extern "C" int xlg_remove_bank(xlg_group *g, int bank_id) {
  if (g == nullptr) return -EINVAL;
  BankHost *k = bank_of(g, bank_id);
  if (k == nullptr) {
    XL_LOG("bank %d does not exist", bank_id);
    return -EINVAL;
  }
  int chans = 0;
  for (const HostClient &h : g->clients) chans += h.active && h.bank == bank_id ? 1 : 0;
  if (chans > 0) {
    XL_LOG("bank %d still has %d channels; remove them first", bank_id, chans);
    return -EBUSY;
  }
  *k = BankHost();
  g->dirty = true;
  return 0;
}

extern "C" int xlg_add_bank_subband(xlg_group *g, int bank_id, int32_t channel, int *subband_id) {
  if (g == nullptr || subband_id == nullptr) return -EINVAL;
  const BankHost *k = bank_of(g, bank_id);
  if (k == nullptr) {
    XL_LOG("bank channel: bank %d does not exist", bank_id);
    return -EINVAL;
  }
  if (channel < -(int32_t)k->D1 || channel >= (int32_t)k->D1) {
    XL_LOG("bank channel: channel %d is outside [-%u, %u)", channel, k->D1, k->D1);
    return -EINVAL;
  }
  for (const HostClient &h : g->clients)
    if (h.active && h.bank == bank_id && h.chan == channel) {
      XL_LOG("bank channel: channel %d of bank %d already exists (sub-band %d)", channel, bank_id, h.sb_id);
      return -EEXIST;
    }
  int cid = -1;
  for (size_t i = 0; i < g->clients.size(); i++)
    if (!g->clients[i].active) {
      cid = (int)i;
      break;
    }
  if (cid < 0) {
    g->clients.emplace_back();
    cid = (int)g->clients.size() - 1;
  }
  HostClient &h = g->clients[cid];
  h = HostClient();
  h.active = true;
  h.D = k->D1;
  h.T = k->T1;
  h.hist = k->hist;
  h.zero_before = k->P;
  h.is_new = true;
  h.bank = bank_id;
  h.chan = channel;
  int id = 0;
  while (id < (int)g->subbands.size() && g->subbands[id] >= 0) id++;
  if (id == (int)g->subbands.size()) g->subbands.push_back(-1);
  g->subbands[id] = cid;
  h.sb = true;
  h.sb_id = id;
  g->dirty = true;
  *subband_id = id;
  return 0;
}

// Samples a block adds at most to the output stream of client index cid (the row capacity rebuild_layout gives
// it): its row, a cascade's final row, a sub-band's or bank channel's n1
static int source_cap(const xlg_group *g, const HostClient &h) {
  const uint64_t half = (uint64_t)g->max_input_len / 2;
  if (h.mem) return stage_b_rows(half / g->clients[h.sb_cid].D + 2, h.b2.geo.L2, h.b2.geo.D2);
  const int cap = (int)(half * h.L / h.D + 2);
  return h.casc ? stage_b_rows((uint64_t)cap, h.b2.geo.L2, h.b2.geo.D2) : cap;
}

// The chirp-z stage's M and tables for width W (xlating_kernels.cuh, "Chirp-z spectra"): c[n] = e^{-i pi (n^2
// mod 2W) / W}, n < W, and Bh, the M-point DFT of b[m] = conj(c[|m|]) for |m| < W wrapped mod M, times 1/M, in
// the position order of the kernels' transform (kern[p] = Bh[bin[p]]); both computed in double and rounded once.
// The DFT is an iterative radix-2 FFT with each twiddle from cos and sin of its own angle.
static int czt_m(int W) { return (int)next_pow2(2 * (size_t)W - 1); }

static void czt_tables(int W, std::vector<float2> &chirp, std::vector<float2> &kern, std::vector<int> &bin) {
  const int M = czt_m(W);
  const double pi = 3.14159265358979323846;
  std::vector<double> cr((size_t)W), ci((size_t)W);
  chirp.resize((size_t)W);
  for (int n = 0; n < W; n++) {
    const uint64_t r = (uint64_t)n * (uint64_t)n % (2 * (uint64_t)W);  // n^2 passes 2^31 at n = 46341
    const double t = pi * (double)r / (double)W;
    cr[n] = cos(t);
    ci[n] = -sin(t);
    chirp[n] = make_float2((float)cr[n], (float)ci[n]);
  }
  std::vector<double> re((size_t)M, 0.0), im((size_t)M, 0.0);
  for (int m = 0; m < W; m++) {
    re[m] = cr[m];
    im[m] = -ci[m];
    if (m > 0) {
      re[M - m] = cr[m];
      im[M - m] = -ci[m];
    }
  }
  for (int i = 1, j = 0; i < M; i++) {  // bit reversal, then decimation in time
    int bit = M >> 1;
    for (; j & bit; bit >>= 1) j ^= bit;
    j ^= bit;
    if (i < j) {
      std::swap(re[i], re[j]);
      std::swap(im[i], im[j]);
    }
  }
  for (int len = 2; len <= M; len <<= 1)
    for (int k = 0; k < len / 2; k++) {
      const double t = -2.0 * pi * (double)k / (double)len, wr = cos(t), wi = sin(t);
      for (int i = k; i < M; i += len) {
        const int h = i + len / 2;
        const double xr = re[h] * wr - im[h] * wi, xi = re[h] * wi + im[h] * wr;
        re[h] = re[i] - xr;
        im[h] = im[i] - xi;
        re[i] += xr;
        im[i] += xi;
      }
    }
  kern.resize((size_t)M);
  bin.resize((size_t)M);
  for (int k = 0; k < M; k++) {
    const int p = bank_fft_pos(k, M);
    bin[p] = k;
    kern[p] = make_float2((float)(re[k] / M), (float)(im[k] / M));
  }
}

// czt_tables(W) into the caller's buffers (xlg_spectrum_any_tables, xlg_bank_any_tables)
static int czt_tables_query(int W, float *chirp, float *kernel, uint32_t *m) {
  if (m) *m = (uint32_t)czt_m(W);
  if (chirp == nullptr && kernel == nullptr) return 0;
  std::vector<float2> c, k;
  std::vector<int> bin;
  czt_tables(W, c, k, bin);
  if (chirp) memcpy(chirp, c.data(), c.size() * sizeof(float2));
  if (kernel) memcpy(kernel, k.data(), k.size() * sizeof(float2));
  return 0;
}

extern "C" int xlg_spectrum_any_tables(uint32_t width, float *chirp, float *kernel, uint32_t *m) {
  if (width <= SPEC_MAX_W || width > SPEC_WIDE_MAX_W || spec_wide((int)width)) return -EINVAL;
  return czt_tables_query((int)width, chirp, kernel, m);
}

extern "C" int xlg_bank_any_tables(uint32_t K, float *chirp, float *kernel, uint32_t *m) {
  if (K < 2 || K > 4096 || K % 2 != 0 || (K & (K - 1)) == 0) return -EINVAL;
  return czt_tables_query((int)K, chirp, kernel, m);
}

// A spectrum of the band (src = -1) or of client index src's output stream, after the checks of its source.
// hop 0 means width; today's spectra are hop = width, reduce = XLG_SPECTRUM_MAX and no window.  any: every width
// up to 65536, those above 4096 that are not powers of two through the chirp-z stage.
static int add_spectrum(xlg_group *g, int src, uint32_t width, uint32_t frames_per_row, uint32_t skip_per_row,
                        uint32_t flags, uint32_t hop, uint32_t reduce, const float *window, bool any,
                        int *spectrum_id) {
  if (any && (width == 0 || width > SPEC_WIDE_MAX_W || frames_per_row == 0)) {
    XL_LOG("spectrum: width %u must be in [1, %d], and frames per row %u at least 1", width, SPEC_WIDE_MAX_W,
           frames_per_row);
    return -EINVAL;
  }
  if (!any && (width == 0 || (width > SPEC_MAX_W && !spec_wide((int)std::min<uint32_t>(width, 1u << 30))) ||
               frames_per_row == 0)) {
    XL_LOG("spectrum: width %u must be in [1, %d] or a power of two up to %d, and frames per row %u at least 1",
           width, SPEC_MAX_W, SPEC_WIDE_MAX_W, frames_per_row);
    return -EINVAL;
  }
  if (hop == 0) hop = width;
  if (8ull * hop < width) {
    XL_LOG("spectrum: a hop of %u is below width / 8 (%u)", hop, width);
    return -EINVAL;
  }
  // (below 2^64: (2^32 - 1)^2 + 2^32 + 4096)
  const uint64_t R = (uint64_t)(frames_per_row - 1) * hop + width + skip_per_row;
  if (R >= (1ull << 31)) {
    XL_LOG("spectrum: a row period of %llu samples is not below 2^31", (unsigned long long)R);
    return -EINVAL;
  }
  if (flags & ~XLG_SPECTRUM_POWER) {
    XL_LOG("spectrum: unknown flags 0x%x", flags & ~XLG_SPECTRUM_POWER);
    return -EINVAL;
  }
  if (reduce != XLG_SPECTRUM_MAX && reduce != XLG_SPECTRUM_MEAN) {
    XL_LOG("spectrum: unknown reduce mode %u", reduce);
    return -EINVAL;
  }
  if (window != nullptr)
    for (uint32_t n = 0; n < width; n++)
      if (!std::isfinite(window[n])) {
        XL_LOG("spectrum: window weight %u is not finite", n);
        return -EINVAL;
      }
  if (g->flags & XLG_TRACK_STATE) {
    XL_LOG("spectrum: an XLG_TRACK_STATE group does not serve spectra");
    return -ENOTSUP;
  }
  CU_OK(cudaSetDevice(g->device));
  SpectrumHost p;
  p.active = true;
  p.power = (flags & XLG_SPECTRUM_POWER) != 0;
  p.W = (int)width;
  p.F = (int)frames_per_row;
  p.S = (int)skip_per_row;
  p.R = (int)R;
  p.H = (int)hop;
  p.mean = reduce == XLG_SPECTRUM_MEAN;
  p.kind = spec_wide(p.W) ? SPEC_WIDE : p.W > SPEC_MAX_W ? SPEC_CZT  // (SPEC_CZT only through xlg_add_spectrum_any)
           : p.H != p.W || window != nullptr || p.mean ? SPEC_EXT : SPEC_PLAIN;
  const bool wide = p.kind == SPEC_WIDE, czt = p.kind == SPEC_CZT;
  p.M = czt ? czt_m(p.W) : 0;
  p.src = src;
  // a source's positions count from here: P = 0 in its own stream
  const uint64_t cap = src < 0 ? (uint64_t)g->max_input_len / 2 : (uint64_t)source_cap(g, g->clients[src]);
  p.P = src < 0 ? g->S : 0;
  p.rows_cap = (int)(cap / R + 1);
  p.NR = p.rows_cap + 1;
  // the frames a block of at most cap samples completes: their last samples are distinct positions of the block,
  // one frame's at least min(H, W + S) after the previous one's (H within a row, W + S from a row's last frame to
  // the next row's first)
  if (p.mean || wide || czt) p.fb_frames = (int)((cap - 1) / std::min<uint64_t>(hop, (uint64_t)width + skip_per_row) + 1);
  // a source's ring holds every sample of the frames a block completes: the block's own and W - 1 before them
  const size_t ring_cap = src < 0 ? 0 : next_pow2((size_t)width - 1 + (size_t)cap);
  p.ring_mask = (unsigned)(ring_cap - 1);
  const int W = p.W, half = W / 2;
  std::vector<int> map((size_t)W);
  for (int j = 0; j < W; j++) {
    // spectrogram.c:156-163: the halves swapped, an odd width's last bin in place
    const int bin = j < half ? half + j : j < 2 * half ? j - half : W - 1;
    map[j] = spec_fft(W) || wide ? bank_fft_pos(bin, W) : bin;
  }
  std::vector<float2> tw = twiddle_table(czt ? p.M : W);
  std::vector<int> czbin;
  if (wide || czt) {  // pass B's table after the W- or M-point one
    const std::vector<float2> tc = twiddle_table(spec_wide_chunk(czt ? p.M : W));
    tw.insert(tw.end(), tc.begin(), tc.end());
  }
  if (czt) {  // then the chirp and Bh
    std::vector<float2> chirp, kern;
    czt_tables(W, chirp, kern, czbin);
    tw.insert(tw.end(), chirp.begin(), chirp.end());
    tw.insert(tw.end(), kern.begin(), kern.end());
  }
  const size_t hold_bytes = (size_t)p.NR * W * sizeof(unsigned);
  if (cudaMalloc(&p.d_tw, tw.size() * sizeof(float2)) != cudaSuccess ||
      cudaMalloc(&p.d_map, W * sizeof(int)) != cudaSuccess || cudaMalloc(&p.d_hold, hold_bytes) != cudaSuccess ||
      (ring_cap > 0 && cudaMalloc(&p.d_ring, ring_cap * sizeof(float2)) != cudaSuccess) ||
      (window != nullptr && cudaMalloc(&p.d_win, W * sizeof(float)) != cudaSuccess) ||
      (p.mean && cudaMalloc(&p.d_fbuf, (size_t)p.fb_frames * W * sizeof(float)) != cudaSuccess) ||
      (wide && cudaMalloc(&p.d_scratch, (size_t)p.fb_frames * W * sizeof(float2)) != cudaSuccess) ||
      (czt && cudaMalloc(&p.d_scratch, 2 * (size_t)p.fb_frames * p.M * sizeof(float2)) != cudaSuccess) ||
      (czt && cudaMalloc(&p.d_bin, (size_t)p.M * sizeof(int)) != cudaSuccess)) {
    for (void *d : p.buffers())
      if (d) cudaFree(d);
    XL_LOG("spectrum: out of device memory");
    return -ENOMEM;
  }
  CU_OK(cudaMemcpy(p.d_tw, tw.data(), tw.size() * sizeof(float2), cudaMemcpyHostToDevice));
  CU_OK(cudaMemcpy(p.d_map, map.data(), W * sizeof(int), cudaMemcpyHostToDevice));
  if (window != nullptr) CU_OK(cudaMemcpy(p.d_win, window, W * sizeof(float), cudaMemcpyHostToDevice));
  if (czt) CU_OK(cudaMemcpy(p.d_bin, czbin.data(), (size_t)p.M * sizeof(int), cudaMemcpyHostToDevice));
  // (on a group stream, finished before the spectrum exists: the kernels' streams do not wait for the legacy one)
  CU_OK(cudaMemsetAsync(p.d_hold, 0, hold_bytes, g->s_in));
  CU_OK(cudaStreamSynchronize(g->s_in));
  int id = 0;
  while (id < (int)g->spectra.size() && g->spectra[id].active) id++;
  if (id == (int)g->spectra.size()) g->spectra.emplace_back();
  g->spectra[id] = p;
  g->dirty = true;  // its rows in the arenas, the input ring's history bound
  *spectrum_id = id;
  return 0;
}

// xlg_add_spectrum_ex, and with any = true xlg_add_spectrum_any
static int add_spectrum_desc(xlg_group *g, int source, int source_id, const xlg_spectrum_desc *desc, bool any,
                             int *spectrum_id) {
  if (g == nullptr || spectrum_id == nullptr) return -EINVAL;
  if (desc == nullptr) {
    XL_LOG("spectrum: no description");
    return -EINVAL;
  }
  int src = -1;
  if (source == XLG_SOURCE_CLIENT) {
    if (source_id < 0 || source_id >= (int)g->clients.size() || !g->clients[source_id].active ||
        g->clients[source_id].sb) {
      XL_LOG("client spectrum: client %d does not exist", source_id);
      return -EINVAL;
    }
    src = source_id;
  } else if (source == XLG_SOURCE_SUBBAND) {
    src = subband_client(g, source_id);
    if (src < 0) {
      XL_LOG("sub-band spectrum: sub-band %d does not exist", source_id);
      return -EINVAL;
    }
  } else if (source != XLG_SOURCE_BAND) {
    XL_LOG("spectrum: unknown source %d", source);
    return -EINVAL;
  }
  return add_spectrum(g, src, desc->width, desc->frames_per_row, desc->skip_per_row, desc->flags, desc->hop,
                      desc->reduce, desc->window, any, spectrum_id);
}

extern "C" int xlg_add_spectrum(xlg_group *g, uint32_t width, uint32_t frames_per_row, uint32_t skip_per_row,
                                uint32_t flags, int *spectrum_id) {
  const xlg_spectrum_desc desc = {width, frames_per_row, skip_per_row, flags, 0, XLG_SPECTRUM_MAX, nullptr};
  return add_spectrum_desc(g, XLG_SOURCE_BAND, 0, &desc, false, spectrum_id);
}

extern "C" int xlg_add_client_spectrum(xlg_group *g, int client_id, uint32_t width, uint32_t frames_per_row,
                                       uint32_t skip_per_row, uint32_t flags, int *spectrum_id) {
  const xlg_spectrum_desc desc = {width, frames_per_row, skip_per_row, flags, 0, XLG_SPECTRUM_MAX, nullptr};
  return add_spectrum_desc(g, XLG_SOURCE_CLIENT, client_id, &desc, false, spectrum_id);
}

extern "C" int xlg_add_subband_spectrum(xlg_group *g, int subband_id, uint32_t width, uint32_t frames_per_row,
                                        uint32_t skip_per_row, uint32_t flags, int *spectrum_id) {
  const xlg_spectrum_desc desc = {width, frames_per_row, skip_per_row, flags, 0, XLG_SPECTRUM_MAX, nullptr};
  return add_spectrum_desc(g, XLG_SOURCE_SUBBAND, subband_id, &desc, false, spectrum_id);
}

extern "C" int xlg_add_spectrum_ex(xlg_group *g, int source, int source_id, const xlg_spectrum_desc *desc,
                                   int *spectrum_id) {
  return add_spectrum_desc(g, source, source_id, desc, false, spectrum_id);
}

extern "C" int xlg_add_spectrum_any(xlg_group *g, int source, int source_id, const xlg_spectrum_desc *desc,
                                    int *spectrum_id) {
  return add_spectrum_desc(g, source, source_id, desc, true, spectrum_id);
}

static SpectrumHost *spectrum_of(xlg_group *g, int id) {
  if (id < 0 || id >= (int)g->spectra.size() || !g->spectra[id].active) return nullptr;
  return &g->spectra[id];
}

extern "C" int xlg_remove_spectrum(xlg_group *g, int spectrum_id) {
  if (g == nullptr) return -EINVAL;
  SpectrumHost *p = spectrum_of(g, spectrum_id);
  if (p == nullptr) {
    XL_LOG("spectrum %d does not exist", spectrum_id);
    return -EINVAL;
  }
  // in-flight tickets still read the tables and the hold: freed at the next re-layout, which drains
  for (void *d : p->buffers())
    if (d) g->dead_spec.push_back(d);
  *p = SpectrumHost();
  g->dirty = true;
  return 0;
}

extern "C" int xlg_spectrum_info(const xlg_group *g, int spectrum_id, int *kernel, uint64_t *rows_done) {
  if (g == nullptr) return -EINVAL;
  const SpectrumHost *p = spectrum_of(const_cast<xlg_group *>(g), spectrum_id);
  if (p == nullptr) return -EINVAL;
  if (kernel) *kernel = p->kind == SPEC_CZT ? 3 : p->kind == SPEC_WIDE ? 2 : spec_fft(p->W) ? 1 : 0;
  if (rows_done) *rows_done = p->rows_done;
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

// One spectrum channel-stage launch, grown over the entries it serves: CTAs along x (0: no launch), along y, and
// dynamic shared memory
struct SpecLaunch {
  int ctas = 0, groups = 0;
  size_t smem = 0;
  void grow(int c, int gr = 1, size_t sm = 0) {
    ctas = std::max(ctas, c);
    groups = std::max(groups, gr);
    smem = std::max(smem, sm);
  }
};

// One block being submitted: where it goes, and what the walks over its clients, banks and sub-bands found (the
// sizes of each kernel family's launch)
struct Block {
  xlg_group *g;
  Slot &s;
  HostOut &ho;
  int64_t ticket;
  long long S;  // stream position of its first sample, on its path
  int n;        // complex samples (src/xlating.c:387)
  bool q15;
  unsigned mask;
  int nc;       // client table entries the kernels walk
  cudaStream_t cs = nullptr, cvs = nullptr;  // its compute stream, the stream of its raw -> ring conversion
  // client walk
  int max_generic_out = 0, poly_warps = 0, max_poly4_out = 0;
  int n_casc = 0, max_n1 = 0;
  int n_crat = 0, max_rat_ctas = 0;  // rational stage B; CTAs per rational client
  size_t casc_poly_smem = 0;
  // bank walk
  int n_bk = 0, max_bk_n1 = 0, max_bk_cg = 0;
  size_t bk_smem = 0;
  int n_bf = 0, max_bf_ctas = 0;  // FFT banks
  size_t bf_smem = 0;
  int n_bz = 0, max_bz_ctas = 0;  // chirp-z banks
  size_t bz_smem = 0;
  // spectrum walk: entries, row values to emit, the end of their rows in the arena; the plain entries' FFT and
  // direct paths
  int n_spec = 0, max_sp_values = 0;
  size_t sp_used = 0;
  SpecLaunch spf, spd;
  // the extended spectra, then the wide, then the chirp-z ones, the last entries: their counts, the values the fold
  // passes over, the extended FFT and direct paths, the wide passes A and B, the chirp-z passes A (and C), B (and D)
  int n_spx = 0, n_spw = 0, n_spc = 0, max_fold_values = 0;
  SpecLaunch spxf, spxd, spwa, spwb, spca, spcb;
  int n_spa = 0, max_spa_n = 0;  // appends to spectrum sources' rings, the longest
  // sub-band walk
  int n_sb = 0, max_sb_n1 = 0, max_sb_n2 = 0;
  int max_sbr_ctas = 0, max_sbr_l2 = 0;  // rational classes: output tiles of the longest residue, largest L2
  size_t sb_smem = 0, sbr_smem = 0;
};

// Clients: each one's outputs in this block (the host mirror of the oscillator pre-pass kernel's integer formula),
// its next window (h.hist) and, for a cascade, its stage-B walk
static void walk_clients(Block &b) {
  xlg_group *g = b.g;
  Slot &s = b.s;
  HostOut &ho = b.ho;
  for (size_t i = 0; i < g->clients.size(); i++) {
    HostClient &h = g->clients[i];
    if (!h.active || h.mem || h.bank >= 0) continue;
    // upsampled coordinates (the same integers for L = 1)
    const long long Su = b.S * h.L, Eu = (b.S + b.n) * h.L;
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
    if (h.kind == 4) b.max_poly4_out = std::max(b.max_poly4_out, n_out);
    if (h.kind == 3) {
      // warps of fir_poly_generic_cf32_kernel: min(L, n_out) residues x groups of G_OPW outputs
      const int per = (int)((n_out + (long long)h.L - 1) / h.L);
      b.poly_warps = std::max(b.poly_warps, (int)std::min<long long>(h.L, n_out) * ((per + G_OPW - 1) / G_OPW));
    }
    if (b.q15 || h.kind == 0) b.max_generic_out = std::max(b.max_generic_out, n_out);
    if (h.casc) {
      const StageBGeom &geo = h.b2.geo;
      const StageBStep w = stage_b_walk(h.b2.geo, h.b2.ring.pos, n_out, h.b2.fin_cap);
      if (geo.L2 == 1) {
        stage_b_fill(h.b2, w, n_out, h.out_off, &s.cblk.h[h.cblk], nullptr);
        s.casc_macs += (uint64_t)w.n2 * geo.T2;
      } else {
        // only the appends read this client's CascBlk; cascade_fir_poly_cf32_kernel reads its CascPolyBlk
        stage_b_fill(h.b2, w, n_out, h.out_off, &s.cblk.h[g->n_casc_int + b.n_crat], &s.pblk.h[b.n_crat]);
        b.n_crat++;
        b.max_rat_ctas = std::max(b.max_rat_ctas, (w.n2 + h.b2.ko - 1) / h.b2.ko);
        b.casc_poly_smem = std::max(b.casc_poly_smem, cascade_poly_smem(h.b2.ko, (int)geo.L2, (int)geo.D2, geo.Tb2));
        s.casc_macs += (uint64_t)w.n2 * (uint64_t)geo.Tb2;
      }
      b.n_casc++;
      h.b2.ring.pos += n_out;
      h.last_n2 = w.n2;
      b.max_n1 = std::max(b.max_n1, n_out);
    }
  }
}

// Banks: each walks the block as an integer client (D1, T1) attached at P; its channels are sub-bands of n1
// samples
static void walk_banks(Block &b) {
  xlg_group *g = b.g;
  Slot &s = b.s;
  s.bk_poly = s.bk_dft = 0;
  s.bf_poly = s.bf_flops = 0;
  for (int bi = 0; bi < (int)g->banks.size(); bi++) {
    BankHost &k = g->banks[bi];
    if (!k.active) continue;
    const long long first = b.S - k.hist;
    const int n1 = xl_walk(&k.hist, b.n, k.T1, k.D1, (int)((uint64_t)g->max_input_len / 2 / k.D1 + 2));
    for (int i : k.cids) {
      g->clients[i].hist = k.hist;
      b.ho.n_out[i] = n1;
      b.ho.out_off[i] = g->clients[i].out_off;
    }
    if (k.cids.empty()) continue;
    BankBlk &e = k.kind == BANK_CZT ? s.bzblk.h[b.n_bz++] : k.kind == BANK_FFT ? s.bfblk.h[b.n_bf++]
                                                                              : s.bkblk.h[b.n_bk++];
    e.taps = g->d_bktaps + k.taps_off;
    e.tw = g->d_bktw + k.tw_off;
    e.chans = g->d_bkch + k.ch_off;
    e.first = first;
    e.zb = k.P;
    e.mask = b.mask;
    e.n1 = n1;
    e.D1 = (int)k.D1;
    e.T1 = (int)k.T1;
    e.K = k.K;
    e.tpad = k.tpad;
    e.n_ch = (int)k.cids.size();
    e.r0 = (int)(((first - k.P) % k.K + k.K) % k.K);
    if (k.kind == BANK_CZT) {
      const int M = bank_czt_m(k.K);
      b.max_bz_ctas = std::max(b.max_bz_ctas, (n1 + bank_czt_frames(M) - 1) / bank_czt_frames(M));
      b.bz_smem = std::max(b.bz_smem, bank_czt_smem(M));
      s.bf_poly += (uint64_t)n1 * k.T1;
      s.bf_flops += (uint64_t)n1 * (2 * xlg_bank_fft_flops((uint32_t)M) + 4ull * k.K + 4ull * M + 4ull * e.n_ch);
      continue;
    }
    if (k.kind == BANK_FFT) {
      b.max_bf_ctas = std::max(b.max_bf_ctas, (n1 + bank_fft_frames(k.K) - 1) / bank_fft_frames(k.K));
      b.bf_smem = std::max(b.bf_smem, bank_fft_smem(k.K));
      s.bf_poly += (uint64_t)n1 * k.T1;
      s.bf_flops += (uint64_t)n1 * xlg_bank_fft_flops((uint32_t)k.K);
      continue;
    }
    b.max_bk_n1 = std::max(b.max_bk_n1, n1);
    b.max_bk_cg = std::max(b.max_bk_cg, (e.n_ch + BK_CG - 1) / BK_CG);
    b.bk_smem = std::max(b.bk_smem, bank_smem((int)k.D1, (int)k.T1));
    s.bk_poly += (uint64_t)n1 * k.T1;
    s.bk_dft += (uint64_t)n1 * k.cids.size() * (uint64_t)k.K;
  }
}

// Spectra: a source's new samples appended to the spectrum's ring, then the frames this block completes (those
// whose last sample it holds) and the rows they complete, in closed form from the frames completed since P.  A
// source's counts are read here, every block (a re-layout moves its row): a cascade's final row is h.last_n2 at
// h.b2.fin_off (ho still holds stage A until launch_stage_b), and a sub-band's or bank channel's ho.n_out is
// zeroed by launch_members after this walk.
static void walk_spectrum(Block &b, int id) {
  xlg_group *g = b.g;
  Slot &s = b.s;
  SpectrumHost &p = g->spectra[id];
  long long E = b.S + b.n;
  if (p.src >= 0) {
    const HostClient &h = g->clients[p.src];
    const int n_src = h.casc ? h.last_n2 : b.ho.n_out[p.src];
    if (n_src > 0) {
      CascBlk &cb = s.spcb.h[b.n_spa++];
      memset(&cb, 0, sizeof(cb));
      cb.ring = p.d_ring;
      cb.a_pos = p.pos;
      cb.mask = p.ring_mask;
      cb.a_off = h.casc ? h.b2.fin_off : h.out_off;
      cb.n1 = n_src;
      b.max_spa_n = std::max(b.max_spa_n, n_src);
    }
    p.pos += n_src;
    E = p.pos;
  }
  const uint64_t d = (uint64_t)(E - p.P), F = (uint64_t)p.F;
  uint64_t total;
  if (p.kind != SPEC_PLAIN) {  // frames completed at offset o of a row: none before W, then one more every H, at most F
    const uint64_t o = d % (uint64_t)p.R;
    total = d / (uint64_t)p.R * F + (o < (uint64_t)p.W ? 0 : std::min<uint64_t>(F, (o - p.W) / (uint64_t)p.H + 1));
  } else {
    total = d / (uint64_t)p.R * F + std::min<uint64_t>(F, d % (uint64_t)p.R / (uint64_t)p.W);
  }
  const int n_frames = (int)(total - (p.rows_done * F + (uint64_t)p.fir));
  const int n_rows = (int)(total / F - p.rows_done);
  b.ho.sp_rows[id] = n_rows;
  b.ho.sp_off[id] = 2 * p.out_off;
  if (n_frames > 0) {
    s.spring.h[b.n_spec] = p.src < 0 ? g->ring : p.d_ring;
    SpecBlk &e = s.spblk.h[b.n_spec++];
    e.tw = p.d_tw;
    e.map = p.d_map;
    e.hold = p.d_hold;
    e.out = reinterpret_cast<float *>(s.d_out) + 2 * (size_t)p.out_off;
    e.base = p.P + (long long)(p.rows_done * (uint64_t)p.R);
    e.mask = p.src < 0 ? b.mask : p.ring_mask;
    e.W = p.W;
    e.F = p.F;
    e.R = p.R;
    e.NR = p.NR;
    e.f0 = (unsigned)p.fir;
    e.n_frames = n_frames;
    e.n_rows = n_rows;
    e.slot0 = (int)(p.rows_done % (uint64_t)p.NR);
    e.power = p.power ? 1 : 0;
    e.inv_w = 1.0f / (float)p.W;
    // a chirp-z frame: two M-point transforms, the chirp's W products and Bh's M (4 instructions each)
    const uint64_t flops = p.kind == SPEC_CZT ? 2 * xlg_bank_fft_flops((uint32_t)p.M) + 4ull * p.W + 4ull * p.M
                           : spec_fft(p.W) || p.kind == SPEC_WIDE ? xlg_bank_fft_flops((uint32_t)p.W)
                                                                  : 4ull * p.W * p.W;
    s.sp_frames += (uint64_t)n_frames;
    s.sp_flops += (uint64_t)n_frames * (flops + 6ull * p.W + (p.d_win ? 2ull * p.W : 0) + (p.mean ? p.W : 0));
    if (p.kind != SPEC_PLAIN) {
      SpecExt &x = s.spext.h[b.n_spx + b.n_spw + b.n_spc];
      x.win = p.d_win;
      x.fbuf = p.d_fbuf;
      x.H = p.H;
      x.mean = p.mean ? 1 : 0;
    }
    if (p.mean)  // values of the rows its frames touch
      b.max_fold_values = std::max(b.max_fold_values, (int)(((long long)p.fir + n_frames - 1) / p.F + 1) * p.W);
    if (p.kind == SPEC_CZT) {
      SpecCzt &c = s.spczt.h[b.n_spc++];
      const int C = spec_wide_chunk(p.M);
      const size_t rows = (size_t)p.fb_frames * p.M;
      c.s1 = p.d_scratch;
      c.s2 = p.d_scratch + rows;
      c.tw_c = p.d_tw + p.M;
      c.chirp = c.tw_c + C;
      c.kern = c.chirp + p.W;
      c.bin = p.d_bin;
      c.M = p.M;
      b.spca.grow(n_frames * (C / SPEC_THREADS));
      b.spcb.grow(n_frames * (p.M / C), 1, (size_t)C * sizeof(float2));
    } else if (p.kind == SPEC_WIDE) {
      SpecWide &w = s.spwide.h[b.n_spw++];
      w.scratch = p.d_scratch;
      w.tw_c = p.d_tw + p.W;
      const int C = spec_wide_chunk(p.W);
      b.spwa.grow(n_frames * (C / SPEC_THREADS));
      b.spwb.grow(n_frames * (p.W / C));
    } else {  // the FFT or the direct path, in the plain or the extended kernels
      const bool x = p.kind == SPEC_EXT;
      b.n_spx += x ? 1 : 0;
      const int Ff = bank_fft_frames(p.W), Fd = spec_direct_frames(p.W);
      if (spec_fft(p.W))
        (x ? b.spxf : b.spf).grow((n_frames + Ff - 1) / Ff, 1, bank_fft_smem(p.W));
      else
        (x ? b.spxd : b.spd).grow((n_frames + Fd - 1) / Fd, spec_direct_groups(p.W), spec_direct_smem(p.W));
    }
    b.max_sp_values = std::max(b.max_sp_values, n_rows * p.W);
    b.sp_used = std::max(b.sp_used, (size_t)p.out_off + ((size_t)n_rows * p.W + 1) / 2);
  }
  p.rows_done = total / F;
  p.fir = (int)(total % F);
}

// every spectrum, by kind: the table is [plain entries | extended entries | wide entries | chirp-z entries]
static void walk_spectra(Block &b) {
  xlg_group *g = b.g;
  b.s.sp_frames = b.s.sp_flops = 0;
  for (int seg = 0; seg < 4; seg++)
    for (int id = 0; id < (int)g->spectra.size(); id++) {
      const SpectrumHost &p = g->spectra[id];
      if (seg == 0) b.ho.sp_w[id] = p.active ? p.W : 0;
      if (p.active && p.kind == seg) walk_spectrum(b, id);
    }
}

// Sub-band members: each class walks its sub-band's n1 new samples (ho.n_out of the sub-band) from the sub-band
// ring's position before them; then the sub-bands' appends
static void walk_subbands(Block &b) {
  xlg_group *g = b.g;
  Slot &s = b.s;
  HostOut &ho = b.ho;
  b.n_sb = (int)g->sb_list.size();
  s.sb_macs = s.sb_rows = 0;
  if (b.n_sb == 0) return;
  for (size_t c = 0; c < g->sb_classes.size(); c++) {
    const SbClassHost &ch = g->sb_classes[c];
    const HostClient &a = g->clients[ch.sb_cid];
    const HostClient &m0 = g->clients[ch.members[0]];
    StageBGeom geo = m0.b2.geo;
    const StageBStep w = stage_b_walk(geo, a.b2.ring.pos, ho.n_out[ch.sb_cid], m0.out_cap);
    const int n2 = w.n2;
    SbBlk &e = s.sbblk.h[c];
    e.ring = a.b2.ring.p;
    e.first = w.first;
    e.zb = ch.zb;
    e.mask = (unsigned)(a.b2.ring.cap - 1);
    e.n2 = n2;
    e.D2 = (int)geo.D2;
    e.T2 = ch.Tb;
    for (int id : ch.members) {
      g->clients[id].b2.geo.hist2 = geo.hist2;
      ho.n_out[id] = n2;
      ho.out_off[id] = g->clients[id].out_off;
    }
    s.sb_macs += (uint64_t)n2 * ch.Tb * ch.members.size();
    if (ch.L2 == 1) {
      b.max_sb_n2 = std::max(b.max_sb_n2, n2);
      b.sb_smem = std::max(b.sb_smem, subband_smem(e.D2, e.T2));
    } else if (n2 > 0) {
      b.max_sbr_ctas = std::max(b.max_sbr_ctas, ((n2 + ch.L2 - 1) / ch.L2 + SB_KO - 1) / SB_KO);
      b.max_sbr_l2 = std::max(b.max_sbr_l2, ch.L2);
      b.sbr_smem = std::max(b.sbr_smem, subband_smem(e.D2, e.T2));
    }
  }
  for (int k = 0; k < b.n_sb; k++) {
    const int i = g->sb_list[k];
    HostClient &a = g->clients[i];
    const int n1 = ho.n_out[i];
    CascBlk &cb = s.sbcb.h[k];
    memset(&cb, 0, sizeof(cb));
    cb.ring = a.b2.ring.p;
    cb.a_pos = a.b2.ring.pos;
    cb.mask = (unsigned)(a.b2.ring.cap - 1);
    cb.a_off = a.out_off;
    cb.n1 = n1;
    a.b2.ring.pos += n1;
    s.sb_rows += (uint64_t)n1;
    b.max_sb_n1 = std::max(b.max_sb_n1, n1);
  }
}

// Input staging, then the conversion (its own stream: never behind the FIR CTAs of earlier blocks that still wait
// for an SM), which the compute stream waits for
static int stage_and_convert(Block &b, int fmt, const void *input, uint32_t flags) {
  xlg_group *g = b.g;
  Slot &s = b.s;
  const int n = b.n;
  const void *d_in = input;
  if (!(flags & XLG_INPUT_DEVICE) && n > 0) {
    const size_t bytes = (size_t)n * 2 * elem_bytes(fmt);
    const bool pinned = page_locked(input);
    const void *src = input;
    if (!pinned) {
      memcpy(s.h_raw, input, bytes);
      src = s.h_raw;
    }
    CU_OK(cudaMemcpyAsync(s.d_raw, src, bytes, cudaMemcpyHostToDevice, g->s_in));
    CU_OK(cudaEventRecord(s.ev_h2d, g->s_in));
    CU_OK(cudaStreamWaitEvent(b.cvs, s.ev_h2d, 0));
    // caller-owned pinned memory is read by the copy engine AFTER this call returns: unless
    // the caller promised to leave it alone (XLG_INPUT_KEEP), wait for the copy (a 256 KiB
    // block is ~10 us) so that the buffer may be reused at once, like a pageable one
    if (pinned && !(flags & XLG_INPUT_KEEP)) CU_OK(cudaEventSynchronize(s.ev_h2d));
    d_in = s.d_raw;
  }

  // (in-order streams: later submits' conversions queue behind this one's, so one wait per event is enough)
  for (size_t i = 0; i < g->n_user_waits; i++) {
    const cudaEvent_t e = g->ev_user[i];
    CU_OK(cudaStreamWaitEvent(b.cvs, e, 0));
    CU_OK(cudaStreamWaitEvent(g->s_in, e, 0));
    if (!g->conv_own_stream)
      for (int c = 0; c < g->n_cs; c++) CU_OK(cudaStreamWaitEvent(g->s_cs[c], e, 0));
  }
  g->n_user_waits = 0;
  // what xlg_input_consumed waits for: the copy out of a host block, the conversion that reads a device block
  s.ev_input = n == 0 ? nullptr : (flags & XLG_INPUT_DEVICE) ? s.ev_conv : s.ev_h2d;
  if (n > 0) {
    if (g->timeline && !g->base_recorded) {
      CU_OK(cudaEventRecord(g->ev_base, b.cvs));
      g->base_recorded = true;
    }
    if (span_begin(g, s, SP_CONV, b.cvs)) return -EIO;
    if (fmt == XLG_FMT_CU8)
      launch_convert<0>(b.q15, d_in, g, b.S, n, b.cvs);
    else if (fmt == XLG_FMT_CS8)
      launch_convert<1>(b.q15, d_in, g, b.S, n, b.cvs);
    else if (fmt == XLG_FMT_CS16)
      launch_convert<2>(b.q15, d_in, g, b.S, n, b.cvs);
    else
      copy_cf32_kernel<<<(n + 255) / 256, 256, 0, b.cvs>>>(static_cast<const float2 *>(d_in), g->ring,
                                                           (unsigned)(g->ring_cap - 1), b.S, n);
    if (span_end(g, s, SP_CONV, b.cvs)) return -EIO;
    CU_OK(cudaEventRecord(s.ev_conv, b.cvs));
  }
  // the FIR reads this block's samples and, as history, the previous blocks'
  // (s_cv is in order: waiting for THIS block's conversion covers the earlier ones -- one driver call less)
  if (g->have_last_conv && (b.cvs == b.cs || n == 0)) CU_OK(cudaStreamWaitEvent(b.cs, g->ev_last_conv_ref, 0));
  if (n > 0) {
    if (b.cvs != b.cs) CU_OK(cudaStreamWaitEvent(b.cs, s.ev_conv, 0));
    g->ev_last_conv_ref = s.ev_conv;
    g->have_last_conv = true;
  }
  return 0;
}

// Banks: after the conversions the FIR kernels wait for, not after the pre-pass (they have no oscillator); the
// direct banks, then the FFT and chirp-z banks in one span
static int launch_banks(Block &b) {
  xlg_group *g = b.g;
  Slot &s = b.s;
  if (b.n_bk > 0 && b.max_bk_n1 > 0) {
    if (span_begin(g, s, SP_BANK, b.cs)) return -EIO;
    CU_OK(s.bkblk.upload((size_t)b.n_bk, b.cs));
    bank_cf32_kernel<<<dim3((b.max_bk_n1 + BK_F - 1) / BK_F, b.n_bk, b.max_bk_cg), BK_THREADS, b.bk_smem, b.cs>>>(
        s.bkblk.d, g->ring, s.d_out);
    if (span_end(g, s, SP_BANK, b.cs)) return -EIO;
  }
  const bool bf = b.n_bf > 0 && b.max_bf_ctas > 0, bz = b.n_bz > 0 && b.max_bz_ctas > 0;
  if (!bf && !bz) return 0;
  if (span_begin(g, s, SP_BANK_FFT, b.cs)) return -EIO;
  if (bf) {
    CU_OK(s.bfblk.upload((size_t)b.n_bf, b.cs));
    bank_fft_cf32_kernel<<<dim3(b.max_bf_ctas, b.n_bf), BF_THREADS, b.bf_smem, b.cs>>>(s.bfblk.d, g->ring, s.d_out);
  }
  if (bz) {
    CU_OK(s.bzblk.upload((size_t)b.n_bz, b.cs));
    bank_czt_cf32_kernel<<<dim3(b.max_bz_ctas, b.n_bz), BZ_THREADS, b.bz_smem, b.cs>>>(s.bzblk.d, g->ring, s.d_out);
  }
  return span_end(g, s, SP_BANK_FFT, b.cs);
}

// Spectra: after the clients' launches (every client, stage-B and member kernel is on b.cs before them), so that no
// client kernel waits for them; each block's after the previous one's, which emptied the hold rows it reuses and
// read the sources' rings it appends to.  One append launch for all sources, then the channel stages and the emit
static int launch_spectra(Block &b) {
  xlg_group *g = b.g;
  Slot &s = b.s;
  if (b.n_spec == 0 && b.n_spa == 0) return 0;
  if (g->have_last_spec) CU_OK(cudaStreamWaitEvent(b.cs, g->ev_last_spec, 0));
  if (span_begin(g, s, SP_SPEC, b.cs)) return -EIO;
  if (b.n_spa > 0) {
    CU_OK(s.spcb.upload((size_t)b.n_spa, b.cs));
    cascade_launch_append(s.spcb.d, b.n_spa, b.max_spa_n, s.d_out, b.cs);
  }
  if (b.n_spec > 0) {
    CU_OK(s.spblk.upload((size_t)b.n_spec, b.cs));
    CU_OK(s.spring.upload((size_t)b.n_spec, b.cs));
  }
  const int n_plain = b.n_spec - b.n_spx - b.n_spw - b.n_spc;
  if (b.spf.ctas > 0)
    spectrum_fft_kernel<<<dim3(b.spf.ctas, n_plain), SPEC_THREADS, b.spf.smem, b.cs>>>(s.spblk.d, s.spring.d);
  if (b.spd.ctas > 0)
    spectrum_direct_kernel<<<dim3(b.spd.ctas, b.spd.groups, n_plain), SPEC_THREADS, b.spd.smem, b.cs>>>(
        s.spblk.d, s.spring.d);
  if (b.n_spx + b.n_spw + b.n_spc > 0) {
    const SpecBlk *xb = s.spblk.d + n_plain;
    const float2 *const *xr = s.spring.d + n_plain;
    CU_OK(s.spext.upload((size_t)(b.n_spx + b.n_spw + b.n_spc), b.cs));
    if (b.spxf.ctas > 0)
      spectrum_fft_ext_kernel<<<dim3(b.spxf.ctas, b.n_spx), SPEC_THREADS, b.spxf.smem, b.cs>>>(xb, xr, s.spext.d);
    if (b.spxd.ctas > 0)
      spectrum_direct_ext_kernel<<<dim3(b.spxd.ctas, b.spxd.groups, b.n_spx), SPEC_THREADS, b.spxd.smem, b.cs>>>(
          xb, xr, s.spext.d);
    if (b.n_spw > 0) {  // the wide entries: pass A into their scratch, then pass B into the hold or frame buffer
      CU_OK(s.spwide.upload((size_t)b.n_spw, b.cs));
      spectrum_wide_a_kernel<<<dim3(b.spwa.ctas, b.n_spw), SPEC_THREADS, 0, b.cs>>>(
          xb + b.n_spx, xr + b.n_spx, s.spext.d + b.n_spx, s.spwide.d);
      spectrum_wide_b_kernel<<<dim3(b.spwb.ctas, b.n_spw), SPEC_THREADS, SPEC_WIDE_SMEM, b.cs>>>(
          xb + b.n_spx, s.spext.d + b.n_spx, s.spwide.d);
    }
    if (b.n_spc > 0) {  // the chirp-z entries: the forward transform and Bh into s2, the second transform
      const int o = b.n_spx + b.n_spw;
      CU_OK(s.spczt.upload((size_t)b.n_spc, b.cs));
      spectrum_czt_a_kernel<<<dim3(b.spca.ctas, b.n_spc), SPEC_THREADS, 0, b.cs>>>(xb + o, xr + o, s.spext.d + o,
                                                                                 s.spczt.d);
      spectrum_czt_b_kernel<<<dim3(b.spcb.ctas, b.n_spc), SPEC_THREADS, b.spcb.smem, b.cs>>>(xb + o, s.spczt.d);
      spectrum_czt_c_kernel<<<dim3(b.spca.ctas, b.n_spc), SPEC_THREADS, 0, b.cs>>>(xb + o, s.spczt.d);
      spectrum_czt_d_kernel<<<dim3(b.spcb.ctas, b.n_spc), SPEC_THREADS, b.spcb.smem, b.cs>>>(xb + o, s.spext.d + o,
                                                                                            s.spczt.d);
    }
    if (b.max_fold_values > 0)
      spectrum_fold_kernel<<<dim3((b.max_fold_values + SPEC_THREADS - 1) / SPEC_THREADS,
                                  b.n_spx + b.n_spw + b.n_spc), SPEC_THREADS, 0, b.cs>>>(xb, s.spext.d);
  }
  if (b.max_sp_values > 0)
    spectrum_emit_kernel<<<dim3((b.max_sp_values + SPEC_THREADS - 1) / SPEC_THREADS, b.n_spec), SPEC_THREADS, 0,
                           b.cs>>>(s.spblk.d);
  if (span_end(g, s, SP_SPEC, b.cs)) return -EIO;
  CU_OK(cudaEventRecord(s.ev_spec, b.cs));
  g->ev_last_spec = s.ev_spec;
  g->have_last_spec = true;
  return 0;
}

// Oscillator pre-pass (own stream: chains only on the previous pre-pass; none without a client to walk), and the
// next block's, speculatively
static int launch_prepass(Block &b) {
  xlg_group *g = b.g;
  Slot &s = b.s;
  const bool q15 = b.q15;
  const int64_t ticket = b.ticket;
  const long long S = b.S;
  const int n = b.n, nc = b.nc;
  if (nc <= 0 || !(q15 || g->n_order > 0)) return 0;
  const bool tl_phase = g->timeline && !(g->spec_valid && !q15);  // a pre-pass that ran ahead was stamped then
  if (span_begin(g, s, SP_PHASE, g->s_ph)) return -EIO;
  if (tl_phase) CU_OK(cudaEventRecord(s.tl_ph[(ticket / XLG_SLOTS) & 1][0], g->s_ph));
  if (g->timeline) s.pf_on[SP_PHASE] = true;  // (harvest_locked writes the block's timeline row by it)
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
  if (span_end(g, s, SP_PHASE, g->s_ph)) return -EIO;
  if (tl_phase) CU_OK(cudaEventRecord(s.tl_ph[(ticket / XLG_SLOTS) & 1][1], g->s_ph));
  if (!ran_ahead) CU_OK(cudaEventRecord(s.ev_phase, g->s_ph));
  CU_OK(cudaStreamWaitEvent(b.cs, s.ev_phase, 0));
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
  return 0;
}

// Integer tiled classes.  Tile shape for this launch: the largest thread tile (best FMA : load ratio) that
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
static int launch_tiled(Block &b) {
  xlg_group *g = b.g;
  Slot &s = b.s;
  HostOut &ho = b.ho;
  if (b.q15 || g->classes.empty()) return 0;
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
  TileBatch t(shape.kt());
  for (TileClassHost &ch : g->classes) {
    int n_out = 0;
    for (int id : ch.real) n_out = std::max(n_out, ho.n_out[id]);
    if (n_out <= 0) continue;
    // merged: the earliest possible window start of this block (history = T-1); every member's window starts
    // delta in [0, D) samples later, read on the device from BlkInfo.  Otherwise identical alignment: recover
    // this block's start from the walked hist
    const HostClient &h0 = g->clients[ch.real[0]];
    const long long first = ch.merged ? b.S - (long long)(ch.T - 1)
                                      : (b.S + b.n) - h0.hist - (long long)ho.n_out[ch.real[0]] * (long long)h0.D;
    s.tile_macs += t.add(ch, first, n_out);
  }
  if (t.ctas == 0) return 0;
  if (span_begin(g, s, SP_TILE, b.cs)) return -EIO;
  long long *trace_ptr = nullptr;
  if (g->d_trace != nullptr && t.ctas <= T_TRACE_CTAS) {
    const int tslot = (int)(g->trace_launches % T_TRACE_LAUNCHES);
    trace_ptr = g->d_trace + (size_t)tslot * T_TRACE_REC * T_TRACE_CTAS;
    g->trace_n[tslot] = t.ctas;
    g->trace_launches++;
    g->trace_ctas = t.ctas;
  }
  shape.kernel<<<t.ctas, shape.threads, t.smem, b.cs>>>(t.P, g->ring, b.mask, (const float2 *)g->d_tile_taps,
                                                        g->d_members, g->d_member_cid, g->d_member_incr, s.d_blk,
                                                        s.d_phases, s.d_out, trace_ptr);
  return span_end(g, s, SP_TILE, b.cs);
}

// Long filters: split-K partial sums, then the ordered reduction
static int launch_long(Block &b) {
  xlg_group *g = b.g;
  Slot &s = b.s;
  HostOut &ho = b.ho;
  if (b.q15 || g->long_classes.empty()) return 0;
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
    k.first = (b.S + b.n) - h0.hist - (long long)n_out * (long long)h0.D;
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
  if (ctas == 0) return 0;
  if (span_begin(g, s, SP_LONG, b.cs)) return -EIO;
  if (pipelined) {
    // the first class gets the tensor map for its strips (all long clients of a stream normally share one D);
    // tmap_w = 0 (no map) sends every stage down the per-strip bulk copies
    strip_map_update(g, P.cls[0].D);
    P.cls[0].tmap_w = g->strip_w;
    fir_long4_cf32_kernel<<<ctas, W4_THREADS, W4_SMEM, b.cs>>>(P, g->ring, b.mask, (const float2 *)g->d_tile_taps,
                                                              s.d_partial, g->strip_map);
  } else {
    fir_long2_cf32_kernel<<<ctas, W2_THREADS, W2_SMEM, b.cs>>>(P, g->ring, b.mask, (const float2 *)g->d_tile_taps,
                                                              s.d_partial);
  }
  dim3 rgrid((max_out + 7) / 8, max_groups, P.n_classes);
  fir_long_reduce_kernel<<<rgrid, 256, 0, b.cs>>>(P, s.d_partial, g->d_members, g->d_member_incr, s.d_phases,
                                                  s.d_out);
  return span_end(g, s, SP_LONG, b.cs);
}

static int launch_generic(Block &b) {
  xlg_group *g = b.g;
  Slot &s = b.s;
  if (b.nc <= 0 || b.max_generic_out <= 0) return 0;
  dim3 grid((b.max_generic_out + G_OPC - 1) / G_OPC, b.nc);
  if (span_begin(g, s, SP_GEN, b.cs)) return -EIO;
  if (b.q15)
    fir_generic_q15_kernel<<<grid, G_THREADS, 0, b.cs>>>(g->d_clients, s.d_blk, g->qring, b.mask, g->d_qtaps,
                                                         s.d_qphases, s.d_qout);
  else
    fir_generic_cf32_kernel<<<grid, G_THREADS, 0, b.cs>>>(g->d_clients, s.d_blk, g->ring, b.mask, g->d_taps,
                                                          s.d_phases, s.d_out);
  return span_end(g, s, SP_GEN, b.cs);
}

// Rational tiled classes: the tiled kernel over one class per polyphase branch, then the placement
static int launch_poly_tiled(Block &b) {
  xlg_group *g = b.g;
  Slot &s = b.s;
  HostOut &ho = b.ho;
  if (b.q15 || g->poly_classes.empty() || b.max_poly4_out <= 0) return 0;
  // largest tile that still gives about two CTAs per SM, among the shapes that fit any CTA count per SM (every
  // one fits: eligibility was checked at 64)
  int si = kTileSmallest;
  for (int i = 0; i <= kTileSmallest; i++) {
    if (kTileShapes[i].min_ctas != 0) continue;
    const int kt = kTileShapes[i].kt();
    int ctas = 0;
    for (const TileClassHost &ch : g->poly_classes)
      ctas += ((ho.n_out[ch.real[0]] / (int)ch.interp + 1 + kt - 1) / kt) * ch.k.n_groups;
    if (ctas >= 2 * g->fir_sms) {
      si = i;
      break;
    }
  }
  const TileShapeHost &shape = kTileShapes[si];
  TileBatch t(shape.kt());
  for (size_t v = 0; v < g->poly_classes.size(); v++) {
    const TileClassHost &ch = g->poly_classes[v];
    const HostClient &h0 = g->clients[ch.real[0]];
    const int n_out = ho.n_out[ch.real[0]];
    const long long L = ch.interp, M = h0.D;
    // this block's first upsampled window (hist was advanced by the walk); branch r serves k = rho + j*L
    const long long first_u = (b.S + b.n) * L - h0.hist - (long long)n_out * M;
    const long long a = (((-(first_u + ch.branch)) % L) + L) % L;
    const long long rho = (a * ch.minv) % L;
    const int nv = rho < n_out ? (int)((n_out - 1 - rho) / L) + 1 : 0;
    s.h_vblk[v].first = (first_u + rho * M + ch.branch) / L;  // exact: the window start is -r mod L
    s.h_vblk[v].n_out = nv;
    s.h_vblk[v].pad_ = 0;
    if (nv > 0) s.tile_macs += t.add(ch, s.h_vblk[v].first, nv);
  }
  if (t.ctas == 0) return 0;
  if (span_begin(g, s, SP_POLY_TILE, b.cs)) return -EIO;
  CU_OK(cudaMemcpyAsync(s.d_vblk, s.h_vblk, g->poly_classes.size() * sizeof(BlkInfo), cudaMemcpyHostToDevice, b.cs));
  shape.kernel<<<t.ctas, shape.threads, t.smem, b.cs>>>(t.P, g->ring, b.mask, (const float2 *)g->d_tile_taps,
                                                        g->d_members, g->d_member_cid, g->d_member_incr, s.d_vblk,
                                                        g->d_ones, s.d_pscratch, nullptr);
  dim3 pgrid((b.max_poly4_out + 255) / 256, g->n_poly4);
  poly_tile_place_cf32_kernel<<<pgrid, 256, 0, b.cs>>>(g->d_clients, g->d_poly4, s.d_blk, s.d_pscratch, s.d_phases,
                                                       s.d_out);
  return span_end(g, s, SP_POLY_TILE, b.cs);
}

static int launch_poly_generic(Block &b) {
  xlg_group *g = b.g;
  Slot &s = b.s;
  if (b.q15 || g->n_poly3 <= 0 || b.poly_warps <= 0) return 0;
  constexpr int warps_per_cta = G_THREADS / 32;
  dim3 grid((b.poly_warps + warps_per_cta - 1) / warps_per_cta, g->n_poly3);
  if (span_begin(g, s, SP_POLY_GEN, b.cs)) return -EIO;
  fir_poly_generic_cf32_kernel<<<grid, G_THREADS, 0, b.cs>>>(g->d_clients, g->d_poly3, s.d_blk, g->ring, b.mask,
                                                             g->d_taps, s.d_phases, s.d_out);
  return span_end(g, s, SP_POLY_GEN, b.cs);
}

// Cascade clients: append the stage-A outputs to their rings, then stage B; from then on a client's results are
// its final row
static int launch_stage_b(Block &b) {
  xlg_group *g = b.g;
  Slot &s = b.s;
  const cudaStream_t cs = b.cs;
  if (b.q15 || b.n_casc == 0) return 0;
  // the rings are appended in block order: after the previous block's stage B, whichever stream ran it
  if (g->have_last_casc) CU_OK(cudaStreamWaitEvent(cs, g->ev_last_casc, 0));
  if (span_begin(g, s, SP_STAGE_B, cs)) return -EIO;
  CU_OK(s.cblk.upload((size_t)b.n_casc, cs));
  if (b.n_crat > 0) CU_OK(s.pblk.upload((size_t)b.n_crat, cs));
  if (b.max_n1 > 0) cascade_launch_append(s.cblk.d, b.n_casc, b.max_n1, s.d_out, cs);
  // integer stage B: one launch per ko, as the drop-in engine launches it (the kernel's summation order
  // depends on ko: with even D2 output k is summed by lane (k mod ko) mod 32)
  for (const xlg_group::CascRun &r : g->casc_runs) {
    int run_n2 = 0;
    size_t smem = 0;
    for (int c = r.c0; c < r.c1; c++) {
      run_n2 = std::max(run_n2, s.cblk.h[c].n2);
      smem = std::max(smem, cascade_smem(r.ko, s.cblk.h[c].D2, s.cblk.h[c].T2));
    }
    if (run_n2 > 0) cascade_launch_fir(s.cblk.d + r.c0, r.c1 - r.c0, run_n2, r.ko, smem, g->d_taps2, s.d_out, cs);
  }
  // rational stage B: each client's CTA size was fixed at attach to fit the shared memory
  if (b.max_rat_ctas > 0)
    cascade_launch_fir_poly(s.pblk.d, b.n_crat, b.max_rat_ctas, b.casc_poly_smem, g->d_taps2, s.d_out, cs);
  if (span_end(g, s, SP_STAGE_B, cs)) return -EIO;
  CU_OK(cudaEventRecord(s.ev_casc, cs));
  g->ev_last_casc = s.ev_casc;
  g->have_last_casc = true;
  for (size_t i = 0; i < g->clients.size(); i++)
    if (g->clients[i].active && g->clients[i].casc) {
      b.ho.n_out[i] = g->clients[i].last_n2;
      b.ho.out_off[i] = g->clients[i].b2.fin_off;
    }
  return 0;
}

// Sub-bands: append their outputs to their rings, then the members' oscillators and FIR
static int launch_members(Block &b) {
  xlg_group *g = b.g;
  Slot &s = b.s;
  const cudaStream_t cs = b.cs;
  if (b.n_sb == 0) return 0;
  // the rings are appended in block order (the cascades' event orders both)
  if (g->have_last_casc) CU_OK(cudaStreamWaitEvent(cs, g->ev_last_casc, 0));
  if (span_begin(g, s, SP_SB, cs)) return -EIO;
  CU_OK(s.sbcb.upload((size_t)b.n_sb, cs));
  if (b.max_sb_n1 > 0) cascade_launch_append(s.sbcb.d, b.n_sb, b.max_sb_n1, s.d_out, cs);
  if (b.max_sb_n2 > 0 || b.max_sbr_ctas > 0) {
    CU_OK(s.sbblk.upload(g->sb_classes.size(), cs));
    subband_phase_kernel<<<(g->n_sb_mem + 31) / 32, 32, 0, cs>>>(g->d_clients, g->d_sbmem, s.sbblk.d, s.d_sbph);
    if (b.max_sb_n2 > 0)
      subband_fir_cf32_kernel<<<dim3((b.max_sb_n2 + SB_KO - 1) / SB_KO, g->n_sb_groups_int), SB_THREADS, b.sb_smem,
                                cs>>>(s.sbblk.d, g->d_sbgrp, g->d_sbtaps, s.d_sbph, s.d_out);
    // rational classes: their groups follow the integer ones, one CTA layer per residue
    if (b.max_sbr_ctas > 0)
      subband_fir_poly_cf32_kernel<<<dim3(b.max_sbr_ctas, g->n_sb_groups - g->n_sb_groups_int, b.max_sbr_l2),
                                     SB_THREADS, b.sbr_smem, cs>>>(s.sbblk.d, g->d_sbgrp + g->n_sb_groups_int,
                                                                   g->d_sbtaps, s.d_sbph, s.d_out);
  }
  if (span_end(g, s, SP_SB, cs)) return -EIO;
  CU_OK(cudaEventRecord(s.ev_casc, cs));
  g->ev_last_casc = s.ev_casc;
  g->have_last_casc = true;
  // a sub-band is not a client: nothing to read, and the D2H copy ends before its row
  for (int i : g->sb_list) {
    b.ho.n_out[i] = 0;
    b.ho.out_off[i] = 0;
  }
  return 0;
}

// Results back to the host (the final rows), or, for XLG_OUT_DEVICE groups, done = FIR done
static int copy_back(Block &b) {
  xlg_group *g = b.g;
  Slot &s = b.s;
  HostOut &ho = b.ho;
  if ((g->flags & XLG_OUT_DEVICE) || g->arena_cap == 0 || (b.nc <= 0 && b.sp_used == 0)) {
    CU_OK(cudaEventRecord(s.ev_done, b.cs));  // results stay on the device: no hop through s_out
    return 0;
  }
  size_t used = 0;
  for (size_t i = 0; i < g->clients.size(); i++)
    if (g->clients[i].active) used = std::max(used, (size_t)ho.out_off[i] + (size_t)ho.n_out[i]);
  used = std::max(used, b.sp_used);
  CU_OK(cudaStreamWaitEvent(g->s_out, s.ev_fir, 0));
  if (used > 0) {
    if (b.q15)
      CU_OK(cudaMemcpyAsync(ho.h_qout, s.d_qout, used * sizeof(short2), cudaMemcpyDeviceToHost, g->s_out));
    else
      CU_OK(cudaMemcpyAsync(ho.h_out, s.d_out, used * sizeof(float2), cudaMemcpyDeviceToHost, g->s_out));
    s.d2h_bytes = used * (b.q15 ? sizeof(short2) : sizeof(float2));
  }
  if ((g->flags & XLG_TRACK_STATE) && !b.q15 && s.d_endph != nullptr && ho.h_endph != nullptr)
    CU_OK(cudaMemcpyAsync(ho.h_endph, s.d_endph, (size_t)b.nc * sizeof(float2), cudaMemcpyDeviceToHost, g->s_out));
  CU_OK(cudaEventRecord(s.ev_done, g->s_out));
  return 0;
}

extern "C" int64_t xlg_submit(xlg_group *g, int fmt, const void *input, size_t input_len, uint32_t flags) {
  if (g == nullptr || (input == nullptr && input_len > 0)) return -EINVAL;
  if (fmt < XLG_FMT_CU8 || fmt > XLG_FMT_CF32) return -EINVAL;
  if (fmt == XLG_FMT_CF32 && (flags & XLG_PATH_Q15)) {
    XL_LOG("the Q15 path takes no cf32 input; submit cf32 without XLG_PATH_Q15");
    return -EINVAL;
  }
  if (input_len > g->max_input_len) {
    XL_LOG("block of %zu elements exceeds max_input_len %u", input_len, g->max_input_len);
    return -EINVAL;
  }
  // the conversion kernels load one complex sample at a time (uchar2 / char2 / short2 / float2); host inputs are staged
  // into an aligned buffer, device inputs are read where they are
  const size_t sample_bytes = 2 * elem_bytes(fmt);
  if ((flags & XLG_INPUT_DEVICE) && input_len > 0 && (uintptr_t)input % sample_bytes != 0) {
    XL_LOG("device input %p is not aligned to one complex sample (%zu bytes)", input, sample_bytes);
    return -EINVAL;
  }
  const bool q15 = (flags & XLG_PATH_Q15) != 0;
  if (q15)
    for (const SpectrumHost &p : g->spectra)
      if (p.active) {
        XL_LOG("the Q15 path does not serve spectra; submit without XLG_PATH_Q15");
        return -ENOTSUP;
      }
  if (q15)
    for (const BankHost &k : g->banks)
      if (k.active) {
        XL_LOG("the Q15 path does not serve banks; submit without XLG_PATH_Q15");
        return -ENOTSUP;
      }
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
  if (fmt == XLG_FMT_CF32 && !(flags & XLG_INPUT_DEVICE) && input_len >= 2) {
    const int rc = grow_raw_cf32(g, s, !page_locked(input));
    if (rc) return rc;
  }
  Block b{g, s, ho, ticket, q15 ? g->qS : g->S, (int)(input_len / 2), q15, (unsigned)(g->ring_cap - 1), g->max_client};
  {
    // consumers read this entry's metadata under the same mutex (xlg_output) / spinlock (xlg_copy_output)
    std::lock_guard<std::mutex> lk(g->mu);
    ho.ticket.store(-1);  // the entry is being recycled (seqlock write-begin for lock-free readers)
    std::atomic_thread_fence(std::memory_order_seq_cst);
    ho.n_out.assign(g->clients.size(), 0);
    ho.out_off.assign(g->clients.size(), 0);
    if (g->flags & XLG_TRACK_STATE) ho.hist_after.assign(g->clients.size(), 0);
    ho.sp_rows.assign(g->spectra.size(), 0);
    ho.sp_off.assign(g->spectra.size(), 0);
    ho.sp_w.assign(g->spectra.size(), 0);
    ho.q15 = q15;
  }
  s.q15 = q15;
  s.tile_macs = s.algo_macs = s.out_samples = s.poly_macs = s.casc_macs = s.d2h_bytes = 0;
  s.in_samples = (uint64_t)b.n;
  std::fill(std::begin(s.pf_on), std::end(s.pf_on), false);
  // The walks, in this order: the client walk advances every client's hist, from which the tiled and long launches
  // recover each class's window start; the bank walk counts its channels' outputs, which the sub-band walk reads.
  walk_clients(b);
  walk_banks(b);
  walk_subbands(b);
  walk_spectra(b);

  // consecutive blocks alternate between two compute streams so that the tail of
  // one block's FIR overlaps the head of the next (each block's launch alone
  // cannot fill 132 SMs evenly); per-kernel profiling keeps a single stream so
  // that event-timed durations are not inflated by the overlap
  b.cs = g->profiling ? g->s_cs[0] : g->s_cs[ticket % g->n_cs];
  b.cvs = g->conv_own_stream ? g->s_cv : b.cs;
  // The launches, in stream order.  Each sizes itself by the walks' counts in ho: stage B switches the cascades'
  // counts to their final rows, and the member launch zeroes the sub-bands', only after their own launches.  Both
  // append to their rings in block order, chained on ev_last_casc.
  if (stage_and_convert(b, fmt, input, flags) || launch_banks(b) || launch_prepass(b) || launch_tiled(b) ||
      launch_long(b) || launch_generic(b) || launch_poly_tiled(b) || launch_poly_generic(b) || launch_stage_b(b) ||
      launch_members(b) || launch_spectra(b))
    return -EIO;
  CU_OK(cudaGetLastError());
  CU_OK(cudaEventRecord(s.ev_fir, b.cs));
  if (copy_back(b)) return -EIO;

  if (q15)
    g->qS += b.n;
  else
    g->S += b.n;
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

// A ticket's rows of a spectrum: where they are, how many, and the width they were made with, read together under
// the group's lock
static int spectrum_rows(xlg_group *g, int64_t ticket, int spectrum_id, const float **rows, size_t *n_rows,
                         uint32_t *width) {
  if (g == nullptr || ticket < 0 || ticket >= g->next_ticket.load()) return -EINVAL;
  HostOut &ho = g->ring_out[ticket % (int64_t)g->ring_out.size()];
  std::lock_guard<std::mutex> lk(g->mu);
  if (ho.ticket.load() != ticket) return -ESTALE;
  if (spectrum_id < 0 || spectrum_id >= (int)ho.sp_w.size() || ho.sp_w[spectrum_id] == 0) return -EINVAL;
  if (n_rows) *n_rows = (size_t)ho.sp_rows[spectrum_id];
  if (width) *width = (uint32_t)ho.sp_w[spectrum_id];
  if (rows) {
    if (g->flags & XLG_OUT_DEVICE) {
      Slot &s = g->slots[ticket % XLG_SLOTS];
      if (s.ticket.load() != ticket) return -ESTALE;  // device arenas live XLG_SLOTS tickets
      *rows = reinterpret_cast<const float *>(s.d_out) + ho.sp_off[spectrum_id];
    } else {
      *rows = reinterpret_cast<const float *>(ho.h_out) + ho.sp_off[spectrum_id];
    }
  }
  return 0;
}

extern "C" int xlg_spectrum_output(xlg_group *g, int64_t ticket, int spectrum_id, const float **rows, size_t *n_rows) {
  return spectrum_rows(g, ticket, spectrum_id, rows, n_rows, nullptr);
}

extern "C" int xlg_spectrum_width(xlg_group *g, int64_t ticket, int spectrum_id, uint32_t *width) {
  if (width == nullptr) return -EINVAL;
  return spectrum_rows(g, ticket, spectrum_id, nullptr, nullptr, width);
}

extern "C" int xlg_read_spectrum(xlg_group *g, int64_t ticket, int spectrum_id, float *dst, size_t cap_rows,
                                 size_t *n_rows) {
  if (g == nullptr || dst == nullptr) return -EINVAL;
  int rc = xlg_wait(g, ticket);
  if (rc != 0) return rc;
  const float *src = nullptr;
  size_t n = 0;
  uint32_t W = 0;
  rc = spectrum_rows(g, ticket, spectrum_id, &src, &n, &W);
  if (rc != 0) return rc;
  if (n_rows) *n_rows = n;
  const size_t bytes = std::min(n, cap_rows) * W * sizeof(float);
  if (bytes == 0) return 0;
  if (g->flags & XLG_OUT_DEVICE) {
    cudaSetDevice(g->device);
    CU_OK(cudaMemcpy(dst, src, bytes, cudaMemcpyDeviceToHost));
    if (g->slots[ticket % XLG_SLOTS].ticket.load() != ticket) return -ESTALE;
  } else {
    const HostOut &ho = g->ring_out[ticket % (int64_t)g->ring_out.size()];
    memcpy(dst, src, bytes);
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
  if (s.ticket.load() != ticket) return 0;  // the slot serves a later ticket: this one's input was read long ago
  if (s.ev_input == nullptr) return 0;      // an empty block reads nothing
  cudaSetDevice(g->device);
  CU_OK(cudaEventSynchronize(s.ev_input));
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
  // symmetry with host inputs).  An event is recorded now and attached to the consuming stream by the next
  // xlg_submit -- which knows the stream (a re-layout in between may switch stream sets) -- so a call costs one
  // record here and one wait there instead of a wait on every stream of the group.  Every call since the last
  // submit keeps its own event: a block may be produced on several streams.
  if (g->n_user_waits == g->ev_user.size()) {
    cudaEvent_t e = nullptr;
    CU_OK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
    g->ev_user.push_back(e);
  }
  CU_OK(cudaEventRecord(g->ev_user[g->n_user_waits], (cudaStream_t)cuda_stream));
  g->n_user_waits++;
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

// one kernel family's counters (the profile structs after xlg_profile)
template <typename P>
static int family_profile_read(xlg_group *g, P xlg_group::*prof, P *p, int reset) {
  if (g == nullptr || p == nullptr) return -EINVAL;
  std::lock_guard<std::mutex> lk(g->mu);
  *p = g->*prof;
  if (reset) memset(&(g->*prof), 0, sizeof(P));
  return 0;
}

extern "C" int xlg_poly_profile_read(xlg_group *g, xlg_poly_profile *p, int reset) {
  return family_profile_read(g, &xlg_group::poly_prof, p, reset);
}

extern "C" int xlg_cascade_profile_read(xlg_group *g, xlg_cascade_profile *p, int reset) {
  return family_profile_read(g, &xlg_group::casc_prof, p, reset);
}

extern "C" int xlg_subband_profile_read(xlg_group *g, xlg_subband_profile *p, int reset) {
  return family_profile_read(g, &xlg_group::sb_prof, p, reset);
}

extern "C" int xlg_bank_profile_read(xlg_group *g, xlg_bank_profile *p, int reset) {
  return family_profile_read(g, &xlg_group::bank_prof, p, reset);
}

extern "C" int xlg_bank_fft_profile_read(xlg_group *g, xlg_bank_fft_profile *p, int reset) {
  return family_profile_read(g, &xlg_group::bank_fft_prof, p, reset);
}

extern "C" int xlg_spectrum_profile_read(xlg_group *g, xlg_spectrum_profile *p, int reset) {
  return family_profile_read(g, &xlg_group::spec_prof, p, reset);
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

// ---- stage-B launchers of both engines (cascade_stage_b.cuh) ----
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
