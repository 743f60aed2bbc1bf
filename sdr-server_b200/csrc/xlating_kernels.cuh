/*
 * csrc/xlating_kernels.cuh -- sm_90a device code of libxlating_b200.
 *
 * The hot path of the reference is, per client and per output sample k
 * (/root/reference/src/xlating.c:52-83):
 *
 *     y[k] = phase_k * sum_{j<T} x[first + k*D + j] * rev[j]          (complex, fp32)
 *
 * with x the wideband input converted to cf32 (:384-414), rev the reversed
 * band-pass taps (:525-534) and phase_k a float oscillator advanced once per
 * output and renormalised once per call (:70-73).  Per input sample and client
 * this is 4*T/D real FMAs against 8/D output bytes: at the client counts the
 * service is built for it is bound by the FP32 FMA pipe, not by HBM and not by
 * tensor cores (DESIGN.md section 4), so the kernels are organised around
 * register tiling and shared-memory operand reuse:
 *
 *   convert_*        raw cu8/cs8/cs16 block -> cf32 (or Q15) ring in HBM, ONCE per
 *                    block instead of once per client
 *   phase_*          the reference's sequential float (or Q15) oscillator, one
 *                    thread per client, bit-exact (unfused mul/add, exact hypotf)
 *   fir_tile_cf32    the dominant kernel: 32 clients x 128 (or 64, 32, 16) outputs per
 *                    CTA, 4 (or 2, 1) outputs x 8 clients per thread in registers, input tile
 *                    staged with coalesced 8-byte cp.async into a bank-conflict-
 *                    free skewed layout, taps streamed by TMA bulk copies
 *                    (cp.async.bulk + mbarrier, 3 stages)
 *   fir_generic_*    any (T, D, alignment): one warp per 4 outputs, lanes split the
 *                    taps, warp-shuffle reduction; also the Q15 integer path
 *   cascade_*        stage B of two-stage clients: a real-tap decimator over each
 *                    client's stage-A history ring, TMA-staged window, register tile
 *
 * The arithmetic shared with the per-filter drop-in engine (conversions, oscillator
 * recursion, generic FIR warp) lives in xlating_common.cuh.
 *
 * Everything here is written for sm_90a (H100) only.
 */
#pragma once

#include <cuda.h>  // CUtensorMap (type only: the encoder is fetched through cudaGetDriverEntryPoint)
#include <cuda_runtime.h>
#include <stdint.h>

#include "xlating_common.cuh"

namespace xl {

// ---------------------------------------------------------------------------
// device-resident tables
// ---------------------------------------------------------------------------
struct ClientDev {
  long long hist;         // history_offset of the reference (src/xlating.c:29), shared by both paths;
                          // in upsampled samples for a rational client (L > 1)
  long long zero_before;  // cf32 ring: samples with absolute index < this read as 0 (attach point)
  long long qzero_before; // same for the Q15 ring
  float2 phase;           // oscillator (src/xlating.c:36)
  float2 incr;            // (src/xlating.c:37)
  short qph_re, qph_im, qinc_re, qinc_im;  // Q15 oscillator (:39-42)
  int D;                  // decimation (M of a rational client)
  int T;                  // taps_len
  int taps_off;           // float2 offset of rev taps in the natural arena (polyphase branches for L > 1)
  int qtaps_off;          // short2 offset in the Q15 arena
  int out_off;            // complex-sample offset in the per-slot output / phase arenas
  int out_cap;
  int active;
  int kind;               // 0 = generic kernel, 1 = tiled kernel, 2 = split-K, 3 / 4 = polyphase generic / tiled
  int renorm;             // 1 = native behaviour (:73), 0 = AVX behaviour (:336-339)
  int ph_off;             // cf32 oscillator table: phase of EVEN output k lives at phases[ph_off + 32*(k/2)]
  int L;                  // interpolation: the client filters the stream zero-stuffed by L (1 = integer client)
  int poly_off;           // kind 4: branch r's unrotated outputs at scratch[poly_off + r * poly_rowcap + k / L]
  int poly_rowcap;
};

struct SpecSave {
  long long hist;
  float2 phase;
};

// ---------------------------------------------------------------------------
// convert: raw interleaved I,Q scalars -> ring  (src/xlating.c:389-390, 399-400,
// 409-410 for cf32; :418, :425, :432 for Q15).  All conversions are exact.
// ---------------------------------------------------------------------------
template <int FMT>
__global__ void convert_cf32_kernel(const void *__restrict__ raw, float2 *__restrict__ ring,
                                    unsigned mask, long long S, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float2 v;
  if (FMT == 0) {
    uchar2 u = reinterpret_cast<const uchar2 *>(raw)[i];
    v = make_float2(cvt_cu8_f32(u.x), cvt_cu8_f32(u.y));
  } else if (FMT == 1) {
    char2 u = reinterpret_cast<const char2 *>(raw)[i];
    v = make_float2(cvt_cs8_f32(u.x), cvt_cs8_f32(u.y));
  } else {
    short2 u = reinterpret_cast<const short2 *>(raw)[i];
    v = make_float2(cvt_cs16_f32(u.x), cvt_cs16_f32(u.y));
  }
  ring[(unsigned)((unsigned long long)(S + i)) & mask] = v;
}

// The same conversion, two samples per thread and step (one 4- or 8-byte load, one 16-byte store, both
// coalesced across the warp), CV_STEPS steps per thread: 8x fewer CTAs -- one wave even on the 8 SMs of
// the oscillator partition, where the conversion runs so that it never queues behind FIR CTAs.  Needs an even
// sample count, an even stream position and a raw pointer aligned to two samples (the launcher checks).
constexpr int CV_STEPS = 4;
template <int FMT>
__global__ void convert_cf32_vec_kernel(const void *__restrict__ raw, float2 *__restrict__ ring, unsigned mask,
                                        long long S, int n) {
  const int pairs = n >> 1;
  int p = blockIdx.x * (blockDim.x * CV_STEPS) + threadIdx.x;
#pragma unroll
  for (int j = 0; j < CV_STEPS; j++, p += blockDim.x) {
    if (p >= pairs) return;
    float4 v;
    if (FMT == 0) {
      const uchar4 u = reinterpret_cast<const uchar4 *>(raw)[p];
      v = make_float4(cvt_cu8_f32(u.x), cvt_cu8_f32(u.y), cvt_cu8_f32(u.z), cvt_cu8_f32(u.w));
    } else if (FMT == 1) {
      const char4 u = reinterpret_cast<const char4 *>(raw)[p];
      v = make_float4(cvt_cs8_f32(u.x), cvt_cs8_f32(u.y), cvt_cs8_f32(u.z), cvt_cs8_f32(u.w));
    } else {
      const short4 u = reinterpret_cast<const short4 *>(raw)[p];
      v = make_float4(cvt_cs16_f32(u.x), cvt_cs16_f32(u.y), cvt_cs16_f32(u.z), cvt_cs16_f32(u.w));
    }
    const unsigned idx = (unsigned)((unsigned long long)(S + 2ll * p)) & mask;  // even: the pair never straddles the wrap
    *reinterpret_cast<float4 *>(ring + idx) = v;
  }
}

template <int FMT>
__global__ void convert_q15_kernel(const void *__restrict__ raw, short2 *__restrict__ ring,
                                   unsigned mask, long long S, int n) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  short2 v;
  if (FMT == 0) {
    uchar2 u = reinterpret_cast<const uchar2 *>(raw)[i];
    v = make_short2(cvt_cu8_q15(u.x), cvt_cu8_q15(u.y));
  } else if (FMT == 1) {
    char2 u = reinterpret_cast<const char2 *>(raw)[i];
    v = make_short2(cvt_cs8_q15(u.x), cvt_cs8_q15(u.y));
  } else {
    v = reinterpret_cast<const short2 *>(raw)[i];
  }
  ring[(unsigned)((unsigned long long)(S + i)) & mask] = v;
}

// ---------------------------------------------------------------------------
// oscillator pre-pass (the recursion itself: xlating_common.cuh).  One thread per
// client replays it and stores the phase of every (even) output of this block.
// ---------------------------------------------------------------------------
constexpr int P_THREADS = 32;   // one warp = one table group of 32 clients
constexpr int P_QTHREADS = 64;  // Q15 variant (one thread per client)

// Oscillator table layout: clients are taken in "table order" (tile classes first,
// in the order the tiled kernel walks them, then the generic clients), 32 per
// group; group g stores phase(2m, lane) at phases[base_g + 32*m + lane].  Lane l of
// the warp owns client order[32*g + l] and walks its recursion sequentially -- the
// dependent chain (2 dependent fp32 ops per output) is the
// only thing on the critical path: the per-output store is one coalesced 256-byte
// line for the whole warp, there is no shared memory, no barrier.  (Earlier
// versions stored [client][k] rows -- first uncoalesced, then through a shared-
// memory transpose with helper warps -- and spent 2/3 of their time on that; and
// storing every output instead of every second one ran at 16.7 cycles/output,
// because a lone warp can only keep ~32 stores in flight.)
__global__ void __launch_bounds__(P_THREADS)
phase_cf32_kernel(ClientDev *__restrict__ cl, const int *__restrict__ order, BlkInfo *__restrict__ blk,
                  float2 *__restrict__ phases, float2 *__restrict__ endph, SpecSave *__restrict__ save, long long S,
                  int n_in) {
  const int c = order[blockIdx.x * 32 + threadIdx.x];
  if (c < 0) return;
  ClientDev *d = cl + c;
  if (!d->active) return;
  if (save != nullptr) {  // a speculative run (the next block's pre-pass, launched early): keep what it overwrites
    save[c].hist = d->hist;
    save[c].phase = d->phase;
  }
  const int D = d->D;
  // stream positions in the client's (upsampled) coordinates: identical integers for L = 1
  const long long Su = S * d->L, Eu = (S + n_in) * d->L;
  const long long first = Su - d->hist;
  const int n_out = outputs_of_call(first, Su, (int)(Eu - Su), d->T, D, d->out_cap);
  BlkInfo b;
  b.first = first;
  b.n_out = n_out;
  b.pad_ = 0;
  blk[c] = b;
  const float2 after = osc_chain_cf32<32>(d->phase, d->incr, phases + d->ph_off, n_out, d->renorm);
  d->phase = after;
  if (endph != nullptr) endph[c] = after;  // XLG_TRACK_STATE: the oscillator after this block, per client id
  d->hist = Eu - (first + (long long)n_out * D);  // src/xlating.c:76
}

// undo a speculative pre-pass that guessed the wrong block length
__global__ void restore_clients_kernel(ClientDev *__restrict__ cl, const SpecSave *__restrict__ save, int n) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n || !cl[c].active) return;
  cl[c].hist = save[c].hist;
  cl[c].phase = save[c].phase;
}

__global__ void __launch_bounds__(P_QTHREADS)
phase_q15_kernel(ClientDev *__restrict__ cl, int n_clients, BlkInfo *__restrict__ blk,
                 short2 *__restrict__ qphases, long long S, int n_in) {
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n_clients) return;
  ClientDev *d = cl + c;
  if (!d->active) return;
  const long long first = S - d->hist;
  const int n_out = outputs_of_call(first, S, n_in, d->T, d->D, d->out_cap);
  BlkInfo b;
  b.first = first;
  b.n_out = n_out;
  b.pad_ = 0;
  blk[c] = b;
  const short2 ph = osc_chain_q15(make_short2(d->qph_re, d->qph_im), make_short2(d->qinc_re, d->qinc_im),
                                  qphases + d->out_off, n_out);
  d->qph_re = ph.x;
  d->qph_im = ph.y;
  d->hist = (S + n_in) - (first + (long long)n_out * d->D);  // src/xlating.c:133
}

// ---------------------------------------------------------------------------
// generic FIR: any T, D, alignment, attach point.  CTA = 8 warps = 32 consecutive
// outputs of one client; each warp owns 4 consecutive outputs, its lanes stride
// over the taps (coalesced float2 loads of ring and taps through L1/L2) and the
// partial dot products are combined with warp shuffles (xlating_common.cuh).
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(G_THREADS)
fir_generic_cf32_kernel(const ClientDev *__restrict__ cl, const BlkInfo *__restrict__ blk,
                        const float2 *__restrict__ ring, unsigned mask,
                        const float2 *__restrict__ taps, const float2 *__restrict__ phases,
                        float2 *__restrict__ out) {
  const int c = blockIdx.y;
  const ClientDev *d = cl + c;
  if (!d->active || d->kind != 0) return;
  const BlkInfo b = blk[c];
  const int kbase = blockIdx.x * G_OPC;
  if (kbase >= b.n_out) return;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int k0 = kbase + warp * G_OPW;
  const float2 mine = fir_warp_cf32(ring, mask, d->zero_before, taps + d->taps_off, d->T, d->D,
                                    b.first + (long long)k0 * d->D, lane);
  const int k = k0 + lane;
  if (lane < G_OPW && k < b.n_out) {
    float2 ph = phases[d->ph_off + (size_t)(k >> 1) * 32];
    if (k & 1) ph = cmul_unfused(ph, d->incr);     // odd outputs: one step from the stored even phase
    out[d->out_off + k] = cmul_unfused(mine, ph);  // src/xlating.c:70
  }
}

// ---------------------------------------------------------------------------
// rational L/M client, any state (kind 3).  The client is the reference filter with
// decimation M fed the zero-stuffed stream u[L*n] = x[n], u[m] = 0 otherwise.  Output
// k's upsampled window starts at w = first + k*M; with r = (-w) mod L and n0 = (w + r)/L
// only the taps rev[r + t*L] meet nonzero samples:
//     y[k] = phase_k * sum_{t < Tb} x[n0 + t] * P[r][t],   P[r][t] = rev[r + t*L] (0 past T),
// Tb = ceil(T / L) taps per output instead of T.  Outputs k and k + L share the branch
// r and their inputs lie M samples apart, so a warp takes G_OPW outputs k0 + i*L and
// runs the integer generic FIR on branch r with decimation M.  Warp q of a client
// serves residue rho = q / groups (outputs rho, rho + L, ...), output group q % groups.
// A padding tap reads one sample past the window; it is finite and weighted by zero.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(G_THREADS)
fir_poly_generic_cf32_kernel(const ClientDev *__restrict__ cl, const int *__restrict__ ids,
                             const BlkInfo *__restrict__ blk, const float2 *__restrict__ ring, unsigned mask,
                             const float2 *__restrict__ taps, const float2 *__restrict__ phases,
                             float2 *__restrict__ out) {
  const int c = ids[blockIdx.y];  // the kind-3 clients only
  const ClientDev *d = cl + c;
  const BlkInfo b = blk[c];
  const int L = d->L, M = d->D;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int per = (b.n_out + L - 1) / L;           // outputs of residue 0 (the most of any residue)
  const int groups = (per + G_OPW - 1) / G_OPW;
  const int q = blockIdx.x * (G_THREADS / 32) + warp;
  if (q >= min(L, b.n_out) * groups) return;       // warp-uniform
  const int rho = q / groups;
  const int k0 = rho + (q - rho * groups) * G_OPW * L;
  if (k0 >= b.n_out) return;
  long long n0;
  const int r = poly_branch(b.first + (long long)k0 * M, L, &n0);
  const int Tb = (d->T + L - 1) / L;
  const float2 mine = fir_warp_cf32(ring, mask, d->zero_before, taps + d->taps_off + (size_t)r * Tb, Tb, M, n0, lane);
  const int k = k0 + lane * L;
  if (lane < G_OPW && k < b.n_out) {
    float2 ph = phases[d->ph_off + (size_t)(k >> 1) * 32];
    if (k & 1) ph = cmul_unfused(ph, d->incr);
    out[d->out_off + k] = cmul_unfused(mine, ph);
  }
}

// ---------------------------------------------------------------------------
// rational L/M clients of a tiled class (kind 4): clients with identical (L, M, T, window
// alignment) and gcd(L, M) = 1.  In a block every branch r serves the outputs
// k = rho_r + j*L (rho_r: the k < L whose window start -(first + k*M) is r mod L) from inputs
// x[n0_r + j*M + t], t < Tb: an integer decimator with decimation M over the Tb taps of
// branch r.  The host launches fir_tile_cf32_kernel with one class per branch (the branch's
// taps packed for its 32-client groups, the class's BlkInfo at blk[class], phase 1 + 0i), which
// leaves y_r[j] unrotated at scratch[poly_off + r * poly_rowcap + j]; this kernel rotates every
// output with the client's oscillator and puts it at k.  Same arithmetic as the polyphase
// generic kernel up to the order of the additions.
// ---------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
poly_tile_place_cf32_kernel(const ClientDev *__restrict__ cl, const int *__restrict__ ids,
                            const BlkInfo *__restrict__ blk, const float2 *__restrict__ scratch,
                            const float2 *__restrict__ phases, float2 *__restrict__ out) {
  const int c = ids[blockIdx.y];  // the kind-4 clients only
  const ClientDev *d = cl + c;
  const BlkInfo b = blk[c];
  const int k = blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= b.n_out) return;
  const int L = d->L;
  const long long w = b.first + (long long)k * d->D;
  const int r = (int)((((-w) % L) + L) % L);
  const float2 y = scratch[d->poly_off + (size_t)r * d->poly_rowcap + k / L];
  float2 ph = phases[d->ph_off + (size_t)(k >> 1) * 32];
  if (k & 1) ph = cmul_unfused(ph, d->incr);
  out[d->out_off + k] = cmul_unfused(y, ph);
}

__global__ void __launch_bounds__(G_THREADS)
fir_generic_q15_kernel(const ClientDev *__restrict__ cl, const BlkInfo *__restrict__ blk,
                       const short2 *__restrict__ ring, unsigned mask,
                       const short2 *__restrict__ qtaps, const short2 *__restrict__ qphases,
                       short2 *__restrict__ out) {
  const int c = blockIdx.y;
  const ClientDev *d = cl + c;
  if (!d->active) return;
  const BlkInfo b = blk[c];
  const int kbase = blockIdx.x * G_OPC;
  if (kbase >= b.n_out) return;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int k0 = kbase + warp * G_OPW;
  const short2 mine = fir_warp_q15(ring, mask, d->qzero_before, qtaps + d->qtaps_off, d->T, d->D,
                                   b.first + (long long)k0 * d->D, lane);
  const int k = k0 + lane;
  if (lane < G_OPW && k < b.n_out)
    out[d->out_off + k] = rotate_q15(mine, qphases[d->out_off + k]);  // src/xlating.c:121-124
}

// ---------------------------------------------------------------------------
// tiled multi-client FIR (the dominant kernel)
// ---------------------------------------------------------------------------
constexpr int T_RC = 8;              // clients per thread
constexpr int T_CG = 32;             // clients per CTA
#ifndef XL_TILE_JC
#define XL_TILE_JC 32
#endif
#ifndef XL_TILE_STAGES
#define XL_TILE_STAGES 3
#endif
#ifndef XL_TILE_MINCTAS
#define XL_TILE_MINCTAS 4
#endif
constexpr int T_JC = XL_TILE_JC;     // flat taps per TMA chunk (multiple of 8)
constexpr int T_STAGES = XL_TILE_STAGES;
#ifndef XL_TILE_UNROLL
#define XL_TILE_UNROLL 8
#endif
constexpr int T_UNROLL = XL_TILE_UNROLL;  // taps per unrolled inner-loop body (L is a multiple of 8)
constexpr int T_CHUNK_F2 = T_JC * T_CG;       // float2 per chunk (1024)
constexpr int T_CHUNK_BYTES = T_CHUNK_F2 * 8;  // 8 KiB
constexpr int T_SMEM_FIXED = T_STAGES * T_CHUNK_BYTES + ((2 * T_STAGES + 1) * 8 + 63) / 64 * 64;  // tap stages + mbarriers
constexpr int T_MAX_CLASSES = 36;    // (D, T) classes per launch: 36 x 104 bytes stays inside the classic 4 KiB parameter space
constexpr int T_TRACE_REC = 6;       // long long per CTA in the XLATING_B200_TRACE timeline
constexpr int T_TRACE_LAUNCHES = 16; // launches kept (ring)
constexpr int T_TRACE_CTAS = 4096;   // CTAs recorded per launch

// Shape of the tile a CTA computes.  LO = number of output lanes in a warp, RK =
// outputs per thread; the thread tile is RK outputs x 8 clients, the CTA tile
// (LO*RK) outputs x 32 clients.  With LO = 16, lane = (h, o), o = lane & 15 the output
// column, h = lane >> 4 the client half; warp = LO*RK outputs x 16 clients, 2 warps per
// output set.  Both half-warps read the same x (one shared-memory wavefront instead of two).
// OS = output sets: OS groups of those warps take consecutive LO*RK-output ranges of
// one input tile and share its tap stages.  OS = 2 with RK = 4 (128 outputs, 4 warps,
// 72 KB at D = 42) runs 3 CTAs per SM with 3 warps on every scheduler, and a CTA that is
// staging or storing leaves 2 warps per scheduler to the others; 2-warp CTAs at 3 per
// SM leave two of the four schedulers a single warp (DESIGN.md section 5).  RK = 4, 2
// or 1 with OS = 1 trade tile size for more (smaller) CTAs when there are few clients
// or few outputs per block (e.g. 64 clients at 250 ksps: 26 CTAs with RK = 4 cannot
// occupy 132 SMs).
template <int LO, int RK, int OS = 1>
struct TileShape {
  static constexpr int kHalves = 32 / LO;                    // client halves per warp
  static constexpr int kWarpClients = kHalves * T_RC;        // 8 or 16
  static constexpr int kClientWarps = T_CG / kWarpClients;   // warps that cover the 32 clients: 4 or 2
  static constexpr int kWarps = kClientWarps * OS;           // OS output sets of them
  static constexpr int kThreads = kWarps * 32;
  static constexpr int kKT = LO * RK * OS;                   // outputs per CTA
  // CTAs per SM the register budget is set for
  static constexpr int kMinCtas = OS == 2 ? 3 : XL_TILE_MINCTAS;
};

// One class = clients with identical (D, T, window alignment).  "Flat" tap index:
// tap j = q*D + r lives at f = q*Dp + r with Dp = D rounded up to odd, so that a
// thread's window x[(k*D + j)] sits at shared address k*Dp + f: consecutive f for
// the inner loop (immediate offsets when unrolled) and an odd stride between the
// lanes' outputs (conflict-free 64-bit shared loads).  Pad slots hold zero taps.
struct TileClass {
  long long first;     // absolute index of output 0's window start (all members)
  long long taps_off;  // float2 offset into the packed tile-tap arena: [group][L][32]
  int n_out;
  int D, Dp, L;        // L = flat length, multiple of 8
  int n_groups;        // CTA groups of 32 clients
  int tiles;           // ceil(n_out / KT)
  int cta_begin;       // first CTA of this class in the launch
  int members_off;     // into the member table: output row offset or -1, 32 per group
  int xs_len;          // float2 in the input tile: (KT-1)*Dp + L
  int ph_stride;       // float2 between the oscillator tables of consecutive client groups
  int n_members;       // real clients in the class (the last group may be partly padding)
  int natural;         // 1: Dp == D, the input tile is ONE contiguous TMA bulk copy (see kernel)
  long long ph_base;   // float2 offset of (group 0, output 0, lane 0) in the oscillator table
  // long-filter (split-K) classes only:
  long long part_off;  // float2 offset of this class in the partial-sum buffer
  int nseg;            // tap segments of W_JS flat taps
  int kpad;            // outputs rounded up to the tile size (row count of the partial buffer)
  int nslab;           // partial-sum slabs the reduction adds: nseg, or ksplit for the pipelined kernel
  int ksplit;          // pipelined long-filter kernel: CTAs along the tap axis per (group, tile)
  int seg_per;         // ... and consecutive segments each of them walks
  int tmap_w;          // long4 with a TMA tensor map for the input strips: width of the map's inner dimension (0 = none)
};

struct TileLaunch {
  int n_classes;
  int pad_;
  TileClass cls[T_MAX_CLASSES];
};
static_assert(sizeof(TileLaunch) <= 4000, "TileLaunch is passed as a __grid_constant__ kernel parameter");

// class of CTA `bid`: the last class whose cta_begin <= bid (classes are laid out in launch order)
__device__ __forceinline__ int class_of_cta(const TileLaunch &P, int bid) {
  int lo = 0, hi = P.n_classes - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    if (P.cls[mid].cta_begin <= bid)
      lo = mid;
    else
      hi = mid - 1;
  }
  return lo;
}

__device__ __forceinline__ void mbar_init(uint64_t *bar, unsigned count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t *bar, unsigned bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t *bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t *bar, unsigned parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(smem_u32(bar)),
      "r"(parity)
      : "memory");
}
// TMA 1-D bulk copy global -> shared, completion signalled on an mbarrier
__device__ __forceinline__ void tma_bulk_g2s(void *dst, const void *src, unsigned bytes, uint64_t *bar) {
  asm volatile(
      "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst)),
      "l"(src), "r"(bytes), "r"(smem_u32(bar))
      : "memory");
}
// TMA 2-D tiled copy global -> shared through a tensor map (one instruction moves a whole box of rows)
__device__ __forceinline__ void tma_tensor2d_g2s(void *dst, const CUtensorMap *map, int c0, int c1, uint64_t *bar) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];" ::"r"(
          smem_u32(dst)),
      "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(smem_u32(bar))
      : "memory");
}
__device__ __forceinline__ void cp_async_8(void *dst, const void *src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(smem_u32(dst)), "l"(src) : "memory");
}

template <int LO, int RK, int OS>
__global__ void __launch_bounds__(TileShape<LO, RK, OS>::kThreads, TileShape<LO, RK, OS>::kMinCtas)
fir_tile_cf32_kernel(const __grid_constant__ TileLaunch P, const float2 *__restrict__ ring, unsigned mask,
                     const float2 *__restrict__ tile_taps, const int *__restrict__ member_off,
                     const int *__restrict__ member_cid, const float2 *__restrict__ member_incr,
                     const BlkInfo *__restrict__ blk, const float2 *__restrict__ phases,
                     float2 *__restrict__ out, long long *__restrict__ trace) {
  using S = TileShape<LO, RK, OS>;
  // optional per-CTA timeline (XLATING_B200_TRACE=1): start, staged, loop done, end
  long long tr0 = 0, tr1 = 0, tr2 = 0;
  if (trace != nullptr) tr0 = clock64();
  constexpr int NT = S::kThreads;
  constexpr int KT = S::kKT;
  extern __shared__ __align__(128) unsigned char smem[];
  float2 *ts = reinterpret_cast<float2 *>(smem);
  uint64_t *bars = reinterpret_cast<uint64_t *>(smem + T_STAGES * T_CHUNK_BYTES);
  float2 *xs = reinterpret_cast<float2 *>(smem + T_SMEM_FIXED);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int o = lane & (LO - 1);   // output column of this lane
  const int h = lane / LO;         // client half of this lane
  const int cbase = (warp % S::kClientWarps) * S::kWarpClients + h * T_RC;  // first of this thread's 8 clients in the group
  const int obase = (warp / S::kClientWarps) * (LO * RK);                  // first output of this warp's output set

  // which class / client group / output tile is this CTA?
  const int ci = class_of_cta(P, (int)blockIdx.x);
  const TileClass &K = P.cls[ci];
  const int local = (int)blockIdx.x - K.cta_begin;
  const int grp = local / K.tiles;
  const int tile = local - grp * K.tiles;
  const int k0 = tile * KT;
  const int D = K.D, Dp = K.Dp, L = K.L;
  const int nchunks = (L + T_JC - 1) / T_JC;

  // bars[0..S): "stage is full" (TMA transaction count); bars[S..2S): "stage is free"
  // (one arrival per warp).  The warps of a CTA never wait for each other inside the
  // tap loop: a warp releases a stage and moves on; the producer thread refills the
  // stage of the PREVIOUS chunk, which every warp has normally left long ago.
  if (tid == 0) {
    for (int s = 0; s < T_STAGES; s++) {
      mbar_init(&bars[s], 1);
      mbar_init(&bars[T_STAGES + s], S::kWarps);
    }
    mbar_init(&bars[2 * T_STAGES], 1);  // input tile landed (natural layout)
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();

  const float2 *gt = tile_taps + K.taps_off + (long long)grp * L * T_CG;
  if (tid == 0) {
    for (int s = 0; s < T_STAGES && s < nchunks; s++) {
      const unsigned bytes = (unsigned)min(T_JC, L - s * T_JC) * T_CG * 8u;
      mbar_expect_tx(&bars[s], bytes);
      tma_bulk_g2s(ts + s * T_CHUNK_F2, gt + (long long)s * T_CHUNK_F2, bytes, &bars[s]);
    }
  }

  // stage the input tile.
  //  natural layout (Dp == D): the tile is a contiguous range of the ring, fetched by ONE
  //    TMA bulk copy (two if it wraps) that costs no issue slots -- the per-element path
  //    below loses issue arbitration to co-resident FMA warps and took 6-16 k cycles.
  //    Used when gcd(D, 16) <= 2: the lane stride D is then at most 2-way bank
  //    conflicting for the 16 output lanes of a half-warp.
  //  skewed layout (Dp = D|1): row r = D consecutive samples stored with pitch Dp,
  //    coalesced 8-byte cp.async per element; conflict-free for any D.
  if (K.natural) {
    const long long w0 = K.first + (long long)k0 * D;
    const unsigned odd = (unsigned)(w0 & 1);  // bulk copies need 16-byte alignment: start one sample early
    if (tid == 0) {
      const unsigned n = ((unsigned)K.xs_len + odd + 1u) & ~1u;
      const unsigned idx = (unsigned)((unsigned long long)(w0 - odd)) & mask;
      const unsigned n1 = min(n, mask + 1u - idx);
      mbar_expect_tx(&bars[2 * T_STAGES], n * 8u);
      tma_bulk_g2s(xs, ring + idx, n1 * 8u, &bars[2 * T_STAGES]);
      if (n1 < n) tma_bulk_g2s(xs + n1, ring, (n - n1) * 8u, &bars[2 * T_STAGES]);
    }
    xs += odd;
  } else {
    const long long w0 = K.first + (long long)k0 * D;
    int row = tid / Dp, col = tid - row * Dp;
    const int drow = NT / Dp, dcol = NT - drow * Dp;
    for (int e = tid; e < K.xs_len; e += NT) {
      if (col < D) {
        const long long ab = w0 + (long long)row * D + col;
        cp_async_8(xs + e, ring + ((unsigned)((unsigned long long)ab) & mask));
      } else {
        xs[e] = make_float2(0.f, 0.f);
      }
      row += drow;
      col += dcol;
      if (col >= Dp) {
        col -= Dp;
        row++;
      }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  }

  // This thread's 8 clients form a subgroup with ONE window alignment: clients of a
  // class share (D, T) but may have been attached at different stream positions, so
  // their windows start delta = first_c - K.first samples (0 <= delta < D) into the
  // tile and they may produce one output less.  Both come from the oscillator
  // pre-pass's per-block record of the subgroup's first client (-1 = all padding).
  int delta = 0, n_out_sub = 0;
  {
    const int cid0 = __ldg(member_cid + K.members_off + grp * T_CG + cbase);
    if (cid0 >= 0) {
      const BlkInfo b = blk[cid0];
      delta = (int)(b.first - K.first);
      n_out_sub = b.n_out;
    }
  }
  // a warp whose subgroups are all padding has nothing to compute (it still takes
  // part in the barriers)
  const bool warp_active = __any_sync(0xffffffffu, n_out_sub > 0);

  if (K.natural) {
    mbar_wait(&bars[2 * T_STAGES], 0);
  } else {
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncthreads();
  }
  if (trace != nullptr) tr1 = clock64();

  float2 acc[RK][T_RC];
#pragma unroll
  for (int i = 0; i < RK; i++)
#pragma unroll
    for (int c = 0; c < T_RC; c++) acc[i][c] = make_float2(0.f, 0.f);

  const float2 *xb[RK];
#pragma unroll
  for (int i = 0; i < RK; i++) xb[i] = xs + (obase + o + LO * i) * Dp + delta;

  for (int ch = 0; ch < nchunks; ch++) {
    const int s = ch % T_STAGES;
    mbar_wait(&bars[s], (unsigned)((ch / T_STAGES) & 1));
    if (warp_active) {
      const int len = min(T_JC, L - ch * T_JC);
      const float4 *tp = reinterpret_cast<const float4 *>(ts + s * T_CHUNK_F2 + cbase);
      const int fbase = ch * T_JC;
#pragma unroll 1
      for (int f = 0; f < len; f += T_UNROLL) {
#pragma unroll
        for (int u = 0; u < T_UNROLL; u++) {
          float2 x[RK];
#pragma unroll
          for (int i = 0; i < RK; i++) x[i] = xb[i][fbase + f + u];
          float4 tq[T_RC / 2];
#pragma unroll
          for (int q = 0; q < T_RC / 2; q++) tq[q] = tp[(f + u) * (T_CG / 2) + q];
#pragma unroll
          for (int i = 0; i < RK; i++) {
#pragma unroll
            for (int q = 0; q < T_RC / 2; q++) {
              float2 &a0 = acc[i][2 * q], &a1 = acc[i][2 * q + 1];
              a0.x = fmaf(x[i].x, tq[q].x, a0.x);
              a0.x = fmaf(-x[i].y, tq[q].y, a0.x);
              a0.y = fmaf(x[i].x, tq[q].y, a0.y);
              a0.y = fmaf(x[i].y, tq[q].x, a0.y);
              a1.x = fmaf(x[i].x, tq[q].z, a1.x);
              a1.x = fmaf(-x[i].y, tq[q].w, a1.x);
              a1.y = fmaf(x[i].x, tq[q].w, a1.y);
              a1.y = fmaf(x[i].y, tq[q].z, a1.y);
            }
          }
        }
      }
    }
    __syncwarp();
    if (lane == 0) mbar_arrive(&bars[T_STAGES + s]);  // this warp is done with stage s
    if (tid == 0 && ch >= 1) {
      const int pc = ch - 1, nx = pc + T_STAGES;
      if (nx < nchunks) {
        const int ps = pc % T_STAGES;
        mbar_wait(&bars[T_STAGES + ps], (unsigned)((pc / T_STAGES) & 1));  // all warps left chunk pc
        const unsigned bytes = (unsigned)min(T_JC, L - nx * T_JC) * T_CG * 8u;
        mbar_expect_tx(&bars[ps], bytes);
        tma_bulk_g2s(ts + ps * T_CHUNK_F2, gt + (long long)nx * T_CHUNK_F2, bytes, &bars[ps]);
      }
    }
  }

  if (trace != nullptr) tr2 = clock64();
  // epilogue: derotate with the pre-computed oscillator and store (coalesced in k).
  // The oscillator table is [k][32 clients]: this thread's 8 clients are 64
  // contiguous bytes per output.  The loads of two outputs (and the clients' output
  // row offsets) are in flight together before the first use.
  if (n_out_sub > 0) {
    int off[T_RC];
    float4 inc[T_RC / 2];  // oscillator steps of the 8 clients, (re, im) pairs
    {
      const int *mo = member_off + K.members_off + grp * T_CG + cbase;
#pragma unroll
      for (int c = 0; c < T_RC; c++) off[c] = __ldg(mo + c);  // -1 = padding slot
      const float4 *mi = reinterpret_cast<const float4 *>(member_incr + K.members_off + grp * T_CG + cbase);
#pragma unroll
      for (int q = 0; q < T_RC / 2; q++) inc[q] = __ldg(mi + q);
    }
    // only even outputs' phases are tabulated; an odd output advances the stored
    // phase by one step, exactly as the reference's recursion does (src/xlating.c:71).
    // k = k0 + obase + o + LO*i has the parity of o (k0, obase and LO are even): uniform per lane.
    const bool odd = (o & 1) != 0;
    const float4 *pt =
        reinterpret_cast<const float4 *>(phases + K.ph_base + (long long)grp * K.ph_stride + cbase);
    constexpr int EB = RK >= 2 ? 2 : 1;  // outputs whose table loads are in flight together
#pragma unroll
    for (int i2 = 0; i2 < RK; i2 += EB) {
      float4 ph[EB][T_RC / 2];
#pragma unroll
      for (int ii = 0; ii < EB; ii++) {
        const int k = min(k0 + obase + o + LO * (i2 + ii), n_out_sub - 1);  // clamped: always a valid row
#pragma unroll
        for (int q = 0; q < T_RC / 2; q++) ph[ii][q] = __ldg(pt + (size_t)(k >> 1) * 16 + q);
      }
#pragma unroll
      for (int ii = 0; ii < EB; ii++) {
        const int i = i2 + ii;
        const int k = k0 + obase + o + LO * i;
        if (k >= n_out_sub) continue;
#pragma unroll
        for (int q = 0; q < T_RC / 2; q++) {
          float2 p0 = make_float2(ph[ii][q].x, ph[ii][q].y), p1 = make_float2(ph[ii][q].z, ph[ii][q].w);
          if (odd) {
            p0 = cmul_unfused(p0, make_float2(inc[q].x, inc[q].y));
            p1 = cmul_unfused(p1, make_float2(inc[q].z, inc[q].w));
          }
          if (off[2 * q] >= 0) out[off[2 * q] + k] = cmul_unfused(acc[i][2 * q], p0);  // src/xlating.c:70
          if (off[2 * q + 1] >= 0) out[off[2 * q + 1] + k] = cmul_unfused(acc[i][2 * q + 1], p1);
        }
      }
    }
  }
  if (trace != nullptr && tid == 0) {
    long long *t = trace + T_TRACE_REC * (size_t)blockIdx.x;
    unsigned smid, wid;
    asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
    asm volatile("mov.u32 %0, %%warpid;" : "=r"(wid));
    unsigned long long gt;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(gt));
    t[0] = tr0;
    t[1] = tr1;
    t[2] = (tr2 & 0x0000ffffffffffffll) | ((long long)smid << 48);  // smid in the top 16 bits
    t[3] = clock64();
    t[4] = (long long)gt;                                          // ns at the END of the CTA
    t[5] = ((long long)ci << 32) | ((long long)wid << 16) | (long long)(L & 0xffff);
  }
}

// ---------------------------------------------------------------------------
// long filters: split-K FIR + ordered reduction
//
// BASELINE configs[4] (61.44 Msps -> 48 ksps) gives D = 1280 and T = 15419 taps with
// only ~52 outputs per 256 KiB block: the window of ONE output (123 KB of cf32) does
// not fit the tiled kernel's shared-memory tile, and (outputs x clients) alone is far
// too little parallelism for 132 SMs.  So the tap range is cut into segments of W_JS
// taps, CTAs along the tap axis write partial sums to [slab][group][output][32 clients]
// (coalesced), and fir_long_reduce_kernel adds the slabs IN ORDER (deterministic),
// derotates with the oscillator table and stores.  Same arithmetic as the other kernels
// up to the order of the fp32 additions.  Two kernels compute the partial sums, both
// with a 7-output x 8-client register tile per thread:
//   * fir_long4 when every long class of the launch has even D (the strips can then be
//     fetched 16-byte aligned by TMA bulk copies);
//   * fir_long2 otherwise (it falls back to 8-byte cp.async for unaligned strips).
// ---------------------------------------------------------------------------
constexpr int W_JS = 128;             // taps per segment
constexpr int W_JSP = W_JS + 2;       // strip pitch: 16-byte aligned rows, 2-way conflicts at most

// ---------------------------------------------------------------------------
// fir_long2: one CTA per (segment, client group, 56-output tile):
//   * the x "strips" of the tile's 56 outputs for this segment (each strip contiguous in
//     the ring) arrive by one TMA bulk copy per output row when the strips are 16-byte
//     aligned (even D and window start), else by 8-byte cp.async; the segment's taps
//     (W_JS x 32 clients, 32 KiB) by one TMA bulk copy;
//   * 4 warps per CTA split the 128-tap segment four ways (32 taps each) and add their
//     partial sums through shared memory in a fixed order -- two CTAs = 8 warps per SM
//     (one warp per scheduler leaves the FMA pipe half idle);
//   * a 56-output tile (8 output lanes x 7 outputs per thread; lane = (client octet,
//     output column), a warp covers all 32 clients): BASELINE configs[4] produces 51-52
//     outputs per 256 KiB block, 7 % of the tile is waste; per tap a thread issues 7 + 4
//     shared loads for 224 FFMA.
// ---------------------------------------------------------------------------
constexpr int W2_LO = 8;               // output lanes per warp
constexpr int W2_RK = 7;               // outputs per thread
constexpr int W2_KT = W2_LO * W2_RK;   // 56 outputs per CTA
constexpr int W2_WARPS = 4;
constexpr int W2_THREADS = 32 * W2_WARPS;
constexpr int W2_JW = W_JS / W2_WARPS;  // taps per warp (32)
constexpr int W2_SMEM = W_JS * T_CG * 8 + 64 + W2_KT * W_JSP * 8;  // 32 KiB taps + barrier + 57 KiB strips
static_assert((W2_WARPS - 1) * 32 * W2_RK * T_RC * 2 * 4 <= W2_KT * W_JSP * 8, "reduction scratch reuses the strips");

__global__ void __launch_bounds__(W2_THREADS, 2)
fir_long2_cf32_kernel(const __grid_constant__ TileLaunch P, const float2 *__restrict__ ring, unsigned mask,
                      const float2 *__restrict__ tile_taps, float2 *__restrict__ partial) {
  extern __shared__ __align__(128) unsigned char smem[];
  float2 *ts = reinterpret_cast<float2 *>(smem);
  uint64_t *bar = reinterpret_cast<uint64_t *>(smem + W_JS * T_CG * 8);
  float2 *xs = reinterpret_cast<float2 *>(smem + W_JS * T_CG * 8 + 64);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int o = lane & (W2_LO - 1), h = lane / W2_LO;  // output column, client octet
  const int cbase = h * T_RC;

  const int ci = class_of_cta(P, (int)blockIdx.x);
  const TileClass &K = P.cls[ci];
  const int local = (int)blockIdx.x - K.cta_begin;
  const int seg = local % K.nseg;
  const int rest = local / K.nseg;
  const int tile = rest % K.tiles;
  const int grp = rest / K.tiles;
  const int k0 = tile * W2_KT;
  const int f0 = seg * W_JS;
  const int len = min(W_JS, K.L - f0);  // multiple of 8
  const int D = K.D;

  if (tid == 0) {
    mbar_init(bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();

  const long long w0 = K.first + (long long)k0 * D + f0;  // first sample of strip 0
  const bool aligned = ((K.first | (long long)D) & 1) == 0;  // f0 and k0*D are even then
  const unsigned strip_bytes = (unsigned)len * 8u;
  if (tid == 0) {
    const unsigned tap_bytes = (unsigned)len * T_CG * 8u;
    mbar_expect_tx(bar, tap_bytes + (aligned ? W2_KT * strip_bytes : 0u));
    tma_bulk_g2s(ts, tile_taps + K.taps_off + ((long long)grp * K.L + f0) * T_CG, tap_bytes, bar);
  }
  __syncthreads();  // expect_tx is posted before any strip copy can complete
  if (aligned) {
    if (tid < W2_KT) {  // one strip per thread: x[(k0 + tid)*D + f0 .. + len), contiguous in the ring
      const unsigned idx = (unsigned)((unsigned long long)(w0 + (long long)tid * D)) & mask;
      const unsigned n1 = min((unsigned)len, mask + 1u - idx);
      tma_bulk_g2s(xs + tid * W_JSP, ring + idx, n1 * 8u, bar);
      if (n1 < (unsigned)len) tma_bulk_g2s(xs + tid * W_JSP + n1, ring, ((unsigned)len - n1) * 8u, bar);
    }
  } else {
    for (int e = tid; e < W2_KT * W_JS; e += W2_THREADS) {
      const int k = e / W_JS, f = e - k * W_JS;
      if (f < len) {
        const long long ab = w0 + (long long)k * D + f;
        cp_async_8(xs + k * W_JSP + f, ring + ((unsigned)((unsigned long long)ab) & mask));
      }
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
    asm volatile("cp.async.wait_group 0;" ::: "memory");
    __syncthreads();
  }
  mbar_wait(bar, 0);

  float2 acc[W2_RK][T_RC];
#pragma unroll
  for (int i = 0; i < W2_RK; i++)
#pragma unroll
    for (int c = 0; c < T_RC; c++) acc[i][c] = make_float2(0.f, 0.f);
  const float2 *xb[W2_RK];
#pragma unroll
  for (int i = 0; i < W2_RK; i++) xb[i] = xs + (o + W2_LO * i) * W_JSP;
  const float4 *tp = reinterpret_cast<const float4 *>(ts + cbase);

  const bool group_active = grp * T_CG < K.n_members;
  const int f_end = min(len, (warp + 1) * W2_JW);
  if (group_active) {
#pragma unroll 1
    for (int f = warp * W2_JW; f < f_end; f += T_UNROLL) {
#pragma unroll
      for (int u = 0; u < T_UNROLL; u++) {
        float2 x[W2_RK];
        float4 tq[T_RC / 2];
#pragma unroll
        for (int i = 0; i < W2_RK; i++) x[i] = xb[i][f + u];
#pragma unroll
        for (int q = 0; q < T_RC / 2; q++) tq[q] = tp[(f + u) * (T_CG / 2) + q];
#pragma unroll
        for (int i = 0; i < W2_RK; i++) {
#pragma unroll
          for (int q = 0; q < T_RC / 2; q++) {
            float2 &a0 = acc[i][2 * q], &a1 = acc[i][2 * q + 1];
            a0.x = fmaf(x[i].x, tq[q].x, a0.x);
            a0.x = fmaf(-x[i].y, tq[q].y, a0.x);
            a0.y = fmaf(x[i].x, tq[q].y, a0.y);
            a0.y = fmaf(x[i].y, tq[q].x, a0.y);
            a1.x = fmaf(x[i].x, tq[q].z, a1.x);
            a1.x = fmaf(-x[i].y, tq[q].w, a1.x);
            a1.y = fmaf(x[i].x, tq[q].w, a1.y);
            a1.y = fmaf(x[i].y, tq[q].z, a1.y);
          }
        }
      }
    }
  }
  // warps 1..3 hand their sums to warp 0 through shared memory (the strips are no longer needed);
  // layout [warp-1][value][lane]: conflict-free both ways, fixed order of addition
  __syncthreads();
  float *red = reinterpret_cast<float *>(xs);
  constexpr int NV = W2_RK * T_RC * 2;  // floats per thread
  if (warp > 0 && group_active) {
    float *dst = red + (size_t)(warp - 1) * NV * 32 + lane;
#pragma unroll
    for (int i = 0; i < W2_RK; i++)
#pragma unroll
      for (int c = 0; c < T_RC; c++) {
        dst[(size_t)((i * T_RC + c) * 2) * 32] = acc[i][c].x;
        dst[(size_t)((i * T_RC + c) * 2 + 1) * 32] = acc[i][c].y;
      }
  }
  __syncthreads();
  if (warp == 0 && group_active) {
#pragma unroll
    for (int w = 0; w < W2_WARPS - 1; w++) {
      const float *src = red + (size_t)w * NV * 32 + lane;
#pragma unroll
      for (int i = 0; i < W2_RK; i++)
#pragma unroll
        for (int c = 0; c < T_RC; c++) {
          acc[i][c].x += src[(size_t)((i * T_RC + c) * 2) * 32];
          acc[i][c].y += src[(size_t)((i * T_RC + c) * 2 + 1) * 32];
        }
    }
    // partial sums: [segment][group][output][32 clients]
    float2 *pp = partial + K.part_off + (((long long)seg * K.n_groups + grp) * K.kpad + k0) * T_CG + cbase;
#pragma unroll
    for (int i = 0; i < W2_RK; i++) {
      float4 *row = reinterpret_cast<float4 *>(pp + (size_t)(o + W2_LO * i) * T_CG);
#pragma unroll
      for (int q = 0; q < T_RC / 2; q++)
        row[q] = make_float4(acc[i][2 * q].x, acc[i][2 * q].y, acc[i][2 * q + 1].x, acc[i][2 * q + 1].y);
    }
  }
}

// ---------------------------------------------------------------------------
// fir_long4: ONE resident CTA per SM walks `seg_per` consecutive 128-tap segments of one (group
// pair, 28-output tile) through a two-stage ring -- while its 8 warps (16 taps of the segment each)
// accumulate segment i, warp 0 has already issued the TMA copies of segment i+1.  No idle time while
// a CTA loads, the prologue and the cross-warp reduction are paid once per ~13 segments instead of
// once per segment, and the partial-sum slabs shrink from one per segment (121 for BASELINE
// configs[4]) to one per CTA along the tap axis (9): the reduction kernel and its traffic shrink
// with them.
// The tile is 28 outputs x 64 clients (4 output lanes x 7 outputs per thread, 8 client octets = TWO
// 32-client groups per CTA), and ~52 outputs per block fit 2 x 28.  Small bulk copies, not FMAs, are
// what a long-filter kernel waits for (~300 cycles per 1 KiB strip copy and SM whatever else it
// does), so a stage is 28 strips + 2 tap blocks = 30 bulk copies where a 56 x 32 tile of the same
// FLOPs needs 57 -- or 3 copies, when the 28 strips arrive as one tensor copy (below).
// ---------------------------------------------------------------------------
constexpr int W4_WARPS = 8;
constexpr int W4_THREADS = 32 * W4_WARPS;
constexpr int W4_STAGES = 2;
constexpr int W4_JW = W_JS / W4_WARPS;  // taps per warp per segment (16)
constexpr int W4_LO = 4;
constexpr int W4_KT = W4_LO * W2_RK;    // 28 outputs per CTA
constexpr int W4_GROUPS = 2;            // client groups per CTA
constexpr int W4_STAGE_BYTES = (W4_GROUPS * W_JS * T_CG * 8 + W4_KT * W_JSP * 8 + 127) / 128 * 128;  // 64 KiB taps + 28.4 KiB strips (128-byte aligned stages: TMA tensor destinations)
constexpr int W4_SMEM = W4_STAGES * W4_STAGE_BYTES + 64;
static_assert((W4_WARPS - 1) * 32 * W2_RK * T_RC * 2 * 4 <= W4_STAGES * W4_STAGE_BYTES, "reduction scratch reuses the stages");

// With a tensor map (K.tmap_w > 0) the 28 input strips of a stage arrive as ONE 2-D tensor copy (box
// 130 x 28 eight-byte elements, row pitch D in the ring) instead of 28 bulk copies of 1 KiB: the stage
// loads, not the FMAs, are what this kernel waits for (ncu: 12 % of warp time on the stage's mbarrier).
// A stage whose box would cross the ring's wrap-around (or the map's inner width), and every stage of a
// class without a map, uses the per-strip copies.
__global__ void __launch_bounds__(W4_THREADS, 1)
fir_long4_cf32_kernel(const __grid_constant__ TileLaunch P, const float2 *__restrict__ ring, unsigned mask,
                      const float2 *__restrict__ tile_taps, float2 *__restrict__ partial,
                      const __grid_constant__ CUtensorMap strips) {
  extern __shared__ __align__(128) unsigned char smem[];
  uint64_t *bars = reinterpret_cast<uint64_t *>(smem + W4_STAGES * W4_STAGE_BYTES);  // full[2], empty[2]

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int o = lane & (W4_LO - 1), h = lane / W4_LO;  // output column, client octet (0..7)
  const int gsel = h >> 2;                              // which of the CTA's two groups
  const int cbase = (h & 3) * T_RC;

  const int ci = class_of_cta(P, (int)blockIdx.x);
  const TileClass &K = P.cls[ci];
  const int local = (int)blockIdx.x - K.cta_begin;
  const int sp = local % K.ksplit;
  const int rest = local / K.ksplit;
  const int tile = rest % K.tiles;
  const int gpair = rest / K.tiles;
  const int k0 = tile * W4_KT;
  const int D = K.D;
  const int seg_begin = sp * K.seg_per;
  const int seg_end = min(seg_begin + K.seg_per, K.nseg);
  const int grp0 = gpair * W4_GROUPS;
  const int n_grp = min(W4_GROUPS, K.n_groups - grp0);           // 1 or 2 real groups in this CTA
  const bool mine_active = gsel < n_grp && (grp0 + gsel) * T_CG < K.n_members;

  if (tid == 0) {
    for (int st = 0; st < W4_STAGES; st++) {
      mbar_init(&bars[st], 1);
      mbar_init(&bars[W4_STAGES + st], W4_WARPS);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();

  const unsigned xoff = (unsigned)(K.first & 1);  // 1: strips start one sample early (see load_segment)
  auto load_segment = [&](int sg, int st) {
    const int f0 = sg * W_JS;
    const int len = min(W_JS, K.L - f0);
    float2 *ts = reinterpret_cast<float2 *>(smem + st * W4_STAGE_BYTES);
    float2 *xs = ts + W4_GROUPS * W_JS * T_CG;
    // bulk copies need 16-byte aligned sources: an odd window start (D is even, so every strip of every
    // segment has the parity of K.first) is fetched from one sample earlier, two samples longer -- the row
    // pitch W_JSP = W_JS + 2 has room -- and the readers skip the extra sample (xoff below)
    const unsigned tap_bytes = (unsigned)len * T_CG * 8u;
    const unsigned slen = (unsigned)len + 2u * xoff, strip_bytes = slen * 8u;
    const long long w0 = K.first + (long long)k0 * D + f0 - (long long)xoff;
    bool boxed = false;
    unsigned q = 0, c0 = 0;
    if (K.tmap_w > 0) {
      const unsigned idx0 = (unsigned)((unsigned long long)w0) & mask;
      q = idx0 / (unsigned)D;
      c0 = idx0 - q * (unsigned)D;
      boxed = (unsigned long long)idx0 + (unsigned long long)(W4_KT - 1) * D + W_JSP <= (unsigned long long)mask + 1ull &&
              c0 + (unsigned)W_JSP <= (unsigned)K.tmap_w;
    }
    if (lane == 0)
      mbar_expect_tx(&bars[st], (unsigned)n_grp * tap_bytes + (boxed ? (unsigned)(W4_KT * W_JSP * 8) : W4_KT * strip_bytes));
    __syncwarp();
    if (lane < n_grp)
      tma_bulk_g2s(ts + lane * W_JS * T_CG, tile_taps + K.taps_off + ((long long)(grp0 + lane) * K.L + f0) * T_CG, tap_bytes,
                   &bars[st]);
    if (boxed) {
      if (lane == 0) tma_tensor2d_g2s(xs, &strips, (int)c0, (int)q, &bars[st]);
    } else if (lane < W4_KT) {
      const unsigned idx = (unsigned)((unsigned long long)(w0 + (long long)lane * D)) & mask;
      const unsigned n1 = min(slen, mask + 1u - idx);
      tma_bulk_g2s(xs + lane * W_JSP, ring + idx, n1 * 8u, &bars[st]);
      if (n1 < slen) tma_bulk_g2s(xs + lane * W_JSP + n1, ring, (slen - n1) * 8u, &bars[st]);
    }
  };

  float2 acc[W2_RK][T_RC];
#pragma unroll
  for (int i = 0; i < W2_RK; i++)
#pragma unroll
    for (int c = 0; c < T_RC; c++) acc[i][c] = make_float2(0.f, 0.f);

  if (seg_begin < seg_end) {
    if (warp == 0) load_segment(seg_begin, 0);
    for (int sg = seg_begin; sg < seg_end; sg++) {
      const int it = sg - seg_begin, st = it % W4_STAGES;
      if (warp == 0 && sg + 1 < seg_end) {
        const int ns = (it + 1) % W4_STAGES;
        if (it >= 1) mbar_wait(&bars[W4_STAGES + ns], (unsigned)(((it - 1) / W4_STAGES) & 1));
        load_segment(sg + 1, ns);
      }
      mbar_wait(&bars[st], (unsigned)((it / W4_STAGES) & 1));
      if (mine_active) {
        const int len = min(W_JS, K.L - sg * W_JS);
        const float2 *ts = reinterpret_cast<const float2 *>(smem + st * W4_STAGE_BYTES);
        const float2 *xs = ts + W4_GROUPS * W_JS * T_CG;
        const float4 *tp = reinterpret_cast<const float4 *>(ts + gsel * W_JS * T_CG + cbase);
        const float2 *xb[W2_RK];
#pragma unroll
        for (int i = 0; i < W2_RK; i++) xb[i] = xs + (o + W4_LO * i) * W_JSP + xoff;
        const int f_end = min(len, (warp + 1) * W4_JW);
#pragma unroll 1
        for (int f = warp * W4_JW; f < f_end; f += T_UNROLL) {
#pragma unroll
          for (int u = 0; u < T_UNROLL; u++) {
            float2 x[W2_RK];
#pragma unroll
            for (int i = 0; i < W2_RK; i++) x[i] = xb[i][f + u];
            float4 tq[T_RC / 2];
#pragma unroll
            for (int q = 0; q < T_RC / 2; q++) tq[q] = tp[(f + u) * (T_CG / 2) + q];
#pragma unroll
            for (int i = 0; i < W2_RK; i++) {
#pragma unroll
              for (int q = 0; q < T_RC / 2; q++) {
                float2 &a0 = acc[i][2 * q], &a1 = acc[i][2 * q + 1];
                a0.x = fmaf(x[i].x, tq[q].x, a0.x);
                a0.x = fmaf(-x[i].y, tq[q].y, a0.x);
                a0.y = fmaf(x[i].x, tq[q].y, a0.y);
                a0.y = fmaf(x[i].y, tq[q].x, a0.y);
                a1.x = fmaf(x[i].x, tq[q].z, a1.x);
                a1.x = fmaf(-x[i].y, tq[q].w, a1.x);
                a1.y = fmaf(x[i].x, tq[q].w, a1.y);
                a1.y = fmaf(x[i].y, tq[q].z, a1.y);
              }
            }
          }
        }
      }
      __syncwarp();
      if (lane == 0) mbar_arrive(&bars[W4_STAGES + st]);  // this warp is done with the stage
    }
  }
  // warps 1..7 hand their sums to warp 0 through shared memory, layout [warp-1][value][lane]
  __syncthreads();
  float *red = reinterpret_cast<float *>(smem);
  constexpr int NV = W2_RK * T_RC * 2;
  if (warp > 0) {
    float *dst = red + (size_t)(warp - 1) * NV * 32 + lane;
#pragma unroll
    for (int i = 0; i < W2_RK; i++)
#pragma unroll
      for (int c = 0; c < T_RC; c++) {
        dst[(size_t)((i * T_RC + c) * 2) * 32] = acc[i][c].x;
        dst[(size_t)((i * T_RC + c) * 2 + 1) * 32] = acc[i][c].y;
      }
  }
  __syncthreads();
  if (warp == 0 && mine_active) {
#pragma unroll 1
    for (int w = 0; w < W4_WARPS - 1; w++) {
      const float *src = red + (size_t)w * NV * 32 + lane;
#pragma unroll
      for (int i = 0; i < W2_RK; i++)
#pragma unroll
        for (int c = 0; c < T_RC; c++) {
          acc[i][c].x += src[(size_t)((i * T_RC + c) * 2) * 32];
          acc[i][c].y += src[(size_t)((i * T_RC + c) * 2 + 1) * 32];
        }
    }
    // partial sums: [tap split][group][output][32 clients]
    float2 *pp = partial + K.part_off + (((long long)sp * K.n_groups + grp0 + gsel) * K.kpad + k0) * T_CG + cbase;
#pragma unroll
    for (int i = 0; i < W2_RK; i++) {
      float4 *row = reinterpret_cast<float4 *>(pp + (size_t)(o + W4_LO * i) * T_CG);
#pragma unroll
      for (int q = 0; q < T_RC / 2; q++)
        row[q] = make_float4(acc[i][2 * q].x, acc[i][2 * q].y, acc[i][2 * q + 1].x, acc[i][2 * q + 1].y);
    }
  }
}

// Adds the segments in order, derotates, stores.  Block = 32 clients (lanes) x 8 outputs.
__global__ void __launch_bounds__(256)
fir_long_reduce_kernel(const __grid_constant__ TileLaunch P, const float2 *__restrict__ partial,
                       const int *__restrict__ member_off, const float2 *__restrict__ member_incr,
                       const float2 *__restrict__ phases, float2 *__restrict__ out) {
  const int ci = blockIdx.z;
  if (ci >= P.n_classes) return;
  const TileClass &K = P.cls[ci];
  const int grp = blockIdx.y;
  if (grp >= K.n_groups) return;
  const int lane = threadIdx.x & 31;
  const int k = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (k >= K.n_out) return;
  const int off = __ldg(member_off + K.members_off + grp * T_CG + lane);
  if (off < 0) return;
  const float2 *pp = partial + K.part_off + ((long long)grp * K.kpad + k) * T_CG + lane;
  const size_t seg_stride = (size_t)K.n_groups * K.kpad * T_CG;
  float2 acc = make_float2(0.f, 0.f);
  // loads in batches of 8 (independent, so their L2 latencies overlap); the additions
  // stay strictly in segment order
  int s = 0;
  for (; s + 8 <= K.nslab; s += 8) {
    float2 v[8];
#pragma unroll
    for (int u = 0; u < 8; u++) v[u] = pp[(size_t)(s + u) * seg_stride];
#pragma unroll
    for (int u = 0; u < 8; u++) {
      acc.x += v[u].x;
      acc.y += v[u].y;
    }
  }
  for (; s < K.nslab; s++) {
    const float2 v = pp[(size_t)s * seg_stride];
    acc.x += v.x;
    acc.y += v.y;
  }
  float2 ph = phases[K.ph_base + (long long)grp * K.ph_stride + (size_t)(k >> 1) * 32 + lane];
  if (k & 1) ph = cmul_unfused(ph, __ldg(member_incr + K.members_off + grp * T_CG + lane));
  out[off + k] = cmul_unfused(acc, ph);  // src/xlating.c:70
}

// ---------------------------------------------------------------------------
// cascade clients (xlg_add_client_cascade).  Stage A is an integer client of the kernels above whose
// outputs land in a row of the slot's arena that is never copied to the host.  Stage B is the reference
// filter at fs / D1 with centre 0: its rotated taps are (h, +-0), its oscillator stays 1 + 0i and the
// renormalisation divides by 1, so it is a real-tap decimator with history,
//     z[k] = sum_{j < T2} y[first + k*D2 + j] * rev2[j]          (2 real FMAs per tap),
// over the client's stage-A stream y, kept in a per-client power-of-two ring in HBM: y at stage-A stream
// position p lives at ring[p & mask], and positions before the attach point read as the ring's zeros.
// ---------------------------------------------------------------------------
struct CascBlk {
  float2 *ring;     // the client's stage-A history ring
  long long a_pos;  // stage-A stream position of this block's first stage-A output
  long long first;  // stage-A stream position where this block's stage-B output 0 starts its window
  unsigned mask;    // ring capacity - 1
  int a_off;        // this block's stage-A outputs in the slot's output arena
  int n1, n2;       // stage-A outputs appended / stage-B outputs computed by this block
  int D2, T2;
  int taps_off;     // float offset of rev2 in the real tap arena, a multiple of 4 (16-byte TMA source)
  int out_off;      // final row in the slot's output arena
};

// companion copy: append this block's stage-A outputs to each client's ring (grid.y = client)
__global__ void __launch_bounds__(256)
cascade_append_kernel(const CascBlk *__restrict__ cb, const float2 *__restrict__ out) {
  const CascBlk &b = cb[blockIdx.y];
  const int n1 = b.n1;
  for (int i = blockIdx.x * 256 + threadIdx.x; i < n1; i += gridDim.x * 256)
    b.ring[(unsigned)((unsigned long long)(b.a_pos + i)) & b.mask] = out[b.a_off + i];
}

constexpr int C_THREADS = 128;
constexpr int C_R = 2;                    // outputs per thread: t and t + C_THREADS
constexpr int C_KO = C_THREADS * C_R;     // outputs per CTA at most (the host lowers it where shared memory runs out)
// shared memory of a CTA with ko outputs: mbarrier, taps padded to 16 bytes, the window (+1 for an odd start, even)
__host__ __device__ constexpr size_t cascade_smem(int ko, int D2, int T2) {
  return 16 + (size_t)((T2 + 3) & ~3) * 4 + (((size_t)(ko - 1) * D2 + T2 + 2) & ~(size_t)1) * 8;
}

// Stage B: CTA (x, c) computes outputs [x*ko, x*ko + ko) of cascade client c.  One TMA bulk copy stages the
// taps, one or two (the ring wraps) stage the window; every thread then keeps C_R outputs in registers.
// Lane l walks the taps starting at j = l (mod T2) when D2 is even: the lanes' samples then lie D2 + 1
// apart in shared memory, an odd stride, so neither the window nor the tap loads have bank conflicts
// (with odd D2 every lane starts at j = 0 and the tap load is a broadcast).
__global__ void __launch_bounds__(C_THREADS)
cascade_fir_cf32_kernel(const CascBlk *__restrict__ cb, const float *__restrict__ taps2, float2 *__restrict__ out,
                        int ko) {
  extern __shared__ __align__(128) unsigned char smem[];
  uint64_t *bar = reinterpret_cast<uint64_t *>(smem);
  const CascBlk &b = cb[blockIdx.y];
  const int n2 = b.n2, k0 = blockIdx.x * ko;
  if (k0 >= n2) return;
  const int D2 = b.D2, T2 = b.T2, tpad = (T2 + 3) & ~3;
  const int nk = min(ko, n2 - k0);
  float *ts = reinterpret_cast<float *>(smem + 16);
  float2 *xs = reinterpret_cast<float2 *>(smem + 16 + tpad * 4);
  const unsigned idx = (unsigned)((unsigned long long)(b.first + (long long)k0 * D2)) & b.mask;
  const unsigned shift = idx & 1u;  // an odd window start is fetched from one sample earlier (16-byte source)
  const int tid = threadIdx.x;
  if (tid == 0) {
    mbar_init(bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();
  if (tid == 0) {
    const unsigned need = ((unsigned)((nk - 1) * D2 + T2) + shift + 1u) & ~1u;
    const unsigned p1 = min(need, b.mask + 1u - (idx - shift));
    mbar_expect_tx(bar, (unsigned)tpad * 4u + need * 8u);
    tma_bulk_g2s(ts, taps2 + b.taps_off, (unsigned)tpad * 4u, bar);
    tma_bulk_g2s(xs, b.ring + (idx - shift), p1 * 8u, bar);
    if (p1 < need) tma_bulk_g2s(xs + p1, b.ring, (need - p1) * 8u, bar);
  }
  mbar_wait(bar, 0);
  if (tid >= nk) return;
  const float2 *x[C_R];
#pragma unroll
  for (int i = 0; i < C_R; i++) x[i] = xs + shift + (size_t)min(tid + C_THREADS * i, nk - 1) * D2;
  float2 acc[C_R];
#pragma unroll
  for (int i = 0; i < C_R; i++) acc[i] = make_float2(0.f, 0.f);
  int j = (D2 & 1) ? 0 : (tid & 31) % T2;
#pragma unroll 4
  for (int s = 0; s < T2; s++) {
    const float h = ts[j];
#pragma unroll
    for (int i = 0; i < C_R; i++) {
      const float2 v = x[i][j];
      acc[i].x = fmaf(v.x, h, acc[i].x);
      acc[i].y = fmaf(v.y, h, acc[i].y);
    }
    if (++j == T2) j = 0;
  }
#pragma unroll
  for (int i = 0; i < C_R; i++)
    if (tid + C_THREADS * i < nk) out[b.out_off + k0 + tid + C_THREADS * i] = acc[i];
}

}  // namespace xl
