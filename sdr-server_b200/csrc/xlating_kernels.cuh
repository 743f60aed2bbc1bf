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
 *   cascade_*        stage B of two-stage clients: a real-tap decimator (or rational
 *                    L2/M2 polyphase filter) over each client's stage-A history ring,
 *                    TMA-staged window, register tile
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

#include "cascade_stage_b.cuh"
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

// cf32 input: the ring holds the submitted values bit for bit (a copy, no arithmetic: NaN payloads, -0.0 and
// subnormals pass unchanged), at S mod cap like every conversion
__global__ void copy_cf32_kernel(const float2 *__restrict__ raw, float2 *__restrict__ ring, unsigned mask,
                                 long long S, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  ring[(unsigned)((unsigned long long)(S + i)) & mask] = raw[i];
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
// cascade clients: stage B (CascBlk, CascPolyBlk and their shared memory in cascade_stage_b.cuh)
// ---------------------------------------------------------------------------

// companion copy: append this block's stage-A outputs to each client's ring (grid.y = client)
__global__ void __launch_bounds__(256)
cascade_append_kernel(const CascBlk *__restrict__ cb, const float2 *__restrict__ out) {
  const CascBlk &b = cb[blockIdx.y];
  const int n1 = b.n1;
  for (int i = blockIdx.x * 256 + threadIdx.x; i < n1; i += gridDim.x * 256)
    b.ring[(unsigned)((unsigned long long)(b.a_pos + i)) & b.mask] = out[b.a_off + i];
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

// Stage B of rational cascade clients: CTA (x, c) computes outputs [x*ko, x*ko + ko) of client c.  One TMA
// bulk copy stages the client's branches, one or two (the ring wraps) the stage-A window from n0 of the
// first output to n0 of the last + Tb2.  Outputs k and k + L2 share a branch and their windows lie M2
// samples apart, so threads take the CTA's outputs residue-major: pair slot (rho, p) computes relative
// outputs rho + p*L2 and rho + (p + P)*L2 on branch r(rho), and consecutive lanes hold consecutive p of one
// residue.  A warp therefore works on one branch (the tap load is a broadcast) wherever the CTA has at
// least 64 outputs per branch, on a few branches otherwise.  Lanes of one residue read the window M2 apart;
// with even M2 they walk the taps skewed (start at t = lane mod Tb2), an odd stride, as the integer stage B
// does for even D2, and the window loads have no bank conflicts.  Two real FMAs per tap.
__global__ void __launch_bounds__(C_THREADS)
cascade_fir_poly_cf32_kernel(const CascPolyBlk *__restrict__ pb, const float *__restrict__ taps2,
                             float2 *__restrict__ out) {
  extern __shared__ __align__(128) unsigned char smem[];
  uint64_t *bar = reinterpret_cast<uint64_t *>(smem);
  const CascPolyBlk &b = pb[blockIdx.y];
  const int n2 = b.n2, ko = b.ko;
  if ((long long)blockIdx.x * ko >= n2) return;
  const int k0 = blockIdx.x * ko;
  const int L2 = b.L2, M2 = b.M2, Tb2 = b.Tb2, tpad = (L2 * Tb2 + 3) & ~3;
  const int nk = min(ko, n2 - k0);
  float *ts = reinterpret_cast<float *>(smem + 16);
  float2 *xs = reinterpret_cast<float2 *>(smem + 16 + tpad * 4);
  long long base, nlast;
  poly_branch(b.first + (long long)k0 * M2, L2, &base);
  poly_branch(b.first + (long long)(k0 + nk - 1) * M2, L2, &nlast);
  const unsigned idx = (unsigned)((unsigned long long)base) & b.mask;
  const unsigned shift = idx & 1u;  // an odd window start is fetched from one sample earlier (16-byte source)
  const int tid = threadIdx.x;
  if (tid == 0) {
    mbar_init(bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();
  if (tid == 0) {
    const unsigned need = ((unsigned)(nlast - base + Tb2) + shift + 1u) & ~1u;
    const unsigned p1 = min(need, b.mask + 1u - (idx - shift));
    mbar_expect_tx(bar, (unsigned)tpad * 4u + need * 8u);
    tma_bulk_g2s(ts, taps2 + b.taps_off, (unsigned)tpad * 4u, bar);
    tma_bulk_g2s(xs, b.ring + (idx - shift), p1 * 8u, bar);
    if (p1 < need) tma_bulk_g2s(xs + p1, b.ring, (need - p1) * 8u, bar);
  }
  mbar_wait(bar, 0);
  const int P = ((nk + L2 - 1) / L2 + 1) / 2;  // pair slots per residue: residue 0 has the most outputs
  const int slots = min(L2, nk) * P;
  for (int ps = tid; ps < slots; ps += C_THREADS) {
    const int rho = ps / P, p = ps - rho * P;
    const int ka = rho + p * L2, kb = ka + P * L2;
    if (ka >= nk) continue;
    long long n0;
    const int r = poly_branch(b.first + (long long)(k0 + rho) * M2, L2, &n0);
    const float *h = ts + r * Tb2;
    const float2 *xa = xs + shift + (size_t)(n0 - base) + (size_t)p * M2;
    const float2 *xb = kb < nk ? xa + (size_t)P * M2 : xa;
    float2 acc_a = make_float2(0.f, 0.f), acc_b = make_float2(0.f, 0.f);
    int t = (M2 & 1) ? 0 : (tid & 31) % Tb2;
#pragma unroll 4
    for (int s = 0; s < Tb2; s++) {
      const float hv = h[t];
      const float2 va = xa[t], vb = xb[t];
      acc_a.x = fmaf(va.x, hv, acc_a.x);
      acc_a.y = fmaf(va.y, hv, acc_a.y);
      acc_b.x = fmaf(vb.x, hv, acc_b.x);
      acc_b.y = fmaf(vb.y, hv, acc_b.y);
      if (++t == Tb2) t = 0;
    }
    out[b.out_off + k0 + ka] = acc_a;
    if (kb < nk) out[b.out_off + k0 + kb] = acc_b;
  }
}

// ---------------------------------------------------------------------------
// sub-band members (xlg_add_client_subband).  A sub-band is an integer client whose outputs are appended to
// a history ring (cascade_append_kernel, as a cascade's stage A).  A member is the reference's float path at
// fs / D1 with its own centre, fed that ring:
//     z[k] = phase_k * sum_{j < T2} y[first + k*D2 + j] * rev2[j]          (complex taps, 4 real FMAs each)
// Members of one sub-band with equal (D2, T2, window alignment, first valid position) form a class: they
// read the same windows, so a CTA stages the windows of a span of outputs once and every staged sample
// feeds SB_MG members.
// A rational member (xlg_add_client_subband_rational, L2 > 1) is the reference's float path with decimation
// M2 at L2 * fs / D1, fed the zero-stuffed ring u[L2*n] = y[n]: output k's upsampled window starts at
// w = first + k*M2, and with r = (-w) mod L2, n0 = (w + r) / L2 (poly_branch) only branch r of its taps meets
// sub-band samples,
//     z[k] = phase_k * sum_{t < Tb2} y[n0 + t] * P[r][t],   P[r][t] = rev2[r + t*L2] (0 past T2).
// Outputs k and k + L2 share r and their n0 lie M2 apart, so the outputs of one residue rho = k mod L2 are an
// integer class with decimation M2 and Tb2 taps, strided by L2.
// ---------------------------------------------------------------------------
constexpr int SB_WARPS = 4;                  // warps of a CTA; warp w serves members [w*SB_RM, (w+1)*SB_RM)
constexpr int SB_THREADS = 32 * SB_WARPS;
constexpr int SB_RM = 4;                     // members per thread
constexpr int SB_RO = 2;                     // outputs per thread: lane and lane + 32
constexpr int SB_MG = SB_WARPS * SB_RM;      // members per CTA (a group)
constexpr int SB_KO = 32 * SB_RO;            // outputs per CTA

struct SbBlk {          // one class, this block
  const float2 *ring;   // its sub-band's history ring
  long long first;      // ring position where output 0's window starts (upsampled position when L2 > 1)
  long long zb;         // ring positions before this read as zero (its members' attach point)
  unsigned mask;        // ring capacity - 1
  int n2, D2, T2;       // L2 > 1: D2 = M2 and T2 = Tb2, the taps per branch
};

struct SbGroup {        // up to SB_MG members of one class (the layout's)
  int cls, n_mem;
  int taps_off;         // float2 offset of the [L2][SB_MG][sb_tpad(T2)] rotated reversed taps (branch-major
                        // when L2 > 1), zero rows for padding
  int l2;               // its class's L2 (1: an integer class)
  int out_off[SB_MG];   // final rows in the slot's output arena
  int ph_off[SB_MG];    // oscillator table: phase of EVEN output k at ph[ph_off + 32 * (k / 2)]
  float2 incr[SB_MG];
};

struct SbMem {          // the member oscillator pre-pass: one entry per member, 32 per table group
  int cid;              // its ClientDev (phase, incr, renorm; inactive for the other kernels), -1 = padding
  int cls;
  int ph_off;
};

__host__ __device__ constexpr int sb_tpad(int T2) { return (T2 + 1) & ~1; }  // 16-byte rows
// shared memory of a CTA: mbarrier, SB_MG tap rows, the window of SB_KO outputs (+1 for an odd start, even)
__host__ __device__ constexpr size_t subband_smem(int D2, int T2) {
  return 16 + (size_t)SB_MG * sb_tpad(T2) * 8 + (((size_t)(SB_KO - 1) * D2 + T2 + 2) & ~(size_t)1) * 8;
}

// The members' oscillators: their output counts are known on the host, so one lane per member replays the
// group's recursion (osc_chain_cf32) on this block's count.  As in phase_cf32_kernel, a warp owns a table
// group of 32 members and stores the even phases interleaved, one coalesced line per step.
__global__ void __launch_bounds__(32)
subband_phase_kernel(ClientDev *__restrict__ cl, const SbMem *__restrict__ mem, const SbBlk *__restrict__ blk,
                     float2 *__restrict__ ph) {
  const SbMem m = mem[blockIdx.x * 32 + threadIdx.x];
  if (m.cid < 0) return;
  ClientDev *d = cl + m.cid;
  d->phase = osc_chain_cf32<32>(d->phase, d->incr, ph + m.ph_off, blk[m.cls].n2, d->renorm);
}

// CTA (x, g) computes outputs [x*SB_KO, x*SB_KO + SB_KO) of the members of group g.  One TMA bulk copy
// stages the group's taps, one or two (the ring wraps) the window; an odd window start is fetched from one
// sample earlier.  Lane l holds outputs l and l + 32 of SB_RM members in registers, so each sample it loads
// feeds SB_RM members and each tap SB_RO outputs.  With even D2 lane l walks the taps from j = l (mod T2):
// its window reads then lie D2 + 1 samples apart, an odd stride, and its tap reads are consecutive, so
// neither has bank conflicts (with odd D2 every lane starts at j = 0 and the tap read is a broadcast).
__global__ void __launch_bounds__(SB_THREADS)
subband_fir_cf32_kernel(const SbBlk *__restrict__ blk, const SbGroup *__restrict__ grp,
                        const float2 *__restrict__ taps, const float2 *__restrict__ ph, float2 *__restrict__ out) {
  extern __shared__ __align__(128) unsigned char smem[];
  uint64_t *bar = reinterpret_cast<uint64_t *>(smem);
  const SbGroup &gp = grp[blockIdx.y];
  const SbBlk b = blk[gp.cls];
  const int k0 = blockIdx.x * SB_KO;
  if (k0 >= b.n2) return;
  const int D2 = b.D2, T2 = b.T2, tpad = sb_tpad(T2);
  const int nk = min(SB_KO, b.n2 - k0);
  float2 *ts = reinterpret_cast<float2 *>(smem + 16);
  float2 *xs = ts + (size_t)SB_MG * tpad;
  const long long w0 = b.first + (long long)k0 * D2;
  const unsigned idx = (unsigned)((unsigned long long)w0) & b.mask;
  const unsigned shift = idx & 1u;
  const unsigned need = ((unsigned)((nk - 1) * D2 + T2) + shift + 1u) & ~1u;
  const int tid = threadIdx.x;
  if (tid == 0) {
    mbar_init(bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();
  if (tid == 0) {
    const unsigned tbytes = (unsigned)(SB_MG * tpad) * 8u;
    const unsigned p1 = min(need, b.mask + 1u - (idx - shift));
    mbar_expect_tx(bar, tbytes + need * 8u);
    tma_bulk_g2s(ts, taps + gp.taps_off, tbytes, bar);
    tma_bulk_g2s(xs, b.ring + (idx - shift), p1 * 8u, bar);
    if (p1 < need) tma_bulk_g2s(xs + p1, b.ring, (need - p1) * 8u, bar);
  }
  mbar_wait(bar, 0);
  const long long base = w0 - (long long)shift;
  if (b.zb > base) {  // a class attached mid-stream: its members read zeros before their attach point
    for (unsigned i = tid; i < need; i += SB_THREADS)
      if (base + (long long)i < b.zb) xs[i] = make_float2(0.f, 0.f);
    __syncthreads();
  }
  const int warp = tid >> 5, lane = tid & 31;
  const int m0 = warp * SB_RM;
  if (m0 >= gp.n_mem) return;
  const float2 *x[SB_RO];
#pragma unroll
  for (int i = 0; i < SB_RO; i++) x[i] = xs + shift + (size_t)min(lane + 32 * i, nk - 1) * D2;
  const float2 *t[SB_RM];
#pragma unroll
  for (int r = 0; r < SB_RM; r++) t[r] = ts + (size_t)(m0 + r) * tpad;
  float2 acc[SB_RO][SB_RM];
#pragma unroll
  for (int i = 0; i < SB_RO; i++)
#pragma unroll
    for (int r = 0; r < SB_RM; r++) acc[i][r] = make_float2(0.f, 0.f);
  int j = (D2 & 1) ? 0 : lane % T2;
#pragma unroll 2
  for (int s = 0; s < T2; s++) {
    float2 v[SB_RO], h[SB_RM];
#pragma unroll
    for (int i = 0; i < SB_RO; i++) v[i] = x[i][j];
#pragma unroll
    for (int r = 0; r < SB_RM; r++) h[r] = t[r][j];
#pragma unroll
    for (int i = 0; i < SB_RO; i++)
#pragma unroll
      for (int r = 0; r < SB_RM; r++) {
        acc[i][r].x = fmaf(v[i].x, h[r].x, acc[i][r].x);
        acc[i][r].x = fmaf(-v[i].y, h[r].y, acc[i][r].x);
        acc[i][r].y = fmaf(v[i].x, h[r].y, acc[i][r].y);
        acc[i][r].y = fmaf(v[i].y, h[r].x, acc[i][r].y);
      }
    if (++j == T2) j = 0;
  }
#pragma unroll
  for (int r = 0; r < SB_RM; r++) {
    const int m = m0 + r;
    if (m >= gp.n_mem) break;
#pragma unroll
    for (int i = 0; i < SB_RO; i++) {
      const int k = k0 + lane + 32 * i;
      if (lane + 32 * i >= nk) continue;
      float2 p = ph[gp.ph_off[m] + 32 * (k >> 1)];
      if (k & 1) p = cmul_unfused(p, gp.incr[m]);     // odd outputs: one step from the stored even phase
      out[gp.out_off[m] + k] = cmul_unfused(acc[i][r], p);  // src/xlating.c:70
    }
  }
}

// Rational classes (SbGroup::l2 > 1), grid (output tiles of the longest residue, groups, largest L2): CTA
// (x, g, rho) computes outputs rho + L2*q, q in [x*SB_KO, x*SB_KO + SB_KO), of the members of group g -- the
// integer class of residue rho: its window from n0 of output rho, decimation M2, and branch r(rho)'s taps,
// staged, walked and rotated as subband_fir_cf32_kernel does.
__global__ void __launch_bounds__(SB_THREADS)
subband_fir_poly_cf32_kernel(const SbBlk *__restrict__ blk, const SbGroup *__restrict__ grp,
                             const float2 *__restrict__ taps, const float2 *__restrict__ ph,
                             float2 *__restrict__ out) {
  extern __shared__ __align__(128) unsigned char smem[];
  uint64_t *bar = reinterpret_cast<uint64_t *>(smem);
  const SbGroup &gp = grp[blockIdx.y];
  const SbBlk b = blk[gp.cls];
  const int L2 = gp.l2, rho = blockIdx.z;
  if (rho >= min(L2, b.n2)) return;
  long long first;  // n0 of output rho: the residue's outputs rho + L2*q start their windows at first + q*M2
  const int br = poly_branch(b.first + (long long)rho * b.D2, L2, &first);
  const int n2 = (b.n2 - rho + L2 - 1) / L2;
  const int k0 = blockIdx.x * SB_KO;
  if (k0 >= n2) return;
  const int D2 = b.D2, T2 = b.T2, tpad = sb_tpad(T2);
  const int nk = min(SB_KO, n2 - k0);
  float2 *ts = reinterpret_cast<float2 *>(smem + 16);
  float2 *xs = ts + (size_t)SB_MG * tpad;
  const long long w0 = first + (long long)k0 * D2;
  const unsigned idx = (unsigned)((unsigned long long)w0) & b.mask;
  const unsigned shift = idx & 1u;
  const unsigned need = ((unsigned)((nk - 1) * D2 + T2) + shift + 1u) & ~1u;
  const int tid = threadIdx.x;
  if (tid == 0) {
    mbar_init(bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();
  if (tid == 0) {
    const unsigned tbytes = (unsigned)(SB_MG * tpad) * 8u;
    const unsigned p1 = min(need, b.mask + 1u - (idx - shift));
    mbar_expect_tx(bar, tbytes + need * 8u);
    tma_bulk_g2s(ts, taps + gp.taps_off + (size_t)br * SB_MG * tpad, tbytes, bar);  // branch br's rows
    tma_bulk_g2s(xs, b.ring + (idx - shift), p1 * 8u, bar);
    if (p1 < need) tma_bulk_g2s(xs + p1, b.ring, (need - p1) * 8u, bar);
  }
  mbar_wait(bar, 0);
  const long long base = w0 - (long long)shift;
  if (b.zb > base) {  // a class attached mid-stream: its members read zeros before their attach point
    for (unsigned i = tid; i < need; i += SB_THREADS)
      if (base + (long long)i < b.zb) xs[i] = make_float2(0.f, 0.f);
    __syncthreads();
  }
  const int warp = tid >> 5, lane = tid & 31;
  const int m0 = warp * SB_RM;
  if (m0 >= gp.n_mem) return;
  const float2 *x[SB_RO];
#pragma unroll
  for (int i = 0; i < SB_RO; i++) x[i] = xs + shift + (size_t)min(lane + 32 * i, nk - 1) * D2;
  const float2 *t[SB_RM];
#pragma unroll
  for (int r = 0; r < SB_RM; r++) t[r] = ts + (size_t)(m0 + r) * tpad;
  float2 acc[SB_RO][SB_RM];
#pragma unroll
  for (int i = 0; i < SB_RO; i++)
#pragma unroll
    for (int r = 0; r < SB_RM; r++) acc[i][r] = make_float2(0.f, 0.f);
  int j = (D2 & 1) ? 0 : lane % T2;
#pragma unroll 2
  for (int s = 0; s < T2; s++) {
    float2 v[SB_RO], h[SB_RM];
#pragma unroll
    for (int i = 0; i < SB_RO; i++) v[i] = x[i][j];
#pragma unroll
    for (int r = 0; r < SB_RM; r++) h[r] = t[r][j];
#pragma unroll
    for (int i = 0; i < SB_RO; i++)
#pragma unroll
      for (int r = 0; r < SB_RM; r++) {
        acc[i][r].x = fmaf(v[i].x, h[r].x, acc[i][r].x);
        acc[i][r].x = fmaf(-v[i].y, h[r].y, acc[i][r].x);
        acc[i][r].y = fmaf(v[i].x, h[r].y, acc[i][r].y);
        acc[i][r].y = fmaf(v[i].y, h[r].x, acc[i][r].y);
      }
    if (++j == T2) j = 0;
  }
#pragma unroll
  for (int r = 0; r < SB_RM; r++) {
    const int m = m0 + r;
    if (m >= gp.n_mem) break;
#pragma unroll
    for (int i = 0; i < SB_RO; i++) {
      if (lane + 32 * i >= nk) continue;
      const int k = rho + L2 * (k0 + lane + 32 * i);  // the member's output
      float2 p = ph[gp.ph_off[m] + 32 * (k >> 1)];
      if (k & 1) p = cmul_unfused(p, gp.incr[m]);     // odd outputs: one step from the stored even phase
      out[gp.out_off[m] + k] = cmul_unfused(acc[i][r], p);  // src/xlating.c:70
    }
  }
}

// ---------------------------------------------------------------------------
// bank sub-bands (xlg_add_bank, xlg_add_bank_subband).  A bank of decimation D1 and real taps h (T1) is a
// 2x-oversampled polyphase filter bank of K = 2 * D1 channels: channel k in [-D1, D1), centred at k * fs / K,
// writes the row
//     y_k[m] = sum_{j < T1} x[s_m + j] * h[T1-1-j] * e^{-2 pi i k (s_m + j - P) / K}
// (P the bank's attach point, x zero before it, s_m the window starts of an integer client (D1, T1) attached
// at P).  With r_m = (s_m - P) mod K and p = j mod K the rotation only depends on p + r_m, so
//     v[m][p] = sum_q x[s_m + p + qK] * h[T1-1-p-qK]                          (phase 1, real taps)
//     y_k[m]  = sum_{p < min(K, T1)} v[m][p] * W[(k (p + r_m)) mod K],   W[j] = e^{-2 pi i j / K}   (phase 2)
// Order (the test model copies it): phase 1 is two fmaf chains (re, im) over q ascending from 0; phase 2 is
// the 4-fmaf complex chain of the member kernels over p ascending from 0.  Both start from +0.
// ---------------------------------------------------------------------------
constexpr int BK_THREADS = 256;
constexpr int BK_F = 32;   // frames per CTA
constexpr int BK_CG = 32;  // channels per CTA (wide banks spread their channel sums over more CTAs)

struct BankBlk {        // one bank, this block
  const float *taps;    // h reversed (h[T1-1-j] at j), zero-padded to bank_tpad
  const float2 *tw;     // W[j], j < K (built in double on the host by quarter turns, rounded once)
  const int2 *chans;    // per materialised channel: (k mod K, its row in the slot's arena)
  long long first;      // stream position of frame 0's window
  long long zb;         // the bank's attach point P: earlier samples read as zero
  unsigned mask;        // input ring capacity - 1
  int n1, D1, T1, K, tpad, n_ch;
  int r0;               // (first - P) mod K
};

// taps padded to a multiple of K and to whole float4s (one bulk copy)
__host__ __device__ constexpr int bank_tpad(int K, int T1) { return ((T1 + K - 1) / K * K + 3) & ~3; }
// shared memory of a CTA: mbarrier, the taps, the window of BK_F frames (+1 for an odd start, even), the
// twiddles and the polyphase sums (rows of K + 1: an odd stride in float2)
__host__ __device__ constexpr size_t bank_smem(int D1, int T1) {
  return 16 + (size_t)bank_tpad(2 * D1, T1) * 4 + (((size_t)(BK_F - 1) * D1 + T1 + 2) & ~(size_t)1) * 8 +
         (size_t)2 * D1 * 8 + (size_t)BK_F * (2 * D1 + 1) * 8;
}

// CTA (x, b, z) computes frames [x*BK_F, x*BK_F + BK_F) of the materialised channels [z*BK_CG, z*BK_CG + BK_CG)
// of bank b.  One TMA bulk copy stages the taps, one or two (the ring wraps) the window; an odd window start
// is fetched from one sample earlier.  Phase 1 gives thread e the sum (frame e / KP, phase e % KP); phase 2
// gives it channel e / BK_F at frame e % BK_F, so a warp stores 32 consecutive samples of one row.
__global__ void __launch_bounds__(BK_THREADS)
bank_cf32_kernel(const BankBlk *__restrict__ blk, const float2 *__restrict__ ring, float2 *__restrict__ out) {
  extern __shared__ __align__(128) unsigned char smem[];
  uint64_t *bar = reinterpret_cast<uint64_t *>(smem);
  const BankBlk b = blk[blockIdx.y];
  const int f0 = blockIdx.x * BK_F, c0 = blockIdx.z * BK_CG;
  if (f0 >= b.n1 || c0 >= b.n_ch) return;
  const int nch = min(BK_CG, b.n_ch - c0);
  const int D1 = b.D1, T1 = b.T1, K = b.K;
  const int nf = min(BK_F, b.n1 - f0);
  float *ts = reinterpret_cast<float *>(smem + 16);
  float2 *xs = reinterpret_cast<float2 *>(ts + b.tpad);
  const long long w0 = b.first + (long long)f0 * D1;
  const unsigned idx = (unsigned)((unsigned long long)w0) & b.mask;
  const unsigned shift = idx & 1u;
  const unsigned need = ((unsigned)((nf - 1) * D1 + T1) + shift + 1u) & ~1u;
  float2 *tw = xs + need;
  float2 *v = tw + K;
  const int tid = threadIdx.x;
  if (tid == 0) {
    mbar_init(bar, 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();
  if (tid == 0) {
    const unsigned tbytes = (unsigned)b.tpad * 4u;
    const unsigned p1 = min(need, b.mask + 1u - (idx - shift));
    mbar_expect_tx(bar, tbytes + need * 8u);
    tma_bulk_g2s(ts, b.taps, tbytes, bar);
    tma_bulk_g2s(xs, ring + (idx - shift), p1 * 8u, bar);
    if (p1 < need) tma_bulk_g2s(xs + p1, ring, (need - p1) * 8u, bar);
  }
  for (int i = tid; i < K; i += BK_THREADS) tw[i] = b.tw[i];
  mbar_wait(bar, 0);
  const long long base = w0 - (long long)shift;
  if (b.zb > base)  // windows that reach back before the attach point read zeros there
    for (unsigned i = tid; i < need; i += BK_THREADS)
      if (base + (long long)i < b.zb) xs[i] = make_float2(0.f, 0.f);
  __syncthreads();
  const int KP = min(K, T1), rs = K + 1;
  for (int e = tid; e < nf * KP; e += BK_THREADS) {
    const int f = e / KP, p = e - f * KP;
    const float2 *x = xs + shift + f * D1 + p;
    const float *h = ts + p;
    float2 acc = make_float2(0.f, 0.f);
    for (int j = 0; j < T1 - p; j += K) {
      const float2 xv = x[j];
      const float hv = h[j];
      acc.x = fmaf(xv.x, hv, acc.x);
      acc.y = fmaf(xv.y, hv, acc.y);
    }
    v[f * rs + p] = acc;
  }
  __syncthreads();
  for (int e = tid; e < nch * BK_F; e += BK_THREADS) {
    const int c = e / BK_F, f = e - c * BK_F;
    if (f >= nf) continue;
    const int2 ch = b.chans[c0 + c];
    const int kk = ch.x;
    const int r = (int)(((long long)b.r0 + (long long)(f0 + f) * D1) % K);
    int t = (int)(((long long)kk * r) % K);
    const float2 *vf = v + f * rs;
    float2 acc = make_float2(0.f, 0.f);
    for (int p = 0; p < KP; p++) {
      const float2 a = vf[p], w = tw[t];
      acc.x = fmaf(a.x, w.x, acc.x);
      acc.x = fmaf(-a.y, w.y, acc.x);
      acc.y = fmaf(a.x, w.y, acc.y);
      acc.y = fmaf(a.y, w.x, acc.y);
      t += kk;
      if (t >= K) t -= K;
    }
    out[ch.y + f0 + f] = acc;
  }
}

// ---------------------------------------------------------------------------
// FFT bank sub-bands (xlg_add_bank_fft).  The channels are the bank's above; only the channel stage differs: a
// K-point FFT, K = 2 * D1 a power of two up to 4096.  Phase 1's sums v[m][p] (p < min(K, T1), the direct bank's
// two fmaf chains over q ascending from +0; zero for T1 <= p < K) are placed at u[(p + r_m) mod K], an exact
// permutation, so that
//     y_k[m] = sum_{p < K} u[p] * W[(k p) mod K]
// which a decimation-in-frequency FFT computes in place: radix-4 stages at lengths L = K, K/4, ... while L >= 4,
// then one radix-2 stage at L = 2 when log2 K is odd.  The radix-4 butterfly at length L, for every block of L
// and j < L/4, reads a_q = u[b + j + q L/4] and writes (component-wise float adds, in this order)
//     t0 = a0 + a2, t1 = a0 - a2, t2 = a1 + a3, t3 = a1 - a3
//     y0 = t0 + t2, y1 = (t1.x + t3.y, t1.y - t3.x), y2 = t0 - t2, y3 = (t1.x - t3.y, t1.y + t3.x)
//     u[b + j + q L/4] = y0 for q = 0, y_q * W[q j K / L] for q = 1, 2, 3
// the radix-2 butterfly (a0, a1) -> (a0 + a1, a0 - a1), and every product y * w is
//     (fmaf(-y.y, w.y, y.x * w.x), fmaf(y.y, w.x, y.x * w.y))     (rounded products, no contraction)
// W is the direct bank's table read at stride K / L, so the quarter turns stay exact.  Channel k then lies at
// the digit reversal of k mod K (bank_fft_pos in xlating_group.cu), which the channel table carries.  The
// spectra use the same transform at K up to 65536 (the wide ones in two passes, spectrum_wide_a/b_kernel).
// ---------------------------------------------------------------------------
constexpr int BF_THREADS = 256;
constexpr int BF_N = 2048;  // sums per CTA: BF_N / K frames, one frame at K = 4096
__host__ __device__ constexpr int bank_fft_frames(int K) { return K >= BF_N ? 1 : BF_N / K; }
__host__ __device__ constexpr size_t bank_fft_smem(int K) { return (size_t)bank_fft_frames(K) * K * 8; }
// taps: a phase's chain is at most max(16, 16384 / K) terms long
__host__ __device__ constexpr long long bank_fft_max_taps(int K) { return 16LL * K > 16384 ? 16LL * K : 16384; }

__device__ __forceinline__ float2 cmul_tw(float2 y, float2 w) {
  return make_float2(fmaf(-y.y, w.y, __fmul_rn(y.x, w.x)), fmaf(y.y, w.x, __fmul_rn(y.x, w.y)));
}

// The in-place decimation-in-frequency FFT of nf rows of K (a power of two, lk = log2 K) in shared memory u, in
// the order the header above states, tw[j] = e^{-2 pi i j / K}; every stage ends with a barrier
template <int THREADS>
__device__ __forceinline__ void fft_dif_rows(float2 *u, int nf, int K, int lk, const float2 *tw, int tid) {
  int L = K;
  for (; L >= 4; L >>= 2) {
    const int q4 = L >> 2, s = K / L;
    for (int e = tid; e < nf * (K >> 2); e += THREADS) {
      const int f = e >> (lk - 2), i = e & ((K >> 2) - 1), j = i & (q4 - 1);
      float2 *x = u + (f << lk) + 4 * (i - j) + j;
      const float2 a0 = x[0], a1 = x[q4], a2 = x[2 * q4], a3 = x[3 * q4];
      const float2 t0 = make_float2(a0.x + a2.x, a0.y + a2.y), t1 = make_float2(a0.x - a2.x, a0.y - a2.y);
      const float2 t2 = make_float2(a1.x + a3.x, a1.y + a3.y), t3 = make_float2(a1.x - a3.x, a1.y - a3.y);
      x[0] = make_float2(t0.x + t2.x, t0.y + t2.y);
      x[q4] = cmul_tw(make_float2(t1.x + t3.y, t1.y - t3.x), __ldg(tw + j * s));
      x[2 * q4] = cmul_tw(make_float2(t0.x - t2.x, t0.y - t2.y), __ldg(tw + 2 * j * s));
      x[3 * q4] = cmul_tw(make_float2(t1.x - t3.y, t1.y + t3.x), __ldg(tw + 3 * j * s));
    }
    __syncthreads();
  }
  if (L == 2) {
    for (int e = tid; e < nf * (K >> 1); e += THREADS) {
      float2 *x = u + 2 * e;
      const float2 a0 = x[0], a1 = x[1];
      x[0] = make_float2(a0.x + a1.x, a0.y + a1.y);
      x[1] = make_float2(a0.x - a1.x, a0.y - a1.y);
    }
    __syncthreads();
  }
}

// Phase p's polyphase sum of the frame whose window starts at stream position w: two fmaf chains from +0 over
// the taps j = p, p + K, ... below T1, the window's samples before the attach point read as zero (taps and ring
// through the L1: T1 is too long to stage)
__device__ __forceinline__ float2 bank_phase_sum(const BankBlk &b, const float2 *__restrict__ ring, long long w,
                                                 int p) {
  float2 acc = make_float2(0.f, 0.f);
  for (int j = p; j < b.T1; j += b.K) {
    const long long pos = w + j;
    const float2 xv = pos < b.zb ? make_float2(0.f, 0.f) : ring[(unsigned)((unsigned long long)pos) & b.mask];
    const float hv = __ldg(b.taps + j);
    acc.x = fmaf(xv.x, hv, acc.x);
    acc.y = fmaf(xv.y, hv, acc.y);
  }
  return acc;
}

// CTA (x, b) computes frames [x F, x F + F) of bank b, F = bank_fft_frames(K): the rotated sums of each frame in
// a row of K in shared memory (taps and window read through the L1: T1 is too long to stage), the FFT of every
// row, then the materialised channels' samples, a channel's frames consecutively.  chans[c].x is the channel's
// position in the transformed row.
__global__ void __launch_bounds__(BF_THREADS)
bank_fft_cf32_kernel(const BankBlk *__restrict__ blk, const float2 *__restrict__ ring, float2 *__restrict__ out) {
  extern __shared__ __align__(16) float2 u[];
  const BankBlk b = blk[blockIdx.y];
  const int K = b.K, F = bank_fft_frames(K);
  const int f0 = blockIdx.x * F;
  if (f0 >= b.n1) return;
  const int nf = min(F, b.n1 - f0), tid = threadIdx.x;
  const int lk = 31 - __clz(K);
  for (int e = tid; e < nf * K; e += BF_THREADS) {
    const int f = e >> lk, p = e & (K - 1);
    const float2 acc = bank_phase_sum(b, ring, b.first + (long long)(f0 + f) * b.D1, p);
    const int r = (int)(((long long)b.r0 + (long long)(f0 + f) * b.D1) & (K - 1));
    u[(f << lk) + ((p + r) & (K - 1))] = acc;
  }
  __syncthreads();
  fft_dif_rows<BF_THREADS>(u, nf, K, lk, b.tw, tid);
  for (int e = tid; e < b.n_ch * F; e += BF_THREADS) {
    const int c = e / F, f = e - c * F;
    if (f >= nf) continue;
    const int2 ch = b.chans[c];
    out[ch.y + f0 + f] = u[(f << lk) + ch.x];
  }
}

// ---------------------------------------------------------------------------
// Chirp-z banks (xlg_add_bank_any, K = 2 * D1 even, at most 4096 and not a power of two).  The channels are the
// bank's above; the channel stage is the K-point DFT of the FFT bank's placed sums u (u[(p + r_m) mod K] = v[m][p],
// r_m = (s_m - P) mod K in 64 bits, taken with %), computed by Bluestein's identity kn = (k^2 + n^2 - (k - n)^2) / 2
// as a circular convolution of length M = next_pow2(2K - 1) (16 to 8192).  With c[n] = e^{-i pi (n^2 mod 2K) / K}
// (period K: K is even) and Bh the chirp-z spectrum's table at W = K (the M-point DFT of conj(c[|m|]), |m| < K,
// wrapped mod M, times 1/M, in position order), in this order (cmul_tw for every complex product):
//   a[n] = cmul_tw(u[n], c[n]) for n < K, +0 for K <= n < M
//   A    = fft_dif_rows' M-point transform of a, in position order
//   Y[p] = cmul_tw(A[p], Bh[p]);  y[bin(p)] = (Y[p].x, -Y[p].y)   (conj(Y) in natural order; bin = fft_bin)
//   v    = the same M-point transform of y, in position order
//   y_k  = cmul_tw((v[q].x, -v[q].y), c[k mod K]),  q = bank_fft_pos(k mod K, M)
// All tables are built in double on the host and rounded once (czt_tables in xlating_group.cu).  FP32
// instructions per frame: 2 xlg_bank_fft_flops(M) + 4 K + 4 M + 4 C for C materialised channels.
// ---------------------------------------------------------------------------
constexpr int BZ_THREADS = 256;
constexpr int BZ_N = 8192;                // points per CTA: BZ_N / M frames, one frame at M = 8192
constexpr int BZ_ST = BZ_N / BZ_THREADS;  // float2 a thread holds while conj(Y) moves to natural order
__host__ __device__ constexpr int bank_czt_m(int K) {  // next_pow2(2K - 1)
  int m = 1;
  while (m < 2 * K - 1) m <<= 1;
  return m;
}
__host__ __device__ constexpr int bank_czt_frames(int M) { return BZ_N / M; }
__host__ __device__ constexpr size_t bank_czt_smem(int M) { return (size_t)bank_czt_frames(M) * M * 8; }

// the bin whose transform output lies at position p of a row of M = 2^lm: bank_fft_pos's inverse (the base-4
// digits of p, most significant first, are the bin's from the least significant, then the radix-2 stage's bit)
__device__ __forceinline__ int fft_bin(int p, int lm) {
  int k = 0, sh = 0, l = lm;
  for (; l >= 2; l -= 2, sh += 2) k |= ((p >> (l - 2)) & 3) << sh;
  return l == 1 ? k | ((p & 1) << sh) : k;
}

// CTA (x, b) computes frames [x F, x F + F) of chirp-z bank b, F = bank_czt_frames(M), each in a row of M in
// shared memory.  b.tw holds the M-point table, then c (K) and Bh (M); chans[c].x is the channel's position in
// the second transform's row in its low 16 bits and k mod K above them.  conj(Y) reaches natural order through
// registers: each thread holds its BZ_ST points across a barrier, then stores them at their bins.
__global__ void __launch_bounds__(BZ_THREADS, 2)
bank_czt_cf32_kernel(const BankBlk *__restrict__ blk, const float2 *__restrict__ ring, float2 *__restrict__ out) {
  extern __shared__ __align__(16) float2 u[];
  const BankBlk b = blk[blockIdx.y];
  const int K = b.K, M = bank_czt_m(K), F = bank_czt_frames(M);
  const int f0 = blockIdx.x * F;
  if (f0 >= b.n1) return;
  const int nf = min(F, b.n1 - f0), tid = threadIdx.x, lm = 31 - __clz(M);
  const float2 *chirp = b.tw + M, *kern = chirp + K;
  for (int e = tid; e < nf * M; e += BZ_THREADS) {
    const int f = e >> lm, n = e & (M - 1);
    if (n >= K) {
      u[e] = make_float2(0.f, 0.f);
      continue;
    }
    const int r = (int)(((long long)b.r0 + (long long)(f0 + f) * b.D1) % K);
    const int p = n >= r ? n - r : n - r + K;  // the phase placed at n
    u[e] = cmul_tw(bank_phase_sum(b, ring, b.first + (long long)(f0 + f) * b.D1, p), __ldg(chirp + n));
  }
  __syncthreads();
  fft_dif_rows<BZ_THREADS>(u, nf, M, lm, b.tw, tid);
  float2 st[BZ_ST];
#pragma unroll
  for (int i = 0; i < BZ_ST; i++) {
    const int e = tid + i * BZ_THREADS;
    if (e < nf * M) {
      const float2 y = cmul_tw(u[e], __ldg(kern + (e & (M - 1))));
      st[i] = make_float2(y.x, -y.y);
    }
  }
  __syncthreads();
#pragma unroll
  for (int i = 0; i < BZ_ST; i++) {
    const int e = tid + i * BZ_THREADS;
    if (e < nf * M) u[(e & ~(M - 1)) + fft_bin(e & (M - 1), lm)] = st[i];
  }
  __syncthreads();
  fft_dif_rows<BZ_THREADS>(u, nf, M, lm, b.tw, tid);
  for (int e = tid; e < b.n_ch * F; e += BZ_THREADS) {
    const int c = e / F, f = e - c * F;
    if (f >= nf) continue;
    const int2 ch = b.chans[c];
    const float2 v = u[(f << lm) + (ch.x & 0xffff)];
    out[ch.y + f0 + f] = cmul_tw(make_float2(v.x, -v.y), __ldg(chirp + (ch.x >> 16)));
  }
}

// ---------------------------------------------------------------------------
// Spectrum rows (xlg_add_spectrum, and xlg_add_client_spectrum / xlg_add_subband_spectrum, whose stream x is a
// source's output, appended by cascade_append_kernel to a ring of the spectrum's own and counted from its attach,
// P = 0).  A spectrum of width W, F frames per row and S samples skipped per row, attached at stream position P,
// has period R = F W + S; row r is the max-hold over the frames
// x[P + r R + f W ... + W), f < F, of the power of each DFT bin (src/spectrogram/spectrogram.c).  Per frame and
// bin, with X the frame's DFT and inv = 1/W rounded to float once, in this order (rounded operations, no
// contraction):
//     c = (X.x * inv, X.y * inv),   p = (c.x * c.x + c.y * c.y) + 1e-20f
// X comes from one of two channel stages:
//   FFT path (W a power of two, 4 <= W <= 4096): the frame in natural order through fft_dif_rows, the FFT bank's
//     radix-4 (then radix-2) decimation in frequency with the twiddle table read at stride W / L; bin k then lies
//     at position bank_fft_pos(k, W) of the row (digit reversal).  FP32 instructions per frame:
//     xlg_bank_fft_flops(W) + 6 W.
//   Direct path (every other W <= 4096): X_k = sum_{n < W} x[n] W_tab[(k n) mod W], two fmaf chains from +0 over
//     n ascending, acc.x = fmaf(-x.y, w.y, fmaf(x.x, w.x, acc.x)), acc.y = fmaf(x.y, w.x, fmaf(x.x, w.y, acc.y)):
//     W complex MACs per input sample, 4 W^2 + 6 W FP32 instructions per frame.
// The table is the banks' e^{-2 pi i m / W}, built in double by quarter turns and rounded once.  Each p goes to
// the spectrum's hold row of its frame's row by atomicMax on its bit pattern: p >= 1e-20 > 0, so integer order
// is float order and the max does not depend on the order CTAs run in (0, the empty hold, is below every p).
// The hold has NR rows used round-robin by row number (NR exceeds the rows a block touches); the emit pass reads
// each row the block completed through the row map (out[j] = hold[map[j]]: the reference's half swap, then the
// FFT path's digit reversal), writes v (XLG_SPECTRUM_POWER) or 10 * log10f(v), and zeroes what it read.
// The two channel stages (spectrum_fft_kernel, spectrum_direct_kernel) share their bodies with the extended
// spectra's, after SpecExt below.  Powers of two from 8192 to 65536 are the wide spectra at the end of this file:
// the FFT path's X at K = W.
// ---------------------------------------------------------------------------
constexpr int SPEC_THREADS = 256;
constexpr int SPEC_MAX_W = 4096;

struct SpecBlk {          // one spectrum, this block
  const float2 *tw;       // e^{-2 pi i m / W}, m < W
  const int *map;         // output bin j reads hold position map[j]
  unsigned *hold;         // NR rows of W: each row's running max (float bits), zero when empty
  float *out;             // its rows in the slot's arena: n_rows x W
  long long base;         // stream position of the first row this block touches: P + r R
  unsigned mask;          // capacity - 1 of the ring it reads
  int W, F, R, NR;
  unsigned f0;            // frames of that row done by earlier blocks
  int n_frames;           // frames completed by this block
  int n_rows;             // rows completed by this block (the first is row r)
  int slot0;              // hold row of row r: r mod NR
  int power;              // XLG_SPECTRUM_POWER: linear rows, else dB
  float inv_w;
};
// (the ring each entry reads comes in a table of its own, rings[s]: the group's input ring or the spectrum's source
// ring, whose capacity - 1 is the entry's mask -- a pointer more in SpecBlk would change spectrum_emit_kernel too)

__host__ __device__ constexpr bool spec_fft(int W) { return W >= 4 && W <= SPEC_MAX_W && (W & (W - 1)) == 0; }
// direct path: frames per CTA (W < SPEC_THREADS: one thread per (frame, bin)), CTAs per frame along y
__host__ __device__ constexpr int spec_direct_frames(int W) { return W >= SPEC_THREADS ? 1 : SPEC_THREADS / W; }
__host__ __device__ constexpr int spec_direct_groups(int W) { return (W + SPEC_THREADS - 1) / SPEC_THREADS; }
__host__ __device__ constexpr size_t spec_direct_smem(int W) {
  return ((size_t)spec_direct_frames(W) * W + W) * sizeof(float2);
}

// frame j of this block: its first sample's stream position and its hold row
struct SpecFrame {
  long long pos;
  int hold_row;
};
__device__ __forceinline__ SpecFrame spec_frame(const SpecBlk &b, int j) {
  const unsigned g = b.f0 + (unsigned)j, rr = g / (unsigned)b.F, ff = g - rr * (unsigned)b.F;
  return {b.base + (long long)rr * b.R + (long long)ff * b.W, (int)(((unsigned)b.slot0 + rr) % (unsigned)b.NR)};
}

__device__ __forceinline__ unsigned spec_power(float2 X, float inv) {
  const float cx = __fmul_rn(X.x, inv), cy = __fmul_rn(X.y, inv);
  return __float_as_uint(__fadd_rn(__fadd_rn(__fmul_rn(cx, cx), __fmul_rn(cy, cy)), 1e-20f));
}

// CTA (x, s) writes values [x 256, x 256 + 256) of the n_rows x W values of the rows spectrum s completed in
// this block, and empties what it read of the hold
__global__ void __launch_bounds__(SPEC_THREADS) spectrum_emit_kernel(const SpecBlk *__restrict__ blk) {
  const SpecBlk b = blk[blockIdx.y];
  const int e = blockIdx.x * SPEC_THREADS + threadIdx.x;
  if (e >= b.n_rows * b.W) return;
  const int i = e / b.W, j = e - i * b.W;
  unsigned *hold = b.hold + (size_t)((b.slot0 + i) % b.NR) * b.W + b.map[j];
  const float v = __uint_as_float(*hold);
  *hold = 0u;
  b.out[e] = b.power ? v : __fmul_rn(10.f, log10f(v));
}

// ---------------------------------------------------------------------------
// Extended spectra (xlg_add_spectrum_ex): a hop H between frame starts, a window and a mean.  Row period
// R = (F - 1) H + W + S; row r covers the frames x[P + r R + f H ... + W), f < F.  Each frame is windowed before
// the transform, z[n] = (x[n].x * w[n], x[n].y * w[n]) (one rounded multiply each; no window: z = x), and goes
// through the same channel stage, spec_power and hold as above: spectrum_fft_ext_kernel and
// spectrum_direct_ext_kernel are the EXT = true instances of the two stages' bodies below, the plain kernels the
// EXT = false ones.  A max spectrum folds by atomicMax as above.  A
// mean spectrum's channel stage stores each frame's powers (position space, as the hold) in the spectrum's frame
// buffer, row j of it for frame j of this block; spectrum_fold_kernel then adds them into the hold in frame order,
//     s = +0;  s = s + p_f for f = 0 .. F - 1 (rounded adds, one frame after the other, across blocks in block order)
// and divides a completed row once, v = s / float(F) (correctly rounded).  The hold carries s between blocks as
// float bits (the empty hold, 0, is +0).  spectrum_emit_kernel then writes and empties the row as for any spectrum.
// The entries are the tail of the block's SpecBlk table, SpecExt holds what only they need (the plain kernels read
// none).
// ---------------------------------------------------------------------------
struct SpecExt {
  const float *win;  // W weights, or nullptr: no window
  float *fbuf;       // mean: the frames' powers, a row of W per frame of this block; max: nullptr
  int H;             // hop
  int mean;
};

__device__ __forceinline__ long long spec_frame_pos(const SpecBlk &b, int H, int j) {
  const unsigned g = b.f0 + (unsigned)j, rr = g / (unsigned)b.F, ff = g - rr * (unsigned)b.F;
  return b.base + (long long)rr * b.R + (long long)ff * H;
}

__device__ __forceinline__ float2 spec_load(const float2 *__restrict__ ring, unsigned mask, long long pos,
                                            const float *__restrict__ win, int n) {
  const float2 v = ring[(unsigned)((unsigned long long)pos) & mask];
  if (win == nullptr) return v;
  const float w = __ldg(win + n);
  return make_float2(__fmul_rn(v.x, w), __fmul_rn(v.y, w));
}

// The FFT path: CTA (x, s) transforms frames [x F, x F + F) of spectrum s, F = bank_fft_frames(W), one row of W
// each in shared memory, and folds their powers into the hold (below W = 256 a CTA first takes the max over runs of
// its frames) or, for a mean, stores them to the frame buffer.  EXT = false: a plain spectrum, hop W, no window
// and the max, without reading a SpecExt.
template <bool EXT>
__device__ __forceinline__ void spectrum_fft_stage(const SpecBlk *__restrict__ blk,
                                                   const float2 *const *__restrict__ rings,
                                                   const SpecExt *__restrict__ ext) {
  extern __shared__ __align__(16) float2 u[];
  const SpecBlk b = blk[blockIdx.y];
  const SpecExt x = EXT ? ext[blockIdx.y] : SpecExt{nullptr, nullptr, b.W, 0};
  const float2 *__restrict__ ring = rings[blockIdx.y];
  if (!spec_fft(b.W)) return;
  const int W = b.W, F = bank_fft_frames(W);
  const int j0 = blockIdx.x * F;
  if (j0 >= b.n_frames) return;
  const int nf = min(F, b.n_frames - j0), tid = threadIdx.x, lw = 31 - __clz(W);
  for (int e = tid; e < nf * W; e += SPEC_THREADS) {
    const int n = e & (W - 1);
    u[e] = spec_load(ring, b.mask, spec_frame_pos(b, x.H, j0 + (e >> lw)) + n, x.win, n);
  }
  __syncthreads();
  fft_dif_rows<SPEC_THREADS>(u, nf, W, lw, b.tw, tid);
  if (EXT && x.mean) {
    float *fb = x.fbuf + (size_t)j0 * W;
    for (int e = tid; e < nf * W; e += SPEC_THREADS) fb[e] = __uint_as_float(spec_power(u[e], b.inv_w));
    return;
  }
  if (W >= SPEC_THREADS) {  // at most 8 frames: one atomicMax per power
    for (int e = tid; e < nf * W; e += SPEC_THREADS) {
      const int h = spec_frame(b, j0 + (e >> lw)).hold_row;
      atomicMax(b.hold + (size_t)h * W + (e & (W - 1)), spec_power(u[e], b.inv_w));
    }
    return;
  }
  // narrow rows, many frames: the powers' bits in place of the transformed rows, then a thread takes one position
  // over a run of frames, keeps their max and issues one atomicMax per hold row the run meets (the max does not
  // depend on the order)
  unsigned *pw = reinterpret_cast<unsigned *>(u);
  for (int e = tid; e < nf * W; e += SPEC_THREADS) pw[2 * e] = spec_power(u[e], b.inv_w);
  __syncthreads();
  // (W divides SPEC_THREADS: thread tid takes position tid mod W over run tid / W)
  const int runs = SPEC_THREADS / W, per = (nf + runs - 1) / runs;
  const int q = tid & (W - 1), f0 = (tid >> lw) * per, f1 = min(nf, f0 + per);
  int h = -1;
  unsigned m = 0u;
  for (int f = f0; f < f1; f++) {
    const int hf = spec_frame(b, j0 + f).hold_row;
    if (hf != h) {
      if (h >= 0) atomicMax(b.hold + (size_t)h * W + q, m);
      h = hf;
      m = 0u;
    }
    m = max(m, pw[2 * ((f << lw) + q)]);
  }
  if (h >= 0) atomicMax(b.hold + (size_t)h * W + q, m);
}

// The direct path: CTA (x, y, s) computes bins [y 256, y 256 + 256) of frames [x Fd, x Fd + Fd) of spectrum s,
// Fd = spec_direct_frames(W): the frames and the table in shared memory, one bin of one frame per thread.  EXT as
// above.
template <bool EXT>
__device__ __forceinline__ void spectrum_direct_stage(const SpecBlk *__restrict__ blk,
                                                      const float2 *const *__restrict__ rings,
                                                      const SpecExt *__restrict__ ext) {
  extern __shared__ __align__(16) float2 sm[];
  const SpecBlk b = blk[blockIdx.z];
  const SpecExt xe = EXT ? ext[blockIdx.z] : SpecExt{nullptr, nullptr, b.W, 0};
  const float2 *__restrict__ ring = rings[blockIdx.z];
  const int W = b.W;
  if (spec_fft(W)) return;
  const int Fd = spec_direct_frames(W), j0 = blockIdx.x * Fd, k0 = blockIdx.y * SPEC_THREADS;
  if (j0 >= b.n_frames || k0 >= W) return;
  const int nf = min(Fd, b.n_frames - j0), tid = threadIdx.x;
  float2 *tw = sm, *xs = sm + W;
  for (int i = tid; i < W; i += SPEC_THREADS) tw[i] = b.tw[i];
  for (int e = tid; e < nf * W; e += SPEC_THREADS) {
    const int f = e / W;
    if constexpr (EXT) {
      const int n = e - f * W;
      xs[e] = spec_load(ring, b.mask, spec_frame_pos(b, xe.H, j0 + f) + n, xe.win, n);
    } else {  // (the plain kernel's own load: through spec_frame_pos and spec_load it compiles to more instructions)
      xs[e] = ring[(unsigned)((unsigned long long)(spec_frame(b, j0 + f).pos + (e - f * W))) & b.mask];
    }
  }
  __syncthreads();
  const int wb = min(W, SPEC_THREADS), f = tid / wb, k = k0 + tid - f * wb;
  if (f >= nf || k >= W) return;
  const float2 *x = xs + f * W;
  float2 acc = make_float2(0.f, 0.f);
  int t = 0;
  for (int n = 0; n < W; n++) {
    const float2 a = x[n], w = tw[t];
    acc.x = fmaf(a.x, w.x, acc.x);
    acc.x = fmaf(-a.y, w.y, acc.x);
    acc.y = fmaf(a.x, w.y, acc.y);
    acc.y = fmaf(a.y, w.x, acc.y);
    t += k;
    if (t >= W) t -= W;
  }
  const unsigned p = spec_power(acc, b.inv_w);
  if (EXT && xe.mean)
    xe.fbuf[(size_t)(j0 + f) * W + k] = __uint_as_float(p);
  else
    atomicMax(b.hold + (size_t)spec_frame(b, j0 + f).hold_row * W + k, p);
}

__global__ void __launch_bounds__(SPEC_THREADS)
spectrum_fft_kernel(const SpecBlk *__restrict__ blk, const float2 *const *__restrict__ rings) {
  spectrum_fft_stage<false>(blk, rings, nullptr);
}

__global__ void __launch_bounds__(SPEC_THREADS)
spectrum_direct_kernel(const SpecBlk *__restrict__ blk, const float2 *const *__restrict__ rings) {
  spectrum_direct_stage<false>(blk, rings, nullptr);
}

__global__ void __launch_bounds__(SPEC_THREADS)
spectrum_fft_ext_kernel(const SpecBlk *__restrict__ blk, const float2 *const *__restrict__ rings,
                        const SpecExt *__restrict__ ext) {
  spectrum_fft_stage<true>(blk, rings, ext);
}

__global__ void __launch_bounds__(SPEC_THREADS)
spectrum_direct_ext_kernel(const SpecBlk *__restrict__ blk, const float2 *const *__restrict__ rings,
                           const SpecExt *__restrict__ ext) {
  spectrum_direct_stage<true>(blk, rings, ext);
}

// CTA (x, s) folds values [x 256, x 256 + 256) of the rows x W that mean spectrum s's frames of this block touch:
// thread (i, q) adds position q of the block's frames in row i, in frame order, to hold row i and divides the sum
// by float(F) if the block completes that row (i < n_rows)
__global__ void __launch_bounds__(SPEC_THREADS)
spectrum_fold_kernel(const SpecBlk *__restrict__ blk, const SpecExt *__restrict__ ext) {
  const SpecBlk b = blk[blockIdx.y];
  const SpecExt x = ext[blockIdx.y];
  if (!x.mean) return;
  const int W = b.W, touched = (int)((b.f0 + (unsigned)b.n_frames - 1u) / (unsigned)b.F) + 1;
  const int e = blockIdx.x * SPEC_THREADS + threadIdx.x;
  if (e >= touched * W) return;
  const int i = e / W, q = e - i * W;
  const long long first = (long long)i * b.F - (long long)b.f0;  // row i's frame 0, as a frame of this block
  const int j1 = (int)min((long long)b.n_frames, first + b.F);
  unsigned *hold = b.hold + (size_t)((b.slot0 + i) % b.NR) * W + q;
  float s = __uint_as_float(*hold);
  for (int j = (int)max(0ll, first); j < j1; j++) s = __fadd_rn(s, x.fbuf[(size_t)j * W + q]);
  *hold = __float_as_uint(i < b.n_rows ? __fdiv_rn(s, (float)b.F) : s);
}

// ---------------------------------------------------------------------------
// Wide spectra (W a power of two from 8192 to SPEC_WIDE_MAX_W = 65536, plain or extended): X is fft_dif_rows'
// transform at K = W, bin k at bank_fft_pos(k, W), but a frame does not fit in one CTA's shared memory.  In the
// decimation in frequency, after the first s radix-4 stages (s = 1 at W <= 16384, s = 2 above) each contiguous
// chunk of C = W / 4^s points (2048 or 4096) only meets itself, and its remaining stages at L <= C read the W-point
// table at stride W / L = (W / C)(C / L): they are fft_dif_rows at K = C with the C-point table, twiddle_table(C),
// which is twiddle_table(W) at stride W / C bit for bit (the double angles differ by a power of two).  So:
//   spectrum_wide_a_kernel: thread (frame j, column i < C) loads the 4^s points i + m C of frame j (spec_load: the
//     hop and the window), runs the first s stages' butterflies on them in registers, each with fft_dif_rows'
//     operations in its order and the W table at stride W / L, and stores them at the same positions of row j of
//     the spectrum's scratch (HBM, frames of this block x W, read back from L2).
//   spectrum_wide_b_kernel: CTA (frame j, chunk c) runs fft_dif_rows on chunk c of row j in shared memory
//     (C float2: 32 KiB at C = 4096) and folds the powers as spectrum_fft_ext_kernel does: atomicMax into the hold
//     row, or a store to the mean's frame buffer.  Position c C + t is the W-point transform's own position.
// The entries are the tail of the block's SpecBlk table, [plain | extended | wide], outside every other channel
// kernel's grid.  Each has a SpecExt (a plain one: H = W, no window, the max), so that spectrum_fold_kernel and
// spectrum_emit_kernel finish their rows unchanged, and a SpecWide.
// ---------------------------------------------------------------------------
constexpr int SPEC_WIDE_MAX_W = 65536;
__host__ __device__ constexpr bool spec_wide(int W) {
  return W > SPEC_MAX_W && W <= SPEC_WIDE_MAX_W && (W & (W - 1)) == 0;
}
// pass A's radix-4 stages, and the chunk length after them
__host__ __device__ constexpr int spec_wide_stages(int W) { return W > 16384 ? 2 : 1; }
__host__ __device__ constexpr int spec_wide_chunk(int W) { return W >> (2 * spec_wide_stages(W)); }
constexpr size_t SPEC_WIDE_SMEM = 4096 * sizeof(float2);  // pass B: the largest chunk

struct SpecWide {
  float2 *scratch;     // pass A's rows: a row of W per frame of this block
  const float2 *tw_c;  // the C-point table
};

// fft_dif_rows' radix-4 butterfly on (a0, a1, a2, a3) = u[j + q L/4], in place, twiddles tw[q j s]
__device__ __forceinline__ void dif_bfly4(float2 &a0, float2 &a1, float2 &a2, float2 &a3, const float2 *tw, int js) {
  const float2 t0 = make_float2(a0.x + a2.x, a0.y + a2.y), t1 = make_float2(a0.x - a2.x, a0.y - a2.y);
  const float2 t2 = make_float2(a1.x + a3.x, a1.y + a3.y), t3 = make_float2(a1.x - a3.x, a1.y - a3.y);
  a0 = make_float2(t0.x + t2.x, t0.y + t2.y);
  a1 = cmul_tw(make_float2(t1.x + t3.y, t1.y - t3.x), __ldg(tw + js));
  a2 = cmul_tw(make_float2(t0.x - t2.x, t0.y - t2.y), __ldg(tw + 2 * js));
  a3 = cmul_tw(make_float2(t1.x - t3.y, t1.y + t3.x), __ldg(tw + 3 * js));
}

// pass A's stages, in place, on a[m] = the point i + m C (m < 4^NS) of a row of the K-point transform, tw the K-point
// table: stage 1 (L = K) on columns i + r C, r < 4^(NS-1), then, for NS = 2, stage 2 (L = K / 4, stride 4) on each
// quarter's points
template <int NS>
__device__ __forceinline__ void pass_a_stages(float2 (&a)[NS == 1 ? 4 : 16], const float2 *__restrict__ tw, int i,
                                              int C) {
  constexpr int Q = NS == 1 ? 1 : 4;
#pragma unroll
  for (int r = 0; r < Q; r++) dif_bfly4(a[r], a[r + Q], a[r + 2 * Q], a[r + 3 * Q], tw, i + r * C);
  if (NS == 2) {
#pragma unroll
    for (int q = 0; q < 4; q++) dif_bfly4(a[4 * q], a[4 * q + 1], a[4 * q + 2], a[4 * q + 3], tw, 4 * i);
  }
}

// pass A on the 4^NS points i + m C of a frame starting at pos (spec_load: the hop and the window)
template <int NS>
__device__ __forceinline__ void spec_wide_pass_a(const float2 *__restrict__ ring, unsigned mask, long long pos,
                                                 const float *__restrict__ win, const float2 *__restrict__ tw,
                                                 float2 *__restrict__ row, int i, int C) {
  constexpr int M = NS == 1 ? 4 : 16;
  float2 a[M];
#pragma unroll
  for (int m = 0; m < M; m++) a[m] = spec_load(ring, mask, pos + i + m * C, win, i + m * C);
  pass_a_stages<NS>(a, tw, i, C);
#pragma unroll
  for (int m = 0; m < M; m++) row[i + m * C] = a[m];
}

// pass B's start: the C points of a chunk at src into shared memory u, then fft_dif_rows on them with the C-point
// table (the barriers included)
__device__ __forceinline__ void spec_chunk_fft(float2 *u, const float2 *src, int C, int lc, const float2 *tw_c,
                                               int tid) {
  for (int t = tid; t < C; t += SPEC_THREADS) u[t] = src[t];
  __syncthreads();
  fft_dif_rows<SPEC_THREADS>(u, 1, C, lc, tw_c, tid);
}

// CTA (x, s): threads [x 256, x 256 + 256) of wide spectrum s's frames x C columns, C = spec_wide_chunk(W)
__global__ void __launch_bounds__(SPEC_THREADS)
spectrum_wide_a_kernel(const SpecBlk *__restrict__ blk, const float2 *const *__restrict__ rings,
                       const SpecExt *__restrict__ ext, const SpecWide *__restrict__ wide) {
  const SpecBlk b = blk[blockIdx.y];
  const SpecExt x = ext[blockIdx.y];
  const float2 *__restrict__ ring = rings[blockIdx.y];
  const int W = b.W, C = spec_wide_chunk(W), lc = 31 - __clz(C);
  const int e = blockIdx.x * SPEC_THREADS + threadIdx.x, j = e >> lc, i = e & (C - 1);
  if (j >= b.n_frames) return;
  float2 *row = wide[blockIdx.y].scratch + (size_t)j * W;
  const long long pos = spec_frame_pos(b, x.H, j);
  if (spec_wide_stages(W) == 1)
    spec_wide_pass_a<1>(ring, b.mask, pos, x.win, b.tw, row, i, C);
  else
    spec_wide_pass_a<2>(ring, b.mask, pos, x.win, b.tw, row, i, C);
}

// CTA (x, s): chunk x mod 4^s of frame x / 4^s of wide spectrum s (at least four CTAs per SM: without that bound
// ptxas aims at eight, 32 registers, and spills)
__global__ void __launch_bounds__(SPEC_THREADS, 4)
spectrum_wide_b_kernel(const SpecBlk *__restrict__ blk, const SpecExt *__restrict__ ext,
                       const SpecWide *__restrict__ wide) {
  extern __shared__ __align__(16) float2 u[];
  const SpecBlk b = blk[blockIdx.y];
  const SpecExt x = ext[blockIdx.y];
  const SpecWide wd = wide[blockIdx.y];
  const int W = b.W, ls = 2 * spec_wide_stages(W), C = W >> ls, lc = 31 - __clz(C), tid = threadIdx.x;
  const int j = blockIdx.x >> ls, c0 = (blockIdx.x & ((1 << ls) - 1)) * C;
  if (j >= b.n_frames) return;
  const size_t off = (size_t)j * W + c0;
  spec_chunk_fft(u, wd.scratch + off, C, lc, wd.tw_c, tid);
  if (x.mean) {
    for (int t = tid; t < C; t += SPEC_THREADS) x.fbuf[off + t] = __uint_as_float(spec_power(u[t], b.inv_w));
    return;
  }
  unsigned *hold = b.hold + (size_t)spec_frame(b, j).hold_row * W + c0;
  for (int t = tid; t < C; t += SPEC_THREADS) atomicMax(hold + t, spec_power(u[t], b.inv_w));
}

// ---------------------------------------------------------------------------
// Chirp-z spectra (xlg_add_spectrum_any, every W up to 65536 that the entries above do not serve: above 4096 and
// not a power of two).  Bluestein's identity kn = (k^2 + n^2 - (k - n)^2) / 2 turns the W-point DFT of a frame z
// (windowed as spec_load does) into a circular convolution of length M = next_pow2(2W - 1) (16384 to 131072),
// which the wide passes' M-point FFT computes.  With c[n] = e^{-i pi (n^2 mod 2W) / W} (the index in 64 bits),
// and Bh[p] the M-point DFT of b[m] = e^{+i pi (m^2 mod 2W) / W}, |m| < W, wrapped mod M, scaled by 1/M and
// stored at the positions p of the transform's output (bin bin[p]; all three tables built in double on the host
// and rounded once to float), in this order (cmul_tw's rounded products and fmaf for every complex product):
//   a[n] = cmul_tw(z[n], c[n]) for n < W, +0 for W <= n < M
//   A    = fft_dif_rows' M-point transform of a (pass A then pass B as for a wide spectrum), in position order
//   Y[p] = cmul_tw(A[p], Bh[p]);  y[bin[p]] = (Y[p].x, -Y[p].y)         (conj(Y), scattered into natural order)
//   v    = the same M-point transform of y;  X_k = conj(v[k]) c[k] for k < W
// |c[k]| = 1, so the rows are defined on v itself: p_k = spec_power(v[k]), with the 1/W of a W-point spectrum;
// no post-chirp is applied.  Four launches serve every chirp-z entry of a block:
//   spectrum_czt_a_kernel: thread (frame j, column i < C) loads the 4^s points i + m C (spec_load, then the chirp;
//     the zero padding is written, never left from an earlier frame), runs pass A's stages and stores them at the
//     same positions of row j of scratch s1 (M float2 per frame)
//   spectrum_czt_b_kernel: CTA (frame j, chunk c) runs fft_dif_rows on chunk c of s1's row j, multiplies by Bh,
//     conjugates and scatters each position p to y[bin[p]] in row j of scratch s2
//   spectrum_czt_c_kernel: pass A of the second transform, in place on s2's row j
//   spectrum_czt_d_kernel: CTA (frame j, chunk c) runs fft_dif_rows on chunk c of s2's row j and folds p of every
//     position whose bin is below W into the hold (atomicMax) or the mean's frame buffer (bins in natural order;
//     positions of bins >= W are dropped)
// M = 131072 takes two pass-A stages and 8192-point chunks in 64 KiB of dynamic shared memory, the same split as
// the wide passes at every other M.  The entries are the tail of the block's table, [plain | extended | wide |
// chirp-z]: each has a SpecExt (fold and emit finish their rows unchanged) and a SpecCzt.
// ---------------------------------------------------------------------------
constexpr int SPEC_CZT_MAX_M = 131072;
constexpr size_t SPEC_CZT_SMEM = (SPEC_CZT_MAX_M >> 4) * sizeof(float2);  // passes B and D: the largest chunk

struct SpecCzt {
  float2 *s1, *s2;        // a row of M per frame of this block each: pass A's output, then y
  const float2 *tw_c;     // the C-point table (SpecBlk.tw is the M-point one)
  const float2 *chirp;    // c[n], n < W
  const float2 *kern;     // Bh, in position order
  const int *bin;         // the bin of each position
  int M;
};

template <int NS>
__device__ __forceinline__ void czt_load_a(const float2 *__restrict__ ring, unsigned mask, long long pos,
                                           const float *__restrict__ win, const float2 *__restrict__ chirp, int W,
                                           const float2 *__restrict__ tw, float2 *__restrict__ row, int i, int C) {
  constexpr int NP = NS == 1 ? 4 : 16;
  float2 a[NP];
#pragma unroll
  for (int m = 0; m < NP; m++) {
    const int n = i + m * C;
    a[m] = n < W ? cmul_tw(spec_load(ring, mask, pos + n, win, n), __ldg(chirp + n)) : make_float2(0.f, 0.f);
  }
  pass_a_stages<NS>(a, tw, i, C);
#pragma unroll
  for (int m = 0; m < NP; m++) row[i + m * C] = a[m];
}

template <int NS>
__device__ __forceinline__ void czt_inplace_a(float2 *__restrict__ row, const float2 *__restrict__ tw, int i, int C) {
  constexpr int NP = NS == 1 ? 4 : 16;
  float2 a[NP];
#pragma unroll
  for (int m = 0; m < NP; m++) a[m] = row[i + m * C];
  pass_a_stages<NS>(a, tw, i, C);
#pragma unroll
  for (int m = 0; m < NP; m++) row[i + m * C] = a[m];
}

// CTA (x, s): threads [x 256, x 256 + 256) of chirp-z spectrum s's frames x C columns (first = true: the chirped
// frames from the ring into s1; else s2 in place)
template <bool FIRST>
__device__ __forceinline__ void spectrum_czt_pass_a(const SpecBlk *__restrict__ blk,
                                                    const float2 *const *__restrict__ rings,
                                                    const SpecExt *__restrict__ ext, const SpecCzt *__restrict__ czt) {
  const SpecBlk b = blk[blockIdx.y];
  const SpecCzt z = czt[blockIdx.y];
  const int M = z.M, C = spec_wide_chunk(M), lc = 31 - __clz(C);
  const int e = blockIdx.x * SPEC_THREADS + threadIdx.x, j = e >> lc, i = e & (C - 1);
  if (j >= b.n_frames) return;
  if (FIRST) {
    const SpecExt x = ext[blockIdx.y];
    const long long pos = spec_frame_pos(b, x.H, j);
    float2 *row = z.s1 + (size_t)j * M;
    if (spec_wide_stages(M) == 1)
      czt_load_a<1>(rings[blockIdx.y], b.mask, pos, x.win, z.chirp, b.W, b.tw, row, i, C);
    else
      czt_load_a<2>(rings[blockIdx.y], b.mask, pos, x.win, z.chirp, b.W, b.tw, row, i, C);
  } else {
    float2 *row = z.s2 + (size_t)j * M;
    if (spec_wide_stages(M) == 1)
      czt_inplace_a<1>(row, b.tw, i, C);
    else
      czt_inplace_a<2>(row, b.tw, i, C);
  }
}

__global__ void __launch_bounds__(SPEC_THREADS)
spectrum_czt_a_kernel(const SpecBlk *__restrict__ blk, const float2 *const *__restrict__ rings,
                      const SpecExt *__restrict__ ext, const SpecCzt *__restrict__ czt) {
  spectrum_czt_pass_a<true>(blk, rings, ext, czt);
}

__global__ void __launch_bounds__(SPEC_THREADS)
spectrum_czt_c_kernel(const SpecBlk *__restrict__ blk, const SpecCzt *__restrict__ czt) {
  spectrum_czt_pass_a<false>(blk, nullptr, nullptr, czt);
}

// CTA (x, s): chunk x mod 4^s of frame x / 4^s of chirp-z spectrum s: pass B of the first transform, the product
// with Bh, the conjugate and the scatter into natural order
__global__ void __launch_bounds__(SPEC_THREADS, 3)
spectrum_czt_b_kernel(const SpecBlk *__restrict__ blk, const SpecCzt *__restrict__ czt) {
  extern __shared__ __align__(16) float2 u[];
  const SpecBlk b = blk[blockIdx.y];
  const SpecCzt z = czt[blockIdx.y];
  const int M = z.M, ls = 2 * spec_wide_stages(M), C = M >> ls, lc = 31 - __clz(C), tid = threadIdx.x;
  const int j = blockIdx.x >> ls, c0 = (blockIdx.x & ((1 << ls) - 1)) * C;
  if (j >= b.n_frames) return;
  spec_chunk_fft(u, z.s1 + (size_t)j * M + c0, C, lc, z.tw_c, tid);
  float2 *dst = z.s2 + (size_t)j * M;
  for (int t = tid; t < C; t += SPEC_THREADS) {
    const float2 y = cmul_tw(u[t], __ldg(z.kern + c0 + t));
    dst[__ldg(z.bin + c0 + t)] = make_float2(y.x, -y.y);
  }
}

// CTA (x, s): chunk x mod 4^s of frame x / 4^s of chirp-z spectrum s: pass B of the second transform and the
// powers of bins below W into the hold or the mean's frame buffer
__global__ void __launch_bounds__(SPEC_THREADS, 3)
spectrum_czt_d_kernel(const SpecBlk *__restrict__ blk, const SpecExt *__restrict__ ext,
                      const SpecCzt *__restrict__ czt) {
  extern __shared__ __align__(16) float2 u[];
  const SpecBlk b = blk[blockIdx.y];
  const SpecExt x = ext[blockIdx.y];
  const SpecCzt z = czt[blockIdx.y];
  const int W = b.W, M = z.M, ls = 2 * spec_wide_stages(M), C = M >> ls, lc = 31 - __clz(C), tid = threadIdx.x;
  const int j = blockIdx.x >> ls, c0 = (blockIdx.x & ((1 << ls) - 1)) * C;
  if (j >= b.n_frames) return;
  spec_chunk_fft(u, z.s2 + (size_t)j * M + c0, C, lc, z.tw_c, tid);
  if (x.mean) {
    float *fb = x.fbuf + (size_t)j * W;
    for (int t = tid; t < C; t += SPEC_THREADS) {
      const int k = __ldg(z.bin + c0 + t);
      if (k < W) fb[k] = __uint_as_float(spec_power(u[t], b.inv_w));
    }
    return;
  }
  unsigned *hold = b.hold + (size_t)spec_frame(b, j).hold_row * W;
  for (int t = tid; t < C; t += SPEC_THREADS) {
    const int k = __ldg(z.bin + c0 + t);
    if (k < W) atomicMax(hold + k, spec_power(u[t], b.inv_w));
  }
}

}  // namespace xl
