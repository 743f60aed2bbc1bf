/*
 * csrc/dropin_kernels.cuh -- device side of the per-filter drop-in ABI
 * (include/xlating.h, host side in xlating_dropin.cu).
 *
 * The reference runs one filter per client on one dsp thread per client
 * (src/dsp_worker.c:41-88), every thread calling process_* on its PRIVATE copy of
 * the SDR block (src/queue.c:114).  Behind the unmodified ABI the library cannot
 * share one input between filters, but it can share LAUNCHES: calls that arrive
 * together from different threads are combined into one batch of "requests"
 * (filter, private input) and served by two kernels:
 *
 *   dropin_front_kernel   blocks [0, n_osc): one warp (lane 0) per request replays
 *                         that filter's oscillator for this call (the dependent
 *                         chain, scheduled first because it is the long pole);
 *                         remaining blocks: convert each request's raw samples
 *                         (16 bytes per lane) into the filter's private ring in HBM.
 *   dropin_fir_kernel     the generic FIR (xlating_common.cuh) per request; each
 *                         CTA writes its 32 outputs as one 256-byte line straight
 *                         into the filter's pinned host output buffer.
 *   dropin_fir_poly_kernel  the same for rational (L/M) filters, one polyphase branch
 *                         per output (launched only when the batch has such a request).
 *
 * So a batch costs one (batched) input copy, two launches (three with rational
 * filters in it) and one stream synchronisation however many filters are in it.
 */
#pragma once

#include "xlating_common.cuh"

namespace xl {

// One drop-in filter (src/xlating.c:17-50).  Rings are private: absolute sample
// index s of the filter's own stream lives at ring[s & mask]; the cf32 and Q15
// paths have separate rings and positions but share `hist`, like the reference's
// two working buffers sharing history_offset.
struct FilterDev {
  float2 *ring;
  short2 *qring;          // allocated on the first Q15 call
  const float2 *taps;     // reversed band-pass taps (:525-534)
  const short2 *qtaps;
  float2 *phases;         // phase of output 2m at phases[m], in HBM
  const float2 *phases_host;  // the same table where the HOST writes it (device address of pinned memory)
  short2 *qphases;        // phase of output k at qphases[k]
  float2 *out;            // device address of the filter's pinned host output buffer (cf32)
  short2 *qout;           // same, Q15 (int16 re,im)
  long long hist;         // history_offset (:29)
  BlkInfo blk;            // this call's window start and output count (written by the oscillator lane)
  float2 phase, incr;     // (:36-37)
  short2 qphase, qincr;   // (:39-42)
  unsigned mask;
  int D, T, out_cap;
  int L;                  // interpolation of a rational filter (1 = integer filter); taps are then its
                          // polyphase branches (xl_poly_pack), hist / blk.first in upsampled samples
};

// One process_* call.  The table lives in pinned host memory and is read by the
// front kernel over PCIe (32 bytes per request).
struct DropinReq {
  const void *raw;  // device address of the staged input (HBM copy, or pinned host memory when zero-copy)
  long long S;      // the path's stream position before this call
  int filter;       // index into the FilterDev table
  int n;            // complex samples in this call
  int fmt;          // XLG_FMT_*
  int q15;          // 1 = Q15 path
  int osc_host;     // cf32 oscillator of this call: 0 = walked by a GPU lane; 1 = already walked by the host
                    // (taps_host.c), table to be copied pinned -> HBM here; 2 = being walked by the host
                    // while this kernel runs, the FIR kernel reads the pinned table itself
  int n_out;        // outputs of this call (host mirror of the oscillator lane's count)
};

constexpr int DF_THREADS = 256;
constexpr int DF_SPT = 8;                        // complex samples per thread (16 bytes of cu8)
constexpr int DF_SPB = DF_THREADS * DF_SPT;      // per block
constexpr int DF_OSC_PER_BLOCK = 4;              // oscillator chains per block (one warp each)

__device__ __forceinline__ void dropin_store(const DropinReq &q, const FilterDev *d, int i, float re, float im,
                                             short qre, short qim) {
  const unsigned idx = (unsigned)((unsigned long long)(q.S + i)) & d->mask;
  if (q.q15)
    d->qring[idx] = make_short2(qre, qim);
  else
    d->ring[idx] = make_float2(re, im);
}

template <int FMT>
__device__ __forceinline__ void dropin_convert8(const DropinReq &q, const FilterDev *d, int base) {
  // 8 complex samples = 16 scalars
  if (FMT == 2) {
    __align__(16) short v[16];
    if (base + DF_SPT <= q.n) {
      const uint4 *p = reinterpret_cast<const uint4 *>(reinterpret_cast<const short *>(q.raw) + 2 * (size_t)base);
      *reinterpret_cast<uint4 *>(v) = p[0];
      *reinterpret_cast<uint4 *>(v + 8) = p[1];
    } else {
      for (int e = 0; e < 2 * (q.n - base); e++) v[e] = reinterpret_cast<const short *>(q.raw)[2 * (size_t)base + e];
    }
#pragma unroll
    for (int e = 0; e < DF_SPT; e++)
      if (base + e < q.n)
        dropin_store(q, d, base + e, cvt_cs16_f32(v[2 * e]), cvt_cs16_f32(v[2 * e + 1]), v[2 * e], v[2 * e + 1]);
  } else {
    __align__(16) unsigned char v[16];
    if (base + DF_SPT <= q.n) {
      *reinterpret_cast<uint4 *>(v) =
          *reinterpret_cast<const uint4 *>(reinterpret_cast<const unsigned char *>(q.raw) + 2 * (size_t)base);
    } else {
      for (int e = 0; e < 2 * (q.n - base); e++)
        v[e] = reinterpret_cast<const unsigned char *>(q.raw)[2 * (size_t)base + e];
    }
#pragma unroll
    for (int e = 0; e < DF_SPT; e++) {
      if (base + e >= q.n) break;
      if (FMT == 0) {
        dropin_store(q, d, base + e, cvt_cu8_f32(v[2 * e]), cvt_cu8_f32(v[2 * e + 1]), cvt_cu8_q15(v[2 * e]),
                     cvt_cu8_q15(v[2 * e + 1]));
      } else {
        const signed char a = (signed char)v[2 * e], b = (signed char)v[2 * e + 1];
        dropin_store(q, d, base + e, cvt_cs8_f32(a), cvt_cs8_f32(b), cvt_cs8_q15(a), cvt_cs8_q15(b));
      }
    }
  }
}

__global__ void __launch_bounds__(DF_THREADS)
dropin_front_kernel(FilterDev *__restrict__ filters, const DropinReq *__restrict__ req, int2 *__restrict__ batch,
                    int n_req, int n_osc_blocks, int conv_blocks_per_req, int osc_lanes) {
  if ((int)blockIdx.x < n_osc_blocks) {
    // ---- oscillator: one request per WARP (lane 0), DF_OSC_PER_BLOCK warps per block ----
    // Not one request per lane: every filter has its own table, so a warp with L active
    // lanes issues L separate 8-byte stores per step, and a warp can only keep ~32 store
    // transactions in flight -- measured on the batch engine's pre-pass, 32 uncoalesced
    // lanes ran the chain 4x slower than its 10.75-cycle dependent latency.  A lone lane
    // stays on that latency; the four warps land on the SM's four schedulers.
    int r;
    if (osc_lanes) {  // A/B variant: 32 requests per block, one per lane of warp 0
      if (threadIdx.x >= 32) return;
      r = blockIdx.x * 32 + threadIdx.x;
    } else {
      const int w = threadIdx.x >> 5;
      if ((threadIdx.x & 31) != 0 || w >= DF_OSC_PER_BLOCK) return;
      r = blockIdx.x * DF_OSC_PER_BLOCK + w;
    }
    if (r >= n_req) return;
    const DropinReq q = req[r];
    FilterDev *d = filters + q.filter;
    batch[r] = make_int2(q.filter, q.q15 | (q.osc_host == 2 ? 2 : 0) | (d->L > 1 ? 4 : 0));
    const int D = d->D;
    // stream positions in the filter's (upsampled) coordinates, as the batch engine's pre-pass
    // computes them: identical integers for L = 1
    const long long Su = q.S * d->L, Eu = (q.S + q.n) * d->L;
    const long long first = Su - d->hist;
    const int n_out = outputs_of_call(first, Su, (int)(Eu - Su), d->T, D, d->out_cap);
    BlkInfo b;
    b.first = first;
    b.n_out = n_out;
    b.pad_ = 0;
    d->blk = b;
    if (q.q15)
      d->qphase = osc_chain_q15(d->qphase, d->qincr, d->qphases, n_out);
    else if (q.osc_host == 0)
      d->phase = osc_chain_cf32<1>(d->phase, d->incr, d->phases, n_out, 1);
    d->hist = Eu - (first + (long long)n_out * D);  // src/xlating.c:76, :133
    return;
  }
  // ---- conversion blocks ----
  __shared__ DropinReq sq;
  const int cb = blockIdx.x - n_osc_blocks;
  const int r = cb / conv_blocks_per_req;
  const int chunk = cb - r * conv_blocks_per_req;
  if (threadIdx.x == 0) sq = req[r];
  __syncthreads();
  const DropinReq q = sq;
  const FilterDev *d = filters + q.filter;
  if (chunk == 0 && q.osc_host == 1 && !q.q15) {
    // host-walked oscillator table: one coalesced pass pinned -> HBM (512 bytes per warp
    // request) instead of one 32-byte PCIe read per FIR warp later
    const int n16 = (((q.n_out + 1) >> 1) + 1) >> 1;  // 16-byte units, two table entries each
    const uint4 *src = reinterpret_cast<const uint4 *>(d->phases_host);
    uint4 *dst = reinterpret_cast<uint4 *>(d->phases);
    for (int i = threadIdx.x; i < n16; i += DF_THREADS) dst[i] = src[i];
  }
  const int base = chunk * DF_SPB + threadIdx.x * DF_SPT;
  if (base >= q.n) return;
  if (q.fmt == 0)
    dropin_convert8<0>(q, d, base);
  else if (q.fmt == 1)
    dropin_convert8<1>(q, d, base);
  else
    dropin_convert8<2>(q, d, base);
}

// Outputs one CTA owns: G_OPC of an integer request (dropin_fir_kernel); for a rational one
// (dropin_fir_poly_kernel) the G_OPC outputs of each of up to DF_POLY_RES residues mod L, so that every
// residue of the span fills whole G_OPW-output groups.
constexpr int DF_POLY_RES = 16;
__host__ __device__ __forceinline__ int dropin_fir_span(int L) {
  return G_OPC * (L < DF_POLY_RES ? L : DF_POLY_RES);
}

// grid = (max over integer requests of ceil(n_out / G_OPC), n_req); rational requests are skipped
__global__ void __launch_bounds__(G_THREADS)
dropin_fir_kernel(const FilterDev *__restrict__ filters, const int2 *__restrict__ batch) {
  __shared__ float2 so[G_OPC];
  const int2 bq = batch[blockIdx.y];
  if (bq.y & 4) return;  // rational: dropin_fir_poly_kernel
  const FilterDev *d = filters + bq.x;
  const BlkInfo b = d->blk;
  const int kbase = blockIdx.x * G_OPC;
  if (kbase >= b.n_out) return;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int k0 = kbase + warp * G_OPW;
  const int k = k0 + lane;
  const long long w0 = b.first + (long long)k0 * d->D;
  // samples before the filter's creation (absolute index < 0) are the reference's
  // zero-initialised working buffer (src/xlating.c:556-565)
  if (bq.y & 1) {
    short2 *sq = reinterpret_cast<short2 *>(so);
    const short2 mine = fir_warp_q15(d->qring, d->mask, 0, d->qtaps, d->T, d->D, w0, lane);
    if (lane < G_OPW && k < b.n_out) sq[warp * G_OPW + lane] = rotate_q15(mine, d->qphases[k]);  // :121-124
    __syncthreads();
    if (threadIdx.x < G_OPC && kbase + (int)threadIdx.x < b.n_out) d->qout[kbase + threadIdx.x] = sq[threadIdx.x];
  } else {
    const float2 mine = fir_warp_cf32(d->ring, d->mask, 0, d->taps, d->T, d->D, w0, lane);
    if (lane < G_OPW && k < b.n_out) {
      float2 ph = ((bq.y & 2) ? d->phases_host : d->phases)[k >> 1];
      if (k & 1) ph = cmul_unfused(ph, d->incr);  // odd outputs: one step from the stored even phase
      so[warp * G_OPW + lane] = cmul_unfused(mine, ph);  // src/xlating.c:70
    }
    __syncthreads();
    if (threadIdx.x < G_OPC && kbase + (int)threadIdx.x < b.n_out) d->out[kbase + threadIdx.x] = so[threadIdx.x];
  }
}

// Rational requests (L > 1), grid = (max over them of ceil(n_out / dropin_fir_span(L)), n_req); the
// integer requests are skipped.  A CTA owns a contiguous span of outputs and computes them as the batch
// engine's polyphase generic kernel (fir_poly_generic_cf32_kernel) does: outputs k0 + i*L (i < G_OPW)
// share the branch r of k0 and read inputs M samples apart, so a warp runs the generic FIR warp on
// branch r with decimation M; the warps loop over the span's (residue, output group) pairs.  Per output
// the arithmetic is that kernel's, so a private rational filter equals the same client in a group bit for
// bit.  A branch's padding tap reads one sample past its window with weight 0: the private ring starts
// zeroed and only ever holds converted samples, so that sample is finite.  The span leaves through
// shared memory as contiguous lines into the filter's pinned output buffer.  (A separate kernel: inlined
// next to the integer path, this loop changed how the compiler scheduled that path's loads.)
__global__ void __launch_bounds__(G_THREADS)
dropin_fir_poly_kernel(const FilterDev *__restrict__ filters, const int2 *__restrict__ batch) {
  __shared__ float2 so[G_OPC * DF_POLY_RES];
  const int2 bq = batch[blockIdx.y];
  if (!(bq.y & 4)) return;
  const FilterDev *d = filters + bq.x;
  const BlkInfo b = d->blk;
  const int L = d->L, M = d->D;
  const int kbase = blockIdx.x * dropin_fir_span(L);
  if (kbase >= b.n_out) return;  // CTA-uniform
  const int n_span = min(dropin_fir_span(L), b.n_out - kbase);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int per = (n_span + L - 1) / L;  // outputs of residue 0 (the most of any residue)
  const int groups = (per + G_OPW - 1) / G_OPW;
  const int pairs = min(L, n_span) * groups;
  const int Tb = (d->T + L - 1) / L;
  const float2 *ph_table = (bq.y & 2) ? d->phases_host : d->phases;
  for (int p = warp; p < pairs; p += G_THREADS / 32) {
    const int rho = p / groups;
    const int kl = rho + (p - rho * groups) * G_OPW * L;  // span-local index of the group's first output
    if (kl >= n_span) continue;                           // warp-uniform
    const int k0 = kbase + kl;
    long long n0;
    const int r = poly_branch(b.first + (long long)k0 * M, L, &n0);
    const float2 mine = fir_warp_cf32(d->ring, d->mask, 0, d->taps + (size_t)r * Tb, Tb, M, n0, lane);
    const int kk = kl + lane * L;
    if (lane < G_OPW && kk < n_span) {
      const int k = kbase + kk;
      float2 ph = ph_table[k >> 1];
      if (k & 1) ph = cmul_unfused(ph, d->incr);  // odd outputs: one step from the stored even phase
      so[kk] = cmul_unfused(mine, ph);             // src/xlating.c:70
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < n_span; i += G_THREADS) d->out[kbase + i] = so[i];
}

}  // namespace xl
