/*
 * csrc/xlating_common.cuh -- device code shared by the batch engine
 * (xlating_kernels.cuh / xlating_group.cu) and the per-filter drop-in engine
 * (dropin_kernels.cuh / xlating_dropin.cu): the arithmetic that has to match the
 * reference bit for bit lives here exactly once.
 *
 *   convert        raw cu8/cs8/cs16 -> cf32 or Q15   (src/xlating.c:389-390, 399-400,
 *                  409-410; :418, :425, :432) -- all conversions are exact
 *   oscillator     the reference's sequential float / Q15 recursion (:70-73, :126-129)
 *   generic FIR    one warp per 4 consecutive outputs of one filter, lanes split the
 *                  taps, warp-shuffle reduction (:62-69, :108-124)
 */
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

namespace xl {

struct BlkInfo {
  long long first;  // absolute sample index where output 0's window starts
  int n_out;
  int pad_;
};

__device__ __forceinline__ float2 cmul_unfused(float2 a, float2 b) {
  // two products and one add per component, each rounded (what libgcc's __mulsc3
  // does for finite operands in the reference's strict build)
  float2 r;
  r.x = __fsub_rn(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y));
  r.y = __fadd_rn(__fmul_rn(a.x, b.y), __fmul_rn(a.y, b.x));
  return r;
}

__device__ __forceinline__ short sat16(int v) {
  return (short)max(-32768, min(32767, v));
}

__device__ __forceinline__ uint32_t smem_u32(const void *p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}

// ---------------------------------------------------------------------------
// sample conversion.  FMT: 0 = cu8, 1 = cs8, 2 = cs16 (include/xlating_group.h).
// ---------------------------------------------------------------------------
__device__ __forceinline__ float cvt_cu8_f32(unsigned char u) { return ((float)u - 127.5f) * 0.0078125f; }
__device__ __forceinline__ float cvt_cs8_f32(signed char u) { return (float)u * 0.0078125f; }
__device__ __forceinline__ float cvt_cs16_f32(short u) { return (float)u * (1.0f / 32768.0f); }
__device__ __forceinline__ short cvt_cu8_q15(unsigned char u) { return (short)(((int)u - 128) << 8); }
__device__ __forceinline__ short cvt_cs8_q15(signed char u) { return (short)((int)u << 8); }

// ---------------------------------------------------------------------------
// oscillator.  The phase sequence does not depend on the data, only on how many
// outputs each call produces -- but it cannot be parallelised or put in closed
// form: parity is against the reference's float recursion (SURVEY.md 0.3), which
// drifts 4e-3 rad per block from exact math.  One thread replays it bit for bit.
//
// Only the phases of EVEN outputs are stored (dst[m * STRIDE] = phase of output
// 2m); a consumer derives an odd output's phase with the same single unfused
// multiply the recursion itself performs (phase_{k+1} = phase_k * incr), so
// nothing changes numerically while the store rate and the table halve.
// Unrolled 16 pairs: a global store keeps its source registers reserved until the
// LSU has read them (a long-scoreboard release, ~100+ cycles); with a short unroll
// the recursion stalls on that write-after-read hazard when the registers come round.
// ---------------------------------------------------------------------------
template <int STRIDE>
__device__ __forceinline__ float2 osc_chain_cf32(float2 p, const float2 inc, float2 *__restrict__ dst, int n_out,
                                                 int renorm) {
  const int n_pairs = n_out >> 1;
#pragma unroll 16
  for (int m = 0; m < n_pairs; m++) {
    dst[(size_t)m * STRIDE] = p;  // phase of output 2m
    p = cmul_unfused(p, inc);     // src/xlating.c:71 (output 2m+1)
    p = cmul_unfused(p, inc);
  }
  if (n_out & 1) {
    dst[(size_t)n_pairs * STRIDE] = p;  // last (even-indexed) output
    p = cmul_unfused(p, inc);
  }
  if (n_out > 0 && renorm) {
    // src/xlating.c:73.  glibc's hypotf is (float)sqrt((double)x*x + (double)y*y)
    // (verified on 5e7 random inputs); the products are exact in double.
    const double m2 = (double)p.x * (double)p.x + (double)p.y * (double)p.y;
    const float mag = (float)sqrt(m2);
    p.x = __fdiv_rn(p.x, mag);
    p.y = __fdiv_rn(p.y, mag);
  }
  return p;
}

// Q15 oscillator (src/xlating.c:126-129, no renormalisation): stores the phase of
// EVERY output, returns the phase after the last one.
__device__ __forceinline__ short2 osc_chain_q15(short2 ph, const short2 inc, short2 *__restrict__ row, int n_out) {
  int pr = ph.x, pi = ph.y;
  const int ir = inc.x, ii = inc.y;
  for (int k = 0; k < n_out; k++) {
    row[k] = make_short2((short)pr, (short)pi);
    const int nr = pr * ir - pi * ii;
    const int ni = pr * ii + pi * ir;
    pr = sat16(nr >> 15);
    pi = sat16(ni >> 15);
  }
  return make_short2((short)pr, (short)pi);
}

// number of outputs of a call: windows of T samples every D, the first starting at
// `first`, the last admissible one at S + n_in - T (src/xlating.c:58-60)
__device__ __forceinline__ int outputs_of_call(long long first, long long S, int n_in, int T, int D, int out_cap) {
  const long long last_ok = S + n_in - T;
  int n_out = 0;
  if (last_ok >= first) n_out = (int)((last_ok - first) / D) + 1;
  return n_out > out_cap ? out_cap : n_out;  // cannot clamp for input_len <= max_input_len
}

// rational L/M filter (the filter at L * fs fed the zero-stuffed stream u[L*n] = x[n]): the output
// whose upsampled window starts at w reads only polyphase branch r = (-w) mod L (floor semantics:
// w < 0 inside the first block), whose first tap meets input sample n0 = (w + r) / L
__device__ __forceinline__ int poly_branch(long long w, int L, long long *n0) {
  const int r = (int)((((-w) % L) + L) % L);
  *n0 = (w + r) / L;
  return r;
}

// ---------------------------------------------------------------------------
// generic FIR, one warp = G_OPW consecutive outputs starting at window w0.  Lane i
// (< G_OPW) returns the dot product of output i; other lanes return output 0's.
// ---------------------------------------------------------------------------
constexpr int G_THREADS = 256;
constexpr int G_OPW = 4;                         // outputs per warp
constexpr int G_OPC = (G_THREADS / 32) * G_OPW;  // outputs per CTA

constexpr int G_STEPS = 4;  // tap steps (of 32 lanes) whose loads are issued together

__device__ __forceinline__ float2 fir_warp_cf32(const float2 *__restrict__ ring, unsigned mask, long long zb,
                                                const float2 *__restrict__ tp, int T, int D, long long w0,
                                                int lane) {
  float2 acc[G_OPW];
#pragma unroll
  for (int i = 0; i < G_OPW; i++) acc[i] = make_float2(0.f, 0.f);
  // A lone call is a fraction of one wave and purely load-latency bound (ncu: 11
  // long-scoreboard stalls per issue slot with one step in flight), so the loads of
  // G_STEPS tap steps are issued before their FMAs.  Loads are unconditional -- any
  // masked index is inside the ring -- and samples before the attach point are zeroed
  // by a select, which keeps the loop free of branches.  The accumulation order per
  // lane is the sequential one.
  int j = lane;
  for (; j + 32 * (G_STEPS - 1) < T; j += 32 * G_STEPS) {
    float2 t[G_STEPS], x[G_STEPS][G_OPW];
#pragma unroll
    for (int u = 0; u < G_STEPS; u++) {
      t[u] = __ldg(tp + j + 32 * u);
#pragma unroll
      for (int i = 0; i < G_OPW; i++) {
        const long long ab = w0 + (long long)i * D + j + 32 * u;
        x[u][i] = ring[(unsigned)((unsigned long long)ab) & mask];
        if (ab < zb) x[u][i] = make_float2(0.f, 0.f);
      }
    }
#pragma unroll
    for (int u = 0; u < G_STEPS; u++)
#pragma unroll
      for (int i = 0; i < G_OPW; i++) {
        acc[i].x = fmaf(x[u][i].x, t[u].x, acc[i].x);
        acc[i].x = fmaf(-x[u][i].y, t[u].y, acc[i].x);
        acc[i].y = fmaf(x[u][i].x, t[u].y, acc[i].y);
        acc[i].y = fmaf(x[u][i].y, t[u].x, acc[i].y);
      }
  }
  for (; j < T; j += 32) {
    const float2 t = __ldg(tp + j);
#pragma unroll
    for (int i = 0; i < G_OPW; i++) {
      const long long ab = w0 + (long long)i * D + j;
      float2 x = ring[(unsigned)((unsigned long long)ab) & mask];
      if (ab < zb) x = make_float2(0.f, 0.f);
      acc[i].x = fmaf(x.x, t.x, acc[i].x);
      acc[i].x = fmaf(-x.y, t.y, acc[i].x);
      acc[i].y = fmaf(x.x, t.y, acc[i].y);
      acc[i].y = fmaf(x.y, t.x, acc[i].y);
    }
  }
#pragma unroll
  for (int i = 0; i < G_OPW; i++) {
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) {
      acc[i].x += __shfl_xor_sync(0xffffffffu, acc[i].x, s);
      acc[i].y += __shfl_xor_sync(0xffffffffu, acc[i].y, s);
    }
  }
  // lane i finishes output i (every lane holds all four sums after the butterfly)
  float2 mine = acc[0];
#pragma unroll
  for (int i = 1; i < G_OPW; i++)
    if (lane == i) mine = acc[i];
  return mine;
}

// Q15 integer path (src/xlating.c:92-140): int16 x int16 products accumulated in
// int64 -- integer addition is associative, so the lane-split + shuffle reduction
// is bit-exact against the reference's sequential loop.  Returns the filter output
// already scaled and saturated (:118-119).
__device__ __forceinline__ short2 fir_warp_q15(const short2 *__restrict__ ring, unsigned mask, long long zb,
                                               const short2 *__restrict__ tp, int T, int D, long long w0,
                                               int lane) {
  long long are[G_OPW], aim[G_OPW];
#pragma unroll
  for (int i = 0; i < G_OPW; i++) are[i] = aim[i] = 0;
#pragma unroll 4
  for (int j = lane; j < T; j += 32) {
    const short2 t = __ldg(tp + j);
#pragma unroll
    for (int i = 0; i < G_OPW; i++) {
      const long long ab = w0 + (long long)i * D + j;
      short2 x = ring[(unsigned)((unsigned long long)ab) & mask];  // unconditional: any masked index is in the ring
      if (ab < zb) x = make_short2(0, 0);
      are[i] += (long long)((int)x.x * (int)t.x) - (long long)((int)x.y * (int)t.y);  // :114
      aim[i] += (long long)((int)x.x * (int)t.y) + (long long)((int)x.y * (int)t.x);  // :115
    }
  }
#pragma unroll
  for (int i = 0; i < G_OPW; i++) {
#pragma unroll
    for (int s = 16; s > 0; s >>= 1) {
      are[i] += __shfl_xor_sync(0xffffffffu, are[i], s);
      aim[i] += __shfl_xor_sync(0xffffffffu, aim[i], s);
    }
  }
  long long mre = are[0], mim = aim[0];
#pragma unroll
  for (int i = 1; i < G_OPW; i++)
    if (lane == i) {
      mre = are[i];
      mim = aim[i];
    }
  return make_short2(sat16((int)(mre >> 15)), sat16((int)(mim >> 15)));  // :118-119
}

// output rotation of the Q15 path (src/xlating.c:121-124)
__device__ __forceinline__ short2 rotate_q15(short2 a, short2 ph) {
  const int rr = (int)a.x * (int)ph.x - (int)a.y * (int)ph.y;
  const int ri = (int)a.x * (int)ph.y + (int)a.y * (int)ph.x;
  return make_short2(sat16(rr >> 15), sat16(ri >> 15));
}

}  // namespace xl
