/*
 * csrc/cascade_stage_b.cuh -- stage B of two-stage (cascade) clients: the tables its kernels read, their
 * shared-memory sizes, launchers for the kernels themselves (defined with the batch engine's kernels in
 * xlating_kernels.cuh, compiled once in xlating_group.cu), and the host half both engines share.  The batch
 * engine (xlating_group.cu) and the per-filter drop-in engine (xlating_dropin.cu) run the same stage-B
 * kernels, whose summation order depends on the thread that computes an output; a cascade filter and the same
 * client in a group produce the same bits because both take their admission rules, taps, outputs per CTA
 * (ko), history reach, per-block walk and tables from the functions here.
 */
#pragma once

#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include <algorithm>
#include <vector>

#include "taps_host.h"

namespace xl {

// dynamic shared memory a CTA of the tiled FIR or of stage B may use (raised per kernel at set-up)
constexpr int kTileMaxSmem = 200 * 1024;

// ---------------------------------------------------------------------------
// cascade clients (xlg_add_client_cascade).  Stage A is an integer client of the FIR kernels whose outputs
// land in a row of an output arena that is never copied to the host.  Stage B is the reference
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

constexpr int C_THREADS = 128;
constexpr int C_R = 2;                    // outputs per thread: t and t + C_THREADS
constexpr int C_KO = C_THREADS * C_R;     // outputs per CTA at most (the host lowers it where shared memory runs out)
// shared memory of a CTA with ko outputs: mbarrier, taps padded to 16 bytes, the window (+1 for an odd start, even)
__host__ __device__ constexpr size_t cascade_smem(int ko, int D2, int T2) {
  return 16 + (size_t)((T2 + 3) & ~3) * 4 + (((size_t)(ko - 1) * D2 + T2 + 2) & ~(size_t)1) * 8;
}

// ---------------------------------------------------------------------------
// rational cascade clients (xlg_add_client_cascade_rational, interp2 = L2 > 1).  Stage B is the reference
// filter with decimation M2 at L2 * fs / D1, centre 0, fed the zero-stuffed stage-A stream u[L2*n] = y[n]:
// output k's upsampled window starts at w = first + k*M2, and with r = (-w) mod L2, n0 = (w + r) / L2
// (poly_branch) only the branch r of the real reversed taps meets stage-A samples,
//     z[k] = sum_{t < Tb2} y[n0 + t] * P[r][t],   P[r][t] = rev2[r + t*L2] (0 past T2),  Tb2 = ceil(T2 / L2).
// The ring, its positions and its zeros before the attach are the integer cascade's (CascBlk appends them).
// ---------------------------------------------------------------------------
struct CascPolyBlk {
  float2 *ring;     // the client's stage-A history ring
  long long first;  // upsampled stream position where this block's output 0 starts its window
  unsigned mask;    // ring capacity - 1
  int n2;           // outputs computed by this block
  int L2, M2, Tb2;
  int ko;           // outputs per CTA (the host sets it per client)
  int taps_off;     // float offset of the branch-major taps P in the real tap arena, a multiple of 4
  int out_off;      // final row in the slot's output arena
};

// shared memory of a CTA with ko outputs: mbarrier, the L2 branches padded to 16 bytes, the window: the
// n0 of ko consecutive outputs span at most ceil((ko - 1) * M2 / L2) samples, plus Tb2 taps (+1 for an odd
// start, even)
__host__ __device__ constexpr size_t cascade_poly_smem(int ko, int L2, int M2, int Tb2) {
  return 16 + (((size_t)L2 * Tb2 + 3) & ~(size_t)3) * 4 +
         ((((size_t)(ko - 1) * M2 + L2 - 1) / L2 + Tb2 + 2) & ~(size_t)1) * 8;
}

// Outputs per CTA of a rational stage B (CascPolyBlk::ko), fixed when the client is attached: about
// 2 * C_THREADS, a whole number per branch where L2 <= C_THREADS; fewer where the window would not fit (the
// attach checks that one output fits).
inline int cascade_poly_ko(int L2, int M2, int Tb2) {
  int ko = L2 <= C_THREADS ? 2 * L2 * (C_THREADS / L2) : C_KO;
  while (ko > 1 && cascade_poly_smem(ko, L2, M2, Tb2) > (size_t)kTileMaxSmem) ko /= 2;
  return ko;
}

// Outputs per CTA of an integer stage B, fixed when the client is attached: C_KO halved until the window fits
// (the attach checks that one output fits).
inline int cascade_ko(int D2, int T2) {
  int ko = C_KO;
  while (ko > 1 && cascade_smem(ko, D2, T2) > (size_t)kTileMaxSmem) ko /= 2;
  return ko;
}

// ---------------------------------------------------------------------------
// host half of stage B
// ---------------------------------------------------------------------------

// Why a cascade client is refused, or nullptr: stage A decimates by D1 a stream of blocks of at most max_in
// scalars, stage B is the filter with T2 taps and decimation M2 at L2 times stage A's rate.
inline const char *cascade_refusal(uint32_t max_in, uint32_t D1, uint32_t L2, uint32_t M2, size_t T2) {
  if (D1 == 0 || L2 == 0 || M2 == 0) return "decimation1, interpolation2 and decimation2 must all be at least 1";
  if (L2 > 1 && (uint64_t)L2 * ((uint64_t)max_in / 2 / D1 + 2) >= (1ull << 31))
    return "interpolation2 x (max_input_len / 2 / decimation1 + 2) upsampled stage-A samples per block reach 2^31";
  if (T2 > (size_t)INT32_MAX ||
      (L2 == 1 ? cascade_smem(1, (int)M2, (int)T2)
               : cascade_poly_smem(1, (int)L2, (int)M2, (int)((T2 + L2 - 1) / L2))) > (size_t)kTileMaxSmem)
    return "stage B's taps and one output's window exceed the stage-B kernels' shared memory";
  return nullptr;
}

// Why a single-stage rational client (the filter with decimation M at L * fs fed the zero-stuffed stream of
// blocks of at most max_in scalars) is refused, or nullptr.
inline const char *rational_refusal(uint32_t fs, uint32_t max_in, uint32_t L, uint32_t M) {
  if (L == 0 || M == 0) return "interpolation and decimation must both be at least 1";
  if ((uint64_t)L * fs > UINT32_MAX) return "the upsampled rate interpolation x sampling rate exceeds UINT32_MAX";
  if ((uint64_t)L * (max_in / 2) >= (1ull << 31))
    return "interpolation x max_input_len / 2 upsampled samples per block reach 2^31";
  return nullptr;
}

// Samples of its input stream that a filter with interpolation L reaches back for its history of at most
// T - 1 upsampled samples: ceil((T - 1) / L), plus one zero-weighted sample its last branch may read past the
// block when L > 1.
inline size_t history_reach(size_t T, uint32_t L) { return L == 1 ? T - 1 : (T - 1 + L - 1) / L + 1; }

// Outputs of one block of a stage B at L2 / D2 fed at most n1_cap samples: n2 <= (L2 * n1 - 1) / D2 + 1 for
// any history.
inline int stage_b_rows(uint64_t n1_cap, uint32_t L2, uint32_t D2) { return (int)(n1_cap * L2 / D2 + 2); }

// A power-of-two history ring in HBM: the sample at stream position q lives at p[q & (cap - 1)], and positions
// before the attach read as the ring's zeros.
struct HistRing {
  float2 *p = nullptr;
  size_t cap = 0;
  long long pos = 0;  // samples appended since the attach: the position of the next one
};

// Stage B's geometry: the filter with T2 taps and decimation D2 at L2 times the rate of the stream it reads
// (zero-stuffed when L2 > 1), and where its next window starts.
struct StageBGeom {
  uint32_t L2 = 1, D2 = 0;
  size_t T2 = 0;
  int Tb2 = 0;          // taps per branch, ceil(T2 / L2)
  long long hist2 = 0;  // history_offset, in upsampled samples
};

inline StageBGeom stage_b_geom(uint32_t L2, uint32_t D2, size_t T2) {
  StageBGeom b;
  b.L2 = L2;
  b.D2 = D2;
  b.T2 = T2;
  b.Tb2 = (int)((T2 + L2 - 1) / L2);
  b.hist2 = (long long)T2 - 1;  // src/xlating.c:552
  return b;
}

// This block's walk of a stage B: where its output 0's window starts (upsampled), and its outputs.
struct StageBStep {
  long long first;
  int n2;
};

// The reference's walk (xl_walk) of stage B over the n1 samples of its input stream from position pos, in
// upsampled coordinates (the zero-stuffed stream u[L2 * n] = y[n]; the same integers for L2 = 1), at most
// out_cap outputs.  Advances b.hist2.
inline StageBStep stage_b_walk(StageBGeom &b, long long pos, int n1, int out_cap) {
  const long long first = (long long)b.L2 * pos - b.hist2;
  const int n2 = xl_walk(&b.hist2, (long long)b.L2 * n1, b.T2, b.D2, out_cap);
  return {first, n2};
}

// Stage B of a cascade client or filter.  A sub-band keeps only `ring` (its members' input) and a sub-band
// member only `geo` (its own filter, in sub-band samples).
struct StageB {
  StageBGeom geo;
  int ko = 0;                    // outputs per CTA: cascade_ko (L2 = 1), cascade_poly_ko (L2 > 1)
  HistRing ring;                 // stage-A history
  std::vector<float> taps;       // real, branch-major, padded to whole float4s (16-byte bulk copies)
  int taps_off = 0;              // taps in the real tap arena, floats
  int fin_off = 0, fin_cap = 0;  // final row: offset and outputs per block at most (stage_b_rows)
};

// A cascade's stage B at L2 * rate1 (rate1 = fs / D1, stage A's output rate): the reference filter with
// decimation M2 and centre 0.  Its rotated taps are (h, +-0), so the real parts of its reversed taps (the
// even-length quirk included) are all it needs, branch-major P[r][t] = rev2[r + t * L2] (xl_poly_pack: the
// reversed taps themselves for L2 = 1); at centre 0 the rate only enters the rotation, so clamping it changes
// nothing.  Returns 0 or -ENOMEM.
inline int stage_b_init(StageB *c, const float *taps2, size_t T2, uint32_t L2, uint32_t M2, uint32_t rate1) {
  const uint64_t rate2 = (uint64_t)L2 * std::max<uint32_t>(rate1, 1);
  xl_client_consts k;
  const int rc = xl_client_consts_build(taps2, T2, M2, 0, (uint32_t)std::min<uint64_t>(rate2, UINT32_MAX), &k);
  if (rc != 0) return rc;
  c->geo = stage_b_geom(L2, M2, T2);
  c->ko = L2 == 1 ? cascade_ko((int)M2, (int)T2) : cascade_poly_ko((int)L2, (int)M2, c->geo.Tb2);
  const size_t n = (size_t)L2 * c->geo.Tb2;
  std::vector<float> packed(2 * n);
  xl_poly_pack(k.rev_cf32, T2, L2, packed.data());
  xl_client_consts_free(&k);
  c->taps.assign((n + 3) & ~(size_t)3, 0.f);
  for (size_t j = 0; j < n; j++) c->taps[j] = packed[2 * j];
  return 0;
}

// This block's stage-B entries of a cascade from its walk w over n1 stage-A outputs at a_off (the ring's
// position not yet advanced): the append and integer entry cb and, for L2 > 1, the rational entry pb.
inline void stage_b_fill(const StageB &c, const StageBStep &w, int n1, int a_off, CascBlk *cb, CascPolyBlk *pb) {
  cb->ring = c.ring.p;
  cb->a_pos = c.ring.pos;
  cb->first = w.first;
  cb->mask = (unsigned)(c.ring.cap - 1);
  cb->a_off = a_off;
  cb->n1 = n1;
  cb->n2 = w.n2;
  cb->D2 = (int)c.geo.D2;
  cb->T2 = (int)c.geo.T2;
  cb->taps_off = c.taps_off;
  cb->out_off = c.fin_off;
  if (c.geo.L2 == 1) return;
  pb->ring = c.ring.p;
  pb->first = w.first;
  pb->mask = cb->mask;
  pb->n2 = w.n2;
  pb->L2 = (int)c.geo.L2;
  pb->M2 = (int)c.geo.D2;
  pb->Tb2 = c.geo.Tb2;
  pb->ko = c.ko;
  pb->taps_off = c.taps_off;
  pb->out_off = c.fin_off;
}

// ---- launchers (xlating_group.cu): the only launch site of each stage-B kernel ----
// Raise the stage-B kernels' dynamic shared memory limit to kTileMaxSmem on the current device.
cudaError_t cascade_stage_b_init();
// cascade_append_kernel: entry c appends cb[c].n1 stage-A outputs from a_rows + cb[c].a_off to its ring.
void cascade_launch_append(const CascBlk *cb, int n, int max_n1, const float2 *a_rows, cudaStream_t s);
// cascade_fir_cf32_kernel over n integer entries with ko outputs per CTA.
void cascade_launch_fir(const CascBlk *cb, int n, int max_n2, int ko, size_t smem, const float *taps2, float2 *out,
                        cudaStream_t s);
// cascade_fir_poly_cf32_kernel over n rational entries; max_ctas = max over them of ceil(n2 / ko).
void cascade_launch_fir_poly(const CascPolyBlk *pb, int n, int max_ctas, size_t smem, const float *taps2,
                             float2 *out, cudaStream_t s);

}  // namespace xl
