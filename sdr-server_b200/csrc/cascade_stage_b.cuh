/*
 * csrc/cascade_stage_b.cuh -- stage B of two-stage (cascade) clients: the tables its kernels read, their
 * shared-memory sizes, and launchers for the kernels themselves (defined with the batch engine's kernels in
 * xlating_kernels.cuh, compiled once in xlating_group.cu).  The batch engine (xlating_group.cu) and the
 * per-filter drop-in engine (xlating_dropin.cu) run the same stage-B kernels, so a cascade filter and the
 * same client in a group produce the same bits.
 */
#pragma once

#include <cuda_runtime.h>
#include <stddef.h>

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

// ---- launchers (xlating_group.cu), for engines that keep their own tables ----
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
