"""References of the chirp-z bank tests (xlg_add_bank_any at a K that is not a power of two).  No GPU.

* bank_czt_model: what bank_czt_cf32_kernel computes, in its exact order (xlating_kernels.cuh, "Chirp-z banks"),
  on the library's own tables (xlg_bank_any_tables: the chirp c and Bh in position order): the FFT bank's
  placed sums u, a = cmul(u, c) padded with zeros to M, A = fft_rows at K = M, Y = cmul(A, Bh) at each position,
  conj(Y) scattered to natural order, v = fft_rows at K = M again, y_k = cmul(conj(v[q]), c[k mod K]) at
  q = bank_fft_pos(k mod K, M).  A `mutation` argument models a plausible kernel bug (MUTATIONS).  Its channels
  are xlg_add_bank's (bank_exact.f64_bank is their float64 definition).
* bank_czt_member_model: bank_czt_model's rows of a channel fed to subband_exact.member_model, bit for bit what a
  member of a chirp-z bank channel computes.
* bank_czt_m, bank_czt_frames, bank_czt_flops: the kernel's transform length, frames per CTA and FP32 count.
"""
import numpy as np

from bank_fft_exact import _cmul, _sums, fft_rows
from spectrum_czt import positions

F = np.float32
MUTATIONS = ("no_final_chirp", "final_conj_missing", "kernel_unscaled", "chirp_phase_f32", "shift_masked")
BZ_N = 8192  # points per CTA (xlating_kernels.cuh)


def bank_czt_m(K):
    """next_pow2(2 K - 1)."""
    return 1 << (2 * K - 2).bit_length()


def bank_czt_frames(M):
    return BZ_N // M


def bank_czt_flops(fft_flops, K, channels):
    """FP32 instructions of one frame's channel stage: 2 xlg_bank_fft_flops(M) + 4 K + 4 M + 4 C (fft_flops: the
    library's xlg_bank_fft_flops)."""
    M = bank_czt_m(K)
    return 2 * fft_flops(M) + 4 * K + 4 * M + 4 * channels


def _chirp(K, tables, mutation):
    chirp = tables[0]
    if mutation == "chirp_phase_f32":  # pi n^2 / K formed in float32 with n^2 unreduced
        n = np.arange(K, dtype=F)
        t = (F(np.pi) * (n * n) / F(K)).astype(np.float64)
        chirp = np.exp(-1j * t).astype(np.complex64)
    return chirp.real.astype(F), chirp.imag.astype(F)


def _placed_sums(taps, D1, x, P, sizes, mutation):
    """_sums' rows u (sums at (p + r_m) mod K); shift_masked places them at (p + ((s_m - P) & (K - 1))) mod K."""
    K, T1 = 2 * D1, len(taps)
    ure, uim, counts = _sums(taps, D1, x, P, sizes, None)
    if mutation == "shift_masked":
        s = -(T1 - 1) + D1 * np.arange(ure.shape[0], dtype=np.int64)  # s_m - P
        p = np.arange(K)[None, :]
        rows = np.arange(ure.shape[0])[:, None]
        v = (ure[rows, (p + (s % K)[:, None]) % K], uim[rows, (p + (s % K)[:, None]) % K])
        ure, uim = np.zeros_like(ure), np.zeros_like(uim)
        dest = (p + (s & (K - 1))[:, None]) % K
        ure[rows, dest], uim[rows, dest] = v
    return ure, uim, counts


def bank_czt_model(taps, D1, channels, x, P, sizes, tables, mutation=None):
    """bank_czt_cf32_kernel's rows of `channels` (arguments as bank_exact.f64_bank; x complex64, the converted
    ring; tables: bank_any_tables(K)): {k: [complex64 array per block]}.

    mutation (MUTATIONS): no_final_chirp returns conj(v) without the product with c[k mod K];
    final_conj_missing multiplies v itself by the chirp; kernel_unscaled reads Bh without its 1/M;
    chirp_phase_f32 builds c from pi n^2 / K in float32, n^2 not reduced mod 2K; shift_masked reduces
    s_m - P with a mask (K - 1) instead of mod K."""
    assert mutation is None or mutation in MUTATIONS, mutation
    K = 2 * D1
    M = tables[2]
    assert M == bank_czt_m(K)
    pos, bins = positions(M)
    cr, ci = _chirp(K, tables, mutation)
    kr, ki = tables[1].real.astype(F), tables[1].imag.astype(F)
    if mutation == "kernel_unscaled":
        kr, ki = kr * F(M), ki * F(M)
    ure, uim, counts = _placed_sums(taps, D1, x, P, sizes, mutation)
    n = ure.shape[0]
    ar, ai = np.zeros((n, M), F), np.zeros((n, M), F)
    ar[:, :K], ai[:, :K] = _cmul(ure, uim, cr[None, :], ci[None, :])
    fft_rows(ar, ai, M)
    yr, yi = _cmul(ar, ai, kr[None, :], ki[None, :])
    vr, vi = np.empty_like(yr), np.empty_like(yi)
    vr[:, bins], vi[:, bins] = yr, -yi
    fft_rows(vr, vi, M)
    out = {}
    for k in channels:
        kk = k % K
        a, b = vr[:, pos[kk]], vi[:, pos[kk]]
        if mutation == "no_final_chirp":
            re, im = a, -b
        elif mutation == "final_conj_missing":
            re, im = _cmul(a, b, cr[kk], ci[kk])
        else:
            re, im = _cmul(a, -b, cr[kk], ci[kk])
        y = np.empty(n, np.complex64)
        y.real, y.imag = re, im
        out[k] = np.split(y, np.cumsum(counts)[:-1])
    return out


def bank_czt_member_model(taps1, D1, k, x, P, sizes, members, fs, tables, mat=0, attach=0):
    """Members of channel k of a chirp-z bank: bank_czt_model's rows of the channel fed to member_model.
    Arguments as bank_exact.bank_member_model, plus the bank's tables."""
    from subband_exact import member_consts, member_model
    rows = bank_czt_model(taps1, D1, [k], x, P, sizes, tables)[k][mat:]
    classes = {}
    for i, (l2, d2, taps2, offset) in enumerate(members):
        classes.setdefault((l2, d2, len(taps2)), []).append(i)
    outs = [None] * len(members)
    for (l2, d2, _), idx in classes.items():
        consts = [member_consts(np.asarray(members[i][2], F), d2, members[i][3], l2, fs // D1) for i in idx]
        got = member_model(rows, attach, l2, d2, [c[0] for c in consts], [c[1] for c in consts])
        for i, y in zip(idx, got):
            outs[i] = y
    return outs
