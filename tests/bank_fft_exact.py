"""References of the FFT bank tests (xlg_add_bank_fft).  No GPU.

* bank_fft_model: what bank_fft_cf32_kernel computes, in its exact order (DESIGN.md section 5, "FFT banks"),
  with a `mutation` argument that models a plausible kernel bug (MUTATIONS).  Its channels are xlg_add_bank's
  (bank_exact.f64_bank is their float64 definition).
* bank_fft_member_model: bank_fft_model's rows of a channel fed to subband_exact.member_model, bit for bit what
  a member of an FFT bank channel computes on any taps and input.
* bank_fft_pos, bank_fft_frames, bank_fft_max_taps, fft_stages: the kernel's row layout, frames per CTA, tap
  bound and butterfly schedule.
"""
import numpy as np

from bank_exact import bank_walk, twiddles
from subband_exact import fmaf

F = np.float32
MUTATIONS = ("twiddle_stride_plus_1", "shift_negated", "no_zero_pad", "stages_swapped")
BF_N = 2048  # sums per CTA (xlating_kernels.cuh)


def bank_fft_frames(K):
    return 1 if K >= BF_N else BF_N // K


def bank_fft_max_taps(K):
    return max(16 * K, 16384)


def fft_stages(K):
    """(L, radix) of each stage in order: radix 4 at L = K, K/4, ... while L >= 4, then radix 2 at L = 2."""
    out, L = [], K
    while L >= 4:
        out.append((L, 4))
        L //= 4
    return out + [(2, 2)] if L == 2 else out


def bank_fft_pos(k, K):
    """Where channel k lies in a transformed row: the digit reversal of k mod K (first stage most significant)."""
    k %= K
    pos = 0
    for L, R in fft_stages(K):
        pos += (k % R) * (L // R)
        k //= R
    return pos


def _sums(taps, D1, x, P, sizes, mutation):
    """Phase 1: every frame's sums v[p] (the direct bank's fmaf chains), zero-padded to K and placed at
    (p + r_m) mod K.  Returns (re, im) float32 arrays of (frames, K) and the per-block frame counts."""
    T1, K = len(taps), 2 * D1
    counts, _ = bank_walk(sizes, T1, D1)
    total = int(sum(counts))
    x = np.asarray(x, np.complex64)
    xr, xi = x.real.astype(F), x.imag.astype(F)
    s = P - (T1 - 1) + D1 * np.arange(total, dtype=np.int64)
    hr = np.asarray(taps, F)[::-1].copy()
    KP = min(K, T1)
    vre = np.zeros((total, K), F)
    vim = np.zeros((total, K), F)
    for q in range(-(-T1 // K)):
        p = np.arange(min(KP, T1 - q * K))
        pos = s[:, None] + q * K + p[None, :]
        ok = (pos >= P) & (pos < x.size)
        at = np.clip(pos, 0, max(x.size - 1, 0))
        a = np.where(ok, xr[at] if x.size else 0, 0).astype(F)
        b = np.where(ok, xi[at] if x.size else 0, 0).astype(F)
        vre[:, p] = fmaf(a, hr[q * K + p], vre[:, p])
        vim[:, p] = fmaf(b, hr[q * K + p], vim[:, p])
    if mutation == "no_zero_pad" and T1 < K:  # the padding phases keep stale sums instead of zeros
        vre[:, T1:] = vre[:, np.arange(T1, K) % T1]
        vim[:, T1:] = vim[:, np.arange(T1, K) % T1]
    r = (P - s) % K if mutation == "shift_negated" else (s - P) % K
    dest = (np.arange(K)[None, :] + r[:, None]) % K
    ure = np.zeros_like(vre)
    uim = np.zeros_like(vim)
    rows = np.arange(total)[:, None]
    ure[rows, dest] = vre
    uim[rows, dest] = vim
    return ure, uim, counts


def _cmul(yr, yi, wr, wi):
    return fmaf(-yi, wi, yr * wr), fmaf(yi, wr, yr * wi)


def fft_rows(ure, uim, K, mutation=None):
    """The kernel's in-place FFT of every row (float32 arrays of (frames, K), changed in place)."""
    W = twiddles(K)
    wr, wi = W.real.astype(F), W.imag.astype(F)
    st = fft_stages(K)
    if mutation == "stages_swapped" and len(st) > 1:
        st[0], st[1] = st[1], st[0]
    for L, R in st:
        if R == 2:
            a, b = np.arange(0, K, L), np.arange(0, K, L) + L // 2
            ar, ai, br, bi = ure[:, a], uim[:, a], ure[:, b], uim[:, b]
            ure[:, a], uim[:, a] = ar + br, ai + bi
            ure[:, b], uim[:, b] = ar - br, ai - bi
            continue
        q4, stride = L // 4, K // L + (1 if mutation == "twiddle_stride_plus_1" else 0)
        i = np.arange(K // 4)
        j = i % q4
        idx = [4 * (i - j) + j + q * q4 for q in range(4)]
        a = [(ure[:, ix], uim[:, ix]) for ix in idx]
        t0 = (a[0][0] + a[2][0], a[0][1] + a[2][1])
        t1 = (a[0][0] - a[2][0], a[0][1] - a[2][1])
        t2 = (a[1][0] + a[3][0], a[1][1] + a[3][1])
        t3 = (a[1][0] - a[3][0], a[1][1] - a[3][1])
        y = [(t0[0] + t2[0], t0[1] + t2[1]), (t1[0] + t3[1], t1[1] - t3[0]),
             (t0[0] - t2[0], t0[1] - t2[1]), (t1[0] - t3[1], t1[1] + t3[0])]
        ure[:, idx[0]], uim[:, idx[0]] = y[0]
        for q in (1, 2, 3):
            t = (q * j * stride) % K
            ure[:, idx[q]], uim[:, idx[q]] = _cmul(y[q][0], y[q][1], wr[t][None, :], wi[t][None, :])
    return ure, uim


def bank_fft_model(taps, D1, channels, x, P, sizes, mutation=None):
    """bank_fft_cf32_kernel's rows of `channels` (arguments as bank_exact.f64_bank; x complex64, the converted
    ring): {k: [complex64 array per block]}.

    mutation (MUTATIONS): twiddle_stride_plus_1 reads W at stride K / L + 1; shift_negated places the sums at
    (p - r_m) mod K; no_zero_pad leaves the padding phases T1 <= p < K with stale sums (v[p mod T1]) instead of
    zeros; stages_swapped runs the first two butterfly stages in the other order."""
    assert mutation is None or mutation in MUTATIONS, mutation
    K = 2 * D1
    ure, uim, counts = _sums(taps, D1, x, P, sizes, mutation)
    fft_rows(ure, uim, K, mutation)
    out = {}
    for k in channels:
        c = bank_fft_pos(k, K)
        y = np.empty(ure.shape[0], np.complex64)
        y.real, y.imag = ure[:, c], uim[:, c]
        out[k] = np.split(y, np.cumsum(counts)[:-1])
    return out


def bank_fft_member_model(taps1, D1, k, x, P, sizes, members, fs, mat=0, attach=0, renorm=True, mutation=None):
    """Members of channel k of an FFT bank: bank_fft_model's rows of the channel fed to member_model.  Arguments
    as bank_exact.bank_member_model; mutation: an entry of MUTATIONS (the bank) or of subband_exact.MUTATIONS
    (the members)."""
    from subband_exact import MUTATIONS as SB_MUTATIONS, member_consts, member_model
    assert mutation is None or mutation in MUTATIONS or mutation in SB_MUTATIONS, mutation
    rows = bank_fft_model(taps1, D1, [k], x, P, sizes, mutation=mutation if mutation in MUTATIONS else None)[k]
    rows = rows[mat:]
    classes = {}
    for i, (l2, d2, taps2, offset) in enumerate(members):
        classes.setdefault((l2, d2, len(taps2)), []).append(i)
    outs = [None] * len(members)
    for (l2, d2, _), idx in classes.items():
        consts = [member_consts(np.asarray(members[i][2], F), d2, members[i][3], l2, fs // D1) for i in idx]
        got = member_model(rows, attach, l2, d2, [c[0] for c in consts], [c[1] for c in consts], renorm=renorm,
                           mutation=mutation if mutation in SB_MUTATIONS else None)
        for i, y in zip(idx, got):
            outs[i] = y
    return outs
