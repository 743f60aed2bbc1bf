"""References of the chirp-z spectrum tests (xlg_add_spectrum_any, W above 4096 and not a power of two).  No GPU.

* czt_model: the rows the chirp-z kernels compute, in their float32 order (xlating_kernels.cuh, "Chirp-z
  spectra"), on the library's own tables (xlg_spectrum_any_tables: the chirp c and Bh in position order):
  a = cmul(z, c) padded with zeros to M, A = fft_rows at K = M, Y = cmul(A, Bh) at each position, conj(Y)
  scattered to natural order, v = fft_rows at K = M again, p = power32 of v at bank_fft_pos(k, M) for k < W.
  Frames, window, max or mean and the half swap are spectrum_welch's.  With two_pass=True both transforms go
  through spectrum_wide.two_pass_rows (the kernels' pass A / pass B split).  A `mutation` argument models a
  plausible bug (MUTATIONS).
* czt_blocks: rows per block, as spectrum_wide.wide_blocks.
* czt_m, chirp_f64, kernel_f64: M and the float64 definitions of the tables.
"""
import functools

import numpy as np

from bank_fft_exact import _cmul, bank_fft_pos, fft_rows
from spectrum_exact import F32, half_swap, power32
from spectrum_welch import frames_done, reduce32, welch_frames, windowed
from spectrum_wide import two_pass_rows

# every M boundary: 4097 and 8191 (M = 16384), 8193 and 12288 (32768), 16385 and 32767 (65536), 32769 to 65535
# (131072); 65521 is prime
CZT_WIDTHS = (4097, 5000, 8191, 8193, 12288, 16385, 32767, 32769, 48000, 65521, 65535)
MUTATIONS = ("chirp_index_32bit", "chirp_sign_flipped", "kernel_natural_order", "scatter_by_pos", "stale_tail",
             "bins_above_w_folded", "kernel_unscaled")


def czt_m(W):
    """next_pow2(2 W - 1)."""
    return 1 << (2 * W - 2).bit_length()


def chirp_f64(W, index32=False):
    """c[n] = e^{-i pi (n^2 mod 2W) / W}, n < W, in float64; index32: n^2 wrapped to a signed 32-bit int first and
    reduced with C's %, the overflow the 64-bit index avoids."""
    n = np.arange(W, dtype=np.int64)
    if index32:
        r = np.fmod((n * n).astype(np.uint32).view(np.int32).astype(np.int64), 2 * W)
    else:
        r = (n * n) % (2 * W)
    return np.exp(-1j * np.pi * r / W)


def kernel_f64(W, c=None):
    """Bh: the M-point DFT of b[m] = conj(c[|m|]), |m| < W, wrapped mod M, over M, natural order, float64."""
    M = czt_m(W)
    c = chirp_f64(W) if c is None else c
    b = np.zeros(M, np.complex128)
    b[:W] = np.conj(c)
    b[M - W + 1:] = np.conj(c[1:])[::-1]
    return np.fft.fft(b) / M


@functools.lru_cache(maxsize=None)
def positions(M):
    """pos[k] = bank_fft_pos(k, M); bins[p]: its inverse."""
    pos = np.array([bank_fft_pos(k, M) for k in range(M)])
    bins = np.empty(M, np.int64)
    bins[pos] = np.arange(M)
    return pos, bins


def _mutated_tables(W, tables, mutation):
    """(c, Bh in position order) as complex64 pairs of float32 arrays, with the mutation's change."""
    chirp, kern, M = tables
    pos, _ = positions(M)
    if mutation == "chirp_index_32bit":  # the host's tables built with the 32-bit index
        c64 = chirp_f64(W, index32=True)
        chirp, kern = c64.astype(np.complex64), kernel_f64(W, c64)[np.argsort(pos)].astype(np.complex64)
    cr, ci = chirp.real.astype(F32), chirp.imag.astype(F32)
    if mutation == "chirp_sign_flipped":
        ci = -ci
    kr, ki = kern.real.astype(F32), kern.imag.astype(F32)
    if mutation == "kernel_natural_order":  # Bh read as if stored by bin
        kr, ki = kr[pos], ki[pos]
    if mutation == "kernel_unscaled":
        kr, ki = kr * F32(M), ki * F32(M)
    return cr, ci, kr, ki


def _transform(ure, uim, M, two_pass):
    if two_pass:
        two_pass_rows(ure, uim, M)
    else:
        fft_rows(ure, uim, M)


def czt_power(z, W, tables, two_pass=False, mutation=None):
    """p of every (windowed) frame z (..., W) complex64: float32 (..., W), bins in natural order."""
    shape = z.shape
    z = z.reshape(-1, W)
    M = tables[2]
    pos, bins = positions(M)
    cr, ci, kr, ki = _mutated_tables(W, tables, mutation)
    ar, ai = np.zeros((z.shape[0], M), F32), np.zeros((z.shape[0], M), F32)
    ar[:, :W], ai[:, :W] = _cmul(z.real.astype(F32), z.imag.astype(F32), cr[None, :], ci[None, :])
    if mutation == "stale_tail":  # the padding left from the previous frame's transformed row
        for f in range(z.shape[0]):
            if f > 0:
                ar[f, W:], ai[f, W:] = ar[f - 1, W:], ai[f - 1, W:]
            r, i = ar[f:f + 1].copy(), ai[f:f + 1].copy()
            _transform(r, i, M, two_pass)
            ar[f], ai[f] = r[0], i[0]
    else:
        _transform(ar, ai, M, two_pass)
    yr, yi = _cmul(ar, ai, kr[None, :], ki[None, :])
    nr, ni = np.empty_like(yr), np.empty_like(yi)
    dst = pos if mutation == "scatter_by_pos" else bins
    nr[:, dst], ni[:, dst] = yr, -yi
    _transform(nr, ni, M, two_pass)
    if mutation == "bins_above_w_folded":  # every bin's power folded into the row at k mod W by the max
        p = power32(nr[:, pos], ni[:, pos], W)
        out = p[:, :W].copy()
        for k0 in range(W, M, W):
            seg = p[:, k0:k0 + W]
            out[:, :seg.shape[1]] = np.maximum(out[:, :seg.shape[1]], seg)
        return out.reshape(shape)
    return power32(nr[:, pos[:W]], ni[:, pos[:W]], W).reshape(shape)


def czt_model(x, W, F, S, tables, H=None, window=None, mean=False, power=True, two_pass=False, mutation=None):
    """The chirp-z spectrum's rows over x (complex64 from the attach point on): (rows, W) float32, linear power or
    (power=False) 10 * log10 in float32."""
    assert mutation is None or mutation in MUTATIONS, mutation
    H = W if H is None else H
    fr = welch_frames(x, W, F, S, H)
    if fr.shape[0] == 0:
        return np.zeros((0, W), F32)
    p = czt_power(windowed(fr, window), W, tables, two_pass, mutation)
    v = half_swap(reduce32(p, F, mean))
    return v if power else F32(10) * np.log10(v).astype(F32)


def czt_blocks(x, sizes, W, F, S, tables, H=None, window=None, mean=False, attach=0, power=True):
    """Rows per block: czt_model's rows of x[attach sample:], each with the block after which frames_done first
    counts all its frames (None before the attach block)."""
    H = W if H is None else H
    ends = np.cumsum([0] + list(sizes))
    P = int(ends[attach])
    rows = czt_model(x[P:ends[-1]], W, F, S, tables, H, window, mean, power)
    out, done = [], 0
    for b in range(len(sizes)):
        if b < attach:
            out.append(None)
            continue
        n = frames_done(int(ends[b + 1]) - P, W, F, S, H) // F
        out.append(rows[done:n])
        done = n
    return out
