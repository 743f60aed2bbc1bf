"""References of the wide spectrum tests (W a power of two from 8192 to 65536).  No GPU.

* wide_model: the rows the wide kernels compute.  X is bank_fft_exact.fft_rows at K = W, bin k at
  bank_fft_pos(k, W); frames, window, power, max or mean and the half swap are spectrum_welch's.  With
  two_pass=True (or a mutation) X comes from two_pass_rows instead, the kernels' split restated: the first
  wide_stages(W) radix-4 stages over the whole frame (spectrum_wide_a_kernel), then fft_rows at K = C on each
  contiguous chunk of C = wide_chunk(W) points with the C-point table (spectrum_wide_b_kernel).  A `mutation`
  argument models a plausible kernel bug (MUTATIONS).
* wide_blocks: rows per block, as spectrum_welch.model_blocks (whose channel stage stops at 4096).
"""
import functools

import numpy as np

from bank_exact import twiddles
from bank_fft_exact import _cmul, bank_fft_pos, fft_rows, fft_stages
from spectrum_exact import F32, half_swap, power32
from spectrum_welch import frames_done, reduce32, welch_frames, windowed

WIDE_WIDTHS = (8192, 16384, 32768, 65536)
MUTATIONS = ("chunk_twiddles_w_table", "pass_a_stage_dropped", "chunks_strided", "positions_of_chunk",
             "window_after_pass_a")


def wide_stages(W):
    """Radix-4 stages of pass A: one at 8192 and 16384, two at 32768 and 65536."""
    return 2 if W > 16384 else 1


def wide_chunk(W):
    return W >> (2 * wide_stages(W))


@functools.lru_cache(maxsize=None)
def _table(K):
    tw = twiddles(K)
    return tw.real.astype(F32), tw.imag.astype(F32)


def _stage4(ure, uim, L, wr, wi, stride):
    """One radix-4 stage at length L over rows of ure.shape[1] points, fft_rows' butterfly, table (wr, wi) read at
    `stride` (in place)."""
    K = ure.shape[1]
    q4 = L // 4
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
        t = q * j * stride
        ure[:, idx[q]], uim[:, idx[q]] = _cmul(y[q][0], y[q][1], wr[t][None, :], wi[t][None, :])


def pass_a(ure, uim, W, mutation=None):
    """The first wide_stages(W) stages of the W-point transform, W table at stride W / L (in place)."""
    wr, wi = _table(W)
    stages = fft_stages(W)[:wide_stages(W)]
    if mutation == "pass_a_stage_dropped":
        stages = stages[:-1]
    for L, _ in stages:
        _stage4(ure, uim, L, wr, wi, W // L)


def two_pass_rows(ure, uim, W, window=None, mutation=None):
    """fft_rows(ure, uim, W) restated as the kernels split it (in place): pass A, then each contiguous chunk of
    C points through fft_rows at K = C."""
    pass_a(ure, uim, W, mutation)
    if mutation == "window_after_pass_a" and window is not None:
        w = np.asarray(window, F32)[None, :]
        ure *= w
        uim *= w
    C = wide_chunk(W)
    n = W // C
    for c in range(n):
        cols = np.arange(c, W, n) if mutation == "chunks_strided" else np.arange(c * C, (c + 1) * C)
        sr, si = ure[:, cols].copy(), uim[:, cols].copy()
        if mutation == "chunk_twiddles_w_table":  # the W-point table read as if it were the C-point one
            wr, wi = _table(W)
            for L, R in fft_stages(C):
                if R == 4:
                    _stage4(sr, si, L, wr, wi, C // L)
                else:
                    ar, ai = sr[:, 0::2].copy(), si[:, 0::2].copy()
                    sr[:, 0::2], si[:, 0::2] = ar + sr[:, 1::2], ai + si[:, 1::2]
                    sr[:, 1::2], si[:, 1::2] = ar - sr[:, 1::2], ai - si[:, 1::2]
        else:
            fft_rows(sr, si, C)
        ure[:, cols], uim[:, cols] = sr, si
    return ure, uim


@functools.lru_cache(maxsize=None)
def positions(W, mutation=None):
    """Where bin k lies in the transformed row: bank_fft_pos(k, W)."""
    K = wide_chunk(W) if mutation == "positions_of_chunk" else W
    return np.array([bank_fft_pos(k, K) for k in range(W)])


def wide_dft32(fr, W, window=None, two_pass=False, mutation=None):
    """X of every frame (..., W) complex64, bins in natural order, as (re, im) float32 arrays; the window is
    applied to the frame as spectrum_welch.windowed does (or, mutated, after pass A)."""
    shape = fr.shape
    z = fr if mutation == "window_after_pass_a" else windowed(fr, window)
    a = z.reshape(-1, W)
    ure, uim = a.real.astype(F32).copy(), a.imag.astype(F32).copy()
    if two_pass or mutation is not None:
        two_pass_rows(ure, uim, W, window, mutation)
    else:
        fft_rows(ure, uim, W)
    pos = positions(W, mutation)
    return ure[:, pos].reshape(shape), uim[:, pos].reshape(shape)


def wide_model(x, W, F, S, H=None, window=None, mean=False, power=True, two_pass=False, mutation=None):
    """The wide spectrum's rows over x (complex64 from the attach point on): (rows, W) float32, linear power or
    (power=False) 10 * log10 in float32."""
    assert mutation is None or mutation in MUTATIONS, mutation
    H = W if H is None else H
    fr = welch_frames(x, W, F, S, H)
    if fr.shape[0] == 0:
        return np.zeros((0, W), F32)
    xr, xi = wide_dft32(fr, W, window, two_pass, mutation)
    v = half_swap(reduce32(power32(xr, xi, W), F, mean))
    return v if power else F32(10) * np.log10(v).astype(F32)


def wide_blocks(x, sizes, W, F, S, H=None, window=None, mean=False, attach=0, power=True):
    """Rows per block: wide_model's rows of x[attach sample:], each with the block after which frames_done first
    counts all its frames (None before the attach block)."""
    H = W if H is None else H
    ends = np.cumsum([0] + list(sizes))
    P = int(ends[attach])
    rows = wide_model(x[P:ends[-1]], W, F, S, H, window, mean, power)
    out, done = [], 0
    for b in range(len(sizes)):
        if b < attach:
            out.append(None)
            continue
        n = frames_done(int(ends[b + 1]) - P, W, F, S, H) // F
        out.append(rows[done:n])
        done = n
    return out
