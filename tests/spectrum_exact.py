"""References of the spectrum tests (xlg_add_spectrum).  No GPU.

* spectrum_model: the rows the kernels compute, in their exact float32 order (xlating_kernels.cuh, "Spectrum
  rows"): spectrum_fft_kernel's FFT (W a power of two from 4 to 4096) or spectrum_direct_kernel's fmaf chains,
  the normalised power, the max over each row's frames and the reference's half swap; linear rows, or dB rows
  through numpy's log10.  A `mutation` argument models a plausible bug (MUTATIONS).
* f64_rows: the float64 definition of the same rows (include/xlating_group.h).
* half_swap: spectrogram.c:156-163's swap, odd widths' quirk included.
* golden_stimulus, read_png, GOLDENS: the reference's spectrogram goldens (tests/golden/spectrogram).
"""
import os
import struct
import zlib

import numpy as np

from bank_exact import twiddles
from bank_fft_exact import bank_fft_pos, fft_rows
from subband_exact import fmaf

F32 = np.float32
MUTATIONS = ("true_fftshift", "skip_ignored", "normalise_after_square", "no_floor")
GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "spectrogram")
# image -> (format, width); every golden is fs = 128 over 256 complex samples
GOLDENS = {"spectrogram_cu8.png": ("cu8", 64), "spectrogram_cs16.png": ("cs16", 64),
           "spectrogram_cf32.png": ("cf32", 64), "spectrogram_cf32_odd.png": ("cf32", 63)}
GOLDEN_FS = 128


def spec_fft(W):
    return 4 <= W <= 4096 and W & (W - 1) == 0


def period(W, F, S, mutation=None):
    return F * W + (0 if mutation == "skip_ignored" else S)


def frames(x, W, F, S, mutation=None):
    """The frames of every row x completes, (rows, F, W) complex64; x starts at the attach point P."""
    x = np.asarray(x, np.complex64)
    R = period(W, F, S, mutation)
    rows = (x.size - F * W) // R + 1 if x.size >= F * W else 0
    if rows == 0:
        return np.zeros((0, F, W), np.complex64)
    start = R * np.arange(rows)[:, None, None] + W * np.arange(F)[None, :, None] + np.arange(W)[None, None, :]
    return x[start]


def half_swap(v, mutation=None):
    """out[j] = v[W/2 + j], out[W/2 + j] = v[j] for j < W/2 (rounded down); odd W keeps v[W-1] at W-1.  The
    true_fftshift mutation rotates by ceil(W/2) instead (differs for odd W only)."""
    W = v.shape[-1]
    h = W // 2
    if mutation == "true_fftshift":
        return np.roll(v, -((W + 1) // 2), axis=-1)
    idx = np.array([h + j if j < h else (j - h if j < 2 * h else W - 1) for j in range(W)], np.int64)
    return v[..., idx]


def dft32(fr, W):
    """X of every frame (..., W) complex64 as the channel stage computes it: (re, im) float32 arrays."""
    shape = fr.shape
    a = fr.reshape(-1, W)
    if spec_fft(W):
        ure, uim = a.real.astype(F32).copy(), a.imag.astype(F32).copy()
        fft_rows(ure, uim, W)
        pos = np.array([bank_fft_pos(k, W) for k in range(W)])
        return ure[:, pos].reshape(shape), uim[:, pos].reshape(shape)
    tw = twiddles(W)
    wr, wi = tw.real.astype(F32), tw.imag.astype(F32)
    ar, ai = a.real.astype(F32), a.imag.astype(F32)
    k = np.arange(W)
    xr = np.zeros(a.shape, F32)
    xi = np.zeros(a.shape, F32)
    for n in range(W):
        t = (k * n) % W
        xr = fmaf(ar[:, n:n + 1], wr[t][None, :], xr)
        xr = fmaf(-ai[:, n:n + 1], wi[t][None, :], xr)
        xi = fmaf(ar[:, n:n + 1], wi[t][None, :], xi)
        xi = fmaf(ai[:, n:n + 1], wr[t][None, :], xi)
    return xr.reshape(shape), xi.reshape(shape)


def power32(xr, xi, W, mutation=None):
    inv = F32(1) / F32(W)
    if mutation == "normalise_after_square":
        p = (xr * xr + xi * xi) * inv
    else:
        cr, ci = xr * inv, xi * inv
        p = cr * cr + ci * ci
    return p if mutation == "no_floor" else p + F32(1e-20)


def spectrum_model(x, W, F, S, power=True, mutation=None):
    """The spectrum's rows over x (complex64 from the attach point on): (rows, W) float32, linear power or
    (power=False) 10 * log10 in float32 (numpy's log10, within an ulp or two of log10f)."""
    assert mutation is None or mutation in MUTATIONS, mutation
    xr, xi = dft32(frames(x, W, F, S, mutation), W)
    v = power32(xr, xi, W, mutation).max(axis=1) if xr.shape[0] else np.zeros((0, W), F32)
    v = half_swap(v, mutation)
    return v if power else F32(10) * np.log10(v).astype(F32)


def f64_rows(x, W, F, S, power=True):
    """The definition in float64: |DFT / W|^2 + 1e-20, max over the row's frames, half swapped."""
    X = np.fft.fft(frames(x, W, F, S).astype(np.complex128), axis=-1) / W
    v = half_swap((np.abs(X) ** 2 + 1e-20).max(axis=1)) if X.shape[0] else np.zeros((0, W))
    return v if power else 10 * np.log10(v)


def model_blocks(x, sizes, W, F, S, attach=0, power=True):
    """Rows per block: the model's rows of x[attach_sample:] returned with the block holding each row's last
    frame sample (attach: the block the spectrum is attached before)."""
    ends = np.cumsum([0] + list(sizes))
    P = int(ends[attach])
    rows = spectrum_model(x[P:ends[-1]], W, F, S, power)
    R = F * W + S
    last = P + R * np.arange(rows.shape[0]) + F * W  # exclusive end of each row's last frame
    out = []
    for b in range(len(sizes)):
        sel = (last > ends[b]) & (last <= ends[b + 1])
        out.append(rows[sel] if b >= attach else None)
    return out


def golden_stimulus(fmt):
    """The 512 scalars of test/utils.c:137-174 for 256 complex samples, as raw elements (cu8, cs16) or
    complex64 (cf32)."""
    i = np.arange(512)
    if fmt == "cu8":
        return (i & 0xFF).astype(np.uint8)
    if fmt == "cs16":
        return (i - 256).astype(np.int16)
    v = np.sin(i.astype(F32)).astype(F32)
    return (v[0::2] + 1j * v[1::2]).astype(np.complex64)


def read_png(path):
    """An 8-bit grey, non-interlaced PNG as a (height, width) uint8 array (zlib and the five row filters)."""
    data = open(path, "rb").read()
    assert data[:8] == b"\x89PNG\r\n\x1a\n"
    pos, idat = 8, b""
    w = h = None
    while pos < len(data):
        n, kind = struct.unpack(">I4s", data[pos:pos + 8])
        body = data[pos + 8:pos + 8 + n]
        if kind == b"IHDR":
            w, h, depth, color, _, _, interlace = struct.unpack(">IIBBBBB", body)
            assert depth == 8 and color == 0 and interlace == 0
        elif kind == b"IDAT":
            idat += body
        pos += 12 + n
    raw = zlib.decompress(idat)
    img = np.zeros((h, w), np.uint8)
    prev = np.zeros(w, np.int64)
    for r in range(h):
        f, line = raw[r * (w + 1)], np.frombuffer(raw[r * (w + 1) + 1:(r + 1) * (w + 1)], np.uint8).astype(np.int64)
        cur = np.zeros(w, np.int64)
        for c in range(w):
            a = cur[c - 1] if c else 0
            b, cc = prev[c], (prev[c - 1] if c else 0)
            if f == 0:
                pred = 0
            elif f == 1:
                pred = a
            elif f == 2:
                pred = b
            elif f == 3:
                pred = (a + b) // 2
            else:
                p = a + b - cc
                pa, pb, pc = abs(p - a), abs(p - b), abs(p - cc)
                pred = a if pa <= pb and pa <= pc else (b if pb <= pc else cc)
            cur[c] = (line[c] + pred) & 0xFF
        img[r] = cur
        prev = cur
    return img


def log10f_bound_db(v):
    """Largest |10 * log10f(v) - 10 * log10(v)| the emit pass can show in float32: log10f's documented 2 ulp
    (CUDA C Programming Guide, single-precision functions), the multiply by 10 and the output's own rounding."""
    y = np.abs(10 * np.log10(np.asarray(v, np.float64)))
    ulp = np.spacing(np.maximum(np.abs(np.log10(np.asarray(v, np.float64))), 1e-30).astype(F32)).astype(np.float64)
    return 10 * 2 * ulp + 2 * np.spacing(y.astype(F32)).astype(np.float64)

