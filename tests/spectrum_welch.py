"""References of the Welch spectrum tests (xlg_add_spectrum_ex).  No GPU.

* welch_model: the rows the extended kernels compute, in their exact float32 order (xlating_kernels.cuh,
  "Extended spectra"): frames every H samples, each sample times the window in one rounded float32 multiply,
  spectrum_exact's channel stage (dft32) and power (power32), then the max of the row's frames or their mean
  (a float32 sum from +0 in frame order, divided once by float32(F)), and the reference's half swap.  A
  `mutation` argument models a plausible bug (MUTATIONS).
* welch_f64: the float64 definition of the same rows (include/xlating_group.h, xlg_add_spectrum_ex).
* frames_done: the walk's closed form of the frames completed after d samples; model_blocks: rows per block.
"""
import numpy as np

from spectrum_exact import F32, dft32, half_swap, power32

MUTATIONS = ("window_reversed", "hop_ignored", "mean_over_f_minus_1", "fold_reversed", "frame_count_off_by_one")


def period(W, F, S, H):
    return (F - 1) * H + W + S


def welch_frames(x, W, F, S, H, mutation=None):
    """The frames of every row x completes, (rows, F, W) complex64; x starts at the attach point P."""
    x = np.asarray(x, np.complex64)
    if mutation == "hop_ignored":
        H = W
    R, span = period(W, F, S, H), (F - 1) * H + W
    rows = (x.size - span) // R + 1 if x.size >= span else 0
    if rows == 0:
        return np.zeros((0, F, W), np.complex64)
    start = R * np.arange(rows)[:, None, None] + H * np.arange(F)[None, :, None] + np.arange(W)[None, None, :]
    return x[start]


def windowed(fr, window, mutation=None):
    """z = (x.re * w, x.im * w), each product rounded to float32; no window: z = x."""
    if window is None:
        return fr
    w = np.asarray(window, F32)
    if mutation == "window_reversed":
        w = w[::-1]
    z = np.empty(fr.shape, np.complex64)
    z.real = fr.real.astype(F32) * w
    z.imag = fr.imag.astype(F32) * w
    return z


def reduce32(p, F, mean, mutation=None):
    """(rows, F, W) powers -> (rows, W): the max, or the float32 sum from +0 in frame order over float32(F)."""
    if not mean:
        return p.max(axis=1)
    s = np.zeros((p.shape[0], p.shape[2]), F32)
    order = range(F - 1, -1, -1) if mutation == "fold_reversed" else range(F)
    for f in order:
        s = s + p[:, f]
    return s / F32(F - 1 if mutation == "mean_over_f_minus_1" and F > 1 else F)


def welch_model(x, W, F, S, H=None, window=None, mean=False, power=True, mutation=None):
    """The spectrum's rows over x (complex64 from the attach point on): (rows, W) float32, linear power or
    (power=False) 10 * log10 in float32 (numpy's log10, within an ulp or two of log10f)."""
    assert mutation is None or mutation in MUTATIONS, mutation
    H = W if H is None else H
    fr = windowed(welch_frames(x, W, F, S, H, mutation), window, mutation)
    if fr.shape[0] == 0:
        return np.zeros((0, W), F32)
    xr, xi = dft32(fr, W)
    v = half_swap(reduce32(power32(xr, xi, W), F, mean, mutation))
    return v if power else F32(10) * np.log10(v).astype(F32)


def welch_f64(x, W, F, S, H=None, window=None, mean=False):
    """The definition in float64: |DFT(x w) / W|^2 + 1e-20, max or mean over the row's frames, half swapped."""
    H = W if H is None else H
    fr = welch_frames(x, W, F, S, H).astype(np.complex128)
    if window is not None:
        fr = fr * np.asarray(window, np.float64)
    if fr.shape[0] == 0:
        return np.zeros((0, W))
    p = np.abs(np.fft.fft(fr, axis=-1) / W) ** 2 + 1e-20
    return half_swap(p.mean(axis=1) if mean else p.max(axis=1))


def frames_done(d, W, F, S, H, mutation=None):
    """Frames completed after d source samples: (d // R) F + g(d % R), g(o) = 0 below W, else
    min(F, (o - W) // H + 1) (xlating_group.cu, walk_spectrum)."""
    R = period(W, F, S, H)
    o = d % R
    g = 0 if o < W else min(F, (o - W) // H + (2 if mutation == "frame_count_off_by_one" else 1))
    return d // R * F + g


def model_blocks(x, sizes, W, F, S, H=None, window=None, mean=False, attach=0, power=True, mutation=None):
    """Rows per block: the model's rows of x[attach sample:], each returned with the block after which
    frames_done first counts all its frames (attach: the block the spectrum is attached before; None before)."""
    H = W if H is None else H
    ends = np.cumsum([0] + list(sizes))
    P = int(ends[attach])
    rows = welch_model(x[P:ends[-1]], W, F, S, H, window, mean, power, mutation)
    out, done = [], 0
    for b in range(len(sizes)):
        if b < attach:
            out.append(None)
            continue
        n = frames_done(int(ends[b + 1]) - P, W, F, S, H, mutation) // F
        out.append(rows[done:n])
        done = n
    return out


def last_sample_blocks(n_rows, sizes, W, F, S, H, attach=0):
    """The block holding each row's last frame sample P + r R + (F - 1) H + W - 1: the definition model_blocks'
    frame count must agree with."""
    ends = np.cumsum([0] + list(sizes))
    last = int(ends[attach]) + period(W, F, S, H) * np.arange(n_rows) + (F - 1) * H + W - 1
    return np.searchsorted(ends, last, side="right") - 1


def fbuf_frames(cap, W, S, H):
    """The frame buffer's rows: the most frames a block of at most cap samples completes (their last samples are
    at least min(H, W + S) apart)."""
    return (cap - 1) // min(H, W + S) + 1


def hann(W):
    """The periodic Hann window in float32 (scipy.signal.get_window('hann', W))."""
    return (0.5 - 0.5 * np.cos(2 * np.pi * np.arange(W) / W)).astype(F32)
