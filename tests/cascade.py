"""Helpers of the cascade-client tests: a float32 restatement of the reference's float path on cf32 input, the
cascade oracle built on it, the float64 reference filter and small dyadic taps.  No GPU."""
import ctypes as C
import importlib

import numpy as np

from exact import reversed_taps
from oracle import pyoracle as po

F = np.float32


class _Consts(C.Structure):
    _fields_ = [("rev_cf32", C.POINTER(C.c_float)), ("rev_q15", C.POINTER(C.c_int16)),
                ("incr_re", C.c_float), ("incr_im", C.c_float), ("qincr_re", C.c_int16), ("qincr_im", C.c_int16)]


def filter_constants(taps, decimation, center, fs):
    """Reversed rotated taps (complex64) and oscillator step of create_frequency_xlating_filter
    (src/xlating.c:519-549), from the library's host constants, which tests/test_abi.py pins bit for bit to
    the oracle's."""
    lib = importlib.import_module("sdr-server_b200").lib()
    fn = lib.xl_client_consts_build
    fn.argtypes = [C.POINTER(C.c_float), C.c_size_t, C.c_uint32, C.c_int32, C.c_uint32, C.POINTER(_Consts)]
    fn.restype = C.c_int
    free = lib.xl_client_consts_free
    free.argtypes = [C.POINTER(_Consts)]
    free.restype = None
    taps = np.ascontiguousarray(taps, dtype=np.float32)
    k = _Consts()
    assert fn(taps.ctypes.data_as(C.POINTER(C.c_float)), taps.size, decimation, center, fs, C.byref(k)) == 0
    rev = np.ctypeslib.as_array(k.rev_cf32, shape=(2 * taps.size,)).copy().view(np.complex64)
    incr = (F(k.incr_re), F(k.incr_im))
    free(C.byref(k))
    return rev, incr


class FloatPath:
    """The reference's float path (src/xlating.c:52-83) fed cf32 samples, in float32 with every product and
    sum rounded as the strict build rounds them (-ffp-contract=off, __mulsc3's two products and one add per
    component): history of T - 1 zeros at creation, windows every D, taps in order per output, the output
    derotated by the oscillator, which advances once per output and is renormalised once per call with
    hypotf = (float)sqrt of the exact double sum.  Stage B of a cascade client is this at centre 0."""

    def __init__(self, decimation, taps, center, fs):
        rev, (self.inc_re, self.inc_im) = filter_constants(taps, decimation, center, fs)
        self.tr, self.ti = rev.real.astype(F), rev.imag.astype(F)
        self.D, self.T = decimation, rev.size
        self.work = np.zeros(self.T - 1, np.complex64)
        self.ph_re, self.ph_im = F(1), F(0)

    @property
    def history(self):
        return self.work.size

    def process_cf32(self, data, renorm=True):
        w = np.concatenate([self.work, np.asarray(data, dtype=np.complex64)])
        T, D = self.T, self.D
        n_out = (w.size - T) // D + 1 if w.size >= T else 0
        xr, xi = w.real.astype(F), w.imag.astype(F)
        start = np.arange(n_out) * D
        acc_re, acc_im = np.zeros(n_out, F), np.zeros(n_out, F)
        with np.errstate(over="ignore", invalid="ignore"):
            for j in range(T):  # :67-69, one complex MAC per tap, in tap order
                a, b = xr[start + j], xi[start + j]
                acc_re = acc_re + (a * self.tr[j] - b * self.ti[j])
                acc_im = acc_im + (a * self.ti[j] + b * self.tr[j])
        out = np.empty(n_out, np.complex64)
        pr, pi = self.ph_re, self.ph_im
        ph_re, ph_im = np.empty(n_out, F), np.empty(n_out, F)
        for k in range(n_out):  # :70-71, the sequential recursion
            ph_re[k], ph_im[k] = pr, pi
            pr, pi = pr * self.inc_re - pi * self.inc_im, pr * self.inc_im + pi * self.inc_re
        out.real = acc_re * ph_re - acc_im * ph_im
        out.imag = acc_re * ph_im + acc_im * ph_re
        if n_out > 0 and renorm:  # :73
            mag = F(np.sqrt(np.float64(pr) * np.float64(pr) + np.float64(pi) * np.float64(pi)))
            pr, pi = pr / mag, pi / mag
        self.ph_re, self.ph_im = pr, pi
        self.work = w[n_out * D:].copy()  # :76-79
        return out


class CascadeOracle:
    """A cascade client (include/xlating_group.h, xlg_add_client_cascade) as two reference filters called
    block by block: stage A = the oracle filter (d1, taps1, center) at fs fed the block, stage B = FloatPath
    (d2, taps2, centre 0) at fs / d1 fed stage A's cf32 outputs of the same block."""

    def __init__(self, d1, taps1, center_freq, d2, taps2, fs, max_input_len):
        self.a = po.OracleFilter(d1, taps1, center_freq, fs, max_input_len)
        self.b = FloatPath(d2, taps2, 0, fs // d1)

    def process_cf32(self, fmt, data, renorm=True):
        return self.b.process_cf32(self.a.process_cf32(fmt, data, renorm=renorm), renorm=renorm)


def cascade_oracle(d1, taps1, center_freq, d2, taps2, fs, max_input_len):
    return CascadeOracle(d1, taps1, center_freq, d2, taps2, fs, max_input_len)


def f64_filter(taps, D, center, fs, blocks):
    """The reference filter in float64 (exact rotation and oscillator), fed complex blocks one call each.
    Returns one complex128 array per block."""
    T = len(taps)
    w0 = 2 * np.pi * center / fs
    rev = reversed_taps(np.asarray(taps, dtype=np.float64) * np.exp(1j * w0 * np.arange(T)))
    x = np.concatenate([np.zeros(T - 1, complex)] + [np.asarray(b, dtype=complex) for b in blocks])
    n_all = (x.size - T) // D + 1 if x.size >= T else 0
    idx = np.arange(n_all)[:, None] * D + np.arange(T)[None, :]
    y = (x[idx] @ rev if n_all else np.zeros(0, complex)) * np.exp(-1j * w0 * D * np.arange(n_all))
    out, done, avail = [], 0, T - 1
    for b in blocks:
        avail += len(b)
        n = (avail - T) // D + 1 if avail >= T else 0
        out.append(y[done:n])
        done = n
    return out


def small_taps(rng, T, bits):
    """T nonzero taps m / 2^bits, 1 <= |m| <= 2^bits - 1, random signs."""
    m = rng.integers(1, 2 ** bits, T) * rng.choice(np.array([-1, 1]), T)
    return (m / 2.0 ** bits).astype(np.float32)
