"""An integer model of the reference's Q15 path (src/xlating.c:92-140) at any centre frequency.

The reference computes, per output, in this order:

* each complex product pair in 32-bit int, `(int32_t)ar * bi + (int32_t)ai * br`, then adds it to an
  int64 accumulator.  The imaginary pair is 2^31 for x = (-32768, -32768) and a tap of (-32768, -32768): it
  wraps to -2^31 (gcc's build; the real pair cannot overflow);
* `saturate_to_int16(acc >> 15)`: an arithmetic (floor) shift, the int64 -> int32 narrowing of the argument
  (it matters once |acc| >= 2^46), then saturation to int16;
* the rotation by the Q15 phase in int arithmetic, >> 15 and saturation;
* the oscillator step phase * incr in int arithmetic, >> 15 and saturation, never renormalised.

The constants come from the host (csrc/taps_host.c, as tests/test_abi.py reads them): the reversed Q15 band-pass
taps (int16)(x * 32768), which wrap for |x * 32768| >= 32768 (gcc converts through int32), and the increment
(int16)(incr * 32767).  `Arith` names each of the rules above so that a test can check each one is needed.

At centre 0 the oscillator decays to 0 within 32767 outputs; at other centres floor rounding holds it in a
limit cycle of nonzero magnitude.  `Osc` walks the recursion and remembers every state it has seen, so it
finds the cycle and returns the phase of any output, 2^32 included, exactly.

numpy only; `host_consts` takes the product's ctypes library from its caller.
"""
import ctypes as C
from dataclasses import dataclass, replace

import numpy as np

from exact import _outputs_per_call, to_q15


@dataclass(frozen=True)
class Arith:
    pair_wrap: bool = True   # each product pair wraps to int32 before the int64 sum
    narrow: bool = True      # (int32)(acc >> 15) before sat16
    sat_fir: bool = True     # sat16 of the filter output
    sat_rot: bool = True     # sat16 of the rotated output
    sat_osc: bool = True     # sat16 of the oscillator step
    floor: bool = True       # >> 15 is a floor shift (False: round half up, (v + 2^14) >> 15)


REF = Arith()
MUTATIONS = {"pair widened to int64": replace(REF, pair_wrap=False),
             "(int32) narrowing dropped": replace(REF, narrow=False),
             "sat16 dropped at the filter output": replace(REF, sat_fir=False),
             "sat16 dropped at the rotation": replace(REF, sat_rot=False),
             "sat16 dropped at the oscillator": replace(REF, sat_osc=False),
             ">> 15 rounds": replace(REF, floor=False)}


def wrap32(v):
    v = np.asarray(v, dtype=np.int64)
    return ((v + 2 ** 31) & 0xFFFFFFFF) - 2 ** 31


def wrap16(v):
    v = np.asarray(v, dtype=np.int64)
    return ((v + 2 ** 15) & 0xFFFF) - 2 ** 15


def sat16(v):
    return np.clip(v, -32768, 32767)


def _shr15(v, a):
    v = np.asarray(v, dtype=np.int64)
    return v >> 15 if a.floor else (v + (1 << 14)) >> 15


def _sat(v, on):
    return sat16(v) if on else v


def q15_of(x):
    """(int16_t)(x * 32768) of float32 values as gcc compiles it (truncate to int32, keep the low 16 bits)."""
    p = np.asarray(x, dtype=np.float32) * np.float32(32768)
    return wrap16(np.trunc(p.astype(np.float64)).astype(np.int64))


# ---------------------------------------------------------------------------
# the oscillator
# ---------------------------------------------------------------------------
class Osc:
    """The Q15 phase of a new filter (32767 + 0i) after k outputs, for any k: the walk is remembered until a
    state repeats, after which the sequence is periodic (mu: first index of the cycle, lam: its length)."""

    def __init__(self, qinc, arith=REF):
        self.ir, self.ii = int(qinc[0]), int(qinc[1])
        self.a = arith
        self.seq = [(32767, 0)]
        self.seen = {(32767, 0): 0}
        self.mu = self.lam = None

    def step(self, pr, pi):
        a = self.a
        nr, ni = pr * self.ir - pi * self.ii, pr * self.ii + pi * self.ir
        if a.floor:
            nr, ni = nr >> 15, ni >> 15
        else:
            nr, ni = (nr + (1 << 14)) >> 15, (ni + (1 << 14)) >> 15
        if a.sat_osc:
            nr, ni = min(32767, max(-32768, nr)), min(32767, max(-32768, ni))
        return nr, ni

    def _walk(self, n):
        while self.lam is None and len(self.seq) < n:
            s = self.step(*self.seq[-1])
            if s in self.seen:
                self.mu = self.seen[s]
                self.lam = len(self.seq) - self.mu
                break
            self.seen[s] = len(self.seq)
            self.seq.append(s)

    def cycle(self, limit=1 << 24):
        """(mu, lam), walking at most `limit` states."""
        self._walk(limit)
        assert self.lam is not None, f"no cycle within {limit} states"
        return self.mu, self.lam

    def phases(self, k0, n):
        """(n, 2) int64: the phases of outputs k0 .. k0 + n - 1."""
        self._walk(k0 + n)
        k = np.arange(k0, k0 + n, dtype=np.int64)
        seq = np.asarray(self.seq, dtype=np.int64).reshape(-1, 2)
        if self.lam is not None:
            k = np.where(k < len(seq), k, self.mu + (k - self.mu) % self.lam)
        return seq[k]

    def magnitude_after(self, k):
        pr, pi = self.phases(k, 1)[0]
        return float(np.hypot(pr, pi))


# ---------------------------------------------------------------------------
# the filter
# ---------------------------------------------------------------------------
def fir(rev, D, xr, xi, starts, arith=REF, chunk=1 << 22):
    """The saturated filter outputs (ar, ai) of the windows starting at `starts` of the stream (xr, xi).
    rev: (T, 2) int Q15 taps in window order."""
    a = arith
    rev = np.asarray(rev, dtype=np.int64)
    T = rev.shape[0]
    tr, ti = rev[:, 0], rev[:, 1]
    Wr = np.lib.stride_tricks.sliding_window_view(xr, T)
    Wi = np.lib.stride_tricks.sliding_window_view(xi, T)
    ar = np.empty(len(starts), np.int64)
    ai = np.empty(len(starts), np.int64)
    step = max(1, chunk // T)
    for s in range(0, len(starts), step):
        idx = starts[s:s + step]
        wr, wi = Wr[idx], Wi[idx]
        pre, pim = wr * tr - wi * ti, wr * ti + wi * tr
        if a.pair_wrap:
            pre, pim = wrap32(pre), wrap32(pim)
        accr, acci = _shr15(pre.sum(axis=1), a), _shr15(pim.sum(axis=1), a)
        if a.narrow:
            accr, acci = wrap32(accr), wrap32(acci)
        ar[s:s + step] = _sat(accr, a.sat_fir)
        ai[s:s + step] = _sat(acci, a.sat_fir)
    return ar, ai


def rotate(ar, ai, ph, arith=REF):
    a = arith
    rr = wrap32(ar * ph[:, 0] - ai * ph[:, 1])
    ri = wrap32(ar * ph[:, 1] + ai * ph[:, 0])
    return _sat(_shr15(rr, a), a.sat_rot), _sat(_shr15(ri, a), a.sat_rot)


def model(rev, qinc, D, fmt, blocks, k0=0, osc=None, arith=REF):
    """A new filter with Q15 taps `rev` (window order) and increment `qinc` fed `blocks` (raw `fmt`
    elements) one call each, its first output taking the oscillator's phase k0 (a fresh filter: 0; the
    window reference of a filter attached m * D samples before blocks[0]: m).  Returns one (n, 2) array per
    block, int16 unless a mutation lets values leave that range (int64 then)."""
    rev = np.asarray(rev, dtype=np.int64).reshape(-1, 2)
    T = rev.shape[0]
    per_call, total = _outputs_per_call(blocks, T, D)
    parts = [to_q15(fmt, b) for b in blocks]
    z = np.zeros(T - 1, dtype=np.int64)
    xr = np.concatenate([z] + [p[0] for p in parts])
    xi = np.concatenate([z] + [p[1] for p in parts])
    if total:
        ar, ai = fir(rev, D, xr, xi, np.arange(total, dtype=np.int64) * D, arith)
        osc = Osc(qinc, arith) if osc is None else osc
        yr, yi = rotate(ar, ai, osc.phases(k0, total), arith)
        y = np.stack([yr, yi], axis=1)
    else:
        y = np.zeros((0, 2), dtype=np.int64)
    if arith == REF or (y.size and y.min() >= -32768 and y.max() <= 32767):
        y = y.astype(np.int16)
    return np.split(y, np.cumsum(per_call)[:-1])


# ---------------------------------------------------------------------------
# constants
# ---------------------------------------------------------------------------
class _Consts(C.Structure):
    _fields_ = [("rev_cf32", C.POINTER(C.c_float)), ("rev_q15", C.POINTER(C.c_int16)),
                ("incr_re", C.c_float), ("incr_im", C.c_float), ("qincr_re", C.c_int16), ("qincr_im", C.c_int16)]


def host_consts(lib, taps, D, center, fs):
    """csrc/taps_host.c's constants of a filter: ((T, 2) int64 reversed Q15 taps, (qincr_re, qincr_im),
    (T,) complex64 reversed band-pass taps)."""
    taps = np.ascontiguousarray(taps, dtype=np.float32)
    fn = lib.xl_client_consts_build
    fn.argtypes = [C.POINTER(C.c_float), C.c_size_t, C.c_uint32, C.c_int32, C.c_uint32, C.POINTER(_Consts)]
    fn.restype = C.c_int
    k = _Consts()
    assert fn(taps.ctypes.data_as(C.POINTER(C.c_float)), len(taps), D, center, fs, C.byref(k)) == 0
    T = len(taps)
    rev = np.ctypeslib.as_array(k.rev_q15, shape=(2 * T,)).astype(np.int64).reshape(T, 2)
    cf = np.ctypeslib.as_array(k.rev_cf32, shape=(2 * T,)).copy().view(np.complex64)
    qinc = (int(k.qincr_re), int(k.qincr_im))
    lib.xl_client_consts_free.argtypes = [C.POINTER(_Consts)]
    lib.xl_client_consts_free(C.byref(k))
    return rev, qinc, cf


class Client:
    """One Q15 filter's model: its host constants and its oscillator walk (shared by every window)."""

    def __init__(self, lib, taps, D, center, fs):
        self.taps, self.D, self.center, self.fs = np.asarray(taps, np.float32), D, center, fs
        self.rev, self.qinc, _ = host_consts(lib, taps, D, center, fs)
        self.osc = Osc(self.qinc)

    def __call__(self, fmt, blocks, k0=0):
        return model(self.rev, self.qinc, self.D, fmt, blocks, k0, self.osc)


# ---------------------------------------------------------------------------
# stimuli
# ---------------------------------------------------------------------------
FS = 2_048_000
WRAP_TAPS = np.array([0, 1.41422, 0], dtype=np.float32)  # at centre -3 fs / 8: the middle tap is (-32768, -32768)
WRAP_CENTER = -3 * FS // 8
LIMIT_CENTERS = (-768000, 640000, 682666, 300000, 12345, -512000)
EDGE_TAPS = np.array([1.0, -1.0, 1 - 2 ** -16, -1 - 2 ** -16, 1.5, -3.0, 2 ** -15, -2 ** -15, 0.5], dtype=np.float32)
FULL = {"cu8": (np.uint8, 0, 255), "cs8": (np.int8, -128, 127), "cs16": (np.int16, -32768, 32767)}


def wrap_input(rng, fmt, n, p=0.25):
    """n complex samples (2n raw elements) of random data, a fraction p of them the most negative sample
    (-32768, -32768) after conversion: cu8 (0, 0), cs8 (-128, -128), cs16 (-32768, -32768)."""
    dt, lo, hi = FULL[fmt]
    x = rng.integers(lo, hi + 1, 2 * n).astype(dt)
    hit = rng.random(n) < p
    x[0::2][hit] = lo
    x[1::2][hit] = lo
    return x


def rail_input(rng, fmt, n):
    """n complex samples at full scale: every part one of the two rails."""
    dt, lo, hi = FULL[fmt]
    return np.where(rng.random(2 * n) < 0.5, lo, hi).astype(dt)


def narrowing_taps(T, center, fs):
    """T real taps whose band-pass Q15 taps at `center` have one part at -32768 each: the larger part of
    cexpf(i * w0) scaled to -32768.5 / 32768 (truncated to -32768, not wrapped)."""
    w0 = np.float32(2 * np.pi * center / fs)
    th = np.arange(T, dtype=np.float32) * w0  # float products, as the host computes them
    c = np.cos(th.astype(np.float64)).astype(np.float32)
    s = np.sin(th.astype(np.float64)).astype(np.float32)
    big = np.where(np.abs(c) >= np.abs(s), c, s).astype(np.float64)
    return (-(32768.5 / 32768) / big).astype(np.float32)


def narrowing_window(rev):
    """cs16 raw elements of one window that drives every imaginary product pair ar * bi + ai * br with the
    window-order Q15 taps `rev` (one part of each at -32768) to at least 2^30: the part at -32768 meets
    -32768, the other part a sample of its own sign (0 where it is -32768 too, so that no pair wraps).  With
    more than 65536 taps the imaginary sum then passes 2^46, and acc >> 15 passes 2^31."""
    br, bi = np.asarray(rev[:, 0]), np.asarray(rev[:, 1])

    def match(b):
        return np.where(b > 0, 32767, np.where(b > -32768, -32768, 0))

    x = np.empty(2 * len(rev), np.int16)
    x[0::2] = np.where(bi == -32768, -32768, match(bi))
    x[1::2] = np.where(bi == -32768, match(br), -32768)
    return x


def narrowing_blocks(rng, rev):
    """cs16 calls for a filter with the Q15 taps `rev` of narrowing_taps(65537, ...) and D = 4096: a designed
    window as the first call (output 16 reads exactly it), random data, then the window again."""
    win = narrowing_window(rev)
    return [win, wrap_input(rng, "cs16", 9000 - 5), wrap_input(rng, "cs16", 5), win]


def edge_clients(rng, fmt, fs=FS):
    """(label, taps, D, centre) of Q15 filters at the edges: the wrapping pair, gain > 1 taps at a 45 degree
    centre, the conversion-edge taps at centre 0 and 300 kHz, the limit-cycle centres, and one-hot taps at
    random centres (as the cf32 phase harness of tests/test_gpu_exact.py)."""
    out = [("wrap", WRAP_TAPS, 1, WRAP_CENTER)]
    out.append(("rails", (rng.uniform(0.6, 0.95, 8) * rng.choice([-1, 1], 8)).astype(np.float32), 3, fs // 8))
    out += [(f"edge taps at {c}", EDGE_TAPS, 2, c) for c in (0, 300000)]
    out += [(f"cycle at {c}", rng.uniform(-0.7, 0.7, 5).astype(np.float32), 1, c) for c in LIMIT_CENTERS]
    for i in range(6):
        D = int(rng.choice([1, 2, 5, 21]))
        T = int(rng.choice([D, 64, 253]))  # T >= D: with D > T the reference's history bookkeeping underflows
        taps = np.zeros(T, np.float32)
        taps[(0, T - 1, int(rng.integers(0, T)))[i % 3]] = rng.choice([0.75, -0.5, 1.0, -1 - 2 ** -16])
        band = fs // 2 - fs // (2 * D)
        out.append((f"one-hot {i}", taps, D, int(rng.integers(-band, band + 1))))
    return out


def edge_blocks(rng, fmt, sizes):
    """Calls of `sizes` complex samples (a negative size: that many samples and one odd trailing element),
    alternating random data with a quarter of wrap samples and full-scale rails."""
    out = []
    for i, n in enumerate(sizes):
        m = abs(n)
        x = wrap_input(rng, fmt, m) if i % 2 == 0 else rail_input(rng, fmt, m)
        if n < 0:
            x = np.concatenate([x, x[:1]])
        out.append(x)
    return out


RAGGED = [4000, 2, 0, 8191, -7, 1, 4000, 16, -2999, 0, 4000, 4000]
