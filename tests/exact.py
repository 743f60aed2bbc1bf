"""Stimuli whose exact answer every summation order reproduces, and their float64 / int64 reference.

With centre frequency 0 the band-pass taps equal the low-pass taps (imaginary part +-0), the
oscillator stays at 1 + 0i and renormalisation divides by 1.  With dyadic taps m / 2^k (|m| <= M)
and inputs on an 8-bit grid, every product is an integer multiple of one grid step and every
partial sum -- in any order -- stays below 2^24 steps as long as T * A * M <= 2^24 (A: largest
input magnitude in steps).  Every partial sum is then an exact float32 number, so every kernel
(tiled, generic, split-K with its ordered reduction, warp shuffles, drop-in) must reproduce the
float64 result bit for bit: a dropped tap, a window shifted by one sample or one history sample
that should read as zero changes outputs by whole grid steps instead of by float noise.

numpy only and no GPU; only oscillator_increment asks the oracle library (for the reference's
cexpf-derived increment).
"""
import numpy as np

# input grid per format: x = n * STEP with |n| <= AMAX (cs16 restricted to multiples of 256)
STEP = {"cu8": 2.0 ** -8, "cs8": 2.0 ** -7, "cs16": 2.0 ** -7}
AMAX = {"cu8": 255, "cs8": 128, "cs16": 128}
EXACT_LIMIT = 2 ** 24


def tap_bits(T, fmt):
    """b such that taps m / 2^b with |m| <= M = 2^b - 1 keep T * AMAX * M <= 2^24 (at most 7 bits)."""
    b = 7
    while b > 1 and T * AMAX[fmt] * (2 ** b - 1) > EXACT_LIMIT:
        b -= 1
    assert T * AMAX[fmt] * (2 ** b - 1) <= EXACT_LIMIT, f"T={T} is too long for exact {fmt} stimuli"
    return b


def dyadic_taps(rng, T, fmt, k=None):
    """T nonzero taps m / 2^k, |m| <= M = 2^b - 1 with b = tap_bits(T, fmt); the first and the last at
    full magnitude M.  k defaults to b (taps in (-1, 1)); a larger k (<= 15) scales them down, which
    keeps Q15 outputs clear of saturation.  The Q15 taps are then m * 2^(15 - k), all nonzero."""
    b = tap_bits(T, fmt)
    k = b if k is None else k
    assert b <= k <= 15
    M = 2 ** b - 1
    m = rng.integers(1, M + 1, T) * rng.choice(np.array([-1, 1]), T)
    m[0] = M * (1 if rng.integers(0, 2) else -1)
    m[-1] = M * (1 if rng.integers(0, 2) else -1)
    return (m / 2.0 ** k).astype(np.float32)


def one_hot_taps(T, j, value=0.5):
    taps = np.zeros(T, dtype=np.float32)
    taps[j] = value
    return taps


def exact_input(rng, fmt, n):
    """n raw elements (interleaved I/Q) on the exact grid: cu8 (2u - 255) / 256 is never zero;
    cs8 k / 128; cs16 multiples of 256, i.e. k / 128 as well."""
    if fmt == "cu8":
        return rng.integers(0, 256, n, dtype=np.uint8)
    if fmt == "cs8":
        return rng.integers(-128, 128, n, dtype=np.int8)
    return (rng.integers(-128, 128, n) * 256).astype(np.int16)


def real_input(rng, n):
    """cs16 with every imaginary sample 0 and every real sample nonzero."""
    x = np.zeros(n, dtype=np.int16)
    re = rng.integers(1, 16384, (n + 1) // 2) * rng.choice(np.array([-1, 1]), (n + 1) // 2)
    x[0::2] = re.astype(np.int16)
    return x


def to_complex(fmt, raw):
    """The reference's sample conversion (all exact), as complex128; a trailing odd element is dropped."""
    raw = np.asarray(raw)
    n = raw.size // 2 * 2
    if fmt == "cu8":
        v = (raw[:n].astype(np.float64) - 127.5) / 128.0
    elif fmt == "cs8":
        v = raw[:n].astype(np.float64) / 128.0
    else:
        v = raw[:n].astype(np.float64) / 32768.0
    return v[0::2] + 1j * v[1::2]


def to_q15(fmt, raw):
    raw = np.asarray(raw)
    n = raw.size // 2 * 2
    if fmt == "cu8":
        v = (raw[:n].astype(np.int64) - 128) << 8
    elif fmt == "cs8":
        v = raw[:n].astype(np.int64) << 8
    else:
        v = raw[:n].astype(np.int64)
    return v[0::2], v[1::2]


def reversed_taps(taps):
    """Taps in window order: reversed, and for even T the middle pair left un-swapped (the reference's
    reversal loop runs one step too far and swaps it back)."""
    rev = np.asarray(taps)[::-1].copy()
    T = rev.size
    if T % 2 == 0:
        a, b = T // 2 - 1, T // 2
        rev[a], rev[b] = rev[b], rev[a]
    return rev


def _outputs_per_call(blocks, T, D):
    n_in = np.array([np.asarray(b).size // 2 for b in blocks], dtype=np.int64)
    cum = np.cumsum(n_in)
    # after a call the stream holds T - 1 + cum samples; window k (start k * D) is complete when
    # k * D + T <= T - 1 + cum
    done = np.where(cum >= 1, (cum - 1) // D + 1, 0)
    return np.diff(np.concatenate([[0], done])).astype(np.int64), int(done[-1]) if len(done) else 0


def ref_f64(taps, D, fmt, blocks, history=None):
    """A filter created with `taps` (centre 0) and fed `blocks` one call each, computed in float64.

    history: the T - 1 complex samples its first window reads before the first block (zeros, as
    for any new filter, when None).  Returns one complex64 array per block."""
    return ref_f64_many([taps], D, fmt, blocks, history)[0]


def ref_f64_many(taps_list, D, fmt, blocks, history=None):
    """ref_f64 for several filters of one length that consume the same blocks (one matrix product;
    every partial sum is an integer number of grid steps below 2^53, so BLAS's order is exact too)."""
    R = np.stack([reversed_taps(np.asarray(t, dtype=np.float64)) for t in taps_list], axis=1)
    T = R.shape[0]
    per_call, total_out = _outputs_per_call(blocks, T, D)
    x = np.concatenate([np.zeros(T - 1, dtype=np.complex128) if history is None else np.asarray(history),
                        *[to_complex(fmt, b) for b in blocks]])
    if total_out:
        starts = np.arange(total_out, dtype=np.int64) * D
        W = np.lib.stride_tricks.sliding_window_view(x, T)[starts]
        y = W.real @ R + 1j * (W.imag @ R)
    else:
        y = np.zeros((0, R.shape[1]), dtype=np.complex128)
    cuts = np.cumsum(per_call)[:-1]
    return [np.split(y[:, c].astype(np.complex64), cuts) for c in range(R.shape[1])]


def _sat16(v):
    return np.clip(v, -32768, 32767)


def q15_phases(n, qinc=(32767, 0)):
    """The Q15 oscillator of a new filter (phase 32767 + 0i, no renormalisation) for n outputs."""
    pr, pi = 32767, 0
    ir, ii = qinc
    out = np.empty((n, 2), dtype=np.int64)
    for k in range(n):
        out[k] = pr, pi
        nr, ni = pr * ir - pi * ii, pr * ii + pi * ir
        pr, pi = int(_sat16(nr >> 15)), int(_sat16(ni >> 15))
    return out


def ref_q15(taps, D, fmt, blocks):
    """Integer twin of ref_f64 for the Q15 path (centre 0): int64 sums, >> 15 and saturation, then
    the rotation by the decaying Q15 oscillator.  Returns one (n, 2) int16 array per block."""
    rev = reversed_taps(np.trunc(np.asarray(taps, dtype=np.float32) * np.float32(32768)).astype(np.int64))
    T = rev.size
    per_call, total_out = _outputs_per_call(blocks, T, D)
    parts = [to_q15(fmt, b) for b in blocks]
    z = np.zeros(T - 1, dtype=np.int64)
    xr = np.concatenate([z] + [p[0] for p in parts])
    xi = np.concatenate([z] + [p[1] for p in parts])
    if total_out:
        starts = np.arange(total_out, dtype=np.int64) * D
        Wr = np.lib.stride_tricks.sliding_window_view(xr, T)[starts]
        Wi = np.lib.stride_tricks.sliding_window_view(xi, T)[starts]
        ar = _sat16((Wr * rev).sum(axis=1) >> 15)
        ai = _sat16((Wi * rev).sum(axis=1) >> 15)
        ph = q15_phases(total_out)
        yr = _sat16((ar * ph[:, 0] - ai * ph[:, 1]) >> 15)
        yi = _sat16((ar * ph[:, 1] + ai * ph[:, 0]) >> 15)
        y = np.stack([yr, yi], axis=1).astype(np.int16)
    else:
        y = np.zeros((0, 2), dtype=np.int16)
    return np.split(y, np.cumsum(per_call)[:-1])


def oscillator_increment(D, center, fs):
    """incr of the oracle: the phase after exactly one output, without renormalisation.  (The filter has
    D taps: with fewer the reference's history bookkeeping underflows.)"""
    from oracle import pyoracle as po
    o = po.OracleFilter(D, np.ones(D, np.float32), center, fs, 4 * D)
    o.process_cf32("cs16", np.zeros(2, np.int16), renorm=False)
    return complex(np.complex64(o.phase))


def oracle_phases(inc, counts, renorm=True):
    """The float32 oscillator recursion of the reference (two unfused products and one add per component,
    renormalised by (float)sqrt((double)re^2 + (double)im^2) after every call that produced outputs):
    the phase of every output of calls with `counts` outputs each, as complex128."""
    f32 = np.float32
    ir, ii = f32(inc.real), f32(inc.imag)
    pr, pi = f32(1), f32(0)
    out = []
    for n in counts:
        for _ in range(int(n)):
            out.append(complex(pr, pi))
            pr, pi = f32(f32(pr * ir) - f32(pi * ii)), f32(f32(pr * ii) + f32(pi * ir))
        if n and renorm:
            mag = f32(np.sqrt(np.float64(pr) * np.float64(pr) + np.float64(pi) * np.float64(pi)))
            pr, pi = f32(pr / mag), f32(pi / mag)
    return np.array(out, dtype=np.complex128)


def _f32(v):
    return np.asarray(v, dtype=np.float32)


def _fma(a, b, c):
    # exact product of two float32 numbers in float64, one rounding to float32 (exact for the sums here:
    # one of the addends is always zero)
    return _f32(a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64))


def _cmul(a_re, a_im, b_re, b_im):
    return (_f32(_f32(a_re * b_re) - _f32(a_im * b_im)), _f32(_f32(a_re * b_im) + _f32(a_im * b_re)))


def gpu_model(rev, inc, D, blocks, renorm=True):
    """What the kernels compute: fmaf chains per accumulator, then the unfused derotation by the
    float32 oscillator recursion."""
    T = rev.size
    tr, ti = _f32(rev.real), _f32(rev.imag)
    x = np.concatenate([np.zeros(T - 1, np.complex64)] + [to_complex("cs16", b).astype(np.complex64) for b in blocks])
    n_in = np.cumsum([b.size // 2 for b in blocks])
    done = np.where(n_in >= 1, (n_in - 1) // D + 1, 0)
    total = int(done[-1])
    W = np.lib.stride_tricks.sliding_window_view(x, T)[np.arange(total) * D]
    xr, xi = _f32(W.real), _f32(W.imag)
    are = np.zeros(total, np.float32)
    aim = np.zeros(total, np.float32)
    for j in range(T):
        are = _fma(xr[:, j], np.full(total, tr[j]), are)
        are = _fma(-xi[:, j], np.full(total, ti[j]), are)
        aim = _fma(xr[:, j], np.full(total, ti[j]), aim)
        aim = _fma(xi[:, j], np.full(total, tr[j]), aim)
    ph = oracle_phases(inc, np.diff(np.concatenate([[0], done])), renorm)
    yr, yi = _cmul(are, aim, _f32(ph.real), _f32(ph.imag))
    y = (yr + 1j * yi.astype(np.complex64)).astype(np.complex64)
    out = np.split(y, np.cumsum(np.diff(np.concatenate([[0], done])))[:-1])
    return out


def assert_exact(got, ref, what="", T=None, D=None, step=None):
    """Bit-for-bit equality of per-block outputs (+0 and -0 count as equal).

    got, ref: one array per block (or one array).  On failure reports the number of mismatching
    outputs, the first block and output index, that output's window start (samples relative to the
    attach point, negative inside the zero history; needs T and D) and the difference in grid steps."""
    if not isinstance(got, (list, tuple)):
        got, ref = [got], [ref]
    assert len(got) == len(ref), f"{what}: {len(got)} blocks != {len(ref)}"
    k0, bad, first = 0, 0, None
    for b, (g, r) in enumerate(zip(got, ref)):
        g, r = np.asarray(g), np.asarray(r)
        assert g.shape == r.shape, f"{what}: block {b}: output shape {g.shape} != {r.shape}"
        neq = g != r
        if neq.ndim > 1:
            neq = neq.any(axis=tuple(range(1, neq.ndim)))
        idx = np.nonzero(neq)[0]
        if idx.size and first is None:
            i = int(idx[0])
            first = (b, i, k0 + i, g[i], r[i])
        bad += idx.size
        k0 += len(r)
    if first is None:
        return
    b, i, k, gv, rv = first
    msg = f"{what}: {bad} outputs differ; first at block {b} output {i} (stream output {k}"
    if T is not None and D is not None:
        msg += f", window start {k * D - (T - 1)}"
    msg += f"): got {gv}, want {rv}"
    if step is not None and np.iscomplexobj(rv):
        d = complex(gv) - complex(rv)
        msg += f", difference {d.real / step:+.3f}{d.imag / step:+.3f}j grid steps"
    raise AssertionError(msg)


def grid_step(taps, fmt):
    """The output grid step of exact stimuli: input step times the finest tap step."""
    t = np.abs(np.asarray(taps, dtype=np.float64))
    # every tap is m / 2^k: the step is 2^-k for the smallest k that makes all of them integers
    k = 0
    while k < 40 and np.any(np.mod(t * 2.0 ** k, 1.0) != 0):
        k += 1
    return STEP[fmt] * 2.0 ** -k
