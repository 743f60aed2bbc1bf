"""Rational (L/M) clients as the reference defines them: the integer filter with decimation M at
L * fs, fed the zero-stuffed stream u[L*n] = x[n], u[m] = 0 otherwise.

Every cu8 or cs8 block maps exactly onto cs16 ((2u - 255) * 128 and v * 256), so one stuffed cs16
stream feeds the strict oracle and the float64 reference of tests/exact.py for all three formats.
"""
import numpy as np

from exact import _cmul, _f32, _fma, oracle_phases, reversed_taps, to_complex

# rows of the rate table: (band fs, format, client rate) -> L / M
ROWS = [(2048000, "cu8", 48000), (3000000, "cs16", 48000), (10000000, "cs16", 48000), (20000000, "cs8", 48000)]


def as_cs16(fmt, raw):
    raw = np.asarray(raw)
    if fmt == "cu8":
        return ((raw.astype(np.int32) * 2 - 255) * 128).astype(np.int16)
    if fmt == "cs8":
        return (raw.astype(np.int32) * 256).astype(np.int16)
    return raw.astype(np.int16)


def stuff(fmt, raw, L):
    """One block as the zero-stuffed cs16 block the reference filter at L * fs is fed."""
    v = as_cs16(fmt, raw)
    n = v.size // 2
    u = np.zeros(2 * L * n, dtype=np.int16)
    u[0::2 * L] = v[0:2 * n:2]
    u[1::2 * L] = v[1:2 * n:2]
    return u


def oracle_filter(po, L, M, taps, center, fs, max_in):
    return po.OracleFilter(M, taps, center, L * fs, L * max_in)


def oracle_run(o, fmt, blocks, L):
    return [o.process_cf32("cs16", stuff(fmt, x, L)) for x in blocks]


def poly_pack_np(rev, L):
    """Numpy restatement of the branch-major polyphase packer: P[r][t] = rev[r + t*L], zero past T."""
    rev = np.asarray(rev)
    Tb = -(-rev.size // L)
    P = np.zeros((L, Tb), dtype=rev.dtype)
    for r in range(L):
        branch = rev[r::L]
        P[r, :branch.size] = branch
    return P


def output_counts(n_in, L, M):
    """Outputs per call of a rational client fed calls of n_in input samples each (the integer filter's
    count on the upsampled lengths L * n): window k is complete once k * M < L * (samples so far)."""
    up = np.cumsum(np.asarray(n_in, dtype=np.int64)) * L
    done = np.where(up >= 1, (up - 1) // M + 1, 0)
    return np.diff(np.concatenate([[0], done])).astype(np.int64)


def poly_windows(k, T, L, M):
    """Output k's window start w = k*M - (T-1) (upsampled samples from the attach point), its branch
    r = (-w) mod L (the first tap that lands on a real sample) and n0 = (w + r) / L, the input sample
    that tap reads.  Tap t of branch r then reads input sample n0 + t."""
    w = np.asarray(k, dtype=np.int64) * M - (T - 1)
    r = (-w) % L
    return w, r, (w + r) // L


class RationalRef:
    """The float64 sum of a rational client at centre 0, one call at a time, computed on the input-rate
    stream without building the L-times-longer stuffed one: y[k] = sum_t x[n0 + t] * P[r][t] with
    poly_windows' r and n0 and P = poly_pack_np(reversed_taps(taps), L).

    history: input-rate complex samples before the attach point (newest last); older samples read as
    zero.  Equal to ref_f64 on the stuffed stream bit for bit on exact stimuli (tests/exact.py)."""

    def __init__(self, taps, L, M, history=None):
        self.P = poly_pack_np(reversed_taps(np.asarray(taps, dtype=np.float64)), L)
        self.T, self.L, self.M, self.Tb = len(taps), L, M, self.P.shape[1]
        self.tail = np.zeros(0, np.complex128) if history is None else np.asarray(history, np.complex128)
        self.lo = -self.tail.size  # input index of the oldest sample ever held
        self.n = self.k = 0        # input samples consumed, outputs produced

    def feed(self, fmt, block):
        x = to_complex(fmt, block)
        buf = np.concatenate([self.tail, x])
        self.n += x.size
        x0 = self.n - buf.size  # input index of buf[0]
        done = (self.n * self.L - 1) // self.M + 1 if self.n else 0
        _, r, n0 = poly_windows(np.arange(self.k, done), self.T, self.L, self.M)
        self.k = done
        idx = n0[:, None] + np.arange(self.Tb)[None, :]
        assert not np.any((idx < x0) & (idx >= self.lo)), "the tail kept too few samples"
        ok = (idx >= x0) & (idx < x0 + buf.size)
        xv = np.where(ok, buf[np.clip(idx - x0, 0, max(buf.size - 1, 0))] if buf.size else 0, 0)
        y = (xv * self.P[r]).sum(axis=1)
        self.tail = buf[-(self.Tb + 1):]
        return y.astype(np.complex64)


def ref_rational_f64(taps, L, M, fmt, blocks, history=None):
    """ref_f64 of tests/exact.py for a rational client (centre 0): one complex64 array per call."""
    ref = RationalRef(taps, L, M, history)
    return [ref.feed(fmt, b) for b in blocks]


def branch_one_hot_taps(rng, T, L):
    """T taps whose reversed, branch-packed form (poly_pack_np(reversed_taps(taps), L)) holds exactly
    one nonzero per branch (none in the branches past T), at a random position and with a value that
    differs from branch to branch and between calls.

    Fed a real input (every imaginary sample 0) every accumulator of every output is then one rounded
    product, whatever the centre and its rotated taps: the kernels' FMA chains and the strict oracle's
    unfused sum over the stuffed stream agree bit for bit, so the oscillator, the branch and the window
    of every output are checked exactly.  A plain one-hot filter would leave all but 1/L of the outputs 0."""
    assert L <= 512
    scale = float(rng.choice([0.75, 1.0, 0.625]))
    rev = np.zeros(T, np.float32)
    for r in range(min(L, T)):
        t = int(rng.integers(0, len(range(r, T, L))))
        rev[r + t * L] = scale * (512 + r) / 1024 * rng.choice([-1, 1])  # |value| differs per branch
    taps = reversed_taps(rev)  # the reversal (with its even-T middle swap) is its own inverse
    assert np.array_equal(reversed_taps(taps), rev)
    return taps


def real_grid_input(rng, n):
    """n raw cs16 elements, real part k * 256 with k in [-128, 127], imaginary part 0: on the exact grid
    of dyadic clients at centre 0 and a real input for branch_one_hot_taps clients at any centre."""
    x = np.zeros(n, dtype=np.int16)
    x[0::2] = (rng.integers(-128, 128, (n + 1) // 2) * 256).astype(np.int16)
    return x


MUTATIONS = ("branch_w_mod_L", "n0_negative_w", "Tb_floor", "odd_phase_no_step")


def poly_model(rev, L, M, inc, blocks, renorm=True, mutation=None):
    """What the polyphase kernels compute for a new client fed cs16 `blocks`: an fmaf chain per
    accumulator over branch r's taps P[r] = poly_pack_np(rev, L) (rev: the rotated, reversed taps),
    then the unfused rotation by the float32 oscillator recursion, odd outputs one step past the stored
    even phase.  `mutation` (one of MUTATIONS) models a plausible kernel bug."""
    T = rev.size
    P = poly_pack_np(np.asarray(rev, np.complex64), L)
    if mutation == "Tb_floor":
        P = P[:, :T // L]  # drops the last tap row when T % L != 0
    Tb = P.shape[1]
    counts = output_counts([np.asarray(b).size // 2 for b in blocks], L, M)
    total = int(counts.sum())
    x = np.concatenate([np.zeros(0, np.complex64)] + [to_complex("cs16", b).astype(np.complex64) for b in blocks])
    w, r, n0 = poly_windows(np.arange(total), T, L, M)
    if mutation == "n0_negative_w":
        n0 = n0 + ((w < 0) & (r != 0))  # ceil by truncating division, wrong below zero
    rb = w % L if mutation == "branch_w_mod_L" else r
    are = np.zeros(total, np.float32)
    aim = np.zeros(total, np.float32)
    for t in range(Tb):
        idx = n0 + t
        ok = (idx >= 0) & (idx < x.size)
        xv = np.where(ok, x[np.clip(idx, 0, max(x.size - 1, 0))] if x.size else 0, 0).astype(np.complex64)
        xr, xi = _f32(xv.real), _f32(xv.imag)
        tr, ti = _f32(P[rb, t].real), _f32(P[rb, t].imag)
        are = _fma(xr, tr, are)
        are = _fma(-xi, ti, are)
        aim = _fma(xr, ti, aim)
        aim = _fma(xi, tr, aim)
    ph = oracle_phases(inc, counts, renorm).astype(np.complex64)
    if mutation == "odd_phase_no_step":
        local = np.arange(total) - np.repeat(np.cumsum(counts) - counts, counts)
        odd = np.nonzero(local % 2 == 1)[0]
        ph[odd] = ph[odd - 1]
    yr, yi = _cmul(are, aim, _f32(ph.real), _f32(ph.imag))
    return np.split((yr + 1j * yi.astype(np.complex64)).astype(np.complex64), np.cumsum(counts)[:-1])
