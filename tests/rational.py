"""Rational (L/M) clients as the reference defines them: the integer filter with decimation M at
L * fs, fed the zero-stuffed stream u[L*n] = x[n], u[m] = 0 otherwise.

Every cu8 or cs8 block maps exactly onto cs16 ((2u - 255) * 128 and v * 256), so one stuffed cs16
stream feeds the strict oracle and the float64 reference of tests/exact.py for all three formats.
"""
import numpy as np

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
