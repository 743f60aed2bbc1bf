"""References of the bank tests (xlg_add_bank, xlg_add_bank_subband).  No GPU.

* bank_walk: the outputs per block of a bank (an integer client (D1, T1) attached at P).
* f64_bank: the definition in float64: channel k's output m is
      sum_{j < T1} x[s_m + j] * h[T1-1-j] * e^{-2 pi i k (s_m + j - P) / K},   K = 2 * D1,
  x zero before P.
* bank_model: what bank_cf32_kernel computes, in its fmaf order (DESIGN.md section 5, "Bank sub-bands"), with
  a `mutation` argument that models a plausible kernel bug (MUTATIONS).
* twiddles: the library's table W[j] = e^{-2 pi i j / K}, built by quarter turns in double and rounded once.
* bank_member_model: bank_model's rows of a channel fed to subband_exact.member_model, bit for bit what a
  member of a bank channel computes on any taps and input.
* ring_cap, bank_ctas: the group's input ring capacity and, per block and bank CTA, its window, parity, wrap
  split and zeroing before P (the edges the GPU tests assert they reached).
"""
import math

import numpy as np

from subband_exact import fmaf

F = np.float32
MUTATIONS = ("twiddle_plus_1", "r0_negated", "zero_point_minus_1", "taps_not_reversed")
XLG_SLOTS = 4  # tickets in flight (include/xlating_group.h)
BK_F = 32      # frames per bank CTA (xlating_kernels.cuh)
BK_CG = 32     # channels per bank CTA


def bank_tpad(K, T1):
    return ((-(-T1 // K) * K) + 3) & ~3


def twiddles(K):
    """W[j] as xlg_add_bank builds it: 4j = qK + rem, t = 2 pi rem / 4K, (-i)^q (cos t, -sin t)."""
    w = np.zeros(K, np.complex64)
    for j in range(K):
        q, rem = divmod(4 * j, K)
        t = 2.0 * math.pi * rem / (4.0 * K)
        c, s = F(math.cos(t)), F(math.sin(t))
        re, im = [(c, -s), (-s, -c), (-c, s), (s, c)][q]
        w.view(np.float32)[2 * j] = F(re)
        w.view(np.float32)[2 * j + 1] = F(im)
    return w


def bank_walk(sizes, T1, D1):
    """Outputs per block of a bank attached before the first of these blocks (sizes in complex samples), and
    the window start of each block's first output relative to P."""
    hist = T1 - 1
    pos = 0
    counts, firsts = [], []
    for n in sizes:
        firsts.append(pos - hist)
        avail = hist + n - T1
        n1 = avail // D1 + 1 if avail >= 0 else 0
        hist += n - n1 * D1
        pos += n
        counts.append(n1)
    return counts, firsts


def _windows(x, P, T1, D1, total):
    """Window start s_m (absolute) of the bank's outputs 0..total-1 and the windows of x zeroed before P."""
    s = P - (T1 - 1) + D1 * np.arange(total, dtype=np.int64)
    pos = s[:, None] + np.arange(T1)[None, :]
    ok = (pos >= P) & (pos < x.size)
    return s, pos, ok


def f64_bank(taps, D1, channels, x, P, sizes):
    """float64 rows of `channels` of a bank attached at stream position P of the complex stream x, whose blocks
    from P on have `sizes` samples.  Returns {k: [complex128 array per block]}."""
    T1 = len(taps)
    K = 2 * D1
    counts, _ = bank_walk(sizes, T1, D1)
    total = int(sum(counts))
    s, pos, ok = _windows(x, P, T1, D1, total)
    X = np.where(ok, np.asarray(x, complex)[np.clip(pos, 0, max(x.size - 1, 0))] if x.size else 0, 0)
    h = np.asarray(taps, np.float64)[::-1]
    out = {}
    for k in channels:
        t = (k * (pos - P)) % K
        rot = np.exp(-2j * np.pi * t / K)
        q = (4 * t) % K == 0
        rot[q] = np.array([1, -1j, -1, 1j])[(4 * t[q]) // K]  # quarter turns exactly
        y = np.sum(X * h[None, :] * rot, axis=1) if total else np.zeros(0, complex)
        out[k] = np.split(y, np.cumsum(counts)[:-1])
    return out


def bank_model(taps, D1, channels, x, P, sizes, mutation=None):
    """bank_cf32_kernel's rows of `channels` (arguments as f64_bank; x complex64, the converted ring).

    Frame m (window s_m, r_m = (s_m - P) mod K): phase 1 sums v[p] = fmaf chains (re, im) over q ascending of
    x[s_m + p + qK] * hr[p + qK], hr[j] = h[T1-1-j], for p < min(K, T1); phase 2 sums y_k = the 4-fmaf complex
    chain over p ascending of v[p] * W[(k mod K) * (p + r_m) mod K].  Both start from +0.  Each step of a
    chain is one fmaf over every (frame, p) or (channel, frame) at once, so wide banks stay affordable.

    mutation (MUTATIONS): twiddle_plus_1 reads W one index further; r0_negated takes r_m = (P - s_m) mod K;
    zero_point_minus_1 reads the sample just before P; taps_not_reversed multiplies x[s_m + j] by h[j]."""
    T1 = len(taps)
    K = 2 * D1
    counts, _ = bank_walk(sizes, T1, D1)
    total = int(sum(counts))
    x = np.asarray(x, np.complex64)
    s, pos, ok = _windows(x, P, T1, D1, total)
    if mutation == "zero_point_minus_1":
        ok = (pos >= P - 1) & (pos >= 0) & (pos < x.size)
    X = np.where(ok, x[np.clip(pos, 0, max(x.size - 1, 0))] if x.size else 0, 0).astype(np.complex64)
    h = np.asarray(taps, F)
    hr = h if mutation == "taps_not_reversed" else h[::-1].copy()
    KP = min(K, T1)
    vre = np.zeros((total, KP), F)
    vim = np.zeros((total, KP), F)
    xr, xi = X.real.astype(F), X.imag.astype(F)
    for q in range(-(-T1 // K)):  # tap p + qK of every phase p that has one
        j = q * K + np.arange(min(KP, T1 - q * K))
        p = j - q * K
        vre[:, p] = fmaf(xr[:, j], hr[j], vre[:, p])
        vim[:, p] = fmaf(xi[:, j], hr[j], vim[:, p])
    W = twiddles(K)
    wre, wim = W.real.astype(F), W.imag.astype(F)
    r = (s - P) % K if mutation != "r0_negated" else (P - s) % K
    chans = list(channels)
    kk = np.array([k % K for k in chans], np.int64)[:, None]
    are = np.zeros((len(chans), total), F)
    aim = np.zeros((len(chans), total), F)
    for p in range(KP):
        t = (kk * (p + r)[None, :]) % K
        if mutation == "twiddle_plus_1":
            t = (t + 1) % K
        a, b, c, d = vre[None, :, p], vim[None, :, p], wre[t], wim[t]
        are = fmaf(a, c, are)
        are = fmaf(-b, d, are)
        aim = fmaf(a, d, aim)
        aim = fmaf(b, c, aim)
    out = {}
    for i, k in enumerate(chans):
        y = np.empty(total, np.complex64)
        y.real, y.imag = are[i], aim[i]
        out[k] = np.split(y, np.cumsum(counts)[:-1])
    return out


def bank_member_model(taps1, D1, k, x, P, sizes, members, fs, mat=0, attach=0, renorm=True, mutation=None):
    """Members of channel k of a bank, as the bank kernel and the member kernels compute them: bank_model's
    rows of the channel fed to member_model.

    The bank (taps1, D1) is attached at stream position P of x; sizes are its blocks from P on.  The channel
    was materialised before block `mat` of them (its ring reads zero before that block) and the members
    (l2, d2, taps2, offset) before block `attach` of the channel's blocks.  Members of one shape form one class,
    in the given order.  Returns per member one complex64 array per block from the attach on.

    mutation: an entry of MUTATIONS (the bank) or of subband_exact.MUTATIONS (the members)."""
    from subband_exact import MUTATIONS as SB_MUTATIONS, member_consts, member_model
    assert mutation is None or mutation in MUTATIONS or mutation in SB_MUTATIONS, mutation
    rows = bank_model(taps1, D1, [k], x, P, sizes, mutation=mutation if mutation in MUTATIONS else None)[k][mat:]
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


def next_pow2(n):
    return 1 << max(0, int(n - 1).bit_length())


def ring_cap(max_in, hist):
    """The group's input ring capacity (ensure_ring): XLG_SLOTS + 1 blocks of max_in / 2 samples, the largest
    history the group has needed (at least 4096) and 64 samples of slack, to a power of two."""
    return next_pow2((XLG_SLOTS + 1) * (max_in // 2) + max(hist, 4096) + 64)


def bank_ctas(sizes, T1, D1, P, cap):
    """Per block of a bank attached at stream position P (sizes: its blocks from P on) and per CTA x of its
    frames (BK_F each), what walk_banks and the kernel prologue compute: (w0, shift, need, split, pre_p) --
    the window start, its parity in the ring, the samples staged, whether the staging is two bulk copies
    (the window straddles the ring's wrap) and whether the CTA zeroes samples before P."""
    counts, firsts = bank_walk(sizes, T1, D1)
    out = []
    for n1, first in zip(counts, firsts):
        ctas = []
        for f0 in range(0, n1, BK_F):
            nf = min(BK_F, n1 - f0)
            w0 = P + first + f0 * D1
            idx = w0 & (cap - 1)
            shift = idx & 1
            need = ((nf - 1) * D1 + T1 + shift + 1) & ~1
            p1 = min(need, cap - (idx - shift))
            ctas.append((w0, shift, need, p1 < need, w0 - shift < P))
        out.append(ctas)
    return out


class BankMemberOracle:
    """A member (d2, taps2, offset, interp2) of channel k of a bank (d1, taps1) attached before the first
    block, fed block by block: the channel's rows by f64_bank's definition, then the reference's float path at
    interp2 * fs / d1 fed them zero-stuffed (RationalSubbandOracle's member).  Keeps only T1 - 1 samples of
    the stream, so it follows long runs."""

    def __init__(self, d1, taps1, k, d2, taps2, offset, interp2, fs):
        from cascade import FloatPath
        self.d1, self.K, self.k, self.l2 = d1, 2 * d1, k, interp2
        self.h = np.asarray(taps1, np.float64)[::-1]
        self.T1 = self.h.size
        self.tail = np.zeros(self.T1 - 1, complex)
        self.S = 0               # stream position of the next block
        self.hist = self.T1 - 1
        self.path = FloatPath(d2, taps2, offset, interp2 * fs // d1)

    def process_cf32(self, fmt, raw):
        from cascade_rational import stuff
        from exact import to_complex
        x = to_complex(fmt, raw)
        buf = np.concatenate([self.tail, x])  # buf[0] is stream position S - (T1 - 1)
        first = self.S - self.hist
        avail = self.hist + x.size - self.T1
        n1 = avail // self.d1 + 1 if avail >= 0 else 0
        self.hist += x.size - n1 * self.d1
        m = np.arange(n1, dtype=np.int64)[:, None] * self.d1 + np.arange(self.T1)[None, :]
        t = (self.k * (first + m)) % self.K
        y = np.sum(buf[first - (self.S - (self.T1 - 1)) + m] * self.h[None, :] * np.exp(-2j * np.pi * t / self.K),
                   axis=1) if n1 else np.zeros(0, complex)
        self.S += x.size
        self.tail = buf[buf.size - (self.T1 - 1):] if self.T1 > 1 else self.tail
        y = y.astype(np.complex64)
        return self.path.process_cf32(stuff(y, self.l2) if self.l2 > 1 else y)
