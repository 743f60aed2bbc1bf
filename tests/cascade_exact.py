"""Exact references of the cascade stage-B tests (xlg_add_client_cascade[_rational], cascade filters).  No GPU.

* mirrors of the host half of stage B (sdr-server_b200/csrc/cascade_stage_b.cuh): cascade_smem, cascade_ko,
  cascade_poly_smem, cascade_poly_ko, the stage-B rule of cascade_refusal and stage_b_walk;
* stage_b_model: what cascade_fir_cf32_kernel (L2 = 1) and cascade_fir_poly_cf32_kernel (L2 > 1) compute for
  one client, summation order included.  Both kernels give each output's accumulators one fmaf chain over its
  taps, but with even D2 (M2) a lane starts its walk at tap lane mod T (T = T2, or Tb2 = ceil(T2 / L2)), and
  which lane computes an output depends on the outputs per CTA, ko.  So on taps that are not exact the bits of
  a client depend on its ko: two engines agree bit for bit only where they launch it at the same ko.  A
  `mutation` argument models a plausible kernel bug (MUTATIONS).
"""
import numpy as np

from cascade import filter_constants
from exact import reversed_taps
from rational import poly_pack_np
from subband_exact import fmaf

C_THREADS = 128
C_KO = 256
TILE_MAX_SMEM = 200 * 1024  # kTileMaxSmem
SLOTS = 4                   # XLG_SLOTS


def cascade_smem(ko, D2, T2):
    return 16 + ((T2 + 3) & ~3) * 4 + (((ko - 1) * D2 + T2 + 2) & ~1) * 8


def cascade_poly_smem(ko, L2, M2, Tb2):
    return 16 + ((L2 * Tb2 + 3) & ~3) * 4 + ((((ko - 1) * M2 + L2 - 1) // L2 + Tb2 + 2) & ~1) * 8


def cascade_ko(D2, T2):
    ko = C_KO
    while ko > 1 and cascade_smem(ko, D2, T2) > TILE_MAX_SMEM:
        ko //= 2
    return ko


def cascade_poly_ko(L2, M2, Tb2):
    ko = 2 * L2 * (C_THREADS // L2) if L2 <= C_THREADS else C_KO
    while ko > 1 and cascade_poly_smem(ko, L2, M2, Tb2) > TILE_MAX_SMEM:
        ko //= 2
    return ko


def stage_b_ko(L2, M2, T2):
    """The outputs per CTA a client is attached with (stage_b_init)."""
    return cascade_ko(M2, T2) if L2 == 1 else cascade_poly_ko(L2, M2, -(-T2 // L2))


def stage_b_refused(L2, M2, T2):
    """cascade_refusal's shared-memory rule: stage B's taps and one output's window exceed TILE_MAX_SMEM."""
    smem = cascade_smem(1, M2, T2) if L2 == 1 else cascade_poly_smem(1, L2, M2, -(-T2 // L2))
    return smem > TILE_MAX_SMEM


# (D2, T2) with odd and with even D2 for every integer stage-B CTA size, D2 just past where C_KO halves that
# often (T2 = 16000 for ko = 1: at T2 = 33 a window of two outputs would need D2 > 25000)
INT_KO_CASES = {256: ((7, 85), (2, 85)), 128: ((101, 33), (102, 33)), 64: ((203, 33), (204, 33)),
                32: ((407, 33), (408, 33)), 16: ((827, 33), (826, 33)), 8: ((1705, 33), (1706, 33)),
                4: ((3651, 33), (3652, 33)), 2: ((8517, 33), (8518, 33)), 1: ((1599, 16000), (1600, 16000))}

# (L2, M2, T2) of rational stage B: ko whole per branch (L2 <= 128: 256, 252, 240, 254, 256), C_KO where
# L2 > 128, halved to a whole number per branch (2, 255) and to one that is not (3, 2000: 31); Tb2 = 1;
# T2 % L2 != 0 wherever Tb2 > 1
RAT_CASES = [(2, 7, 85), (2, 255, 301), (3, 16, 193), (3, 2000, 40), (12, 125, 121), (127, 125, 500),
             (128, 125, 500), (129, 127, 500), (441, 640, 1000), (12, 5, 12), (441, 640, 441)]


def max_t2(L2, M2):
    """The longest stage B the shared memory admits (cascade_refusal): one more tap is refused (for L2 > 1 one
    more tap past a whole number per branch)."""
    T2 = 1
    step = 1 << 20
    while step:
        if not stage_b_refused(L2, M2, T2 + step):
            T2 += step
        step >>= 1
    return T2


def stage_b_walk(n1s, L2, M2, T2):
    """stage_b_walk from the attach point over blocks of n1s stage-A samples: (first, n2) per block, first in
    upsampled stage-A positions (the ring's position 0 is the attach point; earlier positions read zero)."""
    hist, pos, out = T2 - 1, 0, []
    for n1 in n1s:
        avail = hist + L2 * n1 - T2
        n2 = avail // M2 + 1 if avail >= 0 else 0
        out.append((L2 * pos - hist, n2))
        hist += L2 * n1 - n2 * M2
        pos += n1
    return out


def stage_b_taps(taps2, L2, M2, rate1):
    """The real parts of the library's reversed taps at L2 * rate1 (the even-length quirk included),
    branch-major (L2, Tb2): what stage_b_init uploads."""
    rev, _ = filter_constants(taps2, M2, 0, min(L2 * max(rate1, 1), 2 ** 32 - 1))
    return poly_pack_np(rev.real.astype(np.float32), L2)


def ring_cap(T2, L2, out_cap):
    """A group client's stage-A ring: next_pow2(history_reach + (XLG_SLOTS + 1) * out_cap)."""
    reach = T2 - 1 if L2 == 1 else (T2 - 1 + L2 - 1) // L2 + 1
    return 1 << int(reach + (SLOTS + 1) * out_cap - 1).bit_length()


def f64_stage_b(rows, attach, L2, M2, taps2):
    """Stage B in float64 from the attach point (the float64 composition's stage B, tests/cascade_rational.py),
    summed per branch without building the zero-stuffed stream and a block at a time, so that windows of
    tens of thousands of taps stay small: one complex128 array per block from `attach` on."""
    P = poly_pack_np(reversed_taps(np.asarray(taps2, np.float64)), L2)
    T = P.shape[1]
    new = [np.asarray(r, np.complex128) for r in rows[attach:]]
    x = np.concatenate([np.zeros(0, np.complex128)] + new)
    out = []
    for first, n2 in stage_b_walk([r.size for r in new], L2, M2, len(taps2)):
        w = first + np.arange(n2, dtype=np.int64) * M2
        r = (-w) % L2
        n0 = (w + r) // L2
        y = np.zeros(n2, np.complex128)
        for c in range(0, n2, max(1, 2 ** 22 // max(T, 1))):
            idx = n0[c:c + 2 ** 22 // max(T, 1), None] + np.arange(T)[None, :]
            ok = (idx >= 0) & (idx < x.size)
            xv = np.where(ok, x[np.clip(idx, 0, max(x.size - 1, 0))] if x.size else 0, 0)
            y[c:c + idx.shape[0]] = (xv * P[r[c:c + idx.shape[0]]]).sum(axis=1)
        out.append(y)
    return out


def ring_windows(walk, L2, M2, T2, ko, cap):
    """The stage-B windows the kernels stage from a ring of cap samples over a client's walk: (the parities of
    the windows' first ring index, how many windows cross the ring's end)."""
    Tb = -(-T2 // L2)
    parities, wraps = set(), 0
    for first, n2 in walk:
        for k0 in range(0, n2, ko):
            nk = min(ko, n2 - k0)
            lo = first + k0 * M2
            hi = first + (k0 + nk - 1) * M2
            if L2 > 1:
                lo, hi = (lo + (-lo) % L2) // L2, (hi + (-hi) % L2) // L2
            idx = lo & (cap - 1)
            shift = idx & 1
            need = ((hi - lo + (T2 if L2 == 1 else Tb)) + shift + 1) & ~1
            parities.add(shift)
            wraps += (idx - shift) + need > cap
    return parities, wraps


MUTATIONS = ("newest_dropped", "oldest_dropped", "lane_tid_15", "skew_odd", "branch_w_mod_L2", "Tb_floor")
ORDER_MUTATIONS = ("lane_tid_15", "skew_odd")  # change the summation order only: invisible on exact stimuli


def stage_b_lanes(n2, L2, ko, mutation=None):
    """The lane (tid & 31) that computes each of a block's n2 outputs.  Integer kernel: CTA x computes outputs
    k0 = x*ko ... and thread tid the relative outputs tid and tid + C_THREADS.  Rational kernel: relative output
    ka = rho + p*L2 and kb = ka + P*L2 (P = ceil(ceil(nk / L2) / 2)) belong to pair slot ps = rho*P + p, taken
    by thread ps mod C_THREADS."""
    k = np.arange(n2, dtype=np.int64)
    k0 = k // ko * ko
    loc = k - k0
    if L2 == 1:
        tid = loc % C_THREADS
    else:
        nk = np.minimum(ko, n2 - k0)
        P = (-(-nk // L2) + 1) // 2
        rho, q = loc % L2, loc // L2
        tid = (rho * P + np.where(q < P, q, q - P)) % C_THREADS
    return tid & (15 if mutation == "lane_tid_15" else 31)


def stage_b_model(rows, attach, L2, M2, taps2, rate1, ko, mutation=None):
    """A cascade client's stage B as its kernel computes it: one complex64 array per block from `attach` on.

    rows: the client's stage-A outputs, one complex64 array per block since the group was created (stage B
    reads zeros before the block `attach`); taps2, rate1: its stage-B taps and stage-A rate; ko: the outputs per
    CTA it is launched with.  Output k of a block (block-local) has the upsampled window w = first + k*M2,
    branch r = (-w) mod L2 and first stage-A sample n0 = (w + r) / L2 (r = 0, n0 = w for L2 = 1); its lane
    (stage_b_lanes) walks tap t = (lane mod T + s) mod T for s < T with even M2, t = s with odd M2, and .x and
    .y are separate fmaf chains of y[n0 + t] * P[r][t].

    mutation (MUTATIONS): newest_dropped / oldest_dropped skip the tap of the newest / oldest window sample
    (t = T - 1 / t = 0); lane_tid_15 takes the lane from tid & 15; skew_odd skews the walk for odd M2 too;
    branch_w_mod_L2 reads branch w mod L2; Tb_floor walks floor(T2 / L2) taps per branch."""
    P = stage_b_taps(taps2, L2, M2, rate1)
    T2 = len(taps2)
    if mutation == "Tb_floor" and L2 > 1:
        P = P[:, :T2 // L2]
    T = P.shape[1]
    new = [np.asarray(r, np.complex64) for r in rows[attach:]]
    x = np.concatenate([np.zeros(0, np.complex64)] + new)
    walk = stage_b_walk([r.size for r in new], L2, M2, T2)
    counts = [n2 for _, n2 in walk]
    w = np.concatenate([np.zeros(0, np.int64)] + [f + np.arange(n2, dtype=np.int64) * M2 for f, n2 in walk])
    lane = np.concatenate([np.zeros(0, np.int64)] + [stage_b_lanes(n2, L2, ko, mutation) for n2 in counts])
    r = (-w) % L2
    n0 = (w + r) // L2
    rb = w % L2 if mutation == "branch_w_mod_L2" else r
    skew = M2 % 2 == 0 or mutation == "skew_odd"
    t0 = lane % max(T, 1) if skew else np.zeros_like(lane)
    xr, xi = x.real.astype(np.float32), x.imag.astype(np.float32)
    are = np.zeros(w.size, np.float32)
    aim = np.zeros(w.size, np.float32)
    for s in range(T):
        t = (t0 + s) % T
        pos = n0 + t
        ok = (pos >= 0) & (pos < x.size)
        if mutation == "newest_dropped":
            ok &= t != T - 1
        elif mutation == "oldest_dropped":
            ok &= t != 0
        p = np.clip(pos, 0, max(x.size - 1, 0))
        vr = np.where(ok, xr[p] if x.size else 0, 0).astype(np.float32)
        vi = np.where(ok, xi[p] if x.size else 0, 0).astype(np.float32)
        h = P[rb, t]
        are = fmaf(vr, h, are)
        aim = fmaf(vi, h, aim)
    y = (are + 1j * aim.astype(np.complex64)).astype(np.complex64)
    return np.split(y, np.cumsum(counts)[:-1]) if counts else []
