"""Exact references of the sub-band tests (xlg_add_subband, xlg_add_client_subband[_rational]).  No GPU.

* f64_rows / f64_member: a sub-band and its members in float64 at centre 0 (tests/cascade.py's f64_filter,
  members fed the zero-stuffed rows as tests/cascade_rational.py's f64_composition feeds stage B).  On dyadic
  taps and the exact input grid every partial sum of both stages is a whole number of grid steps; exact_bound
  checks that those numbers stay below 2^24, so every float32 summation order -- the strict oracle's, the
  kernels' -- reproduces the float64 result bit for bit, and full-length member filters are summed exactly.
* member_model: what subband_fir_cf32_kernel and subband_fir_poly_cf32_kernel compute for one class of
  members, with a `mutation` argument that models a plausible kernel bug (MUTATIONS).
"""
import numpy as np

from cascade import f64_filter, filter_constants
from cascade_rational import stuff
from exact import AMAX, EXACT_LIMIT, _cmul, _f32, oracle_phases, to_complex
from rational import output_counts, poly_pack_np, poly_windows

SB_MG = 16   # members per CTA group (xlating_kernels.cuh)
SB_KO = 64   # outputs per CTA tile
PH_GROUP = 32  # members per oscillator table group (subband_phase_kernel's warp)
F = np.float32


def sb_tpad(T2):
    return (T2 + 1) & ~1


def tap_units(taps):
    """sum |m| of taps m / 2^k (k the smallest exponent that makes every tap an integer)."""
    t = np.abs(np.asarray(taps, dtype=np.float64))
    k = 0
    while k < 40 and np.any(np.mod(t * 2.0 ** k, 1.0) != 0):
        k += 1
    assert k < 40, "taps are not dyadic"
    return float(np.sum(t * 2.0 ** k))


def exact_bound(taps1, taps2, fmt):
    """(sum |m1|) * A * (sum |m2|) <= 2^24: every partial sum of the stage-A row and of the member's sums
    is a whole number of grid steps below 2^24 (A: the largest input magnitude in steps; real_grid_input
    is cs16 on the same grid)."""
    return tap_units(taps1) * AMAX[fmt] * tap_units(taps2) <= EXACT_LIMIT


def f64_rows(d1, taps1, fs, fmt, raw_blocks):
    """The sub-band (centre 0) in float64, created before raw_blocks[0]: one complex128 row per block."""
    return f64_filter(taps1, d1, 0, fs, [to_complex(fmt, x) for x in raw_blocks])


def f64_member(rows, l2, d2, taps2, fs1):
    """A member at offset 0 attached before the block of rows[0], in float64: the filter (d2, taps2) at
    l2 * fs1 fed the rows zero-stuffed by l2.  One complex64 array per block."""
    return [y.astype(np.complex64) for y in f64_filter(taps2, d2, 0, l2 * fs1, [stuff(y, l2) for y in rows])]


def member_consts(taps2, d2, offset, l2, fs1):
    """Rotated reversed taps (complex64, natural length) and oscillator step of a member, from the library's
    host constants at l2 * fs1 (what xlg_add_client_subband_rational builds)."""
    rev, (ir, ii) = filter_constants(taps2, d2, offset, l2 * fs1)
    return rev, complex(ir, ii)


def fmaf(a, b, c):
    """float32 fmaf, correctly rounded: the product is exact in float64, the sum is rounded to odd in float64
    (53 >= 24 + 2 bits) and then to nearest in float32."""
    a64, b64, c64 = (np.asarray(v, np.float32).astype(np.float64) for v in (a, b, c))
    p = a64 * b64
    s = p + c64
    bb = s - p
    e = (p - (s - bb)) + (c64 - bb)
    odd = (s.view(np.int64) & 1) == 1
    s = np.where((e != 0) & ~odd, np.nextafter(s, np.where(e > 0, np.inf, -np.inf)), s)
    return s.astype(np.float32)


MUTATIONS = ("newest_dropped", "zb_minus_1", "odd_no_step", "tap_stride_T2", "branch_w_mod_L2",
             "phase_row_plus_32")


def member_model(rows, attach, l2, d2, revs, incs, renorm=True, mutation=None):
    """One class of members as the member kernels compute it.

    rows: the sub-band's complex64 rows, one per block since it was created (its ring); attach: the block the
    class was attached before (zb = the samples of the rows before it); revs, incs: the members' rotated
    reversed taps (member_consts) and oscillator steps, in class order (groups of SB_MG consecutive members
    share a tap table of rows sb_tpad(Tb) apart, Tb = ceil(T2 / l2)).

    Output k of a block (block-local) has the upsampled window w = first + k*d2, branch r = (-w) mod l2 and
    n0 = (w + r) / l2; it is computed by the lane (k // l2) % 32 of its tile, which walks branch r's Tb taps
    from j = lane % Tb for even d2 (from 0 for odd), an fmaf chain per accumulator over sub-band samples
    n0 + j (zero before zb), then rotated unfused by its phase: the even phase of the oscillator table, one
    cmul_unfused step further for odd k.  Returns per member one complex64 array per block from `attach` on.

    mutation (MUTATIONS): newest_dropped skips the newest window sample (j = Tb - 1); zb_minus_1 reads the
    last sample before the attach point; odd_no_step gives odd outputs their even neighbour's phase;
    tap_stride_T2 reads tap rows Tb apart instead of sb_tpad(Tb); branch_w_mod_L2 takes branch w mod l2;
    phase_row_plus_32 reads the phases of member m + 32 (mod the class size) for member m."""
    n = len(revs)
    T = revs[0].size
    x = np.concatenate([np.zeros(0, np.complex64)] + [np.asarray(r, np.complex64) for r in rows])
    zb = sum(len(r) for r in rows[:attach])
    counts = output_counts([len(r) for r in rows[attach:]], l2, d2)
    total = int(counts.sum())
    Tb = -(-T // l2)
    tpad = sb_tpad(Tb)
    stride = Tb if mutation == "tap_stride_T2" else tpad
    w, r, n0 = poly_windows(np.arange(total), T, l2, d2)
    rb = w % l2 if mutation == "branch_w_mod_L2" else r
    local = np.arange(total) - np.repeat(np.cumsum(counts) - counts, counts)
    lane = (local // l2) % 32
    j0 = lane % Tb if d2 % 2 == 0 else np.zeros(total, np.int64)
    lo = zb - 1 if mutation == "zb_minus_1" else zb
    outs = []
    for m in range(n):
        g0 = m - m % SB_MG
        tab = np.zeros((l2, SB_MG * tpad + tpad), np.complex64)  # the group's table (+ a row of slack)
        for s in range(min(SB_MG, n - g0)):
            tab[:, s * tpad:s * tpad + Tb] = poly_pack_np(np.asarray(revs[g0 + s], np.complex64), l2)
        slot = m - g0
        are = np.zeros(total, np.float32)
        aim = np.zeros(total, np.float32)
        for s in range(Tb):
            j = (j0 + s) % Tb
            pos = zb + n0 + j
            ok = (pos >= max(lo, 0)) & (pos < x.size)
            if mutation == "newest_dropped":
                ok &= j != Tb - 1
            v = np.where(ok, x[np.clip(pos, 0, max(x.size - 1, 0))] if x.size else 0, 0).astype(np.complex64)
            h = tab[rb, slot * stride + j]
            vr, vi, hr, hi = _f32(v.real), _f32(v.imag), _f32(h.real), _f32(h.imag)
            are = fmaf(vr, hr, are)
            are = fmaf(-vi, hi, are)
            aim = fmaf(vr, hi, aim)
            aim = fmaf(vi, hr, aim)
        inc = incs[(m + PH_GROUP) % n] if mutation == "phase_row_plus_32" else incs[m]
        ph = oracle_phases(inc, counts, renorm).astype(np.complex64)
        if mutation == "odd_no_step":
            odd = np.nonzero(local % 2 == 1)[0]
            ph[odd] = ph[odd - 1]
        yr, yi = _cmul(are, aim, _f32(ph.real), _f32(ph.imag))
        y = (yr + 1j * yi.astype(np.complex64)).astype(np.complex64)
        outs.append(np.split(y, np.cumsum(counts)[:-1]))
    return outs
