"""The rational exact-stimulus harness (tests/rational.py) checked on the CPU, before any GPU test relies on it.

* ref_rational_f64, the float64 polyphase sum on the input-rate stream, equals ref_f64 on the zero-stuffed
  stream bit for bit (and the strict float32 oracle wherever it may run, T >= M: with fewer taps than the
  decimation its history bookkeeping underflows) for T < L, T % L != 0, T < M, gcd(L, M) > 1, M = 1, L > M,
  L up to 441, given history and 0- and 2-element calls;
* branch_one_hot_taps leaves one nonzero per polyphase branch, so the kernels' single-product model equals
  the strict oracle at any centre;
* mutations of the polyphase model (wrong branch, window one sample off before the attach point, the last
  tap row dropped, odd outputs without their oscillator step) fail assert_exact; whether the 1e-5 float
  contract with designed taps sees them is recorded beside each.
"""
import numpy as np
import pytest

from exact import assert_exact, dyadic_taps, exact_input, grid_step, oscillator_increment, ref_f64, to_complex
from oracle import pyoracle as po
from rational import (MUTATIONS, RationalRef, branch_one_hot_taps, oracle_filter, poly_model, poly_pack_np,
                      real_grid_input, ref_rational_f64, stuff)
from util import assert_cf32_close, rand_block

FS = 2048000
FMTS = ("cu8", "cs8", "cs16")
# (L, M, T): T < L, T % L != 0, T < M, gcd(L, M) > 1, M = 1, L > M, L in {16, 17, 36, 37, 160, 441}
SPECS = [(3, 128, 97), (5, 4, 3), (2, 1, 9), (5, 3, 40), (7, 320, 431), (16, 15, 97), (17, 16, 200),
         (36, 35, 300), (37, 36, 300), (6, 256, 400), (4, 2, 9), (160, 147, 1000), (147, 160, 1000),
         (441, 20480, 2000), (17, 16, 5), (37, 5, 36), (2, 1, 1)]
SIZES = [8192, 2, 0, 6002, 7, 4096]


def spec_id(s):
    return "L{}_M{}_T{}".format(*s)


def stuffed_history(hist, L, T):
    """The T - 1 upsampled samples before the attach point of the stuffed stream whose input-rate history
    is `hist` (newest last): u[-L * j] = hist[-j]."""
    hu = np.zeros(T - 1, np.complex128)
    for j in range(1, (T - 1) // L + 1):
        if j <= hist.size:
            hu[T - 1 - L * j] = hist[-j]
    return hu


@pytest.mark.parametrize("spec", SPECS, ids=spec_id)
def test_ref_rational_f64_equals_stuffed_ref_f64(spec):
    L, M, T = spec
    rng = np.random.default_rng(L * 7919 + M * 31 + T)
    fmt = FMTS[(L + T) % 3]
    taps = dyadic_taps(rng, T, fmt)
    blocks = [exact_input(rng, fmt, n) for n in SIZES]
    got = ref_rational_f64(taps, L, M, fmt, blocks)
    want = ref_f64(taps, M, "cs16", [stuff(fmt, x, L) for x in blocks])
    assert_exact(got, want, f"L={L} M={M} T={T} {fmt}", T, M, grid_step(taps, fmt))
    assert sum(np.count_nonzero(y) for y in want) > 0
    if T >= M:
        o = oracle_filter(po, L, M, taps, 0, FS, max(SIZES))
        assert_exact(got, [o.process_cf32("cs16", stuff(fmt, x, L)) for x in blocks], f"oracle L={L} M={M} T={T}")


@pytest.mark.parametrize("spec", [(3, 128, 97), (17, 16, 200), (160, 147, 1000), (4, 2, 9), (37, 5, 100)],
                         ids=spec_id)
def test_ref_rational_f64_history(spec):
    """history: the input-rate samples a client attached mid-stream reads before its first call."""
    L, M, T = spec
    rng = np.random.default_rng(T + 5)
    fmt = "cu8"
    taps = dyadic_taps(rng, T, fmt)
    hist = to_complex(fmt, exact_input(rng, fmt, 2 * (-(-T // L) + 3)))
    blocks = [exact_input(rng, fmt, n) for n in SIZES]
    got = ref_rational_f64(taps, L, M, fmt, blocks, history=hist)
    want = ref_f64(taps, M, "cs16", [stuff(fmt, x, L) for x in blocks], history=stuffed_history(hist, L, T))
    assert_exact(got, want, f"history L={L} M={M} T={T}", T, M, grid_step(taps, fmt))
    # and the history is read: without it the first outputs differ
    with pytest.raises(AssertionError, match="first at block 0 output 0"):
        assert_exact(ref_rational_f64(taps, L, M, fmt, blocks), want, "no history")


def test_ref_rational_f64_block_by_block_carries_state():
    """Feeding one call at a time (the reference the long-stream GPU test keeps) is the one-shot sum."""
    rng = np.random.default_rng(9)
    L, M, T, fmt = 441, 20480, 2000, "cu8"
    taps = dyadic_taps(rng, T, fmt)
    blocks = [exact_input(rng, fmt, n) for n in [65536, 2, 65536, 0, 30001, 65536]]
    ref = RationalRef(taps, L, M)
    assert_exact([ref.feed(fmt, x) for x in blocks], ref_f64(taps, M, "cs16", [stuff(fmt, x, L) for x in blocks]),
                 "block by block")


@pytest.mark.parametrize("T", [199, 200, 5, 6, 1000, 1001])
@pytest.mark.parametrize("L", [3, 16, 17, 36, 37, 160, 441])
def test_branch_one_hot_rows(T, L):
    rng = np.random.default_rng(T * 3 + L)
    taps = branch_one_hot_taps(rng, T, L)
    P = poly_pack_np(reversed_taps_of_library(taps), L)
    nz = np.count_nonzero(P, axis=1)
    assert np.all(nz[:min(L, T)] == 1) and np.all(nz[min(L, T):] == 0), nz
    vals = np.abs(P[np.arange(min(L, T)), np.argmax(P[:min(L, T)] != 0, axis=1)])
    assert np.unique(vals).size == vals.size  # a different value in every branch


def reversed_taps_of_library(taps):
    """The reversal the strict oracle applies (centre 0, taps stay real): its rev_taps with a decimation
    of 1 (no history underflow whatever T)."""
    o = po.OracleFilter(1, taps, 0, FS, 64)
    rev = o.rev_taps
    o.close()
    assert np.all(rev.imag == 0)
    return rev.real


ONE_HOT = [(3, 128, 129), (17, 16, 200), (160, 147, 1000), (441, 20480, 20481), (6, 256, 401), (16, 15, 97),
           (36, 35, 300), (37, 36, 300), (3, 2, 8)]


@pytest.mark.parametrize("center", [-987654, -312000, 1, 400123, 1007999])
@pytest.mark.parametrize("spec", ONE_HOT, ids=spec_id)
def test_branch_one_hot_model_equals_oracle(spec, center):
    """Branch-one-hot taps, a real cs16 input on the grid, any centre: the kernels' arithmetic (FMA chain,
    unfused rotation, odd outputs one step past the stored even phase) is the strict oracle bit for bit."""
    L, M, T = spec
    rng = np.random.default_rng(L + M + T + center % 1000)
    taps = branch_one_hot_taps(rng, T, L)
    o = oracle_filter(po, L, M, taps, center, FS, 8192)
    inc = oscillator_increment(M, center, L * FS)
    blocks = [real_grid_input(rng, n) for n in (8192, 2, 2002, 8192, 0, 6000)]
    want = [o.process_cf32("cs16", stuff("cs16", x, L)) for x in blocks]
    flat = np.concatenate(want)
    assert np.count_nonzero(flat) >= 0.98 * flat.size > 0
    assert_exact(poly_model(o.rev_taps, L, M, inc, blocks), want, f"L={L} M={M} T={T} centre {center}", T, M)


# ---------------------------------------------------------------------------
# mutations of the polyphase model
# ---------------------------------------------------------------------------
MUT = (5, 3, 43)  # T % L = 3, windows before the attach point on every branch, (-w) mod L != w mod L
# does the 1e-5 contract with rational_plan taps (2.048 Msps -> 48 ksps: L = 3, M = 128, T = 1541) accept it?
# None of these: a sample off in the first windows, the 514th tap row of two branches and a missing oscillator
# step all exceed 1e-5 of the largest output.  At centre 0, though, the phase is 1 + 0i and the odd-output step
# cannot be seen by the exact dyadic stimuli: only the branch-one-hot ones at nonzero centres catch it.
CONTRACT_ACCEPTS = {"branch_w_mod_L": False, "n0_negative_w": False, "Tb_floor": False, "odd_phase_no_step": False}


@pytest.mark.parametrize("mutation", MUTATIONS)
def test_mutation_rejected_by_exact_stimuli(pkg, mutation):
    L, M, T = MUT
    rng = np.random.default_rng(61)
    blocks = [real_grid_input(rng, n) for n in (4096, 2, 1001 * 2, 4096)]
    # centre 0, dyadic taps: the model equals the float64 polyphase sum; the mutant does not
    taps = dyadic_taps(rng, T, "cs16")
    one = complex(1, 0)
    good = poly_model(reversed_taps_of_library(taps).astype(np.complex64), L, M, one, blocks)
    want = ref_rational_f64(taps, L, M, "cs16", blocks)
    assert_exact(good, want, "unmutated model, centre 0", T, M)
    bad = poly_model(reversed_taps_of_library(taps).astype(np.complex64), L, M, one, blocks, mutation=mutation)
    if mutation == "odd_phase_no_step":
        assert_exact(bad, want, "at centre 0 the phase is 1 + 0i: invisible")
    else:
        with pytest.raises(AssertionError, match="outputs differ"):
            assert_exact(bad, want, mutation, T, M)
    # branch-one-hot taps at a nonzero centre against the strict oracle (one tap per branch at a random
    # position need not sit in the last row or read a sample next to the attach point: those two mutations
    # are left to the dyadic stimuli above)
    center = 312345
    taps = branch_one_hot_taps(rng, T, L)
    o = oracle_filter(po, L, M, taps, center, FS, 8192)
    inc = oscillator_increment(M, center, L * FS)
    want = [o.process_cf32("cs16", stuff("cs16", x, L)) for x in blocks]
    assert_exact(poly_model(o.rev_taps, L, M, inc, blocks), want, "unmutated model, one-hot", T, M)
    if mutation in ("branch_w_mod_L", "odd_phase_no_step"):
        with pytest.raises(AssertionError, match="outputs differ"):
            assert_exact(poly_model(o.rev_taps, L, M, inc, blocks, mutation=mutation), want, mutation, T, M)

    # the float contract with designed taps
    p = pkg.rational_plan(FS, [48000])[0]
    L, M, taps, center = p["interp"], p["decim"], p["taps"], p["center"]
    assert (L, M, taps.size % L) == (3, 128, 2)
    o = oracle_filter(po, L, M, taps, center, FS, 8192)
    inc = oscillator_increment(M, center, L * FS)
    blocks = [rand_block(rng, "cs16", n) for n in (8192, 8192, 3002, 8192)]
    want = np.concatenate([o.process_cf32("cs16", stuff("cs16", x, L)) for x in blocks])
    assert_cf32_close(np.concatenate(poly_model(o.rev_taps, L, M, inc, blocks)), want, "unmutated, designed")
    try:
        assert_cf32_close(np.concatenate(poly_model(o.rev_taps, L, M, inc, blocks, mutation=mutation)), want)
        accepted = True
    except AssertionError:
        accepted = False
    assert accepted == CONTRACT_ACCEPTS[mutation]
