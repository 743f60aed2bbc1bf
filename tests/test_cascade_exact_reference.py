"""The stage-B model of cascade clients (tests/cascade_exact.py) checked on the CPU, before any GPU test relies on it.

* on exact stimuli the model equals the float64 composition bit for bit at any ko, for L2 = 1 and rational stage
  B up to L2 = 441, with D2 > T2, T2 = 1 and Tb2 = 1, attached at the first block or mid-stream;
* with designed taps (cascade_plan at five band rates) it is within 1e-5 of the composed oracles;
* its bits depend on ko exactly where the kernels' do: with even D2 (M2), not with odd;
* every mutation differs from it on designed taps, those that change which samples or taps are summed also on
  exact stimuli; whether the 1e-5 contract sees each is recorded (CONTRACT_ACCEPTS);
* the ko and refusal mirrors take every CTA size and hold at the shared-memory bound.
"""
import numpy as np
import pytest

from cascade import CascadeOracle, f64_filter, small_taps
from cascade_exact import (C_KO, INT_KO_CASES, MUTATIONS, ORDER_MUTATIONS, RAT_CASES, TILE_MAX_SMEM,
                           cascade_ko, cascade_poly_ko, cascade_poly_smem, cascade_smem, f64_stage_b, max_t2,
                           ring_cap, ring_windows, stage_b_ko, stage_b_model, stage_b_refused, stage_b_walk)
from cascade_rational import RationalCascadeOracle, f64_composition, stuff
from exact import exact_input, to_complex
from subband_exact import exact_bound
from util import assert_cf32_close, rand_block

FS = 2016000
D1 = 6
FS1 = FS // D1
SIZES = [8192, 8192, 1002, 7, 0, 2, 8190, 333, 8192, 8192]

# (L2, M2, T2): odd and even D2, T2 = 1, D2 > T2, T2 around 32 with even D2, and the rational shapes
EXACT_SHAPES = [(1, 7, 85), (1, 2, 85), (1, 3, 1), (1, 4, 1), (1, 9, 4), (1, 10, 3), (1, 2, 31), (1, 2, 32),
                (1, 2, 33), (2, 7, 85), (2, 8, 85), (3, 7, 40), (12, 5, 120), (128, 125, 700), (129, 127, 700),
                (441, 640, 1000), (12, 5, 12)]


def exact_equal(got, want):
    return len(got) == len(want) and all(y.shape == r.shape and np.array_equal(y, r) for y, r in zip(got, want))


def exact_rows(seed):
    """Dyadic stage A (9 taps of 2 bits, D1 = 6, centre 0) on exact cu8 blocks: its float64 rows (exact)."""
    rng = np.random.default_rng(seed)
    t1 = small_taps(rng, 9, 2)
    blocks = [to_complex("cu8", exact_input(rng, "cu8", n)) for n in SIZES]
    return rng, t1, blocks, f64_filter(t1, D1, 0, FS, blocks)


@pytest.mark.parametrize("attach", [0, 2])
@pytest.mark.parametrize("shape", EXACT_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_model_equals_float64_composition(shape, attach):
    L2, M2, T2 = shape
    rng, t1, blocks, rows = exact_rows(T2 + M2)
    t2 = small_taps(rng, T2, 1)
    assert exact_bound(t1, t2, "cu8")
    want = f64_stage_b(rows, attach, L2, M2, t2)
    if attach == 0:
        assert exact_equal(want, f64_composition(D1, t1, L2, M2, t2, FS, blocks))
    else:
        assert exact_equal(want, f64_filter(t2, M2, 0, L2 * FS1, [stuff(y, L2) for y in rows[attach:]]))
    rows32 = [y.astype(np.complex64) for y in rows]
    for ko in sorted({stage_b_ko(L2, M2, T2), C_KO, 64, 16, 3, 1}):
        got = stage_b_model(rows32, attach, L2, M2, t2, FS1, ko)
        assert exact_equal(got, [y.astype(np.complex64) for y in want]), (shape, ko)
    n = sum(y.size for y in want)
    assert n > 100 and np.count_nonzero(np.concatenate(want)) > (0.9 if T2 >= L2 else 0.4) * n


# ---------------------------------------------------------------------------
# designed taps
# ---------------------------------------------------------------------------
PLANS = {2016000: ("cu8", 65536), 2048000: ("cu8", 65536), 10000000: ("cs16", 65536), 20000000: ("cs8", 65536),
         61440000: ("cs16", 131072)}


def planned(pkg, fs, seed=0, n_blocks=5):
    """cascade_plan's 48 kHz client at band rate fs (centre -312000) on random blocks: (plan, stage-A rows of
    the composed oracle, its stage-B outputs)."""
    fmt, max_in = PLANS[fs]
    p = pkg.cascade_plan(fs, [48000])[0]
    rng = np.random.default_rng(fs % 997 + seed)
    blocks = [rand_block(rng, fmt, max_in if b != 2 else max_in // 3 * 2 + 2) for b in range(n_blocks)]
    if p["interp2"] == 1:
        o = CascadeOracle(p["d1"], p["taps1"], p["center"], p["d2"], p["taps2"], fs, max_in)
        rows = [o.a.process_cf32(fmt, x) for x in blocks]
        want = [o.b.process_cf32(y) for y in rows]
    else:
        o = RationalCascadeOracle(p["d1"], p["taps1"], p["center"], p["interp2"], p["d2"], p["taps2"], fs, max_in)
        rows = [o.a.process_cf32(fmt, x) for x in blocks]
        want = [o.b.process_cf32(stuff(y, p["interp2"])) for y in rows]
    return p, rows, want


def model_of(p, fs, rows, ko=None, mutation=None):
    ko = ko or stage_b_ko(p["interp2"], p["d2"], len(p["taps2"]))
    return stage_b_model(rows, 0, p["interp2"], p["d2"], p["taps2"], fs // p["d1"], ko, mutation)


@pytest.mark.parametrize("fs", list(PLANS))
def test_model_within_contract_of_oracle(pkg, fs):
    p, rows, want = planned(pkg, fs)
    got = model_of(p, fs, rows)
    assert [y.size for y in got] == [y.size for y in want]
    assert sum(y.size for y in got) >= 100
    assert_cf32_close(np.concatenate(got), np.concatenate(want), f"{fs}")


def test_bits_depend_on_ko_only_with_even_decimation(pkg):
    """Odd D2 (2.016 Msps: 6 x 7) and odd M2 (10 Msps: 12/125): the same bits at every ko.  Even D2 (61.44 Msps:
    32 x 40) and even M2 (2.048 Msps: 3/16, 20 Msps: 3/50): most outputs whose lane changes get other bits."""
    for fs in (2016000, 10000000):
        p, rows, _ = planned(pkg, fs)
        assert p["d2"] % 2 == 1
        ref = np.concatenate(model_of(p, fs, rows))
        for ko in (C_KO, 16, 4, 1):
            assert np.array_equal(np.concatenate(model_of(p, fs, rows, ko)), ref), (fs, ko)
    for fs in (61440000, 2048000, 20000000):
        p, rows, _ = planned(pkg, fs)
        assert p["d2"] % 2 == 0
        a = np.concatenate(model_of(p, fs, rows))
        b = np.concatenate(model_of(p, fs, rows, 16))
        assert a.size == b.size > 100
        assert np.count_nonzero(a != b) > 0.2 * a.size, fs
        assert_cf32_close(a, b, f"{fs}")


# ---------------------------------------------------------------------------
# mutations of the model
# ---------------------------------------------------------------------------
def exact_harness(mutation):
    """Exact stimuli, L2 = 1 with odd and even D2 and rational shapes with T2 % L2 != 0, attached mid-stream:
    True when the (mutated) model still equals the float64 composition."""
    _, _, _, rows = exact_rows(91)
    rows32 = [y.astype(np.complex64) for y in rows]
    rng = np.random.default_rng(92)
    for L2, M2, T2 in [(1, 7, 85), (1, 2, 33), (3, 7, 40), (3, 16, 193)]:
        t2 = small_taps(rng, T2, 1)
        got = stage_b_model(rows32, 2, L2, M2, t2, FS1, stage_b_ko(L2, M2, T2), mutation)
        if not exact_equal(got, [y.astype(np.complex64) for y in f64_stage_b(rows, 2, L2, M2, t2)]):
            return False
    return True


def designed_differs(pkg, mutation):
    """cascade_plan's taps: integer stage B with odd (2.016 Msps) and even D2 (61.44 Msps), rational with odd
    (10 Msps) and even M2 (2.048 Msps).  One bool per plan: the mutant's bits differ from the model's."""
    out = []
    for fs in (2016000, 61440000, 10000000, 2048000):
        p, rows, _ = planned(pkg, fs, n_blocks=3)
        a, b = np.concatenate(model_of(p, fs, rows)), np.concatenate(model_of(p, fs, rows, mutation=mutation))
        out.append(not np.array_equal(a, b))
    return tuple(out)


def contract_accepts(pkg, mutation):
    """The same four plans: True per plan where the mutant is within 1e-5 of the composed oracle."""
    out = []
    for fs in (2016000, 61440000, 10000000, 2048000):
        p, rows, want = planned(pkg, fs, n_blocks=3)
        try:
            assert_cf32_close(np.concatenate(model_of(p, fs, rows, mutation=mutation)), np.concatenate(want))
            out.append(True)
        except AssertionError:
            out.append(False)
    return tuple(out)


# Plans: 2.016 Msps (odd D2), 61.44 Msps (even D2), 10 Msps (L2 = 12, odd M2), 2.048 Msps (L2 = 3, even M2).
# Where a mutant changes bits it differs from the model (DESIGNED_DIFFERS); whether the 1e-5 contract still
# accepts it is CONTRACT_ACCEPTS.  Both ends of an integer plan's window meet taps of about 1e-9 of the peak, so
# dropping either is invisible to the contract, and so are the order mutations, which only change the rounding.
# At 2.048 Msps (T2 = 193 = 3 * 64 + 1) only branch 0 has a 65th tap, the window's edge: dropping the newest tap
# or walking floor(T2 / L2) taps removes just that one and the contract accepts both; at 10 Msps
# (T2 = 1505 = 12 * 125 + 5) five branches lose their 126th tap and the contract sees it.  The integer plans have branch 0
# only and T2 % 1 == 0, so branch and Tb mutations cannot touch them, and the odd-M2 skew changes nothing for the
# even-M2 plans.
DESIGNED_DIFFERS = {"newest_dropped": (True, True, True, True), "oldest_dropped": (True, True, True, True),
                    "lane_tid_15": (False, True, False, True), "skew_odd": (True, False, True, False),
                    "branch_w_mod_L2": (False, False, True, True), "Tb_floor": (False, False, True, True)}
CONTRACT_ACCEPTS = {"newest_dropped": (True, True, False, True), "oldest_dropped": (True, True, False, False),
                    "lane_tid_15": (True, True, True, True), "skew_odd": (True, True, True, True),
                    "branch_w_mod_L2": (True, True, False, False), "Tb_floor": (True, True, False, True)}


def test_unmutated_model_passes_every_harness(pkg):
    assert exact_harness(None)
    assert designed_differs(pkg, None) == (False,) * 4
    assert contract_accepts(pkg, None) == (True,) * 4


@pytest.mark.parametrize("mutation", MUTATIONS)
def test_mutation(pkg, mutation):
    assert designed_differs(pkg, mutation) == DESIGNED_DIFFERS[mutation]
    # mutations of which samples or taps are summed fail on exact stimuli; the order ones cannot be seen there
    assert exact_harness(mutation) == (mutation in ORDER_MUTATIONS)
    assert contract_accepts(pkg, mutation) == CONTRACT_ACCEPTS[mutation]


# ---------------------------------------------------------------------------
# the host mirrors
# ---------------------------------------------------------------------------
def test_ko_mirrors_take_every_cta_size():
    for ko, cases in INT_KO_CASES.items():
        assert [D2 % 2 for D2, _ in cases] == [1, 0]
        for D2, T2 in cases:
            assert cascade_ko(D2, T2) == ko
            assert cascade_smem(ko, D2, T2) <= TILE_MAX_SMEM
            assert ko == C_KO or cascade_smem(2 * ko, D2, T2) > TILE_MAX_SMEM
    assert cascade_ko(1024, 64) == 16 and cascade_ko(40, 481) == C_KO
    want = [256, 128, 252, 31, 240, 254, 256, 256, 256, 240, 256]
    assert [stage_b_ko(*c) for c in RAT_CASES] == want
    for (L2, M2, T2), ko in zip(RAT_CASES, want):
        Tb2 = -(-T2 // L2)
        assert cascade_poly_ko(L2, M2, Tb2) == ko
        assert cascade_poly_smem(ko, L2, M2, Tb2) <= TILE_MAX_SMEM
        whole = L2 <= 128 and ko % L2 == 0
        assert whole == ((L2, M2) not in ((3, 2000), (129, 127), (441, 640))), (L2, M2)
    # halving from 252 down to 1 at the smallest M2 where each value is reached
    M2s = [7, 306, 614, 1237, 2557, 5478, 12781, 38342]
    assert [cascade_poly_ko(3, M2, 14) for M2 in M2s] == [252, 126, 63, 31, 15, 7, 3, 1]
    assert [cascade_poly_ko(3, M2 - 1, 14) for M2 in M2s[1:]] == [252, 126, 63, 31, 15, 7, 3]


def test_refusal_mirror_at_the_bound():
    for L2, M2 in [(1, 2), (1, 1600), (1, 8518), (3, 3001), (2, 255), (441, 640)]:
        T2 = max_t2(L2, M2)
        assert not stage_b_refused(L2, M2, T2) and stage_b_refused(L2, M2, T2 + 1), (L2, M2)
        assert T2 % L2 == 0
        assert stage_b_ko(L2, M2, T2) >= 1
    assert max_t2(1, 2) == max_t2(1, 1600) == 17064  # one output's window does not depend on D2
    assert max_t2(3, 3001) == 30714


def test_window_bookkeeping():
    """ring_windows sees odd and even window starts and windows across the ring's end."""
    cap = ring_cap(85, 1, 4098)
    assert cap == 32768
    walk = stage_b_walk([683] * 200, 1, 7, 85)
    parities, wraps = ring_windows(walk, 1, 7, 85, 256, cap)
    assert parities == {0, 1} and wraps >= 3
    # before the stream reaches the ring's end only the first window crosses it: it starts before the attach
    # point, at ring index cap - 84
    assert ring_windows(stage_b_walk([683] * 20, 1, 7, 85), 1, 7, 85, 256, cap)[1] == 1
