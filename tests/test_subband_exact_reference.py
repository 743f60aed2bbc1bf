"""The exact sub-band references (tests/subband_exact.py) checked on the CPU, before any GPU test relies on them.

* the float64 composition (stage A at centre 0, members fed its rows zero-stuffed by L2) equals SubbandOracle
  and RationalSubbandOracle bit for bit on dyadic stimuli with full-length member taps -- members attached
  mid-stream, L2 > M2, T2 % L2 != 0 and T2 < L2 included;
* the member kernel model equals the oracles bit for bit at any stage-A centre on one-hot stimuli (a real
  input, one-hot sub-band taps; members at offset 0 with one nonzero tap or one per branch, or at any offset
  with the only nonzero tap at taps2[0]), and is not exact for a one-hot tap elsewhere at a nonzero offset;
* mutations of the model each fail at least one exact harness; whether the 1e-5 contract with subband_plan's
  taps sees them is recorded beside each (CONTRACT_ACCEPTS).
"""
import numpy as np
import pytest

from cascade import small_taps
from exact import exact_input, one_hot_taps
from rational import branch_one_hot_taps, real_grid_input
from subband_exact import (MUTATIONS, exact_bound, f64_member, f64_rows, member_consts, member_model)
from subband_rational import RationalSubbandOracle
from util import assert_cf32_close, rand_block

FS = 2016000
D1 = 6
FS1 = FS // D1
SIZES = [8192, 8192, 1002, 7, 0, 2, 8190, 333, 8192]

# (L2, M2, T2) of full-length dyadic members: odd and even D2, T2 = 1, T2 < 32, L2 > M2, T2 % L2 != 0,
# T2 < L2 (with T2 >= M2), gcd(L2, M2) > 1
MEMBERS = [(1, 5, 23), (1, 2, 8), (1, 1, 1), (1, 7, 7), (1, 4, 40), (3, 7, 40), (2, 5, 33), (12, 5, 60),
           (12, 5, 7), (4, 6, 50), (2, 1, 9)]


def feed(orc, blocks, fmt, attach, renorm=True):
    """Feeds every block; members (key -> (l2, d2, taps2, offset)) attach before block attach[key].  Returns
    {key: outputs per block from its attach block on}."""
    got = {}
    for b, x in enumerate(blocks):
        for key, (at, spec) in attach.items():
            if at == b:
                l2, d2, t2, off = spec
                orc.add_member(key, d2, t2, off, interp2=l2)
                got[key] = []
        for key, y in orc.process_cf32(fmt, x, renorm=renorm).items():
            got[key].append(y)
    return got


@pytest.mark.parametrize("fmt", ["cu8", "cs8", "cs16"])
def test_f64_composition_equals_oracles(fmt):
    rng = np.random.default_rng(len(fmt) * 7 + ord(fmt[-1]))
    t1 = small_taps(rng, 17, 3)
    blocks = [exact_input(rng, fmt, n) for n in SIZES]
    attach = {}
    for i, (l2, d2, T2) in enumerate(MEMBERS):
        t2 = small_taps(rng, T2, 3)
        assert exact_bound(t1, t2, fmt)
        attach[i] = (i % 3 * 2, (l2, d2, t2, 0))  # attached before blocks 0, 2 and 4
    orc = RationalSubbandOracle(D1, t1, 0, FS, max(SIZES))
    got = feed(orc, blocks, fmt, attach)
    rows = f64_rows(D1, t1, FS, fmt, blocks)
    assert all(np.array_equal(a, b) for a, b in zip(rows, orc.rows))
    for key, (at, (l2, d2, t2, _)) in attach.items():
        want = f64_member(rows[at:], l2, d2, t2, FS1)
        assert len(want) == len(got[key])
        for b, (y, r) in enumerate(zip(got[key], want)):
            assert np.array_equal(y, r), (MEMBERS[key], at, b)
        flat = np.concatenate(want)
        # with T2 < L2 the branches past T2 are empty and their outputs 0
        assert np.count_nonzero(flat) > (0.9 if t2.size >= l2 else 0.4) * flat.size
    # and a member attached mid-stream reads zeros before its attach point, not the rows it missed
    l2, d2, t2, _ = attach[1][1]
    assert not all(np.array_equal(a, b) for a, b in zip(f64_member(rows, l2, d2, t2, FS1)[2:], got[1]))


def test_exact_bound_of_the_long_kind():
    """The long kind's 800 stage-A taps of +-1/2 leave room for about sum |m2| <= 160 on the cs16 grid."""
    t1 = np.full(800, 0.5, np.float32)
    assert exact_bound(t1, np.full(163, 0.5, np.float32), "cs16")
    assert not exact_bound(t1, np.full(164, 0.5, np.float32), "cs16")


# ---------------------------------------------------------------------------
# the kernel model at any stage-A centre
# ---------------------------------------------------------------------------
def one_hot_population(rng, attach_mid):
    """{key: (attach block, (l2, d2, taps2, offset))} of members exact on a complex row."""
    pop, k = {}, 0
    for l2, d2, T2 in MEMBERS:
        at = 2 if attach_mid and k % 2 else 0
        if l2 == 1:
            t2 = one_hot_taps(T2, int(rng.integers(0, T2)), float(rng.choice([0.5, -0.75, 0.625])))
        else:
            t2 = branch_one_hot_taps(rng, T2, l2)
        pop[k] = (at, (l2, d2, t2, 0))  # offset 0: the taps stay real
        k += 1
        t0 = one_hot_taps(T2, 0, float(rng.choice([0.5, -0.75])))
        pop[k] = (at, (l2, d2, t0, int(rng.integers(-FS1 // 2, FS1 // 2))))  # only taps2[0]: rotation 1
        k += 1
    return pop


def model_of(orc, key, spec, at, renorm=True, mutation=None, cls=None):
    """member_model of one member (or of the class `cls`, a list of (key, spec)); returns {key: outputs}."""
    cls = cls or [(key, spec)]
    l2, d2 = cls[0][1][0], cls[0][1][1]
    consts = [member_consts(s[2], d2, s[3], l2, FS1) for _, s in cls]
    outs = member_model(orc.rows, at, l2, d2, [c[0] for c in consts], [c[1] for c in consts], renorm, mutation)
    return {k: o for (k, _), o in zip(cls, outs)}


def exact_equal(got, want):
    return len(got) == len(want) and all(y.shape == r.shape and np.array_equal(y, r) for y, r in zip(got, want))


@pytest.mark.parametrize("renorm", [True, False], ids=["renorm", "no_renorm"])
@pytest.mark.parametrize("center", [-1007999, -312000, 0, 17, 251001])
def test_model_equals_oracle_at_any_centre(center, renorm):
    rng = np.random.default_rng(abs(center) % 997 + renorm)
    t1 = one_hot_taps(17, int(rng.integers(0, 17)), 0.75)
    blocks = [real_grid_input(rng, n) for n in SIZES]
    pop = one_hot_population(rng, attach_mid=True)
    orc = RationalSubbandOracle(D1, t1, center, FS, max(SIZES))
    got = feed(orc, blocks, "cs16", pop, renorm=renorm)
    if center:
        assert np.count_nonzero(np.concatenate(orc.rows).imag) > 0.9 * sum(r.size for r in orc.rows)
    for key, (at, spec) in pop.items():
        m = model_of(orc, key, spec, at, renorm)[key]
        assert exact_equal(m, got[key]), (key, spec[:2], spec[3], at)
        # only taps2[0]: one branch of L2 is nonzero
        assert np.count_nonzero(np.concatenate(got[key])) > 0.8 / spec[0] * sum(y.size for y in got[key])
    # a class of members at distinct offsets (two groups of SB_MG) is each member's own filter
    cls = [(100 + i, (1, 5, one_hot_taps(23, 0, 0.5), int(rng.integers(-FS1 // 2, FS1 // 2)))) for i in range(20)]
    orc = RationalSubbandOracle(D1, t1, center, FS, max(SIZES))
    got = feed(orc, blocks, "cs16", {k: (2, s) for k, s in cls}, renorm=renorm)
    for k, m in model_of(orc, None, None, 2, renorm, cls=cls).items():
        assert exact_equal(m, got[k]), k


def test_one_hot_tap_elsewhere_is_not_exact_at_an_offset():
    """A single nonzero tap not at taps2[0] at a nonzero offset is a complex tap on a complex row: the
    kernels' fmaf of two products and the oracle's two rounded products differ in about a third of the
    outputs, so exact tests must not rely on it."""
    rng = np.random.default_rng(5)
    t1 = one_hot_taps(17, 3, 0.75)
    blocks = [real_grid_input(rng, n) for n in [8192] * 8]
    spec = (1, 5, one_hot_taps(23, 11, 0.5), 41234)
    orc = RationalSubbandOracle(D1, t1, 312345, FS, 8192)
    got = feed(orc, blocks, "cs16", {0: (0, spec)})[0]
    m = np.concatenate(model_of(orc, 0, spec, 0)[0])
    want = np.concatenate(got)
    assert m.size == want.size >= 1000
    assert 0.2 * m.size < np.count_nonzero(m != want) < 0.6 * m.size
    assert_cf32_close(m, want)


# ---------------------------------------------------------------------------
# mutations of the kernel model
# ---------------------------------------------------------------------------
def harness_dyadic(mutation):
    """Dyadic stage A at centre 0 on cu8, dyadic full-length classes attached mid-stream (odd Tb, several
    members per class) against the float64 composition.  True when the model is exact."""
    rng = np.random.default_rng(71)
    t1 = small_taps(rng, 17, 3)
    blocks = [exact_input(rng, "cu8", n) for n in SIZES]
    rows = f64_rows(D1, t1, FS, "cu8", blocks)
    rows32 = [r.astype(np.complex64) for r in rows]
    for l2, d2, T2, n in [(1, 5, 9, 3), (1, 4, 9, 2), (3, 7, 37, 3), (2, 5, 33, 2)]:
        taps = [small_taps(rng, T2, 3) for _ in range(n)]
        consts = [member_consts(t, d2, 0, l2, FS1) for t in taps]
        outs = member_model(rows32, 2, l2, d2, [c[0] for c in consts], [c[1] for c in consts], mutation=mutation)
        for t, o in zip(taps, outs):
            if not exact_equal(o, f64_member(rows[2:], l2, d2, t, FS1)):
                return False
    return True


def harness_one_hot(mutation):
    """One-hot stage A at centre 312345 on a real input; a class of 40 members (three groups of SB_MG, two
    oscillator table groups) at distinct offsets with only taps2[0], and a branch-one-hot rational class at
    offset 0, attached mid-stream, against RationalSubbandOracle.  True when the model is exact."""
    rng = np.random.default_rng(73)
    t1 = one_hot_taps(17, 5, 0.75)
    blocks = [real_grid_input(rng, n) for n in SIZES]
    ints = [(i, (1, 5, one_hot_taps(23, 0, 0.5), int(rng.integers(-FS1 // 2, FS1 // 2)))) for i in range(40)]
    rats = [(100 + i, (3, 7, branch_one_hot_taps(rng, 40, 3), 0)) for i in range(3)]
    orc = RationalSubbandOracle(D1, t1, 312345, FS, max(SIZES))
    got = feed(orc, blocks, "cs16", {k: (2, s) for k, s in ints + rats})
    for cls in (ints, rats):
        for k, m in model_of(orc, None, None, 2, mutation=mutation, cls=cls).items():
            if not exact_equal(m, got[k]):
                return False
    return True


def planned_population(pkg, fs):
    """(d1, fs1, taps1, l2, d2, taps2) of 48 kHz members as subband_plan designs them: at 2.016 Msps its
    D1 = 6 plan (one 48 kHz client), integer members of 85 taps at 336 kHz; at 2.048 Msps rational ones."""
    p = pkg.subband_plan(fs, [(312345, 48000)])
    m = p["members"][0]
    return p["d1"], p["fs1"], p["taps1"], m["interp2"], m["d2"], m["taps2"]


def contract_accepts(pkg, mutation):
    """subband_plan's taps (integer members at 2.016 Msps, rational ones at 2.048 Msps): a complex row from the
    strict oracle at sub-band centre 312345 on random cu8 blocks, a class of 40 members at distinct offsets
    attached mid-stream.  One bool per population, True when the model is within 1e-5 of the oracle for every
    member."""
    return tuple(contract_accepts_at(pkg, fs, mutation) for fs in (2016000, 2048000))


def contract_accepts_at(pkg, fs, mutation):
    rng = np.random.default_rng(fs % 1000 + 3)
    d1, fs1, t1, l2, d2, t2 = planned_population(pkg, fs)
    cls = [(i, (l2, d2, t2, int(off))) for i, off in enumerate(np.linspace(-fs1 // 5, fs1 // 5, 40))]
    orc = RationalSubbandOracle(d1, t1, 312345, fs, 16384)
    blocks = [rand_block(rng, "cu8", n) for n in [16384, 16384, 16384, 5002, 16384, 16384]]
    got = feed(orc, blocks, "cu8", {k: (2, s) for k, s in cls})
    consts = [member_consts(t2, d2, s[3], l2, fs1) for _, s in cls]
    outs = member_model(orc.rows, 2, l2, d2, [c[0] for c in consts], [c[1] for c in consts], mutation=mutation)
    for (k, _), o in zip(cls, outs):
        try:
            assert_cf32_close(np.concatenate(o), np.concatenate(got[k]))
        except AssertionError:
            if mutation is None:
                raise
            return False
    return True


def test_planned_populations(pkg):
    d1, fs1, t1, l2, d2, t2 = planned_population(pkg, 2016000)
    assert (d1, l2, d2) == (6, 1, 7) and np.array_equal(t2, pkg.create_low_pass_filter(1.0, 336000, 24000, 9600))
    assert t2.size == 85 and abs(t2[0]) < 1e-8 * np.abs(t2).max()
    d1, fs1, t1, l2, d2, t2 = planned_population(pkg, 2048000)
    assert l2 > 1 and t2.size % l2 != 0


# Does the 1e-5 contract with subband_plan's taps accept the mutant?  (integer population, rational one.)
# The newest window sample of an integer member meets taps2[0], about 1e-9 of the peak: dropping it is
# invisible, while a rational member's branches end on taps of its passband ripple.  The sample before the
# attach point meets taps2[1] (4e-3 of the peak) in the first output and is seen.  The branch of an integer
# member is always 0, so its w mod L2 cannot be wrong.  Everything else exceeds 1e-5.
CONTRACT_ACCEPTS = {"newest_dropped": (True, False), "zb_minus_1": (False, False), "odd_no_step": (False, False),
                    "tap_stride_T2": (False, False), "branch_w_mod_L2": (True, False),
                    "phase_row_plus_32": (False, False)}


def test_unmutated_model_passes_every_harness(pkg):
    assert harness_dyadic(None) and harness_one_hot(None) and contract_accepts(pkg, None) == (True, True)


@pytest.mark.parametrize("mutation", MUTATIONS)
def test_mutation_rejected_by_an_exact_harness(pkg, mutation):
    dyadic, one_hot = harness_dyadic(mutation), harness_one_hot(mutation)
    assert not (dyadic and one_hot), mutation
    assert contract_accepts(pkg, mutation) == CONTRACT_ACCEPTS[mutation]
