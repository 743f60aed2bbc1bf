"""Sub-band members bit for bit with full-length taps, at any sub-band centre, at class, table and tile edges,
through churn and in randomised mixed populations.

Two stimuli make every member output exact (tests/subband_exact.py):
* dyadic taps on both stages at centre 0, on the exact input grid, within exact_bound: every partial sum of
  the sub-band and of a full-length member filter is a whole number of grid steps, so the output equals the
  float64 composition (f64_rows / f64_member) -- a dropped tap, a window one sample off, a tap row read at the
  wrong stride or one pre-attach sample changes it by whole grid steps;
* one-hot sub-band taps at any centre on a real input (each row sample is one product, so the row equals the
  strict oracle's), members at offset 0 with one nonzero tap (branch-one-hot when rational) or at any offset
  with the only nonzero tap at taps2[0]; or a centre-0 dyadic sub-band on a real input (a real row) with
  one-hot members at any offset: every member accumulator is one product, so the output equals
  RationalSubbandOracle's, oscillators included.

Every test asserts the kernel kinds: 6 (xlg_client_info) for members, the stage-A kind (xlg_subband_info).
"""
import errno

import numpy as np
import pytest

from cascade import small_taps
from exact import dyadic_taps, exact_input, one_hot_taps
from rational import real_grid_input
from subband_exact import SB_KO
from subband_rig import Rig, dyadic_member, dyadic_stage_a, one_hot_member, real_row_member

pytestmark = pytest.mark.gpu

GENERIC, TILED, LONG, MEMBER = 0, 1, 2, 6
SLOTS = 4
# sub-band (D1, T1), sub-bands in the group, forced generic: which stage-A kernel serves it
STAGE_A = {"generic": (6, 17, 2, True), "tiled": (6, 17, 8, False), "long": (400, 800, 8, False)}
WANT = {"generic": GENERIC, "tiled": TILED, "long": LONG}


def next_pow2(n):
    return 1 << max(0, int(n - 1).bit_length())


def member_cap(max_in, d1, l2, d2):
    """A member's output row capacity per block (rebuild_layout's out_cap)."""
    return (max_in // 2 // d1 + 2) * l2 // d2 + 2


# ---------------------------------------------------------------------------
# stimuli (tests/subband_rig.py)
# ---------------------------------------------------------------------------
def stage_a_kinds_ok(rig, case):
    want = WANT[case]
    kinds = rig.kinds()
    assert want in kinds and kinds <= {GENERIC, want}, (case, kinds)


# ---------------------------------------------------------------------------
# A. full sums: dyadic full-length members against the float64 composition
# ---------------------------------------------------------------------------
INT_SHAPES = [(5, 23), (4, 8), (7, 7), (2, 31), (1, 1), (3, 9), (6, 40), (40, 1356)]  # (D2, T2)
RAT_SHAPES = [(2, 5, 33), (3, 8, 40), (12, 5, 120), (4, 6, 50), (2, 1, 9), (3, 7, 40), (12, 5, 7)]  # (L2, M2, T2)
FULL = {"generic_cu8": ("generic", "cu8", 8192), "tiled_cs8": ("tiled", "cs8", 8192),
        "long_cs16": ("long", "cs16", 65536)}


@pytest.mark.parametrize("name", list(FULL))
def test_full_sums_against_float64_composition(pkg, monkeypatch, name):
    """Odd and even T2 and D2, T2 < 32 (lane % T2 wraps), T2 = 1, T2 at the shared-memory bound (and one
    past it refused); rational L2 = 2, 3, 12 with gcd(L2, M2) > 1, L2 > M2, T2 % L2 != 0 and T2 < L2; classes
    of three members; members attached at block 0 and mid-stream."""
    case, fmt, max_in = FULL[name]
    d1, T1, n_sb, generic = STAGE_A[case]
    fs = 2016000
    fs1 = fs // d1
    rng = np.random.default_rng(sum(map(ord, name)))
    assert pkg.subband_member_fits(1, 40, 1356) and not pkg.subband_member_fits(1, 40, 1357)
    row = max_in // 2 // d1 + 8  # two sub-bands' members take about 27 rows
    rig = Rig(pkg, monkeypatch, fs, max_in, fmt, flags=pkg.XLG_FORCE_GENERIC if generic else 0, depth=SLOTS,
              reserve=(60 + n_sb) * row)
    sbs = [rig.add_subband(d1, dyadic_stage_a(rng, d1, T1), 0, True) for _ in range(n_sb)]
    with pytest.raises(ValueError) as e:
        rig.g.add_client_subband(sbs[0].sid, 40, np.ones(1357, np.float32), 0)
    assert e.value.args[0] == -errno.EINVAL

    def attach(sb):
        for d2, T2 in INT_SHAPES:
            for _ in range(3 if T2 in (23, 9) else 1):
                rig.add_member(sb, 1, d2, dyadic_member(rng, sb.taps1, T2, fmt), 0, True)
        for l2, m2, T2 in RAT_SHAPES:
            for _ in range(3 if T2 == 40 else 1):
                rig.add_member(sb, l2, m2, dyadic_member(rng, sb.taps1, T2, fmt), 0, True)

    attach(sbs[0])
    sizes = [max_in, max_in, 1002, max_in, 7, 1, 0, max_in - 2, 2 * d1 * 41 + 1] + [max_in] * 8 + [333] * 4
    for b, n in enumerate(sizes):
        if b == 3:
            attach(sbs[1])  # mid-stream: the ring holds nonzero samples before their attach point
        rig.submit(exact_input(rng, fmt, n))
    rig.check()
    stage_a_kinds_ok(rig, case)
    for m in rig.mems:
        flat = np.concatenate(m.got)
        assert flat.size > 0 and np.count_nonzero(flat) > 0.3 * flat.size, m.label()
    rig.close()


# ---------------------------------------------------------------------------
# B. any sub-band centre: one-hot sub-band taps, members exact on a complex row
# ---------------------------------------------------------------------------
ANY_INT = [(5, 23), (4, 8), (1, 1), (3, 9), (2, 31)]
ANY_RAT = [(3, 7, 40), (2, 5, 33), (12, 5, 60)]
ANY_VARIANTS = {  # stage-A case, env, flag, host_ring
    "generic": ("generic", None, None, 0), "tiled": ("tiled", None, None, 0), "long": ("long", None, None, 0),
    "no_renorm": ("tiled", None, "XLG_NO_RENORM", 0),
    "no_speculation": ("tiled", {"XLATING_B200_SPECULATE": "0"}, None, 0),
    "sm_partition": ("tiled", {"XLATING_B200_PARTITION": "1"}, "XLG_SM_PARTITION", 0),
    "out_device": ("tiled", None, "XLG_OUT_DEVICE", 0), "host_ring": ("tiled", None, None, 8),
}


@pytest.mark.parametrize("variant", list(ANY_VARIANTS))
def test_any_subband_centre(pkg, monkeypatch, variant):
    case, env, flag, host_ring = ANY_VARIANTS[variant]
    d1, T1, n_sb, generic = STAGE_A[case]
    fs = 2016000
    fs1 = fs // d1
    max_in = 65536 if case == "long" else 16384
    rng = np.random.default_rng(sum(map(ord, variant)) + 40)
    flags = (getattr(pkg, flag) if flag else 0) | (pkg.XLG_FORCE_GENERIC if generic else 0)
    rig = Rig(pkg, monkeypatch, fs, max_in, "cs16", flags=flags, host_ring=host_ring, depth=SLOTS, env=env)
    centres = [int(rng.integers(-fs // 2 + 1, fs // 2)) for _ in range(n_sb)]
    sbs = [rig.add_subband(d1, one_hot_taps(T1, int(rng.integers(0, T1)), 0.75), c, False) for c in centres]
    for sb in sbs[:2]:
        for d2, T2 in ANY_INT:
            for any_offset in (False, True, True):
                rig.add_member(sb, 1, d2, *one_hot_member(rng, 1, T2, fs1, any_offset), False)
        for l2, m2, T2 in ANY_RAT:
            for any_offset in (False, True):
                rig.add_member(sb, l2, m2, *one_hot_member(rng, l2, T2, fs1, any_offset), False)
    choices = [max_in, max_in, max_in - 2, 2, 0, 7, 2 * d1 * 23 + 1]
    for _ in range(300):
        n = int(rng.choice(choices)) if rng.integers(0, 3) else int(rng.integers(0, max_in // 2)) * 2
        rig.submit(real_grid_input(rng, n))
    rows = rig.check()
    assert all(np.count_nonzero(np.concatenate(rows[sb][0]).imag) > 0 for sb in sbs[:2])
    stage_a_kinds_ok(rig, case)
    rig.close()


# ---------------------------------------------------------------------------
# C. class, oscillator-table and tile edges
# ---------------------------------------------------------------------------
# (sub-band, L2, D2, T2, members): classes of 1, 3, 4, 5, 15, 16, 17, 31, 32, 33 and 48 over three
# sub-bands, integer and rational, 238 members (SbMem groups of 32 straddle classes and the integer/rational
# boundary: the 197 integer members are not a multiple of 32)
CLASSES = [(0, 1, 5, 23, 48), (0, 1, 4, 9, 1), (0, 1, 3, 13, 17), (1, 1, 5, 23, 33), (1, 1, 2, 8, 16),
           (1, 1, 7, 21, 4), (2, 1, 6, 25, 31), (2, 1, 5, 11, 32), (2, 1, 1, 3, 15),
           (0, 3, 7, 40, 3), (1, 2, 5, 33, 5), (2, 12, 5, 60, 17), (0, 4, 6, 50, 16)]
PILOT_INT, PILOT_RAT = 0, 9  # the classes whose counts the block sizes are chosen for
N2_TARGETS = [0, 1, 63, 64, 65, 128, 129]
RESIDUE_TARGETS = [64, 65]


def pilot_sizes(d1, max_in, cls_int, cls_rat, rng):
    """Block sizes (raw elements) such that the integer pilot class's n2 takes every N2_TARGETS value and the
    rational pilot's residue-0 count ceil(n2 / L2) every RESIDUE_TARGETS value, full blocks between them
    (the ring wraps), for classes attached at block 0 of a sub-band created with them."""
    _, _, d2, _, _ = cls_int
    _, l2, m2, _, _ = cls_rat
    cand = np.arange(0, max_in // 2 + 1, dtype=np.int64)  # samples of the next block
    sizes, S = [], 0

    def counts(S_next):
        R0, R1 = (S - 1) // d1 + 1 if S else 0, np.where(S_next >= 1, (S_next - 1) // d1 + 1, 0)
        n_int = np.where(R1 >= 1, (R1 - 1) // d2 + 1, 0) - ((R0 - 1) // d2 + 1 if R0 else 0)
        n_rat = np.where(R1 >= 1, (l2 * R1 - 1) // m2 + 1, 0) - ((l2 * R0 - 1) // m2 + 1 if R0 else 0)
        return n_int, -(-n_rat // l2)

    plan = [("i", t) for t in N2_TARGETS] + [("r", t) for t in RESIDUE_TARGETS]
    rng.shuffle(plan)
    for kind, target in plan:
        for _ in range(int(rng.integers(1, 4))):
            sizes.append(max_in)
            S += max_in // 2
        n_int, n_res = counts(S + cand)
        hit = np.nonzero((n_int if kind == "i" else n_res) == target)[0]
        assert hit.size, (kind, target)
        n = int(rng.choice(hit))
        sizes.append(2 * n)
        S += n
    return sizes


@pytest.mark.parametrize("stimulus", ["dyadic", "one_hot"])
def test_class_table_and_tile_edges(pkg, monkeypatch, stimulus):
    fs, max_in, d1, T1 = 2016000, 16384, 6, 17
    fs1 = fs // d1
    rng = np.random.default_rng(60 + len(stimulus))
    dyadic = stimulus == "dyadic"
    fmt = "cu8" if dyadic else "cs16"
    rig = Rig(pkg, monkeypatch, fs, max_in, fmt, depth=SLOTS)
    sbs = [rig.add_subband(d1, dyadic_stage_a(rng, d1, T1), 0, True) for _ in range(8)]  # tiled
    cls_members = []
    for s, l2, d2, T2, n in CLASSES:
        ms = []
        for _ in range(n):
            if dyadic:
                ms.append(rig.add_member(sbs[s], l2, d2, dyadic_member(rng, sbs[s].taps1, T2, fmt), 0, True))
            else:
                ms.append(rig.add_member(sbs[s], l2, d2, *real_row_member(rng, l2, T2, fs1), False))
        cls_members.append(ms)
    assert len(rig.mems) == 238 and sum(n for _, l2, _, _, n in CLASSES if l2 == 1) % 32 != 0
    sizes = pilot_sizes(d1, max_in, CLASSES[PILOT_INT], CLASSES[PILOT_RAT], rng)
    for n in sizes:
        rig.submit(exact_input(rng, fmt, n) if dyadic else real_grid_input(rng, n))
    rig.check()
    stage_a_kinds_ok(rig, "tiled")

    # the edges, from the test's own bookkeeping: per class and block its n2 (a rational class: the count of
    # residue 0), and per CTA tile of that count its window start parity and whether the window straddles the
    # ring's wrap (the capacity formula of rebuild_subbands)
    n2s, residues, parities, wraps = set(), set(), set(), 0
    for (s, l2, d2, T2, _), ms in zip(CLASSES, cls_members):
        back = max((t2 - 1) if l2_ == 1 else -(-(t2 - 1) // l2_) + 1 for (s_, l2_, _, t2, _) in CLASSES if s_ == s)
        cap = next_pow2(back + (SLOTS + 1) * (max_in // 2 // d1 + 2))
        Tb = -(-T2 // l2)
        K = 0  # outputs before the block
        for n2 in (y.size for y in ms[0].got):
            w = K * d2 - (T2 - 1)  # upsampled window start of the block's output 0 (the class attached at 0)
            if l2 == 1:
                n2s.add(n2)
                n0, count = w, n2
            else:
                residues.add(-(-n2 // l2))
                n0, count = -((-w) // l2), -(-n2 // l2)  # residue 0: n0 = (w + r) / L2
            for k0 in range(0, count, SB_KO):
                w0 = n0 + k0 * d2
                shift = w0 & 1
                parities.add(shift)
                need = ((min(SB_KO, count - k0) - 1) * d2 + Tb + shift + 1) & ~1
                wraps += ((w0 - shift) & (cap - 1)) + need > cap
            K += n2
    assert set(N2_TARGETS) <= n2s, sorted(n2s)
    assert set(RESIDUE_TARGETS) & residues, sorted(residues)
    assert parities == {0, 1} and wraps > 0, (parities, wraps)
    rig.close()


# ---------------------------------------------------------------------------
# D. churn, exactly
# ---------------------------------------------------------------------------
def test_churn_exactly(pkg, monkeypatch):
    """With tickets in flight: members attached while the ring holds older samples; two same-shape members
    attached at different blocks (separate classes) merged by a later re-layout once settled; a longer member
    that grows the ring; a member removed and attached again; a sub-band removed and a new one taking its id,
    which starts from zeros.  A dyadic sub-band and a one-hot one at centre 312345 on a real input."""
    fs, max_in, d1 = 2016000, 8192, 6
    fs1 = fs // d1
    rng = np.random.default_rng(77)
    reserve = 60 * (max_in // 2 // d1 + 8) + 8 * (max_in // 2 // d1 + 8)
    rig = Rig(pkg, monkeypatch, fs, max_in, "cs16", depth=SLOTS, reserve=reserve)
    a = rig.add_subband(d1, dyadic_stage_a(rng, d1, 17), 0, True)
    bsb = rig.add_subband(d1, one_hot_taps(17, 4, 0.75), 312345, False)
    for _ in range(6):
        rig.add_subband(d1, dyadic_stage_a(rng, d1, 17), 0, True)  # the sub-bands' tiled class
    t23 = dyadic_member(rng, a.taps1, 23, "cs16")
    rig.add_member(a, 1, 5, t23, 0, True)
    for _ in range(3):
        rig.add_member(bsb, 1, 5, *one_hot_member(rng, 1, 23, fs1, True), False)
    late, long_m, again = [], None, None
    ring0 = next_pow2(22 + (SLOTS + 1) * (max_in // 2 // d1 + 2))
    for blk in range(48):
        if blk == 3:
            late.append(rig.add_member(a, 1, 5, dyadic_member(rng, a.taps1, 23, "cs16"), 0, True))
            late.append(rig.add_member(a, 3, 7, dyadic_member(rng, a.taps1, 40, "cs16"), 0, True))
            rig.add_member(bsb, 1, 5, *one_hot_member(rng, 1, 23, fs1, True), False)
        if blk == 5:
            late.append(rig.add_member(a, 1, 5, dyadic_member(rng, a.taps1, 23, "cs16"), 0, True))
            rig.add_member(bsb, 3, 7, *one_hot_member(rng, 3, 40, fs1, False), False)
        if blk == 12:  # a re-layout after both have settled: the two classes of (5, 23) merge
            rig.add_member(a, 1, 7, dyadic_member(rng, a.taps1, 21, "cs16"), 0, True)
        if blk == 15:  # grows a's ring: later windows of the others span samples copied into the new ring
            long_m = rig.add_member(a, 1, 5, dyadic_member(rng, a.taps1, 1200, "cs16"), 0, True)
        if blk == 18:
            rig.remove_member(late[0])
        if blk == 20:
            again = rig.add_member(a, 1, 5, late[0].taps2, 0, True)
        if blk == 26:
            for m in [m for m in rig.mems if m.sb is bsb and m.last is None]:
                rig.remove_member(m)
            rig.remove_subband(bsb)
            c = rig.add_subband(d1, one_hot_taps(17, 9, -0.625), -251001, False)
            assert c.sid == bsb.sid  # the id is reused; the new sub-band starts from zeros
            for _ in range(3):
                rig.add_member(c, 1, 5, *one_hot_member(rng, 1, 23, fs1, True), False)
            rig.add_member(c, 2, 5, *one_hot_member(rng, 2, 33, fs1, False), False)
        rig.submit(real_grid_input(rng, max_in if blk % 3 else max_in - 2 * (blk % 5) - 2))
    rig.check()
    stage_a_kinds_ok(rig, "tiled")
    assert 1200 - 1 + (SLOTS + 1) * (max_in // 2 // d1 + 2) > ring0  # the long member grew the ring
    assert len(again.got) == 28 and len(long_m.got) == 33 and late[0].last == 18
    rig.close()


# ---------------------------------------------------------------------------
# E. randomised mixed populations
# ---------------------------------------------------------------------------
E_INT = [(5, 23), (4, 8), (7, 21), (2, 9), (1, 1), (3, 13)]
E_RAT = [(3, 7, 40), (2, 5, 33), (12, 5, 60), (4, 6, 50), (2, 1, 9)]
E_VARIANTS = ["no_renorm", "out_device", "host_ring", "sm_partition"]


def e_class(rng, rig, sb, real, fs1):
    """A class of 1..20 members of one random shape on sub-band sb."""
    if rng.integers(0, 2):
        l2, (d2, T2) = 1, E_INT[int(rng.integers(0, len(E_INT)))]
    else:
        l2, d2, T2 = E_RAT[int(rng.integers(0, len(E_RAT)))]
    for _ in range(int(rng.integers(1, 21))):
        if not sb.dyadic:
            rig.add_member(sb, l2, d2, *one_hot_member(rng, l2, T2, fs1, bool(rng.integers(0, 2))), False)
        elif real and rng.integers(0, 2):
            rig.add_member(sb, l2, d2, *real_row_member(rng, l2, T2, fs1), False)
        else:
            rig.add_member(sb, l2, d2, dyadic_member(rng, sb.taps1, T2, rig.fmt), 0, True)


def e_neighbour(rng, fmt):
    k = int(rng.integers(0, 3))
    if k == 0:
        D, T = [(42, 505), (8, 97), (5, 40)][int(rng.integers(0, 3))]
        return ("i", D, dyadic_taps(rng, T, fmt))
    if k == 1:
        L, M, T = [(3, 128, 97), (5, 3, 40)][int(rng.integers(0, 2))]
        return ("r", L, M, dyadic_taps(rng, T, fmt))
    return ("c", 6, small_taps(rng, 17, 3), 5, small_taps(rng, 23, 3))


@pytest.mark.parametrize("seed", range(12))
def test_random_mixed_populations(pkg, monkeypatch, seed):
    rng = np.random.default_rng(5000 + seed)
    fs = int(rng.choice([2016000, 2400000, 3000000]))
    max_in = int(rng.choice([8192, 16384, 32768]))
    case = ["generic", "tiled", "long"][int(rng.integers(0, 3))]
    d1, T1, n_sb, generic = STAGE_A[case]
    if case == "long":
        max_in *= 4
    real = bool(rng.integers(0, 2))  # a real cs16 input: one-hot sub-bands at any centre beside dyadic ones
    fmt = "cs16" if real else str(rng.choice(["cu8", "cs8", "cs16"]))
    fs1 = fs // d1
    variant = E_VARIANTS[seed % len(E_VARIANTS)]
    flags, env, host_ring = pkg.XLG_FORCE_GENERIC if generic else 0, None, 0
    if variant == "sm_partition":
        flags, env = flags | pkg.XLG_SM_PARTITION, {"XLATING_B200_PARTITION": "1"}
    elif variant == "no_renorm":
        flags |= pkg.XLG_NO_RENORM
    elif variant == "out_device":
        flags |= pkg.XLG_OUT_DEVICE
    else:
        host_ring = 12
    depth = int(rng.integers(1, SLOTS + 1))
    row = max_in // 2 // d1 + 8  # up to 220 members of at most 12/5 of a row each, sub-bands, neighbours
    reserve = 600 * row + n_sb * row + 8 * (max_in // 2 + 8)
    rig = Rig(pkg, monkeypatch, fs, max_in, fmt, flags=flags, host_ring=host_ring, depth=depth, env=env,
              reserve=reserve)
    for _ in range(int(rng.integers(1, 4))):
        rig.add_neighbour(e_neighbour(rng, fmt))
    sbs = []
    for i in range(n_sb):
        if real and i % 2:
            sbs.append(rig.add_subband(d1, one_hot_taps(T1, int(rng.integers(0, T1)), 0.75),
                                       int(rng.integers(-fs // 2 + 1, fs // 2)), False))
        else:
            sbs.append(rig.add_subband(d1, dyadic_stage_a(rng, d1, T1), 0, True))
    for sb in sbs[:3]:
        for _ in range(int(rng.integers(1, 4))):
            e_class(rng, rig, sb, real, fs1)
    choices = [max_in, max_in, max_in - 2, 0, 2, 7, int(rng.integers(1, max_in // 2)) * 2 + 1]
    b1, b2 = sorted(rng.choice(np.arange(2, 13), 2, replace=False).tolist())
    for b in range(14):
        if b in (b1, b2):
            live = [m for m in rig.mems if m.last is None]
            for i in (rng.choice(len(live), min(len(live), int(rng.integers(1, 4))), replace=False) if live else []):
                rig.remove_member(live[i])
            e_class(rng, rig, sbs[int(rng.integers(0, min(3, n_sb)))], real, fs1)
            if rng.integers(0, 2):
                rig.add_neighbour(e_neighbour(rng, fmt))
        n = int(rng.choice(choices))
        rig.submit(real_grid_input(rng, n) if real else exact_input(rng, fmt, n))
    rig.check()
    stage_a_kinds_ok(rig, case)
    rig.close()
