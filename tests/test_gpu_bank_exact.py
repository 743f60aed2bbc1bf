"""Members of bank channels bit for bit on random taps and input: the bank kernel's rows chained into the
member kernels (bank_member_model, tests/bank_exact.py) predicts every member output exactly, at any offset,
for integer and rational members, in banks wider than one channel group and above 256 threads, at frame,
ring and parity edges, with tickets in flight in every pipeline variant, through churn and in randomised mixed
populations.  Members of channels with a copy member from their first block are also checked against
member_model fed the GPU's own rows of that channel (tests/subband_rig.py), so a failure names its stage.

Every member is asserted to be kind 6 (xlg_client_info) on a kind-7 channel (xlg_subband_info).
"""
import errno

import numpy as np
import pytest

from bank_exact import BK_CG, XLG_SLOTS, bank_ctas, bank_walk, ring_cap
from cascade import small_taps
from exact import dyadic_taps, exact_input
from subband_rig import BANK, Rig, dyadic_member, dyadic_stage_a, one_hot_member
from util import rand_block

pytestmark = pytest.mark.gpu

FMTS = ("cu8", "cs8", "cs16")


def rand_taps(rng, T):
    return (rng.standard_normal(T) / np.sqrt(T)).astype(np.float32)


def bound_taps(pkg, d1):
    t = 1
    while pkg.bank_fits(d1, 2 * t):
        t *= 2
    lo, hi = t, 2 * t
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if pkg.bank_fits(d1, mid) else (lo, mid)
    return lo


def refused(fn, *args):
    with pytest.raises(ValueError) as e:
        fn(*args)
    assert e.value.args[0] == -errno.EINVAL


def row(max_in, d1):
    return max_in // 2 // d1 + 8


def banks_ok(rig):
    assert rig.kinds() == {BANK}, rig.kinds()


# ---------------------------------------------------------------------------
# 1. members at any offset
# ---------------------------------------------------------------------------
INT_SHAPES = [(5, 23), (4, 8), (1, 1), (6, 40), (2, 31), (3, 250)]  # (D2, T2): odd/even D2, T2 = 1, < 32, long
RAT_SHAPES = [(2, 5, 33), (3, 7, 40), (12, 5, 60)]                 # (L2, M2, T2)
RAGGED = [16384, 16384, 4005, 0, 7, 16382, 16384, 333, 16384, 16384, 16384, 9001, 16384, 16384]


@pytest.mark.parametrize("fmt", FMTS)
def test_members_at_any_offset(pkg, monkeypatch, fmt):
    """Channels -D1, 0, D1 - 1 from block 0 and an odd and an even one materialised at block 2; integer
    members with odd and even D2, T2 = 1, T2 < 32, long, and at the member shared-memory bound (one tap past
    it refused); rational L2 = 2, 3, 12; offsets 0, +-fs1/4 and arbitrary; attached at the channel's first
    block and at block 5."""
    rng = np.random.default_rng(100 + FMTS.index(fmt))
    fs, max_in, d1 = 2016000, 16384, 7
    fs1 = fs // d1
    offsets = [0, fs1 // 4, -fs1 // 4, int(rng.integers(-fs1 // 2, fs1 // 2))]
    assert pkg.subband_member_fits(1, 40, 1356) and not pkg.subband_member_fits(1, 40, 1357)
    rig = Rig(pkg, monkeypatch, fs, max_in, fmt, depth=XLG_SLOTS, reserve=400 * row(max_in, d1))
    bk = rig.add_bank(d1, rand_taps(rng, 61))

    def attach(sb, n):
        shapes = [(1, d2, T2) for d2, T2 in INT_SHAPES] + RAT_SHAPES
        for i, (l2, d2, T2) in enumerate(shapes[:n]):
            rig.add_member(sb, l2, d2, rand_taps(rng, T2), offsets[(i + sb.chan) % 4], False)

    chans = {}
    for b, n in enumerate(RAGGED):
        if b == 0:
            for k in (-d1, 0, d1 - 1):
                chans[k] = rig.add_channel(bk, k, copy=True)
                attach(chans[k], 9)
            rig.add_member(chans[0], 1, 40, rand_taps(rng, 1356), offsets[3], False)
            refused(rig.g.add_client_subband, chans[0].sid, 40, np.ones(1357, np.float32), 0)
        if b == 2:
            for k in (3, -2):  # materialised after the bank: its rows from here
                chans[k] = rig.add_channel(bk, k, copy=True)
                attach(chans[k], 9)
        if b == 5:
            for k in (-d1, 3):
                attach(chans[k], 9)
        rig.submit(rand_block(rng, fmt, n))
    rig.check()
    banks_ok(rig)
    for m in rig.mems:
        assert np.count_nonzero(np.concatenate(m.got)) > 0, m.label()
    rig.close()


# ---------------------------------------------------------------------------
# 2. banks wider than one channel group
# ---------------------------------------------------------------------------
def picks(table):
    """First, middle and last channel of every group of BK_CG in table order."""
    out = []
    for g0 in range(0, len(table), BK_CG):
        grp = table[g0:g0 + BK_CG]
        out += [grp[0], grp[len(grp) // 2], grp[-1]]
    return list(dict.fromkeys(out))


@pytest.mark.parametrize("d1", [17, 32, 64])
def test_banks_wider_than_one_channel_group(pkg, monkeypatch, d1):
    """Every channel materialised in a shuffled order; copies on the first, middle and last channel of every
    group of 32 in table order, plus a member on each; then channels from the middle of the table removed and
    added again in reverse order (they take the freed slots: the table no longer follows k and other channels
    share each CTA), and the new picks checked too."""
    rng = np.random.default_rng(d1)
    fs, max_in = 2 * d1 * 48000, 8192
    fs1 = fs // d1
    K = 2 * d1
    rig = Rig(pkg, monkeypatch, fs, max_in, "cs16", depth=XLG_SLOTS, reserve=(8 * K + 64) * row(max_in, d1))
    bk = rig.add_bank(d1, rand_taps(rng, 3 * K + 5))
    order = rng.permutation(np.arange(-d1, d1)).tolist()
    sizes = [8192, 8192, 2005, 8190, 8192, 0, 8192, 333, 8192, 8192, 8192]
    for b, n in enumerate(sizes):
        if b == 0:
            sbs = {k: rig.add_channel(bk, k) for k in order}
            first = picks(rig.channel_table(bk))
            assert len(first) >= 3 * (K // BK_CG) and sbs[order[-1]] in rig.channel_table(bk)[-1:]
            for sb in first:
                sb.copy = rig.add_member(sb, 1, 1, np.ones(1, np.float32), 0, False)
                rig.add_member(sb, 1, 5, rand_taps(rng, 23), int(rng.integers(-fs1 // 2, fs1 // 2)), False)
        if b == 5:
            table = rig.channel_table(bk)
            mid = [sb for sb in table[K // 2 - 6:K // 2 + 6] if sb.copy is None][:6]
            for sb in mid:
                rig.remove_subband(sb)
            for sb in mid[::-1]:
                sbs[sb.chan] = rig.add_channel(bk, sb.chan)
            table = rig.channel_table(bk)
            assert [sb.chan for sb in table] != sorted(sb.chan for sb in table)
            for sb in picks(table):
                if sb.copy is None:
                    sb.copy = rig.add_member(sb, 1, 1, np.ones(1, np.float32), 0, False)
                    rig.add_member(sb, 3, 7, rand_taps(rng, 40), int(rng.integers(-fs1 // 2, fs1 // 2)), False)
        rig.submit(rand_block(rng, "cs16", n))
    assert len(rig.channel_table(bk)) == K
    rig.check()
    banks_ok(rig)
    rig.close()


# ---------------------------------------------------------------------------
# 3. K > 256 threads
# ---------------------------------------------------------------------------
BIG = {129: 8666, 200: 4000, 260: 85}  # bank_fits' bounds at fs = 2 * D1 * 48000


@pytest.mark.parametrize("d1,case", [(129, "short"), (129, "K"), (129, "bound"), (200, "short"), (200, "K"),
                                     (200, "bound"), (260, "short"), (260, "bound")])
def test_more_channels_than_threads(pkg, monkeypatch, d1, case):
    """K = 2 D1 > 256: the twiddle staging and both phase loops stride past 256 threads; at D1 = 260 the
    bound (85 taps) is below K, so phase 2 walks part of each twiddle row.  One tap past the bound is refused."""
    assert bound_taps(pkg, d1) == BIG[d1]
    K = 2 * d1
    T1 = {"short": 37, "K": K, "bound": BIG[d1]}[case]
    rng = np.random.default_rng(d1 + T1)
    fs = 2 * d1 * 48000
    fs1 = fs // d1
    max_in = 2 * (T1 + 8192)
    rig = Rig(pkg, monkeypatch, fs, max_in, "cs8", depth=XLG_SLOTS, reserve=64 * row(max_in, d1))
    refused(rig.g.add_bank, d1, np.ones(BIG[d1] + 1, np.float32))
    bk = rig.add_bank(d1, rand_taps(rng, T1))
    chans = [-d1, 0, d1 - 1, 1, int(rng.integers(-d1, d1))]
    for k in dict.fromkeys(chans):
        sb = rig.add_channel(bk, k, copy=True)
        rig.add_member(sb, 1, 4, rand_taps(rng, 23), int(rng.integers(-fs1 // 2, fs1 // 2)), False)
        rig.add_member(sb, 2, 5, rand_taps(rng, 33), fs1 // 4, False)
    for n in [max_in, max_in // 2 + 1, 7, max_in, max_in - 2]:
        rig.submit(rand_block(rng, "cs8", n))
    rig.check()
    banks_ok(rig)
    rig.close()


def test_widest_bank_is_the_kernel_bound(pkg):
    """D1 = 260 at T1 = 1 is accepted and D1 = 261 refused by shared memory alone (2 * 261 divides fs)."""
    assert pkg.bank_fits(260, 1) and not pkg.bank_fits(261, 1)
    g = pkg.Group(2 * 261 * 260 * 4000, 8192)
    try:
        g.add_bank(260, np.ones(1, np.float32))
        refused(g.add_bank, 261, np.ones(1, np.float32))
    finally:
        g.close()


# ---------------------------------------------------------------------------
# 4. frame and ring edges
# ---------------------------------------------------------------------------
N1_TARGETS = [0, 1, 31, 32, 33, 64, 65]


def edge_sizes(rng, max_in, d1, T1, lead):
    """Raw block sizes (from the first bank's attach) making its n1 every N1_TARGETS value, with full and
    random odd blocks between them so that the ring wraps at both window parities."""
    plan = list(N1_TARGETS)
    rng.shuffle(plan)
    sizes = list(lead)
    for target in plan:
        for _ in range(int(rng.integers(2, 5))):
            sizes.append(max_in if rng.integers(0, 2) else int(rng.integers(1, max_in // 2)) * 2 + 1)
        counts = np.array([bank_walk([s // 2 for s in sizes] + [n], T1, d1)[0][-1] for n in range(max_in // 2 + 1)])
        sizes.append(2 * int(rng.choice(np.nonzero(counts == target)[0])))
    return sizes


def test_frame_and_ring_edges(pkg, monkeypatch):
    """Bank A (D1 = 7, T1 = 300 > 32 D1) attached at an even P, bank B (D1 = 4, T1 = 45) at an odd P: A's n1
    takes 0, 1, 31, 32, 33, 64 and 65; the test's bookkeeping (bank_ctas) confirms split windows at both
    parities and a CTA with x > 0 that zeroed samples before P."""
    rng = np.random.default_rng(43)  # (a plan that splits windows at both parities)
    fs, max_in, fmt = 2016000, 8192, "cu8"
    sizes = edge_sizes(rng, max_in, 7, 300, [])
    at_b = next(b for b in range(1, len(sizes)) if sum(n // 2 for n in sizes[:b]) % 2 == 1)
    rig = Rig(pkg, monkeypatch, fs, max_in, fmt, depth=XLG_SLOTS, reserve=64 * row(max_in, 4))
    for b, n in enumerate(sizes):
        if b == 0:
            a = rig.add_bank(7, rand_taps(rng, 300))
            for k in (-7, 3, 6):
                sb = rig.add_channel(a, k, copy=True)
                rig.add_member(sb, 1, 6, rand_taps(rng, 40), 12345, False)
        if b == at_b:
            bb = rig.add_bank(4, rand_taps(rng, 45))
            for k in (-4, 1):
                sb = rig.add_channel(bb, k, copy=True)
                rig.add_member(sb, 3, 7, rand_taps(rng, 40), -20000, False)
        rig.submit(rand_block(rng, fmt, n))
    rig.check()
    banks_ok(rig)
    rig.close()
    S = [n // 2 for n in sizes]
    cap = ring_cap(max_in, 299)
    seen_n1 = set(bank_walk(S, 300, 7)[0])
    assert set(N1_TARGETS) <= seen_n1, sorted(seen_n1)
    splits, pre_x = set(), False
    for (T1, d1, at) in ((300, 7, 0), (45, 4, at_b)):
        for ctas in bank_ctas(S[at:], T1, d1, sum(S[:at]), cap):
            for x, (_, shift, _, split, pre) in enumerate(ctas):
                if split:
                    splits.add(shift)
                pre_x |= pre and x > 0
    assert splits == {0, 1} and pre_x, (splits, pre_x)


# ---------------------------------------------------------------------------
# 5. tickets in flight, every pipeline variant
# ---------------------------------------------------------------------------
PIPE = {"default": ({}, None, 0), "conv_on_compute_stream": ({"XLATING_B200_CONV_STREAM": "0"}, None, 0),
        "no_spec_1stream": ({"XLATING_B200_SPECULATE": "0", "XLATING_B200_CSTREAMS": "1"}, None, 0),
        "partition": ({"XLATING_B200_PARTITION": "1"}, None, 0),
        "no_partition": ({"XLATING_B200_PARTITION": "0"}, None, 0),
        "sm_partition": ({"XLATING_B200_PARTITION": "1"}, "XLG_SM_PARTITION", 0),
        "out_device": ({}, "XLG_OUT_DEVICE", 0), "host_ring": ({}, None, 12)}


@pytest.mark.parametrize("group", ["bank_only", "beside_clients", "switching"])
@pytest.mark.parametrize("variant", list(PIPE))
def test_tickets_in_flight(pkg, monkeypatch, variant, group):
    """A bank-only group (no pre-pass), a bank beside dyadic integer clients (the speculative pre-pass runs),
    and a group that loses its last integer client and gains it back with tickets in flight."""
    env, flag, host_ring = PIPE[variant]
    rng = np.random.default_rng(sum(map(ord, variant + group)))
    fs, max_in, fmt = 2016000, 16384, "cs8"
    fs1 = fs // 7
    depth = host_ring or XLG_SLOTS
    rig = Rig(pkg, monkeypatch, fs, max_in, fmt, flags=getattr(pkg, flag) if flag else 0, host_ring=host_ring,
              depth=depth, env=env, reserve=64 * row(max_in, 7))
    bk = rig.add_bank(7, rand_taps(rng, 61))
    for k in (-7, 2, 5):
        sb = rig.add_channel(bk, k, copy=True)
        rig.add_member(sb, 1, 5, rand_taps(rng, 23), int(rng.integers(-fs1 // 2, fs1 // 2)), False)
        rig.add_member(sb, 3, 7, rand_taps(rng, 40), fs1 // 4, False)
    specs = [("i", 42, dyadic_taps(rng, 505, fmt)), ("i", 8, dyadic_taps(rng, 97, fmt))]
    nbs = {"bank_only": [], "beside_clients": specs, "switching": specs[1:]}[group]
    nbs = [rig.add_neighbour(s) for s in nbs]
    sizes = [max_in] * 5 + [15001, max_in, max_in, 12347, max_in, max_in, max_in - 2, max_in, max_in]
    for b, n in enumerate(sizes):
        if group == "switching" and b == 5:
            rig.remove_neighbour(nbs.pop())  # no pre-pass from here ...
        if group == "switching" and b == 9:
            nbs.append(rig.add_neighbour(specs[1]))  # ... and one again
        rig.submit(exact_input(rng, fmt, n))
    rig.check()
    banks_ok(rig)
    rig.close()


# ---------------------------------------------------------------------------
# 6. churn in flight
# ---------------------------------------------------------------------------
def test_churn_in_flight(pkg, monkeypatch):
    """With tickets in flight: channels and members added and removed, a bank removed and its id reused, and
    a bank longer than the ring's history (12300 taps) that grows the input ring, keeping its samples."""
    rng = np.random.default_rng(66)
    fs, max_in, fmt = 2016000, 8192, "cs16"
    fs1 = fs // 7
    rig = Rig(pkg, monkeypatch, fs, max_in, fmt, depth=XLG_SLOTS, reserve=200 * row(max_in, 4))
    a = rig.add_bank(7, rand_taps(rng, 33))
    ch = {k: rig.add_channel(a, k, copy=True) for k in (-7, 2)}
    tmp = rig.add_channel(a, 5, copy=True)
    m_a = rig.add_member(ch[2], 1, 4, rand_taps(rng, 8), 5000, False)
    b2 = long_b = None
    assert ring_cap(max_in, 12299) > ring_cap(max_in, 4096)
    for blk in range(24):
        if blk == 2:
            rig.remove_member(tmp.copy)
            rig.remove_subband(tmp)
            b2 = rig.add_bank(4, rand_taps(rng, 40))
            sb = rig.add_channel(b2, 1, copy=True)
            rig.add_member(sb, 2, 5, rand_taps(rng, 33), -(fs // 4) // 4, False)  # -fs1 / 4 of that bank
        if blk == 4:
            rig.remove_member(m_a)
            rig.add_member(ch[-7], 1, 5, rand_taps(rng, 23), 777, False)
            rig.add_channel(a, 5, copy=True)  # the same channel again: rows from here
        if blk == 7:
            for m in [m for m in rig.mems if m.sb.bank is b2 and m.last is None]:
                rig.remove_member(m)
            for sb in [sb for sb in rig.sbs if sb.bank is b2 and sb.last is None]:
                rig.remove_subband(sb)
            rig.remove_bank(b2)
            b3 = rig.add_bank(4, rand_taps(rng, 41))
            assert b3.bid == b2.bid  # the id is reused; the new bank starts from P
            sb = rig.add_channel(b3, -4, copy=True)
            rig.add_member(sb, 1, 3, rand_taps(rng, 9), 0, False)
        if blk == 10:  # grows the input ring: later windows span samples copied into the new ring
            long_b = rig.add_bank(32, rand_taps(rng, 12300))
            for k in (-32, 7):
                sb = rig.add_channel(long_b, k, copy=True)
                rig.add_member(sb, 1, 2, rand_taps(rng, 31), 1234, False)
        if blk == 14:
            rig.add_member(ch[2], 12, 5, rand_taps(rng, 60), fs1 // 5, False)
        rig.submit(rand_block(rng, fmt, max_in if blk % 3 else max_in - 2 * (blk % 5) - 3))
    rig.check()
    banks_ok(rig)
    assert long_b.first == 10
    rig.close()


# ---------------------------------------------------------------------------
# 7. randomised mixed populations
# ---------------------------------------------------------------------------
MIX_VARIANTS = ["default", "no_renorm", "out_device", "host_ring", "sm_partition", "no_spec_1stream"]
MIX_D1 = [3, 4, 5, 6, 7, 8, 10, 12, 16, 20, 21, 24, 28, 32]  # 2 D1 divides 2016000


def mix_neighbour(rng, fmt):
    k = int(rng.integers(0, 3))
    if k == 0:
        D, T = [(42, 505), (8, 97), (5, 40)][int(rng.integers(0, 3))]
        return ("i", D, dyadic_taps(rng, T, fmt))
    if k == 1:
        L, M, T = [(3, 128, 97), (5, 3, 40)][int(rng.integers(0, 2))]
        return ("r", L, M, dyadic_taps(rng, T, fmt))
    return ("c", 6, small_taps(rng, 17, 3), 5, small_taps(rng, 23, 3))


def mix_member(rng, rig, sb):
    fs1 = rig.fs // sb.d1
    if sb.bank is None:  # an ordinary dyadic sub-band: the sub-band suite's exact stimuli
        if rng.integers(0, 2):
            l2, d2, T2 = 1, *[(5, 23), (4, 8), (1, 1)][int(rng.integers(0, 3))]
            return rig.add_member(sb, l2, d2, dyadic_member(rng, sb.taps1, T2, rig.fmt), 0, True)
        l2, d2, T2 = [(3, 7, 40), (2, 5, 33)][int(rng.integers(0, 2))]
        return rig.add_member(sb, l2, d2, *one_hot_member(rng, l2, T2, fs1, False), False)
    l2, d2, T2 = [(1, 5, 23), (1, 4, 8), (1, 1, 1), (1, 7, 90), (2, 5, 33), (3, 7, 40), (12, 5, 60)][
        int(rng.integers(0, 7))]
    return rig.add_member(sb, l2, d2, rand_taps(rng, T2), int(rng.integers(-fs1 // 2, fs1 // 2)), False)


@pytest.mark.parametrize("seed", range(12))
def test_random_mixed_populations(pkg, monkeypatch, seed):
    rng = np.random.default_rng(9000 + seed)
    fs = 2016000
    max_in = int(rng.choice([8192, 16384]))
    fmt = str(rng.choice(FMTS))
    variant = MIX_VARIANTS[seed % len(MIX_VARIANTS)]
    flags, env, host_ring = 0, None, 0
    if variant == "sm_partition":
        flags, env = pkg.XLG_SM_PARTITION, {"XLATING_B200_PARTITION": "1"}
    elif variant == "no_renorm":
        flags = pkg.XLG_NO_RENORM
    elif variant == "out_device":
        flags = pkg.XLG_OUT_DEVICE
    elif variant == "no_spec_1stream":
        env = {"XLATING_B200_SPECULATE": "0", "XLATING_B200_CSTREAMS": "1"}
    elif variant == "host_ring":
        host_ring = 12
    depth = int(rng.integers(1, XLG_SLOTS + 1))
    rig = Rig(pkg, monkeypatch, fs, max_in, fmt, flags=flags, host_ring=host_ring, depth=depth, env=env,
              reserve=1200 * row(max_in, 3))
    for _ in range(int(rng.integers(1, 4))):
        rig.add_neighbour(mix_neighbour(rng, fmt))
    chans = []
    for i in range(int(rng.integers(1, 4))):
        wide = i == 0 and seed % 2 == 0  # a bank of more than one channel group
        d1 = int(rng.choice([24, 28, 32] if wide else MIX_D1))
        T1 = int(rng.integers(1, min(400, bound_taps(pkg, d1)) + 1))
        bk = rig.add_bank(d1, rand_taps(rng, T1))
        n_ch = int(rng.integers(BK_CG + 1 if wide else 1, 2 * d1 + 1))
        for k in rng.choice(np.arange(-d1, d1), n_ch, replace=False).tolist():
            chans.append(rig.add_channel(bk, int(k), copy=bool(rng.integers(0, 4) == 0)))
    sbs = [rig.add_subband(6, dyadic_stage_a(rng, 6, 17), 0, True) for _ in range(int(rng.integers(1, 3)))]
    targets = chans + sbs
    for _ in range(int(rng.integers(4, 12))):
        mix_member(rng, rig, targets[int(rng.integers(0, len(targets)))])
    b1, b2 = sorted(rng.choice(np.arange(2, 12), 2, replace=False).tolist())
    choices = [max_in, max_in, max_in - 2, 0, 2, 7, int(rng.integers(1, max_in // 2)) * 2 + 1]
    for b in range(14):
        if b in (b1, b2):
            live = [m for m in rig.mems if m.last is None and m is not m.sb.copy]
            for i in (rng.choice(len(live), min(len(live), int(rng.integers(1, 3))), replace=False) if live else []):
                rig.remove_member(live[i])
            for _ in range(int(rng.integers(1, 4))):
                mix_member(rng, rig, targets[int(rng.integers(0, len(targets)))])
            if rng.integers(0, 2):
                rig.add_neighbour(mix_neighbour(rng, fmt))
        rig.submit(exact_input(rng, fmt, int(rng.choice(choices))))
    rig.check()
    assert BANK in rig.kinds()
    assert seed % 2 or len(rig.channel_table(rig.banks[0])) > BK_CG
    rig.close()
