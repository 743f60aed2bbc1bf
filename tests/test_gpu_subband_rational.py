"""Rational sub-band members (xlg_add_client_subband_rational) on the GPU.

A rational member is by definition the reference's float path with decimation M2 at L2 * fs / d1 and its own
centre, fed its sub-band's zero-stuffed outputs (include/xlating_group.h).  Exact stimuli -- a real input on
the exact grid, dyadic sub-band taps at centre 0 and branch-one-hot member taps at centres across the
sub-band -- must equal RationalSubbandOracle bit for bit, oscillators included; designed taps from
subband_plan are held to the 1e-5 contract.  Tests assert which kernel served each sub-band (xlg_subband_info).
"""
import ctypes as C
import errno
import math

import numpy as np
import pytest

from cascade import small_taps
from exact import one_hot_taps
from rational import branch_one_hot_taps, real_grid_input
from subband_rational import RationalSubbandOracle
from test_gpu_subband import GENERIC, LONG, SLOTS, TILED, Rig, add_neighbour, neighbour_specs
from util import rand_block

pytestmark = pytest.mark.gpu


class RatRig(Rig):
    """Rig whose members may resample: add_member takes interp2."""

    def add_subband(self, d1, t1, c1):
        self.flush()
        sid = self.g.add_subband(d1, t1, c1)
        self.orc[sid] = RationalSubbandOracle(d1, t1, c1, self.fs, self.max_in)
        return sid

    def add_member(self, sid, d2, t2, off, key=None, interp2=1):
        self.flush()
        cid = self.g.add_client_subband(sid, d2, t2, off, interp2=interp2)
        key = cid if key is None else key
        self.orc[sid].add_member(cid, d2, t2, off, interp2=interp2)
        self.of[cid] = sid
        self.want[key], self.got[key], self.kinds[key] = [], [], set()
        self.key = getattr(self, "key", {})
        self.key[cid] = key
        return cid


def centre(rng, fs1):
    return int(rng.integers(-fs1 // 2, fs1 // 2))


# (L2, M2, T2) of the lone rational members: L2 = 2, 3 and 12, gcd(L2, M2) > 1, odd and even M2; T2 >= M2,
# as in the integer tests (with M2 > T2 a window may start past the block, where the reference's history
# length would go negative)
LONE = [(2, 5, 33), (3, 8, 40), (12, 5, 120), (4, 6, 50), (2, 9, 10)]
CLASS = (3, 7, 40)  # 17 members: two groups of one class

# sub-band (D1, T1, taps bits), max_in, sub-bands, forced generic: every sub-band sum is exact,
# T1 * 128 * (2^bits - 1) < 2^24 on real_grid_input
EXACT = {
    "generic": (6, 17, 3, 8192, 2, True),
    "tiled": (6, 17, 3, 8192, 8, False),
    "long": (400, 800, 1, 65536, 8, False),
}


@pytest.mark.parametrize("case", list(EXACT))
def test_exact_stimuli_bit_for_bit(pkg, case):
    d1, T1, bits, max_in, n_sb, generic = EXACT[case]
    fs = 2016000
    fs1 = fs // d1
    rng = np.random.default_rng(20 + len(case))
    rig = RatRig(pkg, fs, max_in, "cs16", flags=pkg.XLG_FORCE_GENERIC if generic else 0, depth=SLOTS)
    sids = [rig.add_subband(d1, small_taps(rng, T1, bits), 0) for _ in range(n_sb)]
    l2, m2, t2 = CLASS
    for _ in range(17):
        rig.add_member(sids[0], m2, branch_one_hot_taps(rng, t2, l2), centre(rng, fs1), interp2=l2)
    for l2, m2, t2 in LONE:
        rig.add_member(sids[0], m2, branch_one_hot_taps(rng, t2, l2), centre(rng, fs1), interp2=l2)
    # integer members beside them, in the same sub-band and in another
    for sid in sids[:2]:
        for d2, t2 in [(5, 23), (5, 23), (2, 8)]:
            rig.add_member(sid, d2, one_hot_taps(t2, int(rng.integers(0, t2))), centre(rng, fs1))
    rig.add_member(sids[1], 7, branch_one_hot_taps(rng, 21, 2), centre(rng, fs1), interp2=2)
    sizes = [max_in, max_in, 1002, max_in, 7, 1, 0, max_in - 2, 2 * d1 * 41 + 1] + [max_in] * 8 + [333] * 8
    for n in sizes:
        rig.submit(real_grid_input(rng, n))
    rig.assert_exact()
    assert sum(y.size for y in rig.got[next(iter(rig.got))]) > 0
    want = {"generic": GENERIC, "tiled": TILED, "long": LONG}[case]
    for key, kinds in rig.kinds.items():
        assert want in kinds and kinds <= {GENERIC, want}, (key, kinds)
    rig.close()


def test_interp2_one_is_add_client_subband(pkg):
    """interp2 = 1 through the rational entry point is xlg_add_client_subband: the same bits and kinds."""
    fs, max_in, fmt = 2016000, 16384, "cu8"
    p = pkg.subband_plan(fs, [(-300000 + 50000 * k, 48000 if k % 2 else 96000) for k in range(12)])
    rng = np.random.default_rng(21)
    g = pkg.Group(fs, max_in)
    sids = [g.add_subband(p["d1"], p["taps1"], sb["center"]) for sb in p["subbands"]]
    pairs = []
    for m in p["members"]:
        a = g.add_client_subband(sids[m["subband"]], m["d2"], m["taps2"], m["offset"], interp2=1)
        t2 = np.ascontiguousarray(m["taps2"], dtype=np.float32)
        cid = C.c_int(-1)
        assert g._L.xlg_add_client_subband(g._h, sids[m["subband"]], m["d2"], t2.ctypes.data_as(C.POINTER(C.c_float)),
                                           t2.size, m["offset"], C.byref(cid)) == 0
        pairs.append((a, cid.value))
    for n in [max_in] * 8 + [7, 0, 333, max_in]:
        t = g.submit(fmt, rand_block(rng, fmt, n))
        g.wait(t)
        for a, b in pairs:
            assert np.array_equal(g.output(t, a).view(np.uint64), g.output(t, b).view(np.uint64))
            assert g.client_info(a) == g.client_info(b) and g.subband_info(a) == g.subband_info(b)
    g.close()


DESIGNED = {  # fs, format, clients, centre span, seed
    "2048k_cu8": (2048000, "cu8", 24, 300000, 3),
    "10M_cs16": (10000000, "cs16", 24, 400000, 4),
    "20M_cs8": (20000000, "cs8", 24, 400000, 5),
}


@pytest.mark.parametrize("name", list(DESIGNED))
def test_designed_taps_within_contract(pkg, name):
    """subband_plan's taps, 20 blocks, 1e-5 against RationalSubbandOracle; the plan's members resample, and it
    has a class of at least 8 members and a lone member."""
    fs, fmt, n, span, seed = DESIGNED[name]
    rng = np.random.default_rng(seed)
    centres = [int(c) for c in rng.integers(-span // 2, span // 2, n)]
    centres[-1] = fs // 3  # a lone member, far from the others
    p = pkg.subband_plan(fs, [(c, 48000) for c in centres])
    assert all(m["interp2"] > 1 for m in p["members"])
    max_in = 131072
    rig = RatRig(pkg, fs, max_in, fmt, depth=SLOTS)
    sids = [rig.add_subband(p["d1"], p["taps1"], sb["center"]) for sb in p["subbands"]]
    per = {}
    for m in p["members"]:
        rig.add_member(sids[m["subband"]], m["d2"], m["taps2"], m["offset"], interp2=m["interp2"])
        per.setdefault(m["subband"], []).append(m)
    assert max(len(v) for v in per.values()) >= 8 and min(len(v) for v in per.values()) == 1
    for _ in range(20):
        rig.submit(rand_block(rng, fmt, max_in))
    rig.assert_close()
    rig.close()


def test_churn(pkg):
    """A rational member attached mid-stream reads zeros before its attach point; a member removed and
    attached again; a longer rational member grows the ring with its samples kept; the ring wraps many
    times."""
    fs, max_in, d1 = 2048000, 4096, 10
    fs1 = fs // d1
    rng = np.random.default_rng(23)
    t1 = pkg.create_low_pass_filter(1.0, fs, fs1 // 2, fs1 // 2 - 40000)
    t2 = pkg.create_low_pass_filter(15.0, 15 * fs1, 24000, 9600)
    t_long = pkg.create_low_pass_filter(15.0, 15 * fs1, 24000, 2400)
    rig = RatRig(pkg, fs, max_in, "cu8", depth=SLOTS)
    a = rig.add_subband(d1, t1, -500000)
    base = [rig.add_member(a, 64, t2, off, interp2=15) for off in (-50000, -20000, 30000)]
    rig.add_member(a, 4, pkg.create_low_pass_filter(1.0, fs1, 25600, 10240), 11000)  # an integer member
    late = None
    for blk in range(90):
        if blk == 3:
            late = rig.add_member(a, 64, t2, 45000, interp2=15)
        if blk == 7:
            rig.remove_member(base[1])
        if blk == 9:
            rig.add_member(a, 64, t2, -20000, key="again", interp2=15)
        if blk == 12:
            rig.add_member(a, 64, t_long, 5000, key="long", interp2=15)
        rig.submit(rand_block(rng, "cu8", max_in if blk % 3 else max_in - 2 * (blk % 5) - 1))
    rig.assert_close()
    assert len(rig.got[late]) == 87 and len(rig.got["again"]) == 81 and len(rig.got["long"]) == 78
    n1 = max_in // 2 // d1
    ring = 1 << int(np.ceil(np.log2(-(-(t_long.size - 1) // 15) + 1 + (SLOTS + 1) * (n1 + 2))))
    assert 90 * n1 > 4 * ring  # the grown ring wrapped several times as well
    assert t_long.size > 2 * t2.size
    rig.close()


def test_profile_counts_branch_taps_and_one_row_per_subband(pkg):
    """member_macs = sum n2 * ceil(T2 / L2) over rational and integer members; row_samples counts each
    sub-band's samples once however many members it has."""
    fs, max_in, d1 = 2048000, 16384, 10
    fs1 = fs // d1
    rng = np.random.default_rng(25)
    t1 = pkg.create_low_pass_filter(1.0, fs, fs1 // 2, fs1 // 2 - 40000)
    t2 = pkg.create_low_pass_filter(15.0, 15 * fs1, 24000, 9600)
    t3 = pkg.create_low_pass_filter(1.0, fs1, 25600, 10240)
    rig = RatRig(pkg, fs, max_in, "cu8")
    sids = [rig.add_subband(d1, t1, c) for c in (100000, -400000)]
    for k in range(10):
        rig.add_member(sids[0], 64, t2, -60000 + 12000 * k, interp2=15)
    rig.add_member(sids[1], 64, t2, 3000, interp2=15)
    rig.add_member(sids[1], 4, t3, -3000)
    rig.submit(rand_block(rng, "cu8", max_in))
    rig.flush()
    rig.g.profile_enable(True)
    rig.g.subband_profile_read(reset=True)
    sizes = [max_in, 999, max_in, 0, max_in]
    for n in sizes:
        rig.submit(rand_block(rng, "cu8", n))
    rig.flush()
    sp = rig.g.subband_profile_read()
    rows = sum(y.size for s in sids for y in rig.orc[s].rows[1:])
    macs = 0
    for s in sids:
        for cid, m in rig.orc[s].members.items():
            l2 = rig.orc[s].interp.get(cid, 1)
            macs += sum(y.size for y in rig.got[rig.key[cid]][1:]) * -(-m.T // l2)
    assert sp["row_samples"] == rows
    assert sp["member_macs"] == macs
    assert sp["member_launches"] == len(sizes) and sp["member_ms"] > 0
    rig.close()


@pytest.mark.parametrize("host_ring", [0, 8])
def test_neighbours_keep_their_bits(pkg, host_ring):
    """Integer, rational and cascade clients, and integer members, give the same bits beside rational members
    as in a twin group without them, at pipeline depth XLG_SLOTS."""
    fs, max_in, fmt = 2016000, 16384, "cu8"
    rng = np.random.default_rng(27)
    specs = neighbour_specs(pkg, fs)
    plan = pkg.subband_plan(fs, [(-400000 + 37000 * k, 48000) for k in range(10)])
    fs1 = plan["fs1"]
    l2, m2 = 44100 // math.gcd(44100, fs1), fs1 // math.gcd(44100, fs1)  # 44.1 kHz members
    rat = pkg.create_low_pass_filter(float(l2), l2 * fs1, 22050, 8820)
    groups = []
    for with_rational in (False, True):
        g = pkg.Group(fs, max_in, host_ring=host_ring)
        ids = [add_neighbour(g, s) for s in specs]
        sids = [g.add_subband(plan["d1"], plan["taps1"], sb["center"]) for sb in plan["subbands"]]
        ids += [g.add_client_subband(sids[m["subband"]], m["d2"], m["taps2"], m["offset"]) for m in plan["members"]]
        if with_rational:
            for k in range(12):
                g.add_client_subband(sids[k % len(sids)], m2, rat, -30000 + 5000 * k, interp2=l2)
        groups.append((g, ids))
    blocks = [rand_block(rng, fmt, n) for n in [max_in] * 6 + [1001, 0, max_in, 64] + [max_in] * 6]
    pend = []
    for x in blocks:
        pend.append([g.submit(fmt, x) for g, _ in groups])
        while len(pend) >= SLOTS:
            ts = pend.pop(0)
            outs = []
            for (g, ids), t in zip(groups, ts):
                g.wait(t)
                outs.append([g.output(t, c) for c in ids])
            for a, b in zip(*outs):
                assert np.array_equal(a.view(np.uint64), b.view(np.uint64))
    for g, _ in groups:
        g.close()


def test_device_outputs_match_host_outputs(pkg):
    fs, max_in, fmt = 2048000, 16384, "cu8"
    plan = pkg.subband_plan(fs, [(-300000 + 50000 * k, 48000) for k in range(12)])
    got = []
    for flags in (0, pkg.XLG_OUT_DEVICE):
        rng = np.random.default_rng(29)
        rig = RatRig(pkg, fs, max_in, fmt, flags=flags, depth=SLOTS)
        sids = [rig.add_subband(plan["d1"], plan["taps1"], sb["center"]) for sb in plan["subbands"]]
        for m in plan["members"]:
            rig.add_member(sids[m["subband"]], m["d2"], m["taps2"], m["offset"], interp2=m["interp2"])
        for n in [max_in] * 5 + [77, max_in]:
            rig.submit(rand_block(rng, fmt, n))
        rig.assert_close()
        got.append([rig.got[k] for k in sorted(rig.got)])
        rig.close()
    for a, b in zip(*got):
        for y, z in zip(a, b):
            assert np.array_equal(y, z)


def test_refusals(pkg, capfd):
    """Each refusal returns its code, logs one <3> line and takes no ticket; the next cf32 submit continues
    bit for bit like a twin group that never saw the refused calls.  subband_member_fits agrees with the
    library on both sides of the shared-memory bound."""
    fs, max_in, fmt = 2016000, 8192, "cu8"
    fs1 = fs // 6
    rng = np.random.default_rng(31)
    t1 = pkg.create_low_pass_filter(1.0, fs, fs1 // 2, fs1 // 2 - 96000)
    t2 = pkg.create_low_pass_filter(21.0, 21 * fs1, 22050, 8820)  # 44.1 kHz: 21 / 160 of 336 kHz
    rigs = [RatRig(pkg, fs, max_in, fmt) for _ in range(2)]
    for r in rigs:
        sid = r.add_subband(6, t1, 250000)
        r.add_member(sid, 160, t2, 31000, interp2=21)
    x = rand_block(rng, fmt, max_in)
    for r in rigs:
        r.submit(x)
    capfd.readouterr()
    g = rigs[0].g
    empty = np.zeros(0, np.float32)
    big = np.ones(1505, np.float32)
    calls = [
        (-errno.EINVAL, lambda: g.add_client_subband(sid, 7, t2, 0, interp2=0)),
        (-errno.EINVAL, lambda: g.add_client_subband(sid, 7, t2, 0, interp2=2 ** 20)),  # 2^20 * 336000 Hz
        (-errno.EINVAL, lambda: g.add_client_subband(sid, 0, t2, 0, interp2=3)),
        (-errno.EINVAL, lambda: g.add_client_subband(sid, 7, empty, 0, interp2=3)),
        (-errno.EINVAL, lambda: g.add_client_subband(99, 7, t2, 0, interp2=3)),
        (-errno.EINVAL, lambda: g.add_client_subband(sid, 625, np.ones(3011, np.float32), 0, interp2=24)),
        (-errno.EINVAL, lambda: g.add_client_subband(sid, 373, big, 0, interp2=12)),
    ]
    for code, call in calls:
        with pytest.raises(ValueError) as e:
            call()
        assert e.value.args[0] == code
        assert capfd.readouterr().err.count("<3>") == 1
    assert g.client_count() == 1
    # the block bound: 2^21 x (2^21 / 2016 + 2) upsampled sub-band samples, at a rate that still fits
    wide = pkg.Group(fs, 1 << 22)
    s = wide.add_subband(2016, small_taps(rng, 5, 2), 0)
    with pytest.raises(ValueError) as e:
        wide.add_client_subband(s, 3, small_taps(rng, 9, 2), 0, interp2=1 << 21)
    assert e.value.args[0] == -errno.EINVAL
    assert capfd.readouterr().err.count("<3>") == 1
    assert wide.client_count() == 0
    wide.close()
    # the shared-memory bound from both sides, against subband_member_fits
    probe = pkg.Group(fs, max_in)
    ps = probe.add_subband(6, t1, 0)
    for l2, m2, n in [(12, 372, 1505), (12, 373, 1505), (1, 40, 1400), (1, 40, 1300), (24, 625, 3011)]:
        try:
            probe.add_client_subband(ps, m2, np.ones(n, np.float32), 0, interp2=l2)
            ok = True
        except ValueError as e:
            assert e.args[0] == -errno.EINVAL
            ok = False
        assert ok == pkg.subband_member_fits(l2, m2, n), (l2, m2, n)
    assert pkg.subband_member_fits(12, 372, 1505) and not pkg.subband_member_fits(12, 373, 1505)
    probe.close()
    capfd.readouterr()
    for _ in range(3):
        x = rand_block(rng, fmt, max_in)
        t = [r.submit(x) for r in rigs]
        assert t[0] == t[1]  # no ticket was taken
    for r in rigs:
        r.flush()
    for k in rigs[0].got:
        for y, z in zip(rigs[0].got[k], rigs[1].got[k]):
            assert np.array_equal(y, z)
    for r in rigs:
        r.assert_close()
        r.close()
