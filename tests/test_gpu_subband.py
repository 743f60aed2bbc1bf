"""Sub-band clients (xlg_add_subband, xlg_add_client_subband) on the GPU.

A member is by definition the reference's float path at fs / d1 with its own centre, fed its sub-band's
outputs (include/xlating_group.h).  Exact stimuli -- a real input on the exact grid, dyadic sub-band taps at
centre 0 and one-hot member taps at centres across the sub-band -- must equal SubbandOracle bit for bit,
oscillators included; designed taps from subband_plan are held to the 1e-5 contract.  Tests assert which
kernel served each sub-band (xlg_subband_info).
"""
import errno

import numpy as np
import pytest

from cascade import small_taps
from exact import one_hot_taps
from rational import real_grid_input
from subband import SubbandOracle
from util import assert_cf32_close, rand_block

pytestmark = pytest.mark.gpu

GENERIC, TILED, LONG, MEMBER = 0, 1, 2, 6
SLOTS = 4


class Rig:
    """One group with sub-bands and members beside the SubbandOracles of its sub-bands.  Outputs are read
    `depth` tickets late; attaching or removing first reads every pending ticket (a re-layout may grow the
    result arenas, which drops the tickets still in them)."""

    def __init__(self, pkg, fs, max_in, fmt, flags=0, host_ring=0, depth=1):
        self.pkg, self.fs, self.max_in, self.fmt, self.flags, self.depth = pkg, fs, max_in, fmt, flags, depth
        self.g = pkg.Group(fs, max_in, flags=flags, host_ring=host_ring)
        self.orc, self.of = {}, {}  # sub-band id -> SubbandOracle; member cid -> its sub-band id
        self.want, self.got, self.kinds = {}, {}, {}
        self.pending = []
        self.blocks = 0

    def add_subband(self, d1, t1, c1):
        self.flush()
        sid = self.g.add_subband(d1, t1, c1)
        self.orc[sid] = SubbandOracle(d1, t1, c1, self.fs, self.max_in)
        return sid

    def remove_subband(self, sid):
        self.flush()
        self.g.remove_subband(sid)
        del self.orc[sid]

    def add_member(self, sid, d2, t2, off, key=None):
        self.flush()
        cid = self.g.add_client_subband(sid, d2, t2, off)
        key = cid if key is None else key
        self.orc[sid].add_member(cid, d2, t2, off)
        self.of[cid] = sid
        self.want[key], self.got[key], self.kinds[key] = [], [], set()
        self.key = getattr(self, "key", {})
        self.key[cid] = key
        return cid

    def remove_member(self, cid):
        self.flush()
        self.g.remove_client(cid)
        self.orc[self.of.pop(cid)].remove_member(cid)
        del self.key[cid]

    def submit(self, x):
        t = self.g.submit(self.fmt, x)
        renorm = not (self.flags & self.pkg.XLG_NO_RENORM)
        for o in self.orc.values():
            for cid, y in o.process_cf32(self.fmt, x, renorm=renorm).items():
                self.want[self.key[cid]].append(y)
        self.pending.append((t, list(self.key.items())))
        self.blocks += 1
        while len(self.pending) >= self.depth:
            self.collect()
        return t

    def collect(self):
        t, members = self.pending.pop(0)
        self.g.wait(t)
        for cid, key in members:
            dev = self.flags & self.pkg.XLG_OUT_DEVICE
            self.got[key].append(self.g.read_output(t, cid) if dev else self.g.output(t, cid))
            if cid in self.of:
                assert self.g.client_info(cid)[1] == MEMBER
                sid, kind, _ = self.g.subband_info(cid)
                assert sid == self.of[cid]
                self.kinds[key].add(kind)

    def flush(self):
        while self.pending:
            self.collect()

    def assert_exact(self):
        self.flush()
        for key in self.want:
            assert len(self.got[key]) == len(self.want[key]), key
            for b, (y, r) in enumerate(zip(self.got[key], self.want[key])):
                assert y.shape == r.shape, (key, b)
                assert np.array_equal(y, r), (key, b, np.max(np.abs(y - r)))

    def assert_close(self):
        self.flush()
        for key in self.want:
            assert len(self.got[key]) == len(self.want[key]), key
            for b, (y, r) in enumerate(zip(self.got[key], self.want[key])):
                assert_cf32_close(y, r, f"member {key} block {b}")

    def close(self):
        self.flush()
        self.g.close()


def exact_members(rig, sid, rng, fs1, n_class, lone):
    """n_class one-hot members of one (D2, T2) -- one class -- and lone members of other shapes, at centres
    across the sub-band: each accumulator is one rounded product of an exact sub-band sample."""
    for _ in range(n_class):
        rig.add_member(sid, 5, one_hot_taps(23, int(rng.integers(0, 23))), int(rng.integers(-fs1 // 2, fs1 // 2)))
    for d2, t2 in lone:
        rig.add_member(sid, d2, one_hot_taps(t2, int(rng.integers(0, t2))), int(rng.integers(-fs1 // 2, fs1 // 2)))


# sub-band (D1, T1, taps bits), format, max_in, sub-bands, flags: every sub-band sum is exact, T1 * 128 *
# (2^bits - 1) < 2^24 on real_grid_input
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
    rng = np.random.default_rng(len(case))
    rig = Rig(pkg, fs, max_in, "cs16", flags=pkg.XLG_FORCE_GENERIC if generic else 0, depth=SLOTS)
    for s in range(n_sb):
        sid = rig.add_subband(d1, small_taps(rng, T1, bits), 0)
        if s < 2:
            lone = [(3, 9), (2, 8), (1, 1), (7, 7)] if d1 < 100 else [(3, 9), (2, 8)]
            exact_members(rig, sid, rng, fs1, 9 if s == 0 else 1, lone)
    sizes = [max_in, max_in, 1002, max_in, 7, 0, max_in - 2, 2 * d1 * 23 + 1] + [max_in] * 8 + [333] * 8
    for n in sizes:
        rig.submit(real_grid_input(rng, n))
    rig.assert_exact()
    want = {"generic": GENERIC, "tiled": TILED, "long": LONG}[case]
    for key, kinds in rig.kinds.items():
        assert want in kinds and kinds <= {GENERIC, want}, (key, kinds)
    rig.close()


DESIGNED = {  # fs, format, clients, centre span, seed
    "61M_cs16": (61440000, "cs16", 48, 2000000, 3),
    "2M_cu8": (2016000, "cu8", 80, 400000, 4),
}


@pytest.mark.parametrize("name", list(DESIGNED))
def test_designed_taps_within_contract(pkg, name):
    """subband_plan's taps, 20 blocks, 1e-5 against SubbandOracle; the plan has a class of at least 8
    members and lone members."""
    fs, fmt, n, span, seed = DESIGNED[name]
    rng = np.random.default_rng(seed)
    rates = [48000] * n if fs > 10 ** 7 else [48000 if i % 2 else 96000 for i in range(n)]
    centres = [int(c) for c in rng.integers(-span // 2, span // 2, n)]
    centres[-1] = fs // 3  # a lone member, far from the others
    p = pkg.subband_plan(fs, list(zip(centres, rates)))
    max_in = 131072
    rig = Rig(pkg, fs, max_in, fmt, depth=SLOTS)
    sids = [rig.add_subband(p["d1"], p["taps1"], sb["center"]) for sb in p["subbands"]]
    per = {}
    for m in p["members"]:
        rig.add_member(sids[m["subband"]], m["d2"], m["taps2"], m["offset"])
        per.setdefault((m["subband"], m["d2"]), []).append(m)
    assert max(len(v) for v in per.values()) >= 8 and min(len(v) for v in per.values()) == 1
    for _ in range(20):
        rig.submit(rand_block(rng, fmt, max_in))
    rig.assert_close()
    rig.close()


def test_first_stage_is_shared(pkg):
    """xlg_profile counts one sub-band's first stage however many members it has; the member counters are
    sum n2 * T2 and the sub-band samples."""
    fs, max_in, d1 = 2016000, 16384, 7
    fs1 = fs // d1
    rng = np.random.default_rng(9)
    t1 = pkg.create_low_pass_filter(1.0, fs, fs1 // 2, fs1 // 2 - 96000)
    t2 = pkg.create_low_pass_filter(1.0, fs1, 24000, 9600)
    rig = Rig(pkg, fs, max_in, "cu8")
    sid = rig.add_subband(d1, t1, 100000)
    for k in range(12):
        rig.add_member(sid, 6, t2, -60000 + 10000 * k)
    rig.submit(rand_block(rng, "cu8", max_in))
    rig.flush()
    rig.g.profile_enable(True)
    rig.g.profile_read(reset=True)
    rig.g.subband_profile_read(reset=True)
    sizes = [max_in, 999, max_in, 0, max_in]
    for n in sizes:
        rig.submit(rand_block(rng, "cu8", n))
    rig.flush()
    prof, sp = rig.g.profile_read(), rig.g.subband_profile_read()
    n1s = [y.size for y in rig.orc[sid].rows[1:]]
    n2s = [y.size for y in rig.got[next(iter(rig.got))][1:]]
    assert prof["algo_macs"] == sum(n1s) * t1.size  # one first stage, not one per member
    assert sp["row_samples"] == sum(n1s)
    assert sp["member_macs"] == 12 * sum(n2s) * t2.size
    assert sp["member_launches"] == len(sizes) and sp["member_ms"] > 0
    rig.close()


def test_churn(pkg):
    """A member attached mid-stream equals a fresh FloatPath fed the sub-band from its attach block on; a
    sub-band attached mid-stream; a member removed and attached again; xlg_remove_subband refuses while
    members remain; the ring wraps many times."""
    fs, max_in, d1 = 2016000, 4096, 6
    fs1 = fs // d1
    rng = np.random.default_rng(11)
    t1 = pkg.create_low_pass_filter(1.0, fs, fs1 // 2, fs1 // 2 - 96000)
    t2 = pkg.create_low_pass_filter(1.0, fs1, 24000, 9600)
    rig = Rig(pkg, fs, max_in, "cu8", depth=SLOTS)
    a = rig.add_subband(d1, t1, -500000)
    base = [rig.add_member(a, 7, t2, off) for off in (-70000, -20000, 30000)]
    late, again, b = None, None, None
    for blk in range(60):
        if blk == 3:
            late = rig.add_member(a, 7, t2, 55000)
        if blk == 5:
            b = rig.add_subband(d1, t1, 400000)
            rig.add_member(b, 7, t2, 12000)
            rig.add_member(b, 14, pkg.create_low_pass_filter(1.0, fs1, 12000, 4800), -41000)
        if blk == 7:
            rig.remove_member(base[1])
        if blk == 9:
            again = rig.add_member(a, 7, t2, -20000, key="again")
        rig.submit(rand_block(rng, "cu8", max_in if blk % 3 else max_in - 2 * (blk % 5) - 1))
    rig.flush()
    with pytest.raises(ValueError) as e:
        rig.g.remove_subband(b)
    assert e.value.args[0] == -errno.EBUSY
    for cid in [c for c, s in rig.of.items() if s == b]:
        rig.remove_member(cid)
    rig.remove_subband(b)
    rig.submit(rand_block(rng, "cu8", max_in))
    rig.assert_close()
    assert late in rig.got and len(rig.got[late]) == 58 and len(rig.got["again"]) == 52
    n1 = max_in // 2 // d1
    ring = 1 << int(np.ceil(np.log2(t2.size - 1 + (SLOTS + 1) * (n1 + 2))))
    assert 60 * n1 > 4 * ring  # the ring wrapped several times
    rig.close()


def neighbour_specs(pkg, fs):
    t = pkg.create_low_pass_filter(1.0, fs, 24000, 9600)
    r = pkg.rational_plan(fs, [44100])[0]
    c = pkg.cascade_plan(fs, [48000])[0]
    return [("i", 42, t, 300000), ("i", 42, t, -250000), ("r", r["interp"], r["decim"], r["taps"], 111000),
            ("c", c["d1"], c["taps1"], -610000, c["d2"], c["taps2"])]


def add_neighbour(g, s):
    if s[0] == "i":
        return g.add_client(*s[1:])
    if s[0] == "r":
        return g.add_client_rational(*s[1:])
    return g.add_client_cascade(*s[1:])


@pytest.mark.parametrize("host_ring", [0, 8])
def test_neighbours_keep_their_bits(pkg, host_ring):
    """Integer, rational and cascade clients give the same bits beside sub-bands as in a twin group without
    them, at pipeline depth XLG_SLOTS."""
    fs, max_in, fmt = 2016000, 16384, "cu8"
    rng = np.random.default_rng(13)
    specs = neighbour_specs(pkg, fs)
    twin = pkg.Group(fs, max_in, host_ring=host_ring)
    tw_ids = [add_neighbour(twin, s) for s in specs]
    rig = Rig(pkg, fs, max_in, fmt, host_ring=host_ring, depth=SLOTS)
    ids = [add_neighbour(rig.g, s) for s in specs]
    plan = pkg.subband_plan(fs, [(-400000 + 37000 * k, 48000) for k in range(10)])
    sids = [rig.add_subband(plan["d1"], plan["taps1"], sb["center"]) for sb in plan["subbands"]]
    for m in plan["members"]:
        rig.add_member(sids[m["subband"]], m["d2"], m["taps2"], m["offset"])
    blocks = [rand_block(rng, fmt, n) for n in [max_in] * 6 + [1001, 0, max_in, 64] + [max_in] * 6]
    pend = []
    for x in blocks:
        pend.append((twin.submit(fmt, x), rig.submit(x)))
        while len(pend) >= SLOTS:
            t0, t1 = pend.pop(0)
            twin.wait(t0)
            rig.g.wait(t1)
            for a, b in zip(tw_ids, ids):
                assert np.array_equal(twin.output(t0, a), rig.g.output(t1, b))
    twin.close()
    rig.assert_close()
    rig.close()


def test_device_outputs_match_host_outputs(pkg):
    fs, max_in, fmt = 2016000, 16384, "cu8"
    plan = pkg.subband_plan(fs, [(-300000 + 50000 * k, 48000 if k % 2 else 96000) for k in range(12)])
    got = []
    for flags in (0, pkg.XLG_OUT_DEVICE):
        rng = np.random.default_rng(15)
        rig = Rig(pkg, fs, max_in, fmt, flags=flags, depth=SLOTS)
        sids = [rig.add_subband(plan["d1"], plan["taps1"], sb["center"]) for sb in plan["subbands"]]
        for m in plan["members"]:
            rig.add_member(sids[m["subband"]], m["d2"], m["taps2"], m["offset"])
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
    bit for bit like a twin group that never saw the refused calls."""
    fs, max_in, fmt = 2016000, 8192, "cu8"
    fs1 = fs // 6
    rng = np.random.default_rng(17)
    t1 = pkg.create_low_pass_filter(1.0, fs, fs1 // 2, fs1 // 2 - 96000)
    t2 = pkg.create_low_pass_filter(1.0, fs1, 24000, 9600)
    rigs = [Rig(pkg, fs, max_in, fmt) for _ in range(2)]
    for r in rigs:
        sid = r.add_subband(6, t1, 250000)
        r.add_member(sid, 7, t2, 31000)
    x = rand_block(rng, fmt, max_in)
    for r in rigs:
        r.submit(x)
    capfd.readouterr()
    g = rigs[0].g
    empty = np.zeros(0, np.float32)
    calls = [
        (-errno.EINVAL, lambda: g.add_subband(0, t1, 0)),
        (-errno.EINVAL, lambda: g.add_subband(6, empty, 0)),
        (-errno.EINVAL, lambda: g.add_subband(11, t1, 0)),  # 2016000 % 11 != 0
        (-errno.EINVAL, lambda: g.add_client_subband(sid, 0, t2, 0)),
        (-errno.EINVAL, lambda: g.add_client_subband(sid, 7, empty, 0)),
        (-errno.EINVAL, lambda: g.add_client_subband(99, 7, t2, 0)),
        (-errno.EINVAL, lambda: g.add_client_subband(sid, 40, np.ones(1400, np.float32), 0)),
        (-errno.EINVAL, lambda: g.remove_subband(99)),
        (-errno.EBUSY, lambda: g.remove_subband(sid)),
    ]
    for code, call in calls:
        with pytest.raises(ValueError) as e:
            call()
        assert e.value.args[0] == code
        assert capfd.readouterr().err.count("<3>") == 1
    q = rand_block(rng, fmt, max_in)
    assert g._L.xlg_submit(g._h, pkg.FMT[fmt], q.ctypes.data, q.size, pkg.XLG_PATH_Q15) == -errno.ENOTSUP
    assert capfd.readouterr().err.count("<3>") == 1
    ts = pkg.Group(fs, max_in, flags=pkg.XLG_TRACK_STATE)
    with pytest.raises(ValueError) as e:
        ts.add_subband(6, t1, 0)
    assert e.value.args[0] == -errno.ENOTSUP
    assert capfd.readouterr().err.count("<3>") == 1
    assert ts.client_count() == 0
    ts.close()
    assert g.client_count() == 1  # the member; the sub-band is not a client
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
