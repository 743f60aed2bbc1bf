"""Bank sub-bands (xlg_add_bank, xlg_add_bank_subband) on the GPU.

A channel's row is observed through a member that copies it: taps [1.0] at decimation 1 and offset 0 (its
oscillator stays 1 + 0i, so the member kernel returns the row bit for bit).  Rows must equal the kernel
model (tests/bank_exact.py) bit for bit on random taps and input, and the float64 definition bit for bit on
exact stimuli; designed taps (subband_plan(bank=True)) are held to 1e-5 of the float64 definition, and the
same clients served by ordinary sub-bands to 1e-5 plus the phase their float oscillators drift by.
"""
import ctypes as C
import errno

import numpy as np
import pytest

from bank_exact import bank_model, bank_walk, f64_bank
from cascade import FloatPath, f64_filter, filter_constants
from cascade_rational import stuff
from exact import dyadic_taps, exact_input, one_hot_taps, to_complex
from oracle import pyoracle as po
from subband_rational import RationalSubbandOracle
from util import assert_cf32_close, rand_block

pytestmark = pytest.mark.gpu

FMTS = ("cu8", "cs8", "cs16")
# ragged, odd (a trailing element is dropped), empty and tiny blocks, in elements
RAGGED = [8192, 8192, 2005, 0, 7, 8190, 8192, 333, 8192, 8192, 8192, 8192, 6000, 8192]


def conv(fmt, raw):
    return to_complex(fmt, raw).astype(np.complex64)


def copy_member(g, sid):
    return g.add_client_subband(sid, 1, np.ones(1, np.float32), 0)


def bound_taps(pkg, d1):
    t = 1
    while pkg.bank_fits(d1, 2 * t):
        t *= 2
    lo, hi = t, 2 * t
    while hi - lo > 1:
        mid = (lo + hi) // 2
        lo, hi = (mid, hi) if pkg.bank_fits(d1, mid) else (lo, mid)
    return lo


def tap_cases(pkg, d1):
    K = 2 * d1
    return {"short": max(1, K - 3), "K": K, "ragged": 3 * K + 5, "bound": bound_taps(pkg, d1)}


def run_rows(pkg, fs, max_in, blocks, fmt, banks, flags=0):
    """Feed `blocks`; banks: list of (d1, taps, attach block, {channel: materialise block}).  Returns the rows
    {(bank index, channel): [per block from its materialisation]}."""
    g = pkg.Group(fs, max_in, flags=flags)
    bids, cids, rows = {}, {}, {}
    try:
        for b, x in enumerate(blocks):
            for i, (d1, taps, at, chans) in enumerate(banks):
                if at == b:
                    bids[i] = g.add_bank(d1, taps)
                for k, mb in chans.items():
                    if mb == b:
                        cids[(i, k)] = copy_member(g, g.add_bank_subband(bids[i], k))
                        rows[(i, k)] = []
            t = g.submit(fmt, x)
            g.wait(t)
            for key, cid in cids.items():
                rows[key].append(g.read_output(t, cid) if flags & pkg.XLG_OUT_DEVICE else g.output(t, cid))
    finally:
        g.close()
    return rows


def model_rows(blocks, fmt, d1, taps, at, chans):
    x = np.concatenate([conv(fmt, r) for r in blocks])
    sizes = [np.asarray(r).size // 2 for r in blocks]
    P = int(sum(sizes[:at]))
    out = bank_model(taps, d1, list(chans), x, P, sizes[at:])
    return {k: out[k][mb - at:] for k, mb in chans.items()}


def assert_rows_equal(got, want, what):
    assert len(got) == len(want), what
    for b, (a, w) in enumerate(zip(got, want)):
        assert a.shape == w.shape, (what, b, a.shape, w.shape)
        assert np.array_equal(a, w), (what, b, np.max(np.abs(a - w)) if a.size else 0)


@pytest.mark.parametrize("d1", [1, 2, 3, 7, 10, 32, 64])
@pytest.mark.parametrize("case", ["short", "K", "ragged", "bound"])
def test_rows_bit_exact_against_the_model(pkg, d1, case):
    T1 = tap_cases(pkg, d1)[case]
    rng = np.random.default_rng(d1 * 31 + T1)
    fs = 2 * d1 * 48000
    chans = {-d1: 0, 0: 0, d1 - 1: 0}
    for k in rng.choice(np.arange(-d1, d1), size=min(3, 2 * d1), replace=False):
        chans.setdefault(int(k), 0)
    if case == "bound":
        # windows of the longest bank the kernel holds: two blocks longer than it (one odd), one format (the
        # model's cost grows with T1 times the frames)
        max_in = 2 * (T1 + 4096)
        sizes, fmts = [max_in, max_in // 2 + 1], ("cs16",)
    else:
        # the ring holds 5 blocks + 4096 samples of history: these 14 blocks wrap it
        max_in, sizes, fmts = 8192, RAGGED, FMTS
    for fmt in fmts:
        taps = rng.standard_normal(T1).astype(np.float32) / np.float32(np.sqrt(T1))
        blocks = [rand_block(rng, fmt, n) for n in sizes]
        rows = run_rows(pkg, fs, max_in, blocks, fmt, [(d1, taps, 0, chans)])
        want = model_rows(blocks, fmt, d1, taps, 0, chans)
        for k in chans:
            assert_rows_equal(rows[(0, k)], want[k], (fmt, d1, T1, k))


def test_taps_past_the_bound_are_refused(pkg):
    for d1 in (1, 2, 3, 7, 10, 32, 64):
        g = pkg.Group(2 * d1 * 48000, 8192)
        try:
            T = bound_taps(pkg, d1)
            g.add_bank(d1, np.ones(T, np.float32))
            with pytest.raises(ValueError) as e:
                g.add_bank(d1, np.ones(T + 1, np.float32))
            assert e.value.args[0] == -errno.EINVAL
        finally:
            g.close()


def test_mid_stream_banks_beside_clients_and_subbands(pkg):
    """Two banks of different D1 and taps, one attached mid-stream, a channel materialised after its bank
    (its rows are the bank's from P), beside integer clients and an ordinary sub-band with a member."""
    rng = np.random.default_rng(11)
    fs, max_in, fmt = 2016000, 8192, "cs8"
    blocks = [rand_block(rng, fmt, n) for n in RAGGED]
    ta = rng.standard_normal(61).astype(np.float32) / 8
    tb = rng.standard_normal(40).astype(np.float32) / 8
    banks = [(7, ta, 0, {-7: 0, 3: 4, 6: 0}), (4, tb, 2, {-4: 2, 1: 5})]
    lpf = pkg.create_low_pass_filter(1.0, fs, 24000, 9600)
    sb_taps = pkg.create_low_pass_filter(1.0, fs, 72000, 40000)
    ids = {}

    def extra(g, b):
        if b == 0:
            ids["int"] = [g.add_client(42, lpf, c) for c in (-300000, 12345, 700000)]
            sid = g.add_subband(7, sb_taps, 144000)
            ids["sb"] = g.add_client_subband(sid, 6, lpf[:47], 1000)

    g = pkg.Group(fs, max_in)
    got = {"int": [[] for _ in range(3)], "sb": []}
    bids, cids, rows = {}, {}, {}
    try:
        for b, x in enumerate(blocks):
            for i, (d1, taps, at, chans) in enumerate(banks):
                if at == b:
                    bids[i] = g.add_bank(d1, taps)
                for k, mb in chans.items():
                    if mb == b:
                        cids[(i, k)] = copy_member(g, g.add_bank_subband(bids[i], k))
                        rows[(i, k)] = []
            extra(g, b)
            t = g.submit(fmt, x)
            g.wait(t)
            for key, cid in cids.items():
                rows[key].append(g.output(t, cid))
            for j, cid in enumerate(ids["int"]):
                got["int"][j].append(g.output(t, cid))
            got["sb"].append(g.output(t, ids["sb"]))
            for key, cid in cids.items():
                assert g.subband_info(cid)[1] == 7
    finally:
        g.close()
    for i, (d1, taps, at, chans) in enumerate(banks):
        want = model_rows(blocks, fmt, d1, taps, at, chans)
        for k in chans:
            assert_rows_equal(rows[(i, k)], want[k], (i, k))
    for j, c in enumerate((-300000, 12345, 700000)):
        o = po.OracleFilter(42, lpf, c, fs, max_in)
        for b, x in enumerate(blocks):
            assert_cf32_close(got["int"][j][b], o.process_cf32(fmt, x), f"client {j} block {b}")
    o = RationalSubbandOracle(7, sb_taps, 144000, fs, max_in)
    o.add_member(0, 6, lpf[:47], 1000)
    for b, x in enumerate(blocks):
        assert_cf32_close(got["sb"][b], o.process_cf32(fmt, x)[0], f"sub-band member block {b}")


@pytest.mark.parametrize("d1", [2, 4, 10])
def test_exact_stimuli_against_float64(pkg, d1):
    """Dyadic taps, grid input, channels whose twiddles are +-1 or +-i: every sum is exact, so the rows and
    one-hot members on them (through the member kernels) equal the float64 definition bit for bit."""
    rng = np.random.default_rng(d1)
    fs, max_in = 2 * d1 * 48000, 8192
    chans = [k for k in range(-d1, d1) if (4 * k) % (2 * d1) == 0]
    for fmt in FMTS:
        T1 = 4 * d1 + 3
        taps = dyadic_taps(rng, T1, fmt)
        blocks = [exact_input(rng, fmt, n - n % 2) for n in RAGGED[:8]]
        g = pkg.Group(fs, max_in)
        try:
            bid = g.add_bank(d1, taps)
            sids = {k: g.add_bank_subband(bid, k) for k in chans}
            copies = {k: copy_member(g, s) for k, s in sids.items()}
            hot = {k: g.add_client_subband(s, 2, one_hot_taps(5, 2, 0.5), 0) for k, s in sids.items()}
            got = {k: [] for k in chans}
            got_hot = {k: [] for k in chans}
            for x in blocks:
                t = g.submit(fmt, x)
                g.wait(t)
                for k in chans:
                    got[k].append(g.output(t, copies[k]))
                    got_hot[k].append(g.output(t, hot[k]))
        finally:
            g.close()
        x = np.concatenate([to_complex(fmt, r) for r in blocks])
        sizes = [r.size // 2 for r in blocks]
        ref = f64_bank(taps, d1, chans, x, 0, sizes)
        for k in chans:
            for a, w in zip(got[k], ref[k]):
                assert np.array_equal(a.astype(complex), w), (fmt, k)
            hot_ref = f64_filter(one_hot_taps(5, 2, 0.5), 2, 0, fs // d1, ref[k])
            for a, w in zip(got_hot[k], hot_ref):
                assert np.array_equal(a.astype(complex), w), (fmt, k, "member")


PLAN_RATES = [(61440000, "cs16", 64), (2016000, "cu8", 48), (2048000, "cu8", 48), (10000000, "cs16", 48),
              (20000000, "cs8", 48)]


def plan_clients(fs, n, rng):
    centres = rng.integers(-fs // 2 + 48000, fs // 2 - 48000, n)
    return [(int(c), 48000 if i % 2 == 0 or fs != 2016000 else 96000) for i, c in enumerate(centres)]


@pytest.mark.parametrize("fs,fmt,n", PLAN_RATES)
def test_designed_taps_within_1e_5_of_float64(pkg, fs, fmt, n):
    """subband_plan(bank=True) at the front-end rates, rational members included: every member within 1e-5
    of the float64 bank rows fed to the reference's float path."""
    rng = np.random.default_rng(fs % 1000 + n)
    max_in = 65536
    p = pkg.subband_plan(fs, plan_clients(fs, n, rng), bank=True)
    d1, fs1 = p["d1"], p["fs1"]
    blocks = [rand_block(rng, fmt, max_in) for _ in range(3)]
    g = pkg.Group(fs, max_in)
    try:
        bid = g.add_bank(d1, p["taps1"])
        sids = [g.add_bank_subband(bid, s["channel"]) for s in p["subbands"]]
        picks = sorted(set(rng.choice(len(p["members"]), size=min(12, len(p["members"])), replace=False).tolist()))
        cids = [g.add_client_subband(sids[m["subband"]], m["d2"], m["taps2"], m["offset"], m["interp2"])
                for m in p["members"]]
        outs = {i: [] for i in picks}
        for x in blocks:
            t = g.submit(fmt, x)
            g.wait(t)
            for i in picks:
                outs[i].append(g.output(t, cids[i]))
    finally:
        g.close()
    x = np.concatenate([to_complex(fmt, r) for r in blocks])
    sizes = [r.size // 2 for r in blocks]
    chans = sorted({p["subbands"][p["members"][i]["subband"]]["channel"] for i in picks})
    rows = f64_bank(p["taps1"], d1, chans, x, 0, sizes)
    for i in picks:
        m = p["members"][i]
        k = p["subbands"][m["subband"]]["channel"]
        path = FloatPath(m["d2"], m["taps2"], m["offset"], m["interp2"] * fs1)
        want = [path.process_cf32(stuff(y.astype(np.complex64), m["interp2"]) if m["interp2"] > 1
                                  else y.astype(np.complex64)) for y in rows[k]]
        assert_cf32_close(np.concatenate(outs[i]), np.concatenate(want), f"member {i} channel {k}")


def subband_drift(d1, k, fs):
    _, (ir, ii) = filter_constants(np.ones(1, np.float32), d1, k * fs // (2 * d1), fs)
    return abs(np.angle(complex(ir, ii) * (-1) ** k))


@pytest.mark.parametrize("fs,fmt", [(2016000, "cu8"), (2048000, "cu8")])
def test_same_clients_as_ordinary_subbands(pkg, fs, fmt):
    """The identity on the GPU (odd T1): members of bank channels and of ordinary sub-bands at the same
    centres agree within 1e-5 norm-wise, plus the phase the sub-bands' float oscillators (step
    cexpf(-float(w0) * D1), not exactly (-1)^k) and float tap rotation drift by."""
    rng = np.random.default_rng(3)
    max_in = 16384
    p = pkg.subband_plan(fs, plan_clients(fs, 24, rng), bank=True)
    d1 = p["d1"]
    assert p["taps1"].size % 2 == 1
    blocks = [rand_block(rng, fmt, max_in) for _ in range(2)]
    g = pkg.Group(fs, max_in)
    try:
        bid = g.add_bank(d1, p["taps1"])
        bank_ids, sb_ids = [], []
        for s in p["subbands"]:
            bs = g.add_bank_subband(bid, s["channel"])
            os_ = g.add_subband(d1, p["taps1"], s["channel"] * fs // (2 * d1))
            bank_ids.append(bs)
            sb_ids.append(os_)
        pairs = [(g.add_client_subband(bank_ids[m["subband"]], m["d2"], m["taps2"], m["offset"], m["interp2"]),
                  g.add_client_subband(sb_ids[m["subband"]], m["d2"], m["taps2"], m["offset"], m["interp2"]), m)
                 for m in p["members"]]
        got = [([], []) for _ in pairs]
        for x in blocks:
            t = g.submit(fmt, x)
            g.wait(t)
            for (a, b, _), (ga, gb) in zip(pairs, got):
                ga.append(g.output(t, a))
                gb.append(g.output(t, b))
    finally:
        g.close()
    n1 = sum(bank_walk([max_in // 2] * len(blocks), p["taps1"].size, d1)[0])
    for (_, _, m), (ga, gb) in zip(pairs, got):
        k = p["subbands"][m["subband"]]["channel"]
        a, b = np.concatenate(ga), np.concatenate(gb)
        assert a.shape == b.shape
        tol = 1e-5 + 2 * subband_drift(d1, k, fs) * n1 + 4e-7 * p["taps1"].size
        assert np.max(np.abs(a - b)) <= tol * np.max(np.abs(b)), (k, m["offset"])


def test_refusals(pkg):
    fs = 2016000
    g = pkg.Group(fs, 8192)
    try:
        t = np.ones(21, np.float32)
        for d1, taps in ((0, t), (7, np.zeros(0, np.float32))):
            with pytest.raises(ValueError) as e:
                g.add_bank(d1, taps)
            assert e.value.args[0] == -errno.EINVAL
        with pytest.raises(ValueError) as e:
            g.add_bank(11, t)  # 2016000 % 22 != 0
        assert e.value.args[0] == -errno.EINVAL
        bid = g.add_bank(7, t)
        for k in (-8, 7, 100):
            with pytest.raises(ValueError) as e:
                g.add_bank_subband(bid, k)
            assert e.value.args[0] == -errno.EINVAL
        with pytest.raises(ValueError) as e:
            g.add_bank_subband(bid + 5, 0)
        assert e.value.args[0] == -errno.EINVAL
        sid = g.add_bank_subband(bid, -7)
        with pytest.raises(ValueError) as e:
            g.add_bank_subband(bid, -7)
        assert e.value.args[0] == -errno.EEXIST
        cid = copy_member(g, sid)
        with pytest.raises(ValueError) as e:
            g.remove_subband(sid)
        assert e.value.args[0] == -errno.EBUSY
        with pytest.raises(ValueError) as e:
            g.remove_bank(bid)
        assert e.value.args[0] == -errno.EBUSY
        x = np.zeros(8192, np.uint8)
        assert g._L.xlg_submit(g._h, pkg.FMT["cu8"], x.ctypes.data_as(C.c_void_p), x.size,
                               pkg.XLG_PATH_Q15) == -errno.ENOTSUP
        g.remove_client(cid)
        g.remove_subband(sid)
        g.remove_bank(bid)
        with pytest.raises(ValueError) as e:
            g.remove_bank(bid)
        assert e.value.args[0] == -errno.EINVAL
        assert g.add_bank(7, t) == bid  # ids are reused
        t_ok = g.submit("cu8", x)  # nothing was enqueued by the refused Q15 submit
        g.wait(t_ok)
    finally:
        g.close()
    g = pkg.Group(fs, 8192, flags=pkg.XLG_TRACK_STATE)
    try:
        with pytest.raises(ValueError) as e:
            g.add_bank(7, np.ones(21, np.float32))
        assert e.value.args[0] == -errno.ENOTSUP
    finally:
        g.close()


def test_churn_device_outputs_host_ring_and_profile(pkg):
    """Channels and members added and removed, bank ids reused, the ring grown by a longer bank, outputs left
    on the device and a deeper host ring: rows stay the model's, and the profile counts are the shapes'."""
    rng = np.random.default_rng(9)
    fs, max_in, fmt = 2016000, 8192, "cs16"
    blocks = [rand_block(rng, fmt, n) for n in RAGGED]
    ta = rng.standard_normal(33).astype(np.float32) / 4
    tb = rng.standard_normal(5000).astype(np.float32) / 64
    for flags in (0, pkg.XLG_OUT_DEVICE):
        g = pkg.Group(fs, max_in, flags=flags, host_ring=8 if flags == 0 else 0)
        g.profile_enable(True)
        rows, cids = {}, {}
        polys = dfts = 0
        try:
            for b, x in enumerate(blocks):
                if b == 0:
                    bid = g.add_bank(7, ta)
                    for k in (-7, 2):
                        cids[k] = copy_member(g, g.add_bank_subband(bid, k))
                        rows[k] = []
                    sid_tmp = g.add_bank_subband(bid, 5)
                    tmp = copy_member(g, sid_tmp)
                if b == 3:
                    g.remove_client(tmp)
                    g.remove_subband(sid_tmp)
                    bid2 = g.add_bank(6, tb)  # a longer history: the input ring grows, keeping its samples
                    sid_b = g.add_bank_subband(bid2, 1)
                    cids[("b", 1)] = copy_member(g, sid_b)
                    rows[("b", 1)] = []
                if b == 7:
                    g.remove_client(cids.pop(("b", 1)))
                    g.remove_subband(sid_b)
                    g.remove_bank(bid2)
                    assert g.add_bank(6, tb) == bid2
                    cids[("c", -6)] = copy_member(g, g.add_bank_subband(bid2, -6))
                    rows[("c", -6)] = []
                t = g.submit(fmt, x)
                g.wait(t)
                for key, cid in cids.items():
                    rows[key].append(g.read_output(t, cid))
        finally:
            prof = g.bank_profile_read()
            g.close()
        want = model_rows(blocks, fmt, 7, ta, 0, {-7: 0, 2: 0})
        for k in (-7, 2):
            assert_rows_equal(rows[k], want[k], (flags, k))
        want = model_rows(blocks[:7], fmt, 6, tb, 3, {1: 3})
        assert_rows_equal(rows[("b", 1)], want[1], (flags, "b"))
        want = model_rows(blocks, fmt, 6, tb, 7, {-6: 7})
        assert_rows_equal(rows[("c", -6)], want[-6], (flags, "c"))
        sizes = [np.asarray(r).size // 2 for r in blocks]
        ca, _ = bank_walk(sizes, 33, 7)
        cb, _ = bank_walk(sizes[3:7], 5000, 6)
        cc, _ = bank_walk(sizes[7:], 5000, 6)
        chans_a = [3] * 3 + [2] * (len(sizes) - 3)
        poly = sum(n * 33 for n in ca) + sum(n * 5000 for n in cb) + sum(n * 5000 for n in cc)
        dft = sum(n * c * 14 for n, c in zip(ca, chans_a)) + sum(n * 12 for n in cb) + sum(n * 12 for n in cc)
        assert prof["poly_macs"] == poly and prof["dft_macs"] == dft
        n_b = [0] * 3 + cb + cc
        assert prof["bank_launches"] == sum(1 for a, b in zip(ca, n_b) if max(a, b) > 0)
        assert prof["bank_ms"] > 0


def test_group_without_banks_profiles_nothing(pkg):
    g = pkg.Group(2016000, 8192)
    try:
        g.profile_enable(True)
        g.add_client(42, pkg.create_low_pass_filter(1.0, 2016000, 24000, 9600), 1000)
        g.wait(g.submit("cu8", np.zeros(8192, np.uint8)))
        assert g.bank_profile_read() == {"bank_ms": 0.0, "bank_launches": 0, "poly_macs": 0, "dft_macs": 0}
    finally:
        g.close()
