"""Chirp-z bank sub-bands (xlg_add_bank_any at a K that is not a power of two) on the GPU.

A channel's row is observed through a member that copies it (taps [1.0] at decimation 1 and offset 0).  Rows
must equal the kernel model (tests/bank_czt_exact.py) bit for bit at every K of CZT_KS, at frame, CTA, ring and
attach edges and past 2^31 and 2^32 stream samples; members of a chirp-z channel equal the model's rows fed to
the member model bit for bit; designed taps (subband_plan(..., any_k=True)) are held to 1e-5 of the float64
definition.  A power-of-two K through xlg_add_bank_any is the FFT bank.  Every other client of a group keeps
its bits when a chirp-z bank joins it.  Refusals and the profile counters are checked too.
"""
import ctypes as C
import errno

import numpy as np
import pytest

from bank_czt_exact import bank_czt_flops, bank_czt_frames, bank_czt_m, bank_czt_member_model, bank_czt_model
from bank_exact import bank_walk, f64_bank
from bank_fft_exact import bank_fft_max_taps, bank_fft_model
from cascade import FloatPath
from cascade_rational import stuff
from exact import to_complex
from test_bank_czt_exact_reference import CZT_KS
from util import assert_cf32_close, rand_block

pytestmark = pytest.mark.gpu

FMTS = ("cu8", "cs8", "cs16")
RAGGED = [8192, 8192, 2005, 0, 7, 8190, 8192, 333, 8192, 8192, 8192, 8192, 6000, 8192]
CZT_KIND, FFT_KIND = 9, 8


def conv(fmt, raw):
    return to_complex(fmt, raw).astype(np.complex64)


def copy_member(g, sid):
    return g.add_client_subband(sid, 1, np.ones(1, np.float32), 0)


def rand_taps(rng, T):
    return (rng.standard_normal(T) / np.sqrt(T)).astype(np.float32)


def run_rows(pkg, fs, max_in, blocks, fmt, banks, flags=0, kind=CZT_KIND):
    """Feed `blocks`; banks: list of (d1, taps, attach block, {channel: materialise block}), each added with
    add_bank_fft(any_k=True).  Returns the rows {(bank index, channel): [per block from its materialisation]}."""
    g = pkg.Group(fs, max_in, flags=flags)
    bids, cids, rows = {}, {}, {}
    try:
        for b, x in enumerate(blocks):
            for i, (d1, taps, at, chans) in enumerate(banks):
                if at == b:
                    bids[i] = g.add_bank_fft(d1, taps, any_k=True)
                for k, mb in chans.items():
                    if mb == b:
                        cids[(i, k)] = copy_member(g, g.add_bank_subband(bids[i], k))
                        rows[(i, k)] = []
            t = g.submit(fmt, x)
            g.wait(t)
            for key, cid in cids.items():
                rows[key].append(g.output(t, cid))
                assert g.subband_info(cid)[1] == kind
    finally:
        g.close()
    return rows


def model_rows(pkg, blocks, fmt, d1, taps, at, chans):
    x = np.concatenate([conv(fmt, r) for r in blocks])
    sizes = [np.asarray(r).size // 2 for r in blocks]
    P = int(sum(sizes[:at]))
    out = bank_czt_model(taps, d1, list(chans), x, P, sizes[at:], pkg.bank_any_tables(2 * d1))
    return {k: out[k][mb - at:] for k, mb in chans.items()}


def assert_rows_equal(got, want, what):
    assert len(got) == len(want), what
    for b, (a, w) in enumerate(zip(got, want)):
        assert a.shape == w.shape, (what, b, a.shape, w.shape)
        assert np.array_equal(a, w), (what, b, np.max(np.abs(a - w)) if a.size else 0)


def refused(fn, *args, code=errno.EINVAL, **kw):
    with pytest.raises(ValueError) as e:
        fn(*args, **kw)
    assert e.value.args[0] == -code


@pytest.mark.parametrize("K", CZT_KS)
@pytest.mark.parametrize("case", ["short", "K", "ragged"])
def test_rows_bit_exact_against_the_model(pkg, K, case):
    """T1 < K, T1 = K and T1 >> K; ragged, odd, empty and tiny blocks that wrap the ring (n1 of 0 and 1 among
    them); channels -D1, 0, D1 - 1 and random ones."""
    d1 = K // 2
    T1 = {"short": max(1, K - 3), "K": K, "ragged": 3 * K + 5}[case]
    rng = np.random.default_rng(K * 37 + T1)
    fs = K * 48000
    chans = {-d1: 0, 0: 0, d1 - 1: 0}
    for k in rng.choice(np.arange(-d1, d1), size=min(4, K), replace=False):
        chans.setdefault(int(k), 0)
    max_in = max(8192, 2 * (T1 + 2 * K))
    sizes = [max_in if n == 8192 else n for n in RAGGED]
    for fmt in FMTS if K <= 1000 else ("cs16",):
        taps = rand_taps(rng, T1)
        blocks = [rand_block(rng, fmt, n) for n in sizes]
        rows = run_rows(pkg, fs, max_in, blocks, fmt, [(d1, taps, 0, chans)])
        want = model_rows(pkg, blocks, fmt, d1, taps, 0, chans)
        for k in chans:
            assert_rows_equal(rows[(0, k)], want[k], (fmt, K, T1, k))


def frame_sizes(rng, max_in, d1, T1, targets, lead):
    """Raw block sizes after `lead` making the n1 of a bank attached before lead every value of targets."""
    sizes = list(lead)
    for target in targets:
        for _ in range(int(rng.integers(1, 3))):
            sizes.append(max_in if rng.integers(0, 2) else int(rng.integers(1, max_in // 2)) * 2 + 1)
        counts = np.array([bank_walk([s // 2 for s in sizes] + [n], T1, d1)[0][-1] for n in range(max_in // 2 + 1)])
        sizes.append(2 * int(rng.choice(np.nonzero(counts == target)[0])))
    return sizes


@pytest.mark.parametrize("K", [6, 100, 1000, 4094])
def test_frames_per_cta_edges_and_mid_stream_attach(pkg, K):
    """n1 at 0, 1 and on both sides of one and two CTAs' frames; bank A attached at block 0, bank B of the same
    K mid-stream at an odd P, channels of both materialised after their attach."""
    d1, F = K // 2, bank_czt_frames(bank_czt_m(K))
    T1 = 2 * K + 3
    rng = np.random.default_rng(K + 3)
    fs, fmt = K * 48000, "cs8"
    max_in = 2 * (2 * F + 2) * d1 + 2 * T1
    sizes = frame_sizes(rng, max_in, d1, T1, sorted({0, 1, max(F - 1, 0), F, F + 1, 2 * F, 2 * F + 1}), [2002])
    at_b = 1  # P = 1001
    ta, tb = rand_taps(rng, T1), rand_taps(rng, K - 1)
    chans_a = {-d1: 0, 1: 0, 2: 2, d1 - 1: 3}
    chans_b = {0: at_b, -1: at_b + 1, min(3, d1 - 1): at_b + 2}
    blocks = [rand_block(rng, fmt, n) for n in sizes]
    rows = run_rows(pkg, fs, max_in, blocks, fmt, [(d1, ta, 0, chans_a), (d1, tb, at_b, chans_b)])
    wa = model_rows(pkg, blocks, fmt, d1, ta, 0, chans_a)
    wb = model_rows(pkg, blocks, fmt, d1, tb, at_b, chans_b)
    for k in chans_a:
        assert_rows_equal(rows[(0, k)], wa[k], ("A", k))
    for k in chans_b:
        assert_rows_equal(rows[(1, k)], wb[k], ("B", k))
    seen = set(bank_walk([n // 2 for n in sizes], T1, d1)[0])
    assert {0, 1, F, F + 1, 2 * F, 2 * F + 1} <= seen, sorted(seen)


def test_every_channel_at_250(pkg):
    """All 250 channels of a K = 250 bank, materialised in a shuffled order."""
    K, d1 = 250, 125
    rng = np.random.default_rng(250)
    fs, max_in, fmt = K * 48000, 16384, "cs16"
    taps = rand_taps(rng, 3 * K + 17)
    chans = {int(k): 0 for k in rng.permutation(np.arange(-d1, d1))}
    blocks = [rand_block(rng, fmt, n) for n in [max_in, max_in, 9001, max_in, 0, max_in]]
    rows = run_rows(pkg, fs, max_in, blocks, fmt, [(d1, taps, 0, chans)])
    want = model_rows(pkg, blocks, fmt, d1, taps, 0, chans)
    for k in chans:
        assert_rows_equal(rows[(0, k)], want[k], k)


@pytest.mark.parametrize("K", [2, 16, 128, 4096])
def test_power_of_two_k_is_the_fft_bank(pkg, K):
    """xlg_add_bank_any at a power-of-two K: kind 8 and the FFT bank model's rows, bit for bit."""
    d1 = K // 2
    rng = np.random.default_rng(K)
    fs, fmt = K * 48000, "cs16"
    taps = rand_taps(rng, 2 * K + 1)
    max_in = max(8192, 2 * (2 * K + 1 + 2 * K))
    sizes = [max_in if n == 8192 else n for n in RAGGED]
    blocks = [rand_block(rng, fmt, n) for n in sizes]
    chans = {-d1: 0, 0: 0, d1 - 1: 2}
    rows = run_rows(pkg, fs, max_in, blocks, fmt, [(d1, taps, 0, chans)], kind=FFT_KIND)
    x = np.concatenate([conv(fmt, r) for r in blocks])
    want = bank_fft_model(taps, d1, list(chans), x, 0, [r.size // 2 for r in blocks])
    for k, mb in chans.items():
        assert_rows_equal(rows[(0, k)], want[k][mb:], k)


INT_SHAPES = [(5, 23), (4, 8), (1, 1), (6, 40), (2, 31), (3, 250)]  # (D2, T2)
RAT_SHAPES = [(2, 5, 33), (3, 7, 40), (12, 5, 60)]                 # (L2, M2, T2)


@pytest.mark.parametrize("fmt", FMTS)
def test_members_at_any_offset(pkg, fmt):
    """Integer and rational members at offsets 0, +-fs1/4 and arbitrary, on channels -D1, 0, 7 and D1 - 1 of
    a K = 100 bank attached after block 0, members attached at the channel's first block: bit for bit the
    model's rows fed to the member model."""
    rng = np.random.default_rng(300 + FMTS.index(fmt))
    d1, fs, max_in = 50, 4800000, 16384
    fs1 = fs // d1
    offsets = [0, fs1 // 4, -fs1 // 4, int(rng.integers(-fs1 // 2, fs1 // 2))]
    taps1 = rand_taps(rng, 157)
    shapes = [(1, d2, T2) for d2, T2 in INT_SHAPES] + RAT_SHAPES
    blocks = [rand_block(rng, fmt, n) for n in [max_in, max_in, 4005, 0, 7, max_in - 2, max_in, 333, max_in]]
    g = pkg.Group(fs, max_in)
    members = {}
    outs = {}
    try:
        for b, x in enumerate(blocks):
            if b == 1:
                bid = g.add_bank_fft(d1, taps1, any_k=True)
                for k in (-d1, 0, 7, d1 - 1):
                    sid = g.add_bank_subband(bid, k)
                    members[k] = []
                    for i, (l2, d2, T2) in enumerate(shapes):
                        t2 = rand_taps(rng, T2)
                        off = offsets[(i + k) % 4]
                        cid = g.add_client_subband(sid, d2, t2, off, l2)
                        members[k].append((cid, (l2, d2, t2, off)))
                        outs[cid] = []
            t = g.submit(fmt, x)
            g.wait(t)
            for cid in outs:
                outs[cid].append(g.output(t, cid))
                assert g.subband_info(cid)[1] == CZT_KIND
    finally:
        g.close()
    xs = np.concatenate([conv(fmt, r) for r in blocks])
    sizes = [r.size // 2 for r in blocks]
    P = sizes[0]
    for k, ms in members.items():
        want = bank_czt_member_model(taps1, d1, k, xs, P, sizes[1:], [m for _, m in ms], fs,
                                     pkg.bank_any_tables(2 * d1))
        for (cid, m), w in zip(ms, want):
            assert_rows_equal(outs[cid], w, (fmt, k, m[0], m[1], m[3]))


PLAN_RATES = [(10000000, "cs16", 64), (20000000, "cs8", 48), (6000000, "cs16", 256)]


@pytest.mark.parametrize("fs,fmt,n", PLAN_RATES)
def test_designed_taps_within_1e_5_of_float64(pkg, fs, fmt, n):
    """subband_plan(bank=True, fft=True, any_k=True) at the front-end rates: every sampled member within 1e-5
    of the float64 bank rows fed to the reference's float path."""
    rng = np.random.default_rng(fs % 997 + n)
    max_in = 65536
    centres = rng.integers(-fs // 2 + 48000, fs // 2 - 48000, n)
    p = pkg.subband_plan(fs, [(int(c), 48000) for c in centres], bank=True, fft=True, any_k=True)
    d1, fs1 = p["d1"], p["fs1"]
    assert p["kernel"] == "czt"
    blocks = [rand_block(rng, fmt, max_in) for _ in range(3)]
    g = pkg.Group(fs, max_in)
    try:
        bid = g.add_bank_fft(d1, p["taps1"], any_k=True)
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


def _population(pkg, g, with_czt):
    """Every other client family on a 4.8 Msps band, the same for both twins; with_czt then adds a K = 100
    chirp-z bank with two channels, so the other clients' ids are the same in both.  Returns the other
    clients' ids, the spectrum's id, the chirp-z bank's id and its copy members."""
    lp = pkg.create_low_pass_filter
    ids = [g.add_client(100, lp(1.0, 4800000, 24000, 9600), 123456),
           g.add_client_rational(2, 125, lp(2.0, 9600000, 19200, 7680), -700001),
           g.add_client_cascade(10, lp(1.0, 4800000, 200000, 80000), 40000, 10, lp(1.0, 480000, 20000, 8000))]
    sb = g.add_subband(25, lp(1.0, 4800000, 96000, 40000), -1000000)
    ids.append(g.add_client_subband(sb, 4, lp(1.0, 192000, 24000, 9600), 3000))
    bf = g.add_bank_fft(32, rand_taps(np.random.default_rng(2), 129))
    ids.append(copy_member(g, g.add_bank_subband(bf, -5)))
    bd = g.add_bank(25, rand_taps(np.random.default_rng(3), 151))
    ids.append(copy_member(g, g.add_bank_subband(bd, 7)))
    spec = g.add_spectrum(1000, 2, 0)
    bz, extra = None, []
    if with_czt:
        bz = g.add_bank_fft(50, rand_taps(np.random.default_rng(1), 301), any_k=True)
        extra = [copy_member(g, g.add_bank_subband(bz, k)) for k in (-50, 11)]
    return ids, spec, bz, extra


@pytest.mark.parametrize("variant", ["default", "out_device", "host_ring"])
def test_other_clients_keep_their_bits(pkg, variant):
    """A group with a chirp-z bank beside integer, rational, cascade and sub-band clients, an FFT bank, a direct
    bank and a spectrum gives every other client the bits of a twin without the chirp-z bank, with three tickets
    in flight and the chirp-z bank churned (its channels and the bank removed, a new one added)."""
    flags = pkg.XLG_OUT_DEVICE if variant == "out_device" else 0
    host_ring = 12 if variant == "host_ring" else 0
    rng = np.random.default_rng(77)
    fmt, max_in = "cs16", 32768
    blocks = [rand_block(rng, fmt, n) for n in [max_in, 7, max_in, 0, 10001, max_in, max_in, 333, max_in, max_in]]
    results = []
    for with_czt in (False, True):
        g = pkg.Group(4800000, max_in, flags=flags, host_ring=host_ring)
        got, rows, pending = None, [], []
        try:
            ids, spec, bz, extra = _population(pkg, g, with_czt)
            got = {i: [] for i in ids}

            def harvest(t):
                for i in ids:
                    got[i].append(np.array(g.read_output(t, i)))
                rows.append(np.array(g.read_spectrum(t, spec)))

            for b, x in enumerate(blocks):
                if with_czt and b == 4:
                    for cid in extra:
                        sid = g.subband_info(cid)[0]
                        g.remove_client(cid)
                        g.remove_subband(sid)
                    g.remove_bank(bz)
                    bz = g.add_bank_fft(50, rand_taps(np.random.default_rng(4), 77), any_k=True)
                    extra = [copy_member(g, g.add_bank_subband(bz, 3))]
                pending.append(g.submit(fmt, x))
                if len(pending) >= 3:
                    t = pending.pop(0)
                    g.wait(t)
                    harvest(t)
            for t in pending:
                g.wait(t)
                harvest(t)
        finally:
            g.close()
        results.append((got, rows))
    (a, ra), (b, rb) = results
    assert a.keys() == b.keys()
    for i in a:
        assert_rows_equal(b[i], a[i], (variant, i))
        assert sum(np.count_nonzero(y) for y in a[i]) > 0, (variant, i)
    assert_rows_equal(rb, ra, (variant, "spectrum"))


def test_refusals_and_profile(pkg):
    """Each refusal is logged, changes nothing and takes no ticket: the next bank still takes id 0.  The
    profile counts a chirp-z bank's frames by the header's formulas."""
    g = pkg.Group(4800000, 8192)
    try:
        t = np.ones(21, np.float32)
        add = g.add_bank_fft
        t0 = g.submit("cu8", np.zeros(8192, np.uint8))
        g.wait(t0)
        refused(add, 0, t, any_k=True)
        refused(add, 50, np.zeros(0, np.float32), any_k=True)
        refused(add, 2500, t, any_k=True)     # K = 5000 > 4096
        refused(add, 4096, t, any_k=True)     # K = 8192, a power of two above 4096
        refused(add, 7, t, any_k=True)        # 4.8 MHz % 14 != 0
        refused(add, 50, np.ones(bank_fft_max_taps(100) + 1, np.float32), any_k=True)
        refused(add, 50, t)                   # xlg_add_bank_fft keeps its refusal of K = 100
        t1 = g.submit("cu8", np.zeros(8192, np.uint8))
        assert t1 == t0 + 1  # no refusal took a ticket
        g.wait(t1)
        bid = add(50, np.ones(bank_fft_max_taps(100), np.float32), any_k=True)
        assert bid == 0
        sid = g.add_bank_subband(bid, -50)
        refused(g.add_bank_subband, bid, 50)
        refused(g.add_bank_subband, bid, -50, code=errno.EEXIST)
        cid = copy_member(g, sid)
        refused(g.remove_bank, bid, code=errno.EBUSY)
        x = np.zeros(8192, np.uint8)
        assert g._L.xlg_submit(g._h, pkg.FMT["cu8"], x.ctypes.data_as(C.c_void_p), x.size,
                               pkg.XLG_PATH_Q15) == -errno.ENOTSUP
        t2 = g.submit("cu8", x)
        assert t2 == t1 + 1  # the refused Q15 submit took no ticket
        g.wait(t2)
        g.remove_client(cid)
        g.remove_subband(sid)
        g.remove_bank(bid)
        assert g.add_bank(24, t) == 0
    finally:
        g.close()
    g = pkg.Group(4800000, 8192, flags=pkg.XLG_TRACK_STATE)
    try:
        refused(g.add_bank_fft, 50, np.ones(21, np.float32), any_k=True, code=errno.ENOTSUP)
    finally:
        g.close()
    rng = np.random.default_rng(5)
    fs, max_in, fmt = 4800000, 8192, "cs16"
    blocks = [rand_block(rng, fmt, n) for n in RAGGED]
    ta, tb = rand_taps(rng, 131), rand_taps(rng, 40)
    g = pkg.Group(fs, max_in)
    try:
        g.profile_enable(True)
        a = g.add_bank_fft(50, ta, any_k=True)       # K = 100, M = 256, three channels
        for k in (-50, 0, 9):
            copy_member(g, g.add_bank_subband(a, k))
        b = g.add_bank_fft(8, tb, any_k=True)        # K = 16: an FFT bank, one channel
        copy_member(g, g.add_bank_subband(b, 1))
        g.bank_fft_profile_read(reset=True)
        for x in blocks:
            g.wait(g.submit(fmt, x))
        prof = g.bank_fft_profile_read()
        direct = g.bank_profile_read()
    finally:
        g.close()
    sizes = [r.size // 2 for r in blocks]
    ca, _ = bank_walk(sizes, 131, 50)
    cb, _ = bank_walk(sizes, 40, 8)
    assert prof["poly_macs"] == sum(ca) * 131 + sum(cb) * 40
    assert prof["butterfly_flops"] == (sum(ca) * bank_czt_flops(pkg.bank_fft_flops, 100, 3) +
                                       sum(cb) * pkg.bank_fft_flops(16))
    assert prof["fft_launches"] == sum(1 for p, q in zip(ca, cb) if max(p, q) > 0)
    assert prof["fft_ms"] > 0
    assert direct["bank_launches"] == 0


def test_long_stream_past_2_31_and_2_32(pkg):
    """A K = 30 chirp-z bank fed XLG_INPUT_DEVICE blocks of N samples (N a multiple of K) from position 0: its
    rows in blocks past 2^31 and 2^32 equal the model's rows of a bank attached at the start of the block
    before (both banks' rotations agree there, and its windows all start after that boundary)."""
    torch = pytest.importorskip("torch")
    from long_stream import N, Pump
    fmt, d1, T1 = "cs16", 15, 97
    rng = np.random.default_rng(31)
    taps = rand_taps(rng, T1)
    bufs = [rand_block(rng, fmt, 2 * N) for _ in range(3)]
    g = pkg.Group(30 * 48000, 2 * N)
    chans = (-15, 0, 7, 14)
    got = {}
    try:
        bid = g.add_bank_fft(d1, taps, any_k=True)
        cids = {k: copy_member(g, g.add_bank_subband(bid, k)) for k in chans}

        def read(t, i):
            got[i] = {k: np.array(g.output(t, c)) for k, c in cids.items()}

        pump = Pump(torch, pkg, g, fmt, bufs, 32, read=read)
        checked = []
        for target in (2 ** 31, 2 ** 32):
            pump.run_to(target)
            pump.watch.update({len(pump.blocks), len(pump.blocks) + 1})
            first = pump.feed()
            pump.feed()
            checked.append(first)
        pump.drain()
    finally:
        g.close()
    assert pump.starts[checked[1] + 1] > 2 ** 32
    tables = pkg.bank_any_tables(30)
    for i in checked:
        x = np.concatenate([conv(fmt, pump.blocks[i]), conv(fmt, pump.blocks[i + 1])])
        want = bank_czt_model(taps, d1, list(chans), x, 0, [N, N], tables)
        for k in chans:
            assert np.array_equal(got[i + 1][k], want[k][1]), (i, k)
