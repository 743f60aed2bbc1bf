"""FFT bank sub-bands (xlg_add_bank_fft) on the GPU.

A channel's row is observed through a member that copies it (taps [1.0] at decimation 1 and offset 0: the
member kernel returns the row bit for bit).  Rows must equal the kernel model (tests/bank_fft_exact.py) bit for
bit on random taps and input at every width up to K = 4096, at frame, ring and attach edges; designed taps
(subband_plan(bank=True, fft=True)) are held to 1e-5 of the float64 definition.  Refusals, id sharing with
direct banks, churn, device outputs, the host ring and the profile counters are checked too.
"""
import ctypes as C
import errno

import numpy as np
import pytest

from bank_exact import bank_walk, f64_bank
from bank_fft_exact import bank_fft_frames, bank_fft_max_taps, bank_fft_model
from bank_exact import bank_model
from cascade import FloatPath
from cascade_rational import stuff
from exact import to_complex
from util import assert_cf32_close, rand_block

pytestmark = pytest.mark.gpu

FMTS = ("cu8", "cs8", "cs16")
RAGGED = [8192, 8192, 2005, 0, 7, 8190, 8192, 333, 8192, 8192, 8192, 8192, 6000, 8192]


def conv(fmt, raw):
    return to_complex(fmt, raw).astype(np.complex64)


def copy_member(g, sid):
    return g.add_client_subband(sid, 1, np.ones(1, np.float32), 0)


def rand_taps(rng, T):
    return (rng.standard_normal(T) / np.sqrt(T)).astype(np.float32)


def run_rows(pkg, fs, max_in, blocks, fmt, banks, flags=0):
    """Feed `blocks`; banks: list of (fft, d1, taps, attach block, {channel: materialise block}).  Returns the
    rows {(bank index, channel): [per block from its materialisation]} and the bank ids."""
    g = pkg.Group(fs, max_in, flags=flags)
    bids, cids, rows = {}, {}, {}
    try:
        for b, x in enumerate(blocks):
            for i, (fft, d1, taps, at, chans) in enumerate(banks):
                if at == b:
                    bids[i] = (g.add_bank_fft if fft else g.add_bank)(d1, taps)
                for k, mb in chans.items():
                    if mb == b:
                        cids[(i, k)] = copy_member(g, g.add_bank_subband(bids[i], k))
                        rows[(i, k)] = []
            t = g.submit(fmt, x)
            g.wait(t)
            for key, cid in cids.items():
                rows[key].append(g.read_output(t, cid) if flags & pkg.XLG_OUT_DEVICE else g.output(t, cid))
                assert g.subband_info(cid)[1] == (8 if banks[key[0]][0] else 7)
    finally:
        g.close()
    return rows, bids


def model_rows(blocks, fmt, d1, taps, at, chans, fft=True):
    x = np.concatenate([conv(fmt, r) for r in blocks])
    sizes = [np.asarray(r).size // 2 for r in blocks]
    P = int(sum(sizes[:at]))
    out = (bank_fft_model if fft else bank_model)(taps, d1, list(chans), x, P, sizes[at:])
    return {k: out[k][mb - at:] for k, mb in chans.items()}


def assert_rows_equal(got, want, what):
    assert len(got) == len(want), what
    for b, (a, w) in enumerate(zip(got, want)):
        assert a.shape == w.shape, (what, b, a.shape, w.shape)
        assert np.array_equal(a, w), (what, b, np.max(np.abs(a - w)) if a.size else 0)


def refused(fn, *args, code=errno.EINVAL):
    with pytest.raises(ValueError) as e:
        fn(*args)
    assert e.value.args[0] == -code


WIDTHS = [2, 4, 8, 64, 128, 512, 1024, 4096]


@pytest.mark.parametrize("K", WIDTHS)
@pytest.mark.parametrize("case", ["short", "K", "ragged", "bound"])
def test_rows_bit_exact_against_the_model(pkg, K, case):
    """T1 < K, T1 = K, T1 % K != 0 and T1 at the bound; ragged, odd, empty and tiny blocks that wrap the ring
    (n1 of 0 and 1 among them); channels -D1, 0, D1 - 1 and random ones, odd and even."""
    d1 = K // 2
    T1 = {"short": max(1, K - 3), "K": K, "ragged": 3 * K + 5, "bound": bank_fft_max_taps(K)}[case]
    rng = np.random.default_rng(K * 31 + T1)
    fs = K * 48000
    chans = {-d1: 0, 0: 0, d1 - 1: 0}
    for k in rng.choice(np.arange(-d1, d1), size=min(4, K), replace=False):
        chans.setdefault(int(k), 0)
    if case == "bound":
        # the longest bank the kernel takes: blocks longer than its window (one odd), one format
        max_in = 2 * (T1 + 4 * K + 4096)
        sizes, fmts = [max_in, max_in // 2 + 1, 7, max_in], ("cs16",)
    else:
        max_in = max(8192, 2 * (T1 + 2 * K))
        sizes, fmts = [max_in if n == 8192 else n for n in RAGGED], FMTS
    for fmt in fmts:
        taps = rand_taps(rng, T1)
        blocks = [rand_block(rng, fmt, n) for n in sizes]
        rows, _ = run_rows(pkg, fs, max_in, blocks, fmt, [(True, d1, taps, 0, chans)])
        want = model_rows(blocks, fmt, d1, taps, 0, chans)
        for k in chans:
            assert_rows_equal(rows[(0, k)], want[k], (fmt, K, T1, k))


def frame_sizes(rng, max_in, d1, T1, targets, lead):
    """Raw block sizes after `lead` making the n1 of a bank attached before lead every value of targets, with
    full and random odd blocks between."""
    sizes = list(lead)
    for target in targets:
        for _ in range(int(rng.integers(1, 3))):
            sizes.append(max_in if rng.integers(0, 2) else int(rng.integers(1, max_in // 2)) * 2 + 1)
        counts = np.array([bank_walk([s // 2 for s in sizes] + [n], T1, d1)[0][-1] for n in range(max_in // 2 + 1)])
        sizes.append(2 * int(rng.choice(np.nonzero(counts == target)[0])))
    return sizes


@pytest.mark.parametrize("K", [16, 128, 1024])
def test_frames_per_cta_edges_and_attach_parity(pkg, K):
    """n1 at 0, 1 and on both sides of one and two CTAs' frames; bank A attached at block 0 (even P), bank B of
    the same width at an odd P, channels of both materialised after their attach."""
    d1, F = K // 2, bank_fft_frames(K)
    T1 = 2 * K + 3
    rng = np.random.default_rng(K + 1)
    fs, fmt = K * 48000, "cs8"
    max_in = 2 * (2 * F + 2) * d1 + 2 * T1
    sizes = frame_sizes(rng, max_in, d1, T1, [0, 1, F - 1, F, F + 1, 2 * F, 2 * F + 1], [2002])
    at_b = 1  # P = 1001
    ta, tb = rand_taps(rng, T1), rand_taps(rng, K - 1)
    chans_a = {-d1: 0, 1: 0, 2: 2, d1 - 1: 3}
    chans_b = {0: at_b, -1: at_b + 1, 3: at_b + 2}
    blocks = [rand_block(rng, fmt, n) for n in sizes]
    rows, _ = run_rows(pkg, fs, max_in, blocks, fmt, [(True, d1, ta, 0, chans_a), (True, d1, tb, at_b, chans_b)])
    wa = model_rows(blocks, fmt, d1, ta, 0, chans_a)
    wb = model_rows(blocks, fmt, d1, tb, at_b, chans_b)
    for k in chans_a:
        assert_rows_equal(rows[(0, k)], wa[k], ("A", k))
    for k in chans_b:
        assert_rows_equal(rows[(1, k)], wb[k], ("B", k))
    seen = set(bank_walk([n // 2 for n in sizes], T1, d1)[0])
    assert {0, 1, F - 1, F, F + 1, 2 * F, 2 * F + 1} <= seen, sorted(seen)


def test_every_channel_at_1024(pkg):
    """All 1024 channels of a K = 1024 bank materialised, in a shuffled order, each through its copy member."""
    K, d1 = 1024, 512
    rng = np.random.default_rng(1024)
    fs, max_in, fmt = K * 48000, 16384, "cs16"
    taps = rand_taps(rng, 3 * K + 17)
    chans = {int(k): 0 for k in rng.permutation(np.arange(-d1, d1))}
    blocks = [rand_block(rng, fmt, n) for n in [max_in, max_in, 9001, max_in, 0, max_in]]
    g_rows, _ = run_rows(pkg, fs, max_in, blocks, fmt, [(True, d1, taps, 0, chans)])
    want = model_rows(blocks, fmt, d1, taps, 0, chans)
    for k in chans:
        assert_rows_equal(g_rows[(0, k)], want[k], k)


def test_direct_and_fft_banks_share_ids(pkg):
    """A direct bank and an FFT bank in one group: ids come from one space and are reused across both kinds;
    each bank's rows are its own kernel's."""
    rng = np.random.default_rng(12)
    fs, max_in, fmt = 2048000, 8192, "cu8"
    g = pkg.Group(fs, max_in)
    rows = {}
    try:
        ta, tb, tc = rand_taps(rng, 61), rand_taps(rng, 100), rand_taps(rng, 37)
        a = g.add_bank(8, ta)
        b = g.add_bank_fft(8, tb)
        assert (a, b) == (0, 1)
        sa = g.add_bank_subband(a, 3)
        cids = {("a", 3): copy_member(g, sa), ("b", 3): copy_member(g, g.add_bank_subband(b, 3))}
        blocks = [rand_block(rng, fmt, n) for n in RAGGED]
        for i, x in enumerate(blocks):
            if i == 4:
                g.remove_client(cids.pop(("a", 3)))
                g.remove_subband(sa)
                g.remove_bank(a)
                c = g.add_bank_fft(16, tc)  # an FFT bank takes the direct bank's id
                assert c == a
                cids[("c", -16)] = copy_member(g, g.add_bank_subband(c, -16))
            if i == 9:
                d = g.add_bank(8, ta)  # and a direct bank the next free one
                assert d == 2
                cids[("d", -8)] = copy_member(g, g.add_bank_subband(d, -8))
            t = g.submit(fmt, x)
            g.wait(t)
            for key, cid in cids.items():
                rows.setdefault(key, []).append(g.output(t, cid))
                assert g.subband_info(cid)[1] == (7 if key[0] in "ad" else 8)
    finally:
        g.close()
    assert_rows_equal(rows[("a", 3)], model_rows(blocks[:4], fmt, 8, ta, 0, {3: 0}, fft=False)[3], "direct a")
    assert_rows_equal(rows[("b", 3)], model_rows(blocks, fmt, 8, tb, 0, {3: 0})[3], "fft b")
    assert_rows_equal(rows[("c", -16)], model_rows(blocks, fmt, 16, tc, 4, {-16: 4})[-16], "fft c")
    assert_rows_equal(rows[("d", -8)], model_rows(blocks, fmt, 8, ta, 9, {-8: 9}, fft=False)[-8], "direct d")


PLAN_RATES = [(61440000, "cs16", 64), (2048000, "cu8", 48), (20000000, "cs8", 48)]


def plan_clients(fs, n, rng):
    centres = rng.integers(-fs // 2 + 48000, fs // 2 - 48000, n)
    return [(int(c), 48000) for c in centres]


@pytest.mark.parametrize("fs,fmt,n", PLAN_RATES)
def test_designed_taps_within_1e_5_of_float64(pkg, fs, fmt, n):
    """subband_plan(bank=True, fft=True) at the front-end rates: every sampled member within 1e-5 of the
    float64 bank rows fed to the reference's float path.  At 20 Msps (K = 50) the plan keeps the direct bank."""
    rng = np.random.default_rng(fs % 1000 + n)
    max_in = 65536
    p = pkg.subband_plan(fs, plan_clients(fs, n, rng), bank=True, fft=True)
    d1, fs1 = p["d1"], p["fs1"]
    assert p["kernel"] == ("direct" if fs == 20000000 else "fft")
    blocks = [rand_block(rng, fmt, max_in) for _ in range(3)]
    g = pkg.Group(fs, max_in)
    try:
        bid = (g.add_bank_fft if p["kernel"] == "fft" else g.add_bank)(d1, p["taps1"])
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


def test_refusals(pkg):
    """Each refusal is logged and changes nothing: the next bank still takes id 0."""
    fs = 2048000
    g = pkg.Group(fs, 8192)
    try:
        t = np.ones(21, np.float32)
        refused(g.add_bank_fft, 0, t)
        refused(g.add_bank_fft, 8, np.zeros(0, np.float32))
        refused(g.add_bank_fft, 3, t)       # K = 6: not a power of two
        refused(g.add_bank_fft, 4096, t)    # K = 8192
        refused(g.add_bank_fft, 8, np.ones(bank_fft_max_taps(16) + 1, np.float32))
        refused(g.add_bank_fft, 2048, np.ones(bank_fft_max_taps(4096) + 1, np.float32))
        h = pkg.Group(1000000, 8192)  # 1 MHz % 128 != 0
        try:
            refused(h.add_bank_fft, 64, t)
        finally:
            h.close()
        bid = g.add_bank_fft(8, np.ones(bank_fft_max_taps(16), np.float32))
        assert bid == 0
        wide = g.add_bank_fft(2048, np.ones(bank_fft_max_taps(4096), np.float32))
        assert wide == 1
        sid = g.add_bank_subband(bid, -8)
        refused(g.add_bank_subband, bid, 8)
        refused(g.add_bank_subband, bid, -8, code=errno.EEXIST)
        cid = copy_member(g, sid)
        refused(g.remove_bank, bid, code=errno.EBUSY)
        x = np.zeros(8192, np.uint8)
        assert g._L.xlg_submit(g._h, pkg.FMT["cu8"], x.ctypes.data_as(C.c_void_p), x.size,
                               pkg.XLG_PATH_Q15) == -errno.ENOTSUP
        g.wait(g.submit("cu8", x))  # nothing was enqueued by the refused Q15 submit
        g.remove_client(cid)
        g.remove_subband(sid)
        g.remove_bank(bid)
        g.remove_bank(wide)
        refused(g.remove_bank, bid)
        assert g.add_bank(8, t) == 0
    finally:
        g.close()
    g = pkg.Group(fs, 8192, flags=pkg.XLG_TRACK_STATE)
    try:
        refused(g.add_bank_fft, 8, np.ones(21, np.float32), code=errno.ENOTSUP)
    finally:
        g.close()


def test_churn_device_outputs_host_ring_and_profile(pkg):
    """Channels added and removed, an FFT bank id reused, the ring grown by a longer FFT bank, outputs left on
    the device and a deeper host ring: rows stay the model's, and the profile counts are the shapes'.  The
    direct banks' profile counts nothing in a group of FFT banks only."""
    rng = np.random.default_rng(9)
    fs, max_in, fmt = 2048000, 8192, "cs16"
    blocks = [rand_block(rng, fmt, n) for n in RAGGED]
    ta = rand_taps(rng, 33)
    tb = rand_taps(rng, 9000)  # a longer history than the ring holds: it grows, keeping its samples
    for flags in (0, pkg.XLG_OUT_DEVICE):
        g = pkg.Group(fs, max_in, flags=flags, host_ring=8 if flags == 0 else 0)
        g.profile_enable(True)
        rows, cids = {}, {}
        try:
            for b, x in enumerate(blocks):
                if b == 0:
                    bid = g.add_bank_fft(8, ta)
                    for k in (-8, 3):
                        cids[k] = copy_member(g, g.add_bank_subband(bid, k))
                        rows[k] = []
                    sid_tmp = g.add_bank_subband(bid, 5)
                    tmp = copy_member(g, sid_tmp)
                if b == 3:
                    g.remove_client(tmp)
                    g.remove_subband(sid_tmp)
                    bid2 = g.add_bank_fft(32, tb)
                    sid_b = g.add_bank_subband(bid2, 1)
                    cids[("b", 1)] = copy_member(g, sid_b)
                    rows[("b", 1)] = []
                if b == 7:
                    g.remove_client(cids.pop(("b", 1)))
                    g.remove_subband(sid_b)
                    g.remove_bank(bid2)
                    assert g.add_bank_fft(32, tb) == bid2
                    cids[("c", -32)] = copy_member(g, g.add_bank_subband(bid2, -32))
                    rows[("c", -32)] = []
                t = g.submit(fmt, x)
                g.wait(t)
                for key, cid in cids.items():
                    rows[key].append(g.read_output(t, cid))
        finally:
            prof = g.bank_fft_profile_read()
            direct = g.bank_profile_read()
            g.close()
        want = model_rows(blocks, fmt, 8, ta, 0, {-8: 0, 3: 0})
        for k in (-8, 3):
            assert_rows_equal(rows[k], want[k], (flags, k))
        assert_rows_equal(rows[("b", 1)], model_rows(blocks[:7], fmt, 32, tb, 3, {1: 3})[1], (flags, "b"))
        assert_rows_equal(rows[("c", -32)], model_rows(blocks, fmt, 32, tb, 7, {-32: 7})[-32], (flags, "c"))
        sizes = [np.asarray(r).size // 2 for r in blocks]
        ca, _ = bank_walk(sizes, 33, 8)
        cb, _ = bank_walk(sizes[3:7], 9000, 32)
        cc, _ = bank_walk(sizes[7:], 9000, 32)
        assert prof["poly_macs"] == sum(n * 33 for n in ca) + sum(n * 9000 for n in cb + cc)
        assert prof["butterfly_flops"] == (sum(ca) * pkg.bank_fft_flops(16) + sum(cb + cc) * pkg.bank_fft_flops(64))
        n_b = [0] * 3 + cb + cc
        assert prof["fft_launches"] == sum(1 for a, b in zip(ca, n_b) if max(a, b) > 0)
        assert prof["fft_ms"] > 0
        assert direct == {"bank_ms": 0.0, "bank_launches": 0, "poly_macs": 0, "dft_macs": 0}


def test_group_without_fft_banks_profiles_nothing(pkg):
    g = pkg.Group(2048000, 8192)
    try:
        g.profile_enable(True)
        g.add_client(32, pkg.create_low_pass_filter(1.0, 2048000, 24000, 9600), 1000)
        copy_member(g, g.add_bank_subband(g.add_bank(8, np.ones(21, np.float32)), 2))
        g.wait(g.submit("cu8", np.zeros(8192, np.uint8)))
        assert g.bank_fft_profile_read() == {"fft_ms": 0.0, "fft_launches": 0, "poly_macs": 0, "butterfly_flops": 0}
        assert g.bank_profile_read()["bank_launches"] == 1
    finally:
        g.close()
