"""Members of FFT bank channels bit for bit on random taps and input: the FFT bank kernel's rows chained into the
member kernels (bank_fft_member_model's chain, tests/bank_fft_exact.py, driven by tests/bank_fft_rig.py)
predicts every member output exactly, for integer and rational members at any offset, with tickets in flight in
every pipeline variant of the bank tests, through churn that grows the input ring and in randomised mixed
populations of FFT banks, direct banks, sub-bands and neighbour clients.  Channels with a copy member from their
first block are also checked against member_model fed the GPU's own rows, so a failure names its stage.

Every member of an FFT bank channel is asserted to be on a kind-8 channel (xlg_subband_info).
"""
import numpy as np
import pytest

from bank_exact import XLG_SLOTS, ring_cap
from bank_fft_rig import FFT_BANK, FftRig, fft_taps
from cascade import small_taps
from exact import dyadic_taps, exact_input
from subband_rig import BANK, dyadic_member, dyadic_stage_a, one_hot_member
from util import rand_block

pytestmark = pytest.mark.gpu

FMTS = ("cu8", "cs8", "cs16")


def row(max_in, d1):
    return max_in // 2 // d1 + 8


INT_SHAPES = [(5, 23), (4, 8), (1, 1), (6, 40), (2, 31), (3, 250)]  # (D2, T2)
RAT_SHAPES = [(2, 5, 33), (3, 7, 40), (12, 5, 60)]                 # (L2, M2, T2)
RAGGED = [16384, 16384, 4005, 0, 7, 16382, 16384, 333, 16384, 16384, 16384, 9001, 16384, 16384]


@pytest.mark.parametrize("fmt", FMTS)
def test_members_at_any_offset(pkg, monkeypatch, fmt):
    """Channels -D1, 0, D1 - 1 from block 0 and an odd and an even one materialised at block 2; integer
    members with odd and even D2, T2 = 1, short and long; rational L2 = 2, 3, 12; offsets 0, +-fs1/4 and
    arbitrary; attached at the channel's first block and at block 5."""
    rng = np.random.default_rng(200 + FMTS.index(fmt))
    fs, max_in, d1 = 2048000, 16384, 8
    fs1 = fs // d1
    offsets = [0, fs1 // 4, -fs1 // 4, int(rng.integers(-fs1 // 2, fs1 // 2))]
    rig = FftRig(pkg, monkeypatch, fs, max_in, fmt, depth=XLG_SLOTS, reserve=400 * row(max_in, d1))
    bk = rig.add_bank_fft(d1, fft_taps(rng, 61))

    def attach(sb, n):
        shapes = [(1, d2, T2) for d2, T2 in INT_SHAPES] + RAT_SHAPES
        for i, (l2, d2, T2) in enumerate(shapes[:n]):
            rig.add_member(sb, l2, d2, fft_taps(rng, T2), offsets[(i + sb.chan) % 4], False)

    chans = {}
    for b, n in enumerate(RAGGED):
        if b == 0:
            for k in (-d1, 0, d1 - 1):
                chans[k] = rig.add_channel(bk, k, copy=True)
                attach(chans[k], 9)
        if b == 2:
            for k in (3, -2):
                chans[k] = rig.add_channel(bk, k, copy=True)
                attach(chans[k], 9)
        if b == 5:
            for k in (-d1, 3):
                attach(chans[k], 9)
        rig.submit(rand_block(rng, fmt, n))
    rig.check()
    assert rig.kinds() == {FFT_BANK}
    for m in rig.mems:
        assert np.count_nonzero(np.concatenate(m.got)) > 0, m.label()
    rig.close()


PIPE = {"default": ({}, None, 0), "conv_on_compute_stream": ({"XLATING_B200_CONV_STREAM": "0"}, None, 0),
        "no_spec_1stream": ({"XLATING_B200_SPECULATE": "0", "XLATING_B200_CSTREAMS": "1"}, None, 0),
        "partition": ({"XLATING_B200_PARTITION": "1"}, None, 0),
        "no_partition": ({"XLATING_B200_PARTITION": "0"}, None, 0),
        "sm_partition": ({"XLATING_B200_PARTITION": "1"}, "XLG_SM_PARTITION", 0),
        "out_device": ({}, "XLG_OUT_DEVICE", 0), "host_ring": ({}, None, 12)}


@pytest.mark.parametrize("group", ["fft_only", "beside_clients_and_a_direct_bank"])
@pytest.mark.parametrize("variant", list(PIPE))
def test_tickets_in_flight(pkg, monkeypatch, variant, group):
    """An FFT-bank-only group (no pre-pass), and an FFT bank beside dyadic integer clients (the speculative
    pre-pass runs) and a direct bank."""
    env, flag, host_ring = PIPE[variant]
    rng = np.random.default_rng(sum(map(ord, variant + group)))
    fs, max_in, fmt = 2048000, 16384, "cs8"
    fs1 = fs // 8
    depth = host_ring or XLG_SLOTS
    rig = FftRig(pkg, monkeypatch, fs, max_in, fmt, flags=getattr(pkg, flag) if flag else 0, host_ring=host_ring,
                 depth=depth, env=env, reserve=64 * row(max_in, 8))
    bk = rig.add_bank_fft(8, fft_taps(rng, 61))
    for k in (-8, 2, 5):
        sb = rig.add_channel(bk, k, copy=True)
        rig.add_member(sb, 1, 5, fft_taps(rng, 23), int(rng.integers(-fs1 // 2, fs1 // 2)), False)
        rig.add_member(sb, 3, 7, fft_taps(rng, 40), fs1 // 4, False)
    if group != "fft_only":
        for s in [("i", 32, dyadic_taps(rng, 505, fmt)), ("i", 8, dyadic_taps(rng, 97, fmt))]:
            rig.add_neighbour(s)
        db = rig.add_bank(8, fft_taps(rng, 45))
        sb = rig.add_channel(db, 3, copy=True)
        rig.add_member(sb, 1, 4, fft_taps(rng, 8), 1000, False)
    sizes = [max_in] * 5 + [15001, max_in, max_in, 12347, max_in, max_in, max_in - 2, max_in, max_in]
    for n in sizes:
        rig.submit(exact_input(rng, fmt, n))
    rig.check()
    assert rig.kinds() == ({FFT_BANK} if group == "fft_only" else {FFT_BANK, BANK})
    rig.close()


def test_churn_in_flight(pkg, monkeypatch):
    """With tickets in flight: channels and members added and removed, an FFT bank removed and its id reused
    by a direct bank, and an FFT bank longer than the ring's history (12300 taps) that grows the input ring,
    keeping its samples."""
    rng = np.random.default_rng(67)
    fs, max_in, fmt = 2048000, 8192, "cs16"
    fs1 = fs // 8
    rig = FftRig(pkg, monkeypatch, fs, max_in, fmt, depth=XLG_SLOTS, reserve=200 * row(max_in, 2))
    a = rig.add_bank_fft(8, fft_taps(rng, 33))
    ch = {k: rig.add_channel(a, k, copy=True) for k in (-8, 2)}
    tmp = rig.add_channel(a, 5, copy=True)
    m_a = rig.add_member(ch[2], 1, 4, fft_taps(rng, 8), 5000, False)
    b2 = long_b = None
    assert ring_cap(max_in, 12299) > ring_cap(max_in, 4096)
    for blk in range(24):
        if blk == 2:
            rig.remove_member(tmp.copy)
            rig.remove_subband(tmp)
            b2 = rig.add_bank_fft(2, fft_taps(rng, 40))
            sb = rig.add_channel(b2, 1, copy=True)
            rig.add_member(sb, 2, 5, fft_taps(rng, 33), -(fs // 2) // 4, False)
        if blk == 4:
            rig.remove_member(m_a)
            rig.add_member(ch[-8], 1, 5, fft_taps(rng, 23), 777, False)
            rig.add_channel(a, 5, copy=True)
        if blk == 7:
            for m in [m for m in rig.mems if m.sb.bank is b2 and m.last is None]:
                rig.remove_member(m)
            for sb in [sb for sb in rig.sbs if sb.bank is b2 and sb.last is None]:
                rig.remove_subband(sb)
            rig.remove_bank(b2)
            b3 = rig.add_bank(4, fft_taps(rng, 41))  # a direct bank takes the FFT bank's id
            assert b3.bid == b2.bid
            sb = rig.add_channel(b3, -4, copy=True)
            rig.add_member(sb, 1, 3, fft_taps(rng, 9), 0, False)
        if blk == 10:
            long_b = rig.add_bank_fft(32, fft_taps(rng, 12300))
            for k in (-32, 7):
                sb = rig.add_channel(long_b, k, copy=True)
                rig.add_member(sb, 1, 2, fft_taps(rng, 31), 1234, False)
        if blk == 14:
            rig.add_member(ch[2], 12, 5, fft_taps(rng, 60), fs1 // 5, False)
        rig.submit(rand_block(rng, fmt, max_in if blk % 3 else max_in - 2 * (blk % 5) - 3))
    rig.check()
    assert rig.kinds() == {FFT_BANK, BANK}
    assert long_b.first == 10
    rig.close()


MIX_VARIANTS = ["default", "no_renorm", "out_device", "host_ring", "sm_partition", "no_spec_1stream"]
MIX_D1 = [1, 2, 4, 8, 16, 32, 64, 128, 256, 512]  # 2 D1 a power of two dividing 2048000 * 2


def mix_neighbour(rng, fmt):
    k = int(rng.integers(0, 3))
    if k == 0:
        D, T = [(32, 505), (8, 97), (5, 40)][int(rng.integers(0, 3))]
        return ("i", D, dyadic_taps(rng, T, fmt))
    if k == 1:
        L, M, T = [(3, 128, 97), (5, 3, 40)][int(rng.integers(0, 2))]
        return ("r", L, M, dyadic_taps(rng, T, fmt))
    return ("c", 8, small_taps(rng, 17, 3), 5, small_taps(rng, 23, 3))


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
    return rig.add_member(sb, l2, d2, fft_taps(rng, T2), int(rng.integers(-fs1 // 2, fs1 // 2)), False)


@pytest.mark.parametrize("seed", range(8))
def test_random_mixed_populations(pkg, monkeypatch, seed):
    """FFT banks of random width and taps (up to their bound at small K) with random channels, a direct bank on
    odd seeds, an ordinary sub-band and neighbours; members added and removed twice with tickets in flight."""
    rng = np.random.default_rng(9100 + seed)
    fs = 4096000
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
    rig = FftRig(pkg, monkeypatch, fs, max_in, fmt, flags=flags, host_ring=host_ring, depth=depth, env=env,
                 reserve=150 * row(max_in, 1))
    for _ in range(int(rng.integers(1, 4))):
        rig.add_neighbour(mix_neighbour(rng, fmt))
    chans = []
    for i in range(int(rng.integers(1, 4))):
        d1 = int(rng.choice(MIX_D1))
        T1 = int(rng.integers(1, min(3000, 16 * 2 * d1) + 1))
        bk = rig.add_bank_fft(d1, fft_taps(rng, T1))
        n_ch = int(rng.integers(1, min(2 * d1, 40) + 1))
        for k in rng.choice(np.arange(-d1, d1), n_ch, replace=False).tolist():
            chans.append(rig.add_channel(bk, int(k), copy=bool(rng.integers(0, 4) == 0)))
    if seed % 2:
        bk = rig.add_bank(5, fft_taps(rng, int(rng.integers(1, 200))))
        chans += [rig.add_channel(bk, int(k)) for k in rng.choice(np.arange(-5, 5), 3, replace=False)]
    sbs = [rig.add_subband(8, dyadic_stage_a(rng, 8, 17), 0, True)]
    targets = chans + sbs
    mix_member(rng, rig, chans[0])  # (an FFT bank's channel)
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
    assert FFT_BANK in rig.kinds()
    rig.close()
