"""The bank references (tests/bank_exact.py) checked on the CPU, before any GPU test relies on them.

* the float64 definition is, for odd T1, the float64 sub-band (the reference filter at k * fs / K) and holds
  the oracle's sub-band to float32 accuracy (the identity);
* the kernel model equals the float64 definition bit for bit on exact stimuli (dyadic taps, grid input,
  channels whose twiddles are +-1 or +-i), and is within float32 accuracy of it at any channel;
* mutations of the model each fail the exact harness;
* bank_member_model (the bank model's rows fed to the member model) equals the float64 composition on exact
  stimuli, stays within float32 accuracy of the streaming oracle on random data, and every mutation of either
  stage changes its output;
* ring_cap and bank_ctas follow the walk;
* subband_plan(bank=True) puts every sub-band on the bank's grid with offsets within fs1 / 4 and counts the
  first stage as one polyphase pass and C channel sums; the default plan is the one of the sub-band workloads.
"""
import os
import sys

import numpy as np
import pytest

import subband_exact
from bank_exact import (MUTATIONS, BankMemberOracle, bank_ctas, bank_member_model, bank_model, bank_walk, f64_bank,
                        ring_cap, twiddles)
from cascade import f64_filter, filter_constants
from exact import dyadic_taps, exact_input, to_complex
from subband_exact import f64_member
from subband_rig import dyadic_member
from oracle import pyoracle as po

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))

SIZES = [4096, 1002, 7, 0, 2, 4094, 333]


def stream(rng, fmt, sizes):
    raw = [exact_input(rng, fmt, 2 * n) for n in sizes]
    return raw, np.concatenate([to_complex(fmt, r) for r in raw])


def exact_channels(D1):
    """Channels whose twiddles are all +-1 or +-i: k * 4 divisible by K = 2 * D1."""
    return sorted({k for k in range(-D1, D1) if (4 * k) % (2 * D1) == 0})


def test_twiddles_are_exact_at_quarter_turns():
    for K in (2, 4, 6, 14, 20, 64, 128):
        w = twiddles(K).astype(complex)
        assert np.max(np.abs(w - np.exp(-2j * np.pi * np.arange(K) / K))) < 1e-7
        for j in range(0, K, 1):
            if (4 * j) % K == 0:
                assert w[j] == [1, -1j, -1, 1j][4 * j // K]


@pytest.mark.parametrize("D1,T1", [(1, 5), (2, 9), (3, 13), (7, 101), (10, 61), (4, 8)])
def test_f64_definition_is_the_subband_for_odd_taps(D1, T1):
    rng = np.random.default_rng(D1 * 100 + T1)
    fs = 2 * D1 * 96000
    taps = rng.standard_normal(T1)
    _, x = stream(rng, "cs16", SIZES)
    chans = list(range(-D1, D1))
    got = f64_bank(taps, D1, chans, x, 0, SIZES)
    blocks = np.split(x, np.cumsum(SIZES)[:-1])
    for k in chans:
        ref = f64_filter(taps, D1, k * fs // (2 * D1), fs, blocks)
        err = max((np.max(np.abs(a - b)) for a, b in zip(got[k], ref) if a.size), default=0.0)
        if T1 % 2:
            assert err < 1e-9, (k, err)
        elif k % (2 * D1) != 0:
            assert err > 1e-6  # the reference's middle-pair swap breaks the identity for even T1


def subband_drift(D1, k, fs):
    """Phase error per output of the reference's sub-band at k * fs / K: its float oscillator step is
    cexpf(-float(w0) * D1), not (-1)^k exactly."""
    _, (ir, ii) = filter_constants(np.ones(1, np.float32), D1, k * fs // (2 * D1), fs)
    return abs(np.angle(complex(ir, ii) * (-1) ** k))


@pytest.mark.parametrize("D1,T1,fmt", [(2, 9, "cu8"), (7, 101, "cs8"), (10, 61, "cs16")])
def test_f64_definition_holds_the_oracle_subband(D1, T1, fmt):
    """Within 1e-5 norm-wise plus the phase the oracle's float oscillator has drifted by its last output."""
    rng = np.random.default_rng(T1)
    fs = 2 * D1 * 100000
    taps = (rng.standard_normal(T1) / T1).astype(np.float32)
    raw, x = stream(rng, fmt, SIZES)
    for k in (-D1, -1, 0, D1 // 2, D1 - 1):
        got = f64_bank(taps, D1, [k], x, 0, SIZES)[k]
        o = po.OracleFilter(D1, taps, k * fs // (2 * D1), fs, 2 * max(SIZES))
        drift, done = subband_drift(D1, k, fs), 0
        scale = max(np.max(np.abs(a)) for a in got if a.size)
        for a, r in zip(got, raw):
            b = o.process_cf32(fmt, r)
            assert a.shape == b.shape
            done += a.size
            if a.size:
                tol = 1e-5 + 2 * drift * done + 4e-7 * T1  # (+ the float rotation of the taps, theta = i * w0)
                assert np.max(np.abs(a - b)) <= tol * scale, (k, drift)


@pytest.mark.parametrize("D1,T1,attach", [(1, 3, 0), (2, 4, 2), (2, 9, 0), (3, 6, 1), (4, 31, 2), (7, 14, 0),
                                          (10, 61, 5), (32, 64, 1), (64, 200, 0)])
def test_model_is_exact_on_exact_stimuli(D1, T1, attach):
    rng = np.random.default_rng(D1 * 7 + T1)
    for fmt in ("cu8", "cs8", "cs16"):
        taps = dyadic_taps(rng, T1, fmt)
        _, x = stream(rng, fmt, SIZES)
        P = int(sum(SIZES[:attach]))
        chans = exact_channels(D1)
        ref = f64_bank(taps, D1, chans, x, P, SIZES[attach:])
        got = bank_model(taps, D1, chans, x.astype(np.complex64), P, SIZES[attach:])
        for k in chans:
            for a, b in zip(got[k], ref[k]):
                assert np.array_equal(a.astype(complex), b), (fmt, k)


@pytest.mark.parametrize("D1,T1", [(3, 13), (7, 101), (10, 61)])
def test_model_is_within_float32_of_the_definition(D1, T1):
    rng = np.random.default_rng(T1)
    taps = (rng.standard_normal(T1) / np.sqrt(T1)).astype(np.float32)
    _, x = stream(rng, "cs8", SIZES)
    chans = list(range(-D1, D1))
    ref = f64_bank(taps, D1, chans, x, 0, SIZES)
    got = bank_model(taps, D1, chans, x.astype(np.complex64), 0, SIZES)
    for k in chans:
        a, b = np.concatenate(got[k]), np.concatenate(ref[k])
        assert np.max(np.abs(a - b)) <= 1e-5 * np.max(np.abs(b)), k


@pytest.mark.parametrize("mutation", MUTATIONS)
def test_every_mutation_fails_the_exact_harness(mutation):
    rng = np.random.default_rng(5)
    D1, T1, attach = 4, 24, 2  # (an odd window phase r_m: r0_negated moves the quarter turns)
    taps = dyadic_taps(rng, T1, "cs8")
    _, x = stream(rng, "cs8", SIZES)
    P = int(sum(SIZES[:attach]))
    chans = exact_channels(D1)
    ref = f64_bank(taps, D1, chans, x, P, SIZES[attach:])
    got = bank_model(taps, D1, chans, x.astype(np.complex64), P, SIZES[attach:], mutation=mutation)
    assert any(not np.array_equal(a.astype(complex), b) for k in chans for a, b in zip(got[k], ref[k]))


def test_walk_is_the_integer_clients():
    counts, firsts = bank_walk([10, 3, 0, 7], 5, 3)
    assert counts == [4, 1, 0, 2] and firsts == [-4, 8, 11, 11]


# subband_plan at the sub-band workloads (tools/subband_bench.py): (d1, sub-bands, FMAs, sum of centres) of
# the default plan as it was before bank=True existed
DEFAULT_PLANS = {"61M_1024": (32, 65, 2863.575, 12097540), "61M_4096": (64, 129, 5850.238, 10889148),
                 "2M_256": (7, 14, 2600.0, 431354), "2048k_256": (10, 20, 1976.0, 81780),
                 "10M_256": (20, 40, 1571.315, -1600680), "20M_256": (20, 41, 1494.258, 5015366)}


@pytest.mark.parametrize("name", sorted(DEFAULT_PLANS))
def test_bank_plan_is_on_the_grid_and_the_default_is_unchanged(pkg, name):
    import subband_bench as sbb
    fs = sbb.WORKLOADS[name][0]
    clients = sbb.workload_clients(name)
    p = pkg.subband_plan(fs, clients)
    assert (p["d1"], len(p["subbands"]), round(p["fmas"], 3), sum(s["center"] for s in p["subbands"])) == \
        DEFAULT_PLANS[name]
    assert all("channel" not in s for s in p["subbands"])
    b = pkg.subband_plan(fs, clients, bank=True)
    d1, fs1 = b["d1"], b["fs1"]
    assert fs % (2 * d1) == 0 and fs1 == fs // d1 and pkg.bank_fits(d1, b["taps1"].size)
    half = fs1 // 2
    chans = [s["channel"] for s in b["subbands"]]
    assert len(set(chans)) == len(chans) and all(-d1 <= k < d1 for k in chans)
    for s in b["subbands"]:
        assert s["center"] == s["channel"] * half
    for m, (c, r) in zip(b["members"], clients):
        assert m["center"] == c and m["rate"] == r
        assert abs(m["offset"]) * 4 <= fs1
        k = b["subbands"][m["subband"]]["channel"]
        assert (c - m["offset"]) % fs == (k * half) % fs  # its own grid point is its channel's centre
    shapes = [(m["rate"], m["taps2"].size, m["interp2"]) for m in b["members"]]
    want = 2.0 * b["taps1"].size / d1 + 8.0 * len(chans) + pkg.subband_fmas(fs, d1, b["taps1"].size, 0, shapes)
    assert b["fmas"] == pytest.approx(want, rel=1e-12)


def test_bank_fits_is_the_kernel_bound(pkg):
    for d1 in (1, 2, 7, 10, 32, 64, 128):
        t = 1
        while pkg.bank_fits(d1, t * 2):
            t *= 2
        lo, hi = t, t * 2
        while hi - lo > 1:
            mid = (lo + hi) // 2
            lo, hi = (mid, hi) if pkg.bank_fits(d1, mid) else (lo, mid)
        K = 2 * d1
        tpad = ((-(-lo // K) * K) + 3) & ~3
        smem = 16 + 4 * tpad + 8 * ((31 * d1 + lo + 2) & ~1) + 8 * K + 8 * 32 * (K + 1)
        assert smem <= 200 * 1024 and not pkg.bank_fits(d1, lo + 1)


def test_streaming_member_oracle_follows_the_definition():
    from bank_exact import BankMemberOracle
    rng = np.random.default_rng(2)
    D1, T1, fs = 5, 37, 960000
    taps = rng.standard_normal(T1).astype(np.float32)
    raw, x = stream(rng, "cu8", SIZES)
    for k in (-5, -2, 0, 4):
        o = BankMemberOracle(D1, taps, k, 1, np.ones(1, np.float32), 0, 1, fs)
        ref = f64_bank(taps, D1, [k], x, 0, SIZES)[k]
        for r, w in zip(raw, ref):
            got = o.process_cf32("cu8", r)
            assert np.array_equal(got, w.astype(np.complex64)) or np.max(np.abs(got - w)) <= 1e-6 * max(
                np.max(np.abs(w)), 1.0)


# ---------------------------------------------------------------------------
# the chain: bank rows into the member kernels
# ---------------------------------------------------------------------------
CHAIN_INT = [(1, 1), (3, 9), (4, 8), (5, 23), (2, 31)]  # (D2, T2)
CHAIN_RAT = [(2, 5, 33), (3, 7, 40), (12, 5, 60)]       # (L2, M2, T2)


@pytest.mark.parametrize("D1,T1,fmt", [(2, 9, "cu8"), (4, 31, "cs8"), (10, 61, "cs16"), (32, 70, "cs8")])
def test_chain_is_exact_on_exact_stimuli(D1, T1, fmt):
    """Dyadic bank taps, quarter-turn channels, dyadic full-length members at offset 0 within exact_bound:
    the chain equals f64_bank's rows fed to f64_member, with the bank attached after block 0, the channel
    materialised a block later and members attached at the channel's first block and two blocks on."""
    rng = np.random.default_rng(D1 * 13 + T1)
    fs = 2 * D1 * 96000
    taps1 = dyadic_taps(rng, T1, fmt)
    _, x = stream(rng, fmt, SIZES)
    P, sizes = SIZES[0], SIZES[1:]
    for k in exact_channels(D1):
        for attach in (0, 2):
            members = [(1, d2, dyadic_member(rng, taps1, T2, fmt), 0) for d2, T2 in CHAIN_INT]
            members += [(l2, m2, dyadic_member(rng, taps1, T2, fmt), 0) for l2, m2, T2 in CHAIN_RAT]
            got = bank_member_model(taps1, D1, k, x.astype(np.complex64), P, sizes, members, fs, mat=1,
                                    attach=attach)
            rows = f64_bank(taps1, D1, [k], x, P, sizes)[k][1:]
            for (l2, d2, taps2, _), y in zip(members, got):
                want = f64_member(rows[attach:], l2, d2, taps2, fs // D1)
                assert len(y) == len(want)
                for a, w in zip(y, want):
                    assert np.array_equal(a, w), (fmt, k, l2, d2, taps2.size, attach)


@pytest.mark.parametrize("D1,T1,fmt", [(3, 13, "cu8"), (7, 101, "cs8"), (20, 45, "cs16")])
def test_chain_is_within_float32_of_the_oracle(D1, T1, fmt):
    """Random taps and input, members at offsets 0, +-fs1/4 and arbitrary: within 1e-5 norm-wise of
    BankMemberOracle (the float64 rows fed to the reference's float path)."""
    rng = np.random.default_rng(T1 + 3)
    fs = 2 * D1 * 48000
    fs1 = fs // D1
    taps1 = (rng.standard_normal(T1) / np.sqrt(T1)).astype(np.float32)
    raw, x = stream(rng, fmt, SIZES)
    offsets = [0, fs1 // 4, -fs1 // 4, int(rng.integers(-fs1 // 2, fs1 // 2))]
    shapes = [(1, d2, T2) for d2, T2 in CHAIN_INT] + list(CHAIN_RAT)
    for k in (-D1, 0, D1 - 1, 1):
        members = [(l2, d2, (rng.standard_normal(T2) / np.sqrt(T2)).astype(np.float32), offsets[i % 4])
                   for i, (l2, d2, T2) in enumerate(shapes)]
        got = bank_member_model(taps1, D1, k, x.astype(np.complex64), 0, SIZES, members, fs)
        for (l2, d2, taps2, off), y in zip(members, got):
            o = BankMemberOracle(D1, taps1, k, d2, taps2, off, l2, fs)
            want = [o.process_cf32(fmt, r) for r in raw]
            a, b = np.concatenate(y), np.concatenate(want)
            assert a.shape == b.shape
            assert np.max(np.abs(a - b)) <= 1e-5 * np.max(np.abs(b)), (k, l2, d2, off)


@pytest.mark.parametrize("mutation", MUTATIONS + subband_exact.MUTATIONS)
def test_every_mutation_changes_the_chain(mutation):
    """Random data: the bank attached at an odd P, the channel materialised with it, a class of 33 integer
    members (odd Tb: tap rows of sb_tpad, not Tb, apart; one phase row past 32) at distinct offsets and a
    rational class of L2 = 3, attached with the channel or (the member mutations) after its rows began."""
    rng = np.random.default_rng(8)
    D1, T1, fs = 5, 37, 960000
    fs1 = fs // D1
    taps1 = rng.standard_normal(T1).astype(np.float32)
    _, x = stream(rng, "cs16", SIZES)
    x = x.astype(np.complex64)
    members = [(1, 4, rng.standard_normal(23).astype(np.float32), int(rng.integers(-fs1 // 2, fs1 // 2)))
               for _ in range(33)]
    members += [(3, 7, rng.standard_normal(40).astype(np.float32), 1000 * i) for i in range(3)]
    P, sizes = sum(SIZES[:3]), SIZES[3:]
    args = (taps1, D1, 3, x, P, sizes, members, fs)
    attach = 0 if mutation in MUTATIONS else 3  # (the bank's: rows whose windows reach back before P)
    base = bank_member_model(*args, attach=attach)
    got = bank_member_model(*args, attach=attach, mutation=mutation)
    assert any(not np.array_equal(a, b) for ya, yb in zip(base, got) for a, b in zip(ya, yb)), mutation


def test_ring_cap_and_bank_ctas_follow_the_walk():
    assert ring_cap(8192, 0) == 32768 and ring_cap(8192, 12300) == 65536 and ring_cap(65536, 4096) == 262144
    sizes, T1, D1, P, cap = [1000, 37, 0, 2001], 300, 7, 5, 64
    counts, firsts = bank_walk(sizes, T1, D1)
    ctas = bank_ctas(sizes, T1, D1, P, cap)
    assert [len(c) for c in ctas] == [-(-n // 32) for n in counts]
    for n1, first, cs in zip(counts, firsts, ctas):
        for x, (w0, shift, need, split, pre) in enumerate(cs):
            nf = min(32, n1 - 32 * x)
            assert w0 == P + first + 32 * x * D1 and shift == w0 % 2 and need % 2 == 0
            assert need >= (nf - 1) * D1 + T1 + shift and split == ((w0 - shift) % cap + need > cap)
            assert pre == (w0 - shift < P)
    assert ctas[0][1][4] and not ctas[3][0][4]  # T1 > 32 D1: CTA 1 of the first block reads before P
