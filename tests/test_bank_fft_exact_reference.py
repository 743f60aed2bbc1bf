"""The FFT bank references (tests/bank_fft_exact.py) checked on the CPU, before any GPU test relies on them.

* the kernel model equals the float64 definition of the bank (bank_exact.f64_bank) bit for bit on exact
  stimuli at K = 2 and 4, where every twiddle is +-1 or +-i, and is within NORM_BOUND of it norm-wise at every
  K up to 4096 (the largest error measured below is 2.3e-7, a margin of more than 4x);
* each mutation of the model fails that harness;
* bank_fft_member_model (the model's rows fed to the member model) equals the float64 composition on exact
  stimuli and stays within 1e-5 of the streaming oracle on random data;
* the row layout, the butterfly count and the tap bound are the kernel's (bank_fft_pos, xlg_bank_fft_flops,
  bank_fft_fits);
* subband_plan(..., fft=False) is the plan of before FFT banks existed on the sub-band workloads, and fft=True
  returns FFT banks only at power-of-two K that the kernel takes, and the cheaper kernel.
"""
import os
import sys

import numpy as np
import pytest

from bank_exact import BankMemberOracle, f64_bank
from bank_fft_exact import (MUTATIONS, bank_fft_max_taps, bank_fft_member_model, bank_fft_model, bank_fft_pos,
                            fft_stages)
from exact import dyadic_taps, exact_input, to_complex
from subband_exact import f64_member
from subband_rig import dyadic_member

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))

SIZES = [4096, 1002, 7, 0, 2, 4094, 333]
NORM_BOUND = 1e-6


def stream(rng, fmt, sizes):
    raw = [exact_input(rng, fmt, 2 * n) for n in sizes]
    return raw, np.concatenate([to_complex(fmt, r) for r in raw])


def norm_err(got, ref, chans):
    return max(np.linalg.norm(np.concatenate(got[k]) - np.concatenate(ref[k])) /
               max(np.linalg.norm(np.concatenate(ref[k])), 1e-30) for k in chans)


@pytest.mark.parametrize("D1,T1,attach", [(1, 1, 0), (1, 2, 1), (1, 9, 0), (2, 1, 2), (2, 3, 1), (2, 4, 0),
                                          (2, 31, 3), (2, 64, 1)])
def test_model_is_exact_on_exact_stimuli(D1, T1, attach):
    """K = 2 and 4: T1 < K, = K and beyond, attached at odd and even P, every channel."""
    rng = np.random.default_rng(D1 * 7 + T1)
    for fmt in ("cu8", "cs8", "cs16"):
        taps = dyadic_taps(rng, T1, fmt)
        _, x = stream(rng, fmt, SIZES)
        P = int(sum(SIZES[:attach]))
        chans = list(range(-D1, D1))
        ref = f64_bank(taps, D1, chans, x, P, SIZES[attach:])
        got = bank_fft_model(taps, D1, chans, x.astype(np.complex64), P, SIZES[attach:])
        for k in chans:
            assert len(got[k]) == len(ref[k])
            for a, b in zip(got[k], ref[k]):
                assert np.array_equal(a.astype(complex), b), (fmt, k)


@pytest.mark.parametrize("D1,T1", [(4, 5), (4, 8), (4, 37), (8, 16), (16, 100), (64, 128), (64, 300),
                                   (128, 1000), (256, 513), (512, 2000), (2048, 5000)])
def test_model_is_within_the_norm_bound_of_the_definition(D1, T1):
    """K = 8 .. 4096 on random taps and input: every channel (K <= 128) or a spread of them within NORM_BOUND
    norm-wise.  Measured: 5.7e-8 at K = 8, 1.2e-7 at K = 128 to 512, 1.5e-7 at K = 1024, 2.3e-7 at
    K = 4096."""
    rng = np.random.default_rng(T1)
    K = 2 * D1
    taps = (rng.standard_normal(T1) / np.sqrt(T1)).astype(np.float32)
    sizes = [3000, 7, 0, 5000]
    _, x = stream(rng, "cs16", [1234] + sizes)
    chans = list(range(-D1, D1)) if K <= 128 else sorted({-D1, -1, 0, 1, 3, D1 // 3, D1 - 1})
    ref = f64_bank(taps, D1, chans, x, 1234, sizes)
    got = bank_fft_model(taps, D1, chans, x.astype(np.complex64), 1234, sizes)
    assert norm_err(got, ref, chans) <= NORM_BOUND


@pytest.mark.parametrize("mutation", MUTATIONS)
def test_every_mutation_fails_the_harness(mutation):
    """K = 32 (radix-4 stages at 32 and 8, then radix 2), T1 = 20 < K, the bank attached at an odd P."""
    rng = np.random.default_rng(5)
    D1, T1 = 16, 20
    taps = (rng.standard_normal(T1) / np.sqrt(T1)).astype(np.float32)
    _, x = stream(rng, "cs8", SIZES)
    P = int(sum(SIZES[:3]))
    assert P % 2 == 1
    chans = list(range(-D1, D1))
    ref = f64_bank(taps, D1, chans, x, P, SIZES[3:])
    assert norm_err(bank_fft_model(taps, D1, chans, x.astype(np.complex64), P, SIZES[3:]), ref, chans) <= NORM_BOUND
    got = bank_fft_model(taps, D1, chans, x.astype(np.complex64), P, SIZES[3:], mutation=mutation)
    assert norm_err(got, ref, chans) > NORM_BOUND, mutation


def test_row_layout_butterflies_and_tap_bound(pkg):
    """bank_fft_pos is a permutation of the row (the exactness tests above show it is the FFT's order), the
    library's butterfly count is the schedule's, and bank_fft_fits is the tap and width bound
    xlg_add_bank_fft enforces."""
    for K in (2, 4, 8, 16, 32, 128, 512, 2048, 4096):
        pos = [bank_fft_pos(k, K) for k in range(-K // 2, K // 2)]
        assert sorted(pos) == list(range(K))
        n = sum(K // 4 * 28 if R == 4 else K // 2 * 4 for _, R in fft_stages(K))
        assert pkg.bank_fft_flops(K) == n
        d1 = K // 2
        assert pkg.bank_fft_fits(d1, bank_fft_max_taps(K)) and not pkg.bank_fft_fits(d1, bank_fft_max_taps(K) + 1)
        assert bank_fft_max_taps(K) >= max(16 * K, 16384)
    assert bank_fft_max_taps(4096) == 65536
    assert not pkg.bank_fft_fits(4096, 1) and not pkg.bank_fft_fits(3, 1) and not pkg.bank_fft_fits(7, 1)
    assert not pkg.bank_fft_fits(4, 0)


CHAIN_INT = [(1, 1), (3, 9), (4, 8), (5, 23), (2, 31)]  # (D2, T2)
CHAIN_RAT = [(2, 5, 33), (3, 7, 40), (12, 5, 60)]       # (L2, M2, T2)


@pytest.mark.parametrize("D1,T1,fmt", [(1, 9, "cu8"), (2, 3, "cs8"), (2, 31, "cs16")])
def test_chain_is_exact_on_exact_stimuli(D1, T1, fmt):
    """Dyadic bank taps at K = 2 and 4, dyadic full-length members at offset 0: the chain equals f64_bank's
    rows fed to f64_member, the bank attached after block 0, the channel materialised a block later and
    members attached at the channel's first block and two blocks on."""
    rng = np.random.default_rng(D1 * 13 + T1)
    fs = 2 * D1 * 96000
    taps1 = dyadic_taps(rng, T1, fmt)
    _, x = stream(rng, fmt, SIZES)
    P, sizes = SIZES[0], SIZES[1:]
    for k in range(-D1, D1):
        for attach in (0, 2):
            members = [(1, d2, dyadic_member(rng, taps1, T2, fmt), 0) for d2, T2 in CHAIN_INT]
            members += [(l2, m2, dyadic_member(rng, taps1, T2, fmt), 0) for l2, m2, T2 in CHAIN_RAT]
            got = bank_fft_member_model(taps1, D1, k, x.astype(np.complex64), P, sizes, members, fs, mat=1,
                                        attach=attach)
            rows = f64_bank(taps1, D1, [k], x, P, sizes)[k][1:]
            for (l2, d2, taps2, _), y in zip(members, got):
                want = f64_member(rows[attach:], l2, d2, taps2, fs // D1)
                assert len(y) == len(want)
                for a, w in zip(y, want):
                    assert np.array_equal(a, w), (fmt, k, l2, d2, taps2.size, attach)


@pytest.mark.parametrize("D1,T1,fmt", [(4, 13, "cu8"), (16, 101, "cs8"), (64, 45, "cs16")])
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
        got = bank_fft_member_model(taps1, D1, k, x.astype(np.complex64), 0, SIZES, members, fs)
        for (l2, d2, taps2, off), y in zip(members, got):
            o = BankMemberOracle(D1, taps1, k, d2, taps2, off, l2, fs)
            want = [o.process_cf32(fmt, r) for r in raw]
            a, b = np.concatenate(y), np.concatenate(want)
            assert a.shape == b.shape
            assert np.max(np.abs(a - b)) <= 1e-5 * np.max(np.abs(b)), (k, l2, d2, off)


# (d1, sub-bands, FMAs, sum of centres, sum of member offsets) of subband_plan(fs, clients) and of
# subband_plan(fs, clients, bank=True) at the sub-band workloads (tools/subband_bench.py), as they were before
# FFT banks existed
PLANS = {
    "10M_256": [(20, 40, 1571.315, -1600680, 2013717), (25, 50, 909.155, -5000000, 2419365)],
    "2048k_256": [(10, 20, 1976.0, 81780, 217905), (16, 31, 1078.625, 0, 279089)],
    "20M_256": [(20, 41, 1494.258, 5015366, 2886018), (25, 50, 904.938, -10000000, 3001474)],
    "2M_256": [(7, 14, 2600.0, 431354, 654351), (7, 13, 1924.857, 0, 189967)],
    "61M_1024": [(32, 65, 2863.575, 12097540, -15647901), (64, 128, 1805.919, -30720000, -5065117)],
    "61M_4096": [(64, 129, 5850.238, 10889148, -2819537), (128, 256, 3608.847, -30720000, 1652015)],
}


def signature(p):
    return (p["d1"], len(p["subbands"]), round(p["fmas"], 3), sum(s["center"] for s in p["subbands"]),
            sum(m["offset"] for m in p["members"]))


@pytest.mark.parametrize("name", sorted(PLANS))
def test_plan_without_fft_is_unchanged(pkg, name):
    import subband_bench as sbb
    fs = sbb.WORKLOADS[name][0]
    clients = sbb.workload_clients(name)
    for bank, want in zip((False, True), PLANS[name]):
        p = pkg.subband_plan(fs, clients, bank=bank, fft=False)
        assert signature(p) == want and "kernel" not in p
        q = pkg.subband_plan(fs, clients, bank=bank)
        assert q.keys() == p.keys() and signature(q) == want
        assert all(np.array_equal(a["taps2"], b["taps2"]) for a, b in zip(p["members"], q["members"]))


@pytest.mark.parametrize("name", sorted(PLANS))
def test_plan_with_fft_takes_the_cheaper_kernel(pkg, name):
    """fft=True: an FFT bank only at a power-of-two K that bank_fft_fits takes; the kernel costed lower at the
    chosen D1 (the direct one on a tie), and a plan never dearer than the direct bank's."""
    import subband_bench as sbb
    fs = sbb.WORKLOADS[name][0]
    clients = sbb.workload_clients(name)
    p = pkg.subband_plan(fs, clients, bank=True, fft=True)
    d1, T1, C = p["d1"], p["taps1"].size, len(p["subbands"])
    K = 2 * d1
    direct = 8.0 * C if pkg.bank_fits(d1, T1) else None
    fft = pkg.bank_fft_flops(K) / d1 if pkg.bank_fft_fits(d1, T1) else None
    assert p["kernel"] in ("direct", "fft")
    if p["kernel"] == "fft":
        assert K & (K - 1) == 0 and K <= 4096 and pkg.bank_fft_fits(d1, T1)
        assert direct is None or fft < direct
    else:
        assert direct is not None and (fft is None or direct <= fft)
    shapes = [(m["rate"], m["taps2"].size, m["interp2"]) for m in p["members"]]
    stage = fft if p["kernel"] == "fft" else direct
    assert p["fmas"] == pytest.approx(2.0 * T1 / d1 + stage + pkg.subband_fmas(fs, d1, T1, 0, shapes), rel=1e-12)
    assert p["fmas"] <= pkg.subband_plan(fs, clients, bank=True)["fmas"]
    with pytest.raises(ValueError):
        pkg.subband_plan(fs, clients, fft=True)
