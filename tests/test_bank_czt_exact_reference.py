"""The chirp-z bank references (tests/bank_czt_exact.py) checked on the CPU, before any GPU test relies on them.

* the model is within NORM_BOUND of the float64 definition of the bank (bank_exact.f64_bank) norm-wise at every K
  of CZT_KS, with T1 < K, T1 = K and T1 >> K, attached at P != 0;
* each mutation of the model fails that harness;
* the library's tables (xlg_bank_any_tables) are the float64 definitions rounded once, and the table query
  refuses every K the chirp-z stage does not serve;
* subband_plan without any_k is unchanged on every sub-band workload, and with any_k takes chirp-z banks at
  10 and 20 Msps, costed by the formula.
"""
import os
import sys

import numpy as np
import pytest

from bank_czt_exact import MUTATIONS, bank_czt_flops, bank_czt_m, bank_czt_model
from bank_exact import f64_bank
from exact import exact_input, to_complex
from spectrum_czt import chirp_f64, kernel_f64, positions

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))

CZT_KS = (6, 10, 14, 50, 100, 250, 800, 1000, 4094)
# Measured below: at most 3.1e-7 (K = 4094, T1 = K); 1e-6 leaves a margin of 3x and sits well inside 1e-5.
NORM_BOUND = 1e-6


def stream(rng, fmt, sizes):
    return np.concatenate([to_complex(fmt, exact_input(rng, fmt, 2 * n)) for n in sizes])


def norm_err(got, ref, chans):
    return max(np.linalg.norm(np.concatenate(got[k]) - np.concatenate(ref[k])) /
               max(np.linalg.norm(np.concatenate(ref[k])), 1e-30) for k in chans)


def chans_of(D1):
    return list(range(-D1, D1)) if D1 <= 64 else sorted({-D1, -D1 + 1, -1, 0, 1, 3, D1 // 3, D1 - 1})


@pytest.mark.parametrize("K", CZT_KS)
@pytest.mark.parametrize("shape", ("short", "equal", "long"))
def test_model_is_within_the_norm_bound_of_the_definition(pkg, K, shape):
    """Random taps and cs16 input, T1 < K, = K and 3 K + 5, attached at P = 1234 (every channel up to K = 128,
    else the edges and a spread)."""
    D1 = K // 2
    T1 = {"short": max(K // 3, 1), "equal": K, "long": 3 * K + 5}[shape]
    rng = np.random.default_rng(K * 3 + T1)
    taps = (rng.standard_normal(T1) / np.sqrt(T1)).astype(np.float32)
    sizes = [3000, 7, 0, max(5000, 3 * K)]
    x = stream(rng, "cs16", [1234] + sizes)
    chans = chans_of(D1)
    ref = f64_bank(taps, D1, chans, x, 1234, sizes)
    got = bank_czt_model(taps, D1, chans, x.astype(np.complex64), 1234, sizes, pkg.bank_any_tables(K))
    assert len(got[chans[0]]) == len(ref[chans[0]])
    assert norm_err(got, ref, chans) <= NORM_BOUND


@pytest.mark.parametrize("mutation", MUTATIONS)
def test_every_mutation_fails_the_harness(pkg, mutation):
    """K = 100 (M = 256), T1 = 70 < K, the bank attached at an odd P."""
    rng = np.random.default_rng(11)
    D1, T1 = 50, 70
    taps = (rng.standard_normal(T1) / np.sqrt(T1)).astype(np.float32)
    sizes = [1001, 4096, 7, 0, 2, 4094]
    x = stream(rng, "cs8", sizes)
    P = sizes[0]
    chans = chans_of(D1)
    tables = pkg.bank_any_tables(2 * D1)
    ref = f64_bank(taps, D1, chans, x, P, sizes[1:])
    assert norm_err(bank_czt_model(taps, D1, chans, x.astype(np.complex64), P, sizes[1:], tables), ref,
                    chans) <= NORM_BOUND
    got = bank_czt_model(taps, D1, chans, x.astype(np.complex64), P, sizes[1:], tables, mutation=mutation)
    assert norm_err(got, ref, chans) > NORM_BOUND, mutation


@pytest.mark.parametrize("K", CZT_KS)
def test_tables_are_the_definitions_rounded(pkg, K):
    """The chirp within 2^-24 of e^{-i pi (n^2 mod 2K) / K} per component, Bh within half a float32 ulp of the
    float64 DFT (plus 1e-12 for the host's double FFT), in position order; M = next_pow2(2K - 1)."""
    chirp, kern, M = pkg.bank_any_tables(K)
    assert M == bank_czt_m(K) and chirp.shape == (K,) and kern.shape == (M,)
    c64 = chirp_f64(K)
    assert np.max(np.abs(chirp.real - c64.real)) <= 2.0 ** -24
    assert np.max(np.abs(chirp.imag - c64.imag)) <= 2.0 ** -24
    _, bins = positions(M)
    k64 = kernel_f64(K)[bins]
    for got, ref in ((kern.real, k64.real), (kern.imag, k64.imag)):
        bound = 0.5 * np.spacing(np.abs(ref).astype(np.float32)).astype(np.float64) + 1e-12
        assert np.all(np.abs(got.astype(np.float64) - ref) <= bound), K


def test_table_query_refusals(pkg):
    for K in (0, 1, 2, 3, 4, 5, 8, 64, 4095, 4096, 4097, 4098, 8190):
        with pytest.raises(ValueError):
            pkg.bank_any_tables(K)
    assert pkg.bank_any_tables(4094)[2] == 8192 and pkg.bank_any_tables(6)[2] == 16


def test_fits_and_flops(pkg):
    """bank_any_fits is xlg_add_bank_any's kernel-side bound; bank_any_flops the header's formula."""
    for K in (2, 6, 100, 1024, 4094, 4096):
        d1 = K // 2
        assert pkg.bank_any_fits(d1, max(16 * K, 16384)) and not pkg.bank_any_fits(d1, max(16 * K, 16384) + 1)
    assert not pkg.bank_any_fits(2049, 1) and not pkg.bank_any_fits(50, 0) and not pkg.bank_any_fits(0, 1)
    for K, C in ((6, 6), (100, 3), (800, 800), (4094, 1)):
        assert pkg.bank_any_flops(K, C) == bank_czt_flops(pkg.bank_fft_flops, K, C)


def _signature(p):
    return (p["d1"], len(p["subbands"]), round(p["fmas"], 3), sum(s["center"] for s in p["subbands"]),
            sum(m["offset"] for m in p["members"]), p.get("kernel"))


def test_plan_without_any_k_is_unchanged(pkg):
    """Every sub-band workload: any_k=False (the default) gives the plan of before, with and without fft."""
    import subband_bench as sbb
    for name, (fs, _, _, _) in sbb.WORKLOADS.items():
        clients = sbb.workload_clients(name)
        for bank, fft in ((False, False), (True, False), (True, True)):
            p = pkg.subband_plan(fs, clients, bank=bank, fft=fft)
            q = pkg.subband_plan(fs, clients, bank=bank, fft=fft, any_k=False)
            assert _signature(p) == _signature(q) and p.keys() == q.keys()
            assert np.array_equal(p["taps1"], q["taps1"])
            assert p.get("kernel") != "czt"
    with pytest.raises(ValueError):
        pkg.subband_plan(10000000, [(0, 48000)], bank=True, any_k=True)


@pytest.mark.parametrize("name,d1", [("10M_256", 50), ("20M_256", 125)])
def test_plan_with_any_k_takes_chirp_z_banks(pkg, name, d1):
    """10 and 20 Msps: a chirp-z bank at D1 = 50 and 125, cheaper than the plan without it, its fmas the
    formula's: 2 T1 / D1 + bank_any_flops(K, C) / D1 + the members'."""
    import subband_bench as sbb
    fs = sbb.WORKLOADS[name][0]
    clients = sbb.workload_clients(name)
    p = pkg.subband_plan(fs, clients, bank=True, fft=True, any_k=True)
    assert p["kernel"] == "czt" and p["d1"] == d1
    K = 2 * d1
    assert K & (K - 1) != 0 and pkg.bank_any_fits(d1, p["taps1"].size)
    shapes = [(m["rate"], m["taps2"].size, m["interp2"]) for m in p["members"]]
    members = pkg.subband_fmas(fs, d1, p["taps1"].size, 0, shapes)
    want = 2.0 * p["taps1"].size / d1 + bank_czt_flops(pkg.bank_fft_flops, K, len(p["subbands"])) / d1 + members
    assert p["fmas"] == pytest.approx(want, rel=1e-12)
    assert p["fmas"] < pkg.subband_plan(fs, clients, bank=True, fft=True)["fmas"]
