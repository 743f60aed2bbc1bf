"""Rational L/M clients on the host: the definition (zero-stuffed oracle) against scipy's upfirdn,
the polyphase packer, and the taps rational_plan designs."""
import numpy as np
import pytest
from scipy.signal import upfirdn

from oracle import pyoracle as po
from rational import ROWS, oracle_filter, oracle_run, poly_pack_np, stuff

# (band fs, client rate) -> (L, M, T) as the issue's rate table gives them
TABLE = {2048000: (3, 128, 1541), 3000000: (2, 125, 1505), 10000000: (3, 625, 7529), 20000000: (3, 1250, 15057)}


@pytest.mark.parametrize("row", ROWS[:3], ids=lambda r: f"{r[0] // 1000}k")
def test_zero_stuffed_oracle_is_upfirdn(pkg, row):
    fs, fmt, rate = row
    p = pkg.rational_plan(fs, [rate])[0]
    L, M, taps = p["interp"], p["decim"], p["taps"]
    rng = np.random.default_rng(3)
    n = 65536
    blocks = [rng.integers(0, 256, n, dtype=np.uint8) if fmt == "cu8" else rng.integers(-8192, 8192, n, dtype=np.int16)
              for _ in range(4)]
    o = oracle_filter(po, L, M, taps, 0, fs, n)
    y = np.concatenate(oracle_run(o, fmt, blocks, L)).astype(np.complex128)
    raw = np.concatenate([stuff(fmt, b, 1) for b in blocks]).astype(np.float64) / 32768.0
    x = raw[0::2] + 1j * raw[1::2]
    ref = upfirdn(taps.astype(np.float64), x, L, M)[:y.size]
    assert y.size > 100 and ref.size == y.size
    err = np.max(np.abs(y - ref)) / np.max(np.abs(ref))
    # the difference is the oracle's float32 sum: 514 and 753 nonzero terms per output stay within
    # 1e-6; row 3's 2510 measured 1.6-2.6e-6 across seeds
    assert err <= (2e-6 if -(-taps.size // L) < 1000 else 4e-6), err


@pytest.mark.parametrize("T,L", [(1541, 3), (1505, 2), (10, 3), (2, 5), (1, 4), (12, 4), (97, 7)])
def test_poly_pack_matches_numpy(pkg, T, L):
    rng = np.random.default_rng(T * 31 + L)
    taps = rng.standard_normal(T).astype(np.float32)
    o = po.OracleFilter(5, taps, 123457, L * 2048000, 4096)  # nonzero centre: complex, rotated taps
    rev = o.rev_taps
    got = pkg.poly_pack(rev, L)
    want = poly_pack_np(rev, L)
    assert got.shape == want.shape == (L, -(-T // L))
    assert np.array_equal(got.view(np.uint64), want.view(np.uint64))


@pytest.mark.parametrize("fs", sorted(TABLE))
def test_rational_plan_table_and_branch_gain(pkg, fs):
    plan = pkg.rational_plan(fs, [48000] * 4)
    ref = pkg.client_plan(fs, [48000] * 4)
    for p, q in zip(plan, ref):
        L, M, T = TABLE[fs]
        assert (p["interp"], p["decim"], p["taps"].size) == (L, M, T)
        assert p["center"] == q["center"]
        for r in range(L):
            assert abs(float(np.sum(p["taps"][r::L], dtype=np.float64)) - 1.0) <= 1e-3, (fs, r)
