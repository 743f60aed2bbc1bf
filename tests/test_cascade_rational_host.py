"""Rational cascade clients (xlg_add_client_cascade_rational) on the CPU: the composed oracle, the planner for
rates that do not divide the band rate, and the host walk in upsampled coordinates.  No GPU."""
import ctypes as C
import math

import numpy as np
import pytest

from cascade_rational import RationalCascadeOracle, f64_composition
from exact import to_complex
from oracle import pyoracle as po

RAGGED = [65536, 30001, 2, 0, 12347, 7, 65534, 4096, 1, 999]


def test_composed_oracle_is_two_filters_in_series(pkg):
    """The composed oracle equals the float64 composition within float32 rounding at centre 0."""
    fs, rate, max_in = 2048000, 48000, 8192
    p = pkg.cascade_plan(fs, [rate])[0]
    assert p["interp2"] == 3
    rng = np.random.default_rng(3)
    raw = [rng.integers(0, 256, n, dtype=np.uint8) for n in (8192, 4097, 30, 8192, 2, 6000, 0, 8192)]
    o = RationalCascadeOracle(p["d1"], p["taps1"], 0, p["interp2"], p["d2"], p["taps2"], fs, max_in)
    got = [o.process_cf32("cu8", x) for x in raw]
    want = f64_composition(p["d1"], p["taps1"], p["interp2"], p["d2"], p["taps2"], fs,
                           [to_complex("cu8", x) for x in raw])
    assert [y.size for y in got] == [y.size for y in want]
    g, w = np.concatenate(got), np.concatenate(want)
    assert np.max(np.abs(g - w)) <= 2e-6 * np.max(np.abs(w))


# band -> 48 kHz: D1, L2 / M2, T1, T2, FMAs per input sample (single stage, cascade) to one decimal
TABLE = [(2048000, 8, 3, 16, 25, 193, 48.2, 15.6), (10000000, 20, 12, 125, 55, 1505, 48.2, 12.2),
         (20000000, 25, 3, 50, 65, 603, 48.2, 11.4), (3000000, 10, 4, 25, 29, 301, 48.2, 14.0),
         (2500000, 8, 96, 625, 23, 7529, 48.2, 14.5)]


@pytest.mark.parametrize("fs,d1,l2,m2,t1,t2,single,fmas", TABLE)
def test_cascade_plan_rational(pkg, fs, d1, l2, m2, t1, t2, single, fmas):
    """The planner picks the split with the fewest FMAs, and its taps are create_low_pass_filter's bit for bit."""
    rate = 48000
    p = pkg.cascade_plan(fs, [rate])[0]
    assert (p["d1"], p["interp2"], p["d2"], p["taps1"].size, p["taps2"].size) == (d1, l2, m2, t1, t2)
    fs1, e = fs // d1, 3 * rate // 5
    assert p["taps1"].tobytes() == po.lpf_design(1.0, fs, fs1 // 2, fs1 - 2 * e).tobytes()
    assert p["taps2"].tobytes() == po.lpf_design(float(l2), l2 * fs1, rate // 2, rate // 5).tobytes()
    assert p["fmas"] == 4.0 * t1 / d1 + 2.0 * math.ceil(t2 / l2) / (fs / rate)
    assert p["fmas"] == pytest.approx(fmas, abs=0.06)  # 15.547 for 2.048 Msps is 15.6 in the table
    r = pkg.rational_plan(fs, [rate])[0]
    assert 4 * math.ceil(r["taps"].size / r["interp"]) * rate / fs == pytest.approx(single, abs=0.05)


def test_cascade_plan_keeps_dividing_rates(pkg):
    """interp2 is 1 wherever the rate divides the band rate (the rest of the entry is test_cascade_plan's)."""
    assert [p["interp2"] for p in pkg.cascade_plan(2016000, [48000, 32000])] == [1, 1]


@pytest.mark.parametrize("fs", [2048000, 10000000])
def test_host_walk_counts_match_the_oracle(pkg, fs):
    """xl_walk in upsampled coordinates, walked over stage A's counts, equals the composed oracle's output
    counts and histories over ragged blocks, including blocks with fewer stage-A samples than stage B's
    history."""
    walk = pkg.lib().xl_walk
    walk.argtypes = [C.POINTER(C.c_longlong), C.c_longlong, C.c_size_t, C.c_uint32, C.c_int]
    walk.restype = C.c_int
    max_in = 65536
    p = pkg.cascade_plan(fs, [48000])[0]
    L2, M2, T2 = p["interp2"], p["d2"], p["taps2"].size
    o = RationalCascadeOracle(p["d1"], p["taps1"], 0, L2, M2, p["taps2"], fs, max_in)
    h1, h2 = C.c_longlong(p["taps1"].size - 1), C.c_longlong(T2 - 1)
    cap1 = max_in // 2 // p["d1"] + 2
    rng = np.random.default_rng(5)
    sizes = RAGGED + [int(v) for v in rng.integers(0, 400, 60)]
    short = 0
    for n in sizes:
        n1 = walk(C.byref(h1), n // 2, p["taps1"].size, p["d1"], cap1)
        short += L2 * n1 < T2 - 1
        n2 = walk(C.byref(h2), L2 * n1, T2, M2, cap1 * L2 // M2 + 2)
        assert o.process_cf32("cu8", rng.integers(0, 256, n, dtype=np.uint8)).size == n2, n
        assert o.a.history == h1.value and o.b.history == h2.value
    assert short > 10
