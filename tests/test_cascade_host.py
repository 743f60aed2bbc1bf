"""Cascade clients (xlg_add_client_cascade) on the CPU: the float-path restatement on cf32 input, the cascade
oracle, the tap planner and the host walk that gives each block's stage-B output count.  No GPU."""
import ctypes as C

import numpy as np
import pytest

from cascade import FloatPath, cascade_oracle, f64_filter
from exact import to_complex
from oracle import pyoracle as po

RAGGED = [65536, 30001, 2, 0, 12347, 7, 65534, 4096, 1, 999]


def cu8_as_cf32(x):
    """The reference's cu8 conversion, exact in float32 (src/xlating.c:389-390)."""
    return ((x.astype(np.float32) - np.float32(127.5)) / np.float32(128.0)).astype(np.float32)


@pytest.mark.skipif(not po.ref_available("strict"), reason="reference build absent (oracle/_ref)")
@pytest.mark.parametrize("center", [0, -312000, 17, 251000, 1000003])
def test_float_path_on_cf32_is_the_reference(center):
    """FloatPath, fed an exactly converted cu8 stream, equals the reference's own process_native_cu8_cf32
    bit for bit, call by call (history, oscillator, renormalisation)."""
    fs, max_in = 2016000, 65536
    taps = po.lpf_design(1.0, fs, 24000, 9600)
    o = FloatPath(42, taps, center, fs)
    r = po.RefFilter(42, taps, center, fs, max_in)
    rng = np.random.default_rng(center & 0xffff)
    for n in RAGGED:
        x = rng.integers(0, 256, n, dtype=np.uint8)
        got = o.process_cf32(cu8_as_cf32(x)[: n // 2 * 2].view(np.complex64))
        want = r.process_cf32("cu8", x)
        assert got.view(np.uint64).tolist() == want.view(np.uint64).tolist(), n


def test_cascade_oracle_is_two_filters_in_series(pkg):
    """cascade_oracle equals the float64 composition within float32 rounding (at centre 0: elsewhere the
    reference's float oscillator drifts from exact math by design, SURVEY.md 0.3)."""
    fs, rate, max_in = 2016000, 48000, 8192
    p = pkg.cascade_plan(fs, [rate])[0]
    rng = np.random.default_rng(3)
    raw = [rng.integers(0, 256, n, dtype=np.uint8) for n in (8192, 4097, 30, 8192, 2, 6000)]
    o = cascade_oracle(p["d1"], p["taps1"], 0, p["d2"], p["taps2"], fs, max_in)
    got = [o.process_cf32("cu8", x) for x in raw]
    a = f64_filter(p["taps1"], p["d1"], 0, fs, [to_complex("cu8", x) for x in raw])
    want = f64_filter(p["taps2"], p["d2"], 0, fs // p["d1"], a)
    g, w = np.concatenate(got), np.concatenate(want)
    assert [y.size for y in got] == [y.size for y in want]
    assert np.max(np.abs(g - w)) <= 2e-6 * np.max(np.abs(w))


@pytest.mark.parametrize("fs,rate,d1,t1,t2", [(61440000, 48000, 32, 79, 481), (2016000, 48000, 6, 17, 85),
                                               (10000000, 250000, 8, 25, 61), (2048000, 32000, 8, 23, 97)])
def test_cascade_plan(pkg, fs, rate, d1, t1, t2):
    """The planner picks the issue's split, and its taps are create_low_pass_filter's bit for bit."""
    p = pkg.cascade_plan(fs, [rate])[0]
    assert (p["d1"], p["d2"], p["taps1"].size, p["taps2"].size) == (d1, fs // rate // d1, t1, t2)
    fs1, e = fs // d1, 3 * rate // 5
    assert p["taps1"].tobytes() == po.lpf_design(1.0, fs, fs1 // 2, fs1 - 2 * e).tobytes()
    assert p["taps2"].tobytes() == po.lpf_design(1.0, fs1, rate // 2, rate // 5).tobytes()
    assert p["fmas"] == pytest.approx(4 * t1 / d1 + 2 * t2 / (fs // rate))


def test_host_walk_counts_match_the_oracle(pkg):
    """xl_walk, which gives each block's stage-B count on the host, walked over stage A's counts, equals
    the cascade oracle's output counts over ragged blocks, including blocks with fewer stage-A outputs
    than stage B's history."""
    walk = pkg.lib().xl_walk
    walk.argtypes = [C.POINTER(C.c_longlong), C.c_longlong, C.c_size_t, C.c_uint32, C.c_int]
    walk.restype = C.c_int
    fs, max_in = 2016000, 65536
    p = pkg.cascade_plan(fs, [48000])[0]
    o = cascade_oracle(p["d1"], p["taps1"], 0, p["d2"], p["taps2"], fs, max_in)
    h1, h2 = C.c_longlong(p["taps1"].size - 1), C.c_longlong(p["taps2"].size - 1)
    cap1 = max_in // 2 // p["d1"] + 2
    rng = np.random.default_rng(5)
    sizes = RAGGED + [int(v) for v in rng.integers(0, 400, 60)]
    for n in sizes:
        n1 = walk(C.byref(h1), n // 2, p["taps1"].size, p["d1"], cap1)
        n2 = walk(C.byref(h2), n1, p["taps2"].size, p["d2"], cap1 // p["d2"] + 2)
        assert o.process_cf32("cu8", rng.integers(0, 256, n, dtype=np.uint8)).size == n2, n
        assert o.a.history == h1.value and o.b.history == h2.value
