"""The exact-stimulus harness (tests/exact.py) checked on the CPU, before any GPU test relies on it.

* its float64 and int64 references equal the strict float32 oracle (oracle/liboracle.so) bit for
  bit on dyadic taps and 8-bit inputs, across the shapes and call patterns the GPU tests use;
* the one-hot, real-input construction makes a fused-multiply-add accumulation (what the kernels
  do) agree bit for bit with the oracle's unfused one at any centre frequency;
* mutations that the float tolerance cannot see with designed (lpf.c) taps -- a dropped first or
  last tap, an un-zeroed oldest history sample, two clients' taps swapped -- fail assert_exact.
"""
import ctypes as C

import numpy as np
import pytest

from exact import (assert_exact, dyadic_taps, exact_input, gpu_model, grid_step, one_hot_taps, real_input, ref_f64,
                   oscillator_increment, ref_q15, reversed_taps, tap_bits, to_complex)
from oracle import pyoracle as po
from util import assert_cf32_close, rand_block

MAX_IN = 1 << 17


def oracle_run(taps, D, fmt, blocks, q15=False, center=0, fs=2016000, renorm=True):
    o = po.OracleFilter(D, taps, center, fs, MAX_IN)
    if q15:
        return [o.process_q15(fmt, x) for x in blocks]
    return [o.process_cf32(fmt, x, renorm=renorm) for x in blocks]


def ragged_blocks(rng, fmt, sizes):
    return [exact_input(rng, fmt, n) for n in sizes]


SIZES = [4096, 0, 2, 7, 1, 3001, 4096, 2, 0, 999]  # empty, 1-sample, odd-length and ragged calls


@pytest.mark.parametrize("T,D", [(64, 7), (1, 1), (33, 1), (43, 42), (85, 42), (253, 21), (297, 42), (8, 8),
                                 (16, 3), (400, 8)])
@pytest.mark.parametrize("fmt", ["cu8", "cs8", "cs16"])
def test_ref_f64_equals_oracle(T, D, fmt):
    rng = np.random.default_rng(T * 1000 + D)
    taps = dyadic_taps(rng, T, fmt)
    blocks = ragged_blocks(rng, fmt, SIZES)
    assert_exact(ref_f64(taps, D, fmt, blocks), oracle_run(taps, D, fmt, blocks), f"T={T} D={D} {fmt}", T, D,
                 grid_step(taps, fmt))


@pytest.mark.parametrize("T,D,fmt", [(4001, 15, "cu8"), (15419, 1280, "cs16"), (24001, 5, "cu8")])
def test_ref_f64_equals_oracle_long_filters(T, D, fmt):
    rng = np.random.default_rng(T)
    taps = dyadic_taps(rng, T, fmt)
    assert tap_bits(T, fmt) == {4001: 4, 15419: 3, 24001: 1}[T]
    blocks = ragged_blocks(rng, fmt, [32768, 32768, 10001, 32768])
    y = ref_f64(taps, D, fmt, blocks)
    assert_exact(y, oracle_run(taps, D, fmt, blocks), f"T={T} D={D}", T, D, grid_step(taps, fmt))
    # a sequential float32 sum in the opposite order gives the same numbers (np.cumsum adds in order)
    rev = reversed_taps(np.asarray(taps, dtype=np.float32))
    x = np.concatenate([np.zeros(T - 1, np.complex64)] + [to_complex(fmt, b).astype(np.complex64) for b in blocks])
    flat = np.concatenate(y)
    assert flat.size > 40
    for i in range(0, flat.size, 7):
        w = x[i * D:i * D + T]
        re = np.cumsum((w.real * rev)[::-1], dtype=np.float32)[-1]
        im = np.cumsum((w.imag * rev)[::-1], dtype=np.float32)[-1]
        assert re == flat[i].real and im == flat[i].imag, i


@pytest.mark.parametrize("T,D,fmt", [(64, 7, "cu8"), (253, 21, "cs8"), (297, 42, "cs16"), (1, 1, "cu8"),
                                     (43, 42, "cu8"), (15419, 1280, "cs16")])
def test_ref_q15_equals_oracle(T, D, fmt):
    rng = np.random.default_rng(T + 7)
    taps = dyadic_taps(rng, T, fmt, k=15)
    assert np.all(np.trunc(taps * np.float32(32768)) != 0)
    blocks = ragged_blocks(rng, fmt, [8192, 0, 2, 7, 4001, 8192] if T < 10000 else [131072, 50002, 131072])
    want = oracle_run(taps, D, fmt, blocks, q15=True)
    assert_exact(ref_q15(taps, D, fmt, blocks), want, f"Q15 T={T} D={D} {fmt}", T, D)
    assert any(np.abs(w).max() > 64 for w in want if len(w))  # not drowned in zeros


def test_ref_f64_history_equals_oracle_state():
    """ref_f64's `history` argument: a filter whose first window reads given samples instead of zeros
    (the oracle's set_state), the situation of a client attached mid-stream with real history."""
    rng = np.random.default_rng(3)
    T, D, fmt = 253, 21, "cu8"
    taps = dyadic_taps(rng, T, fmt)
    hist = to_complex(fmt, exact_input(rng, fmt, 2 * (T - 1)))
    blocks = ragged_blocks(rng, fmt, [4096, 7, 2000])
    o = po.OracleFilter(D, taps, 0, 2016000, MAX_IN)
    lib = po.orc()
    lib.orc_xlating_set_state.argtypes = [C.c_void_p, C.POINTER(C.c_float), C.c_size_t, C.c_float, C.c_float]
    lib.orc_xlating_set_state.restype = C.c_int
    h32 = np.ascontiguousarray(hist.astype(np.complex64)).view(np.float32)
    assert lib.orc_xlating_set_state(o._h, h32.ctypes.data_as(C.POINTER(C.c_float)), T - 1, 1.0, 0.0) == 0
    got = [o.process_cf32(fmt, x) for x in blocks]
    assert_exact(ref_f64(taps, D, fmt, blocks, history=hist), got, "history", T, D, grid_step(taps, fmt))


# ---------------------------------------------------------------------------
# one-hot taps, real input, any centre: FMA accumulation == the oracle's unfused sums
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("center", [-987654, -312000, 1, 400123, 1007999])
@pytest.mark.parametrize("j", [0, 100, 252])
def test_one_hot_real_input_fma_matches_oracle(center, j):
    rng = np.random.default_rng(j + 17)
    fs, D, T = 2016000, 21, 253
    taps = one_hot_taps(T, j, 0.75)
    o = po.OracleFilter(D, taps, center, fs, MAX_IN)
    rev = o.rev_taps
    inc = oscillator_increment(D, center, fs)
    blocks = [real_input(rng, n) for n in (4096, 2, 1001, 4096, 0, 3000)]
    want = [o.process_cf32("cs16", x) for x in blocks]
    assert_exact(gpu_model(rev, inc, D, blocks), want, f"centre {center} j={j}", T, D)


# ---------------------------------------------------------------------------
# mutations: invisible to the float tolerance with designed taps, caught by exact stimuli
# ---------------------------------------------------------------------------
FS, D96 = 2016000, 21


def lpf_taps():
    taps = po.lpf_design(1.0, FS, 48000, 19200)
    assert len(taps) == 253
    return taps


def stream(rng, fmt, n_blocks, exact):
    return [(exact_input if exact else rand_block)(rng, fmt, 8192) for _ in range(n_blocks)]


def zero_tap(taps, i):
    t = np.array(taps, copy=True)
    t[i] = 0
    return t


@pytest.mark.parametrize("which", [0, -1], ids=["first_tap", "last_tap"])
def test_mutation_dropped_edge_tap(which):
    rng = np.random.default_rng(41)
    taps = lpf_taps()
    blocks = stream(rng, "cu8", 3, exact=False)
    want = oracle_run(taps, D96, "cu8", blocks)
    for g, r in zip(ref_f64(zero_tap(taps, which), D96, "cu8", blocks), want):
        assert_cf32_close(g, r)  # the float contract cannot see it
    dt = dyadic_taps(rng, 253, "cu8")
    blocks = stream(rng, "cu8", 3, exact=True)
    bad = ref_f64(zero_tap(dt, which), D96, "cu8", blocks)
    with pytest.raises(AssertionError, match="outputs differ"):
        assert_exact(bad, ref_f64(dt, D96, "cu8", blocks), "mutant", 253, D96, grid_step(dt, "cu8"))
    # every output whose window lies past the zero history reads both edge taps: all of them change
    bad, good = np.concatenate(bad), np.concatenate(ref_f64(dt, D96, "cu8", blocks))
    assert np.all(bad[-(-252 // D96):] != good[-(-252 // D96):])


def test_mutation_oldest_history_sample_not_zeroed():
    """A client attached at stream position P must read samples before P as zero; the mutant reads the
    oldest sample of its first window, P - (T - 1), from the stream."""
    rng = np.random.default_rng(43)
    T = 253
    for taps, exact in ((lpf_taps(), False), (dyadic_taps(rng, T, "cu8"), True)):
        blocks = stream(rng, "cu8", 4, exact)
        late = blocks[2:]
        before = np.concatenate([to_complex("cu8", b) for b in blocks[:2]])
        hist = np.zeros(T - 1, np.complex128)
        hist[0] = before[-(T - 1)]
        bad = ref_f64(taps, D96, "cu8", late, history=hist)
        if not exact:
            for g, r in zip(bad, oracle_run(taps, D96, "cu8", late)):
                assert_cf32_close(g, r)
        else:
            with pytest.raises(AssertionError, match="first at block 0 output 0 .*window start -252"):
                assert_exact(bad, ref_f64(taps, D96, "cu8", late), "mutant", T, D96, grid_step(taps, "cu8"))


def test_mutation_two_clients_taps_swapped():
    """Clients of one class read each other's tap column.  Designed taps are identical across a class,
    so the swap is invisible; distinct dyadic taps per client expose it."""
    rng = np.random.default_rng(47)
    a = b = lpf_taps()
    blocks = stream(rng, "cu8", 2, exact=False)
    for g, r in zip(ref_f64(b, D96, "cu8", blocks), oracle_run(a, D96, "cu8", blocks)):
        assert_cf32_close(g, r)
    a, b = dyadic_taps(rng, 253, "cu8"), dyadic_taps(rng, 253, "cu8")
    blocks = stream(rng, "cu8", 2, exact=True)
    with pytest.raises(AssertionError, match="outputs differ"):
        assert_exact(ref_f64(b, D96, "cu8", blocks), ref_f64(a, D96, "cu8", blocks), "swapped")


def test_dyadic_taps_shape():
    rng = np.random.default_rng(1)
    for T, fmt, M in ((64, "cu8", 127), (518, "cu8", 127), (4386, "cu8", 15), (15419, "cu8", 3), (15419, "cs16", 7),
                      (24001, "cu8", 1), (65793, "cu8", 1)):
        t = dyadic_taps(rng, T, fmt)
        m = t * 2.0 ** tap_bits(T, fmt)
        assert np.all(m != 0) and np.all(m == np.round(m)) and np.max(np.abs(m)) == M
        assert abs(m[0]) == M and abs(m[-1]) == M
        assert T * 255 * M <= 2 ** 24 or fmt != "cu8"
