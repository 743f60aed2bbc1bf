"""The Welch spectrum references (tests/spectrum_welch.py) checked on the CPU, before any GPU test relies on them.

* with H = W, no window and the max, the model is spectrum_exact's model bit for bit, and a window of ones is no
  window bit for bit;
* a mean row is the frame-ordered float32 sum of spectrum_exact's per-frame powers over float32(F), bit for bit;
* the model is within ROW_BOUND of the float64 definition, relative to each row's largest value, at widths from
  1 to 4096 through both channel stages, max and mean, with and without overlap and windows (the largest error
  measured is 7.1e-6, at W = 4095, H = 4000 on the direct path with a Hann window: a margin of 2.8x);
* mean rows with the window w W / sum(w) are scipy.signal.welch's "spectrum" + 1e-20, half swapped, within
  WELCH_BOUND (measured: 6.1e-7, the rounding of the float32 rows);
* the walk's frame count returns each row with the block holding its last frame sample, and the frame buffer's
  bound is reached;
* each mutation of the model fails one of these checks.
"""
import numpy as np
import pytest

from exact import to_complex
from spectrum_exact import F32, dft32, half_swap, power32, spec_fft, spectrum_model
from spectrum_welch import (MUTATIONS, fbuf_frames, frames_done, hann, last_sample_blocks, model_blocks,
                            welch_f64, welch_frames, welch_model)
from util import rand_block

ROW_BOUND = 2e-5
WELCH_BOUND = 2e-6


def cs16(rng, n):
    return to_complex("cs16", rand_block(rng, "cs16", 2 * n)).astype(np.complex64)


def row_err(got, ref):
    return float(np.max(np.abs(got.astype(np.float64) - ref) / ref.max(axis=1, keepdims=True))) if ref.size else 0.0


def random_window(rng, W):
    return rng.uniform(-1.0, 1.5, W).astype(F32)


@pytest.mark.parametrize("W", [1, 3, 4, 63, 64, 100, 1024])
def test_plain_parameters_are_spectrum_exact(W):
    rng = np.random.default_rng(W)
    F, S = 3, 5
    x = cs16(rng, 3 * (F * W + S) + 7)
    for power in (True, False):
        a, b = welch_model(x, W, F, S, power=power), spectrum_model(x, W, F, S, power=power)
        assert a.shape == b.shape and a.shape[0] >= 3
        np.testing.assert_array_equal(a.view(np.uint32), b.view(np.uint32))


@pytest.mark.parametrize("W", [1, 5, 64, 1000])
@pytest.mark.parametrize("mean", [False, True])
def test_window_of_ones_is_no_window(W, mean):
    rng = np.random.default_rng(W + 1)
    H = max(1, W // 2)
    x = cs16(rng, 4 * W + 40)
    a = welch_model(x, W, 3, 1, H, None, mean)
    b = welch_model(x, W, 3, 1, H, np.ones(W, F32), mean)
    assert a.shape[0] > 0
    np.testing.assert_array_equal(a.view(np.uint32), b.view(np.uint32))


def ordered_mean(x, W, F, S, H, window):
    """The mean restated from spectrum_exact's pieces: each row's frames one at a time, float32 adds in order."""
    fr = welch_frames(x, W, F, S, H)
    z = (fr.real.astype(F32) * window) + 1j * (fr.imag.astype(F32) * window)
    z = z.astype(np.complex64)
    out = []
    for r in range(fr.shape[0]):
        s = np.zeros(W, F32)
        for f in range(F):
            xr, xi = dft32(z[r, f][None, :], W)
            s = (s + power32(xr, xi, W)[0]).astype(F32)
        out.append(s / F32(F))
    return half_swap(np.array(out, F32).reshape(-1, W))


def mean_check(mutation):
    rng = np.random.default_rng(5)
    failed = []
    for W, F, S, H in ((64, 8, 3, 16), (100, 7, 0, 50)):
        x = cs16(rng, 3 * ((F - 1) * H + W + S))
        w = random_window(rng, W)
        got, ref = welch_model(x, W, F, S, H, w, True, mutation=mutation), ordered_mean(x, W, F, S, H, w)
        if got.shape != ref.shape or (got.view(np.uint32) != ref.view(np.uint32)).any():
            failed.append(f"ordered mean W={W}")
    return failed


def test_mean_is_the_ordered_sum():
    assert mean_check(None) == []


WIDE = [(1, 2), (2, 1), (3, 1), (4, 1), (5, 3), (8, 1), (16, 4), (63, 8), (64, 16), (100, 25), (128, 64),
        (256, 128), (1000, 500), (1024, 512), (2048, 2048), (4095, 4000), (4096, 512)]


def definition_errors(W, H, mean, window, mutation=None):
    rng = np.random.default_rng(W + 7)
    F, S = (5, 3) if W < 1000 else (2, 1)
    n = 2 * ((F - 1) * H + W + S) + (F - 1) * H + W - 1  # two rows, and a third one sample short
    x = cs16(rng, n)
    w = None if window is None else (hann(W) if window == "hann" else random_window(rng, W))
    got, ref = welch_model(x, W, F, S, H, w, mean, mutation=mutation), welch_f64(x, W, F, S, H, w, mean)
    if got.shape != ref.shape:
        return np.inf
    assert got.shape == (2, W)
    return row_err(got, ref)


@pytest.mark.parametrize("W,H", WIDE)
@pytest.mark.parametrize("mean", [False, True])
def test_model_within_bound_of_definition(W, H, mean):
    for window in (None, "hann", "random"):
        assert definition_errors(W, H, mean, window) <= ROW_BOUND, (W, H, mean, window, spec_fft(W))


@pytest.mark.parametrize("W", [8, 64, 100, 1024])
@pytest.mark.parametrize("hop", ["W/2", "W/4", "W", "3W/2"])
@pytest.mark.parametrize("window", ["hann", "random"])
def test_mean_rows_are_scipy_welch(W, hop, window):
    signal = pytest.importorskip("scipy.signal")
    H = {"W/2": W // 2, "W/4": W // 4, "W": W, "3W/2": 3 * W // 2}[hop]
    rng = np.random.default_rng(W + H)
    F, S = 6, 11
    x = cs16(rng, 2 * ((F - 1) * H + W + S) + 5)
    w = hann(W) if window == "hann" else random_window(rng, W)
    w = (w * F32(W) / w.sum(dtype=F32)).astype(F32)  # scaling="spectrum"
    rows = welch_model(x, W, F, S, H, w, True)
    assert rows.shape == (2, W)
    R = (F - 1) * H + W + S
    for r in range(2):
        # a row's frames as one contiguous stream of F segments (H > W: the frames placed end to end)
        seg = welch_frames(x, W, F, S, H)[r]
        y, noverlap = (x[r * R:r * R + (F - 1) * H + W], W - H) if H <= W else (seg.reshape(-1), 0)
        _, pxx = signal.welch(y.astype(np.complex128), window=w.astype(np.float64), nperseg=W, noverlap=noverlap,
                              detrend=False, return_onesided=False, scaling="spectrum", average="mean")
        ref = half_swap(pxx + 1e-20)
        assert np.max(np.abs(rows[r] - ref)) / ref.max() <= WELCH_BOUND, (W, H, r)


def test_frame_count_and_blocks():
    """frames_done puts each row in the block holding its last frame sample, across ragged and empty blocks."""
    sizes = [5, 0, 1, 300, 17, 64, 0, 999, 3]
    for W, F, S, H in ((8, 3, 0, 2), (8, 3, 5, 8), (8, 2, 1, 13), (5, 4, 0, 1), (64, 2, 3, 60), (1, 1, 0, 1)):
        rows = model_blocks(np.zeros(sum(sizes), np.complex64), sizes, W, F, S, H, power=True)
        n = sum(r.shape[0] for r in rows)
        where = [b for b, r in enumerate(rows) for _ in range(r.shape[0])]
        assert n > 0 and where == list(last_sample_blocks(n, sizes, W, F, S, H)), (W, F, S, H)
        # every offset: g counts the frames whose last sample is below d
        for d in range(3 * ((F - 1) * H + W + S)):
            ends = [r * ((F - 1) * H + W + S) + f * H + W for r in range(4) for f in range(F)]
            assert frames_done(d, W, F, S, H) == sum(e <= d for e in ends), (W, F, S, H, d)


def test_frame_buffer_bound_is_reached():
    """A block of cap samples starting at a frame's last sample completes fbuf_frames frames (one row: F large)."""
    for cap, W, S, H in ((8192, 64, 0, 8), (8192, 4096, 0, 512), (100, 8, 1, 1), (8192, 1000, 3, 125)):
        F = 10 ** 6
        n = frames_done(W - 1 + cap, W, F, S, H) - frames_done(W - 1, W, F, S, H)
        assert n == fbuf_frames(cap, W, S, H), (cap, W, S, H)
        # and no block of cap samples does better, at any start
        assert max(frames_done(a + cap, W, F, S, H) - frames_done(a, W, F, S, H) for a in range(2 * W)) == n
    # H > W + S: rows end closer together than frames within a row
    cap, W, S, H, F = 1000, 8, 2, 40, 3
    best = max(frames_done(a + cap, W, F, S, H) - frames_done(a, W, F, S, H) for a in range(400))
    assert best <= fbuf_frames(cap, W, S, H)


def mutation_checks(mutation):
    failed = mean_check(mutation)
    for W, H, mean, window in ((64, 16, True, "random"), (100, 50, False, "random"), (63, 8, True, None)):
        if definition_errors(W, H, mean, window, mutation) > ROW_BOUND:
            failed.append(f"definition W={W}")
    sizes = [5, 0, 1, 300, 17, 64, 0, 999, 3]
    x = np.zeros(sum(sizes), np.complex64)
    for W, F, S, H in ((8, 3, 0, 2), (8, 2, 1, 13)):
        rows = model_blocks(x, sizes, W, F, S, H, mutation=mutation)
        where = [b for b, r in enumerate(rows) for _ in range(r.shape[0])]
        if where != list(last_sample_blocks(len(where), sizes, W, F, S, H)) or \
                len(where) != welch_model(x, W, F, S, H).shape[0]:
            failed.append(f"blocks W={W}")
    return failed


def test_model_passes_every_check():
    assert mutation_checks(None) == []


@pytest.mark.parametrize("mutation", MUTATIONS)
def test_mutation_is_caught(mutation):
    assert mutation_checks(mutation), f"{mutation} passes every check"
