"""The wide spectrum references (tests/spectrum_wide.py) checked on the CPU, before any GPU test relies on them.

* for every wide W, the kernels' two passes (the first radix-4 stages over the frame, then fft_rows at K = C on
  each contiguous chunk with the C-point table) are fft_rows at K = W bit for bit, and the C-point table is the
  W-point one at stride W / C bit for bit;
* the model is within ROW_BOUND of the float64 definition, relative to each row's largest value, for max and
  mean, with no window, Hann and random weights (a tone 60 dB over noise; the largest error measured is
  2.3e-7, at W = 65536 with random weights and the max);
* mean rows with the window w W / sum(w) are scipy.signal.welch's "spectrum" + 1e-20, half swapped, within
  WELCH_BOUND;
* each mutation of the model fails one of these checks.
"""
import numpy as np
import pytest

from bank_exact import twiddles
from bank_fft_exact import fft_rows
from exact import to_complex
from spectrum_exact import F32, half_swap
from spectrum_welch import frames_done, hann, last_sample_blocks, welch_f64, welch_frames
from spectrum_wide import MUTATIONS, WIDE_WIDTHS, two_pass_rows, wide_blocks, wide_chunk, wide_model
from util import rand_block

ROW_BOUND = 2e-5
WELCH_BOUND = 2e-6


def cs16(rng, n):
    return to_complex("cs16", rand_block(rng, "cs16", 2 * n)).astype(np.complex64)


def tone(rng, n, W):
    """A strong tone between bins over cs16 noise 60 dB down."""
    k = np.arange(n)
    x = 2e4 * np.exp(2j * np.pi * (W / 5 + 0.3) * k / W) + 20 * cs16(rng, n)
    return x.astype(np.complex64)


def row_err(got, ref):
    return float(np.max(np.abs(got.astype(np.float64) - ref) / ref.max(axis=1, keepdims=True))) if ref.size else 0.0


@pytest.mark.parametrize("W", WIDE_WIDTHS)
def test_chunk_table_is_the_wide_table_at_stride(W):
    C = wide_chunk(W)
    a, b = np.ascontiguousarray(twiddles(W)[::W // C]), twiddles(C)
    np.testing.assert_array_equal(a.view(np.uint32), b.view(np.uint32))


@pytest.mark.parametrize("W", WIDE_WIDTHS)
def test_two_passes_are_fft_rows(W):
    rng = np.random.default_rng(W)
    z = np.concatenate([cs16(rng, W), tone(rng, W, W), cs16(rng, W) * np.complex64(1e-3)]).reshape(3, W)
    ure, uim = z.real.astype(F32).copy(), z.imag.astype(F32).copy()
    vre, vim = ure.copy(), uim.copy()
    fft_rows(ure, uim, W)
    two_pass_rows(vre, vim, W)
    np.testing.assert_array_equal(vre.view(np.uint32), ure.view(np.uint32))
    np.testing.assert_array_equal(vim.view(np.uint32), uim.view(np.uint32))


def window_of(kind, W, rng):
    if kind is None:
        return None
    return hann(W) if kind == "hann" else rng.uniform(-1.0, 1.5, W).astype(F32)


def definition_error(W, mean, window, mutation=None):
    rng = np.random.default_rng(W + 3)
    F, S, H = 3, 5, W // 2
    R = (F - 1) * H + W + S
    x = tone(rng, 2 * R, W)
    w = window_of(window, W, rng)
    got = wide_model(x, W, F, S, H, w, mean, mutation=mutation)
    ref = welch_f64(x, W, F, S, H, w, mean)
    return np.inf if got.shape != ref.shape or got.shape[0] != 2 else row_err(got, ref)


@pytest.mark.parametrize("W", WIDE_WIDTHS)
@pytest.mark.parametrize("mean", [False, True])
def test_model_within_bound_of_definition(W, mean):
    for window in (None, "hann", "random"):
        assert definition_error(W, mean, window) <= ROW_BOUND, (W, mean, window)


@pytest.mark.parametrize("W", [8192, 65536])
@pytest.mark.parametrize("hop", ["W/2", "W"])
def test_mean_rows_are_scipy_welch(W, hop):
    signal = pytest.importorskip("scipy.signal")
    H = W // 2 if hop == "W/2" else W
    rng = np.random.default_rng(W + H)
    F, S = 3, 11
    x = tone(rng, 2 * ((F - 1) * H + W + S) + 5, W)
    w = hann(W)
    w = (w * F32(W) / w.sum(dtype=F32)).astype(F32)  # scaling="spectrum"
    rows = wide_model(x, W, F, S, H, w, True)
    assert rows.shape == (2, W)
    R = (F - 1) * H + W + S
    for r in range(2):
        y = x[r * R:r * R + (F - 1) * H + W]
        _, pxx = signal.welch(y.astype(np.complex128), window=w.astype(np.float64), nperseg=W, noverlap=W - H,
                              detrend=False, return_onesided=False, scaling="spectrum", average="mean")
        ref = half_swap(pxx + 1e-20)
        assert np.max(np.abs(rows[r] - ref)) / ref.max() <= WELCH_BOUND, (W, H, r)


def test_blocks_follow_the_last_frame_sample():
    """wide_blocks returns each row with the block holding its last frame sample, across blocks far shorter than
    a frame."""
    W, F, S, H = 8192, 2, 3, 2048
    sizes = [1000, 0, 5000, 8192, 1, 7000, 8192, 8192, 3000]
    rows = wide_blocks(np.zeros(sum(sizes), np.complex64), sizes, W, F, S, H)
    n = sum(r.shape[0] for r in rows)
    where = [b for b, r in enumerate(rows) for _ in range(r.shape[0])]
    assert n == (sum(sizes) - (F - 1) * H - W) // ((F - 1) * H + W + S) + 1
    assert where == list(last_sample_blocks(n, sizes, W, F, S, H))
    assert frames_done(sum(sizes), W, F, S, H) // F == n


def mutation_checks(mutation):
    failed = []
    rng = np.random.default_rng(9)
    for W in (8192, 32768):
        z = welch_frames(tone(rng, 2 * W, W), W, 2, 0, W // 2)
        w = hann(W)
        a = wide_model(z.reshape(-1), W, 1, 0, W, w, two_pass=True, mutation=mutation)
        b = wide_model(z.reshape(-1), W, 1, 0, W, w)
        if a.shape != b.shape or (a.view(np.uint32) != b.view(np.uint32)).any():
            failed.append(f"two passes W={W}")
        if definition_error(W, True, "random", mutation) > ROW_BOUND:
            failed.append(f"definition W={W}")
    return failed


def test_model_passes_every_check():
    assert mutation_checks(None) == []


@pytest.mark.parametrize("mutation", MUTATIONS)
def test_mutation_is_caught(mutation):
    assert mutation_checks(mutation), f"{mutation} passes every check"
