"""The chirp-z spectrum references (tests/spectrum_czt.py) checked on the CPU, before any GPU test relies on them.

* the library's tables (xlg_spectrum_any_tables): the chirp within 2^-24 of e^{-i pi (n^2 mod 2W) / W} per
  component (one rounding of a double), and Bh within half a float32 ulp of each component of the float64 DFT
  plus 1e-12 (the host's double FFT), at every width of CZT_WIDTHS; the refusals of the table query;
* the kernels' pass split (two_pass_rows) is fft_rows at K = M = 131072 bit for bit, and the model with
  two_pass=True equals it;
* the model is within ROW_BOUND of the float64 DFT, relative to each row's largest value, at every width of
  CZT_WIDTHS with a Hann window and the max, and with random weights and the mean (a tone 60 dB over noise; the
  largest error measured is 5.1e-7, at W = 65521 (prime) with a Hann window and the max);
* mean rows with the window w W / sum(w) are scipy.signal.welch's "spectrum" + 1e-20, half swapped, within
  WELCH_BOUND;
* each mutation of the model fails one of these checks.
"""
import numpy as np
import pytest

from bank_fft_exact import fft_rows
from exact import to_complex
from spectrum_czt import CZT_WIDTHS, MUTATIONS, chirp_f64, czt_m, czt_model, kernel_f64, positions
from spectrum_exact import F32, half_swap
from spectrum_welch import hann, welch_f64
from spectrum_wide import two_pass_rows
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


def tables(pkg, W):
    return pkg.spectrum_any_tables(W)


@pytest.mark.parametrize("W", CZT_WIDTHS)
def test_tables_are_the_definitions_rounded(pkg, W):
    chirp, kern, M = tables(pkg, W)
    assert M == czt_m(W) and chirp.shape == (W,) and kern.shape == (M,)
    c64 = chirp_f64(W)
    assert np.max(np.abs(chirp.real - c64.real)) <= 2.0 ** -24
    assert np.max(np.abs(chirp.imag - c64.imag)) <= 2.0 ** -24
    _, bins = positions(M)
    k64 = kernel_f64(W)[bins]
    for got, ref in ((kern.real, k64.real), (kern.imag, k64.imag)):
        bound = 0.5 * np.spacing(np.abs(ref).astype(F32)).astype(np.float64) + 1e-12
        assert np.all(np.abs(got.astype(np.float64) - ref) <= bound), W


def test_table_query_refusals(pkg):
    for W in (0, 1, 4096, 8192, 65536, 65537, 131072):
        with pytest.raises(ValueError):
            pkg.spectrum_any_tables(W)
    assert pkg.spectrum_any_tables(65535)[2] == 131072


def test_two_passes_are_fft_rows_at_131072():
    M = 131072
    rng = np.random.default_rng(M)
    z = np.concatenate([cs16(rng, M), tone(rng, M, 5000)]).reshape(2, M)
    ure, uim = z.real.astype(F32).copy(), z.imag.astype(F32).copy()
    vre, vim = ure.copy(), uim.copy()
    fft_rows(ure, uim, M)
    two_pass_rows(vre, vim, M)
    np.testing.assert_array_equal(vre.view(np.uint32), ure.view(np.uint32))
    np.testing.assert_array_equal(vim.view(np.uint32), uim.view(np.uint32))


@pytest.mark.parametrize("W", [5000, 48000])
def test_model_two_pass_equals_model(pkg, W):
    rng = np.random.default_rng(W)
    x = tone(rng, W, W)
    a = czt_model(x, W, 1, 0, tables(pkg, W), two_pass=True)
    b = czt_model(x, W, 1, 0, tables(pkg, W))
    assert a.shape == (1, W)
    np.testing.assert_array_equal(a.view(np.uint32), b.view(np.uint32))


def definition_error(pkg, W, mean, window, mutation=None):
    rng = np.random.default_rng(W + 3)
    F, S, H = 2, 5, W // 2
    R = (F - 1) * H + W + S
    x = tone(rng, R + (F - 1) * H + W, W)
    w = hann(W) if window == "hann" else rng.uniform(-1.0, 1.5, W).astype(F32)
    got = czt_model(x, W, F, S, tables(pkg, W), H, w, mean, mutation=mutation)
    ref = welch_f64(x, W, F, S, H, w, mean)
    return np.inf if got.shape != ref.shape or got.shape[0] != 2 else row_err(got, ref)


@pytest.mark.parametrize("W", CZT_WIDTHS)
def test_model_within_bound_of_definition(pkg, W):
    for mean, window in ((False, "hann"), (True, "random")):
        assert definition_error(pkg, W, mean, window) <= ROW_BOUND, (W, mean, window)


@pytest.mark.parametrize("W", [5000, 48000])
def test_mean_rows_are_scipy_welch(pkg, W):
    signal = pytest.importorskip("scipy.signal")
    H = W // 2
    rng = np.random.default_rng(W + H)
    F, S = 3, 11
    x = tone(rng, (F - 1) * H + W, W)
    w = hann(W)
    w = (w * F32(W) / w.sum(dtype=F32)).astype(F32)  # scaling="spectrum"
    rows = czt_model(x, W, F, S, tables(pkg, W), H, w, True)
    assert rows.shape == (1, W)
    _, pxx = signal.welch(x.astype(np.complex128), window=w.astype(np.float64), nperseg=W, noverlap=W - H,
                          detrend=False, return_onesided=False, scaling="spectrum", average="mean")
    ref = half_swap(pxx + 1e-20)
    assert np.max(np.abs(rows[0] - ref)) / ref.max() <= WELCH_BOUND, W


def mutation_checks(pkg, mutation):
    """The definition check at W = 12288 (M = 32768, where bank_fft_pos is not its own inverse) and at W = 48000
    (M = 131072, past the 32-bit index's overflow at n = 46341)."""
    return [W for W in (12288, 48000) if definition_error(pkg, W, False, "hann", mutation) > ROW_BOUND]


def test_model_passes_every_check(pkg):
    assert mutation_checks(pkg, None) == []


@pytest.mark.parametrize("mutation", MUTATIONS)
def test_mutation_is_caught(pkg, mutation):
    assert mutation_checks(pkg, mutation), f"{mutation} passes every check"
