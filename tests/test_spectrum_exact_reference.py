"""The spectrum references (tests/spectrum_exact.py) checked on the CPU, before any GPU test relies on them.

* the kernel model reproduces the reference's four spectrogram goldens (tests/golden/spectrogram) pixel for
  pixel through spectrogram_pixels, and so does the float64 definition;
* the model is within ROW_BOUND of the float64 definition, relative to each row's largest value, at every width
  from 1 to 4096 through both channel stages (the largest error measured is 4.8e-6, at W = 4095 on the direct
  path: a margin of 4x);
* each mutation of the model fails a golden or a definition check;
* the Python helpers follow the reference tool's parameter rules and png_util_set_data's pixel rule.
"""

import numpy as np
import pytest

from exact import to_complex
from spectrum_exact import (GOLDEN_DIR, GOLDEN_FS, GOLDENS, MUTATIONS, f64_rows, half_swap, read_png,
                            golden_stimulus, spec_fft, spectrum_model)
from util import rand_block

ROW_BOUND = 2e-5
WIDTHS = [1, 2, 3, 4, 5, 8, 16, 63, 64, 100, 128, 256, 1000, 1024, 2048, 4095, 4096]


def golden_input(fmt):
    raw = golden_stimulus(fmt)
    return raw if fmt == "cf32" else to_complex(fmt, raw).astype(np.complex64)


def golden_pixels(pkg, name, rows_fn):
    fmt, W = GOLDENS[name]
    F, S = pkg.spectrogram_params(GOLDEN_FS, W)
    return pkg.spectrogram_pixels(rows_fn(golden_input(fmt), W, F, S)), read_png(f"{GOLDEN_DIR}/{name}")


def row_err(got, ref):
    return float(np.max(np.abs(got.astype(np.float64) - ref) / ref.max(axis=1, keepdims=True))) if ref.size else 0.0


@pytest.mark.parametrize("name", sorted(GOLDENS))
def test_model_reproduces_golden(pkg, name):
    got, want = golden_pixels(pkg, name, lambda x, W, F, S: spectrum_model(x, W, F, S, power=False))
    assert want.shape == (2, GOLDENS[name][1])
    np.testing.assert_array_equal(got, want)


@pytest.mark.parametrize("name", sorted(GOLDENS))
def test_definition_reproduces_golden(pkg, name):
    got, want = golden_pixels(pkg, name, lambda x, W, F, S: f64_rows(x, W, F, S, power=False).astype(np.float32))
    np.testing.assert_array_equal(got, want)


@pytest.mark.parametrize("W", WIDTHS)
def test_model_within_bound_of_definition(W):
    rng = np.random.default_rng(W)
    F, S = (2, 3) if W < 1000 else (1, 5)
    n = 2 * (F * W + S) + F * W - 1  # two rows, and a third one sample short
    x = to_complex("cs16", rand_block(rng, "cs16", 2 * n)).astype(np.complex64)
    got, ref = spectrum_model(x, W, F, S), f64_rows(x, W, F, S)
    assert got.shape == ref.shape == (2, W)
    assert row_err(got, ref) <= ROW_BOUND, (W, spec_fft(W))


def test_half_swap_is_the_reference_quirk():
    np.testing.assert_array_equal(half_swap(np.arange(6)), [3, 4, 5, 0, 1, 2])
    np.testing.assert_array_equal(half_swap(np.arange(5)), [2, 3, 0, 1, 4])  # not fftshift's [3, 4, 0, 1, 2]
    np.testing.assert_array_equal(half_swap(np.arange(1)), [0])


def mutation_checks(pkg, mutation):
    """The checks a mutation fails: each golden, the definition on random data, and on silence."""
    failed = []
    for name in sorted(GOLDENS):
        got, want = golden_pixels(pkg, name, lambda x, W, F, S: spectrum_model(x, W, F, S, power=False,
                                                                               mutation=mutation))
        if got.shape != want.shape or (got != want).any():
            failed.append(name)
    rng = np.random.default_rng(3)
    for W, F, S in ((63, 2, 2), (64, 3, 70)):
        x = to_complex("cs16", rand_block(rng, "cs16", 2 * 1000)).astype(np.complex64)
        got, ref = spectrum_model(x, W, F, S, mutation=mutation), f64_rows(x, W, F, S)
        if got.shape != ref.shape or row_err(got, ref) > ROW_BOUND:
            failed.append(f"random W={W}")
    silence = np.zeros(256, np.complex64)
    with np.errstate(divide="ignore"):
        got, ref = spectrum_model(silence, 64, 2, 0, power=False, mutation=mutation), f64_rows(silence, 64, 2, 0,
                                                                                              power=False)
    if not np.allclose(got, ref):
        failed.append("silence")
    return failed


def test_model_passes_every_check(pkg):
    assert mutation_checks(pkg, None) == []


@pytest.mark.parametrize("mutation", MUTATIONS)
def test_mutation_is_caught(pkg, mutation):
    assert mutation_checks(pkg, mutation), f"{mutation} passes every golden and definition check"


def test_spectrogram_params(pkg):
    assert pkg.spectrogram_params(128, 64) == (2, 0)
    assert pkg.spectrogram_params(128, 63) == (2, 2)
    assert pkg.spectrogram_params(2048000, 1000) == (2048, 0)
    assert pkg.spectrogram_params(5, 5) == (1, 0)
    for fs, W in ((128, 0), (128, -1), (0, 64), (-128, 64), (128, 129)):
        with pytest.raises(ValueError):
            pkg.spectrogram_params(fs, W)


def test_spectrogram_pixels(pkg):
    db = np.array([[-300.0, -255.5, -255.0, -254.9, -100.25, -0.5, 0.0, 0.99, 3.0]], np.float32)
    np.testing.assert_array_equal(pkg.spectrogram_pixels(db), [[0, 0, 0, 0, 154, 254, 255, 255, 255]])
    assert pkg.spectrogram_pixels(db).dtype == np.uint8
