"""CPU tests of create_rational_frequency_xlating_filter (include/xlating.h): its argument checks come
before any CUDA call, so they hold on a machine without a GPU, and with valid arguments and no
device it fails loudly like create_frequency_xlating_filter."""
import errno

import numpy as np
import pytest
import torch

FS, MAX_IN = 2048000, 65536


def test_empty_taps_is_minus_one(pkg):
    with pytest.raises(ValueError) as e:
        pkg.XlatingFilter.rational(3, 128, np.zeros(0, dtype=np.float32), 0, FS, MAX_IN)
    assert e.value.args[0] == -1


@pytest.mark.parametrize("interp,decim,fs,max_in", [
    (0, 128, FS, MAX_IN),              # L = 0
    (3, 0, FS, MAX_IN),                # M = 0
    (2098, 1, FS, MAX_IN),             # 2098 * 2.048 MHz > UINT32_MAX
    (65536, 1, 1000, MAX_IN),          # 65536 * 32768 = 2^31 upsampled samples per call
    (2, 1, 1000, 2 ** 31),             # 2 * 2^30 = 2^31
], ids=["L_0", "M_0", "rate_over_u32", "block_2e31", "block_2e31_L2"])
def test_invalid_arguments_refused_before_cuda(pkg, capfd, interp, decim, fs, max_in):
    capfd.readouterr()
    with pytest.raises(ValueError) as e:
        pkg.XlatingFilter.rational(interp, decim, np.ones(8, dtype=np.float32), 0, fs, max_in)
    assert e.value.args[0] == -errno.EINVAL
    assert "<3>" in capfd.readouterr().err


def test_limits_just_inside_pass_the_checks(pkg, capfd):
    """One below each limit is not refused as an argument error (it then needs the GPU)."""
    for interp, decim, fs, max_in in [(2097, 1, FS, 64), (65535, 65536, 1000, MAX_IN)]:
        try:
            f = pkg.XlatingFilter.rational(interp, decim, np.ones(8, dtype=np.float32), 0, fs, max_in)
            f.close()
        except ValueError as e:
            assert e.args[0] != -errno.EINVAL, (interp, decim, fs, max_in)


@pytest.mark.skipif(torch.cuda.is_available(), reason="only meaningful on a box without a GPU")
def test_no_gpu_fails_loudly(pkg, capfd):
    """No CPU fallback for rational filters either: valid arguments without a device -> -ENODEV / -EIO."""
    capfd.readouterr()
    for interp in (1, 3):
        with pytest.raises(ValueError) as e:
            pkg.XlatingFilter.rational(interp, 128, np.ones(97, dtype=np.float32), -12000, FS, MAX_IN)
        assert e.value.args[0] in (-errno.ENODEV, -errno.EIO)
    assert "<3>" in capfd.readouterr().err
