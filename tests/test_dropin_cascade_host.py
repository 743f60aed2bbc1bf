"""CPU tests of create_cascade_frequency_xlating_filter (include/xlating.h): its argument checks come before
any CUDA call, so they hold on a machine without a GPU; empty tap vectors are not adopted, refused ones are
freed; and with valid arguments and no device it fails loudly like create_frequency_xlating_filter."""
import ctypes as C
import errno
import os
import subprocess
import sys
import textwrap

import numpy as np
import pytest
import torch

FS, MAX_IN = 61440000, 65536
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class _Mallinfo2(C.Structure):
    _fields_ = [(n, C.c_size_t) for n in ("arena", "ordblks", "smblks", "hblks", "hblkhd", "usmblks", "fsmblks",
                                          "uordblks", "fordblks", "keepcost")]


_libc = C.CDLL("libc.so.6")
_libc.malloc.restype = C.c_void_p
_libc.malloc.argtypes = [C.c_size_t]
_libc.free.argtypes = [C.c_void_p]
_libc.mallinfo2.restype = _Mallinfo2


def _create(pkg, d1, t1_len, d2, t2_len, interp2=1, fs=FS, max_in=MAX_IN, t1=None, t2=None):
    """The C call with malloc()ed vectors of ones; returns (code, t1 pointer, t2 pointer)."""
    lib = pkg.lib()
    t1 = t1 if t1 is not None else (_libc.malloc(4 * t1_len) if t1_len else None)
    t2 = t2 if t2 is not None else (_libc.malloc(4 * t2_len) if t2_len else None)
    for p, n in ((t1, t1_len), (t2, t2_len)):
        if p:
            C.memmove(p, np.ones(n, dtype=np.float32).ctypes.data, 4 * n)
    h = C.c_void_p()
    code = lib.create_cascade_frequency_xlating_filter(d1, t1, t1_len, 0, interp2, d2, t2, t2_len, fs, max_in,
                                                       C.byref(h))
    if code == 0:
        lib.destroy_xlating(h)
    return code, t1, t2


# taps at the stage-B limit: an integer stage B needs 16 + 4 ceil4(T2) + 8 floor2(T2 + 2) <= 200 KiB of shared
# memory for one output (cascade_smem), so T2 = 17064 fits and 17065 does not; a rational one with L2 = 12
# needs 16 + 4 ceil4(12 Tb2) + 8 floor2(Tb2 + 3) (cascade_poly_smem), so Tb2 = 3656 fits and 3657 does not
T2_MAX = 17064


@pytest.mark.parametrize("d1,d2,interp2,t2,max_in", [
    (0, 40, 1, 481, MAX_IN),              # decimation1 = 0
    (32, 0, 1, 481, MAX_IN),              # decimation2 = 0
    (32, 40, 0, 481, MAX_IN),             # interpolation2 = 0
    (2, 1, 4, 4, 2 ** 31),                # 4 * (2^29 + 2) >= 2^31
    (32, 40, 1, T2_MAX + 1, MAX_IN),      # integer stage B does not fit shared memory
    (20, 125, 12, 12 * 3657, MAX_IN),     # rational stage B (12 branches of 3657) does not fit
], ids=["d1_0", "d2_0", "interp2_0", "upsampled_2e31", "smem_integer", "smem_rational"])
def test_invalid_arguments_refused_before_cuda(pkg, capfd, d1, d2, interp2, t2, max_in):
    capfd.readouterr()
    code, _, _ = _create(pkg, d1, 79, d2, t2, interp2=interp2, max_in=max_in)
    assert code == -errno.EINVAL
    err = capfd.readouterr().err
    assert err.count("<3>") == 1, err
    # refused before any CUDA call: on this machine a CUDA call would have logged "no usable CUDA device"
    assert "CUDA" not in err


def test_refused_taps_are_freed(pkg, capfd):
    """Refused vectors are adopted and freed: the heap's in-use bytes return to where they were."""
    n = 20000  # 80 KB each, below glibc's mmap threshold: counted in uordblks
    _create(pkg, 0, n, 40, n)  # warm the library's own allocations up
    before = _libc.mallinfo2().uordblks
    for _ in range(20):
        code, _, _ = _create(pkg, 0, n, 40, n)
        assert code == -errno.EINVAL
    assert _libc.mallinfo2().uordblks - before < 2 * 4 * n


@pytest.mark.parametrize("empty", ["taps1", "taps2", "both"])
def test_empty_taps_is_minus_one_and_not_adopted(pkg, empty):
    """-1 and neither vector adopted: the caller can still free both (in a child process, so that a
    double free would fail that process and not this one)."""
    t1_len = 0 if empty in ("taps1", "both") else 79
    t2_len = 0 if empty in ("taps2", "both") else 481
    code = textwrap.dedent(f"""
        import ctypes as C, importlib, sys
        sys.path.insert(0, {ROOT!r})
        pkg = importlib.import_module("sdr-server_b200")
        libc = C.CDLL("libc.so.6")
        libc.malloc.restype = C.c_void_p
        libc.malloc.argtypes = [C.c_size_t]
        libc.free.argtypes = [C.c_void_p]
        t1, t2 = libc.malloc(4 * 79), libc.malloc(4 * 481)
        h = C.c_void_p()
        rc = pkg.lib().create_cascade_frequency_xlating_filter(32, t1, {t1_len}, 0, 1, 40, t2, {t2_len}, {FS},
                                                               {MAX_IN}, C.byref(h))
        libc.free(t1)
        libc.free(t2)
        print(rc)
    """)
    r = subprocess.run([sys.executable, "-c", code], capture_output=True, text=True, timeout=120)
    assert r.returncode == 0, r.stderr
    assert r.stdout.strip() == "-1"


@pytest.mark.parametrize("d1,d2,interp2,t2,max_in", [
    (1, 1, 1, 481, MAX_IN),                    # every decimation and interpolation at 1
    # 3 * (2^29 + 2) < 2^31 (gigabytes of buffers where a GPU is present)
    pytest.param(2, 1, 3, 4, 2 ** 31, marks=pytest.mark.skipif(torch.cuda.is_available(), reason="no GPU only")),
    (32, 40, 1, T2_MAX, MAX_IN),               # the longest integer stage B
    (20, 125, 12, 12 * 3656, MAX_IN),          # the longest rational stage B with 12 branches
], ids=["ones", "upsampled_below_2e31", "smem_integer", "smem_rational"])
def test_limits_just_inside_pass_the_checks(pkg, capfd, d1, d2, interp2, t2, max_in):
    """One step below each limit is not refused as an argument error: without a GPU it reaches -ENODEV."""
    capfd.readouterr()
    code, _, _ = _create(pkg, d1, 79, d2, t2, interp2=interp2, max_in=max_in)
    assert code != -errno.EINVAL, capfd.readouterr().err
    if not torch.cuda.is_available():
        assert code == -errno.ENODEV


@pytest.mark.skipif(torch.cuda.is_available(), reason="only meaningful on a box without a GPU")
def test_no_gpu_fails_loudly(pkg, capfd):
    """No CPU fallback: valid arguments without a device -> -ENODEV and a <3> line."""
    plan = pkg.cascade_plan(FS, [48000])[0]
    capfd.readouterr()
    with pytest.raises(ValueError) as e:
        pkg.XlatingFilter.cascade(plan["d1"], plan["taps1"], plan["center"], plan["d2"], plan["taps2"], FS, MAX_IN,
                                  interp2=plan["interp2"])
    assert e.value.args[0] == -errno.ENODEV
    assert "<3>" in capfd.readouterr().err
