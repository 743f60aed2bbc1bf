"""sdr-server_b200 -- H100-native frequency-translating FIR decimator.

Thin ctypes bindings over ``lib/libxlating_b200.so`` (C ABI declared in
``include/xlating.h``, ``include/xlating_group.h``, ``include/lpf.h``).  The host
side of the product is C/C++ like the reference; this module only exists so that
the parity tests and ``bench.py`` can drive the C ABI the way the reference's own
callers do (``src/dsp_worker.c:98-124``, ``test/test_xlating.c``):

* :func:`create_low_pass_filter`  -> ``create_low_pass_filter``  (src/lpf.h:6)
* :class:`XlatingFilter`          -> ``create_frequency_xlating_filter`` /
  ``process_{native,optimized}_{cu8,cs8,cs16}_{cf32,cs16}`` / ``destroy_xlating``
  (src/xlating.h:10-38); :meth:`XlatingFilter.rational` and :meth:`XlatingFilter.cascade` -> the
  extensions ``create_rational_frequency_xlating_filter`` and ``create_cascade_frequency_xlating_filter``
* :class:`Group`                  -> the batch extension ``xlg_*``

There is no CPU fallback anywhere: if the shared library is missing, or no sm_90
GPU (H100) is present, the calls fail loudly.

The directory name contains a hyphen; import it with
``importlib.import_module("sdr-server_b200")``.
"""
from __future__ import annotations

import ctypes as C
import math
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
# XLATING_B200_LIB: an A/B measurement switch (another build of the SAME library, e.g. other tile constants)
LIB_PATH = os.environ.get("XLATING_B200_LIB") or os.path.join(HERE, "lib", "libxlating_b200.so")

FMT = {"cu8": 0, "cs8": 1, "cs16": 2, "cf32": 3}
NP_DTYPE = {"cu8": np.uint8, "cs8": np.int8, "cs16": np.int16, "cf32": np.float32}

XLG_OUT_DEVICE = 0x1
XLG_NO_RENORM = 0x2
XLG_FORCE_GENERIC = 0x4
XLG_SM_PARTITION = 0x10
XLG_TRACK_STATE = 0x20
XLG_INPUT_DEVICE = 0x100
XLG_PATH_Q15 = 0x200
XLG_INPUT_KEEP = 0x400
XLG_SPECTRUM_POWER = 0x1  # xlg_add_spectrum flag
XLG_SLOTS = 4

# every symbol the headers declare (checked by tests/test_abi.py)
REFERENCE_SYMBOLS = (
    ["create_frequency_xlating_filter", "destroy_xlating", "SIMD_STATUS", "create_low_pass_filter"]
    + [f"process_{v}_{f}_{o}" for v in ("native", "optimized") for f in ("cu8", "cs8", "cs16") for o in ("cf32", "cs16")]
)
# include/xlating.h's extension of the reference's per-filter ABI
DROPIN_EXTENSION_SYMBOLS = ["create_rational_frequency_xlating_filter", "create_cascade_frequency_xlating_filter"]
GROUP_SYMBOLS = [
    "xlg_create", "xlg_create_ex", "xlg_destroy", "xlg_add_client", "xlg_add_client_ex", "xlg_add_client_rational_ex", "xlg_remove_client", "xlg_reserve", "xlg_client_count", "xlg_submit",
    "xlg_wait", "xlg_input_consumed", "xlg_output", "xlg_read_output", "xlg_copy_output", "xlg_alloc_pinned", "xlg_free_pinned", "xlg_wait_stream", "xlg_partition_active", "xlg_timer_start",
    "xlg_timer_stop", "xlg_profile_enable", "xlg_profile_read", "xlg_client_info", "xlg_add_client_rational", "xlg_poly_profile_read", "xlg_add_client_cascade", "xlg_add_client_cascade_rational", "xlg_cascade_info", "xlg_cascade_profile_read", "xlg_add_subband", "xlg_remove_subband", "xlg_add_client_subband", "xlg_add_client_subband_rational", "xlg_subband_info", "xlg_subband_profile_read", "xlg_add_bank", "xlg_add_bank_subband", "xlg_remove_bank", "xlg_bank_profile_read", "xlg_add_spectrum_any", "xlg_spectrum_any_tables", "xlg_add_bank_any", "xlg_bank_any_tables", "xlg_dropin_stats", "xlg_dropin_stream_stats", "xlg_dropin_stream_times",
]


class XlgProfile(C.Structure):
    _fields_ = [("fir_tile_ms", C.c_double), ("fir_generic_ms", C.c_double), ("phase_ms", C.c_double),
                ("convert_ms", C.c_double), ("fir_tile_launches", C.c_uint64),
                ("fir_generic_launches", C.c_uint64), ("phase_launches", C.c_uint64),
                ("convert_launches", C.c_uint64), ("blocks", C.c_uint64), ("out_samples", C.c_uint64),
                ("in_samples", C.c_uint64), ("tile_macs", C.c_uint64), ("algo_macs", C.c_uint64),
                ("fir_long_ms", C.c_double), ("fir_long_launches", C.c_uint64),
                ("host_submit_ms", C.c_double), ("host_wait_ms", C.c_double), ("submits", C.c_uint64)]


class XlgClientState(C.Structure):
    """xlg_client_state (include/xlating_group.h)."""
    _fields_ = [("valid_history", C.c_int64), ("hist", C.c_int64), ("phase_re", C.c_float), ("phase_im", C.c_float)]


class XlgPolyProfile(C.Structure):
    _fields_ = [("fir_poly_tile_ms", C.c_double), ("fir_poly_generic_ms", C.c_double),
                ("fir_poly_tile_launches", C.c_uint64), ("fir_poly_generic_launches", C.c_uint64),
                ("poly_macs", C.c_uint64)]


class XlgCascadeProfile(C.Structure):
    _fields_ = [("stage_b_ms", C.c_double), ("stage_b_launches", C.c_uint64), ("stage_b_macs", C.c_uint64),
                ("d2h_bytes", C.c_uint64)]


class XlgSubbandProfile(C.Structure):
    _fields_ = [("member_ms", C.c_double), ("member_launches", C.c_uint64), ("member_macs", C.c_uint64),
                ("row_samples", C.c_uint64)]


class XlgBankProfile(C.Structure):
    _fields_ = [("bank_ms", C.c_double), ("bank_launches", C.c_uint64), ("poly_macs", C.c_uint64),
                ("dft_macs", C.c_uint64)]


class XlgBankFftProfile(C.Structure):
    _fields_ = [("fft_ms", C.c_double), ("fft_launches", C.c_uint64), ("poly_macs", C.c_uint64),
                ("butterfly_flops", C.c_uint64)]


class XlgSpectrumProfile(C.Structure):
    _fields_ = [("spectrum_ms", C.c_double), ("spectrum_launches", C.c_uint64), ("frames", C.c_uint64),
                ("channel_flops", C.c_uint64)]


class XlgSpectrumDesc(C.Structure):  # xlg_add_spectrum_ex
    _fields_ = [("width", C.c_uint32), ("frames_per_row", C.c_uint32), ("skip_per_row", C.c_uint32),
                ("flags", C.c_uint32), ("hop", C.c_uint32), ("reduce", C.c_uint32),
                ("window", C.POINTER(C.c_float))]


def build(verbose: bool = False) -> None:
    """Compile lib/libxlating_b200.so for sm_90a (nvcc cross-compiles without a GPU)."""
    subprocess.run(["make", "-C", HERE, "all"], check=True,
                   stdout=None if verbose else subprocess.DEVNULL)


_lib = None


def lib() -> C.CDLL:
    """Load the C ABI.  Raises if the CUDA library has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(f"{LIB_PATH} is missing: run `make -C {HERE}` (or __graft_entry__.build()); "
                           "there is no CPU fallback")
    L = C.CDLL(LIB_PATH)
    vp, sz, u32, i32 = C.c_void_p, C.c_size_t, C.c_uint32, C.c_int32
    L.create_low_pass_filter.argtypes = [C.c_float, u32, u32, u32, C.POINTER(vp), C.POINTER(sz)]
    L.create_low_pass_filter.restype = C.c_int
    L.create_frequency_xlating_filter.argtypes = [u32, vp, sz, i32, u32, u32, C.POINTER(vp)]
    L.create_frequency_xlating_filter.restype = C.c_int
    L.create_rational_frequency_xlating_filter.argtypes = [u32, u32, vp, sz, i32, u32, u32, C.POINTER(vp)]
    L.create_rational_frequency_xlating_filter.restype = C.c_int
    L.create_cascade_frequency_xlating_filter.argtypes = [u32, vp, sz, i32, u32, u32, vp, sz, u32, u32, C.POINTER(vp)]
    L.create_cascade_frequency_xlating_filter.restype = C.c_int
    L.destroy_xlating.argtypes = [vp]
    L.destroy_xlating.restype = None
    for v in ("native", "optimized"):
        for f in ("cu8", "cs8", "cs16"):
            for o in ("cf32", "cs16"):
                fn = getattr(L, f"process_{v}_{f}_{o}")
                fn.argtypes = [vp, sz, C.POINTER(vp), C.POINTER(sz), vp]
                fn.restype = None
    L.xlg_create.argtypes = [C.c_int, u32, u32, u32, C.POINTER(vp)]
    L.xlg_create.restype = C.c_int
    L.xlg_create_ex.argtypes = [C.c_int, u32, u32, u32, u32, C.POINTER(vp)]
    L.xlg_create_ex.restype = C.c_int
    L.xlg_destroy.argtypes = [vp]
    L.xlg_destroy.restype = None
    L.xlg_add_client.argtypes = [vp, u32, C.POINTER(C.c_float), sz, i32, C.POINTER(C.c_int)]
    L.xlg_add_client.restype = C.c_int
    L.xlg_add_client_ex.argtypes = [vp, u32, C.POINTER(C.c_float), sz, i32, C.POINTER(XlgClientState),
                                    C.POINTER(C.c_int)]
    L.xlg_add_client_ex.restype = C.c_int
    L.xlg_add_client_rational.argtypes = [vp, u32, u32, C.POINTER(C.c_float), sz, i32, C.POINTER(C.c_int)]
    L.xlg_add_client_rational.restype = C.c_int
    L.xlg_add_client_rational_ex.argtypes = [vp, u32, u32, C.POINTER(C.c_float), sz, i32, C.POINTER(XlgClientState),
                                             C.POINTER(C.c_int)]
    L.xlg_add_client_rational_ex.restype = C.c_int
    L.xlg_poly_profile_read.argtypes = [vp, C.POINTER(XlgPolyProfile), C.c_int]
    L.xlg_poly_profile_read.restype = C.c_int
    fp = C.POINTER(C.c_float)
    L.xlg_add_client_cascade.argtypes = [vp, u32, fp, sz, i32, u32, fp, sz, C.POINTER(C.c_int)]
    L.xlg_add_client_cascade.restype = C.c_int
    L.xlg_add_client_cascade_rational.argtypes = [vp, u32, fp, sz, i32, u32, u32, fp, sz, C.POINTER(C.c_int)]
    L.xlg_add_client_cascade_rational.restype = C.c_int
    L.xlg_cascade_info.argtypes = [vp, C.c_int, C.POINTER(C.c_int), C.POINTER(sz), C.POINTER(sz)]
    L.xlg_cascade_info.restype = C.c_int
    L.xlg_cascade_profile_read.argtypes = [vp, C.POINTER(XlgCascadeProfile), C.c_int]
    L.xlg_cascade_profile_read.restype = C.c_int
    L.xlg_add_subband.argtypes = [vp, u32, fp, sz, i32, C.POINTER(C.c_int)]
    L.xlg_add_subband.restype = C.c_int
    L.xlg_remove_subband.argtypes = [vp, C.c_int]
    L.xlg_remove_subband.restype = C.c_int
    L.xlg_add_client_subband.argtypes = [vp, C.c_int, u32, fp, sz, i32, C.POINTER(C.c_int)]
    L.xlg_add_client_subband.restype = C.c_int
    L.xlg_add_client_subband_rational.argtypes = [vp, C.c_int, u32, u32, fp, sz, i32, C.POINTER(C.c_int)]
    L.xlg_add_client_subband_rational.restype = C.c_int
    L.xlg_subband_info.argtypes = [vp, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_int), C.POINTER(sz)]
    L.xlg_subband_info.restype = C.c_int
    L.xlg_subband_profile_read.argtypes = [vp, C.POINTER(XlgSubbandProfile), C.c_int]
    L.xlg_subband_profile_read.restype = C.c_int
    L.xlg_add_bank.argtypes = [vp, u32, fp, sz, C.POINTER(C.c_int)]
    L.xlg_add_bank.restype = C.c_int
    L.xlg_add_bank_subband.argtypes = [vp, C.c_int, i32, C.POINTER(C.c_int)]
    L.xlg_add_bank_subband.restype = C.c_int
    L.xlg_remove_bank.argtypes = [vp, C.c_int]
    L.xlg_remove_bank.restype = C.c_int
    L.xlg_bank_profile_read.argtypes = [vp, C.POINTER(XlgBankProfile), C.c_int]
    L.xlg_bank_profile_read.restype = C.c_int
    L.xlg_add_bank_fft.argtypes = [vp, u32, fp, sz, C.POINTER(C.c_int)]
    L.xlg_add_bank_fft.restype = C.c_int
    L.xlg_bank_fft_profile_read.argtypes = [vp, C.POINTER(XlgBankFftProfile), C.c_int]
    L.xlg_bank_fft_profile_read.restype = C.c_int
    L.xlg_bank_fft_flops.argtypes = [u32]
    L.xlg_bank_fft_flops.restype = C.c_uint64
    L.xlg_add_bank_any.argtypes = [vp, u32, fp, sz, C.POINTER(C.c_int)]
    L.xlg_add_bank_any.restype = C.c_int
    L.xlg_bank_any_tables.argtypes = [u32, fp, fp, C.POINTER(C.c_uint32)]
    L.xlg_bank_any_tables.restype = C.c_int
    L.xlg_add_spectrum.argtypes = [vp, u32, u32, u32, u32, C.POINTER(C.c_int)]
    L.xlg_add_spectrum.restype = C.c_int
    L.xlg_add_client_spectrum.argtypes = [vp, C.c_int, u32, u32, u32, u32, C.POINTER(C.c_int)]
    L.xlg_add_client_spectrum.restype = C.c_int
    L.xlg_add_subband_spectrum.argtypes = [vp, C.c_int, u32, u32, u32, u32, C.POINTER(C.c_int)]
    L.xlg_add_subband_spectrum.restype = C.c_int
    L.xlg_add_spectrum_ex.argtypes = [vp, C.c_int, C.c_int, C.POINTER(XlgSpectrumDesc), C.POINTER(C.c_int)]
    L.xlg_add_spectrum_ex.restype = C.c_int
    L.xlg_add_spectrum_any.argtypes = [vp, C.c_int, C.c_int, C.POINTER(XlgSpectrumDesc), C.POINTER(C.c_int)]
    L.xlg_add_spectrum_any.restype = C.c_int
    L.xlg_spectrum_any_tables.argtypes = [u32, fp, fp, C.POINTER(C.c_uint32)]
    L.xlg_spectrum_any_tables.restype = C.c_int
    L.xlg_remove_spectrum.argtypes = [vp, C.c_int]
    L.xlg_remove_spectrum.restype = C.c_int
    L.xlg_spectrum_output.argtypes = [vp, C.c_int64, C.c_int, C.POINTER(C.POINTER(C.c_float)), C.POINTER(sz)]
    L.xlg_spectrum_output.restype = C.c_int
    L.xlg_spectrum_width.argtypes = [vp, C.c_int64, C.c_int, C.POINTER(C.c_uint32)]
    L.xlg_spectrum_width.restype = C.c_int
    L.xlg_read_spectrum.argtypes = [vp, C.c_int64, C.c_int, fp, sz, C.POINTER(sz)]
    L.xlg_read_spectrum.restype = C.c_int
    L.xlg_spectrum_info.argtypes = [vp, C.c_int, C.POINTER(C.c_int), C.POINTER(C.c_uint64)]
    L.xlg_spectrum_info.restype = C.c_int
    L.xlg_spectrum_profile_read.argtypes = [vp, C.POINTER(XlgSpectrumProfile), C.c_int]
    L.xlg_spectrum_profile_read.restype = C.c_int
    L.xl_poly_pack.argtypes = [C.POINTER(C.c_float), sz, u32, C.POINTER(C.c_float)]
    L.xl_poly_pack.restype = None
    L.xlg_reserve.argtypes = [vp, sz]
    L.xlg_reserve.restype = C.c_int
    L.xlg_remove_client.argtypes = [vp, C.c_int]
    L.xlg_remove_client.restype = C.c_int
    L.xlg_client_count.argtypes = [vp]
    L.xlg_client_count.restype = C.c_int
    L.xlg_submit.argtypes = [vp, C.c_int, vp, sz, u32]
    L.xlg_submit.restype = C.c_int64
    L.xlg_wait.argtypes = [vp, C.c_int64]
    L.xlg_wait.restype = C.c_int
    L.xlg_input_consumed.argtypes = [vp, C.c_int64]
    L.xlg_input_consumed.restype = C.c_int
    L.xlg_output.argtypes = [vp, C.c_int64, C.c_int, C.POINTER(vp), C.POINTER(sz)]
    L.xlg_output.restype = C.c_int
    L.xlg_read_output.argtypes = [vp, C.c_int64, C.c_int, vp, sz, C.POINTER(sz)]
    L.xlg_read_output.restype = C.c_int
    L.xlg_copy_output.argtypes = [vp, C.c_int64, C.c_int, vp, sz, C.POINTER(sz), C.POINTER(XlgClientState)]
    L.xlg_copy_output.restype = C.c_int
    L.xlg_alloc_pinned.argtypes = [sz]
    L.xlg_alloc_pinned.restype = vp
    L.xlg_free_pinned.argtypes = [vp]
    L.xlg_free_pinned.restype = None
    L.xlg_wait_stream.argtypes = [vp, vp]
    L.xlg_wait_stream.restype = C.c_int
    L.xlg_partition_active.argtypes = [vp]
    L.xlg_partition_active.restype = C.c_int
    L.xlg_timer_start.argtypes = [vp]
    L.xlg_timer_start.restype = C.c_int
    L.xlg_timer_stop.argtypes = [vp, C.POINTER(C.c_float)]
    L.xlg_timer_stop.restype = C.c_int
    L.xlg_profile_enable.argtypes = [vp, C.c_int]
    L.xlg_profile_enable.restype = C.c_int
    L.xlg_profile_read.argtypes = [vp, C.POINTER(XlgProfile), C.c_int]
    L.xlg_profile_read.restype = C.c_int
    L.xlg_client_info.argtypes = [vp, C.c_int, C.POINTER(sz), C.POINTER(C.c_int)]
    L.xlg_client_info.restype = C.c_int
    _lib = L
    return L


_libc = C.CDLL(None)
_libc.malloc.restype = C.c_void_p
_libc.malloc.argtypes = [C.c_size_t]
_libc.free.argtypes = [C.c_void_p]


def simd_status() -> str:
    return C.c_char_p.in_dll(lib(), "SIMD_STATUS").value.decode()


def dropin_stats(device: int = 0):
    """(batches, calls, shared_inputs) of the per-filter drop-in ABI on `device`: how many
    launches the process_* calls made so far were combined into, and how many calls found
    their input already staged by another filter (csrc/xlating_dropin.cu)."""
    b, c, s = C.c_uint64(0), C.c_uint64(0), C.c_uint64(0)
    fn = lib().xlg_dropin_stats
    fn.argtypes = [C.c_int, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]
    fn.restype = C.c_int
    rc = fn(device, C.byref(b), C.byref(c), C.byref(s))
    if rc != 0:
        raise RuntimeError(f"xlg_dropin_stats -> {rc}")
    return b.value, c.value, s.value


def dropin_stream_stats(device: int = 0) -> dict:
    """Counters of the drop-in engine's stream overlay (csrc/stream_overlay.h)."""
    arr = (C.c_uint64 * 7)()
    fn = lib().xlg_dropin_stream_stats
    fn.argtypes = [C.c_int, C.POINTER(C.c_uint64)]
    fn.restype = C.c_int
    rc = fn(device, arr)
    if rc != 0:
        raise RuntimeError(f"xlg_dropin_stream_stats -> {rc}")
    keys = ("served_by_group", "published", "hits", "desyncs", "joins", "private_matches", "members")
    return dict(zip(keys, [int(v) for v in arr]))


def create_low_pass_filter(gain: float, sampling_freq: int, cutoff_freq: int, transition_width: int) -> np.ndarray:
    """Host tap designer (reference: src/lpf.c:53-99).  Raises ValueError(code) on failure."""
    p = C.c_void_p()
    n = C.c_size_t(0)
    code = lib().create_low_pass_filter(gain, sampling_freq, cutoff_freq, transition_width, C.byref(p), C.byref(n))
    if code != 0:
        raise ValueError(code)
    out = np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_float)), shape=(n.value,)).copy()
    _libc.free(p)
    return out


def _adoptable(taps: np.ndarray):
    """A malloc()ed copy of `taps` for a constructor that adopts (and later free()s) the vector, as the
    reference does; None for an empty vector."""
    if len(taps) == 0:
        return None
    mem = _libc.malloc(taps.nbytes)
    C.memmove(mem, taps.ctypes.data, taps.nbytes)
    return mem


class XlatingFilter:
    """Per-client drop-in filter (reference API: src/xlating.h:10-38)."""

    def __init__(self, decimation: int, taps, center_freq: int, sampling_freq: int, max_input_buffer_length: int,
                 interp: int | None = None, stage_b=None):
        self._L = lib()
        taps = np.ascontiguousarray(taps, dtype=np.float32)
        mem = _adoptable(taps)
        h = C.c_void_p()
        if stage_b is not None:
            interp2, decim2, taps2 = stage_b
            taps2 = np.ascontiguousarray(taps2, dtype=np.float32)
            code = self._L.create_cascade_frequency_xlating_filter(decimation, mem, len(taps), center_freq, interp2,
                                                                   decim2, _adoptable(taps2), len(taps2),
                                                                   sampling_freq, max_input_buffer_length, C.byref(h))
        elif interp is None:
            code = self._L.create_frequency_xlating_filter(decimation, mem, len(taps), center_freq, sampling_freq,
                                                           max_input_buffer_length, C.byref(h))
        else:
            code = self._L.create_rational_frequency_xlating_filter(interp, decimation, mem, len(taps), center_freq,
                                                                    sampling_freq, max_input_buffer_length, C.byref(h))
        self._h = None
        if code != 0:
            raise ValueError(code)
        self._h = h

    @classmethod
    def rational(cls, interp: int, decim: int, taps, center_freq: int, sampling_freq: int,
                 max_input_buffer_length: int) -> "XlatingFilter":
        """A filter at sampling_freq * interp / decim (include/xlating.h,
        create_rational_frequency_xlating_filter): the filter with decimation `decim` at
        interp * sampling_freq fed the zero-stuffed stream.  Taps are designed at interp * sampling_freq."""
        return cls(decim, taps, center_freq, sampling_freq, max_input_buffer_length, interp=interp)

    @classmethod
    def cascade(cls, decim1: int, taps1, center_freq: int, decim2: int, taps2, sampling_freq: int,
                max_input_buffer_length: int, interp2: int = 1) -> "XlatingFilter":
        """A two-stage filter (include/xlating.h, create_cascade_frequency_xlating_filter): the filter
        (decim1, taps1, center_freq) at sampling_freq, followed by the filter (decim2, taps2, centre 0) at
        interp2 * sampling_freq / decim1 fed its zero-stuffed outputs.  Equal, call for call, to the client of
        Group.add_client_cascade with the same arguments.  See cascade_plan for taps."""
        return cls(decim1, taps1, center_freq, sampling_freq, max_input_buffer_length,
                   stage_b=(interp2, decim2, taps2))

    def _call(self, name: str, data: np.ndarray):
        out = C.c_void_p()
        n = C.c_size_t(0)
        getattr(self._L, name)(data.ctypes.data, data.size, C.byref(out), C.byref(n), self._h)
        return out, n.value

    def process_cf32(self, fmt: str, data, variant: str = "native") -> np.ndarray:
        data = np.ascontiguousarray(data, dtype=NP_DTYPE[fmt])
        out, n = self._call(f"process_{variant}_{fmt}_cf32", data)
        if n == 0:
            return np.zeros(0, dtype=np.complex64)
        return np.ctypeslib.as_array(C.cast(out, C.POINTER(C.c_float)), shape=(2 * n,)).copy().view(np.complex64)

    def process_q15(self, fmt: str, data, variant: str = "native") -> np.ndarray:
        data = np.ascontiguousarray(data, dtype=NP_DTYPE[fmt])
        out, n = self._call(f"process_{variant}_{fmt}_cs16", data)
        if n == 0:
            return np.zeros((0, 2), dtype=np.int16)
        return np.ctypeslib.as_array(C.cast(out, C.POINTER(C.c_int16)), shape=(2 * n,)).copy().reshape(-1, 2)

    def close(self):
        if self._h:
            self._L.destroy_xlating(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class Group:
    """Many clients on one wideband stream (include/xlating_group.h)."""

    def __init__(self, sampling_freq: int, max_input_len: int, device: int = 0, flags: int = 0, host_ring: int = 0):
        self._L = lib()
        h = C.c_void_p()
        if host_ring:
            code = self._L.xlg_create_ex(device, sampling_freq, max_input_len, flags, host_ring, C.byref(h))
        else:
            code = self._L.xlg_create(device, sampling_freq, max_input_len, flags, C.byref(h))
        self._h = None
        if code != 0:
            raise RuntimeError(f"xlg_create -> {code} (no CPU fallback)")
        self._h = h
        self.flags = flags
        self.fs = sampling_freq

    def add_client(self, decimation: int, taps, center_freq: int, state=None) -> int:
        """state: an XlgClientState for a client that continues a stream it consumed elsewhere
        (xlg_add_client_ex); None for a fresh client."""
        taps = np.ascontiguousarray(taps, dtype=np.float32)
        cid = C.c_int(-1)
        fp = taps.ctypes.data_as(C.POINTER(C.c_float))
        if state is None:
            code = self._L.xlg_add_client(self._h, decimation, fp, len(taps), center_freq, C.byref(cid))
        else:
            code = self._L.xlg_add_client_ex(self._h, decimation, fp, len(taps), center_freq, C.byref(state),
                                             C.byref(cid))
        if code != 0:
            raise ValueError(code)
        return cid.value

    def add_client_rational(self, interp: int, decim: int, taps, center_freq: int, state=None) -> int:
        """A client at fs * interp / decim: the reference filter at interp * fs fed the zero-stuffed
        stream (include/xlating_group.h, xlg_add_client_rational).  state: an XlgClientState (hist in
        upsampled samples, valid_history in input samples) for a client that continues a stream it
        consumed elsewhere (xlg_add_client_rational_ex); None for a fresh client."""
        taps = np.ascontiguousarray(taps, dtype=np.float32)
        cid = C.c_int(-1)
        fp = taps.ctypes.data_as(C.POINTER(C.c_float))
        if state is None:
            code = self._L.xlg_add_client_rational(self._h, interp, decim, fp, len(taps), center_freq, C.byref(cid))
        else:
            code = self._L.xlg_add_client_rational_ex(self._h, interp, decim, fp, len(taps), center_freq,
                                                      C.byref(state), C.byref(cid))
        if code != 0:
            raise ValueError(code)
        return cid.value

    def add_client_cascade(self, decim1: int, taps1, center_freq: int, decim2: int, taps2, interp2: int = 1) -> int:
        """A two-stage client (include/xlating_group.h, xlg_add_client_cascade_rational): the reference filter
        (decim1, taps1, center_freq) at fs, followed by the reference filter (decim2, taps2, centre 0) at
        interp2 * fs / decim1 fed its zero-stuffed outputs (interp2 = 1: xlg_add_client_cascade).  See
        cascade_plan for taps."""
        t1 = np.ascontiguousarray(taps1, dtype=np.float32)
        t2 = np.ascontiguousarray(taps2, dtype=np.float32)
        cid = C.c_int(-1)
        fp = C.POINTER(C.c_float)
        code = self._L.xlg_add_client_cascade_rational(self._h, decim1, t1.ctypes.data_as(fp), len(t1), center_freq,
                                                       interp2, decim2, t2.ctypes.data_as(fp), len(t2), C.byref(cid))
        if code != 0:
            raise ValueError(code)
        return cid.value

    def cascade_info(self, cid: int):
        """(stage-A kernel kind, stage-A history, stage-B history in stage-A samples) of a cascade client."""
        kind, h1, h2 = C.c_int(0), C.c_size_t(0), C.c_size_t(0)
        code = self._L.xlg_cascade_info(self._h, cid, C.byref(kind), C.byref(h1), C.byref(h2))
        if code != 0:
            raise ValueError(code)
        return kind.value, h1.value, h2.value

    def add_subband(self, decim1: int, taps1, center_freq: int) -> int:
        """A sub-band (include/xlating_group.h, xlg_add_subband): the reference filter (decim1, taps1,
        center_freq) at fs, shared by its members and invisible to the caller.  Returns a sub-band id."""
        t1 = np.ascontiguousarray(taps1, dtype=np.float32)
        sid = C.c_int(-1)
        code = self._L.xlg_add_subband(self._h, decim1, t1.ctypes.data_as(C.POINTER(C.c_float)), len(t1),
                                       center_freq, C.byref(sid))
        if code != 0:
            raise ValueError(code)
        return sid.value

    def remove_subband(self, sid: int) -> None:
        code = self._L.xlg_remove_subband(self._h, sid)
        if code != 0:
            raise ValueError(code)

    def add_client_subband(self, sid: int, decim2: int, taps2, center_offset: int, interp2: int = 1) -> int:
        """A member of sub-band `sid` (xlg_add_client_subband_rational): the reference's float path (decim2,
        taps2, center_offset) at interp2 * fs / decim1 fed the sub-band's zero-stuffed outputs (interp2 = 1:
        xlg_add_client_subband).  Returns an ordinary client id.  See subband_plan for taps."""
        t2 = np.ascontiguousarray(taps2, dtype=np.float32)
        cid = C.c_int(-1)
        code = self._L.xlg_add_client_subband_rational(self._h, sid, interp2, decim2,
                                                       t2.ctypes.data_as(C.POINTER(C.c_float)), len(t2),
                                                       center_offset, C.byref(cid))
        if code != 0:
            raise ValueError(code)
        return cid.value

    def subband_info(self, cid: int):
        """(sub-band id, kind of the kernel serving the sub-band, member history in sub-band samples)."""
        sid, kind, h = C.c_int(0), C.c_int(0), C.c_size_t(0)
        code = self._L.xlg_subband_info(self._h, cid, C.byref(sid), C.byref(kind), C.byref(h))
        if code != 0:
            raise ValueError(code)
        return sid.value, kind.value, h.value

    def add_bank(self, decim1: int, taps1) -> int:
        """A channel bank (include/xlating_group.h, xlg_add_bank): K = 2 * decim1 channels k * fs / K apart,
        each the sub-band (decim1, taps1) centred there, from one polyphase pass.  Returns a bank id."""
        t1 = np.ascontiguousarray(taps1, dtype=np.float32)
        bid = C.c_int(-1)
        code = self._L.xlg_add_bank(self._h, decim1, t1.ctypes.data_as(C.POINTER(C.c_float)), len(t1), C.byref(bid))
        if code != 0:
            raise ValueError(code)
        return bid.value

    def add_bank_fft(self, decim1: int, taps1, *, any_k: bool = False) -> int:
        """An FFT bank (xlg_add_bank_fft): add_bank's channels, cut by a K-point FFT per frame instead of a direct
        sum per channel (K = 2 * decim1 a power of two up to 4096; bank_fft_fits bounds taps1).  any_k=True takes
        every even K up to 4096 (xlg_add_bank_any; bank_any_fits bounds taps1): the K above are served as without
        it, every other K by the chirp-z stage.  Returns a bank id from add_bank's id space."""
        t1 = np.ascontiguousarray(taps1, dtype=np.float32)
        bid = C.c_int(-1)
        add = self._L.xlg_add_bank_any if any_k else self._L.xlg_add_bank_fft
        code = add(self._h, decim1, t1.ctypes.data_as(C.POINTER(C.c_float)), len(t1), C.byref(bid))
        if code != 0:
            raise ValueError(code)
        return bid.value

    def add_bank_subband(self, bid: int, channel: int) -> int:
        """Channel `channel` in [-decim1, decim1) of bank `bid` (xlg_add_bank_subband): an ordinary sub-band id,
        centred at channel * fs / (2 * decim1), that takes members through add_client_subband."""
        sid = C.c_int(-1)
        code = self._L.xlg_add_bank_subband(self._h, bid, channel, C.byref(sid))
        if code != 0:
            raise ValueError(code)
        return sid.value

    def remove_bank(self, bid: int) -> None:
        code = self._L.xlg_remove_bank(self._h, bid)
        if code != 0:
            raise ValueError(code)

    def _add_spectrum_ex(self, source, source_id, width, frames_per_row, skip, power, hop, window, mean,
                         any_width=False):
        """xlg_add_spectrum_ex, or xlg_add_spectrum_any with any_width (hop None: width; window: `width` weights
        or None; mean: the mean of the row's frames instead of their max)."""
        w = None
        if window is not None:
            w = np.ascontiguousarray(window, np.float32)
            if w.shape != (width,):
                raise ValueError(f"window of shape {w.shape}, width {width}")
        desc = XlgSpectrumDesc(width, frames_per_row, skip, XLG_SPECTRUM_POWER if power else 0,
                               0 if hop is None else hop, 1 if mean else 0,
                               None if w is None else w.ctypes.data_as(C.POINTER(C.c_float)))
        sid = C.c_int(-1)
        add = self._L.xlg_add_spectrum_any if any_width else self._L.xlg_add_spectrum_ex
        code = add(self._h, source, source_id, C.byref(desc), C.byref(sid))
        if code != 0:
            raise ValueError(code)
        return sid.value

    def add_spectrum(self, width: int, frames_per_row: int, skip: int = 0, power: bool = False,
                     hop=None, window=None, mean: bool = False, *, any_width: bool = False) -> int:
        """A spectrum (xlg_add_spectrum) attached before the next submitted block: rows of the max-held power of
        `frames_per_row` consecutive `width`-point DFT frames, `skip` samples skipped after each row, half swapped
        as the reference's spectrogram; dB rows, or linear power with power=True.  spectrogram_params(fs, width)
        gives the reference tool's frames_per_row and skip.  Returns a spectrum id.
        `width` is 1 to 4096, or a power of two from 8192 to 65536 (the wide FFT, the same rows as an FFT at K = width).
        With `hop` (samples between frame starts in a row), `window` (`width` float weights) or mean=True (the
        mean of the frames' powers instead of their max) it is a Welch spectrum (xlg_add_spectrum_ex).
        any_width=True takes every width from 1 to 65536 (xlg_add_spectrum_any): the widths above are served
        exactly as without it, every other one by the chirp-z stage (spectrum_info kernel 3)."""
        if any_width or hop is not None or window is not None or mean:
            return self._add_spectrum_ex(0, 0, width, frames_per_row, skip, power, hop, window, mean, any_width)
        sid = C.c_int(-1)
        code = self._L.xlg_add_spectrum(self._h, width, frames_per_row, skip, XLG_SPECTRUM_POWER if power else 0,
                                        C.byref(sid))
        if code != 0:
            raise ValueError(code)
        return sid.value

    def add_client_spectrum(self, cid: int, width: int, frames_per_row: int, skip: int = 0,
                            power: bool = False, hop=None, window=None, mean: bool = False, *,
                            any_width: bool = False) -> int:
        """A spectrum of client `cid`'s output stream (xlg_add_client_spectrum): add_spectrum's rows of what
        output() returns for it from the next submitted block on (a cascade client's final row).
        spectrogram_params(client_rate, width) gives the reference tool's parameters for the client's file.
        width (1 to 4096, or a power of two from 8192 to 65536), hop, window, mean and any_width as for
        add_spectrum."""
        if any_width or hop is not None or window is not None or mean:
            return self._add_spectrum_ex(1, cid, width, frames_per_row, skip, power, hop, window, mean, any_width)
        sid = C.c_int(-1)
        code = self._L.xlg_add_client_spectrum(self._h, cid, width, frames_per_row, skip,
                                               XLG_SPECTRUM_POWER if power else 0, C.byref(sid))
        if code != 0:
            raise ValueError(code)
        return sid.value

    def add_subband_spectrum(self, sbid: int, width: int, frames_per_row: int, skip: int = 0,
                             power: bool = False, hop=None, window=None, mean: bool = False, *,
                             any_width: bool = False) -> int:
        """A spectrum of sub-band (or bank channel) `sbid`'s rows at fs / decim1 (xlg_add_subband_spectrum),
        from the next submitted block on: a zoomed waterfall of the sub-band.  width (1 to 4096, or a power of
        two from 8192 to 65536), hop, window, mean and any_width as for add_spectrum."""
        if any_width or hop is not None or window is not None or mean:
            return self._add_spectrum_ex(2, sbid, width, frames_per_row, skip, power, hop, window, mean, any_width)
        sid = C.c_int(-1)
        code = self._L.xlg_add_subband_spectrum(self._h, sbid, width, frames_per_row, skip,
                                                XLG_SPECTRUM_POWER if power else 0, C.byref(sid))
        if code != 0:
            raise ValueError(code)
        return sid.value

    def remove_spectrum(self, sid: int) -> None:
        code = self._L.xlg_remove_spectrum(self._h, sid)
        if code != 0:
            raise ValueError(code)

    def spectrum_rows(self, ticket: int, sid: int) -> int:
        """Rows spectrum `sid` completed in `ticket` (known when submit returns)."""
        n = C.c_size_t(0)
        code = self._L.xlg_spectrum_output(self._h, ticket, sid, None, C.byref(n))
        if code != 0:
            raise ValueError(code)
        return n.value

    def spectrum_width(self, ticket: int, sid: int) -> int:
        """The width of the rows spectrum `sid` completed in `ticket`: the one the id had when the ticket was
        submitted (xlg_spectrum_width)."""
        w = C.c_uint32(0)
        code = self._L.xlg_spectrum_width(self._h, ticket, sid, C.byref(w))
        if code != 0:
            raise ValueError(code)
        return w.value

    def read_spectrum(self, ticket: int, sid: int) -> np.ndarray:
        """The rows spectrum `sid` completed in `ticket`, a (rows, width) float32 array of the width the ticket's
        rows were made with (xlg_read_spectrum; waits for the ticket)."""
        n = self.spectrum_rows(ticket, sid)
        buf = np.zeros((n, self.spectrum_width(ticket, sid)), np.float32)
        got = C.c_size_t(0)
        code = self._L.xlg_read_spectrum(self._h, ticket, sid, buf.ctypes.data_as(C.POINTER(C.c_float)), n,
                                         C.byref(got))
        if code != 0:
            raise ValueError(code)
        assert got.value == n
        return buf

    def spectrum_info(self, sid: int):
        """(kernel: 0 direct DFT, 1 FFT, 2 wide FFT (width above 4096), 3 chirp-z (any_width, above 4096 and not
        a power of two), rows completed by the blocks submitted so far)."""
        kind, rows = C.c_int(-1), C.c_uint64(0)
        code = self._L.xlg_spectrum_info(self._h, sid, C.byref(kind), C.byref(rows))
        if code != 0:
            raise ValueError(code)
        return kind.value, rows.value

    def remove_client(self, cid: int) -> None:
        code = self._L.xlg_remove_client(self._h, cid)
        if code != 0:
            raise ValueError(code)

    def reserve(self, output_samples_per_block: int) -> None:
        code = self._L.xlg_reserve(self._h, output_samples_per_block)
        if code != 0:
            raise RuntimeError(f"xlg_reserve -> {code}")

    def client_count(self) -> int:
        return self._L.xlg_client_count(self._h)

    def client_info(self, cid: int):
        hist = C.c_size_t(0)
        kind = C.c_int(0)
        code = self._L.xlg_client_info(self._h, cid, C.byref(hist), C.byref(kind))
        if code != 0:
            raise ValueError(code)
        return hist.value, kind.value

    def submit(self, fmt: str, data, flags: int = 0) -> int:
        """data: numpy array (host) -- or (device_ptr, n_elements) with XLG_INPUT_DEVICE.  cf32 takes float32
        (re, im) pairs or complex64, and also a CUDA torch.complex64 tensor, submitted in place through
        XLG_INPUT_DEVICE."""
        if fmt == "cf32" and getattr(data, "is_cuda", False):
            assert str(data.dtype) == "torch.complex64" and data.is_contiguous(), data.dtype
            ptr, n, flags = data.data_ptr(), 2 * data.numel(), flags | XLG_INPUT_DEVICE
        elif flags & XLG_INPUT_DEVICE:
            ptr, n = data
        elif fmt == "cf32" and np.iscomplexobj(data):
            data = np.ascontiguousarray(data, dtype=np.complex64).view(np.float32)
            ptr, n = data.ctypes.data, data.size
        else:
            data = np.ascontiguousarray(data, dtype=NP_DTYPE[fmt])
            ptr, n = data.ctypes.data, data.size
        t = self._L.xlg_submit(self._h, FMT[fmt], ptr, n, flags)
        if t < 0:
            raise RuntimeError(f"xlg_submit -> {t}")
        return t

    def submit_ptr(self, fmt_code: int, ptr: int, n: int, flags: int = 0) -> int:
        """Submit n raw elements at address ptr: page-locked host memory (a PinnedBuffer's ptr, or a pinned torch
        tensor's data_ptr(), plus any byte offset) or, with XLG_INPUT_DEVICE, device memory."""
        t = self._L.xlg_submit(self._h, fmt_code, ptr, n, flags)
        if t < 0:
            raise RuntimeError(f"xlg_submit -> {t}")
        return t

    def input_consumed(self, ticket: int) -> None:
        """xlg_input_consumed: returns once the group has read the ticket's input block."""
        code = self._L.xlg_input_consumed(self._h, ticket)
        if code != 0:
            raise RuntimeError(f"xlg_input_consumed -> {code}")

    def wait(self, ticket: int) -> None:
        code = self._L.xlg_wait(self._h, ticket)
        if code != 0:
            raise RuntimeError(f"xlg_wait -> {code}")

    def output_ptr(self, ticket: int, cid: int):
        out = C.c_void_p()
        n = C.c_size_t(0)
        code = self._L.xlg_output(self._h, ticket, cid, C.byref(out), C.byref(n))
        if code != 0:
            raise RuntimeError(f"xlg_output -> {code}")
        return out.value, n.value

    def output(self, ticket: int, cid: int, q15: bool = False) -> np.ndarray:
        """Host copy of one client's output (host-output groups only)."""
        assert not (self.flags & XLG_OUT_DEVICE)
        ptr, n = self.output_ptr(ticket, cid)
        if q15:
            if n == 0:
                return np.zeros((0, 2), dtype=np.int16)
            return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_int16)), shape=(2 * n,)).copy().reshape(-1, 2)
        if n == 0:
            return np.zeros(0, dtype=np.complex64)
        return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(C.c_float)), shape=(2 * n,)).copy().view(np.complex64)

    def read_output(self, ticket: int, cid: int, q15: bool = False) -> np.ndarray:
        """Copy of one client's output wherever it lives (HBM for XLG_OUT_DEVICE groups)."""
        _, n = self.output_ptr(ticket, cid)
        buf = np.zeros((n, 2), dtype=np.int16) if q15 else np.zeros(n, dtype=np.complex64)
        got = C.c_size_t(0)
        code = self._L.xlg_read_output(self._h, ticket, cid, buf.ctypes.data, n, C.byref(got))
        if code != 0:
            raise RuntimeError(f"xlg_read_output -> {code}")
        assert got.value == n
        return buf

    def copy_output(self, ticket: int, cid: int):
        """xlg_copy_output of a completed ticket with its state_after (XLG_TRACK_STATE groups): (cf32 output,
        XlgClientState after the ticket).  Raises ValueError(code) on a nonzero return."""
        st, n = XlgClientState(), C.c_size_t(0)

        def copy(buf):
            code = self._L.xlg_copy_output(self._h, ticket, cid, buf.ctypes.data, buf.size, C.byref(n), C.byref(st))
            if code != 0:
                raise ValueError(code)
            return buf

        buf = copy(np.zeros(1, dtype=np.complex64))  # reports the count
        if n.value > buf.size:
            buf = copy(np.zeros(n.value, dtype=np.complex64))
        return buf[:n.value].copy(), st

    def wait_stream(self, cuda_stream: int) -> None:
        code = self._L.xlg_wait_stream(self._h, cuda_stream)
        if code != 0:
            raise RuntimeError(f"xlg_wait_stream -> {code}")

    def partition_sms(self) -> int:
        """SMs currently reserved for the oscillator pre-pass (0 = no partition active for this layout)."""
        return int(self._L.xlg_partition_active(self._h))

    def timer_start(self) -> None:
        code = self._L.xlg_timer_start(self._h)
        if code != 0:
            raise RuntimeError(f"xlg_timer_start -> {code}")

    def timer_stop(self) -> float:
        ms = C.c_float(0)
        code = self._L.xlg_timer_stop(self._h, C.byref(ms))
        if code != 0:
            raise RuntimeError(f"xlg_timer_stop -> {code}")
        return ms.value

    def profile_enable(self, on: bool) -> None:
        self._L.xlg_profile_enable(self._h, 1 if on else 0)

    def profile_read(self, reset: bool = True) -> dict:
        p = XlgProfile()
        self._L.xlg_profile_read(self._h, C.byref(p), 1 if reset else 0)
        return {k: getattr(p, k) for k, _ in XlgProfile._fields_}

    def poly_profile_read(self, reset: bool = True) -> dict:
        p = XlgPolyProfile()
        self._L.xlg_poly_profile_read(self._h, C.byref(p), 1 if reset else 0)
        return {k: getattr(p, k) for k, _ in XlgPolyProfile._fields_}

    def cascade_profile_read(self, reset: bool = True) -> dict:
        p = XlgCascadeProfile()
        self._L.xlg_cascade_profile_read(self._h, C.byref(p), 1 if reset else 0)
        return {k: getattr(p, k) for k, _ in XlgCascadeProfile._fields_}

    def subband_profile_read(self, reset: bool = True) -> dict:
        p = XlgSubbandProfile()
        self._L.xlg_subband_profile_read(self._h, C.byref(p), 1 if reset else 0)
        return {k: getattr(p, k) for k, _ in XlgSubbandProfile._fields_}

    def bank_profile_read(self, reset: bool = True) -> dict:
        p = XlgBankProfile()
        self._L.xlg_bank_profile_read(self._h, C.byref(p), 1 if reset else 0)
        return {k: getattr(p, k) for k, _ in XlgBankProfile._fields_}

    def bank_fft_profile_read(self, reset: bool = True) -> dict:
        p = XlgBankFftProfile()
        self._L.xlg_bank_fft_profile_read(self._h, C.byref(p), 1 if reset else 0)
        return {k: getattr(p, k) for k, _ in XlgBankFftProfile._fields_}

    def spectrum_profile_read(self, reset: bool = True) -> dict:
        p = XlgSpectrumProfile()
        self._L.xlg_spectrum_profile_read(self._h, C.byref(p), 1 if reset else 0)
        return {k: getattr(p, k) for k, _ in XlgSpectrumProfile._fields_}

    def close(self):
        if self._h:
            self._L.xlg_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class PinnedBuffer:
    """Page-locked host memory from the library (queue/ingest blocks)."""

    def __init__(self, nbytes: int):
        self._L = lib()
        self.ptr = self._L.xlg_alloc_pinned(nbytes)
        if not self.ptr:
            raise MemoryError("xlg_alloc_pinned failed")
        self.nbytes = nbytes

    def array(self, dtype=np.uint8) -> np.ndarray:
        n = self.nbytes // np.dtype(dtype).itemsize
        return np.ctypeslib.as_array(C.cast(self.ptr, C.POINTER(C.c_uint8)), shape=(self.nbytes,)).view(dtype)[:n]

    def free(self):
        if self.ptr:
            self._L.xlg_free_pinned(self.ptr)
            self.ptr = None

    def __del__(self):
        try:
            self.free()
        except Exception:
            pass


# ---------------------------------------------------------------------------
# workload helpers shared by tests and bench.py (SURVEY.md section 8d)
# ---------------------------------------------------------------------------
def client_plan(fs: int, rates, tw=None):
    """Centre offsets and decimations for C clients spread across the band:
    client c: center = round(-fs/2 + rate/2 + c*(fs-rate)/(C-1))."""
    C_ = len(rates)
    plan = []
    for c, rate in enumerate(rates):
        if C_ > 1:
            center = int(round(-fs / 2 + rate / 2 + c * (fs - rate) / (C_ - 1)))
        else:
            center = -312000 if fs > 700000 else -fs // 4
        plan.append({"rate": rate, "decimation": fs // rate, "center": center,
                     "cutoff": rate // 2, "tw": tw if tw is not None else rate // 5})
    return plan


def poly_pack(rev, interp: int) -> np.ndarray:
    """The library's polyphase packer (csrc/taps_host.c): reversed complex taps -> branch-major
    (interp, ceil(T / interp)) complex64 array, zero-padded."""
    rev = np.ascontiguousarray(rev, dtype=np.complex64)
    T = rev.size
    Tb = -(-T // interp)
    out = np.zeros(interp * Tb, dtype=np.complex64)
    fp = C.POINTER(C.c_float)
    lib().xl_poly_pack(rev.ctypes.data_as(fp), T, interp, out.ctypes.data_as(fp))
    return out.reshape(interp, Tb)


def rational_plan(fs: int, rates, lpf_cutoff_rate: int = 5):
    """Clients at any rate: rate / fs reduced to interp / decim, taps designed at interp * fs with gain
    interp (so every polyphase branch has unit DC gain), cutoff rate / 2 and transition width
    rate / lpf_cutoff_rate.  Centres as client_plan places them."""
    plan = []
    for p, rate in zip(client_plan(fs, rates), rates):
        g = math.gcd(int(rate), int(fs))
        L, M = int(rate) // g, int(fs) // g
        taps = create_low_pass_filter(float(L), L * fs, int(rate) // 2, int(rate) // lpf_cutoff_rate)
        plan.append({"rate": rate, "interp": L, "decim": M, "center": p["center"], "taps": taps})
    return plan


def cascade_fmas(fs: int, rate: int, d1: int, t1: int, t2: int, interp2: int = 1) -> float:
    """Algorithmic real FMAs per input sample of a cascade client: 4 per complex tap of stage A at fs / d1,
    2 per real tap of stage B's polyphase branch (ceil(t2 / interp2) taps) at the client rate."""
    return 4.0 * t1 / d1 + 2.0 * -(-t2 // interp2) / (fs / rate)


def cascade_stages(fs: int, rate: int, d1: int):
    """Taps of the two stages for D1 = d1: stage B is the server's own design at fs1 = fs / d1 (cutoff
    rate / 2, transition rate / 5); stage A passes up to e = 3 * rate / 5 (stage B's passband edge plus half
    its transition) and stops from fs1 - e, so everything it aliases onto the band lands in stage B's
    stopband: create_low_pass_filter(1, fs, fs1 / 2, fs1 - 2e).  Where rate does not divide fs1, stage B
    resamples by L2 / M2 = rate / fs1 (reduced): its taps are designed at L2 * fs1 with gain L2, so that every
    polyphase branch has unit gain (L2 = 1 is the design above)."""
    fs1 = fs // d1
    e = 3 * rate // 5
    L2 = rate // math.gcd(rate, fs1)
    return (create_low_pass_filter(1.0, fs, fs1 // 2, fs1 - 2 * e),
            create_low_pass_filter(float(L2), L2 * fs1, rate // 2, rate // 5))


def cascade_plan(fs: int, rates):
    """Two-stage clients.  For a rate that divides fs, D = fs / rate: the divisor D1 >= 2 of D (with
    D2 = D / D1 >= 2).  For any other rate: a divisor D1 >= 2 of fs with fs1 = fs / D1 > 2e (e = 3 * rate / 5,
    cascade_stages) and fs1 > rate, and a rational stage B L2 / M2 = rate / fs1 reduced.  Of these, the one
    with the fewest estimated FMAs per input sample, 4*T1/D1 + 2*ceil(T2/L2)*rate/fs (cascade_fmas; ties go to
    the smaller D1).  Taps from cascade_stages; centres as client_plan places them."""
    plan = []
    for p, rate in zip(client_plan(fs, rates), rates):
        rate = int(rate)
        if fs % rate == 0:
            D = fs // rate
            cands = [d1 for d1 in range(2, D // 2 + 1) if D % d1 == 0]
        else:
            e = 3 * rate // 5
            cands = [d1 for d1 in range(2, fs // rate + 1) if fs // d1 > 2 * e and fs // d1 > rate]
        best = None
        for d1 in cands:
            if fs % d1 != 0:
                continue
            fs1 = fs // d1
            g = math.gcd(rate, fs1)
            L2, M2 = rate // g, fs1 // g
            t1, t2 = cascade_stages(fs, rate, d1)
            cost = cascade_fmas(fs, rate, d1, t1.size, t2.size, L2)
            if best is None or cost < best[0]:
                best = (cost, d1, L2, M2, t1, t2)
        if best is None:
            raise ValueError(f"{fs} has no divisor D1 >= 2 to split a {rate} Hz client into two stages")
        cost, d1, L2, M2, t1, t2 = best
        plan.append({"rate": rate, "d1": d1, "interp2": L2, "d2": M2, "center": p["center"], "taps1": t1,
                     "taps2": t2, "fmas": cost})
    return plan


def subband_fmas(fs: int, d1: int, t1: int, n_subbands: int, members) -> float:
    """Algorithmic real FMAs per input sample of a sub-band plan: 4 per complex tap of each sub-band at
    fs / d1, and 4 per complex tap of each member's polyphase branch (ceil(t2 / interp2) taps) at its own rate.
    members: (rate, t2) or (rate, t2, interp2) tuples."""
    return 4.0 * n_subbands * t1 / d1 + sum(4.0 * -(-m[1] // (m[2] if len(m) > 2 else 1)) * m[0] / fs
                                           for m in members)


def subband_member_fits(interp2: int, decim2: int, t2: int) -> bool:
    """Whether the member kernel's shared memory holds a member (xlg_add_client_subband_rational refuses the
    others): 16 members' taps of one branch and the window of 64 outputs, subband_smem in csrc/xlating_kernels.cuh
    against the 200 KiB the kernel is given."""
    return (16 + 16 * 8 * ((-(-t2 // interp2) + 1) & ~1) + 8 * ((63 * decim2 - (-t2 // interp2) + 2) & ~1)
            <= 200 * 1024)


def bank_fits(d1: int, t1: int) -> bool:
    """Whether the bank kernel's shared memory holds a bank (xlg_add_bank refuses the others): the taps padded
    to a multiple of K = 2 * d1 and of 4, the window of 32 frames, K twiddles and 32 rows of K + 1 polyphase
    sums, bank_smem in csrc/xlating_kernels.cuh against the 200 KiB the kernel is given."""
    K = 2 * d1
    tpad = ((-(-t1 // K) * K) + 3) & ~3
    return 16 + 4 * tpad + 8 * ((31 * d1 + t1 + 2) & ~1) + 8 * K + 8 * 32 * (K + 1) <= 200 * 1024


def bank_fft_fits(d1: int, t1: int) -> bool:
    """Whether the FFT bank kernel takes a bank (xlg_add_bank_fft refuses the others): K = 2 * d1 a power of two
    up to 4096 and at most max(16 * K, 16384) taps, bank_fft_max_taps in csrc/xlating_kernels.cuh."""
    K = 2 * d1
    return d1 >= 1 and K & (K - 1) == 0 and K <= 4096 and 1 <= t1 <= max(16 * K, 16384)


def bank_fft_flops(K: int) -> int:
    """Real FP32 instructions of the butterflies of one K-point FFT bank frame (xlg_bank_fft_flops)."""
    return int(lib().xlg_bank_fft_flops(K))


def bank_any_fits(d1: int, t1: int) -> bool:
    """Whether xlg_add_bank_any takes a bank on the kernel's side (fs % K is the group's check): K = 2 * d1 at
    most 4096 and at most max(16 * K, 16384) taps, bank_fft_max_taps in csrc/xlating_kernels.cuh."""
    K = 2 * d1
    return d1 >= 1 and K <= 4096 and 1 <= t1 <= max(16 * K, 16384)


def bank_any_m(K: int) -> int:
    """M = next_pow2(2K - 1), the chirp-z bank stage's transform length."""
    return 1 << (2 * K - 2).bit_length()


def bank_any_flops(K: int, channels: int) -> int:
    """Real FP32 instructions of one chirp-z bank frame's channel stage with `channels` materialised channels:
    2 * bank_fft_flops(M) + 4 K + 4 M + 4 C (xlg_bank_fft_profile's butterfly_flops)."""
    M = bank_any_m(K)
    return 2 * bank_fft_flops(M) + 4 * K + 4 * M + 4 * channels


def bank_any_tables(K: int):
    """The chirp-z bank stage's tables for K (even, at most 4096, not a power of two), as the library builds
    them (xlg_bank_any_tables): (chirp: complex64[K], kernel: complex64[M] in the transform's position order, M).
    ValueError for any other K."""
    L = lib()
    m = C.c_uint32(0)
    code = L.xlg_bank_any_tables(K, None, None, C.byref(m))
    if code != 0:
        raise ValueError(code)
    chirp, kern = np.zeros(K, np.complex64), np.zeros(m.value, np.complex64)
    fp = C.POINTER(C.c_float)
    code = L.xlg_bank_any_tables(K, chirp.ctypes.data_as(fp), kern.ctypes.data_as(fp), C.byref(m))
    if code != 0:
        raise ValueError(code)
    return chirp, kern, m.value


def spectrum_any_tables(width: int):
    """The chirp-z stage's tables for `width` (above 4096, at most 65536, not a power of two), as the library
    builds them (xlg_spectrum_any_tables): (chirp: complex64[width], kernel: complex64[M] in the transform's
    position order, M).  ValueError for any other width."""
    L = lib()
    m = C.c_uint32(0)
    code = L.xlg_spectrum_any_tables(width, None, None, C.byref(m))
    if code != 0:
        raise ValueError(code)
    chirp, kern = np.zeros(width, np.complex64), np.zeros(m.value, np.complex64)
    fp = C.POINTER(C.c_float)
    code = L.xlg_spectrum_any_tables(width, chirp.ctypes.data_as(fp), kern.ctypes.data_as(fp), C.byref(m))
    if code != 0:
        raise ValueError(code)
    return chirp, kern, m.value


def spectrogram_params(fs: int, width: int):
    """(frames_per_row, skip) of the reference spectrogram tool at sampling rate fs and width W: one row per fs
    samples, (fs // W, fs % W).  ValueError where the tool refuses: W or fs not positive, W > fs."""
    if width <= 0 or fs <= 0:
        raise ValueError(f"width {width} and sampling rate {fs} must be positive")
    if width > fs:
        raise ValueError(f"width {width} is too wide for sampling rate {fs}")
    return fs // width, fs % width


def spectrogram_pixels(rows) -> np.ndarray:
    """8-bit grey pixels of dB rows, as the reference's png_util_set_data: (int)(dB + 255), truncated toward
    zero, clamped to [0, 255]."""
    v = np.asarray(rows, np.float32) + np.float32(255)
    return np.clip(np.trunc(v), 0, 255).astype(np.uint8)


def subband_plan(fs: int, clients, bank: bool = False, fft: bool = False, any_k: bool = False):
    """Sub-band clients for `clients`, a list of (center, rate).  For every D1 >= 2 that divides fs with
    fs1 = fs / D1 even, fs1 > 2 * max rate and every rate dividing fs1: sub-band centres fs1 / 2 apart from
    the lowest client centre up across the occupied span, each client assigned to the nearest one (so its
    offset |c2| <= fs1 / 4), the sub-bands designed with create_low_pass_filter(1, fs, fs1 / 2, fs1 - 2e),
    e = fs1 / 4 + max rate / 2 (it passes everything a member reads, and everything it aliases lands outside
    [-e, e]), the members with the server's own taps at fs1 (cutoff rate / 2, transition rate / 5).  Of
    these, the D1 with the fewest FMAs per input sample (subband_fmas, counting only sub-bands with members;
    ties go to the smaller D1).  Only where no D1 lets every rate divide fs1, every D1 with fs1 even and
    fs1 > 2 * max rate is a candidate: each member then resamples by interp2 / d2 = rate / fs1 (reduced;
    interp2 = 1 where the rate divides fs1) with taps create_low_pass_filter(interp2, interp2 * fs1, rate / 2,
    rate / 5), and a D1 with a member the kernel would refuse (subband_member_fits) is skipped.  Returns
    {"d1", "taps1", "e", "subbands": [{"center"}], "members": [{"subband", "center", "rate", "interp2", "d2",
    "offset", "taps2"}] in the order of `clients`, "fmas"}.

    bank=True plans the sub-bands as channels of one bank (Group.add_bank, add_bank_subband): each client is
    assigned to the nearest centre j * fs1 / 2 of the bank's grid (|offset| <= fs1 / 4 still), every sub-band
    entry also carries its "channel" k in [-D1, D1) (j wrapped: the channel at +fs / 2 is the one at -fs / 2,
    and a member's offset stays relative to its own grid point), a D1 whose bank the kernel would refuse (bank_fits) is skipped, and the first stage costs
    2 * T1 / D1 + 8 * C FMAs per input sample (one polyphase pass, C channel sums of K complex MACs per frame)
    instead of 4 * T1 / D1 per sub-band.

    fft=True (with bank=True) also considers FFT banks (Group.add_bank_fft) where bank_fft_fits: their channel
    stage costs bank_fft_flops(K) / D1 per input sample instead of 8 * C.  At each D1 the cheaper kernel is
    taken (the direct one on a tie), and the plan carries "kernel": "direct" or "fft".

    any_k=True (with fft=True) also considers chirp-z banks (Group.add_bank_fft(..., any_k=True)) at every D1
    whose K = 2 * D1 is not a power of two, where bank_any_fits: their channel stage costs bank_any_flops(K, C) / D1
    per input sample, and "kernel" is "czt" where one is taken (ties keep the earlier kernel)."""
    if fft and not bank:
        raise ValueError("fft=True plans banks: it needs bank=True")
    if any_k and not fft:
        raise ValueError("any_k=True plans chirp-z banks: it needs fft=True")
    centers = [int(c) for c, _ in clients]
    rates = [int(r) for _, r in clients]
    rmax = max(rates)
    lo, hi = min(centers), max(centers)
    best = None
    for rational in (False, True):
        for d1 in range(2, fs // (2 * rmax) + 1):
            if fs % d1:
                continue
            fs1 = fs // d1
            if fs1 % 2 or fs1 <= 2 * rmax or (not rational and any(fs1 % r for r in rates)):
                continue
            shapes = {}  # rate -> (interp2, d2, taps2)
            for r in set(rates):
                g = math.gcd(r, fs1)
                L2, M2 = r // g, fs1 // g
                shapes[r] = (L2, M2, create_low_pass_filter(float(L2), L2 * fs1, r // 2, r // 5))
            if rational and not all(subband_member_fits(L2, M2, t.size) for L2, M2, t in shapes.values()):
                continue
            half = fs1 // 2
            e = fs1 // 4 + rmax // 2
            t1 = create_low_pass_filter(1.0, fs, fs1 // 2, fs1 - 2 * e)
            kernel = None
            if bank:
                base = 0  # the grid j * half, j = round(c / half), and j's channel
                grid = [(2 * c + half) // (2 * half) for c in centers]
                assign = [(j + d1) % (2 * d1) - d1 for j in grid]
                used = sorted(set(assign))
                stages = [(8.0 * len(used), "direct")] if bank_fits(d1, t1.size) else []
                if fft and bank_fft_fits(d1, t1.size):
                    stages.append((bank_fft_flops(2 * d1) / d1, "fft"))
                elif any_k and bank_any_fits(d1, t1.size):
                    stages.append((bank_any_flops(2 * d1, len(used)) / d1, "czt"))
                if not stages:
                    continue
                stage, kernel = min(stages, key=lambda c: c[0])  # (a tie keeps the direct bank)
                cost = 2.0 * t1.size / d1 + stage + subband_fmas(
                    fs, d1, t1.size, 0, [(r, shapes[r][2].size, shapes[r][0]) for r in rates])
            else:
                base = lo
                grid = None
                n_cent = (hi - lo + half - 1) // half + 1
                assign = [min(range(n_cent), key=lambda k: abs(c - (lo + k * half))) for c in centers]
                used = sorted(set(assign))
                cost = subband_fmas(fs, d1, t1.size, len(used), [(r, shapes[r][2].size, shapes[r][0]) for r in rates])
            if best is None or cost < best[0]:
                best = (cost, d1, fs1, half, e, t1, shapes, used, assign, base, grid, kernel)
        if best is not None:
            break
    if best is None:
        raise ValueError(f"{fs} has no divisor D1 >= 2 whose sub-band rate serves the rates {sorted(set(rates))}")
    cost, d1, fs1, half, e, t1, shapes, used, assign, base, grid, kernel = best
    index = {k: i for i, k in enumerate(used)}
    subbands = [{"center": base + k * half, "channel": k} if bank else {"center": base + k * half} for k in used]
    members = [{"subband": index[k], "center": c, "rate": r, "interp2": shapes[r][0], "d2": shapes[r][1],
                "offset": c - (base + (grid[i] if bank else k) * half), "taps2": shapes[r][2]}
               for i, (c, r, k) in enumerate(zip(centers, rates, assign))]
    plan = {"d1": d1, "fs1": fs1, "taps1": t1, "e": e, "subbands": subbands, "members": members, "fmas": cost}
    if fft:
        plan["kernel"] = kernel
    return plan


# ---------------------------------------------------------------------------
# host-side server model in C (sdr-server_b200/host): ticket queue, dsp_worker,
# stream (sdr_callback fan-out).  Bound here only for the tests.
# ---------------------------------------------------------------------------
HOST_LIB_PATH = os.path.join(HERE, "lib", "libxlating_host.so")


class XlClientConfig(C.Structure):
    _fields_ = [("center_freq", C.c_uint32), ("sampling_rate", C.c_uint32), ("band_freq", C.c_uint32),
                ("destination", C.c_uint8), ("client_socket", C.c_int), ("id", C.c_uint32)]


class XlStreamConfig(C.Structure):
    _fields_ = [("sdr_type", C.c_int), ("band_sampling_rate", C.c_uint32), ("buffer_size", C.c_uint32),
                ("queue_size", C.c_int), ("lpf_cutoff_rate", C.c_int), ("base_path", C.c_char_p),
                ("device", C.c_int), ("use_gzip", C.c_int)]


_host = None


def host_lib() -> C.CDLL:
    global _host
    if _host is not None:
        return _host
    if not os.path.exists(HOST_LIB_PATH):
        raise RuntimeError(f"{HOST_LIB_PATH} is missing: run `make -C {HERE}/host`")
    lib()  # libxlating_b200.so first (rpath $ORIGIN also finds it)
    H = C.CDLL(HOST_LIB_PATH)
    vp = C.c_void_p
    H.xl_tq_create.argtypes = [C.c_int, C.POINTER(vp)]
    H.xl_tq_create.restype = C.c_int
    H.xl_tq_put.argtypes = [vp, C.c_int64]
    H.xl_tq_put.restype = None
    H.xl_tq_take.argtypes = [vp]
    H.xl_tq_take.restype = C.c_int64
    H.xl_tq_complete.argtypes = [vp]
    H.xl_tq_complete.restype = None
    H.xl_tq_interrupt.argtypes = [vp]
    H.xl_tq_interrupt.restype = None
    H.xl_tq_destroy.argtypes = [vp]
    H.xl_tq_destroy.restype = None
    H.xl_tq_overruns.argtypes = [vp]
    H.xl_tq_overruns.restype = C.c_uint64
    H.xl_stream_create.argtypes = [C.POINTER(XlStreamConfig), C.POINTER(vp)]
    H.xl_stream_create.restype = C.c_int
    H.xl_stream_add_client.argtypes = [vp, C.POINTER(XlClientConfig)]
    H.xl_stream_add_client.restype = C.c_int
    H.xl_stream_remove_client.argtypes = [vp, C.c_uint32]
    H.xl_stream_remove_client.restype = C.c_int
    H.xl_stream_push.argtypes = [vp, vp, C.c_uint32]
    H.xl_stream_push.restype = C.c_int
    H.xl_stream_flush.argtypes = [vp]
    H.xl_stream_flush.restype = C.c_int
    H.xl_stream_destroy.argtypes = [vp]
    H.xl_stream_destroy.restype = None
    H.xl_stream_client_count.argtypes = [vp]
    H.xl_stream_client_count.restype = C.c_int
    _host = H
    return H
