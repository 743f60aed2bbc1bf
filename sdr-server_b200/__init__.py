"""sdr-server_b200 -- H100-native frequency-translating FIR decimator.

Thin ctypes bindings over ``lib/libxlating_b200.so`` (C ABI declared in
``include/xlating.h``, ``include/xlating_group.h``, ``include/lpf.h``).  The host
side of the product is C/C++ like the reference; this module only exists so that
the parity tests and ``bench.py`` can drive the C ABI the way the reference's own
callers do (``src/dsp_worker.c:98-124``, ``test/test_xlating.c``):

* :func:`create_low_pass_filter`  -> ``create_low_pass_filter``  (src/lpf.h:6)
* :class:`XlatingFilter`          -> ``create_frequency_xlating_filter`` /
  ``process_{native,optimized}_{cu8,cs8,cs16}_{cf32,cs16}`` / ``destroy_xlating``
  (src/xlating.h:10-38); :meth:`XlatingFilter.rational` -> the extension
  ``create_rational_frequency_xlating_filter``
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

FMT = {"cu8": 0, "cs8": 1, "cs16": 2}
NP_DTYPE = {"cu8": np.uint8, "cs8": np.int8, "cs16": np.int16}

XLG_OUT_DEVICE = 0x1
XLG_NO_RENORM = 0x2
XLG_FORCE_GENERIC = 0x4
XLG_SM_PARTITION = 0x10
XLG_TRACK_STATE = 0x20
XLG_INPUT_DEVICE = 0x100
XLG_PATH_Q15 = 0x200
XLG_INPUT_KEEP = 0x400
XLG_SLOTS = 4

# every symbol the headers declare (checked by tests/test_abi.py)
REFERENCE_SYMBOLS = (
    ["create_frequency_xlating_filter", "destroy_xlating", "SIMD_STATUS", "create_low_pass_filter"]
    + [f"process_{v}_{f}_{o}" for v in ("native", "optimized") for f in ("cu8", "cs8", "cs16") for o in ("cf32", "cs16")]
)
# include/xlating.h's extension of the reference's per-filter ABI
DROPIN_EXTENSION_SYMBOLS = ["create_rational_frequency_xlating_filter"]
GROUP_SYMBOLS = [
    "xlg_create", "xlg_create_ex", "xlg_destroy", "xlg_add_client", "xlg_add_client_ex", "xlg_add_client_rational_ex", "xlg_remove_client", "xlg_reserve", "xlg_client_count", "xlg_submit",
    "xlg_wait", "xlg_input_consumed", "xlg_output", "xlg_read_output", "xlg_copy_output", "xlg_alloc_pinned", "xlg_free_pinned", "xlg_wait_stream", "xlg_partition_active", "xlg_timer_start",
    "xlg_timer_stop", "xlg_profile_enable", "xlg_profile_read", "xlg_client_info", "xlg_add_client_rational", "xlg_poly_profile_read", "xlg_add_client_cascade", "xlg_cascade_info", "xlg_cascade_profile_read", "xlg_dropin_stats", "xlg_dropin_stream_stats", "xlg_dropin_stream_times",
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
    L.xlg_cascade_info.argtypes = [vp, C.c_int, C.POINTER(C.c_int), C.POINTER(sz), C.POINTER(sz)]
    L.xlg_cascade_info.restype = C.c_int
    L.xlg_cascade_profile_read.argtypes = [vp, C.POINTER(XlgCascadeProfile), C.c_int]
    L.xlg_cascade_profile_read.restype = C.c_int
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


class XlatingFilter:
    """Per-client drop-in filter (reference API: src/xlating.h:10-38)."""

    def __init__(self, decimation: int, taps, center_freq: int, sampling_freq: int, max_input_buffer_length: int,
                 interp: int | None = None):
        self._L = lib()
        taps = np.ascontiguousarray(taps, dtype=np.float32)
        mem = None
        if len(taps) > 0:
            # create adopts (and later free()s) the vector, as the reference does
            mem = _libc.malloc(taps.nbytes)
            C.memmove(mem, taps.ctypes.data, taps.nbytes)
        h = C.c_void_p()
        if interp is None:
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

    def add_client(self, decimation: int, taps, center_freq: int) -> int:
        taps = np.ascontiguousarray(taps, dtype=np.float32)
        cid = C.c_int(-1)
        code = self._L.xlg_add_client(self._h, decimation, taps.ctypes.data_as(C.POINTER(C.c_float)), len(taps),
                                      center_freq, C.byref(cid))
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

    def add_client_cascade(self, decim1: int, taps1, center_freq: int, decim2: int, taps2) -> int:
        """A two-stage client (include/xlating_group.h, xlg_add_client_cascade): the reference filter
        (decim1, taps1, center_freq) at fs, followed by the reference filter (decim2, taps2, centre 0) at
        fs / decim1 fed its outputs.  See cascade_plan for taps."""
        t1 = np.ascontiguousarray(taps1, dtype=np.float32)
        t2 = np.ascontiguousarray(taps2, dtype=np.float32)
        cid = C.c_int(-1)
        fp = C.POINTER(C.c_float)
        code = self._L.xlg_add_client_cascade(self._h, decim1, t1.ctypes.data_as(fp), len(t1), center_freq, decim2,
                                              t2.ctypes.data_as(fp), len(t2), C.byref(cid))
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
        """data: numpy array (host) -- or (device_ptr, n_elements) with XLG_INPUT_DEVICE."""
        if flags & XLG_INPUT_DEVICE:
            ptr, n = data
        else:
            data = np.ascontiguousarray(data, dtype=NP_DTYPE[fmt])
            ptr, n = data.ctypes.data, data.size
        t = self._L.xlg_submit(self._h, FMT[fmt], ptr, n, flags)
        if t < 0:
            raise RuntimeError(f"xlg_submit -> {t}")
        return t

    def submit_ptr(self, fmt_code: int, ptr: int, n: int, flags: int = 0) -> int:
        t = self._L.xlg_submit(self._h, fmt_code, ptr, n, flags)
        if t < 0:
            raise RuntimeError(f"xlg_submit -> {t}")
        return t

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


def cascade_fmas(fs: int, rate: int, d1: int, t1: int, t2: int) -> float:
    """Algorithmic real FMAs per input sample of a cascade client: 4 per complex tap of stage A at fs / d1,
    2 per real tap of stage B at the client rate."""
    return 4.0 * t1 / d1 + 2.0 * t2 / (fs // rate)


def cascade_stages(fs: int, rate: int, d1: int):
    """Taps of the two stages for D1 = d1: stage B is the server's own design at fs1 = fs / d1 (cutoff
    rate / 2, transition rate / 5); stage A passes up to e = 3 * rate / 5 (stage B's passband edge plus half
    its transition) and stops from fs1 - e, so everything it aliases onto the band lands in stage B's
    stopband: create_low_pass_filter(1, fs, fs1 / 2, fs1 - 2e)."""
    fs1 = fs // d1
    e = 3 * rate // 5
    return (create_low_pass_filter(1.0, fs, fs1 // 2, fs1 - 2 * e),
            create_low_pass_filter(1.0, fs1, rate // 2, rate // 5))


def cascade_plan(fs: int, rates):
    """Two-stage clients for rates that divide fs: for D = fs / rate, the divisor D1 >= 2 of D (with
    D2 = D / D1 >= 2) with the fewest estimated FMAs per input sample, 4*T1/D1 + 2*T2/D (cascade_fmas;
    ties go to the smaller D1).  Taps from cascade_stages; centres as client_plan places them."""
    plan = []
    for p, rate in zip(client_plan(fs, rates), rates):
        rate = int(rate)
        if fs % rate != 0:
            raise ValueError(f"{rate} does not divide {fs}")
        D = fs // rate
        best = None
        for d1 in range(2, D // 2 + 1):
            if D % d1 != 0 or fs % d1 != 0:
                continue
            t1, t2 = cascade_stages(fs, rate, d1)
            cost = cascade_fmas(fs, rate, d1, t1.size, t2.size)
            if best is None or cost < best[0]:
                best = (cost, d1, t1, t2)
        if best is None:
            raise ValueError(f"decimation {D} has no divisor D1 >= 2 with D / D1 >= 2")
        cost, d1, t1, t2 = best
        plan.append({"rate": rate, "d1": d1, "d2": D // d1, "center": p["center"], "taps1": t1, "taps2": t2,
                     "fmas": cost})
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
