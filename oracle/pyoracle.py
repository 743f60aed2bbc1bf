"""ctypes bindings for the CPU oracle.  TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline /
``--impl reference`` legs may import this module (see oracle/oracle.h).  It wraps

* ``oracle/liboracle.so``  -- our restatement (oracle/xlating_oracle.c, lpf_oracle.c)
* ``oracle/_ref/libref_{strict,release,avx}.so`` -- the unmodified reference
  sources compiled from /root/reference by oracle/Makefile (reference API:
  /root/reference/src/xlating.h:10-38, src/lpf.h:6).

Nothing here reads /root/reference at run time; the ``_ref`` libraries are
prebuilt by ``make -C oracle`` (``__graft_entry__.build()``) and travel with the
repo snapshot.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
FMT = {"cu8": 0, "cs8": 1, "cs16": 2}
NP_DTYPE = {"cu8": np.uint8, "cs8": np.int8, "cs16": np.int16}

_libc = C.CDLL(None)
_libc.malloc.restype = C.c_void_p
_libc.malloc.argtypes = [C.c_size_t]
_libc.free.argtypes = [C.c_void_p]


def build(quiet: bool = True) -> None:
    """make -C oracle: liboracle.so always, _ref/ only when /root/reference exists."""
    subprocess.run(["make", "-C", HERE, "all"], check=True,
                   stdout=subprocess.DEVNULL if quiet else None)


def _load(path: str) -> C.CDLL:
    if not os.path.exists(path):
        build()
    return C.CDLL(path)


# --------------------------------------------------------------------------
# restatement
# --------------------------------------------------------------------------
_orc = None


def orc() -> C.CDLL:
    global _orc
    if _orc is None:
        lib = _load(os.path.join(HERE, "liboracle.so"))
        lib.orc_lpf_design.argtypes = [C.c_float, C.c_uint32, C.c_uint32, C.c_uint32,
                                       C.POINTER(C.POINTER(C.c_float)), C.POINTER(C.c_size_t)]
        lib.orc_lpf_design.restype = C.c_int
        lib.orc_xlating_create.argtypes = [C.c_uint32, C.POINTER(C.c_float), C.c_size_t, C.c_int32,
                                           C.c_uint32, C.c_uint32, C.POINTER(C.c_void_p)]
        lib.orc_xlating_create.restype = C.c_int
        lib.orc_xlating_destroy.argtypes = [C.c_void_p]
        lib.orc_xlating_process_cf32.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t, C.c_int,
                                                 C.POINTER(C.POINTER(C.c_float))]
        lib.orc_xlating_process_cf32.restype = C.c_size_t
        lib.orc_xlating_process_q15.argtypes = [C.c_void_p, C.c_int, C.c_void_p, C.c_size_t,
                                                C.POINTER(C.POINTER(C.c_int16))]
        lib.orc_xlating_process_q15.restype = C.c_size_t
        lib.orc_xlating_history.argtypes = [C.c_void_p]
        lib.orc_xlating_history.restype = C.c_size_t
        lib.orc_xlating_phase.argtypes = [C.c_void_p, C.POINTER(C.c_float), C.POINTER(C.c_float)]
        lib.orc_xlating_taps.argtypes = [C.c_void_p, C.POINTER(C.POINTER(C.c_float))]
        lib.orc_xlating_taps.restype = C.c_size_t
        lib.orc_xlating_q15_consts.argtypes = [C.c_void_p, C.POINTER(C.POINTER(C.c_int16)), C.POINTER(C.c_int16),
                                               C.POINTER(C.c_int16)]
        lib.orc_xlating_q15_consts.restype = C.c_size_t
        lib.orc_xlating_set_state.argtypes = [C.c_void_p, C.POINTER(C.c_float), C.c_size_t, C.c_float, C.c_float]
        lib.orc_xlating_set_state.restype = C.c_int
        _orc = lib
    return _orc


def lpf_design(gain: float, fs: int, cutoff: int, tw: int) -> np.ndarray:
    """Oracle tap designer; raises ValueError on the reference's -1 cases."""
    lib = orc()
    p = C.POINTER(C.c_float)()
    n = C.c_size_t(0)
    code = lib.orc_lpf_design(gain, fs, cutoff, tw, C.byref(p), C.byref(n))
    if code != 0:
        raise ValueError(f"orc_lpf_design -> {code}")
    out = np.ctypeslib.as_array(p, shape=(n.value,)).copy()
    _libc.free(C.cast(p, C.c_void_p))
    return out


class OracleFilter:
    """One client of the restated xlating filter."""

    def __init__(self, decimation: int, taps: np.ndarray, center_freq: int, fs: int, max_input_len: int):
        lib = orc()
        taps = np.ascontiguousarray(taps, dtype=np.float32)
        h = C.c_void_p()
        code = lib.orc_xlating_create(decimation, taps.ctypes.data_as(C.POINTER(C.c_float)), len(taps),
                                      center_freq, fs, max_input_len, C.byref(h))
        if code != 0:
            raise ValueError(f"orc_xlating_create -> {code}")
        self._h = h
        self._lib = lib

    def process_cf32(self, fmt: str, data: np.ndarray, renorm: bool = True) -> np.ndarray:
        data = np.ascontiguousarray(data, dtype=NP_DTYPE[fmt])
        out = C.POINTER(C.c_float)()
        n = self._lib.orc_xlating_process_cf32(self._h, FMT[fmt], data.ctypes.data, data.size,
                                               1 if renorm else 0, C.byref(out))
        if n == 0:
            return np.zeros(0, dtype=np.complex64)
        return np.ctypeslib.as_array(out, shape=(2 * n,)).copy().view(np.complex64)

    def process_q15(self, fmt: str, data: np.ndarray) -> np.ndarray:
        data = np.ascontiguousarray(data, dtype=NP_DTYPE[fmt])
        out = C.POINTER(C.c_int16)()
        n = self._lib.orc_xlating_process_q15(self._h, FMT[fmt], data.ctypes.data, data.size, C.byref(out))
        if n == 0:
            return np.zeros((0, 2), dtype=np.int16)
        return np.ctypeslib.as_array(out, shape=(2 * n,)).copy().reshape(-1, 2)

    @property
    def history(self) -> int:
        return self._lib.orc_xlating_history(self._h)

    @property
    def phase(self) -> complex:
        re, im = C.c_float(), C.c_float()
        self._lib.orc_xlating_phase(self._h, C.byref(re), C.byref(im))
        return complex(re.value, im.value)

    def set_state(self, history: np.ndarray, phase: complex) -> None:
        """Continue from a given state: `history` (complex, oldest first) is what the next window reaches
        back to, its length the history offset; `phase` the oscillator."""
        h = np.ascontiguousarray(np.asarray(history, dtype=np.complex64)).view(np.float32)
        code = self._lib.orc_xlating_set_state(self._h, h.ctypes.data_as(C.POINTER(C.c_float)), h.size // 2,
                                               float(phase.real), float(phase.imag))
        if code != 0:
            raise ValueError(f"orc_xlating_set_state -> {code}")

    @property
    def rev_taps(self) -> np.ndarray:
        p = C.POINTER(C.c_float)()
        n = self._lib.orc_xlating_taps(self._h, C.byref(p))
        return np.ctypeslib.as_array(p, shape=(2 * n,)).copy().view(np.complex64)

    @property
    def q15_consts(self):
        """((T, 2) int16 reversed Q15 taps, (qinc_re, qinc_im))."""
        p = C.POINTER(C.c_int16)()
        qr, qi = C.c_int16(), C.c_int16()
        n = self._lib.orc_xlating_q15_consts(self._h, C.byref(p), C.byref(qr), C.byref(qi))
        return np.ctypeslib.as_array(p, shape=(2 * n,)).copy().reshape(n, 2), (qr.value, qi.value)

    def close(self):
        if self._h:
            self._lib.orc_xlating_destroy(self._h)
            self._h = None

    def __del__(self):
        self.close()


# --------------------------------------------------------------------------
# the compiled reference (oracle/_ref)
# --------------------------------------------------------------------------
_ref_cache: dict = {}


def ref_available(flavor: str = "strict") -> bool:
    return os.path.exists(os.path.join(HERE, "_ref", f"libref_{flavor}.so"))


def ref(flavor: str = "strict") -> C.CDLL:
    """Load oracle/_ref/libref_<flavor>.so (RTLD_LOCAL: the three flavours
    export the same symbol names)."""
    if flavor not in _ref_cache:
        path = os.path.join(HERE, "_ref", f"libref_{flavor}.so")
        if not os.path.exists(path):
            raise FileNotFoundError(path)
        lib = C.CDLL(path, mode=os.RTLD_LOCAL | os.RTLD_NOW)
        lib.create_low_pass_filter.argtypes = [C.c_float, C.c_uint32, C.c_uint32, C.c_uint32,
                                               C.POINTER(C.c_void_p), C.POINTER(C.c_size_t)]
        lib.create_low_pass_filter.restype = C.c_int
        lib.create_frequency_xlating_filter.argtypes = [C.c_uint32, C.c_void_p, C.c_size_t, C.c_int32,
                                                        C.c_uint32, C.c_uint32, C.POINTER(C.c_void_p)]
        lib.create_frequency_xlating_filter.restype = C.c_int
        lib.destroy_xlating.argtypes = [C.c_void_p]
        for variant in ("native", "optimized"):
            for fmt in ("cu8", "cs8", "cs16"):
                for o in ("cf32", "cs16"):
                    fn = getattr(lib, f"process_{variant}_{fmt}_{o}")
                    fn.argtypes = [C.c_void_p, C.c_size_t, C.POINTER(C.c_void_p), C.POINTER(C.c_size_t), C.c_void_p]
                    fn.restype = None
        _ref_cache[flavor] = lib
    return _ref_cache[flavor]


def ref_simd_status(flavor: str) -> str:
    lib = ref(flavor)
    return C.c_char_p.in_dll(lib, "SIMD_STATUS").value.decode()


def ref_lpf_design(gain: float, fs: int, cutoff: int, tw: int, flavor: str = "strict") -> np.ndarray:
    lib = ref(flavor)
    p = C.c_void_p()
    n = C.c_size_t(0)
    code = lib.create_low_pass_filter(gain, fs, cutoff, tw, C.byref(p), C.byref(n))
    if code != 0:
        raise ValueError(f"create_low_pass_filter -> {code}")
    out = np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_float)), shape=(n.value,)).copy()
    _libc.free(p)
    return out


class RefFilter:
    """One client of the compiled reference filter (src/xlating.h API)."""

    def __init__(self, decimation: int, taps: np.ndarray, center_freq: int, fs: int, max_input_len: int,
                 flavor: str = "strict"):
        self._lib = ref(flavor)
        taps = np.ascontiguousarray(taps, dtype=np.float32)
        # the reference adopts (and later free()s) the tap vector: hand it malloc'd memory
        mem = _libc.malloc(taps.nbytes)
        C.memmove(mem, taps.ctypes.data, taps.nbytes)
        h = C.c_void_p()
        code = self._lib.create_frequency_xlating_filter(decimation, mem, len(taps), center_freq, fs,
                                                         max_input_len, C.byref(h))
        if code != 0:
            raise ValueError(f"create_frequency_xlating_filter -> {code}")
        self._h = h

    def _call(self, name: str, data: np.ndarray):
        out = C.c_void_p()
        n = C.c_size_t(0)
        getattr(self._lib, name)(data.ctypes.data, data.size, C.byref(out), C.byref(n), self._h)
        return out, n.value

    def process_cf32(self, fmt: str, data: np.ndarray, variant: str = "native") -> np.ndarray:
        data = np.ascontiguousarray(data, dtype=NP_DTYPE[fmt])
        out, n = self._call(f"process_{variant}_{fmt}_cf32", data)
        if n == 0:
            return np.zeros(0, dtype=np.complex64)
        return np.ctypeslib.as_array(C.cast(out, C.POINTER(C.c_float)), shape=(2 * n,)).copy().view(np.complex64)

    def process_q15(self, fmt: str, data: np.ndarray, variant: str = "native") -> np.ndarray:
        data = np.ascontiguousarray(data, dtype=NP_DTYPE[fmt])
        out, n = self._call(f"process_{variant}_{fmt}_cs16", data)
        if n == 0:
            return np.zeros((0, 2), dtype=np.int16)
        return np.ctypeslib.as_array(C.cast(out, C.POINTER(C.c_int16)), shape=(2 * n,)).copy().reshape(-1, 2)

    def process_raw(self, fmt: str, data_ptr: int, nelem: int, variant: str = "native") -> int:
        """Timing entry: no output copy.  Returns the number of complex outputs."""
        out = C.c_void_p()
        n = C.c_size_t(0)
        getattr(self._lib, f"process_{variant}_{fmt}_cf32")(data_ptr, nelem, C.byref(out), C.byref(n), self._h)
        return n.value

    def close(self):
        if self._h:
            self._lib.destroy_xlating(self._h)
            self._h = None

    def __del__(self):
        self.close()
