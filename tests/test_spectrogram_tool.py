"""CPU tests of the spectrogram tool (sdr-server_b200/host/sdr_spectrogram.c) and its PNG writer (host/png_gray.c).

The writer, driven through tests/png_gray_shim.c, must produce images that decode pixel for pixel with the suite's
own decoder (spectrum_exact.read_png) and with a plain zlib walk of the chunks that checks every CRC.  The tool's
refusals all come before it creates a group: each prints its message on stderr and exits non-zero with no GPU
visible, and leaves no image behind.
"""
import ctypes as C
import os
import struct
import subprocess
import zlib

import numpy as np
import pytest

from spectrum_exact import read_png

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "sdr-server_b200", "host")
TOOL = os.path.join(ROOT, "sdr-server_b200", "bin", "sdr_spectrogram")


@pytest.fixture(scope="module")
def shim(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("png") / "libpng_gray_shim.so")
    subprocess.run(["gcc", "-std=gnu11", "-O2", "-shared", "-fPIC", "-I" + HOST,
                    os.path.join(ROOT, "tests", "png_gray_shim.c"), os.path.join(HOST, "png_gray.c"), "-o", so,
                    "-lz"], check=True)
    L = C.CDLL(so)
    L.png_gray_write_file.argtypes = [C.c_char_p, C.c_uint32, C.c_uint32, C.c_void_p]
    L.png_gray_overrun.argtypes = [C.c_char_p]
    L.png_gray_short.argtypes = [C.c_char_p]
    return L


def zlib_decode(path):
    """(width, height, pixels) of an 8-bit grey PNG whose rows all use filter 0, every chunk's CRC checked."""
    data = open(path, "rb").read()
    assert data[:8] == b"\x89PNG\r\n\x1a\n"
    pos, idat, kinds = 8, b"", []
    while pos < len(data):
        n, kind = struct.unpack(">I4s", data[pos:pos + 8])
        body = data[pos + 8:pos + 8 + n]
        (crc,) = struct.unpack(">I", data[pos + 8 + n:pos + 12 + n])
        assert crc == zlib.crc32(kind + body), kind
        kinds.append(kind)
        if kind == b"IHDR":
            w, h, depth, color, comp, filt, interlace = struct.unpack(">IIBBBBB", body)
            assert (depth, color, comp, filt, interlace) == (8, 0, 0, 0, 0)
        elif kind == b"IDAT":
            idat += body
        pos += 12 + n
    assert kinds[0] == b"IHDR" and kinds[-1] == b"IEND" and b"IDAT" in kinds
    assert pos == len(data)
    raw = np.frombuffer(zlib.decompress(idat), np.uint8).reshape(h, w + 1)
    assert np.all(raw[:, 0] == 0)
    return w, h, raw[:, 1:]


@pytest.mark.parametrize("height", [1, 300])
@pytest.mark.parametrize("width", [1, 63, 64, 4096, 65536])
def test_png_writer_round_trip(shim, tmp_path, width, height):
    rng = np.random.default_rng(width * 1000 + height)
    px = rng.integers(0, 256, (height, width), dtype=np.uint8)
    px[0, 0], px[-1, -1] = 0, 255
    path = str(tmp_path / "x.png")
    assert shim.png_gray_write_file(path.encode(), width, height, px.ctypes.data) == 0
    w, h, got = zlib_decode(path)
    assert (w, h) == (width, height)
    np.testing.assert_array_equal(got, px)
    if width * height <= 65536:  # read_png's per-pixel loop is slow; the zlib walk above checks the large ones
        np.testing.assert_array_equal(read_png(path), px)


def test_png_writer_counts_rows(shim, tmp_path):
    path = str(tmp_path / "x.png").encode()
    assert shim.png_gray_overrun(path) == 0
    assert shim.png_gray_short(path) == 0
    assert shim.png_gray_write_file(path, 0, 1, None) != 0


def tool(*args, cwd=None):
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")  # a refusal must come before any GPU work
    return subprocess.run([TOOL, *map(str, args)], capture_output=True, text=True, env=env, cwd=cwd, timeout=60)


@pytest.fixture
def inp(tmp_path):
    p = tmp_path / "in.cu8"
    p.write_bytes(bytes(2 * 1000))
    return p


REFUSALS = [
    ([], "-i (input file) parameter is missing"),
    (["-i", "{inp}"], "-o (output file) parameter is missing"),
    (["-i", "{inp}", "-o", "{out}", "-w", "0"], "-w (width) should be positive. got: 0"),
    (["-i", "{inp}", "-o", "{out}", "-w", "-3"], "-w (width) should be positive. got: -3"),
    (["-i", "{inp}", "-o", "{out}", "-s", "0"], "-s (sampling_rate) should be positive. got: 0"),
    (["-i", "{inp}", "-o", "{out}", "-s", "0.5"], "-s (sampling_rate) should be positive. got: 0"),
    (["-i", "{inp}", "-o", "{out}", "-w", "100", "-s", "64"], "-w (100) is too wide for sampling rate 64"),
    (["-i", "{inp}", "-o", "{out}", "-d", "cs8"], "unsupported data format: cs8"),
    (["-i", "{inp}", "-o", "{out}", "-d", "f32"], "unsupported data format: f32"),
    (["-i", "{missing}", "-o", "{out}"], "unable to read input file {missing}: No such file or directory"),
    (["-i", "{inp}", "-o", "{out}", "-w", "5000", "-s", "100000"], "-w (5000) is not served"),
    (["-i", "{inp}", "-o", "{out}", "-w", "131072", "-s", "1e6"], "-w (131072) is not served"),
    (["-i", "{inp}", "-o", "{out}", "-s", "2147483648"], "-s (sampling_rate) 2147483648 is too high"),
    (["-i", "{inp}", "-o", "{out}", "-w", "64", "-s", "1001"], "fewer than one row of 1001"),
    (["-i", "{inp}", "-o", "{nodir}", "-w", "64", "-s", "1000"], "unable to write to output: {nodir}"),
]


@pytest.mark.parametrize("args,message", REFUSALS, ids=[m.split(":")[0][:40] for _, m in REFUSALS])
def test_tool_refusals(tmp_path, inp, args, message):
    names = {"inp": str(inp), "out": str(tmp_path / "out.png"), "missing": str(tmp_path / "missing.cu8"),
             "nodir": str(tmp_path / "no" / "out.png")}
    r = tool(*[a.format(**names) for a in args])
    assert r.returncode != 0
    assert message.format(**names) in r.stderr, r.stderr
    assert not (tmp_path / "out.png").exists()


def test_tool_refuses_short_gz(tmp_path):
    p = tmp_path / "in.cs16.gz"
    p.write_bytes(b"\x1f\x8b")
    r = tool("-i", p, "-o", tmp_path / "out.png", "-d", "cs16")
    assert r.returncode != 0 and f"premature end of file {p}" in r.stderr


def test_tool_help_and_unknown_fftw_flag(tmp_path, inp):
    r = tool("-h")
    assert r.returncode == 0 and "-d <data_format> data format: cu8, cs16, cf32 (default: cu8)" in r.stdout
    # an unknown -f prints the reference's fallback line; the unwritable output then stops the run before any GPU
    # work
    r = tool("-i", inp, "-o", tmp_path / "no" / "out.png", "-w", "64", "-s", "1000", "-f", "FFTW_PATIENT")
    assert r.returncode != 0
    assert "unsupported fftw flag: FFTW_PATIENT. Fallback to FFTW_ESTIMATE" in r.stderr
