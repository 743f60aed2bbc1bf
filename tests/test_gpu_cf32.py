"""cf32 input (XLG_FMT_CF32) and the spectrogram tool (bin/sdr_spectrogram) on the GPU.

1. The tool reproduces the reference's four spectrogram goldens pixel for pixel from plain and .gz files, and the
   two cf32 goldens also come back through Group as the cu8 and cs16 ones do in test_gpu_spectrum.py.
2. The tool against the model: random cu8, cs16 and cf32 files from W = 1 to 65536, sizes that are not multiples
   of the row or of the sample, rows across the tool's blocks; pixels are spectrogram_pixels of 10 * log10f (the C
   library's, through ctypes) of spectrum_model's / wide_model's float32 rows.
3. cf32 equals raw: one group holding every client family, banks and band, client and sub-band spectra (plain,
   Welch, wide) fed ragged, odd and empty cu8, cs8 and cs16 blocks, and a twin fed their exact float images
   through every ingest path; every output, row and count is bitwise equal, with device outputs, and on an
   XLG_TRACK_STATE group the state after each ticket as well.
4. Values no integer format produces: spectra of random floats up to 1e30, -0.0 and subnormals against the model
   bit for bit; a NaN or an infinity changes only the outputs whose windows and the rows whose frames hold it.
5. Refusals: a misaligned device block and a Q15 cf32 submit take no ticket.
"""
import ctypes as C
import gzip
import os
import subprocess

import numpy as np
import pytest

from exact import to_complex
from spectrum_exact import GOLDEN_DIR, GOLDEN_FS, GOLDENS, golden_stimulus, read_png, spectrum_model
from spectrum_wide import wide_model
from util import rand_block

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOOL = os.path.join(ROOT, "sdr-server_b200", "bin", "sdr_spectrogram")
F32 = np.float32
EINVAL = -22
_LIBM = C.CDLL("libm.so.6")
_LIBM.log10f.restype = C.c_float
_LIBM.log10f.argtypes = [C.c_float]


def log10f(v):
    """The C library's log10f, the function the tool calls, element by element."""
    v = np.asarray(v, F32)
    return np.array([_LIBM.log10f(float(a)) for a in v.ravel()], F32).reshape(v.shape)


def tool_pixels(pkg, rows):
    return pkg.spectrogram_pixels(F32(10) * log10f(rows))


def image(fmt, raw):
    """The exact float32 image of a raw block, as interleaved (re, im) float32."""
    if fmt == "cu8":
        return ((raw.astype(np.float64) - 127.5) / 128).astype(F32)
    return (raw.astype(np.float64) / (128 if fmt == "cs8" else 32768)).astype(F32)


def file_bytes(fmt, x):
    return np.ascontiguousarray(x).astype({"cu8": np.uint8, "cs16": "<i2", "cf32": "<c8"}[fmt]).tobytes()


def run_tool(*args):
    return subprocess.run([TOOL, *map(str, args)], capture_output=True, text=True, timeout=600)


# ---------------------------------------------------------------------------
# 1. goldens
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("gz", [False, True], ids=["plain", "gz"])
@pytest.mark.parametrize("name", sorted(GOLDENS))
def test_tool_reproduces_golden(tmp_path, name, gz):
    fmt, W = GOLDENS[name]
    data = file_bytes(fmt, golden_stimulus(fmt))
    src = tmp_path / (f"in.{fmt}" + (".gz" if gz else ""))
    if gz:
        with gzip.open(src, "wb") as f:
            f.write(data)
    else:
        src.write_bytes(data)
    out = tmp_path / "out.png"
    r = run_tool("-w", W, "-s", GOLDEN_FS, "-d", fmt, "-i", src, "-o", out)
    assert r.returncode == 0, r.stderr
    np.testing.assert_array_equal(read_png(out), read_png(os.path.join(GOLDEN_DIR, name)))


@pytest.mark.parametrize("name", ["spectrogram_cf32.png", "spectrogram_cf32_odd.png"])
@pytest.mark.parametrize("cuts", [[256], [100, 0, 1, 155]])
def test_cf32_golden_pixels(pkg, name, cuts):
    fmt, W = GOLDENS[name]
    F, S = pkg.spectrogram_params(GOLDEN_FS, W)
    x = golden_stimulus(fmt)
    g = pkg.Group(GOLDEN_FS, 512)
    rows = []
    try:
        sid = g.add_spectrum(W, F, S)
        pos = 0
        for n in cuts:
            rows.append(g.read_spectrum(g.submit("cf32", x[pos:pos + n]), sid))
            pos += n
    finally:
        g.close()
    np.testing.assert_array_equal(pkg.spectrogram_pixels(np.concatenate(rows)), read_png(f"{GOLDEN_DIR}/{name}"))


# ---------------------------------------------------------------------------
# 2. the tool against the model
# ---------------------------------------------------------------------------
# (W, format, fs, complex samples): S = fs % W is nonzero except at W = 64; the tool submits 2^20 samples per block,
# so every file but the direct W = 1000 one spans several blocks, and rows span blocks at the wide widths
TOOL_CASES = [(1, "cu8", 1000, 2_500_123), (3, "cs16", 2000, 2_300_001), (63, "cf32", 10_000, 1_100_003),
              (64, "cu8", 48_000, 3_100_007), (1000, "cs16", 12_345, 80_011), (1024, "cf32", 100_000, 3_000_005),
              (4096, "cu8", 250_000, 3_200_001), (8192, "cs16", 500_000, 4_000_003),
              (65536, "cf32", 200_000, 5_000_001)]


@pytest.mark.parametrize("W,fmt,fs,n", TOOL_CASES, ids=[f"W{c[0]}_{c[1]}" for c in TOOL_CASES])
def test_tool_against_model(pkg, tmp_path, W, fmt, fs, n):
    rng = np.random.default_rng(W)
    if fmt == "cf32":
        x = (rng.standard_normal(n) + 1j * rng.standard_normal(n)).astype(np.complex64)
        data = file_bytes(fmt, x) + b"\x01\x02\x03"  # a partial trailing sample
    else:
        raw = rand_block(rng, fmt, 2 * n)
        x = to_complex(fmt, raw).astype(np.complex64)
        data = file_bytes(fmt, raw) + b"\x07"
    src, out = tmp_path / f"in.{fmt}", tmp_path / "out.png"
    src.write_bytes(data)
    r = run_tool("-w", W, "-s", fs, "-d", fmt, "-i", src, "-o", out)
    src.unlink()  # up to 40 MB: the temporary directory may be memory-backed
    assert r.returncode == 0, r.stderr
    F, S = pkg.spectrogram_params(fs, W)
    height = n // fs
    model = wide_model if W > 4096 else spectrum_model
    rows = model(x[:height * fs], W, F, S)
    assert rows.shape == (height, W)
    got = read_png(out)
    assert got.shape == (height, W)
    np.testing.assert_array_equal(got, tool_pixels(pkg, rows))


def test_tool_truncated_gz_fails(tmp_path):
    """A .gz whose data ends before its trailer's size: non-zero exit, and no image left behind."""
    rng = np.random.default_rng(3)
    data = rand_block(rng, "cu8", 2 * 5000).tobytes()
    whole = gzip.compress(data)
    # keep the trailer (its size announces 5000 samples) but drop compressed data from the middle
    src = tmp_path / "cut.cu8.gz"
    src.write_bytes(whole[:len(whole) // 2] + whole[-8:])
    out = tmp_path / "out.png"
    r = run_tool("-w", 64, "-s", 1000, "-d", "cu8", "-i", src, "-o", out)
    assert r.returncode != 0
    assert not out.exists()


# ---------------------------------------------------------------------------
# 3. cf32 equals raw, bit for bit
# ---------------------------------------------------------------------------
FS_MIX, MAX_MIX = 2048000, 65536


def rtaps(rng, n):
    return rng.standard_normal(n).astype(F32) / n


def population(pkg, g, rng):
    """Every client family, a sub-band, both bank kinds and band, client and sub-band spectra (plain, Welch,
    wide).  Returns (client ids, spectrum ids)."""
    ids = [g.add_client(32, rtaps(rng, 97), -900000 + 110000 * c) for c in range(8)]  # a tiled class
    ids.append(g.add_client(5, rtaps(rng, 40), 300000))  # generic
    ids += [g.add_client(1280, rtaps(rng, 2561), 20000 * c) for c in range(8)]  # a split-K long class
    plan = pkg.rational_plan(FS_MIX, [48000] * 8)
    ids += [g.add_client_rational(p["interp"], p["decim"], p["taps"], p["center"]) for p in plan]
    ids.append(g.add_client_cascade(16, rtaps(rng, 65), 200000, 4, rtaps(rng, 33)))
    sb = g.add_subband(32, rtaps(rng, 129), -400000)
    ids.append(g.add_client_subband(sb, 4, rtaps(rng, 33), 5000))
    bid = g.add_bank(16, rtaps(rng, 257))
    ids.append(g.add_client_subband(g.add_bank_subband(bid, 3), 4, rtaps(rng, 33), 0))
    fid = g.add_bank_fft(16, rtaps(rng, 257))
    ids.append(g.add_client_subband(g.add_bank_subband(fid, -5), 4, rtaps(rng, 33), 0))
    sids = [g.add_spectrum(8192, 1, 100, power=True),
            g.add_client_spectrum(ids[8], 256, 4, 5, power=True, hop=128, window=np.hanning(256).astype(F32),
                                  mean=True),
            g.add_subband_spectrum(sb, 64, 2, 3, power=True)]
    return ids, sids


class CfFeeder:
    """Submits the cf32 image of a block through one ingest path; buffers are overwritten at the earliest moment
    the contract allows."""

    def __init__(self, pkg, g, torch, max_in):
        self.pkg, self.g, self.torch = pkg, g, torch
        self.pinned, self.keep = pkg.PinnedBuffer(4 * max_in), pkg.PinnedBuffer(4 * max_in)
        self.dev = torch.zeros(max_in // 2, dtype=torch.complex64, device="cuda")
        self.src = torch.zeros(max_in // 2, dtype=torch.complex64).pin_memory()
        self.side = torch.cuda.Stream()
        self.pending = []

    def flush(self):
        while self.pending:
            self.pending.pop(0)()

    def close(self):
        self.flush()
        self.pinned.free()
        self.keep.free()

    def submit(self, mode, v):
        """v: interleaved float32 (re, im)."""
        self.flush()
        g, pkg, torch = self.g, self.pkg, self.torch
        n = v.size
        if mode == "pageable":
            buf = v.copy()
            t = g.submit("cf32", buf)
            buf[:] = np.nan
        elif mode in ("pinned", "keep"):
            pb = self.pinned if mode == "pinned" else self.keep
            view = pb.array(np.float32)[:n]
            view[:] = v
            if mode == "pinned":
                t = g.submit_ptr(pkg.FMT["cf32"], pb.ptr, n)
                view[:] = np.nan
            else:
                t = g.submit_ptr(pkg.FMT["cf32"], pb.ptr, n, pkg.XLG_INPUT_KEEP)
                self.pending.append(lambda: (g.input_consumed(t), view.__setitem__(slice(None), np.nan)))
        elif mode == "torch":
            d = torch.from_numpy(v[:n // 2 * 2].copy()).view(torch.complex64).cuda()
            torch.cuda.current_stream().synchronize()
            t = g.submit("cf32", d)
            self.pending.append(lambda: (g.input_consumed(t), d.fill_(float("nan")), torch.cuda.synchronize()))
        elif mode == "stream":
            m = n // 2
            self.src[:m].copy_(torch.from_numpy(v[:2 * m].copy()).view(torch.complex64))
            with torch.cuda.stream(self.side):
                self.dev[:m].copy_(self.src[:m], non_blocking=True)
            g.wait_stream(self.side.cuda_stream)
            t = g.submit_ptr(pkg.FMT["cf32"], self.dev.data_ptr(), n, pkg.XLG_INPUT_DEVICE)

            def release():
                g.input_consumed(t)
                self.side.synchronize()
                self.dev.fill_(float("nan"))
                torch.cuda.synchronize()
            self.pending.append(release)
        else:
            raise ValueError(mode)
        return t


MODES = ["pageable", "pinned", "keep", "torch", "stream"]
RAGGED = [MAX_MIX, MAX_MIX - 2, 0, 30002, 7, MAX_MIX, 1, 4098, MAX_MIX, 2]  # scalars


@pytest.mark.parametrize("flag", [0, "XLG_OUT_DEVICE"], ids=["host_out", "device_out"])
def test_cf32_images_equal_raw(pkg, flag):
    torch = pytest.importorskip("torch")
    flags = getattr(pkg, flag) if flag else 0
    a, b = pkg.Group(FS_MIX, MAX_MIX, flags=flags), pkg.Group(FS_MIX, MAX_MIX, flags=flags)
    ids, sids = population(pkg, a, np.random.default_rng(7))
    assert (ids, sids) == population(pkg, b, np.random.default_rng(7))
    f = CfFeeder(pkg, b, torch, MAX_MIX)
    rng = np.random.default_rng(8)
    fmts = ["cu8", "cs8", "cs16"]
    pend, rows_seen = [], 0

    def collect():
        i, ta, tb = pend.pop(0)
        a.wait(ta)
        b.wait(tb)
        for c in ids:
            ya, yb = a.read_output(ta, c), b.read_output(tb, c)
            assert ya.shape == yb.shape, (i, c)
            assert ya.view(np.uint32).tobytes() == yb.view(np.uint32).tobytes(), f"block {i}: client {c}"
        nonlocal rows_seen
        for s in sids:
            ra, rb = a.read_spectrum(ta, s), b.read_spectrum(tb, s)
            assert ra.shape == rb.shape and ra.tobytes() == rb.tobytes(), f"block {i}: spectrum {s}"
            rows_seen += ra.shape[0]

    for i in range(3 * len(MODES)):
        fmt, n, mode = fmts[i % 3], RAGGED[i % len(RAGGED)], MODES[i % len(MODES)]
        raw = rand_block(rng, fmt, n)
        ta = a.submit(fmt, raw)
        tb = f.submit(mode, image(fmt, raw))
        assert ta == tb
        for c in ids:
            assert a.output_ptr(ta, c)[1] == b.output_ptr(tb, c)[1]
        pend.append((i, ta, tb))
        if len(pend) >= pkg.XLG_SLOTS - 1:
            collect()
    f.close()
    while pend:
        collect()
    kinds = {a.client_info(c)[1] for c in ids}
    a.close()
    b.close()
    assert kinds >= {0, 1, 2, 5, 6} and kinds & {3, 4}, kinds
    assert rows_seen > 0


def test_cf32_images_equal_raw_track_state(pkg):
    torch = pytest.importorskip("torch")
    a = pkg.Group(FS_MIX, MAX_MIX, flags=pkg.XLG_TRACK_STATE)
    b = pkg.Group(FS_MIX, MAX_MIX, flags=pkg.XLG_TRACK_STATE)
    rng = np.random.default_rng(9)
    specs = [(32, rtaps(rng, 97), 110000 * c) for c in range(8)] + [(5, rtaps(rng, 40), -300000)]
    ids = [a.add_client(*s) for s in specs]
    assert ids == [b.add_client(*s) for s in specs]
    f = CfFeeder(pkg, b, torch, MAX_MIX)
    for i in range(2 * len(MODES)):
        fmt, n = ["cu8", "cs8", "cs16"][i % 3], RAGGED[i % len(RAGGED)]
        raw = rand_block(rng, fmt, n)
        ta = a.submit(fmt, raw)
        tb = f.submit(MODES[i % len(MODES)], image(fmt, raw))
        f.flush()
        a.wait(ta)
        b.wait(tb)
        for c in ids:
            (ya, sa), (yb, sb) = a.copy_output(ta, c), b.copy_output(tb, c)
            assert ya.tobytes() == yb.tobytes(), (i, c)
            assert (sa.hist, sa.phase_re, sa.phase_im) == (sb.hist, sb.phase_re, sb.phase_im), (i, c)
    f.close()
    a.close()
    b.close()


# ---------------------------------------------------------------------------
# 4. values no integer format produces
# ---------------------------------------------------------------------------
def wild(rng, n):
    """n complex samples of random sign and magnitude from 1e-45 (subnormal) to 1e30, with -0.0 and +0.0."""
    mag = 10.0 ** rng.uniform(-45, 30, 2 * n)
    v = (np.where(rng.integers(0, 2, 2 * n) == 1, -1, 1) * mag).astype(F32)
    v[rng.integers(0, 2 * n, n // 50)] = -0.0
    v[rng.integers(0, 2 * n, n // 50)] = 0.0
    return v


@pytest.mark.parametrize("W,F,S", [(63, 2, 5), (1024, 1, 300), (8192, 1, 0)])
def test_wild_floats_spectra_bit_exact(pkg, W, F, S):
    rng = np.random.default_rng(W)
    sizes = [20000, 0, 1, 16384, 9999]
    blocks = [wild(rng, n) for n in sizes]
    g = pkg.Group(FS_MIX, 2 * 20000)
    got = []
    try:
        sid = g.add_spectrum(W, F, S, power=True)
        for v in blocks:
            got.append(g.read_spectrum(g.submit("cf32", v), sid))
    finally:
        g.close()
    x = np.concatenate(blocks).view(np.complex64)
    model = wide_model if W > 4096 else spectrum_model
    with np.errstate(all="ignore"):
        ref = model(x, W, F, S)
    got = np.concatenate(got)
    assert got.shape == ref.shape and got.shape[0] > 0
    np.testing.assert_array_equal(got.view(np.uint32), ref.view(np.uint32))


def differing(ya, yb):
    """Indices where two float arrays differ bitwise (+0 / -0 equal)."""
    a, b = np.asarray(ya).view(F32).ravel(), np.asarray(yb).view(F32).ravel()
    same = (a == b) | (np.isnan(a) & np.isnan(b))
    return np.flatnonzero(~same)


@pytest.mark.parametrize("bad", [np.nan, np.inf], ids=["nan", "inf"])
def test_non_finite_sample_stays_local(pkg, bad):
    """One NaN or infinity in block 2 changes only a contiguous run of each client's outputs around the sample, no
    longer than its window allows, and only the spectrum row whose frames hold it; everything after is bit-exact."""
    rng = np.random.default_rng(11)
    n, n_blocks = 16384, 8
    blocks = [rng.standard_normal(2 * n).astype(F32) for _ in range(n_blocks)]
    p = 2 * n + 5001  # the sample's stream position
    bad_blocks = [v.copy() for v in blocks]
    bad_blocks[2][2 * 5001] = bad
    groups, outs = [], []
    for bl in (blocks, bad_blocks):
        g = pkg.Group(FS_MIX, 2 * n)
        r = np.random.default_rng(12)
        cl = {"generic": (g.add_client(5, rtaps(r, 40), 300000), 5, 40)}
        cl["tiled"] = ([g.add_client(32, rtaps(r, 97), 10000 * c) for c in range(8)][3], 32, 97)
        cl["long"] = ([g.add_client(1280, rtaps(r, 2561), 1000 * c) for c in range(8)][0], 1280, 2561)
        cl["cascade"] = (g.add_client_cascade(16, rtaps(r, 65), 200000, 4, rtaps(r, 33)), 64, 65 + 16 * 33)
        fid = g.add_bank_fft(16, rtaps(r, 257))
        cl["fft_bank_member"] = (g.add_client_subband(g.add_bank_subband(fid, 2), 4, rtaps(r, 33), 0), 64,
                                 257 + 16 * 33)
        sid = g.add_spectrum(1000, 4, 96, power=True)  # R = 4096
        o = {k: [] for k in cl}
        rows = []
        for v in bl:
            t = g.submit("cf32", v)
            g.wait(t)
            for k, (c, _, _) in cl.items():
                o[k].append(g.output(t, c))
            rows.append(g.read_spectrum(t, sid))
        outs.append((o, np.concatenate(rows)))
        groups.append(g)
    kinds = {k: groups[0].client_info(c)[1] for k, (c, _, _) in cl.items()}
    for g in groups:
        g.close()
    assert kinds["tiled"] == 1 and kinds["long"] == 2 and kinds["generic"] == 0, kinds
    (oa, ra), (ob, rb) = outs
    for k, (_, D, T) in cl.items():
        ya, yb = np.concatenate(oa[k]), np.concatenate(ob[k])
        d = np.unique(differing(ya, yb) // 2)
        assert d.size > 0, k
        assert d[0] * D >= p - T - D, (k, d[0])  # nothing before the sample's window
        assert d[-1] - d[0] + 1 == d.size and d.size <= T // D + 4, (k, d)  # one run, a window long
    d = differing(ra, rb)
    assert np.unique(d // 1000).tolist() == [p // 4096]


# ---------------------------------------------------------------------------
# 5. refusals
# ---------------------------------------------------------------------------
def test_refusals_take_no_ticket(pkg):
    torch = pytest.importorskip("torch")
    g = pkg.Group(FS_MIX, 4096)
    try:
        d = torch.zeros(2048, dtype=torch.complex64, device="cuda")
        with pytest.raises(RuntimeError, match=str(EINVAL)):
            g.submit_ptr(pkg.FMT["cf32"], d.data_ptr() + 4, 1024, pkg.XLG_INPUT_DEVICE)
        v = np.ones(1024, F32)
        with pytest.raises(RuntimeError, match=str(EINVAL)):
            g.submit("cf32", v, pkg.XLG_PATH_Q15)
        g.profile_enable(True)
        assert g.submit("cf32", v) == 0
        g.wait(0)
        prof = g.profile_read()
        assert prof["convert_launches"] == 1 and prof["in_samples"] == 512
        assert g.submit_ptr(pkg.FMT["cf32"], d.data_ptr() + 8, 1024, pkg.XLG_INPUT_DEVICE) == 1
        g.wait(1)
    finally:
        g.close()
