"""Chirp-z spectrum rows (xlg_add_spectrum_any: W above 4096 and not a power of two) on the GPU.

XLG_SPECTRUM_POWER rows must equal the model (tests/spectrum_czt.py, on the library's own tables) bit for bit: at
widths on both sides of every M boundary, hops from W / 8 to 3 W, no window, Hann and random weights, max and
mean, S = 0, 1 and > W; every input format; blocks far shorter than a frame; band, client (tiled, rational,
cascade), sub-band, direct and FFT bank channel sources; the scratches and the mean's frame buffer filled to their
bound; device outputs, device and kept pinned inputs with XLG_SLOTS tickets in flight; and streams past 2^31 and
2^32 samples.  xlg_add_spectrum_any equals xlg_add_spectrum_ex on the widths the latter serves.  Clients of every
family and plain, Welch and wide spectra keep their outputs bit for bit beside chirp-z spectra; ids pass between
kinds; dB rows are held to the power rows through log10f's documented error; refusals, info and the profile
counters are checked; bin/sdr_spectrogram -a matches the model's pixels.
"""
import ctypes as C
import errno
import functools
import os
import subprocess

import numpy as np
import pytest

from exact import to_complex
from long_stream import N, Pump
from spectrum_czt import CZT_WIDTHS, czt_blocks, czt_m, czt_model
from spectrum_exact import log10f_bound_db, read_png
from spectrum_welch import fbuf_frames, frames_done, hann, model_blocks
from spectrum_wide import wide_blocks
from util import rand_block

pytestmark = pytest.mark.gpu

FS = 2048000
MAX_IN = 2 * 8192
RAGGED = [8192, 8192, 2005, 0, 7, 8190, 8192, 333, 8192, 1, 8192, 8192, 6000, 8192]  # complex samples
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOOL = os.path.join(ROOT, "sdr-server_b200", "bin", "sdr_spectrogram")


@functools.lru_cache(maxsize=None)
def tables_of(W):
    import importlib
    return importlib.import_module("sdr-server_b200").spectrum_any_tables(W)


def conv(fmt, raw):
    if fmt == "cf32":
        return raw.view(np.complex64)
    return to_complex(fmt, raw).astype(np.complex64)


def block(rng, fmt, n):
    if fmt == "cf32":
        return (rng.standard_normal(2 * n) * 100).astype(np.float32)
    return rand_block(rng, fmt, 2 * n)


def blocks_of(rng, fmt, sizes):
    return [block(rng, fmt, n) for n in sizes]


def ragged_to(total):
    sizes = []
    while sum(sizes) < total:
        sizes += RAGGED
    return sizes


def window_of(kind, W, seed=0):
    if kind is None:
        return None
    if kind == "hann":
        return hann(W)
    return np.random.default_rng(seed + W).uniform(-1.0, 1.5, W).astype(np.float32)


class Spec:
    """One spectrum through xlg_add_spectrum_any: W, F, S, hop H, window kind, mean, attach and remove blocks."""

    def __init__(self, W, F, S=0, H=None, win=None, mean=False, at=0, rm=None):
        self.W, self.F, self.S, self.H, self.win, self.mean, self.at, self.rm = W, F, S, H, win, mean, at, rm
        self.w = window_of(win, W)

    def add(self, g, power=True):
        return g.add_spectrum(self.W, self.F, self.S, power=power, hop=self.H, window=self.w, mean=self.mean,
                              any_width=True)

    def refs(self, x, sizes, attach=0, power=True):
        H = self.H or self.W
        if self.W <= 4096:
            return model_blocks(x, sizes, self.W, self.F, self.S, H, self.w, self.mean, attach=attach, power=power)
        if self.W & (self.W - 1) == 0:
            return wide_blocks(x, sizes, self.W, self.F, self.S, H, self.w, self.mean, attach=attach, power=power)
        return czt_blocks(x, sizes, self.W, self.F, self.S, tables_of(self.W), H, self.w, self.mean, attach=attach,
                          power=power)

    def __repr__(self):
        return f"W={self.W} F={self.F} S={self.S} H={self.H} win={self.win} mean={self.mean}"


def run(pkg, fmt, blocks, specs, flags=0, max_in=MAX_IN, power=True):
    g = pkg.Group(FS, max_in, flags=flags)
    sids, got = {}, [[None] * len(blocks) for _ in specs]
    try:
        for b, x in enumerate(blocks):
            for i, sp in enumerate(specs):
                if sp.rm == b:
                    g.remove_spectrum(sids.pop(i))
                if sp.at == b:
                    sids[i] = sp.add(g, power)
            t = g.submit(fmt, x)
            for i, sid in sids.items():
                got[i][b] = g.read_spectrum(t, sid)
    finally:
        g.close()
    return got


def check(fmt, blocks, sp, got, label=""):
    x = np.concatenate([conv(fmt, r) for r in blocks])
    sizes = [len(r) // 2 for r in blocks]
    end = len(blocks) if sp.rm is None else sp.rm
    ref = sp.refs(x[:sum(sizes[:end])], sizes[:end], attach=sp.at)
    total = 0
    for b in range(sp.at, end):
        assert got[b].shape == ref[b].shape, f"{label} {sp} block {b}: {got[b].shape} rows, model {ref[b].shape}"
        np.testing.assert_array_equal(got[b].view(np.uint32), ref[b].view(np.uint32), err_msg=f"{label} {sp} b{b}")
        total += got[b].shape[0]
    return total


@pytest.mark.parametrize("W", CZT_WIDTHS)
def test_widths_hops_windows(pkg, W):
    """Hops ceil(W / 8) (the most overlap served), W / 2 - 1, W and 3 W (a gap between frames), the three windows,
    max and mean and the three skip classes in one group; the band arrives in blocks of at most 8192 samples, so a
    frame spans up to nine."""
    rng = np.random.default_rng(W)
    specs = [Spec(W, 2, 0, -(-W // 8), "hann", True), Spec(W, 2, 1, W // 2 - 1, "random", False),
             Spec(W, 1, W + 3, None, None, False), Spec(W, 2, 1, 3 * W, None, True)]
    blocks = blocks_of(rng, "cs16", ragged_to(3 * W + 7))
    got = run(pkg, "cs16", blocks, specs)
    for sp, rows in zip(specs, got):
        n = check("cs16", blocks, sp, rows)
        assert n > 0 or sp.H == 3 * W, sp


@pytest.mark.parametrize("fmt", ["cu8", "cs8", "cs16", "cf32"])
def test_formats(pkg, fmt):
    rng = np.random.default_rng(7)
    blocks = blocks_of(rng, fmt, [3000, 63, 0, 8192, 1, 8192, 8192, 40, 5000, 8192, 8192, 64, 8191, 8192])
    specs = [Spec(5000, 3, 5, 2500, "hann", True), Spec(8193, 2, 0, 4096, "random", False),
             Spec(12288, 1, 1, None, None, False)]
    got = run(pkg, fmt, blocks, specs)
    for sp, rows in zip(specs, got):
        assert check(fmt, blocks, sp, rows, fmt) > 0


# widths xlg_add_spectrum_ex serves: direct, FFT and wide paths
SERVED = [(1, 3, 0, None, None, False), (7, 4, 2, 3, "hann", True), (1000, 2, 1, 500, "random", True),
          (1024, 2, 0, None, None, False), (4096, 2, 3, 1024, "hann", False), (8192, 2, 0, 4096, "hann", True),
          (65536, 1, 0, None, None, False)]


def test_any_equals_ex_on_served_widths(pkg):
    rng = np.random.default_rng(3)
    blocks = blocks_of(rng, "cs16", ragged_to(2 * 65536 + 10))
    g_any, g_ex = pkg.Group(FS, MAX_IN), pkg.Group(FS, MAX_IN)
    try:
        ids = []
        for W, F, S, H, win, mean in SERVED:
            w = window_of(win, W)
            a = g_any.add_spectrum(W, F, S, power=True, hop=H, window=w, mean=mean, any_width=True)
            e = g_ex.add_spectrum(W, F, S, power=True, hop=H, window=w, mean=mean)
            assert g_any.spectrum_info(a) == g_ex.spectrum_info(e), W
            ids.append((a, e))
        total = 0
        for x in blocks:
            ta, te = g_any.submit("cs16", x), g_ex.submit("cs16", x)
            for a, e in ids:
                ra, re = g_any.read_spectrum(ta, a), g_ex.read_spectrum(te, e)
                np.testing.assert_array_equal(ra.view(np.uint32), re.view(np.uint32))
                total += ra.shape[0]
        assert total > 0
        for a, e in ids:
            assert g_any.spectrum_info(a) == g_ex.spectrum_info(e)
    finally:
        g_any.close()
        g_ex.close()


def test_attach_remove_churn_and_id_reuse(pkg):
    """Ids pass between chirp-z, wide, Welch and plain spectra."""
    rng = np.random.default_rng(14)
    blocks = blocks_of(rng, "cs16", ragged_to(120000))
    specs = [Spec(6000, 1, 10, None, None, False, 0, 5),     # chirp-z, removed: its id goes to the next one
             Spec(1000, 2, 0, 500, "hann", True, 5, 9),       # Welch on the chirp-z's id, removed
             Spec(10000, 2, 0, 5000, "hann", True, 9, None),  # chirp-z on the Welch's id
             Spec(16384, 1, 0, None, None, False, 2, 12),     # wide, attached mid-stream, removed
             Spec(48000, 1, 0, None, None, False, 12, None),  # chirp-z on the wide's id
             Spec(64, 3, 1, None, None, False, 4, None)]
    got = run(pkg, "cs16", blocks, specs)
    for sp, rows in zip(specs, got):
        assert check("cs16", blocks, sp, rows) > 0, sp


def client_outputs(pkg, blocks, with_czt):
    """Clients of every family, a plain, a Welch and a wide spectrum, and (with_czt) two chirp-z spectra."""
    def taps(rng, T):
        return (rng.standard_normal(T) / np.sqrt(T)).astype(np.float32)

    rng = np.random.default_rng(21)
    g = pkg.Group(FS, MAX_IN)
    lp = pkg.create_low_pass_filter(1.0, FS, 20000, 10000)
    cids = [g.add_client(32, lp, 100000), g.add_client_rational(3, 64, taps(rng, 301), -50000),
            g.add_client_cascade(8, taps(rng, 63), 200000, 4, taps(rng, 41))]
    sid = g.add_subband(16, taps(rng, 127), -300000)
    cids.append(g.add_client_subband(sid, 4, taps(rng, 33), 1000))
    bid = g.add_bank(16, taps(rng, 200))
    cids.append(g.add_client_subband(g.add_bank_subband(bid, 3), 2, taps(rng, 21), 0))
    fid = g.add_bank_fft(16, taps(rng, 200))
    cids.append(g.add_client_subband(g.add_bank_subband(fid, 5), 2, taps(rng, 21), 0))
    spectra = [g.add_spectrum(1000, 2, 7, power=True),
               g.add_spectrum(1024, 3, 0, power=True, hop=512, window=hann(1024), mean=True),
               g.add_spectrum(8192, 2, 0, power=True, hop=4096, window=hann(8192), mean=True)]
    czt = [g.add_spectrum(5000, 2, 0, power=True, any_width=True),
           g.add_spectrum(12288, 2, 0, power=True, hop=6144, window=hann(12288), mean=True, any_width=True)] \
        if with_czt else []
    outs, rows = [], []
    try:
        for x in blocks:
            t = g.submit("cs16", x)
            g.wait(t)
            outs.append([g.output(t, c) for c in cids] + [g.read_spectrum(t, s) for s in spectra])
            rows.append([g.read_spectrum(t, s) for s in czt])
    finally:
        g.close()
    return outs, rows


def test_clients_and_spectra_unchanged_beside(pkg):
    rng = np.random.default_rng(22)
    blocks = blocks_of(rng, "cs16", ragged_to(70000))
    without, _ = client_outputs(pkg, blocks, False)
    beside, rows = client_outputs(pkg, blocks, True)
    for b, (a, c) in enumerate(zip(without, beside)):
        for i, (ya, yc) in enumerate(zip(a, c)):
            np.testing.assert_array_equal(ya.view(np.uint32), yc.view(np.uint32), err_msg=f"block {b} output {i}")
    for k, sp in enumerate((Spec(5000, 2, 0), Spec(12288, 2, 0, 6144, "hann", True))):
        assert check("cs16", blocks, sp, [r[k] for r in rows]) > 0, sp


def test_sources(pkg):
    """Client (tiled, rational, cascade), sub-band, direct and FFT bank channel sources; the reference stream of a
    sub-band or bank channel is a pass-through member's output."""
    def taps(rng, T):
        return (rng.standard_normal(T) / np.sqrt(T)).astype(np.float32)

    rng = np.random.default_rng(23)
    g = pkg.Group(FS, 2 * 65536)
    one = np.ones(1, np.float32)
    sb = g.add_subband(8, taps(rng, 64), 250000)
    bank_sb = g.add_bank_subband(g.add_bank(16, taps(rng, 200)), 5)
    fft_sb = g.add_bank_subband(g.add_bank_fft(16, taps(rng, 300)), 7)
    src = {"tiled": (g.add_client(4, taps(rng, 129), -40000), 1, None),
           "rational": (g.add_client_rational(3, 8, taps(rng, 90), 50000), 1, None),
           "cascade": (g.add_client_cascade(2, taps(rng, 17), -20000, 2, taps(rng, 29), interp2=3), 1, None),
           "subband": (g.add_client_subband(sb, 1, one, 0), 2, sb),
           "bank": (g.add_client_subband(bank_sb, 1, one, 0), 2, bank_sb),
           "bank_fft": (g.add_client_subband(fft_sb, 1, one, 0), 2, fft_sb)}
    specs = {}
    for name, (cid, kind, sbid) in src.items():
        for k, sp in enumerate((Spec(6000, 2, 1, 3000, "hann", True), Spec(10000, 1, 70, None, "random", False))):
            add = g.add_client_spectrum if kind == 1 else g.add_subband_spectrum
            specs[(name, k)] = (sp, add(cid if kind == 1 else sbid, sp.W, sp.F, sp.S, power=True, hop=sp.H,
                                        window=sp.w, mean=sp.mean, any_width=True))
            assert g.spectrum_info(specs[(name, k)][1])[0] == 3
    band = Spec(48000, 2, 5, 24000, "hann", True)
    band_id = band.add(g)
    sizes = [65536, 8192, 2005, 0, 7, 1, 65536, 333, 40000, 65536, 65536, 65536, 30000, 65536]
    blocks = blocks_of(rng, "cs16", sizes)
    outs = {n: [] for n in src}
    rows = {key: [] for key in specs}
    band_rows = []
    try:
        for x in blocks:
            t = g.submit("cs16", x)
            for n, (cid, _, _) in src.items():
                outs[n].append(g.read_output(t, cid))
            for key, (_, sid) in specs.items():
                rows[key].append(g.read_spectrum(t, sid))
            band_rows.append(g.read_spectrum(t, band_id))
    finally:
        g.close()
    assert check("cs16", blocks, band, band_rows) > 0
    for (name, k), (sp, _) in specs.items():
        ys = outs[name]
        ref = sp.refs(np.concatenate(ys), [len(y) for y in ys])
        assert sum(r.shape[0] for r in ref) > 0, (name, sp)
        for b, (a, c) in enumerate(zip(rows[(name, k)], ref)):
            assert a.shape == c.shape, (name, sp, b)
            np.testing.assert_array_equal(a.view(np.uint32), c.view(np.uint32), err_msg=f"{name} {sp} block {b}")


@pytest.mark.parametrize("W,S,H,mean", [(5000, 0, 625, True), (12288, 3, 1536, False)])
def test_scratch_and_frame_buffer_bound_reached(pkg, W, S, H, mean):
    """A block of max_input_len / 2 samples that starts at a frame's last sample completes the most frames any
    block can: the scratches' rows (and a mean's frame buffer's), fbuf_frames(cap, W, S, H)."""
    max_in = 2 * 16384
    cap = max_in // 2
    F = 2 * fbuf_frames(cap, W, S, H) - 3
    rng = np.random.default_rng(W)
    blocks = blocks_of(rng, "cs16", [W - 1, cap, cap, 5])
    g = pkg.Group(FS, max_in)
    frames, got = [], []
    sp = Spec(W, F, S, H, "hann", mean)
    try:
        sid = sp.add(g)
        g.profile_enable(True)
        for x in blocks:
            g.spectrum_profile_read()
            t = g.submit("cs16", x)
            g.wait(t)
            frames.append(g.spectrum_profile_read()["frames"])
            got.append(g.read_spectrum(t, sid))
    finally:
        g.close()
    assert fbuf_frames(cap, W, S, H) >= 8
    assert frames[1] == fbuf_frames(cap, W, S, H)
    assert check("cs16", blocks, sp, got) >= 1


@pytest.mark.parametrize("mode", ["pageable", "out_device", "input_device", "input_keep"])
def test_ingest_paths_with_tickets_in_flight(pkg, mode):
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(31)
    sizes = [8192, 5000, 0, 8192, 77, 8192, 8192, 4096, 8192, 8192, 8192, 8192, 1, 8192]
    blocks = blocks_of(rng, "cu8", sizes)
    specs = [Spec(5000, 3, 64, 1250, "hann", True), Spec(8193, 2, 2, 8191, "random", False), Spec(32767, 1, 0)]
    g = pkg.Group(FS, MAX_IN, flags=pkg.XLG_OUT_DEVICE if mode == "out_device" else 0)
    sids = [sp.add(g) for sp in specs]
    got = [[None] * len(blocks) for _ in specs]
    keep = []
    try:
        pending = []
        for b, x in enumerate(blocks):
            if mode == "input_device":
                d = torch.from_numpy(x.copy()).cuda()
                torch.cuda.current_stream().synchronize()
                keep.append(d)
                t = g.submit_ptr(pkg.FMT["cu8"], d.data_ptr(), x.size, pkg.XLG_INPUT_DEVICE)
            elif mode == "input_keep":
                buf = pkg.PinnedBuffer(max(x.size, 1))
                buf.array(np.uint8)[:x.size] = x
                keep.append(buf)
                t = g.submit_ptr(pkg.FMT["cu8"], buf.ptr, x.size, pkg.XLG_INPUT_KEEP)
            else:
                t = g.submit("cu8", x)
            pending.append((t, b))
            if len(pending) == pkg.XLG_SLOTS:
                t0, b0 = pending.pop(0)
                for i, sid in enumerate(sids):
                    got[i][b0] = g.read_spectrum(t0, sid)
        for t0, b0 in pending:
            for i, sid in enumerate(sids):
                got[i][b0] = g.read_spectrum(t0, sid)
    finally:
        g.close()
    for sp, rows in zip(specs, got):
        assert check("cu8", blocks, sp, rows, mode) > 0


def test_db_rows_within_log10f_bound(pkg):
    rng = np.random.default_rng(41)
    blocks = blocks_of(rng, "cs16", ragged_to(3 * 6000))
    for sp in (Spec(6000, 2, 0, 3000, "hann", True), Spec(4097, 2, 2, 1024, "random", False)):
        db = run(pkg, "cs16", blocks, [sp], power=False)[0]
        pw = run(pkg, "cs16", blocks, [sp], power=True)[0]
        assert sum(r.shape[0] for r in pw) > 0
        for b in range(len(blocks)):
            assert db[b].shape == pw[b].shape
            ref = 10 * np.log10(pw[b].astype(np.float64))
            assert np.all(np.abs(db[b] - ref) <= log10f_bound_db(pw[b])), (sp, b)


def any_(pkg, g, source=0, source_id=0, **kw):
    """xlg_add_spectrum_any with a raw desc (fields as keywords); returns the code."""
    w = kw.pop("window", None)
    d = pkg.XlgSpectrumDesc(kw.get("width", 5000), kw.get("frames_per_row", 1), kw.get("skip_per_row", 0),
                            kw.get("flags", 0), kw.get("hop", 0), kw.get("reduce", 0),
                            None if w is None else w.ctypes.data_as(C.POINTER(C.c_float)))
    sid = C.c_int(-1)
    return g._L.xlg_add_spectrum_any(g._h, source, source_id, C.byref(d), C.byref(sid))


def czt_flops(pkg, W, window=False, mean=False):
    """The header's channel_flops of one chirp-z frame."""
    M = czt_m(W)
    return 2 * pkg.bank_fft_flops(M) + 4 * W + 4 * M + 6 * W + (2 * W if window else 0) + (W if mean else 0)


def test_refusals_info_and_profile(pkg):
    EINVAL = -errno.EINVAL
    g = pkg.Group(FS, MAX_IN)
    try:
        cid = g.add_client(32, pkg.create_low_pass_filter(1.0, FS, 20000, 10000), 0)
        sb = g.add_subband(16, np.ones(16, np.float32) / 16, 0)
        for W in (0, 65537, 98304, 131072, 2 ** 31, 2 ** 32 - 1):
            for source, source_id in ((0, 0), (1, cid), (2, sb)):
                assert any_(pkg, g, source, source_id, width=W) == EINVAL, W
        nan = np.ones(5000, np.float32)
        nan[5] = np.nan
        for kw in (dict(hop=624), dict(window=nan), dict(reduce=2), dict(flags=2), dict(frames_per_row=0),
                   dict(width=48000, frames_per_row=2 ** 16, hop=2 ** 15)):
            assert any_(pkg, g, **kw) == EINVAL, kw
        assert any_(pkg, g, 1, 99) == EINVAL and any_(pkg, g, 2, 99) == EINVAL and any_(pkg, g, 3, 0) == EINVAL
        with pytest.raises(ValueError):  # nothing was attached
            g.spectrum_info(0)
        assert g.client_count() == 1
        # the first ticket is the first a twin group without the refusals hands out
        twin = pkg.Group(FS, MAX_IN)
        try:
            assert g.submit("cs16", np.zeros(64, np.int16)) == twin.submit("cs16", np.zeros(64, np.int16))
        finally:
            twin.close()
        for W in (4097, 6144, 8191, 12288, 65535):  # every source, with and without the Welch parameters
            for s in (g.add_spectrum(W, 1, any_width=True), g.add_client_spectrum(cid, W, 1, any_width=True),
                      g.add_subband_spectrum(sb, W, 1, any_width=True),
                      g.add_spectrum(W, 2, hop=-(-W // 8), window=hann(W), mean=True, any_width=True)):
                assert g.spectrum_info(s) == (3, 0), W
                g.remove_spectrum(s)
        for W, kind in ((4096, 1), (1000, 0), (8192, 2), (65536, 2)):
            s = g.add_spectrum(W, 1, any_width=True)
            assert g.spectrum_info(s) == (kind, 0), W
            g.remove_spectrum(s)
        s = g.add_spectrum(5000, 2, hop=2500, mean=True, any_width=True)
        with pytest.raises(RuntimeError, match=str(-errno.ENOTSUP)):
            g.submit("cs16", np.zeros(100, np.int16), pkg.XLG_PATH_Q15)
        g.remove_spectrum(s)
        # profile: a plain chirp-z spectrum beside a windowed mean one
        a = g.add_spectrum(6000, 1, 3, any_width=True)
        b = g.add_spectrum(5000, 3, 1, hop=1250, window=hann(5000), mean=True, any_width=True)
        x = np.zeros(2 * 8000, np.int16)
        g.profile_enable(True)
        g.spectrum_profile_read()
        for _ in range(4):
            g.wait(g.submit("cs16", x))
        p = g.spectrum_profile_read()

        def done(n):
            return frames_done(n, 6000, 1, 3, 6000), frames_done(n, 5000, 3, 1, 1250)

        frames_a, frames_b = done(32000)
        assert (frames_a, frames_b) == (5, 12)
        assert p["spectrum_launches"] == 4
        assert p["frames"] == frames_a + frames_b
        assert p["channel_flops"] == frames_a * czt_flops(pkg, 6000) + frames_b * czt_flops(pkg, 5000, True, True)
        assert g.spectrum_info(a) == (3, 5) and g.spectrum_info(b) == (3, 4)
    finally:
        g.close()
    g = pkg.Group(FS, MAX_IN, flags=pkg.XLG_TRACK_STATE)
    try:
        assert any_(pkg, g, width=5000) == -errno.ENOTSUP
    finally:
        g.close()


def test_long_stream_equals_fresh(pkg):
    """Rows after a block boundary B with (B - P) = 0 (mod R) are a fresh spectrum's attached at B, past 2^31 and
    2^32 samples."""
    torch = pytest.importorskip("torch")
    specs = [Spec(6144, 1, 0), Spec(12288, 2, 0, 6144, "hann", True), Spec(36864, 1, 0, None, "random", False)]
    lcm = 36864  # R = 6144, 18432, 36864
    rng = np.random.default_rng(51)
    bufs = [rand_block(rng, "cs16", 2 * N) for _ in range(3)]
    g = pkg.Group(FS, 2 * N)
    sids = [sp.add(g) for sp in specs]
    got = {}

    def read(t, i):
        got[i] = [g.read_spectrum(t, s) for s in sids]

    p = Pump(torch, pkg, g, "cs16", bufs, 52, read=read)
    try:
        for target in (2 ** 31, 2 ** 32):
            p.run_to(target - 2000000)
            gap = (target - 250000) // lcm * lcm - p.S
            while gap > 0:
                p.feed(None, 0, min(gap, N))
                gap -= min(gap, N)
            assert p.S % lcm == 0 and p.S < target < p.S + 470007
            c0 = len(p.blocks)
            for off, n in ((0, 70000), (70000, 7), (70007, 0), (70007, 300000), (370007, 100000)):
                p.watch.add(len(p.blocks))
                p.feed(0, off, n)
            p.drain()
            idx = range(c0, len(p.blocks))
            x = np.concatenate([conv("cs16", p.blocks[i]) for i in idx])
            for k, sp in enumerate(specs):
                ref = sp.refs(x, [len(p.blocks[i]) // 2 for i in idx])
                assert sum(r.shape[0] for r in ref) > 0
                for j, i in enumerate(idx):
                    np.testing.assert_array_equal(got[i][k].view(np.uint32), ref[j].view(np.uint32),
                                                  err_msg=f"{target}: {sp} block {i}")
    finally:
        g.close()


# ---------------------------------------------------------------------------
# bin/sdr_spectrogram -a
# ---------------------------------------------------------------------------
_LIBM = C.CDLL("libm.so.6")
_LIBM.log10f.restype = C.c_float
_LIBM.log10f.argtypes = [C.c_float]


def tool_pixels(pkg, rows):
    """The tool's pixels of power rows: 10 * log10f(v) in float with the C library's log10f, then the reference's
    clamp (spectrogram_pixels)."""
    v = np.asarray(rows, np.float32)
    lg = np.array([_LIBM.log10f(float(a)) for a in v.ravel()], np.float32).reshape(v.shape)
    return pkg.spectrogram_pixels(np.float32(10) * lg)


def run_tool(*args):
    return subprocess.run([TOOL, *map(str, args)], capture_output=True, text=True, timeout=600)


@pytest.mark.parametrize("W,fmt,fs,n", [(5000, "cs16", 100000, 300_007), (48000, "cu8", 48000, 150_001)])
def test_tool_any_width_against_model(pkg, tmp_path, W, fmt, fs, n):
    rng = np.random.default_rng(W)
    raw = rand_block(rng, fmt, 2 * n)
    x = to_complex(fmt, raw).astype(np.complex64)
    src, out = tmp_path / f"in.{fmt}", tmp_path / "out.png"
    src.write_bytes(raw.astype({"cu8": np.uint8, "cs16": "<i2"}[fmt]).tobytes())
    r = run_tool("-a", "-w", W, "-s", fs, "-d", fmt, "-i", src, "-o", out)
    src.unlink()
    assert r.returncode == 0, r.stderr
    F, S = pkg.spectrogram_params(fs, W)
    height = n // fs
    rows = czt_model(x[:height * fs], W, F, S, tables_of(W))
    assert rows.shape == (height, W)
    got = read_png(out)
    assert got.shape == (height, W)
    np.testing.assert_array_equal(got, tool_pixels(pkg, rows))


@pytest.mark.parametrize("W,fs", [(1000, 12345), (1024, 100000), (4096, 250000)])
def test_tool_any_width_same_png_where_served(tmp_path, W, fs):
    rng = np.random.default_rng(W)
    src = tmp_path / "in.cs16"
    src.write_bytes(rand_block(rng, "cs16", 2 * (2 * fs + 17)).astype("<i2").tobytes())
    outs = []
    for flag in ([], ["-a"]):
        out = tmp_path / f"out{len(flag)}.png"
        r = run_tool(*flag, "-w", W, "-s", fs, "-d", "cs16", "-i", src, "-o", out)
        assert r.returncode == 0, r.stderr
        outs.append(out.read_bytes())
    assert outs[0] == outs[1]
