"""Windowed, overlapped and averaged spectrum rows (xlg_add_spectrum_ex) on the GPU.

XLG_SPECTRUM_POWER rows must equal the kernel model (tests/spectrum_welch.py) bit for bit on both channel stages:
widths from 1 to 4096, hops from ceil(W / 8) to 3 W, no window, ones, Hann and random weights with negative
entries, max and mean, every skip class and input format; ragged, odd, empty and sub-frame blocks, many rows per
block and one mean row across hundreds of blocks; band, client (tiled, rational, cascade), sub-band and bank
channel sources, a source's reference being its own outputs read back from the same group; the frame buffer
filled to its bound; device outputs, device and kept pinned inputs with XLG_SLOTS tickets in flight; and a mean
spectrum past 2^31 and 2^32 samples.  An extended spectrum with a window of ones, H = W and the max has a plain
spectrum's rows; a plain spectrum and every client keep their outputs bit for bit beside an extended one; ids are
shared with plain spectra.  dB rows are held to the power rows through log10f's documented error, and every
refusal and the profile counters are checked.
"""
import ctypes as C
import errno

import numpy as np
import pytest

from exact import to_complex
from long_stream import N, Pump
from spectrum_exact import log10f_bound_db, spec_fft
from spectrum_welch import fbuf_frames, hann, model_blocks
from util import rand_block

pytestmark = pytest.mark.gpu

FS = 2048000
MAX_IN = 2 * 8192
RAGGED = [8192, 8192, 2005, 0, 7, 8190, 8192, 333, 8192, 1, 8192, 8192, 6000, 8192]  # complex samples
SHORT = [8192, 100, 0, 5000, 1, 8192]


def conv(fmt, raw):
    return to_complex(fmt, raw).astype(np.complex64)


def blocks_of(rng, fmt, sizes):
    return [rand_block(rng, fmt, 2 * n) for n in sizes]


def window_of(kind, W, seed=0):
    if kind is None:
        return None
    if kind == "ones":
        return np.ones(W, np.float32)
    if kind == "hann":
        return hann(W)
    return np.random.default_rng(seed + W).uniform(-1.0, 1.5, W).astype(np.float32)


class Spec:
    """One spectrum of the band: W, F, S, hop H, window kind, mean, attach block, remove block (or None)."""

    def __init__(self, W, F, S=0, H=None, win=None, mean=False, at=0, rm=None):
        self.W, self.F, self.S, self.H, self.win, self.mean, self.at, self.rm = W, F, S, H, win, mean, at, rm
        self.w = window_of(win, W)

    def add(self, g, power=True):
        return g.add_spectrum(self.W, self.F, self.S, power=power, hop=self.H, window=self.w, mean=self.mean)

    def __repr__(self):
        return f"W={self.W} F={self.F} S={self.S} H={self.H} win={self.win} mean={self.mean}"


def run(pkg, fmt, blocks, specs, flags=0, max_in=MAX_IN, power=True):
    """Feed `blocks`, one ticket at a time; returns per spec the rows read per block (None outside its life)."""
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
    H = sp.W if sp.H is None else sp.H
    ref = model_blocks(x[:sum(sizes[:end])], sizes[:end], sp.W, sp.F, sp.S, H, sp.w, sp.mean, attach=sp.at)
    total = 0
    for b in range(sp.at, end):
        assert got[b].shape == ref[b].shape, f"{label} {sp} block {b}: {got[b].shape} rows, model {ref[b].shape}"
        np.testing.assert_array_equal(got[b].view(np.uint32), ref[b].view(np.uint32), err_msg=f"{label} {sp} b{b}")
        total += got[b].shape[0]
    return total


def hops(W):
    """ceil(W / 8), W / 4, W / 2, W - 1, W, W + 1, 3 W: the allowed, distinct ones."""
    hs = [-(-W // 8), W // 4, W // 2, W - 1, W, W + 1, 3 * W]
    return [h for i, h in enumerate(hs) if h >= 1 and 8 * h >= W and h not in hs[:i]]


@pytest.mark.parametrize("W", [1, 3, 4, 63, 64, 100, 1000, 1024, 4095, 4096])
def test_widths_hops_windows(pkg, W):
    """Every hop of the width in one group, cycling through the windows, max and mean and the skip classes."""
    rng = np.random.default_rng(W)
    big_direct = W >= 1000 and not spec_fft(W)
    blocks = blocks_of(rng, "cs16", SHORT if big_direct else RAGGED)
    wins, skips = [None, "ones", "hann", "random"], [0, 1, W + 3]
    specs = []
    for i, H in enumerate(hops(W)):
        if big_direct and i % 2:  # (the model's direct DFT is slow at these widths: every other hop)
            continue
        F = 2 if W >= 1000 else 3
        specs.append(Spec(W, F, skips[i % 3], H, wins[i % 4], mean=i % 2 == 0))
        specs.append(Spec(W, F, skips[(i + 1) % 3], H, wins[(i + 2) % 4], mean=i % 2 == 1))
    got = run(pkg, "cs16", blocks, specs)
    for sp, rows in zip(specs, got):
        assert check("cs16", blocks, sp, rows) > 0, sp


@pytest.mark.parametrize("fmt", ["cu8", "cs8", "cs16"])
def test_formats(pkg, fmt):
    rng = np.random.default_rng(7)
    blocks = blocks_of(rng, fmt, [3000, 63, 0, 8192, 1, 40, 5000, 8192, 64, 8191])
    specs = [Spec(64, 4, 5, 16, "hann", True), Spec(63, 3, 1, 40, "random", False), Spec(100, 2, 0, 150, None, True)]
    got = run(pkg, fmt, blocks, specs)
    for sp, rows in zip(specs, got):
        assert check(fmt, blocks, sp, rows, fmt) > 0


def test_many_rows_per_block(pkg):
    rng = np.random.default_rng(11)
    blocks = blocks_of(rng, "cs16", [8192, 8192, 4001])
    specs = [Spec(8, 2, 0, 1, "hann", True), Spec(16, 3, 0, 2, "random", False)]  # R = 9, 20
    got = run(pkg, "cs16", blocks, specs)
    assert [r.shape[0] for r in got[0]] == [910, 910, 445]
    for sp, rows in zip(specs, got):
        check("cs16", blocks, sp, rows)


def test_mean_row_across_hundreds_of_blocks(pkg):
    rng = np.random.default_rng(12)
    blocks = blocks_of(rng, "cu8", [100] * 800)
    specs = [Spec(64, 1200, 3, 32, "hann", True), Spec(100, 500, 7, 77, "random", True)]
    got = run(pkg, "cu8", blocks, specs, max_in=200)
    assert sum(r.shape[0] for r in got[0]) == 2  # R = 38435: 385 blocks per row
    for sp, rows in zip(specs, got):
        check("cu8", blocks, sp, rows)


def test_extended_path_equals_plain(pkg):
    """A window of ones, H = W and the max through the extended kernels: the plain spectrum's rows bit for bit."""
    rng = np.random.default_rng(13)
    blocks = blocks_of(rng, "cs16", RAGGED)
    for W, F, S in ((64, 2, 5), (1000, 1, 3), (4096, 2, 1), (3, 5, 2)):
        got = run(pkg, "cs16", blocks, [Spec(W, F, S), Spec(W, F, S, W, "ones", False)])
        assert sum(r.shape[0] for r in got[0]) > 0
        for b, (a, c) in enumerate(zip(*got)):
            np.testing.assert_array_equal(a.view(np.uint32), c.view(np.uint32), err_msg=f"W={W} block {b}")


def test_attach_remove_churn_and_id_reuse(pkg):
    rng = np.random.default_rng(14)
    blocks = blocks_of(rng, "cs16", RAGGED)
    specs = [Spec(64, 3, 10, None, None, False, 0, 4),     # plain, removed: its id goes to the next one
             Spec(100, 2, 0, 50, "hann", True, 4, 9),       # extended on the plain's id, removed
             Spec(64, 2, 0, None, None, False, 9, None),    # plain on the extended's id
             Spec(16, 5, 0, 4, "random", True, 2, None),    # attached mid-stream
             Spec(1024, 2, 1, 256, "hann", True, 6, 11)]
    got = run(pkg, "cs16", blocks, specs)
    for sp, rows in zip(specs, got):
        assert check("cs16", blocks, sp, rows) > 0, sp


@pytest.mark.parametrize("flags", [0, 1])
def test_old_tickets_keep_their_width(pkg, flags):
    rng = np.random.default_rng(61)
    blocks = blocks_of(rng, "cs16", [8192] * 3)
    specs = [Spec(1000, 1, 0), Spec(512, 2, 0, 256, "hann", True), Spec(2000, 1, 0, 1000, None, True)]
    g = pkg.Group(FS, MAX_IN, flags=pkg.XLG_OUT_DEVICE if flags else 0)
    try:
        g.reserve(1 << 16)
        tickets, sid = [], None
        for x, sp in zip(blocks, specs):
            if sid is not None:
                g.remove_spectrum(sid)
            sid = sp.add(g)
            assert sid == 0
            tickets.append(g.submit("cs16", x))
        for t, x, sp in zip(tickets, blocks, specs):
            assert g.spectrum_width(t, 0) == sp.W
            rows = g.read_spectrum(t, 0)
            ref = model_blocks(conv("cs16", x), [x.size // 2], sp.W, sp.F, sp.S, sp.H or sp.W, sp.w, sp.mean)[0]
            assert rows.shape == ref.shape and rows.shape[0] > 0
            np.testing.assert_array_equal(rows.view(np.uint32), ref.view(np.uint32), err_msg=str(sp))
    finally:
        g.close()


def client_outputs(pkg, blocks, with_ext):
    """Integer, rational, cascade, sub-band member and bank member clients and a plain spectrum, and (with_ext)
    a Welch spectrum beside them."""
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
    plain = g.add_spectrum(1000, 2, 7, power=True)
    ext = g.add_spectrum(1024, 3, 0, power=True, hop=512, window=hann(1024), mean=True) if with_ext else None
    outs, rows = [], []
    try:
        for x in blocks:
            t = g.submit("cs16", x)
            g.wait(t)
            outs.append([g.output(t, c) for c in cids] + [g.read_spectrum(t, plain)])
            if ext is not None:
                rows.append(g.read_spectrum(t, ext))
    finally:
        g.close()
    return outs, rows


def test_clients_and_plain_spectrum_unchanged_beside(pkg):
    rng = np.random.default_rng(22)
    blocks = blocks_of(rng, "cs16", RAGGED)
    without, _ = client_outputs(pkg, blocks, False)
    beside, rows = client_outputs(pkg, blocks, True)
    for b, (a, c) in enumerate(zip(without, beside)):
        for i, (ya, yc) in enumerate(zip(a, c)):
            np.testing.assert_array_equal(ya.view(np.uint32), yc.view(np.uint32), err_msg=f"block {b} output {i}")
    assert check("cs16", blocks, Spec(1024, 3, 0, 512, "hann", True), rows) > 0


def test_sources(pkg):
    """Client (tiled, rational, cascade), sub-band and bank channel sources; the reference stream of a sub-band
    or bank channel is a pass-through member's output."""
    def taps(rng, T):
        return (rng.standard_normal(T) / np.sqrt(T)).astype(np.float32)

    rng = np.random.default_rng(23)
    g = pkg.Group(FS, 2 * 65536)
    one = np.ones(1, np.float32)
    sb = g.add_subband(8, taps(rng, 64), 250000)
    bank_sb = g.add_bank_subband(g.add_bank(16, taps(rng, 200)), 5)
    src = {"tiled": (g.add_client(4, taps(rng, 129), -40000), 1, None),
           "rational": (g.add_client_rational(3, 8, taps(rng, 90), 50000), 1, None),
           "cascade": (g.add_client_cascade(2, taps(rng, 17), -20000, 2, taps(rng, 29), interp2=3), 1, None),
           "subband": (g.add_client_subband(sb, 1, one, 0), 2, sb),
           "bank": (g.add_client_subband(bank_sb, 1, one, 0), 2, bank_sb)}
    specs = {}
    for name, (cid, kind, sbid) in src.items():
        for k, sp in enumerate((Spec(64, 3, 1, 16, "hann", True), Spec(100, 2, 70, 101, "random", False),
                                Spec(1024, 2, 0, 512, "random", True))):
            add = g.add_client_spectrum if kind == 1 else g.add_subband_spectrum
            specs[(name, k)] = (sp, add(cid if kind == 1 else sbid, sp.W, sp.F, sp.S, power=True, hop=sp.H,
                                        window=sp.w, mean=sp.mean))
    sizes = [65536, 8192, 2005, 0, 7, 1, 65536, 333, 40000, 65536]
    outs = {n: [] for n in src}
    rows = {key: [] for key in specs}
    try:
        for x in blocks_of(rng, "cs16", sizes):
            t = g.submit("cs16", x)
            for n, (cid, _, _) in src.items():
                outs[n].append(g.read_output(t, cid))
            for key, (_, sid) in specs.items():
                rows[key].append(g.read_spectrum(t, sid))
    finally:
        g.close()
    for (name, k), (sp, _) in specs.items():
        ys = outs[name]
        ref = model_blocks(np.concatenate(ys), [len(y) for y in ys], sp.W, sp.F, sp.S, sp.H, sp.w, sp.mean)
        assert sum(r.shape[0] for r in ref) > 0, (name, sp)
        for b, (a, c) in enumerate(zip(rows[(name, k)], ref)):
            assert a.shape == c.shape, (name, sp, b)
            np.testing.assert_array_equal(a.view(np.uint32), c.view(np.uint32), err_msg=f"{name} {sp} block {b}")


@pytest.mark.parametrize("W,S,H", [(64, 0, 8), (100, 3, 13), (4096, 0, 512)])
def test_frame_buffer_bound_reached(pkg, W, S, H):
    """A block of max_input_len / 2 samples that starts at a frame's last sample completes the most frames any
    block can: the frame buffer's rows, fbuf_frames(cap, W, S, H)."""
    cap = MAX_IN // 2
    F = 2 * fbuf_frames(cap, W, S, H) - 3
    rng = np.random.default_rng(W)
    sizes = [W - 1, cap, cap, cap, 5]
    blocks = blocks_of(rng, "cs16", sizes)
    g = pkg.Group(FS, MAX_IN)
    frames, got = [], []
    try:
        sid = g.add_spectrum(W, F, S, power=True, hop=H, window=hann(W), mean=True)
        g.profile_enable(True)
        for x in blocks:
            g.spectrum_profile_read()
            t = g.submit("cs16", x)
            g.wait(t)
            frames.append(g.spectrum_profile_read()["frames"])
            got.append(g.read_spectrum(t, sid))
    finally:
        g.close()
    assert frames[1] == fbuf_frames(cap, W, S, H)
    assert check("cs16", blocks, Spec(W, F, S, H, "hann", True), got) >= 1


@pytest.mark.parametrize("mode", ["out_device", "input_device", "input_keep"])
def test_ingest_paths_with_tickets_in_flight(pkg, mode):
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(31)
    sizes = [8192, 5000, 0, 8192, 77, 8192, 8192, 4096, 8192]
    blocks = blocks_of(rng, "cu8", sizes)
    specs = [Spec(128, 4, 64, 32, "hann", True), Spec(63, 2, 2, 21, "random", False), Spec(64, 3, 0)]
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
    blocks = blocks_of(rng, "cs16", RAGGED)
    for sp in (Spec(64, 2, 0, 32, "hann", True), Spec(63, 2, 2, 9, "random", False)):
        db = run(pkg, "cs16", blocks, [sp], power=False)[0]
        pw = run(pkg, "cs16", blocks, [sp], power=True)[0]
        for b in range(len(blocks)):
            assert db[b].shape == pw[b].shape
            ref = 10 * np.log10(pw[b].astype(np.float64))
            assert np.all(np.abs(db[b] - ref) <= log10f_bound_db(pw[b])), (sp, b)


def ex(pkg, g, source=0, source_id=0, desc=None, **kw):
    """xlg_add_spectrum_ex with a raw desc (fields as keywords); returns the code."""
    d = None
    if desc is not False:
        w = kw.pop("window", None)
        d = pkg.XlgSpectrumDesc(kw.get("width", 64), kw.get("frames_per_row", 1), kw.get("skip_per_row", 0),
                                kw.get("flags", 0), kw.get("hop", 0), kw.get("reduce", 0),
                                None if w is None else w.ctypes.data_as(C.POINTER(C.c_float)))
    sid = C.c_int(-1)
    return g._L.xlg_add_spectrum_ex(g._h, source, source_id, None if d is None else C.byref(d), C.byref(sid))


def test_refusals_info_and_profile(pkg):
    EINVAL = -errno.EINVAL
    g = pkg.Group(FS, MAX_IN)
    try:
        cid = g.add_client(32, pkg.create_low_pass_filter(1.0, FS, 20000, 10000), 0)
        sb = g.add_subband(16, np.ones(16, np.float32) / 16, 0)
        nan = np.ones(64, np.float32)
        nan[5] = np.nan
        inf = np.ones(64, np.float32)
        inf[63] = -np.inf
        refused = [dict(desc=False), dict(source=3), dict(source=-1), dict(source=1, source_id=99),
                   dict(source=1, source_id=-1), dict(source=2, source_id=99), dict(source=2, source_id=-1),
                   dict(width=0), dict(width=4097), dict(frames_per_row=0), dict(flags=2), dict(reduce=2),
                   dict(hop=7), dict(width=4096, hop=511), dict(window=nan), dict(window=inf),
                   dict(width=4096, frames_per_row=2 ** 20, hop=2048), dict(frames_per_row=2, hop=2 ** 31),
                   dict(frames_per_row=2 ** 32 - 1, hop=2 ** 32 - 1, skip_per_row=2 ** 32 - 1)]
        for kw in refused:
            assert ex(pkg, g, **kw) == EINVAL, kw
        assert g.client_count() == 1
        code = g._L.xlg_add_spectrum(g._h, 64, 1, 0, 0x2, C.byref(C.c_int()))  # still an unknown flag
        assert code == EINVAL
        # the edges that are allowed: 8 H = W, R = 2^31 - 1, every source
        r_max = 2 ** 31 - 1 - 64  # (F - 1) H + S of R = 2^31 - 1 at W = 64, H = 8
        for kw in (dict(width=4096, hop=512), dict(hop=8, frames_per_row=r_max // 8 + 1, skip_per_row=r_max % 8),
                   dict(source=1, source_id=cid, reduce=1), dict(source=2, source_id=sb, hop=8)):
            assert ex(pkg, g, **kw) == 0, kw
        for s in range(4):
            g.remove_spectrum(s)
        for W in (1, 3, 4, 63, 64, 100, 1000, 1024, 4095, 4096):
            s = g.add_spectrum(W, 1, hop=W, window=hann(W))
            assert g.spectrum_info(s) == (1 if spec_fft(W) else 0, 0)
            g.remove_spectrum(s)
        s = g.add_spectrum(64, 2, hop=32, mean=True)
        with pytest.raises(RuntimeError, match=str(-errno.ENOTSUP)):
            g.submit("cs16", np.zeros(100, np.int16), pkg.XLG_PATH_Q15)
        g.remove_spectrum(s)
        # profile: a windowed mean spectrum beside a plain one
        a = g.add_spectrum(64, 2, 3)
        b = g.add_spectrum(100, 3, 1, hop=40, window=hann(100), mean=True)
        x = np.zeros(2 * 4000, np.int16)
        g.profile_enable(True)
        g.spectrum_profile_read()
        for _ in range(2):
            g.wait(g.submit("cs16", x))
        p = g.spectrum_profile_read()
        frames_a = 8000 // 131 * 2 + min(2, 8000 % 131 // 64)
        R = 2 * 40 + 100 + 1
        o = 8000 % R
        frames_b = 8000 // R * 3 + (0 if o < 100 else min(3, (o - 100) // 40 + 1))
        assert p["spectrum_launches"] == 2
        assert p["frames"] == frames_a + frames_b
        assert p["channel_flops"] == frames_a * (pkg.bank_fft_flops(64) + 6 * 64) + \
            frames_b * (4 * 100 ** 2 + 6 * 100 + 2 * 100 + 100)
        assert g.spectrum_info(b) == (0, 8000 // R * 1 + (1 if o >= 2 * 40 + 100 else 0))
    finally:
        g.close()
    g = pkg.Group(FS, MAX_IN, flags=pkg.XLG_TRACK_STATE)
    try:
        assert ex(pkg, g, hop=32, reduce=1) == -errno.ENOTSUP
        with pytest.raises(ValueError):
            g.add_spectrum(64, 2, hop=32)
    finally:
        g.close()


def test_long_stream_mean_equals_fresh(pkg):
    """Rows after a block boundary B with (B - P) = 0 (mod R) are a fresh spectrum's attached at B, past 2^31 and
    2^32 samples."""
    torch = pytest.importorskip("torch")
    specs = [Spec(64, 3, 0, 32, "hann", True), Spec(105, 2, 0, 35, "random", True), Spec(8, 1, 0, 1, None, True)]
    lcm = 4480  # R = 128, 140, 8
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
            p.run_to(target - 20000)
            gap = (target - 9000) // lcm * lcm - p.S
            while gap > 0:
                p.feed(None, 0, min(gap, N))
                gap -= min(gap, N)
            assert p.S % lcm == 0 and p.S < target < p.S + 20000
            c0 = len(p.blocks)
            for off, n in ((0, 4000), (4000, 7), (4007, 0), (4007, 9000), (13007, 5000)):
                p.watch.add(len(p.blocks))
                p.feed(0, off, n)
            p.drain()
            idx = range(c0, len(p.blocks))
            for k, sp in enumerate(specs):
                ref = model_blocks(np.concatenate([conv("cs16", p.blocks[i]) for i in idx]),
                                   [len(p.blocks[i]) // 2 for i in idx], sp.W, sp.F, sp.S, sp.H, sp.w, sp.mean)
                for j, i in enumerate(idx):
                    np.testing.assert_array_equal(got[i][k].view(np.uint32), ref[j].view(np.uint32),
                                                  err_msg=f"{target}: {sp} block {i}")
    finally:
        g.close()
