"""Wide spectrum rows (W = 8192, 16384, 32768 and 65536) on the GPU.

XLG_SPECTRUM_POWER rows must equal the model (tests/spectrum_wide.py: fft_rows at K = W) bit for bit: hops from
W / 8 to 3 W, no window, ones, Hann and random weights with negative entries, max and mean, S = 0, 1 and > W; every
input format; ragged, empty and sub-frame blocks, W = 65536 fed blocks of at most 8192 samples so that every frame
spans many blocks; band, client (tiled, rational, cascade), sub-band, direct and FFT bank channel sources, a
source's reference being its own outputs read back from the same group; the scratch and the mean's frame buffer
filled to their bound; device outputs, device and kept pinned inputs with XLG_SLOTS tickets in flight; and streams
past 2^31 and 2^32 samples.  Clients of every family, a plain and a Welch spectrum of W <= 4096 keep their outputs
bit for bit beside wide spectra; ids pass between wide and narrow widths and old tickets keep theirs; dB rows are
held to the power rows through log10f's documented error; refusals, info and the profile counters are checked.
"""
import ctypes as C
import errno

import numpy as np
import pytest

from exact import to_complex
from long_stream import N, Pump
from spectrum_exact import log10f_bound_db
from spectrum_welch import fbuf_frames, frames_done, hann, model_blocks
from spectrum_wide import WIDE_WIDTHS, wide_blocks
from util import rand_block

pytestmark = pytest.mark.gpu

FS = 2048000
MAX_IN = 2 * 8192
RAGGED = [8192, 8192, 2005, 0, 7, 8190, 8192, 333, 8192, 1, 8192, 8192, 6000, 8192]  # complex samples


def conv(fmt, raw):
    return to_complex(fmt, raw).astype(np.complex64)


def blocks_of(rng, fmt, sizes):
    return [rand_block(rng, fmt, 2 * n) for n in sizes]


def ragged_to(total):
    """RAGGED repeated until the sizes reach `total` samples."""
    sizes = []
    while sum(sizes) < total:
        sizes += RAGGED
    return sizes


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

    def refs(self, x, sizes, attach=0, power=True):
        """The model's rows per block (spectrum_welch's for the narrow widths some tests mix in)."""
        blocks = wide_blocks if self.W > 4096 else model_blocks
        return blocks(x, sizes, self.W, self.F, self.S, self.H or self.W, self.w, self.mean, attach=attach,
                      power=power)

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
    ref = sp.refs(x[:sum(sizes[:end])], sizes[:end], attach=sp.at)
    total = 0
    for b in range(sp.at, end):
        assert got[b].shape == ref[b].shape, f"{label} {sp} block {b}: {got[b].shape} rows, model {ref[b].shape}"
        np.testing.assert_array_equal(got[b].view(np.uint32), ref[b].view(np.uint32), err_msg=f"{label} {sp} b{b}")
        total += got[b].shape[0]
    return total


def hops(W):
    """W / 8, W / 4, W / 2, W - 1, W, W + 1, 3 W."""
    return [W // 8, W // 4, W // 2, W - 1, W, W + 1, 3 * W]


@pytest.mark.parametrize("W", WIDE_WIDTHS)
def test_widths_hops_windows(pkg, W):
    """Every hop of the width in one group, cycling through the windows, max and mean and the skip classes; the
    band arrives in blocks of at most 8192 samples, so at W = 65536 each frame spans at least eight of them."""
    rng = np.random.default_rng(W)
    blocks = blocks_of(rng, "cs16", ragged_to(6 * W))
    wins, skips = [None, "ones", "hann", "random"], [0, 1, W + 3]
    specs = []
    for i, H in enumerate(hops(W)):
        specs.append(Spec(W, 2, skips[i % 3], H, wins[i % 4], mean=i % 2 == 0))
        if H <= W:
            specs.append(Spec(W, 3, skips[(i + 1) % 3], H, wins[(i + 2) % 4], mean=i % 2 == 1))
    got = run(pkg, "cs16", blocks, specs)
    for sp, rows in zip(specs, got):
        assert check("cs16", blocks, sp, rows) > 0, sp


@pytest.mark.parametrize("fmt", ["cu8", "cs8", "cs16"])
def test_formats(pkg, fmt):
    rng = np.random.default_rng(7)
    blocks = blocks_of(rng, fmt, [3000, 63, 0, 8192, 1, 8192, 8192, 40, 5000, 8192, 8192, 64, 8191, 8192, 8192])
    specs = [Spec(8192, 3, 5, 2048, "hann", True), Spec(16384, 2, 0, 16384, "random", False),
             Spec(32768, 1, 1, None, None, True)]
    got = run(pkg, fmt, blocks, specs)
    for sp, rows in zip(specs, got):
        assert check(fmt, blocks, sp, rows, fmt) > 0


def test_plain_and_windowed_of_ones_agree(pkg):
    """A plain wide spectrum and the same one through xlg_add_spectrum_ex with a window of ones: the same rows."""
    rng = np.random.default_rng(13)
    blocks = blocks_of(rng, "cs16", ragged_to(3 * 65536))
    for W, F, S in ((8192, 2, 5), (65536, 1, 3)):
        got = run(pkg, "cs16", blocks, [Spec(W, F, S), Spec(W, F, S, W, "ones", False)])
        assert sum(r.shape[0] for r in got[0]) > 0
        for b, (a, c) in enumerate(zip(*got)):
            np.testing.assert_array_equal(a.view(np.uint32), c.view(np.uint32), err_msg=f"W={W} block {b}")
        assert check("cs16", blocks, Spec(W, F, S), got[0]) > 0


def test_attach_remove_churn_and_id_reuse(pkg):
    rng = np.random.default_rng(14)
    blocks = blocks_of(rng, "cs16", ragged_to(200000))
    specs = [Spec(16384, 1, 10, None, None, False, 0, 9),     # wide, removed: its id goes to the next one
             Spec(1000, 2, 0, 500, "hann", True, 9, 20),      # narrow on the wide's id, removed
             Spec(65536, 1, 0, 32768, "hann", True, 20, None),  # wide on the narrow's id
             Spec(8192, 2, 0, 4096, "random", True, 2, None),  # attached mid-stream
             Spec(64, 3, 1, None, None, False, 4, 25)]
    got = run(pkg, "cs16", blocks, specs)
    for sp, rows in zip(specs, got):
        assert check("cs16", blocks, sp, rows) > 0, sp


@pytest.mark.parametrize("flags", [0, 1])
def test_old_tickets_keep_their_width(pkg, flags):
    rng = np.random.default_rng(61)
    blocks = blocks_of(rng, "cs16", [65536] * 4)
    specs = [Spec(65536, 1, 0), Spec(1000, 2, 0, 500, "hann", True), Spec(16384, 2, 0, 8192, None, True),
             Spec(4096, 1, 0)]
    g = pkg.Group(FS, 2 * 65536, flags=pkg.XLG_OUT_DEVICE if flags else 0)
    try:
        g.reserve(1 << 18)
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
            ref = sp.refs(conv("cs16", x), [x.size // 2])[0]
            assert rows.shape == ref.shape and rows.shape[0] > 0
            np.testing.assert_array_equal(rows.view(np.uint32), ref.view(np.uint32), err_msg=str(sp))
    finally:
        g.close()


def client_outputs(pkg, blocks, with_wide):
    """Integer, rational, cascade, sub-band member and bank member clients, a plain and a Welch spectrum, and
    (with_wide) two wide spectra beside them."""
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
    plain = g.add_spectrum(1000, 2, 7, power=True)
    welch = g.add_spectrum(1024, 3, 0, power=True, hop=512, window=hann(1024), mean=True)
    wide = [g.add_spectrum(65536, 1, 0, power=True),
            g.add_spectrum(8192, 3, 0, power=True, hop=4096, window=hann(8192), mean=True)] if with_wide else []
    outs, rows = [], []
    try:
        for x in blocks:
            t = g.submit("cs16", x)
            g.wait(t)
            outs.append([g.output(t, c) for c in cids] + [g.read_spectrum(t, plain), g.read_spectrum(t, welch)])
            rows.append([g.read_spectrum(t, s) for s in wide])
    finally:
        g.close()
    return outs, rows


def test_clients_and_narrow_spectra_unchanged_beside(pkg):
    rng = np.random.default_rng(22)
    blocks = blocks_of(rng, "cs16", ragged_to(140000))
    without, _ = client_outputs(pkg, blocks, False)
    beside, rows = client_outputs(pkg, blocks, True)
    for b, (a, c) in enumerate(zip(without, beside)):
        for i, (ya, yc) in enumerate(zip(a, c)):
            np.testing.assert_array_equal(ya.view(np.uint32), yc.view(np.uint32), err_msg=f"block {b} output {i}")
    for k, sp in enumerate((Spec(65536, 1, 0), Spec(8192, 3, 0, 4096, "hann", True))):
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
        for k, sp in enumerate((Spec(8192, 2, 1, 4096, "hann", True), Spec(8192, 2, 70, 1024, "random", False),
                                Spec(16384, 1, 0, None, None, False))):
            add = g.add_client_spectrum if kind == 1 else g.add_subband_spectrum
            specs[(name, k)] = (sp, add(cid if kind == 1 else sbid, sp.W, sp.F, sp.S, power=True, hop=sp.H,
                                        window=sp.w, mean=sp.mean))
    band = Spec(65536, 2, 5, 16384, "hann", True)
    band_id = band.add(g)
    sizes = [65536, 8192, 2005, 0, 7, 1, 65536, 333, 40000, 65536, 65536, 65536, 65536, 30000, 65536, 65536]
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


@pytest.mark.parametrize("W,S,H,mean", [(8192, 0, 1024, True), (65536, 3, 8192, True), (32768, 0, 4096, False)])
def test_scratch_and_frame_buffer_bound_reached(pkg, W, S, H, mean):
    """A block of max_input_len / 2 samples that starts at a frame's last sample completes the most frames any
    block can: the scratch's rows (and a mean's frame buffer's), fbuf_frames(cap, W, S, H)."""
    max_in = 2 * 65536
    cap = max_in // 2
    F = 2 * fbuf_frames(cap, W, S, H) - 3
    rng = np.random.default_rng(W)
    sizes = [W - 1, cap, cap, cap, 5]
    blocks = blocks_of(rng, "cs16", sizes)
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


@pytest.mark.parametrize("mode", ["out_device", "input_device", "input_keep"])
def test_ingest_paths_with_tickets_in_flight(pkg, mode):
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(31)
    sizes = [8192, 5000, 0, 8192, 77, 8192, 8192, 4096, 8192, 8192, 8192, 8192, 1, 8192]
    blocks = blocks_of(rng, "cu8", sizes)
    specs = [Spec(8192, 4, 64, 2048, "hann", True), Spec(16384, 2, 2, 8191, "random", False), Spec(32768, 1, 0)]
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
    blocks = blocks_of(rng, "cs16", ragged_to(3 * 16384))
    for sp in (Spec(16384, 2, 0, 8192, "hann", True), Spec(8192, 2, 2, 1024, "random", False)):
        db = run(pkg, "cs16", blocks, [sp], power=False)[0]
        pw = run(pkg, "cs16", blocks, [sp], power=True)[0]
        assert sum(r.shape[0] for r in pw) > 0
        for b in range(len(blocks)):
            assert db[b].shape == pw[b].shape
            ref = 10 * np.log10(pw[b].astype(np.float64))
            assert np.all(np.abs(db[b] - ref) <= log10f_bound_db(pw[b])), (sp, b)


def ex(pkg, g, source=0, source_id=0, **kw):
    """xlg_add_spectrum_ex with a raw desc (fields as keywords); returns the code."""
    w = kw.pop("window", None)
    d = pkg.XlgSpectrumDesc(kw.get("width", 8192), kw.get("frames_per_row", 1), kw.get("skip_per_row", 0),
                            kw.get("flags", 0), kw.get("hop", 0), kw.get("reduce", 0),
                            None if w is None else w.ctypes.data_as(C.POINTER(C.c_float)))
    sid = C.c_int(-1)
    return g._L.xlg_add_spectrum_ex(g._h, source, source_id, C.byref(d), C.byref(sid))


def test_refusals_info_and_profile(pkg):
    EINVAL = -errno.EINVAL
    g = pkg.Group(FS, MAX_IN)
    try:
        cid = g.add_client(32, pkg.create_low_pass_filter(1.0, FS, 20000, 10000), 0)
        sb = g.add_subband(16, np.ones(16, np.float32) / 16, 0)
        for W in (0, 4097, 6144, 8191, 8193, 12288, 65535, 65537, 98304, 131072, 2 ** 31, 2 ** 32 - 1):
            assert ex(pkg, g, width=W) == EINVAL, W
            for add in (lambda: g._L.xlg_add_spectrum(g._h, W, 1, 0, 0, C.byref(C.c_int())),
                        lambda: g._L.xlg_add_client_spectrum(g._h, cid, W, 1, 0, 0, C.byref(C.c_int())),
                        lambda: g._L.xlg_add_subband_spectrum(g._h, sb, W, 1, 0, 0, C.byref(C.c_int()))):
                assert add() == EINVAL, W
        nan = np.ones(8192, np.float32)
        nan[5] = np.nan
        for kw in (dict(hop=1023), dict(window=nan), dict(reduce=2), dict(flags=2), dict(frames_per_row=0),
                   dict(width=65536, frames_per_row=2 ** 16, hop=2 ** 15)):
            assert ex(pkg, g, **kw) == EINVAL, kw
        assert g.client_count() == 1
        for W in WIDE_WIDTHS:  # every entry point, every source
            for s in (g.add_spectrum(W, 1), g.add_client_spectrum(cid, W, 1), g.add_subband_spectrum(sb, W, 1),
                      g.add_spectrum(W, 2, hop=W // 8, window=hann(W), mean=True),
                      g.add_client_spectrum(cid, W, 1, mean=True), g.add_subband_spectrum(sb, W, 1, hop=W // 2)):
                assert g.spectrum_info(s) == (2, 0), W
                g.remove_spectrum(s)
        assert g.spectrum_info(g.add_spectrum(4096, 1)) == (1, 0)
        g.remove_spectrum(0)
        s = g.add_spectrum(8192, 2, hop=4096, mean=True)
        with pytest.raises(RuntimeError, match=str(-errno.ENOTSUP)):
            g.submit("cs16", np.zeros(100, np.int16), pkg.XLG_PATH_Q15)
        g.remove_spectrum(s)
        # profile: a plain wide spectrum beside a windowed mean one
        a = g.add_spectrum(16384, 1, 3)
        b = g.add_spectrum(8192, 3, 1, hop=2048, window=hann(8192), mean=True)
        x = np.zeros(2 * 8000, np.int16)
        g.profile_enable(True)
        g.spectrum_profile_read()
        for _ in range(4):
            g.wait(g.submit("cs16", x))
        p = g.spectrum_profile_read()
        def done(n):
            return frames_done(n, 16384, 1, 3, 16384), frames_done(n, 8192, 3, 1, 2048)

        frames_a, frames_b = done(32000)
        assert (frames_a, frames_b) == (1, 6)
        assert p["spectrum_launches"] == sum(done(8000 * k) != done(8000 * (k + 1)) for k in range(4)) == 3
        assert p["frames"] == frames_a + frames_b
        assert p["channel_flops"] == frames_a * (pkg.bank_fft_flops(16384) + 6 * 16384) + \
            frames_b * (pkg.bank_fft_flops(8192) + 6 * 8192 + 2 * 8192 + 8192)
        assert g.spectrum_info(a) == (2, 1) and g.spectrum_info(b) == (2, 2)
    finally:
        g.close()
    g = pkg.Group(FS, MAX_IN, flags=pkg.XLG_TRACK_STATE)
    try:
        assert ex(pkg, g, width=65536) == -errno.ENOTSUP
        assert g._L.xlg_add_spectrum(g._h, 8192, 1, 0, 0, C.byref(C.c_int())) == -errno.ENOTSUP
    finally:
        g.close()


def test_long_stream_equals_fresh(pkg):
    """Rows after a block boundary B with (B - P) = 0 (mod R) are a fresh spectrum's attached at B, past 2^31 and
    2^32 samples."""
    torch = pytest.importorskip("torch")
    specs = [Spec(65536, 1, 0), Spec(8192, 2, 0, 4096, "hann", True), Spec(16384, 2, 0, 2048, "random", False)]
    lcm = 589824  # R = 65536, 12288, 18432
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
            assert p.S % lcm == 0 and p.S < target < p.S + 870007
            c0 = len(p.blocks)
            for off, n in ((0, 70000), (70000, 7), (70007, 0), (70007, 600000), (670007, 200000)):
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
