"""Spectrum rows (xlg_add_spectrum) on the GPU.

XLG_SPECTRUM_POWER rows must equal the kernel model (tests/spectrum_exact.py) bit for bit, on both channel
stages, at widths from 1 to 4096, with and without skip, on every input format, through ragged, odd, empty and
sub-frame blocks, many rows per block and one row across hundreds of blocks, attach mid-stream, removal and
re-adding, two spectra in one group, device outputs, device and kept pinned inputs with XLG_SLOTS tickets in
flight, and past 2^31 and 2^32 stream samples.  Clients of every family keep their outputs bit for bit beside
a spectrum.  dB rows are held to the model's power through log10f's documented error, and a group at fs = 128
fed the reference's own stimuli reproduces its spectrogram goldens pixel for pixel.
"""
import ctypes as C
import errno

import numpy as np
import pytest

from exact import to_complex
from long_stream import N, Pump
from spectrum_exact import (GOLDEN_DIR, GOLDEN_FS, GOLDENS, golden_stimulus, log10f_bound_db, model_blocks,
                            read_png, spec_fft)
from util import rand_block

pytestmark = pytest.mark.gpu

FS = 2048000
MAX_IN = 2 * 8192
RAGGED = [8192, 8192, 2005, 0, 7, 8190, 8192, 333, 8192, 1, 8192, 8192, 6000, 8192]  # complex samples


def conv(fmt, raw):
    return to_complex(fmt, raw).astype(np.complex64)


def blocks_of(rng, fmt, sizes):
    return [rand_block(rng, fmt, 2 * n) for n in sizes]


def run(pkg, fmt, blocks, specs, flags=0, max_in=MAX_IN, power=True):
    """Feed `blocks`, one ticket at a time; specs: list of (W, F, S, attach block, remove block or None).
    Returns per spec the rows read per block (None outside its life)."""
    g = pkg.Group(FS, max_in, flags=flags)
    sids, got = {}, [[None] * len(blocks) for _ in specs]
    try:
        for b, x in enumerate(blocks):
            for i, (W, F, S, at, rm) in enumerate(specs):
                if rm == b:
                    g.remove_spectrum(sids.pop(i))
                if at == b:
                    sids[i] = g.add_spectrum(W, F, S, power=power)
            t = g.submit(fmt, x)
            for i, sid in sids.items():
                got[i][b] = g.read_spectrum(t, sid)
    finally:
        g.close()
    return got


def check(fmt, blocks, spec, got, label=""):
    W, F, S, at, rm = spec
    x = np.concatenate([conv(fmt, r) for r in blocks])
    sizes = [len(r) // 2 for r in blocks]
    end = len(blocks) if rm is None else rm
    ref = model_blocks(x[:sum(sizes[:end])], sizes[:end], W, F, S, attach=at)
    total = 0
    for b in range(at, end):
        assert got[b].shape == ref[b].shape, f"{label} block {b}: {got[b].shape} rows, model {ref[b].shape}"
        np.testing.assert_array_equal(got[b].view(np.uint32), ref[b].view(np.uint32), err_msg=f"{label} block {b}")
        total += got[b].shape[0]
    return total


# (W, F, S): every width of both channel stages, F = 1, S in {0, 1, W - 1, > W}, rows longer than a block
WIDTHS = [(1, 1, 0), (2, 1, 1), (3, 5, 2), (4, 1, 3), (8, 7, 9), (63, 2, 2), (64, 2, 0), (100, 3, 101),
          (128, 1, 127), (1000, 1, 0), (1024, 20, 5), (4096, 3, 1)]


@pytest.mark.parametrize("W,F,S", WIDTHS)
def test_rows_bit_exact(pkg, W, F, S):
    rng = np.random.default_rng(W)
    blocks = blocks_of(rng, "cs16", RAGGED)
    spec = (W, F, S, 0, None)
    got = run(pkg, "cs16", blocks, [spec])
    assert check("cs16", blocks, spec, got[0], f"W={W}") > 0


@pytest.mark.parametrize("W,F,S", [(3000, 2, 1), (4095, 1, 3)])
def test_wide_direct_rows_bit_exact(pkg, W, F, S):
    """The direct path above 48 KiB of shared memory (16 W bytes) and with up to 16 CTAs per frame."""
    rng = np.random.default_rng(W)
    blocks = blocks_of(rng, "cs16", [8192, 100, 0, 8192, 5000])
    spec = (W, F, S, 0, None)
    got = run(pkg, "cs16", blocks, [spec])
    assert check("cs16", blocks, spec, got[0], f"W={W}") > 0


@pytest.mark.parametrize("flags", [0, 1])
def test_old_tickets_keep_their_width(pkg, flags):
    """An id removed and added again with a smaller, then a larger width: tickets submitted before each change
    still return their own rows, at their own width, with XLG_SLOTS tickets outstanding."""
    rng = np.random.default_rng(61)
    blocks = blocks_of(rng, "cs16", [8192] * 3)
    widths = [1000, 512, 2000]
    g = pkg.Group(FS, MAX_IN, flags=pkg.XLG_OUT_DEVICE if flags else 0)
    try:
        g.reserve(1 << 16)  # no arena growth between the submits
        tickets, sid = [], None
        for x, W in zip(blocks, widths):
            if sid is not None:
                g.remove_spectrum(sid)
            sid = g.add_spectrum(W, 1, 0, power=True)
            assert sid == 0
            tickets.append(g.submit("cs16", x))
        for t, x, W in zip(tickets, blocks, widths):
            assert g.spectrum_width(t, 0) == W
            rows = g.read_spectrum(t, 0)
            ref = model_blocks(conv("cs16", x), [x.size // 2], W, 1, 0)[0]
            assert rows.shape == ref.shape == (8192 // W, W)
            np.testing.assert_array_equal(rows.view(np.uint32), ref.view(np.uint32), err_msg=f"W={W}")
        with pytest.raises(ValueError):
            g.spectrum_width(tickets[-1], 1)
    finally:
        g.close()


@pytest.mark.parametrize("fmt", ["cu8", "cs8", "cs16"])
def test_formats_and_two_spectra(pkg, fmt):
    rng = np.random.default_rng(7)
    blocks = blocks_of(rng, fmt, [3000, 63, 0, 8192, 1, 40, 5000, 8192, 64, 8191])
    specs = [(64, 2, 5, 0, None), (63, 3, 1, 0, None)]
    got = run(pkg, fmt, blocks, specs)
    for spec, rows in zip(specs, got):
        assert check(fmt, blocks, spec, rows, f"{fmt} W={spec[0]}") > 0


def test_many_rows_per_block(pkg):
    rng = np.random.default_rng(11)
    blocks = blocks_of(rng, "cs16", [8192, 8192, 4001])
    spec = (4, 1, 0, 0, None)
    got = run(pkg, "cs16", blocks, [spec])
    assert [r.shape[0] for r in got[0]] == [2048, 2048, 1000]
    check("cs16", blocks, spec, got[0])


def test_row_across_hundreds_of_blocks(pkg):
    rng = np.random.default_rng(12)
    blocks = blocks_of(rng, "cu8", [100] * 800)
    spec = (64, 600, 3, 0, None)  # R = 38403 samples: 384 blocks per row
    got = run(pkg, "cu8", blocks, [spec], max_in=200)
    assert sum(r.shape[0] for r in got[0]) == 2
    check("cu8", blocks, spec, got[0])


def test_attach_remove_readd(pkg):
    rng = np.random.default_rng(13)
    blocks = blocks_of(rng, "cs16", RAGGED)
    specs = [(64, 3, 10, 3, 6), (100, 2, 0, 6, None), (16, 5, 0, 0, None)]  # spectrum 1 re-uses spectrum 0's id
    got = run(pkg, "cs16", blocks, specs)
    for i, spec in enumerate(specs):
        assert check("cs16", blocks, spec, got[i], f"spectrum {i}") > 0


def client_outputs(pkg, blocks, with_spectrum):
    """Integer, rational, cascade, sub-band member and bank member clients (and a spectrum) on one group."""
    def fft_taps(rng, T):
        return (rng.standard_normal(T) / np.sqrt(T)).astype(np.float32)

    rng = np.random.default_rng(21)
    g = pkg.Group(FS, MAX_IN)
    lp = pkg.create_low_pass_filter(1.0, FS, 20000, 10000)
    cids = [g.add_client(32, lp, 100000), g.add_client_rational(3, 64, fft_taps(rng, 301), -50000),
            g.add_client_cascade(8, fft_taps(rng, 63), 200000, 4, fft_taps(rng, 41))]
    sid = g.add_subband(16, fft_taps(rng, 127), -300000)
    cids.append(g.add_client_subband(sid, 4, fft_taps(rng, 33), 1000))
    bid = g.add_bank(16, fft_taps(rng, 200))
    cids.append(g.add_client_subband(g.add_bank_subband(bid, 3), 2, fft_taps(rng, 21), 0))
    spec = g.add_spectrum(1000, 2, 7, power=True) if with_spectrum else None
    outs, rows = [], []
    try:
        for x in blocks:
            t = g.submit("cs16", x)
            g.wait(t)
            outs.append([g.output(t, c) for c in cids])
            if spec is not None:
                rows.append(g.read_spectrum(t, spec))
        assert g.client_count() == len(cids)
    finally:
        g.close()
    return outs, rows


def test_clients_unchanged_beside_a_spectrum(pkg):
    rng = np.random.default_rng(22)
    blocks = blocks_of(rng, "cs16", RAGGED)
    without, _ = client_outputs(pkg, blocks, False)
    beside, rows = client_outputs(pkg, blocks, True)
    for b, (a, c) in enumerate(zip(without, beside)):
        for i, (ya, yc) in enumerate(zip(a, c)):
            np.testing.assert_array_equal(ya.view(np.uint32), yc.view(np.uint32), err_msg=f"block {b} client {i}")
    check("cs16", blocks, (1000, 2, 7, 0, None), rows)


@pytest.mark.parametrize("mode", ["out_device", "input_device", "input_keep"])
def test_ingest_paths_with_tickets_in_flight(pkg, mode):
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(31)
    sizes = [8192, 5000, 0, 8192, 77, 8192, 8192, 4096, 8192]
    blocks = blocks_of(rng, "cu8", sizes)
    specs = [(128, 4, 64, 0, None), (63, 2, 2, 0, None)]
    flags = pkg.XLG_OUT_DEVICE if mode == "out_device" else 0
    g = pkg.Group(FS, MAX_IN, flags=flags)
    sids = [g.add_spectrum(W, F, S, power=True) for W, F, S, _, _ in specs]
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
            if len(pending) == pkg.XLG_SLOTS:  # XLG_SLOTS tickets in flight before the oldest is read
                t0, b0 = pending.pop(0)
                for i, sid in enumerate(sids):
                    got[i][b0] = g.read_spectrum(t0, sid)
        for t0, b0 in pending:
            for i, sid in enumerate(sids):
                got[i][b0] = g.read_spectrum(t0, sid)
    finally:
        g.close()
    for spec, rows in zip(specs, got):
        assert check("cu8", blocks, spec, rows, mode) > 0


def test_info_refusals_and_profile(pkg):
    g = pkg.Group(FS, MAX_IN)
    try:
        for W in (1, 2, 3, 4, 8, 63, 64, 100, 1000, 1024, 4095, 4096):
            sid = g.add_spectrum(W, 1)
            assert g.spectrum_info(sid) == (1 if spec_fft(W) else 0, 0)
            g.remove_spectrum(sid)
        for W, F, S, flags in ((0, 1, 0, 0), (4097, 1, 0, 0), (64, 0, 0, 0), (4096, 524288, 0, 0),
                               (1, 2 ** 31 - 1, 1, 0)):
            with pytest.raises(ValueError) as e:
                g.add_spectrum(W, F, S)
            assert e.value.args[0] == -errno.EINVAL, (W, F, S)
        code = g._L.xlg_add_spectrum(g._h, 64, 1, 0, 0x2, C.byref(C.c_int()))  # an unknown flag
        assert code == -errno.EINVAL
        sid = g.add_spectrum(4096, 524287, 4095)  # R = 2^31 - 1
        g.remove_spectrum(sid)
        with pytest.raises(ValueError):
            g.remove_spectrum(sid)
        with pytest.raises(ValueError):
            g.spectrum_info(sid)
        a, b = g.add_spectrum(64, 2, 3), g.add_spectrum(100, 1)
        assert g.client_count() == 0
        x = np.zeros(2 * 4000, np.int16)
        with pytest.raises(RuntimeError, match=str(-errno.ENOTSUP)):
            g.submit("cs16", x, pkg.XLG_PATH_Q15)
        g.profile_enable(True)
        g.profile_read()
        g.spectrum_profile_read()
        t = g.submit("cs16", x)
        assert t == 0  # the refused Q15 submit took no ticket
        g.wait(t)
        t = g.submit("cs16", x)
        g.wait(t)
        p = g.spectrum_profile_read()
        frames_a, frames_b = 8000 // 131 * 2 + min(2, 8000 % 131 // 64), 80
        assert p["spectrum_launches"] == 2 and p["spectrum_ms"] > 0
        assert p["frames"] == frames_a + frames_b
        assert p["channel_flops"] == frames_a * (pkg.bank_fft_flops(64) + 6 * 64) + frames_b * (4 * 100 ** 2 + 600)
        assert g.spectrum_info(a)[1] == 8000 // 131 + (1 if 8000 % 131 >= 128 else 0)
        assert g.spectrum_info(b) == (0, 80)
        with pytest.raises(ValueError):
            g.spectrum_rows(t, 7)
    finally:
        g.close()
    g = pkg.Group(FS, MAX_IN, flags=pkg.XLG_TRACK_STATE)
    try:
        with pytest.raises(ValueError) as e:
            g.add_spectrum(64, 1)
        assert e.value.args[0] == -errno.ENOTSUP
    finally:
        g.close()


def test_db_rows_within_log10f_bound(pkg):
    rng = np.random.default_rng(41)
    blocks = blocks_of(rng, "cs16", RAGGED)
    for W, F, S in ((64, 2, 0), (63, 2, 2), (1024, 1, 3)):
        db = run(pkg, "cs16", blocks, [(W, F, S, 0, None)], power=False)[0]
        pw = run(pkg, "cs16", blocks, [(W, F, S, 0, None)], power=True)[0]
        for b in range(len(blocks)):
            assert db[b].shape == pw[b].shape
            ref = 10 * np.log10(pw[b].astype(np.float64))
            assert np.all(np.abs(db[b] - ref) <= log10f_bound_db(pw[b])), (W, b)


@pytest.mark.parametrize("name", ["spectrogram_cu8.png", "spectrogram_cs16.png"])
@pytest.mark.parametrize("cuts", [[256], [100, 0, 1, 155]])
def test_golden_pixels(pkg, name, cuts):
    fmt, W = GOLDENS[name]
    F, S = pkg.spectrogram_params(GOLDEN_FS, W)
    raw = golden_stimulus(fmt)
    g = pkg.Group(GOLDEN_FS, 512)
    rows = []
    try:
        sid = g.add_spectrum(W, F, S)
        pos = 0
        for n in cuts:
            t = g.submit(fmt, raw[2 * pos:2 * (pos + n)])
            rows.append(g.read_spectrum(t, sid))
            pos += n
    finally:
        g.close()
    np.testing.assert_array_equal(pkg.spectrogram_pixels(np.concatenate(rows)), read_png(f"{GOLDEN_DIR}/{name}"))


def test_long_stream_rows_equal_fresh(pkg):
    """Rows after a block boundary B with (B - P) = 0 (mod R) are a fresh spectrum's attached at B, past 2^31
    and 2^32 samples (W = 1: more than 2^32 rows and frames)."""
    torch = pytest.importorskip("torch")
    specs = [(64, 3, 0), (105, 2, 0), (1, 1, 0)]  # R = 192, 210, 1: all divide N
    lcm = 6720
    rng = np.random.default_rng(51)
    bufs = [rand_block(rng, "cs16", 2 * N) for _ in range(3)]
    g = pkg.Group(FS, 2 * N)
    sids = [g.add_spectrum(W, F, S, power=True) for W, F, S in specs]
    got = {}

    def read(t, i):
        got[i] = [g.read_spectrum(t, s) for s in sids]

    p = Pump(torch, pkg, g, "cs16", bufs, 52, read=read)
    try:
        for target in (2 ** 31, 2 ** 32):
            p.run_to(target - 20000)
            gap = (target - 9000) // lcm * lcm - p.S  # up to a multiple of lcm (and so of every R)
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
            for k, (W, F, S) in enumerate(specs):
                ref = model_blocks(np.concatenate([conv("cs16", p.blocks[i]) for i in idx]),
                                   [len(p.blocks[i]) // 2 for i in idx], W, F, S)
                for j, i in enumerate(idx):
                    np.testing.assert_array_equal(got[i][k].view(np.uint32), ref[j].view(np.uint32),
                                                  err_msg=f"{target}: W={W} block {i}")
            assert g.spectrum_info(sids[2])[1] == p.S
    finally:
        g.close()
