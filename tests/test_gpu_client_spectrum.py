"""Spectrum rows of a source's output (xlg_add_client_spectrum, xlg_add_subband_spectrum) on the GPU.

A source spectrum's XLG_SPECTRUM_POWER rows must equal the kernel model (tests/spectrum_exact.py) bit for bit over
the source's own output, read back from the same group ticket by ticket (xlg_read_output) and concatenated, with
the per-ticket output counts as the block sizes.  A sub-band or bank channel has no host-visible output: its
reference stream is a pass-through member (D2 = 1, one tap 1.0, offset 0), an exact copy of its rows.  Covered:
every source family and kernel kind, widths of both channel stages with and without skip, the reference tool's
parameters at the client rate, ragged, empty and 1-sample blocks, rows across hundreds of blocks and many rows
per block, every attach timing, removal refusals, id reuse and churn, 256 client spectra beside a band spectrum,
device outputs and inputs with tickets in flight, a client carried past 2^31 and 2^32 outputs, the identity
client against the band and the reference's goldens, refusals and the profile counters.
"""
import errno

import numpy as np
import pytest

from exact import to_complex
from long_stream import N, Pump
from spectrum_exact import GOLDEN_DIR, GOLDEN_FS, GOLDENS, golden_stimulus, model_blocks, read_png
from util import rand_block

pytestmark = pytest.mark.gpu

FS = 2048000
MAX_IN = 2 * 65536
RAGGED = [65536, 8192, 2005, 0, 7, 1, 65536, 333, 40000, 1, 65536, 0, 30001, 65536]  # complex samples


def taps(rng, T):
    return (rng.standard_normal(T) / np.sqrt(T)).astype(np.float32)


def blocks_of(rng, fmt, sizes):
    return [rand_block(rng, fmt, 2 * n) for n in sizes]


class Rig:
    """A group, its sources (name -> (reference client id, spectrum source)), its spectra (name -> spectrum id,
    source name, W, F, S, attach block) and, per block, every source's output and every spectrum's rows."""

    def __init__(self, pkg, fs=FS, max_in=MAX_IN, flags=0):
        self.pkg, self.g = pkg, pkg.Group(fs, max_in, flags=flags)
        self.src, self.spec = {}, {}
        self.outs, self.rows = [], []  # per block: {source: output}, {spectrum: rows}

    def client(self, name, cid):
        self.src[name] = (cid, ("client", cid))

    def subband(self, name, sbid):
        """A sub-band (or bank channel) source, read through a pass-through member."""
        self.src[name] = (self.g.add_client_subband(sbid, 1, np.ones(1, np.float32), 0), ("sub", sbid))

    def attach(self, name, source, W, F, S=0):
        kind, i = self.src[source][1]
        add = self.g.add_client_spectrum if kind == "client" else self.g.add_subband_spectrum
        self.spec[name] = [add(i, W, F, S, power=True), source, W, F, S, len(self.outs)]

    def collect(self, t):
        self.outs.append({s: self.g.read_output(t, cid) for s, (cid, _) in self.src.items()})
        self.rows.append({s: self.g.read_spectrum(t, v[0]) for s, v in self.spec.items()})

    def feed(self, fmt, blocks):
        for x in blocks:
            self.collect(self.g.submit(fmt, x))

    def check(self, name, min_rows=1):
        sid, source, W, F, S, at = self.spec[name]
        ys = [o.get(source) for o in self.outs[at:]]
        x = np.concatenate(ys) if ys else np.zeros(0, np.complex64)
        ref = model_blocks(x, [len(y) for y in ys], W, F, S)
        total = 0
        for j, b in enumerate(range(at, len(self.outs))):
            got = self.rows[b][name]
            assert got.shape == ref[j].shape, f"{name} block {b}: {got.shape} rows, model {ref[j].shape}"
            np.testing.assert_array_equal(got.view(np.uint32), ref[j].view(np.uint32), err_msg=f"{name} block {b}")
            total += got.shape[0]
        assert total >= min_rows, f"{name}: {total} rows"
        return total

    def close(self):
        self.g.close()


def population(r, rng):
    """Every source family; returns {name: expected kind} of the clients (xlg_client_info)."""
    g, kinds = r.g, {}

    def client(name, cid, kind):
        r.client(name, cid)
        kinds[name] = kind

    for i in range(2):
        client(f"generic{i}", g.add_client(5, taps(rng, 16), 30000 * i), 0)
    for i in range(8):
        client(f"tiled{i}", g.add_client(21, taps(rng, 129), -400000 + 90000 * i), 1)
    for i in range(8):
        client(f"long{i}", g.add_client(1280, taps(rng, 2561), -300000 + 70000 * i), 2)
    for i in range(8):
        client(f"rat_tiled{i}", g.add_client_rational(3, 128, taps(rng, 390), 50000 * i), 4)
    client("rat_generic", g.add_client_rational(63, 640, taps(rng, 1764), 12345), 3)
    client("casc_int", g.add_client_cascade(6, taps(rng, 25), 100000, 7, taps(rng, 29)), 5)
    client("casc_rat", g.add_client_cascade(8, taps(rng, 17), -200000, 16, taps(rng, 47), interp2=3), 5)
    sb = g.add_subband(32, taps(rng, 64), 250000)
    client("member_int", g.add_client_subband(sb, 4, taps(rng, 33), 1000), None)
    client("member_rat", g.add_client_subband(sb, 40, taps(rng, 61), -2000, interp2=3), None)
    r.subband("subband", sb)
    r.subband("bank", g.add_bank_subband(g.add_bank(16, taps(rng, 200)), 5))
    r.subband("bank_fft", g.add_bank_subband(g.add_bank_fft(16, taps(rng, 64)), -3))
    return kinds


@pytest.mark.parametrize("W,F,S", [(64, 2, 5), (63, 3, 1)])
def test_every_source_family(pkg, W, F, S):
    rng = np.random.default_rng(W)
    r = Rig(pkg)
    try:
        kinds = population(r, rng)
        for s in r.src:
            r.attach(s, s, W, F, S)
        r.feed("cs16", blocks_of(rng, "cs16", RAGGED))
        for name, kind in kinds.items():
            if kind is not None:
                assert r.g.client_info(r.src[name][0])[1] == kind, name
        for s in r.spec:
            r.check(s, min_rows=0 if s.startswith("long") else 1)  # D = 1280: a row every few blocks
        assert sum(r.check(s, 0) for s in r.spec if s.startswith("long")) > 0
    finally:
        r.close()


# every width of both channel stages, with and without skip, on a D = 2 client (4096 outputs per 8192 samples)
WIDTHS = [(1, 1, 0), (2, 1, 1), (3, 5, 2), (4, 1, 0), (4, 2, 3), (63, 2, 0), (63, 1, 70), (64, 2, 0), (64, 3, 9),
          (1000, 1, 0), (1000, 2, 17), (1024, 1, 0), (1024, 3, 5), (4096, 1, 0), (4096, 2, 1)]


@pytest.mark.parametrize("W,F,S", WIDTHS)
def test_widths(pkg, W, F, S):
    rng = np.random.default_rng(1000 + W + S)
    r = Rig(pkg)
    try:
        r.client("d2", r.g.add_client(2, taps(rng, 33), 70000))
        r.client("casc", r.g.add_client_cascade(2, taps(rng, 9), 0, 2, taps(rng, 13)))
        r.attach("d2", "d2", W, F, S)
        r.attach("casc", "casc", W, F, S)
        r.feed("cs16", blocks_of(rng, "cs16", RAGGED))
        r.check("d2")
        r.check("casc")
    finally:
        r.close()


def test_tool_parameters_rows_across_hundreds_of_blocks(pkg):
    """The reference tool's parameters at a 32 ksps client rate: one row per 32000 outputs, 2.048 M input
    samples, across 250 blocks of 8192; and at W = 1 on a D = 1 client, 8192 rows in one block."""
    rng = np.random.default_rng(5)
    r = Rig(pkg, max_in=2 * 8192)
    try:
        r.client("slow", r.g.add_client(64, taps(rng, 301), -500000))
        r.client("fast", r.g.add_client(1, taps(rng, 3), 0))
        F, S = pkg.spectrogram_params(FS // 64, 64)
        r.attach("tool64", "slow", 64, F, S)
        F2, S2 = pkg.spectrogram_params(FS // 64, 1000)
        r.attach("tool1000", "slow", 1000, F2, S2)
        r.attach("w1", "fast", 1, 1, 0)
        r.feed("cu8", blocks_of(rng, "cu8", [8192] * 520))
        assert r.check("tool64") == 2 and r.check("tool1000") == 2
        assert r.rows[0]["w1"].shape == (8192, 1)
        r.check("w1")
    finally:
        r.close()


def test_attach_timing(pkg):
    """A spectrum attached mid-stream to a running client; a client attached mid-stream together with its
    spectrum, through its zero-history window and the re-layout that moves it into its tiled class."""
    rng = np.random.default_rng(9)
    r = Rig(pkg)
    try:
        for i in range(8):
            r.client(f"tiled{i}", r.g.add_client(21, taps(rng, 129), -400000 + 90000 * i))
        r.client("cascade", r.g.add_client_cascade(6, taps(rng, 25), 100000, 7, taps(rng, 29)))
        blocks = blocks_of(rng, "cs16", RAGGED + RAGGED[:6])
        r.feed("cs16", blocks[:3])
        r.attach("mid", "tiled3", 64, 2, 1)
        r.attach("casc_mid", "cascade", 63, 1, 0)
        r.feed("cs16", blocks[3:5])
        for i in range(8):  # a class of its own once their windows have passed the attach point
            r.client(f"late{i}", r.g.add_client(21, taps(rng, 129), 333000 - 80000 * i))
        r.attach("late0", "late0", 128, 1, 7)
        r.attach("late7", "late7", 1000, 2, 0)
        r.feed("cs16", blocks[5:])
        assert r.g.client_info(r.src["late0"][0])[1] == 1  # settled into a tiled class
        for s in ("mid", "casc_mid", "late0", "late7"):
            r.check(s)
    finally:
        r.close()


def test_removal_refusals_id_reuse_and_churn(pkg):
    rng = np.random.default_rng(17)
    r = Rig(pkg)
    g = r.g
    try:
        r.client("a", g.add_client(8, taps(rng, 65), 120000))
        r.client("m", g.add_client(16, taps(rng, 65), -90000))
        sb = g.add_subband(16, taps(rng, 64), -250000)  # a sub-band without members
        bid = g.add_bank(16, taps(rng, 100))
        ch = g.add_bank_subband(bid, 2)
        band = g.add_spectrum(1000, 1, 0, power=True)
        assert band == 0
        blocks = blocks_of(rng, "cs16", RAGGED)
        t0 = g.submit("cs16", blocks[0])
        r.outs.append({s: g.read_output(t0, c) for s, (c, _) in r.src.items()})
        r.rows.append({})
        g.remove_spectrum(band)
        r.attach("a", "a", 512, 1, 0)
        assert r.spec["a"][0] == 0  # the band spectrum's id, now a client spectrum's
        s_sb = g.add_subband_spectrum(sb, 64, 1, power=True)
        s_ch = g.add_subband_spectrum(ch, 32, 2, power=True)
        for call, arg in ((g.remove_client, r.src["a"][0]), (g.remove_subband, sb), (g.remove_subband, ch),
                          (g.remove_bank, bid)):
            with pytest.raises(ValueError) as e:
                call(arg)
            assert e.value.args[0] == -errno.EBUSY
        # the band spectrum's ticket keeps its width; the new ticket has the client spectrum's
        assert g.spectrum_width(t0, 0) == 1000
        band_rows = g.read_spectrum(t0, 0)
        ref = model_blocks(to_complex("cs16", blocks[0]).astype(np.complex64), [RAGGED[0]], 1000, 1, 0)[0]
        np.testing.assert_array_equal(band_rows.view(np.uint32), ref.view(np.uint32))
        churn = []
        for b, x in enumerate(blocks[1:], 1):
            if b % 3 == 1:
                churn.append(g.add_client(8, taps(rng, 65), 10000 * b))
            elif b % 3 == 2 and churn:
                g.remove_client(churn.pop(0))
            r.collect(g.submit("cs16", x))
            assert g.spectrum_width(len(r.outs) - 1, 0) == 512
        r.check("a")
        g.remove_spectrum(s_sb)
        g.remove_spectrum(s_ch)
        g.remove_subband(sb)
        g.remove_subband(ch)
        g.remove_bank(bid)
        g.remove_spectrum(r.spec["a"][0])
        g.remove_client(r.src["a"][0])
    finally:
        r.close()


def test_unaffected_outputs_with_256_client_spectra(pkg):
    """The cfg2-style group (256 clients at 48 and 96 ksps of 2.016 Msps, cu8) with a spectrum on every client
    and one on the band: every client's output is the output of the group without spectra, the band rows are
    those of a group with the band spectrum alone, and every client spectrum matches its model."""
    fs, max_in = 2016000, 2 * 65536
    plan = pkg.client_plan(fs, [48000 if c % 2 == 0 else 96000 for c in range(256)])
    rng = np.random.default_rng(23)
    blocks = blocks_of(rng, "cu8", [65536, 1000, 0, 65536, 77, 65536])

    def run(client_spectra, band):
        r = Rig(pkg, fs, max_in)
        try:
            for i, p in enumerate(plan):
                r.client(i, r.g.add_client(p["decimation"], pkg.create_low_pass_filter(1.0, fs, p["cutoff"], p["tw"]),
                                           p["center"]))
                if client_spectra:
                    r.attach(i, i, 64, 2, 3)
            b = r.g.add_spectrum(1024, 1, 0, power=True) if band else None
            rows = []
            for x in blocks:
                t = r.g.submit("cu8", x)
                r.collect(t)
                rows.append(r.g.read_spectrum(t, b) if band else None)
            if client_spectra:
                for i in range(len(plan)):
                    r.check(i)
            return r.outs, rows
        finally:
            r.close()

    plain, _ = run(False, False)
    band_only, band_rows = run(False, True)
    both, rows = run(True, True)
    for b in range(len(blocks)):
        np.testing.assert_array_equal(rows[b].view(np.uint32), band_rows[b].view(np.uint32), err_msg=f"block {b}")
        for i in range(len(plan)):
            for other in (band_only, both):
                np.testing.assert_array_equal(other[b][i].view(np.uint32), plain[b][i].view(np.uint32),
                                              err_msg=f"block {b} client {i}")


@pytest.mark.parametrize("mode", ["out_device", "input_device", "input_keep"])
def test_ingest_paths_with_tickets_in_flight(pkg, mode):
    torch = pytest.importorskip("torch")
    rng = np.random.default_rng(31)
    sizes = [65536, 5000, 0, 65536, 77, 1, 65536, 4096, 65536, 30000]
    blocks = blocks_of(rng, "cu8", sizes)
    r = Rig(pkg, flags=pkg.XLG_OUT_DEVICE if mode == "out_device" else 0)
    try:
        r.client("c", r.g.add_client(4, taps(rng, 41), 150000))
        r.client("casc", r.g.add_client_cascade(4, taps(rng, 17), -60000, 3, taps(rng, 21)))
        r.subband("sb", r.g.add_subband(8, taps(rng, 48), 300000))
        for s in ("c", "casc", "sb"):
            r.attach(s, s, 128, 3, 17)
        keep, pending = [], []
        for x in blocks:
            if mode == "input_device":
                d = torch.from_numpy(x.copy()).cuda()
                torch.cuda.current_stream().synchronize()
                keep.append(d)
                t = r.g.submit_ptr(pkg.FMT["cu8"], d.data_ptr(), x.size, pkg.XLG_INPUT_DEVICE)
            elif mode == "input_keep":
                buf = pkg.PinnedBuffer(max(x.size, 1))
                buf.array(np.uint8)[:x.size] = x
                keep.append(buf)
                t = r.g.submit_ptr(pkg.FMT["cu8"], buf.ptr, x.size, pkg.XLG_INPUT_KEEP)
            else:
                t = r.g.submit("cu8", x)
            pending.append(t)
            if len(pending) == pkg.XLG_SLOTS:  # XLG_SLOTS tickets in flight before the oldest is read
                r.collect(pending.pop(0))
        for t in pending:
            r.collect(t)
        for s in ("c", "casc", "sb"):
            r.check(s)
    finally:
        r.close()


def identity(g):
    return g.add_client(1, np.ones(1, np.float32), 0)


def test_identity_client_equals_band(pkg):
    rng = np.random.default_rng(41)
    g = pkg.Group(FS, MAX_IN)
    try:
        cid = identity(g)
        pairs = [(g.add_spectrum(W, F, S, power=True), g.add_client_spectrum(cid, W, F, S, power=True))
                 for W, F, S in ((64, 2, 5), (63, 3, 1), (4096, 1, 7), (1, 1, 0))]
        dbs = (g.add_spectrum(1000, 2, 0), g.add_client_spectrum(cid, 1000, 2, 0))
        for x in blocks_of(rng, "cs16", RAGGED):
            t = g.submit("cs16", x)
            np.testing.assert_array_equal(g.read_output(t, cid), to_complex("cs16", x).astype(np.complex64))
            for a, b in pairs + [dbs]:
                np.testing.assert_array_equal(g.read_spectrum(t, b).view(np.uint32),
                                              g.read_spectrum(t, a).view(np.uint32))
    finally:
        g.close()


@pytest.mark.parametrize("name", ["spectrogram_cu8.png", "spectrogram_cs16.png"])
@pytest.mark.parametrize("cuts", [[256], [100, 0, 1, 155]])
def test_golden_pixels(pkg, name, cuts):
    fmt, W = GOLDENS[name]
    F, S = pkg.spectrogram_params(GOLDEN_FS, W)
    raw = golden_stimulus(fmt)
    g = pkg.Group(GOLDEN_FS, 512)
    rows = []
    try:
        sid = g.add_client_spectrum(identity(g), W, F, S)
        pos = 0
        for n in cuts:
            t = g.submit(fmt, raw[2 * pos:2 * (pos + n)])
            rows.append(g.read_spectrum(t, sid))
            pos += n
    finally:
        g.close()
    np.testing.assert_array_equal(pkg.spectrogram_pixels(np.concatenate(rows)), read_png(f"{GOLDEN_DIR}/{name}"))


def test_long_stream_client_past_2_32(pkg):
    """A D = 1 client carried past 2^31 and 2^32 outputs: after a boundary B that every row period divides, its
    rows are a fresh spectrum's over the outputs read from B on."""
    torch = pytest.importorskip("torch")
    specs = [(64, 3, 0), (105, 2, 0), (1, 1, 0)]
    lcm = 6720
    rng = np.random.default_rng(51)
    bufs = [rand_block(rng, "cs16", 2 * N) for _ in range(3)]
    g = pkg.Group(FS, 2 * N)
    cid = g.add_client(1, taps(rng, 5), 0)
    sids = [g.add_client_spectrum(cid, W, F, S, power=True) for W, F, S in specs]
    got = {}

    def read(t, i):
        got[i] = (g.read_output(t, cid), [g.read_spectrum(t, s) for s in sids])

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
            ys = [got[i][0] for i in idx]
            assert [len(y) for y in ys] == [len(p.blocks[i]) // 2 for i in idx]  # D = 1: one output per sample
            for k, (W, F, S) in enumerate(specs):
                ref = model_blocks(np.concatenate(ys), [len(y) for y in ys], W, F, S)
                for j, i in enumerate(idx):
                    np.testing.assert_array_equal(got[i][1][k].view(np.uint32), ref[j].view(np.uint32),
                                                  err_msg=f"{target}: W={W} block {i}")
        assert g.spectrum_info(sids[2])[1] == p.S
    finally:
        g.close()


def test_refusals_and_profile(pkg):
    rng = np.random.default_rng(61)
    g = pkg.Group(FS, MAX_IN)
    try:
        cid = g.add_client(4, taps(rng, 33), 0)
        sb = g.add_subband(8, taps(rng, 32), 0)
        for call, i in ((g.add_client_spectrum, 7), (g.add_client_spectrum, -1), (g.add_subband_spectrum, 3),
                        (g.add_subband_spectrum, -1)):
            with pytest.raises(ValueError) as e:
                call(i, 64, 1)
            assert e.value.args[0] == -errno.EINVAL, (call, i)
        for W, F, S in ((0, 1, 0), (4097, 1, 0), (64, 0, 0), (1, 2 ** 31 - 1, 1)):
            for call, i in ((g.add_client_spectrum, cid), (g.add_subband_spectrum, sb)):
                with pytest.raises(ValueError) as e:
                    call(i, W, F, S)
                assert e.value.args[0] == -errno.EINVAL
        a = g.add_client_spectrum(cid, 64, 2, 3)
        b = g.add_subband_spectrum(sb, 100, 1)
        x = np.zeros(2 * 4000, np.int16)
        with pytest.raises(RuntimeError, match=str(-errno.ENOTSUP)):
            g.submit("cs16", x, pkg.XLG_PATH_Q15)
        g.profile_enable(True)
        g.profile_read()
        g.spectrum_profile_read()
        t = g.submit("cs16", x)
        assert t == 0  # the refused Q15 submit took no ticket
        g.wait(t)
        n_c = len(g.read_output(t, cid))
        p = g.spectrum_profile_read()
        frames_a, frames_b = n_c // 131 * 2 + min(2, n_c % 131 // 64), g.spectrum_info(b)[1]  # (F = 1 for b)
        assert frames_b > 0
        assert p["spectrum_launches"] == 1 and p["spectrum_ms"] > 0
        assert p["frames"] == frames_a + frames_b
        assert p["channel_flops"] == frames_a * (pkg.bank_fft_flops(64) + 6 * 64) + frames_b * (4 * 100 ** 2 + 600)
        assert g.spectrum_info(a) == (1, n_c // 131 + (1 if n_c % 131 >= 128 else 0))
        assert g.spectrum_info(b)[0] == 0
    finally:
        g.close()
    g = pkg.Group(FS, MAX_IN, flags=pkg.XLG_TRACK_STATE)
    try:
        cid = g.add_client(4, taps(rng, 33), 0)
        with pytest.raises(ValueError) as e:
            g.add_client_spectrum(cid, 64, 1)
        assert e.value.args[0] == -errno.ENOTSUP
    finally:
        g.close()
