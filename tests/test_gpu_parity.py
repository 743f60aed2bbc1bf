"""GPU parity tests: the CUDA path, called through the C ABI, against the oracle.

* the reference's own known-answer fixtures (tests/golden/reference_fixtures.json)
  with the reference's own assert semantics (test/utils.c:176-196);
* seeded random streams vs oracle/liboracle.so: float path within the contract's
  norm-wise tolerance (tests/util.py: max|d| <= 1e-5 * max|ref|), Q15 path bit-exact
  (tests/test_gpu_exact.py checks every kernel bit for bit on exact stimuli);
* the reference's edge cases: too-short input -> 0 outputs (test_xlating.c:63-81),
  ragged call sizes, state carry-over, even tap counts, mid-stream attach.
"""
import numpy as np
import pytest

from oracle import pyoracle as po
from exact import oracle_phases, oscillator_increment, to_complex
from util import RTOL, assert_cf32_close, ramp, rand_block, trunc4

pytestmark = pytest.mark.gpu


def fixture_filter(pkg, fixtures, max_input):
    s = fixtures["xlating"]["setup"]
    taps = pkg.create_low_pass_filter(s["lpf"]["gain"], s["sampling_freq"], s["lpf"]["cutoff"],
                                      s["lpf"]["transition_width"])
    assert len(taps) == s["ntaps"]
    return pkg.XlatingFilter(s["decimation"], taps, s["center_freq"], s["sampling_freq"], max_input)


def assert_golden_cf32(y, expected):
    """Reference semantics: (int32)(x*10000) equality.  The truncation is brittle
    within float noise of a multiple of 1e-4, so a mismatch is accepted only if the
    values agree to 1e-6 absolute (never needed so far)."""
    exp = np.asarray(expected, dtype=np.float32)
    got = np.asarray(y).view(np.float32)
    assert got.shape == exp.shape
    bad = np.nonzero(trunc4(got) != trunc4(exp))[0]
    for i in bad:
        assert abs(float(got[i]) - float(exp[i])) <= 1e-6, (i, got[i], exp[i])


# ---------------------------------------------------------------------------
# reference fixtures through the drop-in ABI
# ---------------------------------------------------------------------------
def test_fixture_full_block(pkg, fixtures):
    """test/test_xlating.c:24-37"""
    g = fixtures["xlating"]["max_input_buffer_size"]
    f = fixture_filter(pkg, fixtures, g["max_input"])
    x = ramp("cu8", 0, g["input_len"])
    y = f.process_cf32("cu8", x)
    assert len(y) == len(g["cf32"]) // 2
    assert_golden_cf32(y, g["cf32"])
    q = f.process_q15("cu8", x)
    np.testing.assert_array_equal(q.reshape(-1), np.array(g["cs16"], dtype=np.int16))
    f.close()


def test_fixture_partial_blocks(pkg, fixtures):
    """test/test_xlating.c:39-61 -- history and phase carry over between calls"""
    g = fixtures["xlating"]["partial_input_buffer_size"]
    f = fixture_filter(pkg, fixtures, g["max_input"])
    x0 = ramp("cu8", 0, g["input_len"])
    assert_golden_cf32(f.process_cf32("cu8", x0), g["cf32"])
    np.testing.assert_array_equal(f.process_q15("cu8", x0).reshape(-1), np.array(g["cs16"], dtype=np.int16))
    x1 = ramp("cu8", 200, g["input_len"])
    assert_golden_cf32(f.process_cf32("cu8", x1), g["next_cf32"])
    np.testing.assert_array_equal(f.process_q15("cu8", x1).reshape(-1), np.array(g["next_cs16"], dtype=np.int16))
    f.close()


def test_fixture_small_input(pkg, fixtures):
    """test/test_xlating.c:63-81 -- not enough data for an output"""
    g = fixtures["xlating"]["small_input_data"]
    f = fixture_filter(pkg, fixtures, g["max_input"])
    x = ramp("cu8", 0, g["first_len"])
    assert len(f.process_cf32("cu8", x)) == 20
    assert len(f.process_q15("cu8", x)) == 20
    x = ramp("cu8", 200, g["second_len"])
    assert len(f.process_cf32("cu8", x)) == g["expected_outputs"]
    assert len(f.process_q15("cu8", x)) == g["expected_outputs"]
    f.close()


@pytest.mark.parametrize("fmt,key", [("cu8", "rtlsdr_cu8"), ("cs16", "airspy_cs16"), ("cs8", "hackrf_cs8")])
def test_fixture_tcp_server(pkg, fixtures, fmt, key):
    """test/test_tcp_server.c:154-248: dsp_worker_start's filter on the mock SDR ramps"""
    s = fixtures["tcp_server"]["setup"]
    taps = pkg.create_low_pass_filter(1.0, s["band_sampling_rate"], s["lpf"]["cutoff"], s["lpf"]["transition_width"])
    f = pkg.XlatingFilter(s["decimation"], taps, s["center_offset"], s["band_sampling_rate"], s["buffer_size"])
    y = f.process_cf32(fmt, ramp(fmt, 0, s["input_elements"]))
    assert len(y) == len(fixtures["tcp_server"][key]) // 2
    assert_golden_cf32(y, fixtures["tcp_server"][key])
    f.close()


# ---------------------------------------------------------------------------
# drop-in ABI vs oracle on random streams
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("variant", ["native", "optimized"])
@pytest.mark.parametrize("fmt", ["cu8", "cs8", "cs16"])
@pytest.mark.parametrize("fs,rate,tw,center", [(48000, 9600, 2000, -12000), (2016000, 48000, 16400, -312000),
                                               (2016000, 96000, 19200, 400123), (10000000, 250000, 50000, 1234567)])
def test_dropin_stream_vs_oracle(pkg, fmt, variant, fs, rate, tw, center):
    rng = np.random.default_rng(99)
    taps = pkg.create_low_pass_filter(1.0, fs, rate // 2, tw)
    D = fs // rate
    max_in = 40000
    f = pkg.XlatingFilter(D, taps, center, fs, max_in)
    o = po.OracleFilter(D, taps, center, fs, max_in)
    fq = pkg.XlatingFilter(D, taps, center, fs, max_in)
    oq = po.OracleFilter(D, taps, center, fs, max_in)
    for n in [40000, 2, 38, 12346, 0, 40000, 20000, 4, 39998, 40000]:
        x = rand_block(rng, fmt, n)
        assert_cf32_close(f.process_cf32(fmt, x, variant), o.process_cf32(fmt, x), f"{fmt} n={n}")
        np.testing.assert_array_equal(fq.process_q15(fmt, x, variant), oq.process_q15(fmt, x))
    f.close()
    fq.close()


def test_dropin_even_taps_and_tiny_filter(pkg):
    """even tap counts keep the reference's reversal quirk; T=1 and D=1 edge cases.
    (D > T is excluded: there the reference's history_offset underflows,
    src/xlating.c:76 -- undefined behaviour, so there is nothing to be on par with.)"""
    rng = np.random.default_rng(5)
    for T, D in [(8, 2), (1, 1), (4, 3), (33, 1), (64, 7)]:
        taps = rng.standard_normal(T).astype(np.float32) * 0.2
        f = pkg.XlatingFilter(D, taps, 1000, 48000, 4096)
        o = po.OracleFilter(D, taps, 1000, 48000, 4096)
        for n in [4096, 10, 4096, 1024]:
            x = rand_block(rng, "cu8", n)
            assert_cf32_close(f.process_cf32("cu8", x), o.process_cf32("cu8", x), f"T={T} D={D} n={n}")
        f.close()


def test_dropin_long_stream_phase_drift(pkg):
    """300 consecutive full blocks: a closed-form oscillator would exceed 1e-5 by
    block ~10 (SURVEY.md 0.3); the replayed float recursion must not drift."""
    rng = np.random.default_rng(7)
    fs, rate = 2016000, 48000
    taps = pkg.create_low_pass_filter(1.0, fs, rate // 2, 16400)
    f = pkg.XlatingFilter(fs // rate, taps, -312000, fs, 65536)
    o = po.OracleFilter(fs // rate, taps, -312000, fs, 65536)
    worst = 0.0
    for b in range(300):
        x = rand_block(rng, "cu8", 65536)
        worst = max(worst, assert_cf32_close(f.process_cf32("cu8", x), o.process_cf32("cu8", x), f"block {b}"))
    assert worst < 1e-5
    f.close()


# ---------------------------------------------------------------------------
# batch ABI
# ---------------------------------------------------------------------------
def make_group(pkg, fs, max_in, plan, flags=0):
    g = pkg.Group(fs, max_in, flags=flags)
    oracles, ids = [], []
    for p in plan:
        taps = pkg.create_low_pass_filter(1.0, fs, p["cutoff"], p["tw"])
        ids.append(g.add_client(p["decimation"], taps, p["center"]))
        oracles.append(po.OracleFilter(p["decimation"], taps, p["center"], fs, max_in))
    return g, ids, oracles


@pytest.mark.parametrize("flags", [0, 4])  # 4 = XLG_FORCE_GENERIC
@pytest.mark.parametrize("fmt", ["cu8", "cs16"])
def test_group_mixed_clients_vs_oracle(pkg, fmt, flags):
    """40 clients, mixed 48/96 ksps (two tiled classes of 20 each) + 3 odd ones
    (generic kernel) on one shared input, several ragged blocks."""
    rng = np.random.default_rng(11)
    fs, max_in = 2016000, 65536
    plan = pkg.client_plan(fs, [48000 if c % 2 == 0 else 96000 for c in range(40)], tw=None)
    plan += [{"rate": 252000, "decimation": 8, "center": 100000, "cutoff": 100000, "tw": 60000},
             {"rate": 48000, "decimation": 42, "center": -5000, "cutoff": 24000, "tw": 16400},
             {"rate": 16000, "decimation": 126, "center": 777777, "cutoff": 8000, "tw": 3200}]
    g, ids, oracles = make_group(pkg, fs, max_in, plan, flags)
    kinds = set()
    for blk, n in enumerate([65536, 65536, 30000, 2, 65536, 12346, 65536]):
        x = rand_block(rng, fmt, n)
        t = g.submit(fmt, x)
        g.wait(t)
        for cid, o in zip(ids, oracles):
            assert_cf32_close(g.output(t, cid), o.process_cf32(fmt, x), f"block {blk} client {cid}")
            assert g.client_info(cid)[0] == o.history
        kinds |= {g.client_info(cid)[1] for cid in ids}
    assert kinds == ({0} if flags else {0, 1})
    g.close()


@pytest.mark.parametrize("env", [{}, {"XLATING_B200_CONV_STREAM": "0"}, {"XLATING_B200_CSTREAMS": "1"},
                                 {"XLATING_B200_SPECULATE": "0", "XLATING_B200_CSTREAMS": "1"},
                                 {"XLATING_B200_PARTITION": "1"}, {"XLATING_B200_PARTITION": "0"}],
                         ids=["default", "conv_on_compute_stream", "1stream", "no_spec_1stream", "partition", "no_partition"])
def test_group_pipelined_tickets(pkg, monkeypatch, env):
    """XLG_SLOTS blocks in flight before the first wait; outputs stay valid -- in every pipeline variant the
    measurement switches select (conversion stream, speculation, stream count, SM partition)."""
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    rng = np.random.default_rng(13)
    fs, max_in = 2016000, 32768
    plan = pkg.client_plan(fs, [48000] * 16, tw=16400)
    g, ids, oracles = make_group(pkg, fs, max_in, plan)
    blocks = [rand_block(rng, "cu8", max_in) for _ in range(12)]
    refs = [[o.process_cf32("cu8", x) for o in oracles] for x in blocks]
    pending = []
    for b, x in enumerate(blocks):
        pending.append((b, g.submit("cu8", x)))
        if len(pending) == pkg.XLG_SLOTS:
            bb, t = pending.pop(0)
            g.wait(t)
            for cid, r in zip(ids, refs[bb]):
                assert_cf32_close(g.output(t, cid), r, f"block {bb} client {cid}")
    for bb, t in pending:
        g.wait(t)
        for cid, r in zip(ids, refs[bb]):
            assert_cf32_close(g.output(t, cid), r, f"block {bb} client {cid}")
    g.close()


def test_group_attach_and_detach_midstream(pkg):
    """A client added at stream position P behaves like a reference filter created
    at that moment (zero history, phase 1): src/xlating.c:543-565."""
    rng = np.random.default_rng(17)
    fs, max_in = 2016000, 32768
    plan = pkg.client_plan(fs, [48000] * 12, tw=16400)
    g, ids, oracles = make_group(pkg, fs, max_in, plan)
    for _ in range(3):
        x = rand_block(rng, "cu8", max_in)
        t = g.submit("cu8", x)
        g.wait(t)
        for cid, o in zip(ids, oracles):
            assert_cf32_close(g.output(t, cid), o.process_cf32("cu8", x))
    # attach 10 more (one aligned class of its own) + 1 loner, detach two
    late = pkg.client_plan(fs, [96000] * 10, tw=19200) + [
        {"rate": 48000, "decimation": 42, "center": 1234, "cutoff": 24000, "tw": 9600}]
    for p in late:
        taps = pkg.create_low_pass_filter(1.0, fs, p["cutoff"], p["tw"])
        ids.append(g.add_client(p["decimation"], taps, p["center"]))
        oracles.append(po.OracleFilter(p["decimation"], taps, p["center"], fs, max_in))
    for victim in (ids[1], ids[5]):
        g.remove_client(victim)
    keep = [(c, o) for c, o in zip(ids, oracles) if c not in (ids[1], ids[5])]
    assert g.client_count() == len(keep)
    for blk in range(5):
        n = max_in if blk != 2 else 1000
        x = rand_block(rng, "cu8", n)
        t = g.submit("cu8", x)
        g.wait(t)
        for cid, o in keep:
            assert_cf32_close(g.output(t, cid), o.process_cf32("cu8", x), f"block {blk} client {cid}")
    g.close()


def test_group_q15_path_bit_exact(pkg):
    rng = np.random.default_rng(19)
    fs, max_in = 2016000, 32768
    plan = pkg.client_plan(fs, [48000, 96000, 48000, 96000], tw=None)
    g, ids, oracles = make_group(pkg, fs, max_in, plan)
    for n in [max_in, 500, max_in]:
        x = rand_block(rng, "cs16", n)
        t = g.submit("cs16", x, flags=pkg.XLG_PATH_Q15)
        g.wait(t)
        for cid, o in zip(ids, oracles):
            np.testing.assert_array_equal(g.output(t, cid, q15=True), o.process_q15("cs16", x))
    g.close()


def test_group_full_size_cfg2_sampled(pkg):
    """BASELINE configs[1] at full size: 256 clients, mixed 48/96 ksps, 262144-byte
    cu8 blocks; 8 sampled clients are checked against the oracle on 3 blocks, all
    clients' output counts on every block."""
    rng = np.random.default_rng(23)
    fs, max_in = 2016000, 262144
    plan = pkg.client_plan(fs, [48000 if c % 2 == 0 else 96000 for c in range(256)], tw=None)
    g = pkg.Group(fs, max_in)
    ids = []
    tapsets = {}
    for p in plan:
        key = (p["cutoff"], p["tw"])
        if key not in tapsets:
            tapsets[key] = pkg.create_low_pass_filter(1.0, fs, p["cutoff"], p["tw"])
        ids.append(g.add_client(p["decimation"], tapsets[key], p["center"]))
    sample = [0, 1, 2, 101, 128, 200, 254, 255]
    oracles = {c: po.OracleFilter(plan[c]["decimation"], tapsets[(plan[c]["cutoff"], plan[c]["tw"])],
                                  plan[c]["center"], fs, max_in) for c in sample}
    for blk in range(3):
        x = rand_block(rng, "cu8", max_in)
        t = g.submit("cu8", x)
        g.wait(t)
        for c in sample:
            assert_cf32_close(g.output(t, ids[c]), oracles[c].process_cf32("cu8", x), f"block {blk} client {c}")
        counts = [g.output_ptr(t, cid)[1] for cid in ids]
        assert all(n in (3120, 3121, 3122) for n in counts[0::2]) and all(n in (6241, 6242, 6243) for n in counts[1::2])
    assert all(g.client_info(cid)[1] == 1 for cid in ids)  # all on the tiled kernel
    g.close()


def test_group_linearity_full_size(pkg):
    """Size-independent property at full size: the cs16 converter has no offset
    (x/32768, src/xlating.c:409-410), so the whole path is linear in the input:
    y(a) + y(b) == y(a + b) up to float rounding of the sums."""
    rng = np.random.default_rng(29)
    fs, max_in = 2016000, 262144
    taps = pkg.create_low_pass_filter(1.0, fs, 24000, 16400)
    plan = pkg.client_plan(fs, [48000] * 64, tw=16400)
    outs = []
    a = rng.integers(-8000, 8000, max_in, dtype=np.int16)
    b = rng.integers(-8000, 8000, max_in, dtype=np.int16)
    for x in (a, b, (a + b).astype(np.int16)):
        g = pkg.Group(fs, max_in)
        ids = [g.add_client(p["decimation"], taps, p["center"]) for p in plan]
        t = g.submit("cs16", x)
        g.wait(t)
        outs.append(np.stack([g.output(t, c) for c in ids]))
        g.close()
    ya, yb, yab = outs
    err = np.max(np.abs((ya + yb) - yab)) / np.max(np.abs(yab))
    assert err < 5e-6, err


# ---------------------------------------------------------------------------
# more edge cases of the batch ABI
# ---------------------------------------------------------------------------
def test_group_cs8_and_no_renorm_variant(pkg):
    """HackRF format through the batch path, and XLG_NO_RENORM = the reference's AVX
    process_optimized_cf32, which never renormalises the phase (src/xlating.c:336-339)."""
    rng = np.random.default_rng(37)
    fs, max_in = 2016000, 32768
    plan = pkg.client_plan(fs, [48000] * 12, tw=16400)
    for flags, renorm in ((0, True), (pkg.XLG_NO_RENORM, False)):
        g = pkg.Group(fs, max_in, flags=flags)
        taps = pkg.create_low_pass_filter(1.0, fs, 24000, 16400)
        ids = [g.add_client(p["decimation"], taps, p["center"]) for p in plan]
        oracles = [po.OracleFilter(p["decimation"], taps, p["center"], fs, max_in) for p in plan]
        for blk in range(6):
            x = rand_block(rng, "cs8", max_in)
            t = g.submit("cs8", x)
            g.wait(t)
            for cid, o in zip(ids, oracles):
                assert_cf32_close(g.output(t, cid), o.process_cf32("cs8", x, renorm=renorm), f"blk {blk} c{cid}")
        g.close()


def test_group_very_long_filter_config5_shape(pkg):
    """BASELINE configs[4] shape: 61.44 Msps cs16 -> 48 ksps, D = 1280, the server's
    designer gives T = 15419 taps; 65536 samples per block -> 51/52 outputs."""
    rng = np.random.default_rng(41)
    fs, max_in = 61440000, 131072
    taps = pkg.create_low_pass_filter(1.0, fs, 24000, 9600)
    assert len(taps) == 15419
    g = pkg.Group(fs, max_in)
    centers = [-20000000, 1234567, 30000000]
    ids = [g.add_client(1280, taps, c) for c in centers]
    oracles = [po.OracleFilter(1280, taps, c, fs, max_in) for c in centers]
    for blk in range(3):
        x = rand_block(rng, "cs16", max_in)
        t = g.submit("cs16", x)
        g.wait(t)
        for cid, o in zip(ids, oracles):
            r = o.process_cf32("cs16", x)
            assert len(r) in (39, 51, 52)
            assert_cf32_close(g.output(t, cid), r, f"blk {blk} c{cid}")
    g.close()


def test_group_long_filter_split_k_kernel(pkg):
    """>= 8 aligned clients with a filter too long for a shared-memory tile use the
    split-K long-filter kernel (kernel kind 2): config-5 shape (aligned TMA strips) and an
    odd-decimation case (cp.async strips, many output tiles)."""
    rng = np.random.default_rng(67)
    # (a) BASELINE configs[4] shape
    fs, max_in = 61440000, 131072
    taps = pkg.create_low_pass_filter(1.0, fs, 24000, 9600)
    g = pkg.Group(fs, max_in)
    centers = [int(-30000000 + c * 4100000) for c in range(12)]
    ids = [g.add_client(1280, taps, c) for c in centers]
    oracles = [po.OracleFilter(1280, taps, c, fs, max_in) for c in centers]
    for blk, n in enumerate([max_in, max_in, 50000, max_in]):
        x = rand_block(rng, "cs16", n)
        t = g.submit("cs16", x)
        g.wait(t)
        for cid, o in zip(ids, oracles):
            assert_cf32_close(g.output(t, cid), o.process_cf32("cs16", x), f"(a) blk {blk} c{cid}")
    assert {g.client_info(c)[1] for c in ids} == {2}
    g.close()
    # (b) odd decimation, 24001 taps, 1638 outputs per block (26 output tiles, unaligned strips)
    fs, max_in, D, T = 1000000, 16384, 5, 24001
    taps = (rng.standard_normal(T) * 0.01).astype(np.float32)
    g = pkg.Group(fs, max_in)
    centers = [int(-400000 + c * 90000) for c in range(9)]
    ids = [g.add_client(D, taps, c) for c in centers]
    oracles = [po.OracleFilter(D, taps, c, fs, max_in) for c in centers]
    for blk in range(2):
        x = rand_block(rng, "cu8", max_in)
        t = g.submit("cu8", x)
        g.wait(t)
        for cid, o in zip(ids, oracles):
            assert_cf32_close(g.output(t, cid), o.process_cf32("cu8", x), f"(b) blk {blk} c{cid}")
    assert {g.client_info(c)[1] for c in ids} == {2}
    g.close()


@pytest.mark.parametrize("env", [{}, {"XLATING_B200_LONG_TMAP": "0"}], ids=["default", "no_tmap"])
def test_group_long_filter_odd_window_starts_and_variants(pkg, monkeypatch, env):
    """configs[4] shape with ODD block lengths in between: the window start of the long-filter class changes
    parity from block to block (the pipelined kernel then fetches its strips from one sample earlier; the
    TMA tensor-map path and the strip path must both give the oracle's answer), plus a ring wrap-around (the
    ring holds 5 blocks + history)."""
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    rng = np.random.default_rng(6701)
    fs, max_in = 61440000, 131072
    taps = pkg.create_low_pass_filter(1.0, fs, 24000, 9600)
    g = pkg.Group(fs, max_in)
    centers = [int(-30000000 + c * 2300000) for c in range(40)]  # two 32-client groups, the second partly padding
    ids = [g.add_client(1280, taps, c) for c in centers]
    check = [0, 7, 31, 32, 39]
    oracles = {c: po.OracleFilter(1280, taps, centers[c], fs, max_in) for c in check}
    sizes = [max_in, 50002, max_in, max_in, 30006, max_in, max_in, 131070, max_in, max_in, max_in, max_in]
    blocks, got, want = [], {c: [] for c in check}, {c: [] for c in check}
    for blk, n in enumerate(sizes):
        x = rand_block(rng, "cs16", n)
        blocks.append(x)
        t = g.submit("cs16", x)
        g.wait(t)
        for c in check:
            got[c].append(g.output(t, ids[c]))
            want[c].append(oracles[c].process_cf32("cs16", x))
            assert_cf32_close(got[c][-1], want[c][-1], f"{env} blk {blk} c{c}")
    assert {g.client_info(c)[1] for c in ids} == {2}
    g.close()
    # the margin on record: norm-wise error of the GPU and of the float32 oracle itself against the same
    # filter summed in float64 (the reference's float32 band-pass taps and oscillator phases)
    x = np.concatenate([np.zeros(len(taps) - 1)] + [to_complex("cs16", b) for b in blocks])
    counts = [len(y) for y in want[check[0]]]
    W = np.lib.stride_tricks.sliding_window_view(x, len(taps))[np.arange(sum(counts)) * 1280]
    for c in check:
        y64 = (W @ oracles[c].rev_taps.astype(np.complex128)) * oracle_phases(
            oscillator_increment(1280, centers[c], fs), counts)
        scale = np.max(np.abs(y64))
        e_gpu = np.max(np.abs(np.concatenate(got[c]) - y64)) / scale
        e_orc = np.max(np.abs(np.concatenate(want[c]) - y64)) / scale
        print(f"{env} c{c}: norm-wise error vs float64: GPU {e_gpu:.2e}, float32 oracle {e_orc:.2e}")
        assert e_gpu <= RTOL, (c, e_gpu, e_orc)


def test_group_partition_is_chosen_per_layout(pkg, monkeypatch):
    """XLG_SM_PARTITION offers the 8-SM oscillator partition; the group takes it where the pre-pass chain
    would pace the pipeline (many outputs per block, little FIR work) and declines it where the FIR dominates
    (configs[4] shape: 51 outputs per block, 15419 taps) -- and the answers do not depend on the choice."""
    monkeypatch.delenv("XLATING_B200_PARTITION", raising=False)
    rng = np.random.default_rng(6702)
    # (a) chain-bound: 64 clients at 96 ksps from 2.016 Msps, 253 taps
    fs, max_in = 2016000, 262144
    taps = pkg.create_low_pass_filter(1.0, fs, 48000, 19200)
    g = pkg.Group(fs, max_in, flags=pkg.XLG_SM_PARTITION)
    centers = [int(-900000 + c * 28000) for c in range(64)]
    ids = [g.add_client(21, taps, c) for c in centers]
    oracles = {c: po.OracleFilter(21, taps, centers[c], fs, max_in) for c in (0, 33, 63)}
    for blk in range(3):
        x = rand_block(rng, "cu8", max_in)
        t = g.submit("cu8", x)
        g.wait(t)
        for c, o in oracles.items():
            assert_cf32_close(g.output(t, ids[c]), o.process_cf32("cu8", x), f"(a) blk {blk} c{c}")
    sms_a = g.partition_sms()
    g.close()
    # (b) FIR-bound: 384 clients with the configs[4] filter
    fs, max_in = 61440000, 131072
    taps = pkg.create_low_pass_filter(1.0, fs, 24000, 9600)
    g = pkg.Group(fs, max_in, flags=pkg.XLG_SM_PARTITION)
    centers = [int(-30000000 + c * 150000) for c in range(384)]
    ids = [g.add_client(1280, taps, c) for c in centers]
    oracles = {c: po.OracleFilter(1280, taps, centers[c], fs, max_in) for c in (0, 200, 383)}
    for blk in range(3):
        x = rand_block(rng, "cs16", max_in)
        t = g.submit("cs16", x)
        g.wait(t)
        for c, o in oracles.items():
            assert_cf32_close(g.output(t, ids[c]), o.process_cf32("cs16", x), f"(b) blk {blk} c{c}")
    sms_b = g.partition_sms()
    g.close()
    # green contexts may be unavailable on a driver (then both are 0 and the group said so in its log)
    assert sms_a in (0, 8) and sms_b == 0, (sms_a, sms_b)
    if sms_a == 0:
        pytest.skip("green contexts unavailable: the partition could not be offered")


def test_decimation_larger_than_the_filter_is_defined_here(pkg):
    """D > T: in the reference `history_offset` underflows (src/xlating.c:76, undefined behaviour; its oracle
    restatement crashes there as well), so there is nothing to be bit-identical with.  Here the decimator simply
    skips the samples between windows.  Checked against the definition itself in float64,
        y[k] = p^k * sum_j x[k*D + j - (T-1)] * rev[j],   x = 0 before the stream starts,
    through the batch ABI and the per-filter ABI, over ragged blocks."""
    rng = np.random.default_rng(6703)
    fs, max_in = 2400000, 8192
    for D, T in ((48, 39), (100, 31)):
        taps = (rng.standard_normal(T) * 0.05).astype(np.float32)
        center = 123000
        w0 = np.float32(2 * np.pi * center / fs)
        bpf = taps.astype(np.complex128) * np.exp(1j * (np.arange(T, dtype=np.float32) * w0).astype(np.float64))
        rev = bpf[::-1]
        if T % 2 == 0:  # the reference re-swaps the middle pair of an even-length vector (src/xlating.c:530-534)
            a, b = T // 2 - 1, T // 2
            rev[a], rev[b] = rev[b], rev[a]
        # the oscillator step as the reference forms it: float product, cexpf, float components (src/xlating.c:544)
        inc = complex(np.complex64(np.exp(1j * np.float64(np.float32(-w0 * np.float32(D))))))
        g = pkg.Group(fs, max_in)
        cid = g.add_client(D, taps, center)
        f = pkg.XlatingFilter(D, taps, center, fs, max_in)
        xs, got_g, got_f = [], [], []
        for n in (max_in, 1000, 2, max_in, 4098, 600, max_in):
            raw = rand_block(rng, "cu8", n)
            t = g.submit("cu8", raw)
            g.wait(t)
            got_g.append(np.array(g.output(t, cid)))
            got_f.append(np.array(f.process_cf32("cu8", raw)))
            xs.append((raw.astype(np.float64)[0::2] - 127.5) / 128.0 + 1j * (raw.astype(np.float64)[1::2] - 127.5) / 128.0)
        x = np.concatenate([np.zeros(T - 1, dtype=np.complex128)] + xs)
        n_out = (len(x) - T) // D + 1
        ref = np.array([np.dot(x[k * D:k * D + T], rev) for k in range(n_out)]) * inc ** np.arange(n_out)
        for name, got in (("batch", np.concatenate(got_g)), ("per-filter", np.concatenate(got_f))):
            assert got.shape == ref.shape, f"D={D} T={T} {name}: {got.shape} outputs, definition {ref.shape}"
            err = np.max(np.abs(got - ref)) / np.max(np.abs(ref))
            assert err < 1e-4, f"D={D} T={T} {name}: {err:.2e} from the definition"
        g.close()
        f.close()


def test_group_rejects_oversized_block(pkg, capfd):
    """the reference overflows its work buffer here (src/xlating.c:353); we refuse"""
    g = pkg.Group(48000, 1000)
    g.add_client(5, pkg.create_low_pass_filter(1.0, 48000, 4800, 2000), -12000)
    with pytest.raises(RuntimeError):
        g.submit("cu8", np.zeros(1002, dtype=np.uint8))
    assert "<3>" in capfd.readouterr().err
    t = g.submit("cu8", np.zeros(1000, dtype=np.uint8))  # still usable
    g.wait(t)
    g.close()


def test_group_stale_tickets_and_host_ring(pkg):
    """outputs live XLG_SLOTS tickets by default, host_ring tickets with xlg_create_ex"""
    rng = np.random.default_rng(43)
    fs, max_in = 48000, 2000
    taps = pkg.create_low_pass_filter(1.0, fs, 4800, 2000)
    for ring in (0, 12):
        g = pkg.Group(fs, max_in, host_ring=ring)
        cid = g.add_client(5, taps, -12000)
        o = po.OracleFilter(5, taps, -12000, fs, max_in)
        keep = ring if ring else pkg.XLG_SLOTS
        tickets, refs = [], []
        for _ in range(keep + 3):
            x = rand_block(rng, "cu8", max_in)
            tickets.append(g.submit("cu8", x))
            refs.append(o.process_cf32("cu8", x))
        for i, t in enumerate(tickets):
            if i < 3:
                with pytest.raises(RuntimeError):
                    g.wait(t)  # overwritten: -ESTALE
            else:
                g.wait(t)
                assert_cf32_close(g.output(t, cid), refs[i], f"ticket {t}")
        g.close()


def test_group_concurrent_consumers(pkg):
    """many dsp threads wait on the same tickets concurrently (thread-per-client model)"""
    import threading
    rng = np.random.default_rng(47)
    fs, max_in = 2016000, 32768
    plan = pkg.client_plan(fs, [48000] * 24, tw=16400)
    g, ids, oracles = make_group(pkg, fs, max_in, plan)
    blocks = [rand_block(rng, "cu8", max_in) for _ in range(3)]
    refs = [[o.process_cf32("cu8", x) for x in blocks] for o in oracles]
    tickets = [g.submit("cu8", x) for x in blocks]
    errors = []

    def consumer(idx):
        try:
            for b, t in enumerate(tickets):
                g.wait(t)
                assert_cf32_close(g.output(t, ids[idx]), refs[idx][b], f"client {idx} block {b}")
        except Exception as e:  # noqa: BLE001
            errors.append(e)

    threads = [threading.Thread(target=consumer, args=(i,)) for i in range(len(ids))]
    for th in threads:
        th.start()
    for th in threads:
        th.join()
    assert not errors, errors[0]
    g.close()


def test_group_full_size_cfg3_sampled(pkg):
    """BASELINE configs[2] at full size: 64 clients at 250 ksps on a 10 Msps cs16 stream,
    1201-tap filters (tw = 20060), 262144-byte blocks."""
    rng = np.random.default_rng(53)
    fs, max_in = 10000000, 131072
    taps = pkg.create_low_pass_filter(1.0, fs, 125000, 20060)
    assert len(taps) == 1201
    plan = pkg.client_plan(fs, [250000] * 64, tw=20060)
    g = pkg.Group(fs, max_in)
    ids = [g.add_client(p["decimation"], taps, p["center"]) for p in plan]
    sample = [0, 7, 31, 32, 63]
    oracles = {c: po.OracleFilter(40, taps, plan[c]["center"], fs, max_in) for c in sample}
    for blk in range(3):
        x = rand_block(rng, "cs16", max_in)
        t = g.submit("cs16", x)
        g.wait(t)
        for c in sample:
            assert_cf32_close(g.output(t, ids[c]), oracles[c].process_cf32("cs16", x), f"blk {blk} c{c}")
    assert all(g.client_info(c)[1] == 1 for c in ids)
    g.close()


def test_dropin_many_filters_thread_per_client(pkg):
    """The unmodified reference server: one filter + one dsp thread per client, all
    processing copies of the same blocks concurrently (src/dsp_worker.c:41-88)."""
    import threading
    rng = np.random.default_rng(59)
    fs, max_in, n_clients = 2016000, 65536, 24
    plan = pkg.client_plan(fs, [48000 if c % 3 else 96000 for c in range(n_clients)])
    blocks = [rand_block(rng, "cu8", max_in) for _ in range(4)]
    filters, refs = [], []
    for p in plan:
        taps = pkg.create_low_pass_filter(1.0, fs, p["cutoff"], p["tw"])
        filters.append(pkg.XlatingFilter(p["decimation"], taps, p["center"], fs, max_in))
        o = po.OracleFilter(p["decimation"], taps, p["center"], fs, max_in)
        refs.append([o.process_cf32("cu8", x) for x in blocks])
    errors = []

    def dsp_thread(i):
        try:
            for b, x in enumerate(blocks):
                own_copy = x.copy()  # queue_put memcpy'd a private copy per client (src/queue.c:114)
                assert_cf32_close(filters[i].process_cf32("cu8", own_copy), refs[i][b], f"client {i} block {b}")
        except Exception as e:  # noqa: BLE001
            errors.append(e)

    threads = [threading.Thread(target=dsp_thread, args=(i,)) for i in range(n_clients)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors[0]
    for f in filters:
        f.close()


def test_dropin_combined_calls_mixed_paths_formats_sizes(pkg):
    """Calls that arrive together are combined into one launch (csrc/xlating_dropin.cu):
    a batch may mix input formats, the cf32 and the Q15 path, filter shapes and ragged
    call sizes, and the result must not depend on how the calls were batched."""
    import threading
    rng = np.random.default_rng(71)
    fs, max_in = 2016000, 40000
    shapes = [(42, 24000, 9600, -312000), (21, 48000, 19200, 400000), (7, 100000, 60000, 0), (3, 300000, 200000, -7)]
    fmts = ["cu8", "cs8", "cs16"]
    sizes = [40000, 2, 39998, 1234, 0, 20000, 36]  # ragged, incl. too-short (test_xlating.c:63-81) and empty calls
    jobs = []
    for i in range(18):
        D, cutoff, tw, center = shapes[i % len(shapes)]
        fmt, q15 = fmts[i % 3], (i % 5 == 1)
        taps = pkg.create_low_pass_filter(1.0, fs, cutoff, tw)
        f = pkg.XlatingFilter(D, taps, center + 1000 * i, fs, max_in)
        o = po.OracleFilter(D, taps, center + 1000 * i, fs, max_in)
        blocks = [rand_block(rng, fmt, sizes[(b + i) % len(sizes)]) for b in range(6)]
        ref = [(o.process_q15(fmt, x) if q15 else o.process_cf32(fmt, x)) for x in blocks]
        jobs.append((f, fmt, q15, blocks, ref))
    b0, c0, _ = pkg.dropin_stats()
    s0 = pkg.dropin_stream_stats()["served_by_group"]
    errors = []
    barrier = threading.Barrier(len(jobs))

    def dsp_thread(i):
        f, fmt, q15, blocks, ref = jobs[i]
        try:
            for b, x in enumerate(blocks):
                barrier.wait()  # arrive together, like the dsp threads woken by one sdr_callback
                if q15:
                    np.testing.assert_array_equal(f.process_q15(fmt, x), ref[b], err_msg=f"client {i} block {b}")
                else:
                    y = f.process_cf32(fmt, x)
                    assert len(y) == len(ref[b]), (i, b, len(y), len(ref[b]))
                    if len(y):
                        assert_cf32_close(y, ref[b], f"client {i} block {b}")
        except Exception as e:  # noqa: BLE001
            errors.append(e)
            barrier.abort()

    threads = [threading.Thread(target=dsp_thread, args=(i,)) for i in range(len(jobs))]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    assert not errors, errors[0]
    b1, c1, _ = pkg.dropin_stats()
    n_calls = sum(1 for (_, _, _, blocks, _) in jobs for x in blocks if len(x) >= 2)
    # every non-empty call went through the combined engine, or was served by the band's batch
    # group (csrc/stream_overlay.h: a filter whose own blocks form "the stream" becomes its member)
    served_by_group = pkg.dropin_stream_stats()["served_by_group"] - s0
    assert (c1 - c0) + served_by_group == n_calls
    assert 0 < b1 - b0 <= n_calls        # ... in at most that many launches
    for f, *_ in jobs:
        f.close()


def test_dropin_private_group_model(pkg, monkeypatch):
    """XLATING_B200_DROPIN=group: each filter a private one-client batch group (the
    older model, kept for A/B measurements) -- same results."""
    monkeypatch.setenv("XLATING_B200_DROPIN", "group")
    rng = np.random.default_rng(73)
    fs, max_in = 2016000, 32768
    taps = pkg.create_low_pass_filter(1.0, fs, 24000, 9600)
    f = pkg.XlatingFilter(42, taps, -312000, fs, max_in)
    o = po.OracleFilter(42, taps, -312000, fs, max_in)
    for n in (max_in, 1000, max_in):
        x = rand_block(rng, "cu8", n)
        assert_cf32_close(f.process_cf32("cu8", x), o.process_cf32("cu8", x), f"n={n}")
    f.close()


def test_group_empty_blocks_and_client_churn(pkg):
    """zero-length blocks, removing every client, re-adding, growing the arenas"""
    rng = np.random.default_rng(61)
    fs, max_in = 2016000, 32768
    taps = pkg.create_low_pass_filter(1.0, fs, 24000, 16400)
    g = pkg.Group(fs, max_in)
    t = g.submit("cu8", np.zeros(0, dtype=np.uint8))  # no clients, no data
    g.wait(t)
    ids = [g.add_client(42, taps, 1000 * c) for c in range(3)]
    oracles = [po.OracleFilter(42, taps, 1000 * c, fs, max_in) for c in range(3)]
    for n in (0, max_in, 0, 2, max_in):
        x = rand_block(rng, "cu8", n)
        t = g.submit("cu8", x)
        g.wait(t)
        for cid, o in zip(ids, oracles):
            assert_cf32_close(g.output(t, cid), o.process_cf32("cu8", x), f"n={n}")
    for cid in ids:
        g.remove_client(cid)
    assert g.client_count() == 0
    t = g.submit("cu8", rand_block(rng, "cu8", max_in))  # stream advances with nobody listening
    g.wait(t)
    # 40 new clients (arenas and tables grow); they start with zero history at the current position
    plan = pkg.client_plan(fs, [48000] * 40, tw=16400)
    ids = [g.add_client(p["decimation"], taps, p["center"]) for p in plan]
    oracles = [po.OracleFilter(p["decimation"], taps, p["center"], fs, max_in) for p in plan]
    for blk in range(3):
        x = rand_block(rng, "cu8", max_in)
        t = g.submit("cu8", x)
        g.wait(t)
        for cid, o in zip(ids, oracles):
            assert_cf32_close(g.output(t, cid), o.process_cf32("cu8", x), f"blk {blk} c{cid}")
    g.close()


def test_group_mixed_alignment_classes(pkg):
    """Clients of one (D, T) attached at different stream positions have different
    window alignments; with the natural input layout they still share a tiled class
    (8-client subgroups of equal alignment), lone alignments stay on the generic
    kernel.  Everything must match a reference filter created at the attach moment."""
    rng = np.random.default_rng(71)
    fs, max_in = 2016000, 32768
    taps = pkg.create_low_pass_filter(1.0, fs, 24000, 16400)
    g = pkg.Group(fs, max_in)
    ids, oracles = [], []

    def attach(n, base):
        for c in range(n):
            center = base + 7000 * c
            ids.append(g.add_client(42, taps, center))
            oracles.append(po.OracleFilter(42, taps, center, fs, max_in))

    def push(n):
        x = rand_block(rng, "cu8", n)
        t = g.submit("cu8", x)
        g.wait(t)
        for cid, o in zip(ids, oracles):
            assert_cf32_close(g.output(t, cid), o.process_cf32("cu8", x), f"client {cid} n={n}")

    attach(10, -900000)
    push(max_in)
    for step, (n_new, n_samples) in enumerate([(3, 20002), (1, 1234), (2, 30000), (5, 32768), (2, 2 * 997)]):
        attach(n_new, -500000 + 100000 * step)   # joins at a new alignment
        push(n_samples)                          # first block: zero-history window -> generic
        push(max_in)
    for _ in range(3):
        push(max_in)
    kinds = [g.client_info(c)[1] for c in ids]
    assert kinds.count(1) >= 10 + 3 + 2 + 5 + 2   # every alignment with >= 2 clients is tiled
    assert kinds.count(0) >= 1                    # the lone one is not
    hist = sorted({g.client_info(c)[0] for c in ids})
    assert len(hist) >= 4                         # several different alignments are live
    g.close()


def test_group_speculative_prepass_hits_and_rollbacks(pkg):
    """The oscillator pre-pass of block t+1 is launched with block t for "the same length
    again" (csrc/xlating_group.cu).  Right guesses, wrong lengths, a Q15 block in between
    (the two paths share history_offset, src/xlating.c:29), a client joining and one leaving
    between blocks: every output must still be the reference's."""
    rng = np.random.default_rng(89)
    fs, max_in = 2016000, 32768
    plan = pkg.client_plan(fs, [48000 if c % 2 == 0 else 96000 for c in range(20)], tw=None)
    g, ids, oracles = make_group(pkg, fs, max_in, plan)
    # (Q15 blocks only at the end: the reference's two paths keep separate sample buffers under one
    # shared history_offset, src/xlating.c:29, so alternating them on one filter is not meaningful)
    script = [("cf32", max_in), ("cf32", max_in), ("cf32", max_in), ("cf32", 2), ("cf32", max_in),
              ("cf32", 10000), ("cf32", 10000), ("add", 0), ("cf32", 10000), ("cf32", max_in), ("remove", 0),
              ("cf32", max_in), ("cf32", max_in), ("cf32", 31000), ("cf32", max_in), ("cf32", max_in),
              ("q15", max_in), ("q15", 2000)]
    for step, (what, n) in enumerate(script):
        if what == "add":
            p = {"rate": 48000, "decimation": 42, "center": 4321, "cutoff": 24000, "tw": 9600}
            taps = pkg.create_low_pass_filter(1.0, fs, p["cutoff"], p["tw"])
            ids.append(g.add_client(p["decimation"], taps, p["center"]))
            oracles.append(po.OracleFilter(p["decimation"], taps, p["center"], fs, max_in))
            continue
        if what == "remove":
            g.remove_client(ids.pop(3))
            oracles.pop(3)
            continue
        x = rand_block(rng, "cu8", n)
        if what == "q15":
            t = g.submit("cu8", x, flags=pkg.XLG_PATH_Q15)
            g.wait(t)
            for cid, o in zip(ids, oracles):
                np.testing.assert_array_equal(g.output(t, cid, q15=True), o.process_q15("cu8", x), err_msg=f"step {step}")
        else:
            t = g.submit("cu8", x)
            g.wait(t)
            for cid, o in zip(ids, oracles):
                assert_cf32_close(g.output(t, cid), o.process_cf32("cu8", x), f"step {step} client {cid}")
    g.close()


def test_group_reserve_keeps_unread_results_when_clients_are_added(pkg):
    """ADVICE round 1: growing the result arenas used to invalidate every ticket still waiting in the
    ring.  With xlg_reserve sized for the final client count, results submitted before 60 more
    clients attach stay readable (the reference never drops data for the others when a client
    joins, src/tcp_server.c:301-384)."""
    rng = np.random.default_rng(97)
    fs, max_in = 2016000, 32768
    taps = pkg.create_low_pass_filter(1.0, fs, 24000, 16400)
    plan = pkg.client_plan(fs, [48000] * 72, tw=16400)
    g = pkg.Group(fs, max_in, host_ring=8)
    g.reserve(72 * (max_in // 2 // 42 + 6))
    ids = [g.add_client(p["decimation"], taps, p["center"]) for p in plan[:12]]
    oracles = [po.OracleFilter(p["decimation"], taps, p["center"], fs, max_in) for p in plan[:12]]
    early = []
    for _ in range(3):
        x = rand_block(rng, "cu8", max_in)
        early.append((g.submit("cu8", x), [o.process_cf32("cu8", x) for o in oracles]))
    late_ids = [g.add_client(p["decimation"], taps, p["center"]) for p in plan[12:]]
    late_or = [po.OracleFilter(p["decimation"], taps, p["center"], fs, max_in) for p in plan[12:]]
    x = rand_block(rng, "cu8", max_in)
    t = g.submit("cu8", x)  # layout rebuilt for 72 clients; the arenas do not grow
    g.wait(t)
    for cid, o in zip(ids + late_ids, oracles + late_or):
        assert_cf32_close(g.output(t, cid), o.process_cf32("cu8", x), f"client {cid}")
    for t0, refs in early:  # still there
        g.wait(t0)
        for cid, r in zip(ids, refs):
            assert_cf32_close(g.output(t0, cid), r, f"early ticket {t0} client {cid}")
    g.close()
