"""Rational L/M clients (xlg_add_client_rational) on the GPU.

A rational client is the reference filter with decimation M at L * fs fed the zero-stuffed stream
(tests/rational.py).  Designed taps are held to the 1e-5 float contract against the strict oracle
on that stream; exact stimuli (tests/exact.py: centre 0, dyadic taps, inputs on a grid) must equal
the float64 sum on it bit for bit, which sees a wrong branch, a window one sample off or a stuffed
position that leaked a sample.
"""

import numpy as np
import pytest

from exact import assert_exact, dyadic_taps, exact_input, grid_step, ref_f64
from oracle import pyoracle as po
from rational import ROWS, oracle_filter, stuff
from util import assert_cf32_close, oracle_stream, rand_block

pytestmark = pytest.mark.gpu

FS, MAX_IN = 2016000, 65536
GENERIC, TILED = 3, 4  # rational client kinds: polyphase generic kernel, tiled classes
POLY_GENERIC = {"XLATING_B200_POLY_TILE": "0"}
RAGGED = [65536, 65536, 30001, 2, 0, 65536, 12347, 65536, 7, 65534]


class Client:
    def __init__(self, cid, L, M, taps, first_block):
        self.cid, self.L, self.M, self.taps, self.first = cid, L, M, taps, first_block
        self.last = None
        self.got, self.kinds = [], set()


def drive_exact(pkg, monkeypatch, plan, sizes, fmt="cu8", fs=FS, max_in=MAX_IN, env=None, flags=0, host_ring=0,
                attach=None, detach=None, depth=1, seed=0, want=TILED):
    """Exact stimuli through a group; plan / attach entries are (L, M, T) (L = 0: an integer client
    added with xlg_add_client and decimation M).  Checks every output of every client bit for bit, and
    that the rational clients ran on kind `want` (TILED: at least one block on it, GENERIC: only there)."""
    for k, v in (env or {}).items():
        monkeypatch.setenv(k, v)
    rng = np.random.default_rng(seed)
    g = pkg.Group(fs, max_in, flags=flags, host_ring=host_ring)
    clients = []

    def add(specs, b):
        for L, M, T in specs:
            taps = dyadic_taps(rng, T, fmt)
            cid = g.add_client(M, taps, 0) if L == 0 else g.add_client_rational(L, M, taps, 0)
            clients.append(Client(cid, max(L, 1), M, taps, b))

    add(plan, 0)
    blocks = [exact_input(rng, fmt, n) for n in sizes]
    pending = []

    def collect(b, t):
        g.wait(t)
        for c in clients:
            if c.first <= b and (c.last is None or b < c.last):
                y = g.read_output(t, c.cid) if flags & pkg.XLG_OUT_DEVICE else g.output(t, c.cid)
                c.got.append(np.array(y, copy=True))
                c.kinds.add(g.client_info(c.cid)[1])

    for b, x in enumerate(blocks):
        if (attach and b in attach) or (detach and b in detach):
            while pending:
                collect(*pending.pop(0))
            for i in (detach or {}).get(b, []):
                g.remove_client(clients[i].cid)
                clients[i].last = b
            add((attach or {}).get(b, []), b)
        pending.append((b, g.submit(fmt, x)))
        if len(pending) >= depth:
            collect(*pending.pop(0))
    while pending:
        collect(*pending.pop(0))
    g.close()
    rational = set().union(*[c.kinds for c in clients if c.L > 1])
    assert rational <= {GENERIC, TILED} and (want in rational) and (want == TILED or rational == {GENERIC}), rational
    for c in clients:
        seen = [stuff(fmt, x, c.L) for x in blocks[c.first:c.last]]
        ref = ref_f64(c.taps, c.M, "cs16", seen)
        assert_exact(c.got, ref, f"{env or ''} flags={flags} client {c.cid} (L={c.L}, M={c.M}, T={c.taps.size})",
                     c.taps.size, c.M, grid_step(c.taps, fmt))
    return clients


def test_interp_one_is_add_client(pkg):
    """add_client_rational(1, D, ...) is add_client(D, ...): same kernels (tiled, generic, split-K), same bits."""
    cases = [(FS, MAX_IN, 0, [(42, 48000)] * 16 + [(8, 252000)], {1, 0}),
             (FS, MAX_IN, pkg.XLG_FORCE_GENERIC, [(42, 48000)] * 4, {0}),
             (61440000, 131072, 0, [(1280, 48000)] * 8, {2})]
    for fs, max_in, flags, spec, want_kinds in cases:
        plan = pkg.client_plan(fs, [r for _, r in spec])
        taps = [pkg.create_low_pass_filter(1.0, fs, p["cutoff"], p["tw"]) for p in plan]
        rng = np.random.default_rng(fs % 97)
        blocks = [rand_block(rng, "cs16", n) for n in (max_in, max_in, 1001, max_in)]
        outs, kinds = [], []
        for rational in (False, True):
            g = pkg.Group(fs, max_in, flags=flags)
            ids = [g.add_client_rational(1, D, t, p["center"]) if rational else g.add_client(D, t, p["center"])
                   for (D, _), t, p in zip(spec, taps, plan)]
            got = []
            for x in blocks:
                t = g.submit("cs16", x)
                g.wait(t)
                got.append([g.output(t, c) for c in ids])
            kinds.append([g.client_info(c) for c in ids])
            outs.append(got)
            g.close()
        assert kinds[0] == kinds[1]
        assert {k for _, k in kinds[0]} == want_kinds, kinds[0]
        for a, b in zip(outs[0], outs[1]):
            for ya, yb in zip(a, b):
                assert np.array_equal(ya.view(np.uint64), yb.view(np.uint64))


@pytest.mark.parametrize("kind", [TILED, GENERIC], ids=["tiled", "generic"])
@pytest.mark.parametrize("row", ROWS, ids=lambda r: f"{r[0] // 1000}k_{r[1]}")
def test_rows_against_zero_stuffed_oracle(pkg, monkeypatch, row, kind):
    """The rate table's rows, 8 clients across the band, 20 ragged blocks with ring wraps.  Rows 3 and 4
    (branches of 2510 and 5019 taps at M = 625 and 1250) exceed the tiled kernel's shared memory and stay
    on the generic kernel."""
    fs, fmt, rate = row
    if kind == GENERIC:
        monkeypatch.setenv("XLATING_B200_POLY_TILE", "0")
    plan = pkg.rational_plan(fs, [rate] * 8)
    rng = np.random.default_rng(fs % 1009)
    blocks = [rand_block(rng, fmt, n) for n in RAGGED * 2]
    g = pkg.Group(fs, MAX_IN)
    ids = [g.add_client_rational(p["interp"], p["decim"], p["taps"], p["center"]) for p in plan]
    got = [[] for _ in ids]
    for x in blocks:
        t = g.submit(fmt, x)
        g.wait(t)
        for i, c in enumerate(ids):
            got[i].append(g.output(t, c))
    kinds = {g.client_info(c)[1] for c in ids}
    g.close()
    assert kinds == ({kind} if fs <= 3000000 else {GENERIC}), kinds
    L = plan[0]["interp"]
    oracles = [oracle_filter(po, L, p["decim"], p["taps"], p["center"], fs, MAX_IN) for p in plan]
    ref = oracle_stream(oracles, "cs16", [stuff(fmt, x, L) for x in blocks])
    for i, p in enumerate(plan):
        assert [len(y) for y in got[i]] == [len(y) for y in ref[i]]
        assert_cf32_close(np.concatenate(got[i]), np.concatenate(ref[i]), f"row {fs} client {i} centre {p['center']}")


SMALL = [16384, 16384, 7001, 2, 0, 16384, 3, 16382, 16384, 16384]


@pytest.mark.parametrize("spec", [(3, 128, 97), (5, 4, 3), (2, 1, 9), (5, 3, 40), (7, 320, 431)],
                         ids=["T_not_multiple_of_L", "T_below_L", "M_1", "L_above_M", "44k1_of_2016k"])
@pytest.mark.parametrize("fmt", ["cu8", "cs16"])
@pytest.mark.parametrize("kind", [TILED, GENERIC], ids=["tiled", "generic"])
def test_exact(pkg, monkeypatch, spec, fmt, kind):
    drive_exact(pkg, monkeypatch, [spec] * 8, SMALL, fmt=fmt, max_in=16384, want=kind,
                env=POLY_GENERIC if kind == GENERIC else None)


def test_integer_clients_unchanged_by_rational_ones(pkg):
    """In a mixed group the integer clients' outputs are those of the same group without rational clients."""
    fs = FS
    plan = pkg.client_plan(fs, [48000] * 16 + [252000])
    rplan = pkg.rational_plan(fs, [44100] * 8)
    rng = np.random.default_rng(11)
    blocks = [rand_block(rng, "cu8", n) for n in RAGGED]
    outs = []
    for mixed in (False, True):
        g = pkg.Group(fs, MAX_IN)
        ids = [g.add_client(p["decimation"], pkg.create_low_pass_filter(1.0, fs, p["cutoff"], p["tw"]), p["center"])
               for p in plan]
        rids = [g.add_client_rational(p["interp"], p["decim"], p["taps"], p["center"]) for p in rplan] if mixed else []
        got = []
        for x in blocks:
            t = g.submit("cu8", x)
            g.wait(t)
            got.append([g.output(t, c) for c in ids])
        if mixed:
            assert {g.client_info(c)[1] for c in rids} == {TILED}
        g.close()
        outs.append(got)
    for a, b in zip(*outs):
        for ya, yb in zip(a, b):
            assert np.array_equal(ya.view(np.uint64), yb.view(np.uint64))


@pytest.mark.parametrize("variant", ["default", "out_device", "host_ring", "sm_partition", "cstreams1", "cstreams4",
                                     "no_renorm"])
def test_attach_detach_pipelined(pkg, monkeypatch, variant):
    """Rational clients join and leave mid-stream next to tiled integer clients, three tickets in flight,
    with blocks of repeated and of changing sizes.  A tiled rational class falls back to the generic kernel
    when detaches leave it under 8 members; clients attached mid-stream start there and join a tiled class
    once their zero-history window has passed."""
    flags, env, host_ring = 0, None, 0
    if variant == "out_device":
        flags = pkg.XLG_OUT_DEVICE
    elif variant == "host_ring":
        host_ring = 16
    elif variant == "sm_partition":
        flags, env = pkg.XLG_SM_PARTITION, {"XLATING_B200_PARTITION": "1"}
    elif variant == "cstreams1":
        env = {"XLATING_B200_CSTREAMS": "1"}
    elif variant == "cstreams4":
        env = {"XLATING_B200_CSTREAMS": "4"}
    elif variant == "no_renorm":
        flags = pkg.XLG_NO_RENORM
    plan = [(0, 42, 505)] * 16 + [(3, 128, 97)] * 8
    sizes = [65536, 65536, 65536, 30001, 30001, 65536, 2, 65536, 65536, 12347, 65536, 65536]
    drive_exact(pkg, monkeypatch, plan, sizes, env=env, flags=flags, host_ring=host_ring, depth=3,
                attach={3: [(7, 320, 431)] * 8, 10: [(5, 3, 40)] * 2}, detach={5: [16, 17], 9: [24]})


def test_track_state_hist_and_oscillator(pkg):
    """XLG_TRACK_STATE: hist in upsampled samples and the oscillator equal the oracle's after every block."""
    fs = 2048000
    plan = pkg.rational_plan(fs, [48000] * 3)
    g = pkg.Group(fs, MAX_IN, flags=pkg.XLG_TRACK_STATE)
    ids = [g.add_client_rational(p["interp"], p["decim"], p["taps"], p["center"]) for p in plan]
    oracles = [oracle_filter(po, p["interp"], p["decim"], p["taps"], p["center"], fs, MAX_IN) for p in plan]
    rng = np.random.default_rng(5)
    for n in RAGGED:
        x = rand_block(rng, "cu8", n)
        t = g.submit("cu8", x)
        g.wait(t)
        for c, o, p in zip(ids, oracles, plan):
            r = o.process_cf32("cs16", stuff("cu8", x, p["interp"]))
            got, st = g.copy_output(t, c)
            assert len(got) == len(r)
            assert st.hist == o.history == g.client_info(c)[0]
            assert complex(st.phase_re, st.phase_im) == complex(np.complex64(o.phase))
    g.close()


def test_q15_refused_and_group_usable(pkg):
    fs = 2048000
    p = pkg.rational_plan(fs, [48000])[0]
    g = pkg.Group(fs, MAX_IN)
    cid = g.add_client_rational(p["interp"], p["decim"], p["taps"], p["center"])
    o = oracle_filter(po, p["interp"], p["decim"], p["taps"], p["center"], fs, MAX_IN)
    rng = np.random.default_rng(9)
    got, ref = [], []
    for b in range(3):
        if b == 1:
            with pytest.raises(RuntimeError, match="-95"):  # -ENOTSUP
                g.submit("cu8", rand_block(rng, "cu8", MAX_IN), flags=pkg.XLG_PATH_Q15)
        x = rand_block(rng, "cu8", MAX_IN)
        t = g.submit("cu8", x)
        g.wait(t)
        got.append(g.output(t, cid))
        ref.append(o.process_cf32("cs16", stuff("cu8", x, p["interp"])))
    g.close()
    assert [len(y) for y in got] == [len(y) for y in ref]
    assert_cf32_close(np.concatenate(got), np.concatenate(ref), "after a refused Q15 submit")


def test_argument_errors(pkg):
    taps = np.ones(8, dtype=np.float32)
    g = pkg.Group(2048000, MAX_IN)
    for L, M in [(0, 5), (3, 0), (2098, 1)]:  # 2098 * 2048000 > UINT32_MAX
        with pytest.raises(ValueError, match="-22"):
            g.add_client_rational(L, M, taps, 0)
    with pytest.raises(ValueError, match="-1"):
        g.add_client_rational(3, 128, np.zeros(0, np.float32), 0)
    assert g.client_count() == 0
    g.close()
    g = pkg.Group(1000, MAX_IN)
    with pytest.raises(ValueError, match="-22"):  # 65536 * 32768 = 2^31 upsampled samples per block
        g.add_client_rational(65536, 1, taps, 0)
    g.remove_client(g.add_client_rational(65535, 65536, taps, 0))
    g.close()


@pytest.mark.parametrize("kind", [TILED, GENERIC], ids=["tiled", "generic"])
def test_counters_and_kind(pkg, monkeypatch, kind):
    if kind == GENERIC:
        monkeypatch.setenv("XLATING_B200_POLY_TILE", "0")
    fs = 2048000
    plan = pkg.rational_plan(fs, [48000] * 8)
    g = pkg.Group(fs, MAX_IN)
    g.profile_enable(True)
    ids = [g.add_client_rational(p["interp"], p["decim"], p["taps"], p["center"]) for p in plan]
    rng = np.random.default_rng(2)
    want, launched = 0, 0
    for n in RAGGED:
        t = g.submit("cu8", rand_block(rng, "cu8", n))
        g.wait(t)
        counts = [len(g.output(t, c)) for c in ids]
        launched += max(counts) > 0
        want += sum(k * -(-p["taps"].size // p["interp"]) for k, p in zip(counts, plan))
    assert {g.client_info(c)[1] for c in ids} == {kind}
    pp, prof = g.poly_profile_read(), g.profile_read()
    g.close()
    assert pp["poly_macs"] == prof["algo_macs"] == want > 0
    name, other = ("tile", "generic") if kind == TILED else ("generic", "tile")
    assert pp[f"fir_poly_{name}_launches"] == launched and pp[f"fir_poly_{name}_ms"] > 0
    assert pp[f"fir_poly_{other}_launches"] == 0
    assert prof["fir_generic_launches"] == 0 and prof["fir_tile_launches"] == 0
