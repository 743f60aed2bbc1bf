"""Every FIR kernel, bit for bit, against the float64 reference on exactly representable stimuli.

Centre frequency 0, distinct dyadic taps per client and inputs on an 8-bit grid (tests/exact.py):
every partial sum in every order is an exact float32 number, so the tiled, generic and split-K
kernels, the warp-shuffle and ordered reductions and the drop-in engine must all return exactly
the float64 result.  Unlike the 1e-5 float contract this sees a dropped first or last tap, a
window one sample off, a history sample that should read as zero, and a client reading another
client's taps.  The Q15 path is checked against the int64 twin on the same stimuli.

The phase harness then covers the oscillator at any centre: with one-hot taps and a real input
each accumulator is a single rounded product in the oracle and on the GPU alike, so the output
must equal the strict float32 oracle bit for bit -- the even/odd phase step, the group stride,
ph_base, per-call renormalisation and speculation with restore after client churn.
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from exact import (assert_exact, dyadic_taps, exact_input, grid_step, one_hot_taps, real_input, ref_f64_many,
                   ref_q15)
from oracle import pyoracle as po

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

FS, MAX_IN = 2016000, 65536
FS5, MAX_IN5 = 61440000, 131072
GENERIC, TILED, LONG = 0, 1, 2


class Client:
    def __init__(self, cid, D, taps, first_block):
        self.cid, self.D, self.taps, self.first = cid, D, taps, first_block
        self.last = None  # first block it no longer sees (detached)
        self.got, self.kinds = [], set()


def drive(pkg, monkeypatch, plan, sizes, fmt="cu8", fs=FS, max_in=MAX_IN, env=None, flags=0, host_ring=0,
          attach=None, detach=None, depth=1, q15=False, seed=0, profile=False):
    """Run a group over exact stimuli and check every output of every client of every block.

    plan: [(D, T)] at block 0; attach: {block: [(D, T)]} joins before that block; detach:
    {block: [client index]} leaves before it.  depth > 1 keeps that many tickets in flight.
    Returns (clients, profile counters or None)."""
    for k, v in (env or {}).items():
        monkeypatch.setenv(k, v)
    rng = np.random.default_rng(seed)
    g = pkg.Group(fs, max_in, flags=flags, host_ring=host_ring)
    if profile:
        g.profile_enable(True)
    clients = []

    def add(specs, b):
        for D, T in specs:
            taps = dyadic_taps(rng, T, fmt, k=15 if q15 else None)
            clients.append(Client(g.add_client(D, taps, 0), D, taps, b))

    add(plan, 0)
    blocks = [exact_input(rng, fmt, n) for n in sizes]
    pending = []

    def collect(b, t):
        g.wait(t)
        for c in clients:
            if c.first <= b and (c.last is None or b < c.last):
                if flags & pkg.XLG_OUT_DEVICE:
                    y = g.read_output(t, c.cid, q15=q15)
                else:
                    y = g.output(t, c.cid, q15=q15)
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
        pending.append((b, g.submit(fmt, x, flags=pkg.XLG_PATH_Q15 if q15 else 0)))
        if len(pending) >= depth:
            collect(*pending.pop(0))
    while pending:
        collect(*pending.pop(0))
    prof = g.profile_read() if profile else None
    g.close()

    # references: clients of one (D, T) that saw the same blocks share one matrix product
    groups = {}
    for c in clients:
        groups.setdefault((c.D, c.taps.size, c.first, c.last), []).append(c)
    for (D, T, first, last), cs in groups.items():
        seen = blocks[first:last]
        if q15:
            refs = [ref_q15(c.taps, D, fmt, seen) for c in cs]
        else:
            refs = ref_f64_many([c.taps for c in cs], D, fmt, seen)
        for c, r in zip(cs, refs):
            assert_exact(c.got, r, f"{env or ''} flags={flags} client {c.cid} (D={D}, T={T}, from block {first})",
                         T, D, None if q15 else grid_step(c.taps, fmt))
    return clients, prof


def kinds_of(clients, pick=lambda c: True):
    out = set()
    for c in clients:
        if pick(c):
            out |= c.kinds
    return out


# mixed classes of the 2.016 Msps band: natural layout (D = 42, 21), skewed layout (D = 8)
MIXED = [(42, 505)] * 16 + [(21, 253)] * 16 + [(8, 97)] * 8
RAGGED = [65536, 65536, 30001, 2, 0, 65536, 12347, 65536, 7, 65534]


# ---------------------------------------------------------------------------
# batch ABI: every kernel kind
# ---------------------------------------------------------------------------
def test_generic_kernel(pkg, monkeypatch):
    """XLG_FORCE_GENERIC, and classes too small for a tile (< 8 clients), T = 1 and even T among them."""
    cl, prof = drive(pkg, monkeypatch, MIXED + [(1, 1)] * 3 + [(2, 2)] * 2 + [(7, 64)] * 3, RAGGED,
                     flags=pkg.XLG_FORCE_GENERIC, profile=True, seed=1)
    assert kinds_of(cl) == {GENERIC}
    assert prof["fir_tile_launches"] == 0 and prof["fir_long_launches"] == 0 and prof["fir_generic_launches"] > 0
    cl, _ = drive(pkg, monkeypatch, [(42, 505)] * 7 + [(21, 254)] * 5 + [(1, 1)] * 3 + [(5, 40)] * 2, RAGGED, seed=2)
    assert kinds_of(cl) == {GENERIC}


@pytest.mark.parametrize("shape", [None, "1642", "1641", "1621", "1611", "3241", "1651"])
def test_tiled_kernel_shapes(pkg, monkeypatch, shape):
    """Every tile shape on the natural and the skewed layout, ragged and odd-length blocks, and a
    second wave of clients that attaches mid-stream (generic until its zero history has passed,
    then its own window alignment inside a merged class).  3241 (the retired LO = 32 shape) and
    1651 are not shapes: they are ignored and the automatic choice runs."""
    env = {"XLATING_B200_TILE": shape} if shape else {}
    cl, prof = drive(pkg, monkeypatch, MIXED, RAGGED, env=env, attach={2: [(42, 505)] * 8 + [(21, 253)] * 8},
                     profile=True, seed=3)
    assert kinds_of(cl, lambda c: c.first == 0) == {TILED}
    assert TILED in kinds_of(cl, lambda c: c.first > 0)
    assert prof["fir_tile_launches"] > 0


@pytest.mark.parametrize("env", [{"XLATING_B200_SKEWED": "1"}, {"XLATING_B200_NO_MERGE": "1"}],
                         ids=["skewed", "no_merge"])
def test_tiled_kernel_layout_switches(pkg, monkeypatch, env):
    cl, _ = drive(pkg, monkeypatch, MIXED, RAGGED, env=env, attach={2: [(42, 505)] * 8}, seed=4)
    assert kinds_of(cl, lambda c: c.first == 0) == {TILED}


def test_tiled_kernel_tap_counts(pkg, monkeypatch):
    """T over every residue mod 8 (the flat rows are padded to L, a multiple of 8), just below, at and
    above multiples of D, even T: one class of 8 clients each."""
    Ts = [160, 161, 162, 163, 164, 165, 166, 167, 168, 169, 125, 126, 127, 189, 190]
    plan = [(21, T) for T in Ts for _ in range(8)] + [(8, T) for T in (63, 64, 65) for _ in range(8)]
    cl, _ = drive(pkg, monkeypatch, plan, [65536, 30001, 65536, 3, 65536], seed=5)
    assert kinds_of(cl) == {TILED}


LONG_PLAN = [(1280, 2561)] * 8 + [(1280, 1407)] * 12 + [(1280, 1281)] * 8 + [(1280, 3840)] * 8
LONG_SIZES = [MAX_IN5, 50002, MAX_IN5, MAX_IN5, 30006, MAX_IN5, MAX_IN5, 131070, MAX_IN5, MAX_IN5, MAX_IN5, 2]


@pytest.mark.parametrize("plan, env", [(LONG_PLAN, {}), (LONG_PLAN, {"XLATING_B200_LONG_TMAP": "0"}),
                                       ([(1280, 2561)] * 8 + [(1279, 2561)] * 8, {})],
                         ids=["default", "no_tmap", "mixed_parity"])
def test_split_k_kernels(pkg, monkeypatch, plan, env):
    """The split-K long-filter kernels: T just above and below multiples of D and of the 128-tap
    segment, odd window starts (odd block lengths), and a ring wrap-around.  fir_long4 with and without
    its strip tensor map; an odd-D class in the group sends the even-D class to fir_long2 as well,
    whose strips then alternate between aligned bulk copies and cp.async with the window start."""
    cl, prof = drive(pkg, monkeypatch, plan, LONG_SIZES, fmt="cs16", fs=FS5, max_in=MAX_IN5, env=env,
                     profile=True, seed=6)
    assert kinds_of(cl) == {LONG}
    assert prof["fir_long_launches"] > 0 and prof["fir_tile_launches"] == 0


def test_split_k_disabled(pkg, monkeypatch):
    cl, prof = drive(pkg, monkeypatch, LONG_PLAN[:16], LONG_SIZES[:4], fmt="cs16", fs=FS5, max_in=MAX_IN5,
                     env={"XLATING_B200_NO_LONG": "1"}, profile=True, seed=7)
    assert kinds_of(cl) == {GENERIC}
    assert prof["fir_long_launches"] == 0


def test_split_k_odd_decimation(pkg, monkeypatch):
    """Odd D (cp.async strips, many output tiles) with 24001 taps (M = 1)."""
    cl, _ = drive(pkg, monkeypatch, [(5, 24001)] * 9, [16384, 16383, 16384], fs=1000000, max_in=16384, seed=8)
    assert kinds_of(cl) == {LONG}


# ---------------------------------------------------------------------------
# stream edges and pipeline variants
# ---------------------------------------------------------------------------
def test_attach_detach_and_ring_wrap(pkg, monkeypatch):
    """Clients join while the stream runs (their first windows overlap real history that must read as
    zero) and leave; empty, 1-sample and ragged blocks; enough blocks to wrap the ring many times."""
    sizes = [32768, 2, 0, 32767, 32768, 1000, 32768, 32768, 5, 32768] * 4
    cl, _ = drive(pkg, monkeypatch, [(42, 505)] * 12 + [(21, 253)] * 9 + [(8, 97)] * 3, sizes, max_in=32768,
                  attach={3: [(42, 505)] * 9 + [(21, 300)] * 2, 11: [(21, 253)] * 8, 25: [(8, 97)] * 8},
                  detach={5: [0, 13], 20: [2, 3, 4]}, seed=9)
    assert {GENERIC, TILED} <= kinds_of(cl)


PIPE_ENVS = [{}, {"XLATING_B200_CONV_STREAM": "0"}, {"XLATING_B200_SPECULATE": "0", "XLATING_B200_CSTREAMS": "1"},
             {"XLATING_B200_PARTITION": "1"}, {"XLATING_B200_PARTITION": "0"}]


@pytest.mark.parametrize("env", PIPE_ENVS, ids=["default", "conv_on_compute_stream", "no_spec_1stream", "partition",
                                                "no_partition"])
def test_tickets_in_flight(pkg, monkeypatch, env):
    drive(pkg, monkeypatch, MIXED + [(5, 40)] * 2, [65536] * 5 + [30001, 65536, 65536, 12347, 65536], env=env,
          depth=pkg.XLG_SLOTS, seed=10)


def test_partition_device_output_and_host_ring(pkg, monkeypatch):
    drive(pkg, monkeypatch, MIXED, RAGGED, flags=pkg.XLG_SM_PARTITION, seed=11)
    drive(pkg, monkeypatch, MIXED + [(5, 40)] * 2, RAGGED, flags=pkg.XLG_OUT_DEVICE, seed=12)
    drive(pkg, monkeypatch, MIXED, RAGGED + RAGGED, host_ring=12, depth=12, seed=13)


def test_q15_path(pkg, monkeypatch):
    cl, _ = drive(pkg, monkeypatch, [(42, 505)] * 8 + [(21, 253)] * 9 + [(1, 1)] * 2 + [(8, 64)] * 3,
                  [32768, 30001, 2, 0, 32768], fmt="cs8", max_in=32768, q15=True, seed=14)
    cl, _ = drive(pkg, monkeypatch, [(21, 253)] * 4, [32768, 7, 32768], fmt="cu8", max_in=32768, q15=True,
                  attach={1: [(21, 253)] * 2}, seed=15)


# ---------------------------------------------------------------------------
# full-size shapes, every client checked
# ---------------------------------------------------------------------------
def test_full_size_cfg2(pkg, monkeypatch):
    """BASELINE configs[1]: 256 clients at 48 / 96 ksps from 2.016 Msps, 262144-byte cu8 blocks."""
    T48 = len(pkg.create_low_pass_filter(1.0, FS, 24000, 9600))
    T96 = len(pkg.create_low_pass_filter(1.0, FS, 48000, 19200))
    plan = [(42, T48) if c % 2 == 0 else (21, T96) for c in range(256)]
    cl, _ = drive(pkg, monkeypatch, plan, [262144] * 3, max_in=262144, seed=16)
    assert kinds_of(cl) == {TILED}


def test_full_size_config5_shape(pkg, monkeypatch):
    """BASELINE configs[4]'s filter: 61.44 Msps cs16, D = 1280, T = 15419 (M = 7)."""
    T = len(pkg.create_low_pass_filter(1.0, FS5, 24000, 9600))
    assert T == 15419
    cl, _ = drive(pkg, monkeypatch, [(1280, T)] * 40, [MAX_IN5, 50002, MAX_IN5, MAX_IN5], fmt="cs16", fs=FS5,
                  max_in=MAX_IN5, seed=17)
    assert kinds_of(cl) == {LONG}


# ---------------------------------------------------------------------------
# the phase harness: one-hot taps, real input, any centre -> bit-exact against the strict oracle
# ---------------------------------------------------------------------------
def phase_harness(pkg, monkeypatch, fs, max_in, D, T, n_clients, n_blocks, env=None, flags=0, seed=0):
    for k, v in (env or {}).items():
        monkeypatch.setenv(k, v)
    rng = np.random.default_rng(seed)
    g = pkg.Group(fs, max_in, flags=flags)
    live = []  # [cid, oracle, label]
    band = fs // 2 - fs // (2 * D)

    def add(i):
        j = (0, T - 1, int(rng.integers(1, T - 1)) if T > 2 else 0)[i % 3]
        center = int(rng.integers(-band, band))
        taps = one_hot_taps(T, j, float(rng.choice([0.75, -0.5, 0.3125])))
        live.append([g.add_client(D, taps, center), po.OracleFilter(D, taps, center, fs, max_in),
                     f"j={j} centre={center}"])

    for i in range(n_clients):
        add(i)
    renorm = not (flags & pkg.XLG_NO_RENORM)
    kinds, added = set(), n_clients
    for b in range(n_blocks):
        if b % 37 == 20:  # churn: one client leaves, one joins (speculation must restore)
            g.remove_client(live.pop(int(rng.integers(0, len(live))))[0])
            add(added)
            added += 1
        n = int(rng.choice([max_in, max_in, max_in - 2, int(rng.integers(0, max_in // 2)) * 2, 2]))
        x = real_input(rng, n)
        t = g.submit("cs16", x)
        g.wait(t)
        for cid, o, label in live:
            assert_exact(g.output(t, cid), o.process_cf32("cs16", x, renorm=renorm), f"{env} block {b} {label}")
            kinds.add(g.client_info(cid)[1])
    g.close()
    return kinds


PHASE_VARIANTS = [({}, 0), ({}, "XLG_NO_RENORM"), ({"XLATING_B200_SPECULATE": "0"}, 0),
                  ({"XLATING_B200_PARTITION": "1"}, "XLG_SM_PARTITION")]


@pytest.mark.parametrize("env,flag", PHASE_VARIANTS, ids=["default", "no_renorm", "no_speculation", "partition"])
def test_phase_harness(pkg, monkeypatch, env, flag):
    flags = getattr(pkg, flag) if flag else 0
    kinds = phase_harness(pkg, monkeypatch, FS, 16384, 21, 253, 20, 300, env, flags, seed=18)
    assert TILED in kinds
    kinds = phase_harness(pkg, monkeypatch, FS, 16384, 42, 200, 4, 300, env, flags | pkg.XLG_FORCE_GENERIC, seed=19)
    assert kinds == {GENERIC}
    kinds = phase_harness(pkg, monkeypatch, FS5, 16384, 1280, 1407, 10, 300, env, flags, seed=20)
    assert LONG in kinds


# ---------------------------------------------------------------------------
# per-filter drop-in ABI
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("variant", ["native", "optimized"])
@pytest.mark.parametrize("fmt", ["cu8", "cs8", "cs16"])
def test_dropin_filters(pkg, fmt, variant):
    rng = np.random.default_rng(21)
    sizes = [40000, 2, 39, 12346, 0, 40000, 7, 40000]
    for D, T in ((21, 253), (42, 505), (1, 1), (7, 64), (8, 8)):
        taps = dyadic_taps(rng, T, fmt)
        qtaps = dyadic_taps(rng, T, fmt, k=15)
        f = pkg.XlatingFilter(D, taps, 0, FS, 40000)
        fq = pkg.XlatingFilter(D, qtaps, 0, FS, 40000)
        blocks = [exact_input(rng, fmt, n) for n in sizes]
        got = [f.process_cf32(fmt, x, variant) for x in blocks]
        gotq = [fq.process_q15(fmt, x, variant) for x in blocks]
        assert_exact(got, ref_f64_many([taps], D, fmt, blocks)[0], f"{fmt} {variant} D={D} T={T}", T, D,
                     grid_step(taps, fmt))
        assert_exact(gotq, ref_q15(qtaps, D, fmt, blocks), f"Q15 {fmt} {variant} D={D} T={T}", T, D)
        f.close()
        fq.close()


def run_overlay(scenario, env=None, clients=24, blocks=16):
    e = dict(os.environ)
    e.update(env or {})
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "_dropin_overlay_worker.py"), scenario,
                        str(clients), str(blocks), "exact"], capture_output=True, text=True, timeout=600, env=e)
    assert r.stdout.strip(), r.stderr[-2000:]
    line = json.loads(r.stdout.strip().splitlines()[-1])
    assert r.returncode == 0 and not line["errors"], (line, r.stderr[-1500:])
    return line["stream"]


@pytest.mark.parametrize("scenario", ["steady", "drops", "late", "lag"])
def test_dropin_overlay_exact(scenario):
    """Filters of one band handed into and out of a batch group: the state handed over (history,
    valid_history, phase) is right to the sample."""
    st = run_overlay(scenario, env={"XLATING_B200_STREAM_RING": "4"} if scenario == "lag" else None)
    assert st["joins"] > 0


@pytest.mark.parametrize("env", [{"XLATING_B200_LANES": "1"}, {"XLATING_B200_LANES": "8"},
                                 {"XLATING_B200_SHARE": "0"}, {"XLATING_B200_OSC": "lanes"},
                                 {"XLATING_B200_OSC": "host"}, {"XLATING_B200_OSC": "device"},
                                 {"XLATING_B200_STREAM": "0", "XLATING_B200_LANES": "2"}],
                         ids=["lanes1", "lanes8", "no_share", "osc_lanes", "osc_host", "osc_device", "private_lanes2"])
def test_dropin_engine_switches(env):
    run_overlay("drops", env=env, clients=16, blocks=10)
