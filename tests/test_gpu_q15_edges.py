"""The Q15 path (process_*_cs16, XLG_PATH_Q15) bit for bit at the edges of integer arithmetic, against the model of
tests/q15.py and, where it is cheap, the strict oracle.

* test_group_edges: a batch group per format with every filter of q15.edge_clients -- the product pair that
  wraps in 32 bits (x = tap = (-32768, -32768)) mixed into random data, gain > 1 taps on full-scale rails at a
  45 degree centre, the taps whose Q15 conversion wraps, the limit-cycle centres and one-hot taps at random
  centres -- fed ragged, odd and empty blocks with XLG_SLOTS tickets in flight.
* test_group_narrowing: 65537 taps whose windows take acc >> 15 past 2^31 at a nonzero centre, so that the
  (int32) narrowing before sat16 decides the output.
* test_dropin_edges: the same filters and the 65537-tap one on the per-filter engine, native and optimized, on
  its own kernels, through XLATING_B200_DROPIN=group, and with combined calls on one lane without the shared
  input cache (tests/_q15_edges_worker.py, a subprocess each).
* test_limit_cycles_past_2_32: Q15 clients at nonzero centres, whose oscillator keeps a limit cycle of nonzero
  magnitude, past 2^31 and 2^32 input samples, checked on windows against the model with the phase walked to
  the window's first output (tests/long_stream.py).
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

import q15
from exact import assert_exact
from long_stream import N, SLOTS, Pump, window_start
from oracle import pyoracle as po

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FS = q15.FS
MAX_IN = 2 * 70000


def run_group(pkg, fmt, clients, blocks):
    """Feed `blocks` to a group with `clients` [(label, taps, D, centre)], SLOTS tickets in flight; returns
    the outputs per client and block."""
    g = pkg.Group(FS, MAX_IN)
    ids = [g.add_client(D, taps, c) for _, taps, D, c in clients]
    got = [[] for _ in clients]
    pending = []

    def retire():
        t, _ = pending.pop(0)
        g.wait(t)
        for i, cid in enumerate(ids):
            got[i].append(g.output(t, cid, q15=True))

    for x in blocks:
        pending.append((g.submit(fmt, x, flags=pkg.XLG_PATH_Q15), x))  # the block stays alive until waited for
        if len(pending) >= SLOTS:
            retire()
    while pending:
        retire()
    g.close()
    return got


def check(pkg, fmt, clients, blocks, got, oracle_below=1000):
    lib = pkg.lib()
    for (label, taps, D, c), y in zip(clients, got):
        want = q15.Client(lib, taps, D, c, FS)(fmt, blocks)
        assert_exact(y, want, f"{fmt} {label} D={D} T={len(taps)} centre={c}: group", len(taps), D)
        if len(taps) < oracle_below:
            o = po.OracleFilter(D, taps, c, FS, MAX_IN)
            assert_exact(want, [o.process_q15(fmt, x) for x in blocks], f"{fmt} {label}: model against the oracle")


@pytest.mark.parametrize("fmt", ["cu8", "cs8", "cs16"])
def test_group_edges(pkg, fmt):
    rng = np.random.default_rng({"cu8": 51, "cs8": 52, "cs16": 53}[fmt])
    clients = q15.edge_clients(rng, fmt)
    blocks = q15.edge_blocks(rng, fmt, q15.RAGGED + q15.RAGGED[::-1])
    got = run_group(pkg, fmt, clients, blocks)
    check(pkg, fmt, clients, blocks, got)
    # the wrap case met some outputs, not all: the widened pair gives other outputs there
    lib = pkg.lib()
    rev, qinc, _ = q15.host_consts(lib, q15.WRAP_TAPS, 1, q15.WRAP_CENTER, FS)
    wide = q15.model(rev, qinc, 1, fmt, blocks, arith=q15.MUTATIONS["pair widened to int64"])
    n = sum(int(np.sum(np.any(a != b, axis=1))) for a, b in zip(wide, got[0]))
    assert 0 < n < sum(len(y) for y in got[0]) // 2, n


def test_group_narrowing(pkg):
    rng = np.random.default_rng(54)
    taps = q15.narrowing_taps(65537, 300000, FS)
    rev, _, _ = q15.host_consts(pkg.lib(), taps, 4096, 300000, FS)
    assert np.all((rev == -32768).any(axis=1))
    blocks = q15.narrowing_blocks(rng, rev)
    clients = [("narrowing", taps, 4096, 300000), ("wrap", q15.WRAP_TAPS, 1, q15.WRAP_CENTER)]
    got = run_group(pkg, "cs16", clients, blocks)
    check(pkg, "cs16", clients, blocks, got, oracle_below=70000)
    wide = q15.model(rev, q15.host_consts(pkg.lib(), taps, 4096, 300000, FS)[1], 4096, "cs16", blocks,
                     arith=q15.MUTATIONS["(int32) narrowing dropped"])
    assert np.any(wide[0][16] != got[0][0][16])


@pytest.mark.parametrize("variant,env", [("native", {}), ("optimized", {}),
                                         ("native", {"XLATING_B200_DROPIN": "group"}),
                                         ("optimized", {"XLATING_B200_LANES": "1", "XLATING_B200_SHARE": "0"})],
                         ids=["native", "optimized", "dropin_group", "lanes1_noshare"])
def test_dropin_edges(variant, env):
    e = dict(os.environ)
    e.update(env)
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "_q15_edges_worker.py"), variant],
                       capture_output=True, text=True, timeout=900, env=e)
    assert r.stdout.strip(), r.stderr[-3000:]
    line = json.loads(r.stdout.strip().splitlines()[-1])
    print(f"\n{line}")
    assert r.returncode == 0 and not line["errors"], (line, r.stderr[-2000:])
    assert line["checked"] == line["filters"] >= 3 * 14 + 1
    if env.get("XLATING_B200_DROPIN") != "group":
        batches, calls, _ = line["stats"]
        assert batches < calls  # calls of many filters were combined into one launch


# ---------------------------------------------------------------------------
# past 2^32 input samples
# ---------------------------------------------------------------------------
LONG_FS = 61_440_000
P31, P32 = 2 ** 31, 2 ** 32


def test_limit_cycles_past_2_32(pkg):
    """The limit-cycle centres of q15.LIMIT_CENTERS scaled to 61.44 Msps (the same w0), at D = 5 and 21, and
    a wrap-case client; checked near the start, across 2^31 and across 2^32 (a ragged pair of odd lengths
    there), and a client attached past 2^32."""
    rng = np.random.default_rng(61)
    g = pkg.Group(LONG_FS, 2 * N)
    lib = pkg.lib()
    live = []  # [cid, D, taps, centre, attach block, model]
    got = {}

    def add(at, D, taps, c):
        live.append([g.add_client(D, taps, c), D, taps, c, at, q15.Client(lib, taps, D, c, LONG_FS)])

    for i, c in enumerate(q15.LIMIT_CENTERS):
        add(0, (5, 21)[i % 2], rng.uniform(-0.9, 0.9, (16, 33)[i % 2]).astype(np.float32), 30 * c)
    add(0, 5, q15.WRAP_TAPS, 30 * q15.WRAP_CENTER)

    def read(t, i):
        got[i] = {cl[0]: g.output(t, cl[0], q15=True) for cl in live if cl[4] <= i}

    bufs = [q15.wrap_input(rng, "cs16", N) if k % 2 else q15.rail_input(rng, "cs16", N) for k in range(4)]
    p = Pump(torch, pkg, g, "cs16", bufs, 62, flags=pkg.XLG_PATH_Q15, read=read)
    live_data = []

    def check(idx, label):
        p.drain()
        c0, c1 = idx[0], idx[-1] + 1
        for cid, D, taps, c, at, model in live:
            if at > c0:
                continue
            b = window_start(p.starts, c0, p.starts[at], D, len(taps))
            k0 = (p.starts[b] - p.starts[at]) // D
            want = model("cs16", p.blocks[b:c1], k0=k0)[c0 - b:]
            ys = [got[i][cid] for i in range(c0, c1)]
            assert_exact(ys, want, f"{label}: Q15 client {cid} D={D} T={len(taps)} centre={c} attached at block "
                         f"{at}, window from block {b} (output {k0})", len(taps), D)
            live_data.append(any(np.any(y) for y in ys))
        for i in range(c0, c1):
            got.pop(i, None)

    def watch_feed(n):
        idx = list(range(len(p.blocks), len(p.blocks) + n))
        p.watch.update(idx)
        for _ in range(n):
            p.feed()
        return idx

    check(watch_feed(2), "control")
    for pos in (P31, P32):
        p.run_to(pos - N)
        idx = watch_feed(1)
        a = pos - pos // N * N + 101
        a += 1 - a % 2  # odd
        p.watch.update({len(p.blocks), len(p.blocks) + 1})
        i = p.pair(a)
        check(idx + [i, i + 1] + watch_feed(1), f"2^{31 if pos == P31 else 32}")
    p.feed(0, 0, 12347)  # odd: the next block starts at a position no D divides
    p.drain()
    add(len(p.blocks), 21, rng.uniform(-0.9, 0.9, 33).astype(np.float32), 30 * 640000)
    check(watch_feed(2), "attached past 2^32")
    assert p.S > P32
    # past 2^32 most oscillators still turn: their outputs carry data
    assert sum(live_data[-len(live):]) >= len(live) - 2, live_data[-len(live):]
    g.close()
