"""Every kernel family bit for bit past 2^31 and 2^32 input samples.

A group at 61.44 Msps is pumped with device blocks of N = 967680 complex cs16 samples (tests/long_stream.py)
past 2^32 input samples, about 4440 submits with no PCIe traffic and no outputs read except on the checked
ranges.  Each range is checked, block by block and for every live client, against the float64 (or bit-exact
model) reference of a fresh client fed the blocks from a boundary whose distance from the client's attach
point is a multiple of its period (the window argument of tests/long_stream.py, checked on CPU by
tests/test_long_stream_reference.py).  At 2^31 and 2^32 one block is replaced by a ragged pair of odd lengths
whose first part ends 101 samples past the power of two: windows straddle it, and the stream's parity flips
between the two parts.

* test_every_family_past_2_32: one group with every family (generic, tiled natural and skewed, split-K long
  on fir_long4, rational tiled and generic, integer and rational cascades, a sub-band with an integer and an
  L2 > 1 member, members of two banks, K = 30 and K = 32).  Ranges: a control near the start, 2^31, 2^32,
  and the blocks where the rational clients' (63/640, 3/128) upsampled positions pass 2^31 and 2^32.  After 2^32, inside a
  second ragged pair, older clients are detached and new ones attached at a new alignment: two that merge into
  the natural D = 21 class as their own subgroup, a lone one that stays generic, an odd-D long class (which
  moves the long launch to fir_long2), a rational tiled class, a cascade, a sub-band with members and a new
  channel of the K = 30 bank; each is checked from its attach point.  The pipeline variants (one compute
  stream without speculation, the SM partition, device outputs) run the same group, with the odd-D long class
  from the start, past 2^31 only, which keeps the file's wall time down.
* test_q15_past_2_32: integer clients on the Q15 path.  The reference's Q15 oscillator is never
  renormalised and reaches 0 after 32767 outputs, so clients running since the start are checked for their
  output counts and zeros, and fresh clients attached before 2^31, before 2^32 and after 2^32 against ref_q15.
* test_dropin_past_2_32: drop-in filters (integer, rational, cascade) on the per-filter engine, and two
  integer filters of one band served by the stream overlay's batch group, past 2^32 (a subprocess each).
"""
import json
import os
import subprocess
import sys
import time

import numpy as np
import pytest

from cascade import small_taps
from exact import assert_exact, dyadic_taps, exact_input, ref_q15
from long_stream import N, Pump, fresh_refs, history, period, window_start
from subband_rig import dyadic_member, dyadic_stage_a

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FS, FMT, MAX_IN = 61_440_000, "cs16", 2 * N
P31, P32 = 2 ** 31, 2 ** 32
N_BUFS = 4


def ragged(pos, avoid=1):
    """a: the first part of the ragged pair replacing the block that holds pos, odd, ending 101 or more samples
    past pos, and (avoid > 1) leaving the second part at a position that is not a multiple of avoid."""
    a = pos - pos // N * N + 101
    while a % 2 == 0 or (avoid > 1 and a % avoid == 0):
        a += 2
    return a


def bufs(seed):
    rng = np.random.default_rng(seed)
    return [exact_input(rng, FMT, 2 * N) for _ in range(N_BUFS)]


class Cl:
    """A client: spec (tests/long_stream.py), the kind xlg_client_info must report (sub-band members: the
    sub-band kind too), its attach block, and for a bank channel materialised late the block it was."""

    def __init__(self, cid, spec, kind, attach, mat=None):
        self.cid, self.spec, self.kind, self.attach, self.mat = cid, spec, kind, attach, mat


def add_population(g, rng, odd_long, attach=0):
    """Every family at centre 0 with exact stimuli; returns [Cl]."""
    cl = []

    def ints(D, T, n, kind):
        for _ in range(n):
            t = dyadic_taps(rng, T, FMT)
            cl.append(Cl(g.add_client(D, t, 0), ("int", D, t), kind, attach))

    ints(5, 16, 2, 0)        # a class smaller than 8: generic
    ints(21, 129, 8, 1)      # natural layout
    ints(42, 64, 8, 1)
    ints(8, 24, 8, 1)        # skewed layout
    ints(1280, 2561, 8, 2)   # split-K long class, even D: fir_long4
    if odd_long:
        ints(945, 4001, 8, 2)  # odd D: the long launch runs fir_long2
    for _ in range(8):       # rational tiled class: 3/128, ceil(T/L) = 130
        t = dyadic_taps(rng, 390, FMT)
        cl.append(Cl(g.add_client_rational(3, 128, t, 0), ("rat", 3, 128, t), 4, attach))
    t = dyadic_taps(rng, 1764, FMT)  # 63/640: no tile holds its branches (L * fs must stay below 2^32)
    cl.append(Cl(g.add_client_rational(63, 640, t, 0), ("rat", 63, 640, t), 3, attach))
    for d1, t1, l2, d2, t2 in ((6, 25, 1, 7, 29), (8, 17, 3, 16, 47)):
        a, b = small_taps(rng, t1, 3), small_taps(rng, t2, 3)
        cl.append(Cl(g.add_client_cascade(d1, a, 0, d2, b, interp2=l2), ("casc", d1, a, l2, d2, b), 5, attach))
    cl += subband(g, rng, attach)
    for d1, t1, chans in ((15, 60, ((3, 4, 33), (-7, 4, 17))), (16, 64, ((5, 5, 21),))):
        taps1 = small_taps(rng, t1, 2)
        bid = g.add_bank(d1, taps1)
        for k, d2, t2 in chans:
            taps2 = small_taps(rng, t2, 3)
            cid = g.add_client_subband(g.add_bank_subband(bid, k), d2, taps2, 0)
            cl.append(Cl(cid, ("bank", d1, taps1, k, d2, taps2), (6, 7), attach))
        if d1 == 15:
            bank15 = (bid, taps1)  # K = 30: not a power of two, so r0 depends on every bit of a position
    return cl, bank15


def subband(g, rng, attach):
    t1 = dyadic_stage_a(rng, 32, 64)
    sid = g.add_subband(32, t1, 0)
    out = []
    for l2, d2, t2 in ((1, 16, 33), (3, 40, 61)):
        taps2 = dyadic_member(rng, t1, t2, FMT)
        cid = g.add_client_subband(sid, d2, taps2, 0, interp2=l2)
        out.append(Cl(cid, ("sub", 32, t1, l2, d2, taps2), (6, (0, 1, 2)), attach))
    return out


def kind_ok(g, c):
    if isinstance(c.kind, tuple):
        ck, sk = c.kind
        _, got_sk, _ = g.subband_info(c.cid)
        return g.client_info(c.cid)[1] == ck and (got_sk in sk if isinstance(sk, tuple) else got_sk == sk)
    return g.client_info(c.cid)[1] == c.kind


class Run:
    """One group, its clients and the outputs of the watched blocks."""

    def __init__(self, pkg, flags, odd_long, seed):
        self.g = pkg.Group(FS, MAX_IN, flags=flags)
        self.rng = np.random.default_rng(seed)
        self.clients, self.bank15 = add_population(self.g, self.rng, odd_long)
        self.got = {}
        self.pump = Pump(torch, pkg, self.g, FMT, bufs(seed + 1), seed + 2, read=self.read)
        self.checked = []

    def read(self, t, i):
        dev = self.g.flags & 0x1
        self.got[i] = {c.cid: (self.g.read_output(t, c.cid) if dev else self.g.output(t, c.cid))
                       for c in self.clients if c.attach <= i}

    def watched(self, n_blocks, first=None):
        """Feed n_blocks watched full blocks (or, first = (k, off, n), that block first)."""
        idx = []
        if first is not None:
            self.pump.watch.add(len(self.pump.blocks))
            idx.append(self.pump.feed(*first))
        for _ in range(n_blocks):
            self.pump.watch.add(len(self.pump.blocks))
            idx.append(self.pump.feed())
        return idx

    def watched_pair(self, pos, extra=1):
        a = ragged(pos)
        self.pump.watch.update(range(len(self.pump.blocks), len(self.pump.blocks) + 2))
        i = self.pump.pair(a)
        return [i, i + 1] + self.watched(extra)

    def check(self, idx, label, which=lambda c: True):
        """Every live client (of `which`) on blocks idx (consecutive) against its window reference."""
        self.pump.drain()
        p = self.pump
        c0, c1 = idx[0], idx[-1] + 1
        groups = {}
        for c in self.clients:
            if c.attach > c0 or not which(c):
                continue
            if c.mat is not None:  # a bank channel materialised late: the bank's frames from a multiple of K
                b = c.mat - 1
                assert p.starts[b] % (2 * c.spec[1]) == 0
                y = fresh_refs([c.spec], FMT, FS, p.blocks[b:c1], mat=1)[0][c0 - c.mat:]
                self.compare(c, y, c0, c1, label, b)
                continue
            b = window_start(p.starts, c0, p.starts[c.attach], period(c.spec), history(c.spec))
            groups.setdefault(b, []).append(c)
        for b, cs in groups.items():
            ys = fresh_refs([c.spec for c in cs], FMT, FS, p.blocks[b:c1])
            for c, y in zip(cs, ys):
                self.compare(c, y[c0 - b:], c0, c1, label, b)
        for i in idx:
            self.got.pop(i, None)
        self.checked.append((label, c0, c1, p.starts[c0], p.starts[c1]))

    def compare(self, c, ref, c0, c1, label, b):
        got = [self.got[i][c.cid] for i in range(c0, c1)]
        s = c.spec
        assert_exact(got, ref, f"{label}: client {c.cid} {s[0]} {[v for v in s[1:] if np.isscalar(v)]} "
                     f"T={len(s[-1])} attached at block {c.attach}, blocks {c0}..{c1 - 1} (positions "
                     f"{self.pump.starts[c0]}..{self.pump.starts[c1]}), window from block {b}")

    def assert_kinds(self, label):
        bad = [(c.cid, c.spec[0], c.kind, self.g.client_info(c.cid)[1]) for c in self.clients if not kind_ok(self.g, c)]
        assert not bad, f"{label}: kinds {bad}"


def rational(c):
    return c.spec[0] == "rat"


def run_group(pkg, flags, odd_long, stop, late):
    r = Run(pkg, flags, odd_long, seed=500 + flags + 10 * odd_long)
    p = r.pump
    t0 = time.perf_counter()
    p.feed()
    p.feed()
    r.check(r.watched(2), "control")
    r.assert_kinds("start")
    # the rational clients' upsampled positions pass 2^31 and 2^32 (63/640 near the start, 3/128 later)
    for pos, L, e in sorted((u // L, L, e) for L in (63, 3) for u, e in ((P31, 31), (P32, 32))):
        p.run_to(pos - N)  # three blocks: the one holding pos, and one that starts past it
        r.check(r.watched(3), f"L = {L}: upsampled position 2^{e} (input {pos})", rational)
    p.run_to(P31)
    r.check(r.watched_pair(P31), "2^31")
    r.assert_kinds("2^31")
    if stop == 31:
        p.drain()
        r.g.close()
        return r, (len(p.blocks), p.S, time.perf_counter() - t0)
    p.run_to(P32)
    r.check(r.watched_pair(P32), "2^32")
    r.assert_kinds("2^32")
    rate = (len(p.blocks), p.S, time.perf_counter() - t0)
    if late:
        late_attaches(r)
    p.drain()
    r.g.close()
    return r, rate


def late_attaches(r):
    """Inside a ragged pair past 2^32: detach older clients, attach one of each family, check them from there."""
    p, g, rng = r.pump, r.g, r.rng
    k = 0
    p.feed()
    a = ragged(p.S, avoid=21)  # odd, so the second part starts at a multiple of neither 21 nor 42
    p.feed(k, 0, a)
    p.drain()
    at = len(p.blocks)
    assert p.S % 21 and p.S % 42 and p.S > P32
    gone = [c for c in r.clients if c.spec[0] == "int" and c.spec[1] == 5] + \
           [c for c in r.clients if c.spec[0] == "casc" and c.spec[3] == 1]
    for c in gone:
        g.remove_client(c.cid)
        r.clients.remove(c)
    new = []

    def int_client(D, T, kind):
        t = dyadic_taps(rng, T, FMT)
        new.append(Cl(g.add_client(D, t, 0), ("int", D, t), kind, at))

    int_client(21, 129, 1)   # two at a new alignment: their own subgroup of the natural D = 21 class
    int_client(21, 129, 1)
    int_client(42, 64, 0)    # a lone alignment: generic
    for _ in range(8):
        int_client(945, 4001, 2)
    for _ in range(8):
        t = dyadic_taps(rng, 390, FMT)
        new.append(Cl(g.add_client_rational(3, 128, t, 0), ("rat", 3, 128, t), 4, at))
    ta, tb = small_taps(rng, 25, 3), small_taps(rng, 29, 3)
    new.append(Cl(g.add_client_cascade(6, ta, 0, 7, tb), ("casc", 6, ta, 1, 7, tb), 5, at))
    new += subband(g, rng, at)
    bid, taps1 = r.bank15
    t2 = small_taps(rng, 33, 3)
    cid = g.add_client_subband(g.add_bank_subband(bid, 10), 4, t2, 0)
    new.append(Cl(cid, ("bank", 15, taps1, 10, 4, t2), (6, 7), at, mat=at))
    reused = {c.cid for c in gone} & {c.cid for c in new}
    assert reused, "client slots were not reused"
    r.clients += new
    r.check(r.watched(4, first=(k, a, N - a)), "attached past 2^32")
    r.assert_kinds("after the attaches")  # settled: the new integer and rational clients joined their classes


VARIANTS = [({}, 0), ({"XLATING_B200_SPECULATE": "0", "XLATING_B200_CSTREAMS": "1"}, 0),
            ({"XLATING_B200_PARTITION": "1"}, "XLG_SM_PARTITION"), ({}, "XLG_OUT_DEVICE")]


@pytest.mark.parametrize("env,flag", VARIANTS, ids=["default", "no_spec_1stream", "partition", "device_out"])
def test_every_family_past_2_32(pkg, monkeypatch, env, flag):
    """Default: past 2^32 with the late attaches; the other variants past 2^31 with fir_long2 from the start."""
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    default = not env and not flag
    flags = getattr(pkg, flag) if flag else 0
    r, (blocks, S, secs) = run_group(pkg, flags, odd_long=not default, stop=32 if default else 31, late=default)
    print(f"\npump: {blocks} blocks, {S} samples in {secs:.1f} s, checks included: {blocks / secs:.0f} blocks/s")
    assert [c[0] for c in r.checked][-1] in ("attached past 2^32", "2^31")


# ---------------------------------------------------------------------------
# the Q15 path
# ---------------------------------------------------------------------------
def test_q15_past_2_32(pkg):
    rng = np.random.default_rng(700)
    g = pkg.Group(FS, MAX_IN)
    shapes = ((21, 129), (21, 129), (5, 16), (640, 1281))
    live = []  # (cid, D, taps, attach block)
    got = {}

    def add(at):
        for D, T in shapes:
            t = dyadic_taps(rng, T, FMT, k=15)
            live.append((g.add_client(D, t, 0), D, t, at))

    def read(t, i):
        got[i] = {cid: g.output(t, cid, q15=True) for cid, _, _, at in live if at <= i}

    p = Pump(torch, pkg, g, FMT, bufs(701), 702, flags=pkg.XLG_PATH_Q15, read=read)
    add(0)

    def check(idx, label):
        p.drain()
        c0, c1 = idx[0], idx[-1] + 1
        for cid, D, t, at in live:
            if at > c0:
                continue
            ys = [got[i][cid] for i in range(c0, c1)]
            if (p.starts[c0] - p.starts[at]) // D > 32768:  # decayed oscillator: zeros, in the window reference's counts
                b = window_start(p.starts, c0, 0, D, len(t))
                ref = ref_q15(t, D, FMT, p.blocks[b:c1])[c0 - b:]
                assert [len(y) for y in ys] == [len(y) for y in ref], f"{label}: client {cid} counts"
                assert all(not np.any(y) for y in ys), f"{label}: client {cid} is not decayed"
            else:        # fresh: data, against ref_q15 from the attach
                ref = ref_q15(t, D, FMT, p.blocks[at:c1])[c0 - at:]
                assert_exact(ys, ref, f"{label}: Q15 client {cid} D={D} T={len(t)} attached at block {at}", len(t), D)
                assert any(np.any(y) for y in ys)
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
        p.drain()
        add(len(p.blocks))  # fresh clients a block before the block at pos: zero_before below 2^31 / 2^32
        idx = watch_feed(1)
        a = ragged(pos)
        p.watch.update({len(p.blocks), len(p.blocks) + 1})
        i = p.pair(a)
        check(idx + [i, i + 1] + watch_feed(1), f"2^{31 if pos == P31 else 32}")
    p.feed()
    p.drain()
    for cid, _, _, at in live[:4]:
        g.remove_client(cid)
    live[:4] = []
    add(len(p.blocks))  # qzero_before past 2^32
    check(watch_feed(2), "attached past 2^32")
    assert p.S > P32
    g.close()


# ---------------------------------------------------------------------------
# drop-in filters
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("scenario", ["engine", "overlay"])
def test_dropin_past_2_32(scenario):
    """engine: an integer, a rational and a cascade filter on the per-filter engine (the stream overlay off);
    overlay: two integer filters of one band, served by the overlay's batch group.  Checked on windows at
    2^31 and 2^32 (tests/_long_stream_dropin_worker.py)."""
    env = dict(os.environ)
    if scenario == "engine":
        env["XLATING_B200_STREAM"] = "0"
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tests", "_long_stream_dropin_worker.py"), scenario],
                       capture_output=True, text=True, timeout=1800, env=env)
    assert r.stdout.strip(), r.stderr[-3000:]
    line = json.loads(r.stdout.strip().splitlines()[-1])
    print(f"\n{line}")
    assert r.returncode == 0 and not line["errors"], (line, r.stderr[-2000:])
    assert line["position"] > P32 and line["checked"] >= 2 * line["filters"]
    if scenario == "overlay":
        assert line["stream"]["served_by_group"] > 0
    else:
        assert line["stream"]["served_by_group"] == 0
