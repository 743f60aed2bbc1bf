"""Worker for tests/test_gpu_dropin_rational.py: rational filters of the per-filter drop-in ABI
(create_rational_frequency_xlating_filter).  Runs in a subprocess because the engine reads its
environment switches (XLATING_B200_STREAM, _OSC, _DROPIN, _STREAM_RING) once per process.

usage: _dropin_rational_worker.py <scenario> [arg]   -> one JSON line, exit code 1 on any error

  interp1 designed|exact   L = 1 filters equal create_frequency_xlating_filter bit for bit (cf32, Q15)
  private <dump_dir>       every rate-table row: counts and 1e-5 against the strict oracle on the
                           zero-stuffed stream, bits against the same clients in a Group on the
                           polyphase generic kernel; outputs saved to <dump_dir>
  exact                    exact stimuli, five L/M/T specs and integer filters, all three formats,
                           one thread per filter: every output equals the float64 sum bit for bit
  combined                 rational, integer cf32 and integer Q15 filters across formats and ragged
                           sizes meet at a barrier every block: every call within the contract
  neighbours               integer filters give the same bits with rational filters alive
  overlay steady|drops|late|lag   24 rational + 4 integer filters of one band, exact stimuli
  q15refuse                a refused Q15 call leaves a member filter's stream untouched
  wide                     exact stimuli at L from 4 to 441 (L >= 16: a call's span of residues is cut at 16;
                           calls with fewer outputs than L), every output equal to the float64 sum
  phase                    branch-one-hot filters at nonzero centres on a real cs16 stream: every output equal
                           to the strict oracle on the zero-stuffed stream bit for bit (oscillator included)
"""
import importlib
import json
import os
import sys
import threading
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import pyoracle as po  # noqa: E402  (checker)
from exact import assert_exact, dyadic_taps, exact_input, grid_step  # noqa: E402
from rational import (ROWS, branch_one_hot_taps, oracle_filter, real_grid_input, ref_rational_f64,  # noqa: E402
                      stuff)
from util import assert_cf32_close, rand_block  # noqa: E402

pkg = importlib.import_module("sdr-server_b200")
RAGGED = [65536, 65536, 30001, 2, 0, 65536, 12347, 65536, 7, 65534]
SMALL = [16384, 16384, 7001, 2, 0, 16384, 3, 16382, 16384, 16384]
SPECS = [(3, 128, 97), (5, 4, 3), (2, 1, 9), (5, 3, 40), (7, 320, 431)]  # test_gpu_rational.py::test_exact
FS = 2016000


def u64(y):
    return np.ascontiguousarray(y).view(np.uint64) if np.iscomplexobj(y) else np.ascontiguousarray(y)


def same_bits(a, b, what):
    assert len(a) == len(b), f"{what}: {len(a)} blocks != {len(b)}"
    for i, (x, y) in enumerate(zip(a, b)):
        assert x.shape == y.shape and np.array_equal(u64(x), u64(y)), f"{what}: block {i} differs"


class F:
    """One drop-in filter and what it consumed.  L = 0: integer filter (decimation M); q15: Q15 calls."""

    def __init__(self, L, M, taps, center, fs, max_in, fmt, q15=False, rational_ctor=None):
        self.L, self.M, self.taps, self.center, self.fmt, self.q15 = L, M, taps, center, fmt, q15
        if L == 0 and not rational_ctor:
            self.f = pkg.XlatingFilter(M, taps, center, fs, max_in)
        else:
            self.f = pkg.XlatingFilter.rational(max(L, 1), M, taps, center, fs, max_in)
        self.seen, self.got = [], []

    def call(self, x):
        y = self.f.process_q15(self.fmt, x) if self.q15 else self.f.process_cf32(self.fmt, x)
        self.seen.append(x)
        self.got.append(y)
        return y

    def check_exact(self, what):
        L = max(self.L, 1)
        assert_exact(self.got, ref_rational_f64(self.taps, L, self.M, self.fmt, self.seen),
                     f"{what} L={L} M={self.M} T={self.taps.size} {self.fmt}", self.taps.size, self.M,
                     grid_step(self.taps, self.fmt))

    def check_oracle_exact(self, fs, max_in, what):
        L = max(self.L, 1)
        assert self.taps.size >= self.M  # the oracle's history bookkeeping underflows with fewer taps
        o = oracle_filter(po, L, self.M, self.taps, self.center, fs, max_in)
        ref = [o.process_cf32("cs16", stuff(self.fmt, x, L)) for x in self.seen]
        o.close()
        assert_exact(self.got, ref, f"{what} L={L} M={self.M} T={self.taps.size} centre {self.center}",
                     self.taps.size, self.M)

    def check_oracle(self, fs, max_in, what):
        L = max(self.L, 1)
        o = oracle_filter(po, L, self.M, self.taps, self.center, fs, max_in)
        if self.q15:
            ref = [o.process_q15(self.fmt, x) for x in self.seen]
            for b, (g, r) in enumerate(zip(self.got, ref)):
                assert np.array_equal(np.asarray(g).reshape(-1, 2), np.asarray(r).reshape(-1, 2)), f"{what} Q15 block {b}"
        else:
            ref = [o.process_cf32("cs16", stuff(self.fmt, x, L)) for x in self.seen]
            assert [len(y) for y in self.got] == [len(y) for y in ref], f"{what}: output counts"
            assert_cf32_close(np.concatenate(self.got), np.concatenate(ref), what)
        o.close()

    def close(self):
        self.f.close()


def run_threads(filters, blocks_for, n_blocks, window=4, skip=None, pause=None):
    """One dsp thread per filter; they meet at a barrier every `window` blocks.  blocks_for(i, b) is
    filter i's private copy of block b; skip(i, b) drops it; pause(i, b) sleeps before it."""
    errors = []
    bar = threading.Barrier(len(filters))

    def dsp(i):
        try:
            for b in range(n_blocks):
                x = blocks_for(i, b).copy()  # the queue's private copy, made before the threads are woken
                if b % window == 0:
                    bar.wait()
                if skip is not None and skip(i, b):
                    continue
                if pause is not None and pause(i, b):
                    time.sleep(0.5)
                filters[i].call(x)
        except Exception as e:  # noqa: BLE001
            errors.append(repr(e))
            bar.abort()

    ts = [threading.Thread(target=dsp, args=(i,)) for i in range(len(filters))]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    return errors


def checked(errors, fn, *args):
    try:
        fn(*args)
    except AssertionError as e:
        errors.append(str(e)[:600])


def scenario_interp1(stim):
    fs, max_in = FS, 65536
    rng = np.random.default_rng(3)
    exact = stim == "exact"
    pairs = []
    for c, p in enumerate(pkg.client_plan(fs, [48000, 96000, 48000, 96000, 48000, 96000])):
        q15 = c >= 4
        taps = pkg.create_low_pass_filter(1.0, fs, p["cutoff"], p["tw"])
        center = p["center"]
        if exact and not q15:
            taps, center = dyadic_taps(rng, len(taps), "cu8"), 0
        pairs.append([F(0, p["decimation"], taps, center, fs, max_in, "cu8", q15),
                      F(0, p["decimation"], taps, center, fs, max_in, "cu8", q15, rational_ctor=True)])
    filters = [f for pr in pairs for f in pr]
    gen = exact_input if exact else rand_block
    blocks = [gen(rng, "cu8", n) for n in RAGGED * 2]
    errors = run_threads(filters, lambda i, b: blocks[b], len(blocks))
    for c, (a, r) in enumerate(pairs):
        checked(errors, same_bits, a.got, r.got, f"pair {c} ({'Q15' if a.q15 else 'cf32'})")
        if exact and not a.q15:
            checked(errors, r.check_exact, f"pair {c}")
    for f in filters:
        f.close()
    return {"errors": errors}


def scenario_private(dump_dir):
    """Rows of the rate table through the drop-in ABI, one thread, and the same clients in a Group whose
    rational clients run on the polyphase generic kernel (kind 3)."""
    os.environ["XLATING_B200_POLY_TILE"] = "0"
    max_in = 65536
    errors, kinds = [], set()
    for row, (fs, fmt, rate) in enumerate(ROWS):
        plan = pkg.rational_plan(fs, [rate] * 3)
        rng = np.random.default_rng(fs % 1013)
        blocks = [rand_block(rng, fmt, n) for n in RAGGED * 2]
        filters = [F(p["interp"], p["decim"], p["taps"], p["center"], fs, max_in, fmt) for p in plan]
        g = pkg.Group(fs, max_in)
        ids = [g.add_client_rational(p["interp"], p["decim"], p["taps"], p["center"]) for p in plan]
        want = [[] for _ in ids]
        for x in blocks:
            for f in filters:
                f.call(x)
            t = g.submit(fmt, x)
            g.wait(t)
            for i, c in enumerate(ids):
                want[i].append(g.output(t, c))
        kinds |= {g.client_info(c)[1] for c in ids}
        g.close()
        for i, f in enumerate(filters):
            checked(errors, same_bits, f.got, want[i], f"row {row} client {i} vs group kind 3")
            checked(errors, f.check_oracle, fs, max_in, f"row {row} client {i}")
            np.save(os.path.join(dump_dir, f"row{row}_client{i}.npy"),
                    np.concatenate(f.got) if f.got else np.zeros(0, np.complex64))
            f.close()
    return {"errors": errors, "group_kinds": sorted(kinds)}


def exact_filters(rng, fmt, fs, max_in, rational_specs, n_integer):
    out = [F(L, M, dyadic_taps(rng, T, fmt), 0, fs, max_in, fmt) for L, M, T in rational_specs]
    out += [F(0, 42, dyadic_taps(rng, 97, fmt), 0, fs, max_in, fmt) for _ in range(n_integer)]
    return out


def scenario_exact():
    errors, stream = [], []
    for fmt in ("cu8", "cs8", "cs16"):
        rng = np.random.default_rng(17)
        filters = exact_filters(rng, fmt, FS, 16384, SPECS * 2, 2)
        blocks = [exact_input(rng, fmt, n) for n in SMALL * 2]
        errors += run_threads(filters, lambda i, b: blocks[b], len(blocks))
        for i, f in enumerate(filters):
            checked(errors, f.check_exact, f"filter {i}")
            f.close()
        stream.append(pkg.dropin_stream_stats())
    return {"errors": errors, "stream": stream[-1]}


def mixed_filters(rng, fs, max_in, with_rational=True):
    fmts = ["cu8", "cs8", "cs16", "cu8"]
    ip = pkg.client_plan(fs, [64000] * 8)
    out = []
    for c, p in enumerate(ip):
        taps = pkg.create_low_pass_filter(1.0, fs, p["cutoff"], p["tw"])
        out.append(F(0, p["decimation"], taps, p["center"], fs, max_in, fmts[c % 4], q15=c >= 4))
    if with_rational:
        for c, p in enumerate(pkg.rational_plan(fs, [48000] * 4)):
            out.append(F(p["interp"], p["decim"], p["taps"], p["center"], fs, max_in, fmts[c]))
    return out


def ragged_feed(rng, filters, n_blocks, max_in):
    sizes = [max_in, max_in, 30001, 2, 0, max_in, 12347, 7, max_in - 2]
    data = {}
    for i, f in enumerate(filters):
        data[i] = [rand_block(rng, f.fmt, sizes[(b + i) % len(sizes)]) for b in range(n_blocks)]
    return lambda i, b: data[i][b]


def scenario_combined():
    fs, max_in = 2048000, 65536
    rng = np.random.default_rng(23)
    filters = mixed_filters(rng, fs, max_in) + mixed_filters(rng, fs, max_in)
    feed = ragged_feed(rng, filters, 12, max_in)
    b0, c0, _ = pkg.dropin_stats()
    errors = run_threads(filters, feed, 12, window=1)
    b1, c1, _ = pkg.dropin_stats()
    for i, f in enumerate(filters):
        checked(errors, f.check_oracle, fs, max_in, f"filter {i} ({'rational' if f.L else 'Q15' if f.q15 else 'cf32'})")
        f.close()
    return {"errors": errors, "batches": b1 - b0, "calls": c1 - c0}


def scenario_neighbours():
    fs, max_in = 2048000, 65536
    runs = []
    for with_rational in (False, True):
        rng = np.random.default_rng(29)
        filters = mixed_filters(rng, fs, max_in, with_rational)
        feed = ragged_feed(np.random.default_rng(31), filters[:8], 12, max_in)
        errors = run_threads(filters, lambda i, b: feed(i % 8, b), 12, window=1)
        runs.append([f.got for f in filters[:8]])
        for f in filters:
            f.close()
        if errors:
            return {"errors": errors}
    errors = []
    for i in range(8):
        checked(errors, same_bits, runs[0][i], runs[1][i], f"integer filter {i}")
    return {"errors": errors}


def scenario_overlay(mode):
    rng = np.random.default_rng(41)
    n_blocks = 16
    filters = exact_filters(rng, "cu8", FS, 65536, [(3, 128, 97), (7, 320, 431)] * 12, 4)
    blocks = [exact_input(rng, "cu8", 65536) for _ in range(n_blocks)]
    r = np.random.default_rng(5)
    drop = {(i, b) for i in range(len(filters)) for b in range(3, n_blocks) if i % 3 == 0 and r.integers(0, 5) == 0}
    skip = {"drops": lambda i, b: (i, b) in drop,
            "late": lambda i, b: b < (i % 4) * 3}.get(mode)
    pause = (lambda i, b: i == 1 and b == 6) if mode == "lag" else None
    errors = run_threads(filters, lambda i, b: blocks[b], n_blocks, window=12 if mode == "lag" else 4, skip=skip,
                         pause=pause)
    calls = sum(len(f.got) for f in filters)
    stream = pkg.dropin_stream_stats()
    for i, f in enumerate(filters):
        checked(errors, f.check_exact, f"filter {i}")
        f.close()
    return {"errors": errors, "stream": stream, "calls": calls, "filters": len(filters)}


def scenario_q15refuse():
    rng = np.random.default_rng(43)
    filters = exact_filters(rng, "cu8", FS, 65536, [(3, 128, 97)] * 4, 0)
    blocks = [exact_input(rng, "cu8", 65536) for _ in range(12)]
    refused = []

    def feed(i, b):
        if i == 0 and b == 5:
            for _ in range(2):  # logged once per filter
                refused.append(len(filters[0].f.process_q15("cu8", exact_input(rng, "cu8", 65536))))
        return blocks[b]

    errors = run_threads(filters, feed, len(blocks))
    stream = pkg.dropin_stream_stats()  # before the filters leave
    for i, f in enumerate(filters):
        checked(errors, f.check_exact, f"filter {i}")
        f.close()
    return {"errors": errors, "refused": refused, "stream": stream}


# (L, M, T): the drop-in span boundary (16, 17), the batch engine's class budget (36, 37), gcd(L, M) = 2,
# 48 kHz from 44.1 kHz and back, 44.1 kHz from 2.048 Msps (T < M, fewer outputs than L per call), T < L
WIDE = [(16, 15, 97), (17, 16, 200), (36, 35, 300), (37, 36, 300), (6, 256, 400), (4, 2, 9), (160, 147, 1000),
        (147, 160, 1000), (441, 20480, 2000), (17, 16, 5)]
# T >= M for the strict oracle
PHASE = [(3, 128, 385), (7, 320, 431), (17, 16, 200), (6, 256, 401), (16, 15, 97), (36, 35, 300), (37, 36, 300),
         (160, 147, 1000)]


def scenario_wide():
    errors, spans = [], 0
    for fmt in ("cu8", "cs8", "cs16"):
        rng = np.random.default_rng(59)
        filters = exact_filters(rng, fmt, 2048000, 16384, WIDE, 2)
        blocks = [exact_input(rng, fmt, n) for n in SMALL * 2]
        errors += run_threads(filters, lambda i, b: blocks[b], len(blocks))
        for i, f in enumerate(filters):
            checked(errors, f.check_exact, f"filter {i}")
            spans += sum(len(y) > f.L > 16 for y in f.got)
            f.close()
    few = sum(0 < len(y) < 441 for y in filters[WIDE.index((441, 20480, 2000))].got)
    return {"errors": errors, "long_spans": spans, "fewer_than_L": few}


def scenario_phase():
    fs, max_in = 2048000, 16384
    rng = np.random.default_rng(67)
    filters = []
    for k, (L, M, T) in enumerate(PHASE * 2):
        center = int(rng.integers(-fs // 2 + 30000, fs // 2 - 30000))
        filters.append(F(L, M, branch_one_hot_taps(rng, T, L), center, fs, max_in, "cs16"))
    blocks = [real_grid_input(rng, n) for n in SMALL * 2]
    errors = run_threads(filters, lambda i, b: blocks[b], len(blocks))
    for i, f in enumerate(filters):
        checked(errors, f.check_oracle_exact, fs, max_in, f"filter {i}")
        f.close()
    return {"errors": errors, "stream": pkg.dropin_stream_stats()}


def main():
    scenario = sys.argv[1]
    arg = sys.argv[2] if len(sys.argv) > 2 else None
    fn = globals()[f"scenario_{scenario}"]
    res = fn(arg) if arg is not None else fn()
    res["scenario"] = scenario
    res["errors"] = res["errors"][:4]
    print(json.dumps(res))
    return 1 if res["errors"] else 0


if __name__ == "__main__":
    sys.exit(main())
