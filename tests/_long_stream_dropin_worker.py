"""Worker of tests/test_gpu_long_stream.py::test_dropin_past_2_32 (a subprocess, so that the drop-in engine
reads the environment the scenario sets: it is read once per process).

usage: _long_stream_dropin_worker.py engine|overlay   -> one JSON line

engine: an integer, a rational and a cascade XlatingFilter (the caller turns the stream overlay off), each fed
the same N-sample cs16 blocks, past 2^32 input samples, with a ragged pair of odd lengths at 2^31 and 2^32.
overlay: two integer filters of one band fed the same blocks, which the overlay's batch group serves.
Every filter's outputs on the blocks around 2^31 and 2^32 are checked against a fresh float64 reference fed
the blocks from a boundary a multiple of its period after its creation (tests/long_stream.py).
"""
import importlib
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from cascade import small_taps  # noqa: E402
from exact import assert_exact, dyadic_taps, exact_input  # noqa: E402
from long_stream import N, fresh_refs, history, period, window_start  # noqa: E402

FS, FMT = 61_440_000, "cs16"


def main():
    scenario = sys.argv[1]
    pkg = importlib.import_module("sdr-server_b200")
    rng = np.random.default_rng(800 if scenario == "engine" else 801)
    bufs = [exact_input(rng, FMT, 2 * N) for _ in range(4)]
    specs = []
    if scenario == "engine":
        specs.append(("int", 21, dyadic_taps(rng, 129, FMT)))
        specs.append(("rat", 3, 128, dyadic_taps(rng, 390, FMT)))
        specs.append(("casc", 8, small_taps(rng, 17, 3), 3, 16, small_taps(rng, 47, 3)))
    else:
        specs.append(("int", 21, dyadic_taps(rng, 129, FMT)))
        specs.append(("int", 42, dyadic_taps(rng, 64, FMT)))
    filters = []
    for s in specs:
        if s[0] == "int":
            filters.append(pkg.XlatingFilter(s[1], s[2], 0, FS, 2 * N))
        elif s[0] == "rat":
            filters.append(pkg.XlatingFilter.rational(s[1], s[2], s[3], 0, FS, 2 * N))
        else:
            filters.append(pkg.XlatingFilter.cascade(s[1], s[2], 0, s[4], s[5], FS, 2 * N, interp2=s[3]))
    blocks, starts, got, errors, checked = [], [0], {}, [], 0

    def feed(x, watch):
        blocks.append(x)
        starts.append(starts[-1] + x.size // 2)
        ys = [f.process_cf32(FMT, x) for f in filters]
        if watch:
            got[len(blocks) - 1] = ys

    def check(c0, c1, label):
        nonlocal checked
        for j, s in enumerate(specs):
            b = window_start(starts, c0, 0, period(s), history(s))
            ref = fresh_refs([s], FMT, FS, blocks[b:c1])[0][c0 - b:]
            try:
                assert_exact([got[i][j] for i in range(c0, c1)], ref, f"{label}: filter {s[0]} {s[1]}")
            except AssertionError as e:
                errors.append(str(e))
            checked += 1
        for i in range(c0, c1):
            got.pop(i)

    def full(watch=False):
        feed(bufs[int(rng.integers(0, len(bufs)))], watch)

    for _ in range(3):
        full(True)
    check(1, 3, "control")
    for pos, label in ((2 ** 31, "2^31"), (2 ** 32, "2^32")):
        while starts[-1] + N <= pos:
            full()
        c0 = len(blocks)
        a = pos - starts[-1] + 101
        a += 1 - a % 2
        x = bufs[int(rng.integers(0, len(bufs)))]
        feed(x[:2 * a], True)
        feed(x[2 * a:], True)
        full(True)
        check(c0, c0 + 3, label)
    st = pkg.dropin_stream_stats()
    for f in filters:
        f.close()
    print(json.dumps({"scenario": scenario, "errors": errors[:3], "position": int(starts[-1]), "checked": checked,
                      "filters": len(filters), "stream": st}))
    return 1 if errors else 0


if __name__ == "__main__":
    sys.exit(main())
