"""Worker for tests/test_gpu_stream_overlay.py and tests/test_gpu_exact.py (run in a subprocess so that
the engine's environment switches -- read once per process -- can differ per scenario).

usage: _dropin_overlay_worker.py <scenario> <clients> <blocks> [exact|phase]   -> one JSON line
Every filter has its own dsp thread and its own private copy of each block
(src/dsp_worker.c:41-88, src/queue.c:114); every output is compared with an oracle filter
that consumed exactly the blocks this filter consumed.

exact: every filter gets its own dyadic taps at centre 0 and the blocks lie on the exact input
grid (tests/exact.py); each filter's outputs must then equal the float64 result over the blocks
it consumed bit for bit, so the state handed over when it joins or leaves a band group (history,
valid history) is checked to the sample.

phase: one real cs16 stream on the same grid (tests/rational.py real_grid_input).  Half of the
filters have dyadic taps at centre 0, checked as in exact; the other half one tap at the first, the
last or a random position at their plan's centre, where every accumulator is one rounded product,
so their outputs must equal the strict oracle bit for bit, oscillator included: the phase handed
over at every join and leave is checked to the bit.

late_short: the late filters (i % 4 in (1, 2)) start with calls of 2, 3 and 7001 elements, so they
can join while they have consumed fewer than taps - 1 samples; the band's older samples must read
as zero for them.  The stream counters are taken after their first two calls ("short").
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
from exact import assert_exact, dyadic_taps, exact_input, one_hot_taps, ref_f64  # noqa: E402
from rational import real_grid_input  # noqa: E402
from util import assert_cf32_close, rand_block  # noqa: E402

SHORT_AT = 4  # late_short: the blocks of 2, 3 and 7001 elements


def main():
    scenario, n_clients, n_blocks = sys.argv[1], int(sys.argv[2]), int(sys.argv[3])
    stim = sys.argv[4] if len(sys.argv) > 4 else None
    exact = stim in ("exact", "phase")
    pkg = importlib.import_module("sdr-server_b200")
    rng = np.random.default_rng(7)
    fs, max_in = 2016000, 65536
    fmt = "cs16" if stim == "phase" else "cu8"
    plan = pkg.client_plan(fs, [48000 if c % 2 == 0 else 96000 for c in range(n_clients)])
    sizes = [max_in] * n_blocks
    if scenario == "late_short":
        sizes[SHORT_AT:SHORT_AT + 3] = [2, 3, 7001]
    if stim == "phase":
        blocks = [real_grid_input(rng, n) for n in sizes]
        other = [real_grid_input(rng, n) for n in sizes]
    else:
        gen = exact_input if exact else rand_block
        blocks = [gen(rng, fmt, n) for n in sizes]
        other = [gen(rng, fmt, n) for n in sizes]  # a second SDR source
    filters, oracles, tapsets, centres = [], [], [], []
    for c, p in enumerate(plan):
        taps = pkg.create_low_pass_filter(1.0, fs, p["cutoff"], p["tw"])
        center = p["center"]
        if stim == "phase" and (c // 2) % 2 == 0:
            T = len(taps)
            taps = one_hot_taps(T, (0, T - 1, int(rng.integers(0, T)))[c % 3], float(rng.choice([0.75, -0.5])))
        elif exact:
            taps, center = dyadic_taps(rng, len(taps), fmt), 0
        tapsets.append(taps)
        centres.append(center)
        filters.append(pkg.XlatingFilter(p["decimation"], taps, center, fs, max_in))
        oracles.append(po.OracleFilter(p["decimation"], taps, center, fs, max_in))
    errors, worst, short = [], [0.0], {}
    seen = [[] for _ in plan]  # exact: (block, output) per filter, checked after the run
    window = {"lag": 12, "late_short": 1}.get(scenario, 4)  # lag: let the others run a whole (4-entry) ring ahead
    bar = threading.Barrier(n_clients)

    def dsp_thread(i):
        r = np.random.default_rng(100 + i)
        try:
            for b in range(n_blocks):
                if b % window == 0:
                    bar.wait()  # bounded queues: nobody runs a whole queue ahead (src/config.c:183)
                if scenario == "late_short" and b == SHORT_AT + 2:
                    bar.wait()  # every filter has made the calls of 2 and 3 elements
                    if i == 0:
                        short.update(pkg.dropin_stream_stats())
                    bar.wait()
                if scenario == "drops" and i % 3 == 0 and b > 2 and r.integers(0, 5) == 0:
                    continue    # this client's queue overwrote the block (src/queue.c:90-94)
                if scenario == "late" and b < (i % 4) * 3:
                    continue    # attached later: never saw the first blocks
                if scenario == "late_short" and i % 4 in (1, 2) and b < SHORT_AT:
                    continue
                if scenario == "lag" and i == 1 and b == 6:
                    time.sleep(0.5)
                src = other if (scenario == "two_sources" and i % 2 == 1) else blocks
                own = src[b].copy()  # queue_put's private copy (src/queue.c:114)
                y = filters[i].process_cf32(fmt, own)
                if exact:
                    seen[i].append((src[b], y))
                    continue
                ref = oracles[i].process_cf32(fmt, own)
                worst[0] = max(worst[0], assert_cf32_close(y, ref, f"client {i} block {b}"))
        except Exception as e:  # noqa: BLE001
            errors.append(repr(e))
            bar.abort()

    threads = [threading.Thread(target=dsp_thread, args=(i,)) for i in range(n_clients)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    if exact and not errors:
        for i, p in enumerate(plan):
            T, D = len(tapsets[i]), p["decimation"]
            got, xs = [y for _, y in seen[i]], [x for x, _ in seen[i]]
            try:
                if centres[i] == 0:
                    assert_exact(got, ref_f64(tapsets[i], D, fmt, xs), f"client {i}", T, D)
                else:
                    assert_exact(got, [oracles[i].process_cf32(fmt, x) for x in xs], f"client {i} centre {centres[i]}",
                                 T, D)
            except AssertionError as e:
                errors.append(str(e))
    st = pkg.dropin_stream_stats()
    for f in filters:
        f.close()
    print(json.dumps({"scenario": scenario, "errors": errors[:3], "worst": worst[0], "stream": st, "short": short}))
    return 1 if errors else 0


if __name__ == "__main__":
    sys.exit(main())
