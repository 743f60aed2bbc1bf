"""Worker for tests/test_gpu_stream_overlay.py (run in a subprocess so that the engine's
environment switches -- read once per process -- can differ per scenario).

usage: _dropin_overlay_worker.py <scenario> <clients> <blocks> [exact]   -> one JSON line
Every filter has its own dsp thread and its own private copy of each block
(src/dsp_worker.c:41-88, src/queue.c:114); every output is compared with an oracle filter
that consumed exactly the blocks this filter consumed.

exact: every filter gets its own dyadic taps at centre 0 and the blocks lie on the exact input
grid (tests/exact.py); each filter's outputs must then equal the float64 result over the blocks
it consumed bit for bit, so the state handed over when it joins or leaves a band group (history,
valid history, phase) is checked to the sample."""
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
from exact import assert_exact, dyadic_taps, exact_input, ref_f64  # noqa: E402
from util import assert_cf32_close, rand_block  # noqa: E402


def main():
    scenario, n_clients, n_blocks = sys.argv[1], int(sys.argv[2]), int(sys.argv[3])
    exact = len(sys.argv) > 4 and sys.argv[4] == "exact"
    pkg = importlib.import_module("sdr-server_b200")
    rng = np.random.default_rng(7)
    fs, max_in = 2016000, 65536
    plan = pkg.client_plan(fs, [48000 if c % 2 == 0 else 96000 for c in range(n_clients)])
    gen = exact_input if exact else rand_block
    blocks = [gen(rng, "cu8", max_in) for _ in range(n_blocks)]
    other = [gen(rng, "cu8", max_in) for _ in range(n_blocks)]  # a second SDR source
    filters, oracles, tapsets = [], [], []
    for p in plan:
        taps = pkg.create_low_pass_filter(1.0, fs, p["cutoff"], p["tw"])
        center = p["center"]
        if exact:
            taps, center = dyadic_taps(rng, len(taps), "cu8"), 0
        tapsets.append(taps)
        filters.append(pkg.XlatingFilter(p["decimation"], taps, center, fs, max_in))
        oracles.append(po.OracleFilter(p["decimation"], taps, center, fs, max_in))
    errors, worst = [], [0.0]
    seen = [[] for _ in plan]  # exact: (block, output) per filter, checked after the run
    window = 12 if scenario == "lag" else 4  # lag: let the others run a whole (4-entry) ring ahead
    bar = threading.Barrier(n_clients)

    def dsp_thread(i):
        r = np.random.default_rng(100 + i)
        try:
            for b in range(n_blocks):
                if b % window == 0:
                    bar.wait()  # bounded queues: nobody runs a whole queue ahead (src/config.c:183)
                if scenario == "drops" and i % 3 == 0 and b > 2 and r.integers(0, 5) == 0:
                    continue    # this client's queue overwrote the block (src/queue.c:90-94)
                if scenario == "late" and b < (i % 4) * 3:
                    continue    # attached later: never saw the first blocks
                if scenario == "lag" and i == 1 and b == 6:
                    time.sleep(0.5)
                src = other if (scenario == "two_sources" and i % 2 == 1) else blocks
                own = src[b].copy()  # queue_put's private copy (src/queue.c:114)
                y = filters[i].process_cf32("cu8", own)
                if exact:
                    seen[i].append((src[b], y))
                    continue
                ref = oracles[i].process_cf32("cu8", own)
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
            try:
                assert_exact([y for _, y in seen[i]], ref_f64(tapsets[i], D, "cu8", [x for x, _ in seen[i]]),
                             f"client {i}", T, D)
            except AssertionError as e:
                errors.append(str(e))
    st = pkg.dropin_stream_stats()
    for f in filters:
        f.close()
    print(json.dumps({"scenario": scenario, "errors": errors[:3], "worst": worst[0], "stream": st}))
    return 1 if errors else 0


if __name__ == "__main__":
    sys.exit(main())
