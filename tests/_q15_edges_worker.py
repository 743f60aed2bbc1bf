"""Worker for tests/test_gpu_q15_edges.py: Q15 drop-in filters (process_*_cs16) at the edges of the integer
path.  Runs in a subprocess because the per-filter engine reads its environment switches (XLATING_B200_DROPIN,
_LANES, _SHARE) once per process.

usage: _q15_edges_worker.py <variant>   -> one JSON line, exit code 1 on any error

Every filter of tests/q15.py's edge_clients, for cu8, cs8 and cs16, and the 65537-tap filter whose acc >> 15
passes 2^31, each on its own dsp thread; the threads meet at a barrier before every call, so calls of many
filters are combined.  Every output is checked bit for bit against the model of tests/q15.py and the cheap
filters against the strict oracle too.
"""
import importlib
import json
import os
import sys
import threading

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import pyoracle as po  # noqa: E402  (checker)
import q15  # noqa: E402
from exact import assert_exact  # noqa: E402

pkg = importlib.import_module("sdr-server_b200")
FS = q15.FS
MAX_IN = 2 * 70000


def main():
    variant = sys.argv[1]
    lib = pkg.lib()
    rng = np.random.default_rng(41)
    jobs = []  # (label, fmt, taps, D, centre, blocks)
    for fmt in ("cu8", "cs8", "cs16"):
        blocks = q15.edge_blocks(rng, fmt, q15.RAGGED)
        for label, taps, D, c in q15.edge_clients(rng, fmt):
            jobs.append((f"{fmt} {label}", fmt, taps, D, c, blocks))
    taps = q15.narrowing_taps(65537, 300000, FS)
    rev, _, _ = q15.host_consts(lib, taps, 4096, 300000, FS)
    jobs.append(("narrowing", "cs16", taps, 4096, 300000, q15.narrowing_blocks(rng, rev)))
    n_calls = max(len(j[5]) for j in jobs)
    filters = [pkg.XlatingFilter(D, taps, c, FS, MAX_IN) for _, _, taps, D, c, _ in jobs]
    got = [[] for _ in jobs]
    errors = []
    bar = threading.Barrier(len(jobs))

    def dsp(i):
        try:
            _, fmt, _, _, _, blocks = jobs[i]
            for b in range(n_calls):
                bar.wait()
                if b < len(blocks):
                    got[i].append(filters[i].process_q15(fmt, blocks[b].copy(), variant))
        except Exception as e:  # noqa: BLE001
            errors.append(repr(e))
            bar.abort()

    ts = [threading.Thread(target=dsp, args=(i,)) for i in range(len(jobs))]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    checked = 0
    for i, (label, fmt, taps, D, c, blocks) in enumerate(jobs):
        try:
            want = q15.Client(lib, taps, D, c, FS)(fmt, blocks)
            assert_exact(got[i], want, f"{variant} {label} D={D} T={len(taps)} centre={c}: model", len(taps), D)
            if len(taps) < 1000:
                o = po.OracleFilter(D, taps, c, FS, MAX_IN)
                assert_exact(want, [o.process_q15(fmt, x) for x in blocks], f"{label}: model against the oracle")
            checked += 1
        except AssertionError as e:
            errors.append(str(e)[:600])
    for f in filters:
        f.close()
    group_model = os.environ.get("XLATING_B200_DROPIN") == "group"  # no per-filter engine, no engine stats
    print(json.dumps({"variant": variant, "filters": len(jobs), "checked": checked, "errors": errors[:6],
                      "n_errors": len(errors), "stats": None if group_model else pkg.dropin_stats()}))
    return 1 if errors else 0


if __name__ == "__main__":
    sys.exit(main())
