"""Throughput of cascade clients (xlg_add_client_cascade) against single-stage clients of the same rate.

    python tools/cascade_bench.py [--blocks K] [--warmup W] [--rounds R]

Workloads (one JSON line each per round, single stage and cascade alternated within a round):
  61M_single     512 clients at 48 kHz on a 61.44 Msps cs16 stream (BASELINE configs[4]): D = 1280, T = 15419
  61M_32x40      the same clients as cascades 32 x 40, taps 79 / 481 (cascade_plan)
  2M_single      256 clients at 48 kHz on a 2.016 Msps cu8 stream (configs[1]): D = 42, T = 505
  2M_6x7         the same as cascades 6 x 7, taps 17 / 85 (cascade_plan's choice)
  2M_7x6         the same as cascades 7 x 6 (cascade_stages with D1 = 7): a shorter stage-A oscillator chain
  10M_single     64 clients at 48 kHz on a 10 Msps cs16 stream: rational 3/625, ceil(T / L) = 2510 (kind 3)
  10M_cascade    the same as the planner's cascades: 20 x 12/125, taps 55 / 1505
  20M_single     64 clients at 48 kHz on a 20 Msps cs8 stream: rational 3/1250 (kind 3)
  20M_cascade    the same as the planner's cascades: 25 x 3/50, taps 65 / 603
  2M048_single   256 clients at 48 kHz on a 2.048 Msps cu8 stream: rational 3/128 (kind 4)
  2M048_cascade  the same as the planner's cascades: 8 x 3/16, taps 25 / 193

Per workload: input MS/s over K pipelined blocks (CUDA events, xlg_timer_*), algorithmic real FMAs per input
sample (4 T / D, 4 ceil(T / L) L / M, or cascade_fmas), and from a profiled run of its own (one compute stream, CUDA events
around each launch) the stage-B kernel's time per block as a share of the pipelined step, and the oscillator
pre-pass time per block against the step: a pre-pass as long as the step paces the pipeline.  The last timed
block of two sampled cascade clients is checked against cascade_oracle, or the composed oracle of a rational
cascade (1e-5 norm-wise).  Blocks are 262144
bytes, as in bench.py.  Nothing is written to the tree.
"""
import argparse
import importlib
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
pkg = importlib.import_module("sdr-server_b200")

BLOCK = 262144
WORKLOADS = {  # fs, format, clients, D1 (0 = single stage, PLAN = cascade_plan's choice)
    "61M_single": (61440000, "cs16", 512, 0),
    "61M_32x40": (61440000, "cs16", 512, 32),
    "2M_single": (2016000, "cu8", 256, 0),
    "2M_6x7": (2016000, "cu8", 256, 6),
    "2M_7x6": (2016000, "cu8", 256, 7),
    "10M_single": (10000000, "cs16", 64, 0),
    "10M_cascade": (10000000, "cs16", 64, -1),
    "20M_single": (20000000, "cs8", 64, 0),
    "20M_cascade": (20000000, "cs8", 64, -1),
    "2M048_single": (2048000, "cu8", 256, 0),
    "2M048_cascade": (2048000, "cu8", 256, -1),
}
PLAN = -1
RATE = 48000


def clients(name):
    fs, _, n, d1 = WORKLOADS[name]
    plan = pkg.client_plan(fs, [RATE] * n)
    if d1 == 0 and fs % RATE:
        r = pkg.rational_plan(fs, [RATE] * n)
        L, M, T = r[0]["interp"], r[0]["decim"], r[0]["taps"].size
        return [("r", p["interp"], p["decim"], p["taps"], p["center"]) for p in r], 4.0 * -(-T // L) * L / M
    if d1 == 0:
        taps = pkg.create_low_pass_filter(1.0, fs, RATE // 2, RATE // 5)
        return [("i", fs // RATE, taps, p["center"]) for p in plan], 4.0 * taps.size / (fs // RATE)
    if d1 == PLAN:
        c = pkg.cascade_plan(fs, [RATE] * n)
        return [("c", p["d1"], p["taps1"], p["center"], p["d2"], p["taps2"], p["interp2"]) for p in c], c[0]["fmas"]
    t1, t2 = pkg.cascade_stages(fs, RATE, d1)
    return ([("c", d1, t1, p["center"], fs // RATE // d1, t2) for p in plan],
            pkg.cascade_fmas(fs, RATE, d1, t1.size, t2.size))


def make_group(name, specs, profile):
    fs = WORKLOADS[name][0]
    g = pkg.Group(fs, BLOCK)
    add = {"i": g.add_client, "r": g.add_client_rational, "c": g.add_client_cascade}
    ids = [add[s[0]](*s[1:]) for s in specs]
    if profile:
        g.profile_enable(True)
    return g, ids


def run(name, blocks, warmup):
    fs, fmt, n, d1 = WORKLOADS[name]
    specs, fmas = clients(name)
    rng = np.random.default_rng(0)
    dtype = pkg.NP_DTYPE[fmt]
    elems = BLOCK // np.dtype(dtype).itemsize
    data = [rng.integers(np.iinfo(dtype).min, np.iinfo(dtype).max, elems, dtype=dtype, endpoint=True) for _ in range(4)]
    res = {"workload": name, "fs": fs, "fmt": fmt, "clients": n, "blocks": blocks, "fmas_per_input_sample": fmas}
    # end to end: the real pipeline (all streams, speculation on)
    g, ids = make_group(name, specs, False)
    for i in range(warmup):
        g.wait(g.submit(fmt, data[i % 4]))
    g.timer_start()
    t = None
    for i in range(blocks):
        t = g.submit(fmt, data[(warmup + i) % 4])
    g.wait(t)
    ms = g.timer_stop()
    res["input_msps"] = blocks * elems / 2 / (ms * 1e-3) / 1e6
    res["ms_per_block"] = ms / blocks
    if d1:
        # the last timed block of two sampled clients against the cascade oracle fed the whole stream
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        from cascade import cascade_oracle  # the tests' checkers
        from cascade_rational import RationalCascadeOracle
        worst = 0.0
        for k in (0, n // 2):
            s = specs[k]
            if len(s) > 6:
                o = RationalCascadeOracle(s[1], s[2], s[3], s[6], s[4], s[5], fs, BLOCK)
            else:
                o = cascade_oracle(s[1], s[2], s[3], s[4], s[5], fs, BLOCK)
            for i in range(warmup + blocks):
                r = o.process_cf32(fmt, data[i % 4])
            y = g.output(t, ids[k])
            assert y.shape == r.shape
            worst = max(worst, float(np.max(np.abs(y - r)) / np.max(np.abs(r))))
        assert worst <= 1e-5, worst
        res["checked_error"] = worst
        res["stage_a_kinds"] = sorted({g.cascade_info(c)[0] for c in ids})
    else:
        res["kinds"] = sorted({g.client_info(c)[1] for c in ids})
    g.close()
    # kernel times: a profiled run of its own
    g, ids = make_group(name, specs, True)
    for i in range(warmup):
        g.wait(g.submit(fmt, data[i % 4]))
    g.profile_read(reset=True)
    g.cascade_profile_read(reset=True)
    for i in range(blocks):
        g.wait(g.submit(fmt, data[i % 4]))
    prof, cp = g.profile_read(), g.cascade_profile_read()
    g.close()
    per = max(prof["blocks"], 1)
    res["phase_ms_per_block"] = prof["phase_ms"] / per
    res["prepass_over_step"] = res["phase_ms_per_block"] / res["ms_per_block"]
    res["fir_ms_per_block"] = (prof["fir_tile_ms"] + prof["fir_generic_ms"] + prof["fir_long_ms"]) / per
    res["stage_b_ms_per_block"] = cp["stage_b_ms"] / per
    res["stage_b_share_of_step"] = res["stage_b_ms_per_block"] / res["ms_per_block"]
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    print(json.dumps({"card": card}), flush=True)
    for r in range(args.rounds):
        for name in WORKLOADS:
            res = run(name, args.blocks, args.warmup)
            res["round"] = r
            print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
