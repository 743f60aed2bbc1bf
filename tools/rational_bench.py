"""Throughput of rational L/M clients against the integer yardstick with about the same MACs per input.

    python tools/rational_bench.py [--blocks K] [--warmup W] [--rounds R]

Workloads (one JSON line each per round, workloads alternated within a round):
  poly_tile     256 clients at 48 kHz on a 2.048 Msps cu8 stream: L/M = 3/128, ceil(T/L) = 514 taps per output,
                tiled rational classes (kind 4)
  poly_generic  the same, forced onto the polyphase generic kernel (XLATING_B200_POLY_TILE=0, kind 3)
  integer_tile  256 clients at 48 kHz on a 2.016 Msps cu8 stream: D = 42, T = 505, the tiled kernel
  poly_10M      64 clients at 48 kHz on a 10 Msps cs16 stream: 3/625, ceil(T/L) = 2510 (generic: its branches
                exceed the tiled kernel's shared memory)

Per workload: input MS/s over K pipelined blocks (CUDA events, xlg_timer_*), algorithmic complex MACs
per second (sum n_out * ceil(T/L)), the FIR kernel's own time per block from a profiled run of its own
(one compute stream, CUDA events around each launch), and both rates as a fraction of the FP32 FMA
peak that tools/bin/microbench measures in the same run (4 real FMA per complex MAC).  Blocks are
262144 bytes, as in bench.py.  Nothing is written to the tree.
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
WORKLOADS = {
    "poly_tile": (2048000, "cu8", 256, True),
    "poly_generic": (2048000, "cu8", 256, True),
    "integer_tile": (2016000, "cu8", 256, False),
    "poly_10M": (10000000, "cs16", 64, True),
}


def make_group(name, profile):
    fs, _, n, rational = WORKLOADS[name]
    if name == "poly_generic":
        os.environ["XLATING_B200_POLY_TILE"] = "0"  # read at group creation
    g = pkg.Group(fs, BLOCK)
    os.environ.pop("XLATING_B200_POLY_TILE", None)
    if rational:
        for p in pkg.rational_plan(fs, [48000] * n):
            g.add_client_rational(p["interp"], p["decim"], p["taps"], p["center"])
    else:
        for p in pkg.client_plan(fs, [48000] * n):
            g.add_client(p["decimation"], pkg.create_low_pass_filter(1.0, fs, p["cutoff"], p["tw"]), p["center"])
    if profile:
        g.profile_enable(True)
    return g


def run(name, blocks, warmup, peak_tfma):
    fs, fmt, n, rational = WORKLOADS[name]
    rng = np.random.default_rng(0)
    dtype = pkg.NP_DTYPE[fmt]
    elems = BLOCK // np.dtype(dtype).itemsize
    data = [rng.integers(np.iinfo(dtype).min, np.iinfo(dtype).max, elems, dtype=dtype, endpoint=True) for _ in range(4)]
    res = {"workload": name, "fs": fs, "fmt": fmt, "clients": n, "blocks": blocks}
    # end to end: the real pipeline (all streams, speculation on)
    g = make_group(name, False)
    for i in range(warmup):
        g.wait(g.submit(fmt, data[i % 4]))
    g.timer_start()
    t = None
    for i in range(blocks):
        t = g.submit(fmt, data[i % 4])
    g.wait(t)
    ms = g.timer_stop()
    g.close()
    # kernel time and algorithmic MACs: a profiled run of its own
    g = make_group(name, True)
    for i in range(warmup):
        g.wait(g.submit(fmt, data[i % 4]))
    g.profile_read(reset=True)
    g.poly_profile_read(reset=True)
    for i in range(blocks):
        g.wait(g.submit(fmt, data[i % 4]))
    prof, pp = g.profile_read(), g.poly_profile_read()
    kinds = sorted({g.client_info(c)[1] for c in range(n)})
    g.close()
    macs_per_block = prof["algo_macs"] / prof["blocks"]
    if rational:
        k_ms = (pp["fir_poly_tile_ms"] + pp["fir_poly_generic_ms"]) / max(
            pp["fir_poly_tile_launches"], pp["fir_poly_generic_launches"], 1)
    else:
        k_ms = prof["fir_tile_ms"] / max(prof["fir_tile_launches"], 1)
    in_samples = blocks * elems / 2
    res.update({
        "kernel_kinds": kinds,
        "input_msps": in_samples / (ms * 1e-3) / 1e6,
        "ms_per_block": ms / blocks,
        "cmacs_per_s": macs_per_block * blocks / (ms * 1e-3),
        "fir_kernel_ms": k_ms,
        "fir_kernel_cmacs_per_s": macs_per_block / (k_ms * 1e-3),
        "fp32_peak_tfma": peak_tfma,
    })
    res["frac_step"] = 4 * res["cmacs_per_s"] / (peak_tfma * 1e12)
    res["frac_kernel"] = 4 * res["fir_kernel_cmacs_per_s"] / (peak_tfma * 1e12)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    out = subprocess.run([os.path.join(ROOT, "tools", "bin", "microbench"), "4000"], capture_output=True, text=True,
                         timeout=120, check=True).stdout
    peak = max(json.loads(ln)["tfma_per_s"] for ln in out.splitlines() if '"ffma"' in ln)
    print(json.dumps({"card": card, "fp32_peak_tfma": peak, "peak_source": "tools/bin/microbench ffma"}), flush=True)
    for r in range(args.rounds):
        for name in WORKLOADS:
            res = run(name, args.blocks, args.warmup, peak)
            res["round"] = r
            print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
