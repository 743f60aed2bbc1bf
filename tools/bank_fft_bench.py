"""The bank kernels alone: the FFT bank (xlg_add_bank_fft), or at a K that is not a power of two the chirp-z bank
(xlg_add_bank_any), against the direct bank (xlg_add_bank) on the same bank with every channel materialised.

    python tools/bank_fft_bench.py [--blocks K] [--warmup W] [--rounds R] [--widths K,...]

Per width K (one JSON line per kernel and round, the kernels alternated within every round; the direct bank
wherever its shared memory holds the bank, bank_fits): a 61.44 Msps
cs16 stream in blocks of 262144 bytes, as in bench.py, feeding one bank of D1 = K / 2 whose taps are
subband_plan's first stage at that D1 (create_low_pass_filter(1, fs, fs1 / 2, fs1 - 2e), e = fs1 / 4 + 24 kHz),
all K channels materialised and no members.  Reported: the bank kernel's time per block from a profiled run
(CUDA events around each launch, xlg_bank_profile / xlg_bank_fft_profile) and the kernel's counted work.  The
card's name, power limit and clocks are printed first, read in the same call.  Nothing is written to the tree.
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

FS, FMT, BLOCK = 61440000, "cs16", 262144


def taps_at(d1):
    fs1 = FS // d1
    e = fs1 // 4 + 24000
    return pkg.create_low_pass_filter(1.0, FS, fs1 // 2, fs1 - 2 * e)


def run(K, kernel, blocks, warmup, data):
    """kernel: "direct", "fft" or "czt"."""
    d1 = K // 2
    taps = taps_at(d1)
    fft = kernel != "direct"
    g = pkg.Group(FS, BLOCK)
    try:
        bid = g.add_bank_fft(d1, taps, any_k=kernel == "czt") if fft else g.add_bank(d1, taps)
        g.reserve(K * (BLOCK // 4 // d1 + 8))
        for k in range(-d1, d1):
            g.add_bank_subband(bid, k)
        g.profile_enable(True)
        for i in range(warmup):
            g.wait(g.submit(FMT, data[i % len(data)]))
        read = g.bank_fft_profile_read if fft else g.bank_profile_read
        read(reset=True)
        for i in range(blocks):
            g.wait(g.submit(FMT, data[i % len(data)]))
        p = read()
    finally:
        g.close()
    ms = p["fft_ms" if fft else "bank_ms"]
    n = p["fft_launches" if fft else "bank_launches"]
    work = {"butterfly_flops": p["butterfly_flops"]} if fft else {"dft_macs": p["dft_macs"]}
    return {"K": K, "d1": d1, "taps1": int(taps.size), "kernel": kernel, "blocks": blocks,
            "launches": n, "kernel_us_per_block": 1e3 * ms / max(n, 1), "poly_macs": p["poly_macs"], **work}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--widths", default="128,256", help="even K up to 4096, comma-separated")
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                           "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()[0]
    print(json.dumps({"card": card}), flush=True)
    rng = np.random.default_rng(0)
    data = [rng.integers(-32768, 32767, BLOCK // 2, dtype=np.int16, endpoint=True) for _ in range(4)]
    for r in range(args.rounds):
        for K in [int(k) for k in args.widths.split(",")]:
            kernels = ["direct"] if pkg.bank_fits(K // 2, taps_at(K // 2).size) else []
            for kernel in kernels + ["fft" if K & (K - 1) == 0 else "czt"]:
                res = run(K, kernel, args.blocks, args.warmup, data)
                res["round"] = r
                print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
