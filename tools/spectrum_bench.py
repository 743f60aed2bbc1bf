"""Spectrum rows (xlg_add_spectrum): the spectrum kernels alone, and what a spectrum adds to a step of clients.

    python tools/spectrum_bench.py [--blocks K] [--warmup W] [--rounds R] [--widths W,...]

1. Per width W (one JSON line per width and round): a 61.44 Msps cs16 stream in blocks of 262144 bytes, as in
   bench.py, feeding one spectrum with the reference tool's parameters (F = fs // W, S = fs % W: one row per
   second of stream).  Reported: the spectrum span's time per block from a profiled run (CUDA events around the
   channel stage and the emit pass, xlg_spectrum_profile), its kernel (fft or direct) and counted work.
2. bench.py's cfg2 workload (256 clients at 48 and 96 ksps on a 2.016 Msps cu8 stream, blocks of 262144 bytes,
   device inputs and outputs) without and with a W = 1024 spectrum (F = 1968, S = 768), the two alternated in
   every round: the step time per block between device events (xlg_timer_start / _stop), profiling off.

The card's name, power limit and clocks are printed first, read in the same call.  Nothing is written to the tree.
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


def kernel_run(W, blocks, warmup, data):
    F, S = pkg.spectrogram_params(FS, W)
    g = pkg.Group(FS, BLOCK)
    try:
        sid = g.add_spectrum(W, F, S)
        g.profile_enable(True)
        for i in range(warmup):
            g.wait(g.submit(FMT, data[i % len(data)]))
        g.spectrum_profile_read(reset=True)
        for i in range(blocks):
            g.wait(g.submit(FMT, data[i % len(data)]))
        p = g.spectrum_profile_read()
        kernel = "fft" if g.spectrum_info(sid)[0] == 1 else "direct"
    finally:
        g.close()
    n = p["spectrum_launches"]
    return {"W": W, "F": F, "S": S, "kernel": kernel, "blocks": blocks, "launches": n,
            "kernel_us_per_block": 1e3 * p["spectrum_ms"] / max(n, 1), "frames": p["frames"],
            "channel_flops": p["channel_flops"]}


def step_run(torch, with_spectrum, blocks, warmup):
    import bench
    wl = bench.workload("cfg2", "default")
    host = bench.synth_blocks(wl["fmt"], 8, wl["block_elems"], seed=3)
    dev = torch.from_numpy(host.view(np.uint8).reshape(8, -1)).cuda()
    torch.cuda.synchronize()
    g = pkg.Group(wl["fs"], wl["block_elems"], flags=pkg.XLG_OUT_DEVICE)
    try:
        taps = {}
        for c in wl["plan"]:
            key = (c["cutoff"], c["tw"])
            if key not in taps:
                taps[key] = pkg.create_low_pass_filter(1.0, wl["fs"], c["cutoff"], c["tw"])
            g.add_client(c["decimation"], taps[key], c["center"])
        if with_spectrum:
            g.add_spectrum(1024, *pkg.spectrogram_params(wl["fs"], 1024))
        code = pkg.FMT[wl["fmt"]]

        def feed(k):
            last = -1
            for i in range(k):
                last = g.submit_ptr(code, dev.data_ptr() + (i % 8) * dev.stride(0), wl["block_elems"],
                                    pkg.XLG_INPUT_DEVICE)
            g.wait(last)

        feed(warmup)
        g.timer_start()
        feed(blocks)
        ms = g.timer_stop()
    finally:
        g.close()
    return {"workload": "cfg2", "spectrum": "W=1024" if with_spectrum else "none", "blocks": blocks,
            "step_us_per_block": 1e3 * ms / blocks}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--widths", default="64,1000,1024,4096")
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                           "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()[0]
    print(json.dumps({"card": card}), flush=True)
    import torch
    rng = np.random.default_rng(0)
    data = [rng.integers(-32768, 32767, BLOCK // 2, dtype=np.int16, endpoint=True) for _ in range(4)]
    for r in range(args.rounds):
        for W in [int(w) for w in args.widths.split(",")]:
            print(json.dumps({**kernel_run(W, args.blocks, args.warmup, data), "round": r}), flush=True)
    for r in range(args.rounds):
        for with_spectrum in (False, True):
            print(json.dumps({**step_run(torch, with_spectrum, 10 * args.blocks, args.warmup), "round": r}),
                  flush=True)


if __name__ == "__main__":
    main()
