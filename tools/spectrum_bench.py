"""Spectrum rows (xlg_add_spectrum): the spectrum kernels alone, and what a spectrum adds to a step of clients.

    python tools/spectrum_bench.py [--blocks K] [--warmup W] [--rounds R] [--widths W,...] [--variants V,...]
                                   [--no-step]

1. Per width W and variant (one JSON line each, the variants alternated within every round): a 61.44 Msps cs16
   stream in blocks of 262144 bytes, as in bench.py, feeding one spectrum with the reference tool's parameters
   (F = fs // W, S = fs % W: one row per second of stream).  Variants: "plain" (xlg_add_spectrum), "hann" (a Hann
   window, H = W, max) and "hann_mean" (a Hann window, H = W / 2, the mean: Welch's method at 50 % overlap, with
   F = 2 fs // W - 1 so that a row still spans about a second).  Reported: the spectrum span's time per block
   from a profiled run (CUDA events around the channel stages, the fold and the emit pass, xlg_spectrum_profile),
   its kernel (direct, fft, wide_fft at powers of two above W = 4096, or czt: every other width above 4096, served
   through xlg_add_spectrum_any) and counted work.
2. bench.py's cfg2 workload (256 clients at 48 and 96 ksps on a 2.016 Msps cu8 stream, blocks of 262144 bytes,
   device inputs and outputs) without a spectrum, with a W = 1024 spectrum (F = 1968, S = 768) and with a
   W = 1024, H = 512 Hann mean spectrum (F = 3935, S = 768), alternated in every round: the step time per block
   between device events (xlg_timer_start / _stop), profiling off.  --no-step leaves this part out.

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


def hann(W):
    return (0.5 - 0.5 * np.cos(2 * np.pi * np.arange(W) / W)).astype(np.float32)


def add(g, fs, W, variant):
    """One spectrum of the band in the given variant, at the reference tool's row length."""
    F, S = pkg.spectrogram_params(fs, W)
    any_width = W > 4096 and W & (W - 1) != 0  # the chirp-z stage
    if variant == "plain":
        return g.add_spectrum(W, F, S, any_width=any_width), F, S
    if variant == "hann":
        return g.add_spectrum(W, F, S, hop=W, window=hann(W), any_width=any_width), F, S
    F = 2 * F - 1  # (F - 1) W / 2 + W + S = the plain row's F W + S
    return g.add_spectrum(W, F, S, hop=W // 2, window=hann(W), mean=True, any_width=any_width), F, S


def kernel_run(W, variant, blocks, warmup, data):
    g = pkg.Group(FS, BLOCK)
    try:
        sid, F, S = add(g, FS, W, variant)
        g.profile_enable(True)
        for i in range(warmup):
            g.wait(g.submit(FMT, data[i % len(data)]))
        g.spectrum_profile_read(reset=True)
        for i in range(blocks):
            g.wait(g.submit(FMT, data[i % len(data)]))
        p = g.spectrum_profile_read()
        kernel = ("direct", "fft", "wide_fft", "czt")[g.spectrum_info(sid)[0]]
    finally:
        g.close()
    n = p["spectrum_launches"]
    return {"W": W, "variant": variant, "F": F, "S": S, "kernel": kernel, "blocks": blocks, "launches": n,
            "kernel_us_per_block": 1e3 * p["spectrum_ms"] / max(n, 1), "frames": p["frames"],
            "channel_flops": p["channel_flops"]}


def step_run(torch, spectrum, blocks, warmup):
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
        if spectrum != "none":
            add(g, wl["fs"], 1024, spectrum)
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
    label = spectrum if spectrum == "none" else f"W=1024 {spectrum}"
    return {"workload": "cfg2", "spectrum": label, "blocks": blocks,
            "step_us_per_block": 1e3 * ms / blocks}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--widths", default="64,1000,1024,4096")
    ap.add_argument("--variants", default="plain,hann,hann_mean")
    ap.add_argument("--no-step", action="store_true")
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                           "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()[0]
    print(json.dumps({"card": card}), flush=True)
    import torch
    rng = np.random.default_rng(0)
    data = [rng.integers(-32768, 32767, BLOCK // 2, dtype=np.int16, endpoint=True) for _ in range(4)]
    variants = args.variants.split(",")
    for r in range(args.rounds):
        for W in [int(w) for w in args.widths.split(",")]:
            for v in variants:
                print(json.dumps({**kernel_run(W, v, args.blocks, args.warmup, data), "round": r}), flush=True)
    for r in range(0 if args.no_step else args.rounds):
        for spectrum in ["none"] + [v for v in variants if v != "hann"]:
            print(json.dumps({**step_run(torch, spectrum, 10 * args.blocks, args.warmup), "round": r}), flush=True)


if __name__ == "__main__":
    main()
