"""Client spectra (xlg_add_client_spectrum): what a spectrum on every client adds to a step of clients.

    python tools/client_spectrum_bench.py [--blocks K] [--warmup W] [--rounds R]

bench.py's cfg2 workload (256 clients at 48 and 96 ksps on a 2.016 Msps cu8 stream, blocks of 262144 bytes,
device inputs and outputs) without spectra and with one W = 1024 spectrum per client at the reference tool's
parameters for the client's rate (spectrogram_params(rate, 1024): one row per second of the client's output).
The two versions alternate in every round; each reports the step time per block between device events
(xlg_timer_start / _stop), profiling off.  A separate profiled run with the spectra reports the spectrum span per
block (CUDA events around the appends, the channel stages and the emit pass, xlg_spectrum_profile) and its work.

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
W = 1024


def run(torch, with_spectra, blocks, warmup, profile=False):
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
            cid = g.add_client(c["decimation"], taps[key], c["center"])
            if with_spectra:
                g.add_client_spectrum(cid, W, *pkg.spectrogram_params(wl["fs"] // c["decimation"], W))
        code = pkg.FMT[wl["fmt"]]

        def feed(k):
            last = -1
            for i in range(k):
                last = g.submit_ptr(code, dev.data_ptr() + (i % 8) * dev.stride(0), wl["block_elems"],
                                    pkg.XLG_INPUT_DEVICE)
            g.wait(last)

        if profile:
            g.profile_enable(True)
        feed(warmup)
        g.spectrum_profile_read(reset=True)
        g.timer_start()
        feed(blocks)
        ms = g.timer_stop()
        p = g.spectrum_profile_read()
    finally:
        g.close()
    out = {"workload": "cfg2", "spectra": f"{len(wl['plan'])} x W={W}" if with_spectra else "none",
           "blocks": blocks}
    if profile:
        n = max(p["spectrum_launches"], 1)
        out.update({"profiled": True, "spectrum_us_per_block": 1e3 * p["spectrum_ms"] / n,
                    "launches": p["spectrum_launches"], "frames": p["frames"], "channel_flops": p["channel_flops"]})
    else:
        out["step_us_per_block"] = 1e3 * ms / blocks
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=2000)
    ap.add_argument("--warmup", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                           "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()[0]
    print(json.dumps({"card": card}), flush=True)
    import torch
    for r in range(args.rounds):
        for with_spectra in (False, True):
            print(json.dumps({**run(torch, with_spectra, args.blocks, args.warmup), "round": r}), flush=True)
    print(json.dumps(run(torch, True, args.blocks, args.warmup, profile=True)), flush=True)


if __name__ == "__main__":
    main()
