"""cf32 ingest and the spectrogram tool on the GPU.

    python tools/spectrogram_bench.py [--gib G] [--blocks K] [--warmup W] [--rounds R] [--no-tool]

1. bin/sdr_spectrogram's input rate in MS/s on a generated 61.44 Msps cs16 file of G GiB (default 3) in a temporary
   directory, at W = 1024, 4096 and 65536 (-s 61440000).  Beside it, the rate of reading the same file alone (64 MiB
   reads, page cache as the tool finds it): if the two are close, disk reads bound the tool, otherwise the group.
2. bench.py's cfg2 workload (256 clients at 48 and 96 ksps on a 2.016 Msps stream, blocks of 262144 elements,
   device outputs) fed the same values as cs16 ((2u - 255) * 128) and as cf32 (their exact float images), from
   device memory and from pageable host memory, alternated in every round.  Each reports the step time per block
   between device events (xlg_timer_start / _stop), profiling off, and the H2D bytes per block of a host input.

The card's name, power limit and clocks are printed first, read in the same call.  Nothing is written to the tree.
"""
import argparse
import importlib
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
pkg = importlib.import_module("sdr-server_b200")
TOOL = os.path.join(ROOT, "sdr-server_b200", "bin", "sdr_spectrogram")
FS = 61440000


def tool_rates(gib):
    out = []
    with tempfile.TemporaryDirectory() as d:
        path = os.path.join(d, "band.cs16")
        rng = np.random.default_rng(5)
        chunk = rng.integers(-8192, 8192, 32 << 20, dtype=np.int16)  # 64 MiB, written over and over
        n_chunks = max(1, (gib << 30) // chunk.nbytes)
        with open(path, "wb") as f:
            for i in range(n_chunks):
                chunk[i % chunk.size] ^= 1  # no two chunks alike
                f.write(chunk.tobytes())
        samples = n_chunks * chunk.size // 2
        t0 = time.perf_counter()
        with open(path, "rb", buffering=0) as f:
            while f.read(64 << 20):
                pass
        read_s = time.perf_counter() - t0
        for W in (1024, 4096, 65536):
            png = os.path.join(d, f"w{W}.png")
            t0 = time.perf_counter()
            r = subprocess.run([TOOL, "-w", str(W), "-s", str(FS), "-d", "cs16", "-i", path, "-o", png],
                               capture_output=True, text=True)
            s = time.perf_counter() - t0
            if r.returncode != 0:
                raise RuntimeError(r.stderr)
            rows = samples // FS
            out.append({"tool": "sdr_spectrogram", "W": W, "file_gib": round(samples * 4 / 2 ** 30, 2),
                        "rows": rows, "seconds": round(s, 3), "input_msps": round(rows * FS / s / 1e6, 1),
                        "read_alone_msps": round(samples / read_s / 1e6, 1)})
    return out


def cfg2_run(torch, fmt, ingest, blocks, warmup):
    import bench
    wl = bench.workload("cfg2", "default")
    u = bench.synth_blocks(wl["fmt"], 8, wl["block_elems"], seed=3)
    if fmt == "cs16":
        host = ((u.astype(np.int32) * 2 - 255) * 128).astype(np.int16)
    else:
        host = ((u.astype(np.float64) - 127.5) / 128).astype(np.float32)
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
        code = pkg.FMT[fmt]

        def feed(k):
            last = -1
            for i in range(k):
                if ingest == "device":
                    last = g.submit_ptr(code, dev.data_ptr() + (i % 8) * dev.stride(0), wl["block_elems"],
                                        pkg.XLG_INPUT_DEVICE)
                else:
                    last = g.submit(fmt, host[i % 8])
            g.wait(last)

        feed(warmup)
        g.timer_start()
        feed(blocks)
        ms = g.timer_stop()
    finally:
        g.close()
    return {"workload": "cfg2", "fmt": fmt, "ingest": ingest, "blocks": blocks,
            "step_us_per_block": round(1e3 * ms / blocks, 2),
            "h2d_bytes_per_block": 0 if ingest == "device" else host[0].nbytes}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gib", type=int, default=3)
    ap.add_argument("--blocks", type=int, default=2000)
    ap.add_argument("--warmup", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--no-tool", action="store_true")
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                           "--format=csv,noheader"], capture_output=True, text=True).stdout.strip().splitlines()[0]
    print(json.dumps({"card": card}), flush=True)
    if not args.no_tool:
        for r in tool_rates(args.gib):
            print(json.dumps(r), flush=True)
    import torch
    for r in range(args.rounds):
        for ingest in ("device", "host"):
            for fmt in ("cs16", "cf32"):
                print(json.dumps({**cfg2_run(torch, fmt, ingest, args.blocks, args.warmup), "round": r}), flush=True)


if __name__ == "__main__":
    main()
