"""Throughput of sub-band clients (xlg_add_subband + xlg_add_client_subband) and of bank sub-bands
(xlg_add_bank + xlg_add_bank_subband) against single-stage and per-client cascade clients of the same centres
and rates.

    python tools/subband_bench.py [--blocks K] [--warmup W] [--rounds R] [--only NAME,...] [--plans P,...]

Workloads (centres drawn uniformly across the band from a fixed seed):
  61M_1024   1024 clients at 48 kHz on a 61.44 Msps cs16 stream
  61M_4096   4096 clients at 48 kHz on a 61.44 Msps cs16 stream
  2M_256     256 clients on a 2.016 Msps cu8 stream, 48 and 96 kHz alternating
  2048k_256  256 clients at 48 kHz on a 2.048 Msps cu8 stream (RTL-SDR)
  10M_256    256 clients at 48 kHz on a 10 Msps cs16 stream (Airspy)
  20M_256    256 clients at 48 kHz on a 20 Msps cs8 stream (HackRF)
Plans, alternated within every round: "single" (one client each: client_plan's taps as an integer client, or
rational_plan's as a rational client where the rate does not divide fs), "cascade" (cascade_plan) and
"subband" (subband_plan; at the last three rates its members resample by a rational L2 / M2), "bank"
(subband_plan(bank=True): the same kind of members on the channels of one bank) and "bank_fft"
(subband_plan(bank=True, fft=True): the same with a direct or an FFT bank, whichever the planner costs lower)
and "bank_any" (subband_plan(bank=True, fft=True, any_k=True): chirp-z banks of any even K are candidates too).

Per workload and plan (one JSON line each): input MS/s and step time over K pipelined blocks (CUDA events,
xlg_timer_*), algorithmic real FMAs per input sample from the shapes, and from a profiled run of its own (one
compute stream, CUDA events around each launch) the time per block of the oscillator pre-pass, the integer
FIR kernels, the cascades' stage B and the sub-band members' work (ring appends, member oscillators and
member kernel), the bank kernel and the FFT bank kernel.  Every run checks its last timed block of sampled clients against the tests' oracles (1e-5
norm-wise; a bank's members against the float64 bank rows fed to the reference's float path, since the bank
has no float oscillator to share with an oracle).  Blocks are 262144 bytes, as in bench.py.  The card's name and power limit are printed first,
read in the same call.  Nothing is written to the tree.
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
sys.path.insert(0, os.path.join(ROOT, "tests"))
pkg = importlib.import_module("sdr-server_b200")

BLOCK = 262144
WORKLOADS = {  # fs, format, clients, rates
    "61M_1024": (61440000, "cs16", 1024, (48000,)),
    "61M_4096": (61440000, "cs16", 4096, (48000,)),
    "2M_256": (2016000, "cu8", 256, (48000, 96000)),
    "2048k_256": (2048000, "cu8", 256, (48000,)),
    "10M_256": (10000000, "cs16", 256, (48000,)),
    "20M_256": (20000000, "cs8", 256, (48000,)),
}
PLANS = ("single", "cascade", "subband", "bank", "bank_fft", "bank_any")
SAMPLED = 3


def workload_clients(name):
    fs, _, n, rates = WORKLOADS[name]
    rng = np.random.default_rng(7)
    rmax = max(rates)
    centres = rng.integers(-fs // 2 + rmax, fs // 2 - rmax, n)
    return [(int(c), rates[i % len(rates)]) for i, c in enumerate(centres)]


def build(name, plan, profile):
    """The group of one plan, its client ids, FMAs per input sample, and oracles of SAMPLED clients
    (callables block -> cf32 outputs)."""
    from cascade import cascade_oracle
    from cascade_rational import RationalCascadeOracle
    from oracle import pyoracle as po
    from rational import oracle_filter, stuff
    from bank_exact import BankMemberOracle
    from subband_rational import RationalSubbandOracle
    fs, fmt, n, _ = WORKLOADS[name]
    clients = workload_clients(name)
    g = pkg.Group(fs, BLOCK)
    picks = [0, n // 2, n - 1]
    oracles = []
    shape = {}
    if plan == "single" and any(fs % r for _, r in clients):
        rp = pkg.rational_plan(fs, [r for _, r in clients])
        ids = [g.add_client_rational(q["interp"], q["decim"], q["taps"], c) for q, (c, _) in zip(rp, clients)]
        fmas = sum(4.0 * -(-q["taps"].size // q["interp"]) * q["rate"] / fs for q in rp)
        for k in picks:
            q, (c, _) = rp[k], clients[k]
            o = oracle_filter(po, q["interp"], q["decim"], q["taps"], c, fs, BLOCK)
            oracles.append((ids[k], lambda x, o=o, L=q["interp"]: o.process_cf32("cs16", stuff(fmt, x, L))))
    elif plan == "single":
        taps = {r: pkg.create_low_pass_filter(1.0, fs, r // 2, r // 5) for _, r in clients}
        ids = [g.add_client(fs // r, taps[r], c) for c, r in clients]
        fmas = sum(4.0 * taps[r].size / (fs // r) for _, r in clients)
        for k in picks:
            c, r = clients[k]
            o = po.OracleFilter(fs // r, taps[r], c, fs, BLOCK)
            oracles.append((ids[k], lambda x, o=o: o.process_cf32(fmt, x)))
    elif plan == "cascade":
        plans = {r: pkg.cascade_plan(fs, [r])[0] for _, r in clients}
        ids = [g.add_client_cascade(plans[r]["d1"], plans[r]["taps1"], c, plans[r]["d2"], plans[r]["taps2"],
                                    plans[r]["interp2"]) for c, r in clients]
        fmas = sum(plans[r]["fmas"] for _, r in clients)
        for k in picks:
            c, r = clients[k]
            p = plans[r]
            o = (RationalCascadeOracle(p["d1"], p["taps1"], c, p["interp2"], p["d2"], p["taps2"], fs, BLOCK)
                 if p["interp2"] > 1 else cascade_oracle(p["d1"], p["taps1"], c, p["d2"], p["taps2"], fs, BLOCK))
            oracles.append((ids[k], lambda x, o=o: o.process_cf32(fmt, x)))
    else:
        banked = plan in ("bank", "bank_fft", "bank_any")
        p = (pkg.subband_plan(fs, clients, bank=True, fft=True, any_k=plan == "bank_any")
             if plan in ("bank_fft", "bank_any") else pkg.subband_plan(fs, clients, bank=banked))
        shape = {"d1": p["d1"], "subbands": len(p["subbands"]), "kernel": p.get("kernel")}
        if banked:
            kernel = p.get("kernel")
            bid = (g.add_bank_fft(p["d1"], p["taps1"], any_k=kernel == "czt") if kernel in ("fft", "czt") else
                   g.add_bank(p["d1"], p["taps1"]))
            sids = [g.add_bank_subband(bid, sb["channel"]) for sb in p["subbands"]]
        else:
            sids = [g.add_subband(p["d1"], p["taps1"], sb["center"]) for sb in p["subbands"]]
        ids = [g.add_client_subband(sids[m["subband"]], m["d2"], m["taps2"], m["offset"], m["interp2"])
               for m in p["members"]]
        fmas = p["fmas"]
        for k in picks:
            m = p["members"][k]
            if banked:
                o = BankMemberOracle(p["d1"], p["taps1"], p["subbands"][m["subband"]]["channel"], m["d2"], m["taps2"],
                                     m["offset"], m["interp2"], fs)
                oracles.append((ids[k], lambda x, o=o: o.process_cf32(fmt, x)))
                continue
            o = RationalSubbandOracle(p["d1"], p["taps1"], p["subbands"][m["subband"]]["center"], fs, BLOCK)
            o.add_member(0, m["d2"], m["taps2"], m["offset"], m["interp2"])
            oracles.append((ids[k], lambda x, o=o: o.process_cf32(fmt, x)[0]))
    if profile:
        g.profile_enable(True)
    return g, ids, fmas, oracles, shape


def run(name, plan, blocks, warmup):
    fs, fmt, n, _ = WORKLOADS[name]
    rng = np.random.default_rng(0)
    dtype = pkg.NP_DTYPE[fmt]
    elems = BLOCK // np.dtype(dtype).itemsize
    data = [rng.integers(np.iinfo(dtype).min, np.iinfo(dtype).max, elems, dtype=dtype, endpoint=True) for _ in range(4)]
    g, ids, fmas, oracles, shape = build(name, plan, False)
    res = {"workload": name, "plan": plan, "fs": fs, "fmt": fmt, "clients": n, "blocks": blocks,
           "fmas_per_input_sample": fmas, **shape}
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
    worst = 0.0
    for cid, o in oracles:
        for i in range(warmup + blocks):
            r = o(data[i % 4])
        y = g.output(t, cid)
        assert y.shape == r.shape, (name, plan, y.shape, r.shape)
        worst = max(worst, float(np.max(np.abs(y - r)) / np.max(np.abs(r))))
    assert worst <= 1e-5, (name, plan, worst)
    res["checked_error"] = worst
    g.close()
    g, ids, _, _, _ = build(name, plan, True)
    for i in range(warmup):
        g.wait(g.submit(fmt, data[i % 4]))
    for read in (g.profile_read, g.cascade_profile_read, g.subband_profile_read, g.bank_profile_read,
                 g.bank_fft_profile_read):
        read(reset=True)
    for i in range(blocks):
        g.wait(g.submit(fmt, data[i % 4]))
    prof, cp, sp, bp = g.profile_read(), g.cascade_profile_read(), g.subband_profile_read(), g.bank_profile_read()
    fp = g.bank_fft_profile_read()
    g.close()
    per = max(prof["blocks"], 1)
    res["phase_ms_per_block"] = prof["phase_ms"] / per
    res["fir_ms_per_block"] = (prof["fir_tile_ms"] + prof["fir_generic_ms"] + prof["fir_long_ms"]) / per
    res["stage_b_ms_per_block"] = cp["stage_b_ms"] / per
    res["member_ms_per_block"] = sp["member_ms"] / per
    res["bank_ms_per_block"] = bp["bank_ms"] / per
    res["fft_ms_per_block"] = fp["fft_ms"] / per
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--blocks", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--only", default=None, help="workloads, comma-separated")
    ap.add_argument("--plans", default=",".join(PLANS), help="plans to alternate, comma-separated")
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip().splitlines()[0]
    print(json.dumps({"card": card}), flush=True)
    names = args.only.split(",") if args.only else list(WORKLOADS)
    for r in range(args.rounds):
        for name in names:
            for plan in args.plans.split(","):
                res = run(name, plan, args.blocks, args.warmup)
                res["round"] = r
                print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
