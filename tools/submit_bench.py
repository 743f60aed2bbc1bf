"""(from the repo root: python tools/submit_bench.py [workload] [blocks])
host time inside xlg_submit per block (xlg_profile's host_submit_ms over its submits) on bench.py's timed path:
device-resident inputs, device outputs, the workload's clients; prints one JSON line"""
import importlib, json, os, sys, time
import numpy as np
sys.path.insert(0, os.getcwd())
import bench, torch
pkg = importlib.import_module("sdr-server_b200")
name = sys.argv[1] if len(sys.argv) > 1 else "cfg2"
K = int(sys.argv[2]) if len(sys.argv) > 2 else 2000
wl = bench.workload(name, "default")
NB = 8
host_blocks = bench.synth_blocks(wl["fmt"], NB, wl["block_elems"], seed=3)
dev = torch.from_numpy(host_blocks.view(np.uint8).reshape(NB, -1)).cuda()
fmt = pkg.FMT[wl["fmt"]]
tapsets = {}
g = pkg.Group(wl["fs"], wl["block_elems"], flags=pkg.XLG_OUT_DEVICE | pkg.XLG_SM_PARTITION)
for p in wl["plan"]:
    key = (p["cutoff"], p["tw"])
    if key not in tapsets:
        tapsets[key] = pkg.create_low_pass_filter(1.0, wl["fs"], p["cutoff"], p["tw"])
    g.add_client(p["decimation"], tapsets[key], p["center"])
def run(k):
    last = -1
    for i in range(k):
        last = g.submit_ptr(fmt, dev.data_ptr() + (i % NB) * dev.stride(0), wl["block_elems"], pkg.XLG_INPUT_DEVICE)
    g.wait(last)
run(200)
g.profile_read(reset=True)
torch.cuda.synchronize(); t0 = time.perf_counter()
run(K)
torch.cuda.synchronize(); wall = time.perf_counter() - t0
p = g.profile_read(reset=True)
g.close()
print(json.dumps({"workload": name, "blocks": int(p["submits"]),
                  "host_submit_us_per_block": round(p["host_submit_ms"] * 1e3 / p["submits"], 3),
                  "host_wait_us_per_block": round(p["host_wait_ms"] * 1e3 / p["submits"], 3),
                  "wall_us_per_block": round(wall * 1e6 / K, 3),
                  "gpu": torch.cuda.get_device_name(0)}), flush=True)
