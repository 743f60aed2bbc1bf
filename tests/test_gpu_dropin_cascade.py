"""Cascade (two-stage) filters of the per-filter drop-in ABI (create_cascade_frequency_xlating_filter) on the
GPU.

A cascade filter is, call for call, the client of xlg_add_client_cascade_rational attached to a fresh group of
the same band and fed the filter's calls as its blocks (include/xlating.h).  The scenarios run in
tests/_dropin_cascade_worker.py, one subprocess per engine configuration (the engine reads its switches once
per process)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
PRIVATE = {"XLATING_B200_STREAM": "0"}


def run(scenario, *args, env=None):
    e = dict(os.environ)
    e.update(env or {})
    cmd = [sys.executable, os.path.join(ROOT, "tests", "_dropin_cascade_worker.py"), scenario] + [str(a) for a in args]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=e)
    assert r.stdout.strip(), r.stderr[-2000:]
    line = json.loads(r.stdout.strip().splitlines()[-1])
    assert r.returncode == 0 and not line["errors"], (line, r.stderr[-1500:])
    line["stderr"] = r.stderr
    return line


def same_dumps(a, b):
    names = sorted(os.listdir(a))
    assert names == sorted(os.listdir(b)) and names
    for n in names:
        x, y = np.load(a / n), np.load(b / n)
        assert x.size > 0 and np.array_equal(x.view(np.uint64), y.view(np.uint64)), n


def test_exact_stimuli_every_format():
    """Integer cascades (odd and even D2), L2 = 2, 3, 12 and gcd(L2, M2) > 1 over full, 30001, 2, 0, 7 and
    65534-element calls and enough full calls to wrap every stage-A ring: the float64 composition bit for bit."""
    line = run("exact")
    assert line["filters"] == 18 and line["ring_wraps"] == 18


@pytest.fixture(scope="module")
def designed(tmp_path_factory):
    """The designed-taps scenario on the default engine: counts of the composed oracle, 1e-5 against it, and
    the bits of a Group(flags=XLG_FORCE_GENERIC) fed the same blocks."""
    d = tmp_path_factory.mktemp("designed")
    line = run("designed", d)
    return d, line


def test_designed_taps_against_oracle_and_group(designed):
    _, line = designed
    assert line["cascades"] == 14 and set(line["kinds"]) == {"c", "i", "r"}
    # integer stage B with even and odd D2, rational with even and odd M2
    assert line["d2_parity"] == [[False, 0], [False, 1], [True, 0], [True, 1]]
    assert line["shared"] > 0


def test_group_model_gives_the_same_bits(designed, tmp_path):
    """XLATING_B200_DROPIN=group: each filter a private one-client group."""
    run("designed", tmp_path, env={"XLATING_B200_DROPIN": "group"})
    same_dumps(designed[0], tmp_path)


@pytest.mark.parametrize("case", ["lone", "lanes1", "no_share", "osc_host", "osc_device", "osc_lanes"])
def test_engine_paths_give_the_same_bits(designed, tmp_path, case):
    """lone: one filter alive at a time (each call walks its host oscillator while the front kernel converts);
    lanes1: one launch lane for all the threads, so cascade, rational, integer and Q15 calls share batches;
    no_share: every call stages its own input; osc_*: every oscillator walk."""
    env = {"lanes1": {"XLATING_B200_LANES": "1"}, "no_share": {"XLATING_B200_SHARE": "0"},
           "osc_host": {"XLATING_B200_OSC": "host"}, "osc_device": {"XLATING_B200_OSC": "device"},
           "osc_lanes": {"XLATING_B200_OSC": "lanes"}}.get(case)
    line = run("designed", tmp_path, *(["lone"] if case == "lone" else []), env=env)
    same_dumps(designed[0], tmp_path)
    if case == "lanes1":
        assert 0 < line["batches"] < line["calls"]
    if case == "lone":
        assert line["batches"] == line["calls"] > 0
    if case == "no_share":
        assert line["shared"] == 0 and line["calls"] > 0


def test_neighbours_keep_their_bits_and_their_group():
    """Overlay on: integer and rational filters of one band give the same bits with and without cascade
    filters alive, still join their band's group and are served by it; no cascade filter is a member."""
    line = run("neighbours")
    before, after = line["stream"]["before"], line["stream"]["after"]
    # read while each run's filters were alive: the band's stream counts (joins, members) are those of that
    # run's stream; served_by_group counts the process
    assert before["joins"] > 0 and after["joins"] > 0
    assert before["served_by_group"] > 0 and after["served_by_group"] > before["served_by_group"]
    assert before["members"] == after["members"] == line["filters"]


def test_refused_q15_call_consumes_nothing():
    """process_*_cs16 on a cascade filter: 0 outputs, one <3> line for two calls, and the cf32 stream carries
    on bit for bit as if the calls had not been made."""
    line = run("q15refuse", env=PRIVATE)
    assert line["refused"] == [0, 0]
    assert line["stderr"].count("Q15 output is not available for a cascade filter") == 1
    assert line["stderr"].count("<3>") == 1


def test_pool_reuse_starts_from_zero_history(tmp_path):
    """Cascade, rational and integer filters created and destroyed interleaved, the cascade arena growing under
    filters that have run: every cascade filter's calls equal those of one filter in a fresh process."""
    line = run("pool", tmp_path)
    run("pool", tmp_path, "fresh")
    pool, fresh = np.load(tmp_path / "pool.npz"), np.load(tmp_path / "fresh.npz")
    calls = [fresh[f"c{b}"] for b in range(4)]
    seen = set()
    for i in range(line["filters"]):
        n = int(pool[f"n{i}"])
        want = np.concatenate(calls[:n])
        assert np.array_equal(pool[f"f{i}"].view(np.uint64), want.view(np.uint64)), i
        seen.add(n)
    assert seen == {4}


@pytest.mark.parametrize("workload,taps", [("cascade", "79 481"), ("wide", "15419")])
def test_dropin_bench_workloads(workload, taps):
    """bin/dropin_bench's cascade and wide workloads complete and design the taps of cascade_plan(61.44 Msps,
    48 kHz) and of the server's single-stage designer."""
    exe = os.path.join(ROOT, "sdr-server_b200", "bin", "dropin_bench")
    r = subprocess.run([exe, "4", "4", "0", "1", workload], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    assert f"taps {taps}" in r.stdout + r.stderr, (r.stdout, r.stderr[-500:])
