"""Rational (L/M) filters of the per-filter drop-in ABI (create_rational_frequency_xlating_filter) on the
GPU, and xlg_add_client_rational_ex, through which the drop-in engine hands such a filter's state to its
band's batch group.

A rational filter is the filter with decimation M at L * fs fed the zero-stuffed stream
(tests/rational.py).  The drop-in scenarios run in tests/_dropin_rational_worker.py, one subprocess per
engine configuration (the engine reads its switches once per process)."""
import errno
import json
import os
import subprocess
import sys

import numpy as np
import pytest

from oracle import pyoracle as po
from rational import oracle_filter, stuff
from util import assert_cf32_close, rand_block

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MAX_IN = 65536
RAGGED = [65536, 65536, 30001, 2, 0, 65536, 12347, 65536, 7, 65534]
PRIVATE = {"XLATING_B200_STREAM": "0"}


def run(scenario, arg=None, env=None):
    e = dict(os.environ)
    e.update(env or {})
    cmd = [sys.executable, os.path.join(ROOT, "tests", "_dropin_rational_worker.py"), scenario]
    if arg is not None:
        cmd.append(str(arg))
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=900, env=e)
    assert r.stdout.strip(), r.stderr[-2000:]
    line = json.loads(r.stdout.strip().splitlines()[-1])
    assert r.returncode == 0 and not line["errors"], (line, r.stderr[-1500:])
    line["stderr"] = r.stderr
    return line


@pytest.mark.parametrize("stream", ["1", "0"], ids=["overlay", "private"])
@pytest.mark.parametrize("osc", ["host", "device"])
def test_interp_one_is_the_integer_filter(osc, stream):
    """interpolation = 1 is create_frequency_xlating_filter bit for bit, cf32 and Q15.  With the overlay on,
    exact stimuli make the bits independent of which engine served a call."""
    run("interp1", "exact" if stream == "1" else "designed", {"XLATING_B200_OSC": osc, "XLATING_B200_STREAM": stream})


def test_private_engine_rows_and_group_model(tmp_path):
    """Every rate-table row over ragged blocks (0- and 2-element calls, ring wraps): output counts of the
    strict oracle on the zero-stuffed stream, 1e-5 against it, and the bits of the same clients in a Group
    on the polyphase generic kernel.  XLATING_B200_DROPIN=group gives the private engine's bits."""
    priv, grp = tmp_path / "private", tmp_path / "group"
    priv.mkdir()
    grp.mkdir()
    assert run("private", priv, PRIVATE)["group_kinds"] == [3]
    run("private", grp, {"XLATING_B200_DROPIN": "group"})
    names = sorted(os.listdir(priv))
    assert names == sorted(os.listdir(grp)) and len(names) == 12
    for n in names:
        a, b = np.load(priv / n), np.load(grp / n)
        assert a.size > 0 and np.array_equal(a.view(np.uint64), b.view(np.uint64)), n


@pytest.mark.parametrize("env", [None, PRIVATE], ids=["overlay", "private"])
def test_exact_stimuli_every_format(env):
    line = run("exact", env=env)
    if env is None:
        assert line["stream"]["served_by_group"] > 0


@pytest.mark.parametrize("env", [None, PRIVATE], ids=["overlay", "private"])
def test_wide_interpolations_exact(env):
    """L from 4 to 441 on exact stimuli: dropin_fir_poly_kernel's span of residues cut at 16 (L >= 16) and
    calls with fewer outputs than L (441/20480)."""
    line = run("wide", env=env)
    assert line["long_spans"] > 0 and line["fewer_than_L"] > 0


@pytest.mark.parametrize("stream", ["1", "0"], ids=["overlay", "private"])
@pytest.mark.parametrize("osc", ["host", "device", "lanes"])
def test_phase_one_hot_at_any_centre(osc, stream):
    """Branch-one-hot rational and one-hot integer filters at nonzero centres on a real input equal the strict
    oracle bit for bit under every oscillator walk (the host one mirrors the output count in upsampled
    coordinates), and dyadic integer filters at centre 0 on the same stream the float64 sum.  With the
    overlay on and the host walk, filters join the band's group: the phase is handed over and back."""
    line = run("phase", env={"XLATING_B200_OSC": osc, "XLATING_B200_STREAM": stream})
    if stream == "1" and osc == "host":
        st = line["stream"]
        assert st["joins"] > 0 and st["served_by_group"] > 0 and st["published"] > 0


@pytest.mark.parametrize("case", ["lone", "lanes1", "no_share"])
def test_phase_one_hot_engine_paths(case):
    """The phase scenario on the private engine's other paths.  lone: one filter alive at a time, so each call
    walks its host oscillator while the front kernel converts; lanes1: one launch lane, so calls share
    batches; no_share: every call stages its own input."""
    if case == "lone":
        line = run("phase", "lone")
        # no filter ever had a band group (which appears with a second live filter of the band, see the
        # overlay case of test_phase_one_hot_at_any_centre) and every batch held one call
        assert line["alone"] == line["filters"] > 0 and line["batches"] == line["calls"] > 0
    elif case == "lanes1":
        line = run("phase", env={**PRIVATE, "XLATING_B200_LANES": "1"})
        assert 0 < line["batches"] < line["calls"]
    else:
        assert run("phase", env=PRIVATE)["shared"] > 0  # the same calls share staged inputs by default
        line = run("phase", env={**PRIVATE, "XLATING_B200_SHARE": "0"})
        assert line["shared"] == 0 and line["calls"] > 0


def test_combined_calls_mix_rational_integer_and_q15():
    """24 threads released together; one launch lane, so calls that overlap must share a batch."""
    line = run("combined", env={**PRIVATE, "XLATING_B200_LANES": "1"})
    assert 0 < line["batches"] < line["calls"]


def test_integer_filters_unchanged_by_rational_neighbours():
    run("neighbours", env=PRIVATE)


def test_overlay_steady():
    line = run("overlay", "steady")
    st, n = line["stream"], line["filters"]
    assert st["joins"] == n and st["desyncs"] == 0 and st["members"] == n
    assert st["served_by_group"] >= 0.8 * line["calls"]


def test_overlay_drops_desync_and_rejoin():
    line = run("overlay", "drops")
    st, n = line["stream"], line["filters"]
    assert st["desyncs"] >= 1 and st["joins"] > n and st["served_by_group"] > 0


def test_overlay_late_attachers_join():
    line = run("overlay", "late")
    st, n = line["stream"], line["filters"]
    assert st["desyncs"] == 0 and st["joins"] >= 0.75 * n and st["served_by_group"] > 0


def test_overlay_lagging_filter_is_served_privately():
    line = run("overlay", "lag", {"XLATING_B200_STREAM_RING": "4"})
    assert line["stream"]["desyncs"] >= 1


def test_refused_q15_call_consumes_nothing():
    """process_*_cs16 on a rational filter: 0 outputs, one <3> line for two calls, the cf32 stream carries
    on as if the call had not been made (bit-exact), and the filter stays a member of its band's group."""
    line = run("q15refuse")
    assert line["refused"] == [0, 0]
    assert line["stderr"].count("Q15 output is not available") == 1
    assert "<3>" in line["stderr"]
    assert line["stream"]["members"] == 4 and line["stream"]["desyncs"] == 0


# ---- xlg_add_client_rational_ex ----

@pytest.mark.parametrize("interp_one", [False, True], ids=["rational", "interp1"])
def test_reattach_continues_bit_for_bit(pkg, monkeypatch, interp_one):
    """A client re-attached mid-stream to a second group with the XLG_TRACK_STATE state of the first
    equals the uninterrupted client bit for bit (both on the generic kernels)."""
    monkeypatch.setenv("XLATING_B200_POLY_TILE", "0")
    fs = 2048000
    p = pkg.rational_plan(fs, [48000])[0]
    L, M, taps = (1, 32, pkg.create_low_pass_filter(1.0, fs, 32000, 12800)) if interp_one else \
        (p["interp"], p["decim"], p["taps"])
    rng = np.random.default_rng(13)
    blocks = [rand_block(rng, "cu8", n) for n in RAGGED]
    a = pkg.Group(fs, MAX_IN, flags=pkg.XLG_TRACK_STATE)
    b = pkg.Group(fs, MAX_IN)
    ca = a.add_client_rational(L, M, taps, p["center"])
    b.add_client(64, np.ones(5, np.float32), 0)  # B runs the stream before the hand-over
    cut, consumed, st, want, got = 6, 0, None, [], []
    for i, x in enumerate(blocks):
        if i == cut:
            st.valid_history = consumed
            cb = b.add_client_rational(L, M, taps, p["center"], state=st)
        ta, tb = a.submit("cu8", x), b.submit("cu8", x)
        a.wait(ta)
        b.wait(tb)
        y, st = a.copy_output(ta, ca)
        want.append(y)
        if i >= cut:
            got.append(b.output(tb, cb))
        consumed += x.size // 2
    a.close()
    b.close()
    for i, (y, r) in enumerate(zip(got, want[cut:])):
        assert np.array_equal(y.view(np.uint64), r.view(np.uint64)), f"block {cut + i}"
    o = oracle_filter(po, L, M, taps, p["center"], fs, MAX_IN)
    ref = [o.process_cf32("cs16", stuff("cu8", x, L)) for x in blocks]
    assert_cf32_close(np.concatenate(got), np.concatenate(ref[cut:]), "re-attached client")


def test_interp_one_is_add_client_ex(pkg):
    fs = 2016000
    taps = pkg.create_low_pass_filter(1.0, fs, 24000, 9600)
    rng = np.random.default_rng(19)
    blocks = [rand_block(rng, "cs16", n) for n in RAGGED[:6]]
    outs = []
    for rational in (False, True):
        g = pkg.Group(fs, MAX_IN)
        st = pkg.XlgClientState(0, 100, 0.6, 0.8)
        if rational:
            cid = g.add_client_rational(1, 42, taps, -312000, state=st)
        else:
            cid = g.add_client(42, taps, -312000, state=st)
        got = []
        for x in blocks:
            t = g.submit("cs16", x)
            g.wait(t)
            got.append(g.output(t, cid))
        outs.append(got)
        g.close()
    for a, b in zip(*outs):
        assert np.array_equal(a.view(np.uint64), b.view(np.uint64))


def test_rational_ex_argument_errors(pkg):
    taps = np.ones(97, dtype=np.float32)
    g = pkg.Group(2048000, MAX_IN)
    for st in (pkg.XlgClientState(0, -1, 1, 0), pkg.XlgClientState(0, 98, 1, 0), pkg.XlgClientState(-1, 10, 1, 0)):
        with pytest.raises(ValueError, match=str(-errno.EINVAL)):
            g.add_client_rational(3, 128, taps, 0, state=st)
    with pytest.raises(ValueError, match=str(-errno.EINVAL)):
        g.add_client_rational(0, 128, taps, 0, state=pkg.XlgClientState(0, 10, 1, 0))
    assert g.client_count() == 0
    g.remove_client(g.add_client_rational(3, 128, taps, 0, state=pkg.XlgClientState(0, 97, 1, 0)))
    g.close()
