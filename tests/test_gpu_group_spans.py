"""The batch group's timed spans on the GPU: the XLATING_B200_TIMELINE file, and every kernel family's profile
counters in one mixed group (each family's launches and time land in its own counters, not a neighbour's)."""
import numpy as np
import pytest

from util import rand_block

pytestmark = pytest.mark.gpu

FS = 2048000
MAX_IN = 65536
TILED, GENERIC, POLY_GENERIC, POLY_TILED, CASCADE, MEMBER = 1, 0, 3, 4, 5, 6


def taps(rng, n):
    return rng.standard_normal(n).astype(np.float32) / n


def tiled_clients(g, rng):
    """16 clients of one (D, T): a tiled class."""
    return [g.add_client(64, taps(rng, 257), -900000 + 110000 * c) for c in range(16)]


def test_timeline_rows(pkg, monkeypatch, tmp_path):
    """One row per block with a tiled launch: every ticket once (xlg_destroy harvests the last slots in slot
    order, not ticket order), and each span's stamps in order."""
    path = tmp_path / "timeline.txt"
    monkeypatch.setenv("XLATING_B200_TIMELINE", str(path))
    rng = np.random.default_rng(1)
    g = pkg.Group(FS, MAX_IN)
    try:
        ids = tiled_clients(g, rng)
        N = 9
        for _ in range(N):
            t = g.submit("cu8", rand_block(rng, "cu8", MAX_IN))
            g.wait(t)
        assert {g.client_info(c)[1] for c in ids} == {TILED}
    finally:
        g.close()
    lines = path.read_text().splitlines()
    assert lines[0].startswith("# ticket conv_ready conv_done phase_start phase_done fir_ready fir_done")
    rows = [[float(v) for v in line.split()] for line in lines[1:]]
    assert len(rows) == N
    assert sorted(int(r[0]) for r in rows) == list(range(N))
    for _, conv_ready, conv_done, phase_start, phase_done, fir_ready, fir_done in rows:
        assert conv_ready <= conv_done
        assert phase_start <= phase_done
        assert fir_ready <= fir_done


def test_every_span_in_one_group(pkg):
    """Tiled, generic, rational tiled, rational generic, cascade stage B, sub-band members and a bank all launch
    in every block of one profiled group: each family counts exactly its own launches, with time > 0."""
    rng = np.random.default_rng(2)
    g = pkg.Group(FS, MAX_IN)
    try:
        g.profile_enable(True)
        kinds = {}
        for c in tiled_clients(g, rng):
            kinds[c] = TILED
        kinds[g.add_client(32, taps(rng, 101), 300000)] = GENERIC
        plan = pkg.rational_plan(FS, [48000] * 8)
        for p in plan:
            kinds[g.add_client_rational(p["interp"], p["decim"], p["taps"], p["center"])] = POLY_TILED
        p = plan[0]  # another tap count: a class of one, on the polyphase generic kernel
        kinds[g.add_client_rational(p["interp"], p["decim"], p["taps"][:-3], -p["center"])] = POLY_GENERIC
        kinds[g.add_client_cascade(16, taps(rng, 65), 200000, 4, taps(rng, 33))] = CASCADE
        sid = g.add_subband(32, taps(rng, 129), -400000)
        kinds[g.add_client_subband(sid, 4, taps(rng, 33), 5000)] = MEMBER
        bid = g.add_bank(16, taps(rng, 257))
        g.add_bank_subband(bid, 3)
        for r in (g.profile_read, g.poly_profile_read, g.cascade_profile_read, g.subband_profile_read,
                  g.bank_profile_read):
            r(reset=True)
        N = 6
        for _ in range(N):
            t = g.submit("cu8", rand_block(rng, "cu8", MAX_IN))
            g.wait(t)
        assert {c: g.client_info(c)[1] for c in kinds} == kinds
        prof, poly, casc = g.profile_read(), g.poly_profile_read(), g.cascade_profile_read()
        sub, bank = g.subband_profile_read(), g.bank_profile_read()
    finally:
        g.close()
    spans = [(prof, "convert"), (prof, "phase"), (prof, "fir_tile"), (prof, "fir_generic"),
             (poly, "fir_poly_tile"), (poly, "fir_poly_generic"), (casc, "stage_b"), (sub, "member"),
             (bank, "bank")]
    for counters, name in spans:
        assert counters[f"{name}_launches"] == N, name
        assert counters[f"{name}_ms"] > 0, name
    assert prof["fir_long_launches"] == 0 and prof["fir_long_ms"] == 0
