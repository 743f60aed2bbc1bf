"""Cascade stage B bit for bit on the GPU: designed and random taps against the kernel model (tests/cascade_exact.py),
exact stimuli against the float64 composition, at every CTA size of both stage-B kernels, at the shared-memory
bound, and with clients of different CTA sizes in one group.

Every cascade client is paired with an integer client (D1, taps1, centre) in the same group: that client's
outputs are the cascade's stage-A rows (tests/test_gpu_cascade.py's single-tap test shows it bit for bit), and
both are asserted to run on the same stage-A kind.  Every comparison is on the bits.
"""
import errno

import numpy as np
import pytest

from cascade import small_taps
from cascade_exact import (INT_KO_CASES, RAT_CASES, SLOTS, f64_stage_b, max_t2, ring_cap, ring_windows,
                           stage_b_ko, stage_b_model, stage_b_walk)
from exact import exact_input
from subband_exact import exact_bound
from test_gpu_cascade_rational import run_group
from util import rand_block

pytestmark = pytest.mark.gpu

CENTRES = [0, -312000, 17, 251001, -1000003]


def spec_pair(d1, t1, centre, m2, t2, l2=1):
    """A cascade client and its stage-A twin."""
    return [("c", d1, t1, centre, m2, t2, l2), ("i", d1, t1, centre)]


def pairs(clients):
    """(cascade client, its twin) of a client list built from spec_pair, each pair on one stage-A kind."""
    out = []
    for c, ci in zip(clients[0::2], clients[1::2]):
        assert c["spec"][0] == "c" and ci["spec"][0] == "i" and c["first"] == ci["first"]
        assert c["spec"][1] == ci["spec"][1] and c["spec"][3] == ci["spec"][3]
        assert c["kinds"] == ci["kinds"], (c["kinds"], ci["kinds"])
        out.append((c, ci))
    return out


def model_diff(c, ci, fs, ko=None):
    """(block, output indices) where the cascade client differs from stage_b_model of its twin's rows at ko
    (default: its own)."""
    _, d1, _, _, m2, t2, l2 = c["spec"]
    ko = ko or stage_b_ko(l2, m2, len(t2))
    want = stage_b_model(ci["got"], 0, l2, m2, t2, fs // d1, ko)
    assert [y.size for y in c["got"]] == [r.size for r in want], c["cid"]
    return [(b, np.flatnonzero(y != r)) for b, (y, r) in enumerate(zip(c["got"], want)) if np.any(y != r)]


def check_model(c, ci, fs):
    bad = model_diff(c, ci, fs)
    assert not bad, (f"client {c['cid']} {c['spec'][4:7:2]}: {len(bad)} blocks differ from the model, first "
                     f"block {bad[0][0]} outputs {bad[0][1][:8]}")
    return sum(y.size for y in c["got"])


def check_exact(c, ci):
    _, _, _, _, m2, t2, l2 = c["spec"]
    want = f64_stage_b(ci["got"], 0, l2, m2, t2)
    assert len(want) == len(c["got"])
    for b, (y, r) in enumerate(zip(c["got"], want)):
        assert np.array_equal(r.astype(np.complex64).astype(np.complex128), r)  # exact stimuli
        assert y.shape == r.shape and np.array_equal(y, r.astype(np.complex64)), (c["cid"], b)


# ---------------------------------------------------------------------------
# designed taps at any centre, stage-A kinds 0, 1 and 2
# ---------------------------------------------------------------------------
DESIGNED = {  # fs, fmt, max_in, XLG_FORCE_GENERIC, stage-A kind
    "2M016_generic": (2016000, "cu8", 65536, True, 0), "2M016": (2016000, "cu8", 65536, False, 1),
    "2M048": (2048000, "cu8", 65536, False, 1), "10M": (10000000, "cs16", 65536, False, 1),
    "20M": (20000000, "cs8", 65536, False, 1), "61M44": (61440000, "cs16", 131072, False, 1),
    "long": (2016000, "cs16", 32768, False, 2)}


@pytest.mark.parametrize("case", list(DESIGNED))
def test_designed_taps_at_any_centre(pkg, case):
    """cascade_plan's 48 kHz client (for "long" a stage A at D1 = 400 and an even-D2 stage B) at five centres,
    300 ragged blocks with XLG_SLOTS tickets in flight: the kernel model of the twin's rows."""
    fs, fmt, max_in, generic, kind = DESIGNED[case]
    if case == "long":
        p = {"d1": 400, "taps1": pkg.create_low_pass_filter(1.0, fs, 1260, 504), "d2": 4, "interp2": 1,
             "taps2": pkg.create_low_pass_filter(1.0, fs // 400, 600, 240)}
    else:
        p = pkg.cascade_plan(fs, [48000])[0]
    specs = []
    for ce in CENTRES:
        specs += spec_pair(p["d1"], p["taps1"], ce, p["d2"], p["taps2"], p["interp2"])
    rng = np.random.default_rng(len(case))
    sizes = [int(v) * 2 for v in rng.integers(max_in // 8, max_in // 2 + 1, 300)]
    sizes[3], sizes[7] = 0, 2
    blocks = [rand_block(rng, fmt, n) for n in sizes]
    clients = run_group(pkg, fs, max_in, fmt, specs, blocks, flags=pkg.XLG_FORCE_GENERIC if generic else 0,
                        depth=SLOTS)
    n = 0
    for c, ci in pairs(clients):
        assert kind in c["kinds"] and c["kinds"] <= {0, kind}, c["kinds"]
        n += check_model(c, ci, fs)
    assert n > 1000


# ---------------------------------------------------------------------------
# every CTA size: exact taps against the float64 composition, random taps against the model
# ---------------------------------------------------------------------------
FS = 2016000
MAX_IN = 131072  # D1 = 1: up to 65536 stage-A samples per block
OUT_CAP = MAX_IN // 2 + 2


def n2_of(hist, L2, M2, T2, n):
    avail = hist + L2 * n - T2
    return avail // M2 + 1 if avail >= 0 else 0


def block_lengths(rng, L2, M2, T2, ko, n_fill=30):
    """Stage-A samples per block (D1 = 1 and a 3-tap stage A: a block of n samples gives n of them) for which
    stage B computes n2 = 0, 1, ko - 1, ko, ko + 1 and 2*ko + 1 outputs wherever the walk can hit them (one
    stage-A sample moves it by L2 upsampled samples), then n_fill random blocks that wrap the ring."""
    targets = [0, 1, max(ko - 1, 0), ko, ko + 1, 2 * ko + 1]
    hist, n1s = T2 - 1, []
    for t in targets:
        lo = 0 if t == 0 else max(0, (T2 - hist + (t - 1) * M2) // L2)
        n = min(next((n for n in range(lo, lo + M2 + 2) if n2_of(hist, L2, M2, T2, n) == t), lo), OUT_CAP - 2)
        n1s.append(n)
        hist += L2 * n - M2 * n2_of(hist, L2, M2, T2, n)
    return n1s + [int(v) for v in rng.integers(MAX_IN // 8, MAX_IN // 2 + 1, n_fill)], targets


def run_cta_case(pkg, L2, M2, T2, seed, flags=0, host_ring=0):
    """A twin, an exact client (1-bit taps) and a random-tap client at (L2, M2, T2) over block_lengths."""
    rng = np.random.default_rng(seed)
    ko = stage_b_ko(L2, M2, T2)
    t1 = small_taps(rng, 3, 1)
    t2e = small_taps(rng, T2, 1)
    assert exact_bound(t1, t2e, "cs16")
    t2r = (rng.standard_normal(T2) / np.sqrt(T2)).astype(np.float32)
    n1s, targets = block_lengths(rng, L2, M2, T2, ko)
    walk = stage_b_walk(n1s, L2, M2, T2)
    n2s = [n2 for _, n2 in walk]
    if L2 == 1:
        assert n2s[:6] == targets, (n2s[:6], targets)
    else:
        assert n2s[0] == 0 and max(n2s[:6]) > ko, n2s[:6]
    # windows across the ring's end besides the first; both parities of the window start, except that with
    # even D2 every start first + k*D2 keeps the parity of the first block's 1 - T2
    parities, wraps = ring_windows(walk, L2, M2, T2, ko, ring_cap(T2, L2, OUT_CAP))
    assert wraps >= 2 and parities == ({(T2 - 1) % 2} if L2 == 1 and M2 % 2 == 0 else {0, 1}), (parities, wraps)
    blocks = [exact_input(rng, "cs16", 2 * n) for n in n1s]
    specs = [("c", 1, t1, 0, M2, t2e, L2), ("c", 1, t1, 0, M2, t2r, L2), ("i", 1, t1, 0)]
    clients = run_group(pkg, FS, MAX_IN, "cs16", specs, blocks, flags=flags, host_ring=host_ring,
                        depth=12 if host_ring else SLOTS)
    ce, cr, ci = clients
    assert ce["kinds"] == cr["kinds"] == ci["kinds"]
    assert [y.size for y in ci["got"]] == n1s
    assert [y.size for y in ce["got"]] == n2s
    check_exact(ce, ci)
    check_model(cr, ci, FS)


INT_CASES = [(D2, T2) for cases in INT_KO_CASES.values() for D2, T2 in cases]
INT_CASES += [(3, 1), (4, 1), (9, 4), (10, 3), (2, 31), (2, 32), (2, 33), (3, 33), (1600, max_t2(1, 1600))]


@pytest.mark.parametrize("D2,T2", INT_CASES)
def test_integer_cta_sizes(pkg, D2, T2):
    """cascade_ko 256 ... 1 with odd and even D2 (INT_KO_CASES), T2 = 1, D2 > T2, T2 around 32 with even D2 (the
    lane skew wraps), and the longest stage B the shared memory admits."""
    run_cta_case(pkg, 1, D2, T2, D2 * 7 + T2)


@pytest.mark.parametrize("L2,M2,T2", RAT_CASES + [(3, 3001, max_t2(3, 3001))])
def test_rational_cta_sizes(pkg, L2, M2, T2):
    """cascade_poly_ko whole per branch, C_KO past L2 = 128, halved to a whole number per branch and to one
    that is not, Tb2 = 1, T2 % L2 != 0, and the longest stage B the shared memory admits."""
    run_cta_case(pkg, L2, M2, T2, L2 * 1000 + M2 + T2)


@pytest.mark.parametrize("mode", ["out_device", "host_ring"])
def test_cta_sizes_out_device_and_host_ring(pkg, mode):
    for L2, M2, T2 in [(1, 826, 33), (1, 2, 33), (3, 2000, 40)]:
        if mode == "out_device":
            run_cta_case(pkg, L2, M2, T2, 5, flags=pkg.XLG_OUT_DEVICE)
        else:
            run_cta_case(pkg, L2, M2, T2, 6, host_ring=16)


@pytest.mark.parametrize("L2,M2", [(1, 2), (1, 1600), (3, 3001), (441, 640)])
def test_one_tap_past_the_bound_is_refused(pkg, capfd, L2, M2):
    """-EINVAL, logged, no ticket taken: the next submit is ticket 0 and the group serves its other client."""
    T2 = max_t2(L2, M2) + 1
    g = pkg.Group(FS, MAX_IN)
    with pytest.raises(ValueError) as e:
        g.add_client_cascade(1, np.full(3, 0.25, np.float32), 0, M2, np.full(T2, 0.5, np.float32), interp2=L2)
    assert e.value.args[0] == -errno.EINVAL
    assert "<3>" in capfd.readouterr().err
    assert g.client_count() == 0
    cid = g.add_client_cascade(1, np.full(3, 0.25, np.float32), 0, M2, np.full(T2 - 1, 0.5, np.float32),
                               interp2=L2)
    t = g.submit("cs16", np.zeros(MAX_IN, np.int16))
    assert t == 0
    g.wait(t)
    assert g.client_count() == 1 and g.output(t, cid).size > 0
    g.close()


# ---------------------------------------------------------------------------
# clients of different CTA sizes in one group
# ---------------------------------------------------------------------------
def neighbour_taps(rng, T):
    return (rng.standard_normal(T) / np.sqrt(T)).astype(np.float32)


MIXED = {  # fs, fmt, max_in, rate; stage-B (D2, T2) of the small-ko neighbours, attached and removed mid-stream
    "61M44": (61440000, "cs16", 131072, 48000),
    "2M016_even": (2016000, "cu8", 65536, 48000),
}


@pytest.mark.parametrize("mode", ["default", "out_device", "host_ring"])
@pytest.mark.parametrize("case", list(MIXED))
def test_mixed_cta_sizes_in_one_group(pkg, case, mode):
    """cascade_plan's clients (ko 256; at 2.016 Msps one with an even D2 = 14 added) share a group with a ko = 16
    neighbour (D2 = 1024) and a ko = 4 neighbour (D2 = 5000), attached at block 40 and removed at block 110 with
    tickets in flight.  Every client equals the model at its own ko, and the plan clients equal the same
    clients in a group without the neighbours."""
    fs, fmt, max_in, rate = MIXED[case]
    plan = pkg.cascade_plan(fs, [rate] * 3)
    rng = np.random.default_rng(41)
    base = []
    for p in plan:
        base += spec_pair(p["d1"], p["taps1"], p["center"], p["d2"], p["taps2"], p["interp2"])
    if case == "2M016_even":
        p = plan[0]
        base += spec_pair(p["d1"], p["taps1"], 251001, 14, pkg.create_low_pass_filter(1.0, fs // p["d1"], 12000, 4800))
    assert any(s[0] == "c" and s[4] % 2 == 0 for s in base)
    # the neighbours' stage A has two taps fewer, so it never shares a tiled class with the plan clients'
    d1, t1n = plan[0]["d1"], plan[0]["taps1"][1:-1].copy()
    neigh = spec_pair(d1, t1n, -17, 1024, neighbour_taps(rng, 64))
    neigh += spec_pair(d1, t1n, 100003, 5000, neighbour_taps(rng, 64))
    assert [stage_b_ko(1, s[4], len(s[5])) for s in neigh[0::2]] == [16, 4]
    sizes = [max_in if b % 7 else max_in // 2 + 2 for b in range(160)]
    blocks = [rand_block(rng, fmt, n) for n in sizes]
    kw = {"out_device": {"flags": pkg.XLG_OUT_DEVICE, "depth": SLOTS}, "host_ring": {"host_ring": 16, "depth": 12},
          "default": {"depth": SLOTS}}[mode]
    nb = len(base)
    mixed = run_group(pkg, fs, max_in, fmt, base, blocks, attach={40: neigh},
                      detach={110: list(range(nb, nb + len(neigh)))}, **kw)
    alone = run_group(pkg, fs, max_in, fmt, base, blocks, **kw)
    failures = []
    for c, ci in pairs(mixed):
        bad = model_diff(c, ci, fs)
        if bad:
            failures.append(f"client {c['cid']} (D2 {c['spec'][4]}, ko {stage_b_ko(1, c['spec'][4], len(c['spec'][5]))})"
                            f" differs from the model in {len(bad)} blocks, first block {bad[0][0]} outputs "
                            f"{bad[0][1][:8]}")
    for ci, a in zip(mixed[1:nb:2], alone[1::2]):  # the stage-A rows do not depend on the neighbours
        assert all(np.array_equal(y, z) for y, z in zip(ci["got"], a["got"])), ci["cid"]
    for c, a in zip(mixed[:nb:2], alone[0::2]):
        for b, (y, z) in enumerate(zip(c["got"], a["got"])):
            if not np.array_equal(y, z):
                failures.append(f"client {c['cid']} (D2 {c['spec'][4]}) differs from the same client alone in block "
                                f"{b}: outputs {np.flatnonzero(y != z)[:8]}")
                break
    assert not failures, "\n".join(failures)
    assert [len(c["got"]) for c in mixed[nb:]] == [70] * len(neigh)
