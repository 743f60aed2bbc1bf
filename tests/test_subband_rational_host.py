"""Rational sub-band members on the CPU: the extended checker against the float64 composition, and
subband_plan's rules where no sub-band rate is a multiple of every client rate.  No GPU."""
import math

import numpy as np
import pytest

from cascade_rational import stuff
from exact import to_complex
from subband_rational import RationalSubbandOracle
from test_subband_host import f64_float_osc, response
from util import assert_cf32_close


def test_oracle_against_float64_composition(pkg):
    """RationalSubbandOracle = the float64 sub-band filter followed by each member's float64
    filter at interp2 * fs / d1 on its zero-stuffed outputs (both with the float oscillator), for members
    attached before block 0 and before block 3, to the 1e-5 contract; an interp2 = 1 member beside them."""
    fs, max_in, d1, c1 = 2048000, 8192, 10, -301000
    rng = np.random.default_rng(6)
    fs1 = fs // d1
    t1 = pkg.create_low_pass_filter(1.0, fs, fs1 // 2, fs1 // 2 - 40000)
    specs = {"a": (15, 64, pkg.create_low_pass_filter(15.0, 15 * fs1, 24000, 9600), 41000, 0),
             "b": (3, 8, pkg.create_low_pass_filter(3.0, 3 * fs1, 38400, 15360), -35000, 0),
             "c": (15, 64, pkg.create_low_pass_filter(15.0, 15 * fs1, 24000, 9600), 7000, 3),
             "d": (1, 4, pkg.create_low_pass_filter(1.0, fs1, 25600, 10240), 12000, 3)}
    blocks = [rng.integers(0, 256, n, dtype=np.uint8) for n in (max_in, 4002, 7, max_in, 1000, max_in, 2)]
    o = RationalSubbandOracle(d1, t1, c1, fs, max_in)
    got = {k: [] for k in specs}
    for b, x in enumerate(blocks):
        for k, (l2, d2, t2, off, first) in specs.items():
            if first == b:
                o.add_member(k, d2, t2, off, interp2=l2)
        for k, y in o.process_cf32("cu8", x).items():
            got[k].append(y)
    a = f64_float_osc(t1, d1, c1, fs, [to_complex("cu8", x) for x in blocks])
    for k, (l2, d2, t2, off, first) in specs.items():
        ref = f64_float_osc(t2, d2, off, l2 * fs1, [stuff(y, l2) for y in a[first:]])
        assert len(got[k]) == len(ref)
        assert sum(y.size for y in ref) > 20
        for b, (y, r) in enumerate(zip(got[k], ref)):
            assert y.shape == r.shape
            assert_cf32_close(y, r, f"{k} block {b}")


def band_clients(fs, seed, n=256):
    rng = np.random.default_rng(seed)
    return [(int(c), 48000) for c in rng.integers(-int(0.45 * fs), int(0.45 * fs), n)]


RATIONAL = {"2048k": 2048000, "10M": 10000000, "20M": 20000000}


def admissible(pkg, fs, rates):
    """Every D1 the rational rule may choose, with its members' (interp2, d2, taps2) by rate."""
    rmax = max(rates)
    for d1 in range(2, fs // (2 * rmax) + 1):
        fs1 = fs // d1
        if fs % d1 or fs1 % 2 or fs1 <= 2 * rmax:
            continue
        shapes = {}
        for r in set(rates):
            g = math.gcd(r, fs1)
            shapes[r] = (r // g, fs1 // g, pkg.create_low_pass_filter(float(r // g), r // g * fs1, r // 2, r // 5))
        if all(pkg.subband_member_fits(l2, m2, t.size) for l2, m2, t in shapes.values()):
            yield d1, shapes


@pytest.mark.parametrize("name", list(RATIONAL))
def test_rational_plan_rules(pkg, name):
    fs = RATIONAL[name]
    clients = band_clients(fs, 1)
    rates = [r for _, r in clients]
    p = pkg.subband_plan(fs, clients)
    d1, fs1, e, t1 = p["d1"], p["fs1"], p["e"], p["taps1"]
    assert fs % d1 == 0 and fs1 == fs // d1 and fs1 % 2 == 0 and fs1 > 2 * max(rates)
    assert fs1 % 48000 != 0  # no sub-band rate divides into these clients: every member resamples
    assert e == fs1 // 4 + max(rates) // 2
    assert len(p["members"]) == len(clients)
    used = set()
    for (c, r), m in zip(clients, p["members"]):
        g = math.gcd(r, fs1)
        assert (m["interp2"], m["d2"]) == (r // g, fs1 // g) and m["interp2"] > 1
        assert np.array_equal(m["taps2"], pkg.create_low_pass_filter(float(m["interp2"]), m["interp2"] * fs1,
                                                                     r // 2, r // 5))
        assert pkg.subband_member_fits(m["interp2"], m["d2"], m["taps2"].size)
        sb = p["subbands"][m["subband"]]
        used.add(m["subband"])
        assert m["center"] == c and m["rate"] == r and m["offset"] == c - sb["center"]
        assert abs(m["offset"]) <= fs1 // 4 and abs(m["offset"]) + r // 2 <= e
    assert used == set(range(len(p["subbands"])))
    # the first stage's passband and alias rules, as for integer members
    dc = response(t1, [0.0], fs)[0]
    assert np.min(response(t1, np.linspace(0, e, 64), fs)) >= 0.92 * dc
    assert np.array_equal(t1, pkg.create_low_pass_filter(1.0, fs, fs1 // 2, fs1 - 2 * e))
    assert np.max(response(t1, np.linspace(fs1 - e, fs / 2, 2048), fs)) <= 10 ** (-26 / 20) * dc
    # the cost model: 4 T1 / D1 per sub-band plus 4 ceil(T2 / L2) rate / fs per member
    want = 4.0 * len(p["subbands"]) * t1.size / d1 + sum(
        4.0 * -(-m["taps2"].size // m["interp2"]) * m["rate"] / fs for m in p["members"])
    assert p["fmas"] == pytest.approx(want, rel=1e-12)
    assert pkg.subband_fmas(fs, d1, t1.size, len(p["subbands"]),
                            [(m["rate"], m["taps2"].size, m["interp2"]) for m in p["members"]]) == \
        pytest.approx(want, rel=1e-12)


@pytest.mark.parametrize("name", list(RATIONAL))
def test_rational_plan_takes_the_cheapest_d1_that_fits(pkg, name):
    """The chosen D1 has the fewest FMAs among every D1 whose members all fit the kernel; a D1 that would be
    cheaper but holds a member the kernel refuses is never chosen."""
    fs = RATIONAL[name]
    clients = band_clients(fs, 2)
    rates = [r for _, r in clients]
    p = pkg.subband_plan(fs, clients)
    lo = min(c for c, _ in clients)
    fits = set()
    for d1, shapes in admissible(pkg, fs, rates):
        fits.add(d1)
        fs1 = fs // d1
        half = fs1 // 2
        n_used = len({min(range((max(c for c, _ in clients) - lo + half - 1) // half + 1),
                          key=lambda k: abs(c - (lo + k * half))) for c, _ in clients})
        e = fs1 // 4 + max(rates) // 2
        t1 = pkg.create_low_pass_filter(1.0, fs, fs1 // 2, fs1 - 2 * e).size
        cost = pkg.subband_fmas(fs, d1, t1, n_used, [(r, shapes[r][2].size, shapes[r][0]) for r in rates])
        assert p["fmas"] <= cost * (1 + 1e-12), (d1, cost, p["d1"], p["fmas"])
    assert p["d1"] in fits
    refused = [d1 for d1 in range(2, fs // 96000 + 1) if fs % d1 == 0 and (fs // d1) % 2 == 0
               and fs // d1 > 96000 and d1 not in fits]
    if fs >= 10000000:
        assert refused  # the bound rules some D1 out here (D1 = 8 at 10 Msps: 24/625)


def test_member_fit_bound(pkg):
    """subband_member_fits is subband_smem(M2, ceil(T2 / L2)) <= 200 KiB; 12/125 with 1505 taps fits (about
    80 KB), 24/625 does not, and interp2 = 1 is the integer member's bound."""
    def smem(l2, m2, t2):
        tb = -(-t2 // l2)
        return 16 + 16 * ((tb + 1) & ~1) * 8 + ((63 * m2 + tb + 2) & ~1) * 8
    for l2, m2, t2 in [(12, 125, 1505), (24, 625, 3011), (1, 40, 1400), (1, 7, 161), (15, 64, 771), (6, 125, 1505)]:
        assert pkg.subband_member_fits(l2, m2, t2) == (smem(l2, m2, t2) <= 200 * 1024)
    assert pkg.subband_member_fits(12, 125, 1505) and 78000 < smem(12, 125, 1505) < 82000
    assert not pkg.subband_member_fits(24, 625, 3011)
    assert not pkg.subband_member_fits(1, 40, 1400)


def old_rule_plan(pkg, fs, clients):
    """subband_plan as it was before rational members: only D1 where every rate divides fs1."""
    centers = [int(c) for c, _ in clients]
    rates = [int(r) for _, r in clients]
    rmax = max(rates)
    lo, hi = min(centers), max(centers)
    best = None
    for d1 in range(2, fs // (2 * rmax) + 1):
        if fs % d1:
            continue
        fs1 = fs // d1
        if fs1 % 2 or fs1 <= 2 * rmax or any(fs1 % r for r in rates):
            continue
        half = fs1 // 2
        n_cent = (hi - lo + half - 1) // half + 1
        assign = [min(range(n_cent), key=lambda k: abs(c - (lo + k * half))) for c in centers]
        used = sorted(set(assign))
        e = fs1 // 4 + rmax // 2
        t1 = pkg.create_low_pass_filter(1.0, fs, fs1 // 2, fs1 - 2 * e)
        designs = {r: pkg.create_low_pass_filter(1.0, fs1, r // 2, r // 5) for r in set(rates)}
        cost = 4.0 * len(used) * t1.size / d1 + sum(4.0 * designs[r].size * r / fs for r in rates)
        if best is None or cost < best[0]:
            best = (cost, d1, fs1, half, e, t1, designs, used, assign)
    cost, d1, fs1, half, e, t1, designs, used, assign = best
    index = {k: i for i, k in enumerate(used)}
    return {"d1": d1, "fs1": fs1, "taps1": t1, "e": e, "subbands": [{"center": lo + k * half} for k in used],
            "members": [{"subband": index[k], "center": c, "rate": r, "d2": fs1 // r, "offset": c - (lo + k * half),
                         "taps2": designs[r]} for c, r, k in zip(centers, rates, assign)], "fmas": cost}


EXISTING = {  # the integer sub-band workloads: fs, clients
    "61M": (61440000, lambda rng: [(int(c), 48000) for c in rng.integers(-30696000, 30696000, 256)]),
    "61M_4096": (61440000, lambda rng: [(int(c), 48000) for c in rng.integers(-30696000, 30696000, 4096)]),
    "2M": (2016000, lambda rng: [(int(c), 48000 if i % 2 else 96000)
                                 for i, c in enumerate(rng.integers(-960000, 960000, 64))]),
    "2M_close": (2016000, lambda rng: [(-400000 + 37000 * k, 48000) for k in range(10)]),
}


@pytest.mark.parametrize("name", list(EXISTING))
def test_integer_plans_unchanged(pkg, name):
    """Where some D1 serves every rate, the plan is the one the integer rule gives, with interp2 = 1."""
    fs, make = EXISTING[name]
    clients = make(np.random.default_rng(3))
    p, q = pkg.subband_plan(fs, clients), old_rule_plan(pkg, fs, clients)
    assert (p["d1"], p["fs1"], p["e"], p["subbands"], p["fmas"]) == (q["d1"], q["fs1"], q["e"], q["subbands"],
                                                                       q["fmas"])
    assert np.array_equal(p["taps1"], q["taps1"])
    for m, n in zip(p["members"], q["members"]):
        assert m.pop("interp2") == 1
        t, u = m.pop("taps2"), n.pop("taps2")
        assert m == n and np.array_equal(t, u)


def test_plan_refuses_rates_no_sub_band_serves(pkg):
    with pytest.raises(ValueError):
        pkg.subband_plan(2048000, [(0, 1000000)])
