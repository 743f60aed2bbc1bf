"""Sub-band clients on the CPU: the checker against the float64 composition, and subband_plan's design rules.
No GPU."""
import numpy as np
import pytest

from cascade import f64_filter, filter_constants
from exact import oracle_phases, to_complex
from subband import SubbandOracle
from util import assert_cf32_close


def f64_float_osc(taps, D, center, fs, blocks):
    """f64_filter with the reference's float32 oscillator in place of the exact one: exact math drifts from
    the float recursion by about 1e-7 rad per output, more than the contract over a few hundred outputs."""
    out = f64_filter(taps, D, center, fs, blocks)
    counts = [y.size for y in out]
    _, (ir, ii) = filter_constants(taps, D, center, fs)
    k = np.arange(sum(counts))
    fix = oracle_phases(complex(ir, ii), counts) / np.exp(-1j * 2 * np.pi * center / fs * D * k)
    return np.split(np.concatenate(out) * fix, np.cumsum(counts)[:-1])


def test_oracle_against_float64_composition(pkg):
    """SubbandOracle = the float64 sub-band filter followed by each member's float64 filter at fs / d1 on its
    outputs (both with the float oscillator), for members attached before block 0 and before block 3, to the
    1e-5 contract."""
    fs, max_in, d1, c1 = 2016000, 8192, 7, -301000
    rng = np.random.default_rng(5)
    t1 = pkg.create_low_pass_filter(1.0, fs, 144000, 120000)
    fs1 = fs // d1
    specs = {"a": (6, pkg.create_low_pass_filter(1.0, fs1, 24000, 9600), 41000, 0),
             "b": (3, pkg.create_low_pass_filter(1.0, fs1, 48000, 19200), -55000, 0),
             "c": (6, pkg.create_low_pass_filter(1.0, fs1, 24000, 9600), 7000, 3)}
    blocks = [rng.integers(0, 256, n, dtype=np.uint8) for n in (max_in, 4002, 7, max_in, 1000, max_in)]
    o = SubbandOracle(d1, t1, c1, fs, max_in)
    got = {k: [] for k in specs}
    for b, x in enumerate(blocks):
        for k, (d2, t2, off, first) in specs.items():
            if first == b:
                o.add_member(k, d2, t2, off)
        for k, y in o.process_cf32("cu8", x).items():
            got[k].append(y)
    a = f64_float_osc(t1, d1, c1, fs, [to_complex("cu8", x) for x in blocks])
    for k, (d2, t2, off, first) in specs.items():
        ref = f64_float_osc(t2, d2, off, fs1, a[first:])
        assert len(got[k]) == len(ref)
        for b, (y, r) in enumerate(zip(got[k], ref)):
            assert_cf32_close(y, r, f"{k} block {b}")


WORKLOADS = {  # fs, clients as (centre, rate), seeded
    "61M": (61440000, lambda rng: [(int(c), 48000) for c in rng.integers(-30696000, 30696000, 256)]),
    "2M": (2016000, lambda rng: [(int(c), 48000 if i % 2 else 96000)
                                 for i, c in enumerate(rng.integers(-960000, 960000, 64))]),
}


def response(taps, f, fs):
    n = np.arange(taps.size)
    return np.abs(np.exp(-2j * np.pi * np.outer(f, n) / fs) @ taps.astype(np.float64))


@pytest.mark.parametrize("name", list(WORKLOADS))
def test_plan_passes_every_member_and_stops_its_aliases(pkg, name):
    fs, make = WORKLOADS[name]
    clients = make(np.random.default_rng(1))
    p = pkg.subband_plan(fs, clients)
    d1, fs1, e, t1 = p["d1"], p["fs1"], p["e"], p["taps1"]
    assert fs % d1 == 0 and fs1 == fs // d1 and fs1 > 2 * max(r for _, r in clients)
    assert e == fs1 // 4 + max(r for _, r in clients) // 2
    assert len(p["members"]) == len(clients)
    used = set()
    for (c, r), m in zip(clients, p["members"]):
        sb = p["subbands"][m["subband"]]
        used.add(m["subband"])
        assert m["center"] == c and m["rate"] == r and m["d2"] * r == fs1
        assert m["offset"] == c - sb["center"]
        assert abs(m["offset"]) <= fs1 // 4  # the nearest centre of a grid fs1 / 2 apart
        assert abs(m["offset"]) + r // 2 <= e  # inside the sub-band's passband
    assert used == set(range(len(p["subbands"])))  # only sub-bands with members
    # the design: passband edge e, stopband from fs1 - e on (cutoff fs1 / 2, transition fs1 - 2e)
    # (the planner's Hamming-windowed designs are up to about 0.7 dB down at their passband edge)
    dc = response(t1, [0.0], fs)[0]
    assert np.min(response(t1, np.linspace(0, e, 64), fs)) >= 0.92 * dc
    assert np.array_equal(t1, pkg.create_low_pass_filter(1.0, fs, fs1 // 2, fs1 - 2 * e))
    assert fs1 // 2 + (fs1 - 2 * e) // 2 >= fs1 - e  # the nominal stopband edge, cutoff + transition / 2
    # (the window's estimate of the transition is short: at the nominal edge the design is about 28 dB down,
    # 40 dB a little further on)
    assert np.max(response(t1, np.linspace(fs1 - e, fs / 2, 2048), fs)) <= 10 ** (-26 / 20) * dc


@pytest.mark.parametrize("name", list(WORKLOADS))
def test_plan_takes_the_cheapest_d1(pkg, name):
    """subband_fmas is 4 T1 / D1 per sub-band with members plus 4 T2 rate / fs per member, and the chosen D1
    has the fewest among every admissible D1."""
    fs, make = WORKLOADS[name]
    clients = make(np.random.default_rng(2))
    p = pkg.subband_plan(fs, clients)
    rmax = max(r for _, r in clients)
    n_sb = len(p["subbands"])
    want = 4.0 * n_sb * p["taps1"].size / p["d1"] + sum(4.0 * m["taps2"].size * m["rate"] / fs for m in p["members"])
    assert p["fmas"] == pytest.approx(want, rel=1e-12)
    assert pkg.subband_fmas(fs, p["d1"], p["taps1"].size, n_sb,
                            [(m["rate"], m["taps2"].size) for m in p["members"]]) == pytest.approx(want, rel=1e-12)
    lo = min(c for c, _ in clients)
    for d1 in range(2, fs // (2 * rmax) + 1):
        fs1 = fs // d1
        if fs % d1 or fs1 % 2 or fs1 <= 2 * rmax or any(fs1 % r for _, r in clients):
            continue
        half = fs1 // 2
        n_used = len({int(np.floor((c - lo) / half + 0.5)) if (c - lo) % half != half // 2 else (c - lo) // half
                      for c, _ in clients})
        e = fs1 // 4 + rmax // 2
        t1 = pkg.create_low_pass_filter(1.0, fs, fs1 // 2, fs1 - 2 * e).size
        t2 = {r: pkg.create_low_pass_filter(1.0, fs1, r // 2, r // 5).size for _, r in clients}
        cost = pkg.subband_fmas(fs, d1, t1, n_used, [(r, t2[r]) for _, r in clients])
        assert p["fmas"] <= cost * (1 + 1e-12), (d1, cost, p["d1"], p["fmas"])


def test_plan_refuses_rates_no_sub_band_serves(pkg):
    with pytest.raises(ValueError):
        pkg.subband_plan(2016000, [(0, 1000000)])
