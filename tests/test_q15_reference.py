"""The Q15 model (tests/q15.py) against the strict oracle and, where oracle/_ref is built, the compiled
reference, on the stimuli where integer code goes wrong: the product pair that wraps in 32 bits, both
saturation rails at the filter and at the rotation, taps whose (int16_t)(x * 32768) conversion wraps, a window
whose acc >> 15 passes 2^31, and the oscillator in its limit cycle at nonzero centres.  Each rule of the
model is needed: dropping it makes some stimulus disagree with the oracle.  No GPU."""
import numpy as np
import pytest

import q15
from exact import assert_exact
from oracle import pyoracle as po

FS = q15.FS
MAX_IN = 2 * 70000


def blocks_of(x, sizes):
    """x (raw elements) cut into calls of `sizes` complex samples."""
    cuts = np.cumsum([2 * s for s in sizes])
    assert cuts[-1] == x.size
    return np.split(x, cuts[:-1])


def stimuli():
    """name -> (taps, D, centre, fmt, blocks)."""
    rng = np.random.default_rng(31)
    out = {}
    for fmt in ("cu8", "cs8", "cs16"):
        lo = q15.FULL[fmt][1]
        first = np.full(16, lo, dtype=q15.FULL[fmt][0])  # the wrap case on every full window
        sizes = [9, 1, 0, 4000, 3, 2048]
        out[f"wrap_{fmt}"] = (q15.WRAP_TAPS, 1, q15.WRAP_CENTER, fmt,
                              [first] + blocks_of(q15.wrap_input(rng, fmt, sum(sizes)), sizes))
        # gain > 1: sums of eight taps of magnitude near 0.9 on full-scale samples reach both rails, and at
        # centre fs / 8 the rotation by a phase near 45 degrees takes them past the rails again
        taps = (rng.uniform(0.6, 0.95, 8) * rng.choice([-1, 1], 8)).astype(np.float32)
        sizes = [5000, 7, 1, 3001]
        out[f"rails_{fmt}"] = (taps, 3, FS // 8, fmt, blocks_of(q15.rail_input(rng, fmt, sum(sizes)), sizes))
    for center in (0, 300000):
        sizes = [3000, 11, 2000]
        x = np.concatenate([q15.rail_input(rng, "cs16", 1000), q15.wrap_input(rng, "cs16", sum(sizes) - 1000)])
        out[f"edge_taps_{center}"] = (q15.EDGE_TAPS, 2, center, "cs16", blocks_of(x, sizes))
    # acc >> 15 past 2^31: 65537 taps with one Q15 part at -32768 each and a window that meets each of them
    T, D, center = 65537, 4096, 300000
    taps = q15.narrowing_taps(T, center, FS)
    rev = po.OracleFilter(D, taps, center, FS, MAX_IN).q15_consts[0].astype(np.int64)
    out["narrowing"] = (taps, D, center, "cs16", q15.narrowing_blocks(rng, rev))
    # the oscillator into its limit cycle (mu up to 111550 outputs at D = 1)
    for center in q15.LIMIT_CENTERS:
        taps = (rng.uniform(-0.7, 0.7, 5)).astype(np.float32)
        sizes = [32768, 32768, 1, 32767, 40000, 3]
        out[f"cycle_{center}"] = (taps, 1, center, "cs16", blocks_of(q15.wrap_input(rng, "cs16", sum(sizes)),
                                                                     sizes))
    return out


STIMULI = stimuli()


def oracle_outputs(spec, flavor=None):
    taps, D, center, fmt, blocks = spec
    if flavor is None:
        o = po.OracleFilter(D, taps, center, FS, MAX_IN)
        return [o.process_q15(fmt, b) for b in blocks]
    r = po.RefFilter(D, taps, center, FS, MAX_IN, flavor=flavor)
    return [r.process_q15(fmt, b) for b in blocks]


def model_outputs(spec, arith=q15.REF):
    taps, D, center, fmt, blocks = spec
    rev, qinc = po.OracleFilter(D, taps, center, FS, MAX_IN).q15_consts
    return q15.model(rev, qinc, D, fmt, blocks, arith=arith)


_ORACLE = {}


def oracle_cached(name):
    if name not in _ORACLE:
        _ORACLE[name] = oracle_outputs(STIMULI[name])
    return _ORACLE[name]


@pytest.mark.parametrize("name", sorted(STIMULI))
def test_model_equals_oracle(name):
    spec = STIMULI[name]
    want = oracle_cached(name)
    assert_exact(model_outputs(spec), want, f"{name}: model", len(spec[0]), spec[1])
    if po.ref_available("strict"):
        assert_exact(oracle_outputs(spec, "strict"), want, f"{name}: libref_strict", len(spec[0]), spec[1])


def test_stimuli_reach_their_edges(pkg):
    """Each stimulus does what it is named for."""
    lib = pkg.lib()
    # the wrap case: output 1 of 16 zero bytes is (23168, 23169); with the pair widened it flips sign
    for fmt in ("cu8", "cs8", "cs16"):
        spec = STIMULI[f"wrap_{fmt}"]
        assert tuple(oracle_cached(f"wrap_{fmt}")[0][1]) == (23168, 23169)
        wide = model_outputs(spec, q15.MUTATIONS["pair widened to int64"])
        assert tuple(wide[0][1]) == (-23168, -23169)
        y = np.concatenate(oracle_cached(f"wrap_{fmt}")[1:])
        n_diff = int(np.sum(np.any(np.concatenate(wide[1:]) != y, axis=1)))
        assert 0 < n_diff < len(y) // 2, (fmt, n_diff, len(y))  # only some outputs meet it in random data
    rev, _, _ = q15.host_consts(lib, q15.WRAP_TAPS, 1, q15.WRAP_CENTER, FS)
    assert rev[1].tolist() == [-32768, -32768]
    # both rails, at the filter and at the rotation
    for fmt in ("cu8", "cs8", "cs16"):
        y = np.concatenate(oracle_cached(f"rails_{fmt}"))
        for v in (-32768, 32767):
            assert np.sum(y == v) > 100, (fmt, v)
    # acc >> 15 past 2^31 at the designed windows
    taps, D, center, fmt, blocks = STIMULI["narrowing"]
    rev, _, _ = q15.host_consts(lib, taps, D, center, FS)
    assert np.all((rev == -32768).any(axis=1))
    diff = [np.any(a != b, axis=1) for a, b in
            zip(model_outputs(STIMULI["narrowing"], q15.MUTATIONS["(int32) narrowing dropped"]),
                oracle_cached("narrowing"))]
    assert diff[0][16] and diff[3].any()
    # limit cycles of nonzero magnitude (the issue's table, at D = 1)
    want = {-768000: 5537, 640000: 3913, 682666: 10894, 300000: 659, 12345: 174, -512000: 0}
    for center, mag in want.items():
        _, qinc, _ = q15.host_consts(lib, np.ones(3, np.float32), 1, center, FS)
        osc = q15.Osc(qinc)
        mu, lam = osc.cycle()
        assert round(osc.magnitude_after(2 ** 32)) == mag, center
        assert mu < 120000 and lam < 1000, (center, mu, lam)


EDGE_SETS = {"edge": q15.EDGE_TAPS, "wrap": q15.WRAP_TAPS, "narrowing": q15.narrowing_taps(101, 300000, FS),
             "designed": po.lpf_design(1.0, FS, 24000, 16400)}


@pytest.mark.parametrize("center", [0, 300000, -768000, q15.WRAP_CENTER + 1, 12345])
@pytest.mark.parametrize("which", sorted(EDGE_SETS))
def test_host_q15_constants_equal_oracle(pkg, which, center):
    """csrc/taps_host.c's Q15 taps and increment == the oracle's == (int16_t)(x * 32768) as gcc converts
    (through int32, keeping the low 16 bits: 1.0 -> -32768, 1.5 -> -16384, -3 -> -32768)."""
    taps = EDGE_SETS[which]
    D = 4
    rev, qinc, cf = q15.host_consts(pkg.lib(), taps, D, center, FS)
    o = po.OracleFilter(D, taps, center, FS, 64)
    orev, oqinc = o.q15_consts
    np.testing.assert_array_equal(rev, orev)
    assert qinc == oqinc
    np.testing.assert_array_equal(rev, q15.q15_of(cf.view(np.float32)).reshape(-1, 2))
    if center == 0 and which == "edge":
        assert rev[::-1, 0].tolist() == [-32768, -32768, 32767, -32768, -16384, -32768, 1, -1, 16384]


@pytest.mark.parametrize("mutation", [m for m in q15.MUTATIONS if m != "sat16 dropped at the oscillator"])
def test_model_mutation_is_caught(mutation):
    """Each rule of the model is needed: with it changed, some stimulus disagrees with the oracle."""
    caught = []
    for name, spec in STIMULI.items():
        got = model_outputs(spec, q15.MUTATIONS[mutation])
        if any(g.shape != w.shape or np.any(g != w) for g, w in zip(got, oracle_cached(name))):
            caught.append(name)
    print(f"\n{mutation}: caught by {caught}")
    assert caught, mutation


def test_oscillator_saturation_never_fires(pkg):
    """The oscillator's sat16 is the one rule no stimulus can reach: |incr| <= 32767, so from 32767 + 0i
    |phase * incr| >> 15 stays inside int16, and floor rounding never carries the walk past 32767 (checked on
    every limit-cycle centre at D = 1, 8 and 1280, and on 20000 random increments for 20000 steps)."""
    lib = pkg.lib()
    incs = []
    for center in q15.LIMIT_CENTERS + (q15.WRAP_CENTER, 256000, 1):
        for D in (1, 8, 1280):
            incs.append(q15.host_consts(lib, np.ones(3, np.float32), D, center, FS)[1])
    for qinc in incs:
        a, b = q15.Osc(qinc), q15.Osc(qinc, q15.MUTATIONS["sat16 dropped at the oscillator"])
        mu, lam = a.cycle()
        np.testing.assert_array_equal(a.phases(0, mu + lam), b.phases(0, mu + lam))
    rng = np.random.default_rng(5)
    ang = rng.uniform(-np.pi, np.pi, 20000)
    ir = np.trunc(np.cos(ang).astype(np.float32) * np.float32(32767)).astype(np.int64)
    ii = np.trunc(np.sin(ang).astype(np.float32) * np.float32(32767)).astype(np.int64)
    pr, pi = np.full(ang.size, 32767, np.int64), np.zeros(ang.size, np.int64)
    for _ in range(20000):
        pr, pi = (pr * ir - pi * ii) >> 15, (pr * ii + pi * ir) >> 15
        assert pr.min() >= -32768 and pr.max() <= 32767 and pi.min() >= -32768 and pi.max() <= 32767


def test_window_reference_with_walked_phase(pkg):
    """The long-run window reference: the outputs of a filter attached m * D samples before a block equal the
    data part of a fresh filter fed from that block, rotated by the walked phases from output m."""
    rng = np.random.default_rng(9)
    D, center = 7, -768000
    taps = rng.uniform(-0.9, 0.9, 31).astype(np.float32)
    c = q15.Client(pkg.lib(), taps, D, center, FS)
    sizes = [7000] * 30 + [7 * 11, 5]
    blocks = blocks_of(q15.wrap_input(rng, "cs16", sum(sizes)), sizes)
    o = po.OracleFilter(D, taps, center, FS, MAX_IN)
    full = [o.process_q15("cs16", b) for b in blocks]
    b0 = 25  # 25 * 7000 samples = 25000 periods of D
    got = c("cs16", blocks[b0 - 1:], k0=(b0 - 1) * 7000 // D)[1:]
    assert_exact(got, full[b0:], "window reference")
    assert np.any(np.concatenate(full[b0:]))
