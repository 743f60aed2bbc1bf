"""Rational L/M clients bit for bit at interpolations up to 441, at any centre and in randomised mixed groups.

Two stimuli make every output of every kernel exact (tests/rational.py):
* dyadic taps at centre 0 on the 8-bit grid: the float64 polyphase sum ref_rational_f64, which sees a wrong
  branch, a window one sample off or a dropped tap row;
* branch-one-hot taps (one nonzero per polyphase branch) at any centre fed a real cs16 stream: every
  accumulator is one rounded product, so the output equals the strict float32 oracle on the zero-stuffed
  stream, which sees the oscillator -- even/odd phase lookup, renormalisation, speculation with restore.

Every test asserts client_info's kind so that it proves which kernel ran: 1 the tiled integer kernel,
3 fir_poly_generic_cf32_kernel, 4 one tiled class per polyphase branch and poly_tile_place_cf32_kernel.
"""
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from exact import assert_exact, dyadic_taps, exact_input, grid_step, ref_f64
from oracle import pyoracle as po
from rational import RationalRef, branch_one_hot_taps, real_grid_input, ref_rational_f64, stuff

pytestmark = pytest.mark.gpu

TILED_INT, GENERIC, TILED = 1, 3, 4
POLY_GENERIC = {"XLATING_B200_POLY_TILE": "0"}
SMALL = [16384, 16384, 7001, 2, 0, 16384, 3, 16382, 16384, 16384]


class Client:
    """spec (L, M, T, centre): L = 0 is an integer client (add_client, decimation M); centre None gives
    dyadic taps at centre 0, a number branch-one-hot taps at that centre."""

    def __init__(self, g, rng, spec, fmt, first):
        self.L, self.M, self.T, self.center = spec
        self.Lr = max(self.L, 1)
        if self.center is None:
            self.taps = dyadic_taps(rng, self.T, fmt)
        else:
            self.taps = branch_one_hot_taps(rng, self.T, self.Lr)
        c = 0 if self.center is None else self.center
        self.cid = g.add_client(self.M, self.taps, c) if self.L == 0 else g.add_client_rational(self.L, self.M,
                                                                                                   self.taps, c)
        self.first, self.last = first, None
        self.got, self.kinds = [], {}  # kinds: block -> client_info kind

    def label(self):
        return f"client {self.cid} L={self.L} M={self.M} T={self.T} centre={self.center} from block {self.first}"


def outputs_per_block(spec, max_in):
    L, M, _, _ = spec
    return max(L, 1) * (max_in // 2) // M + 2


def run_group(pkg, monkeypatch, fs, max_in, plan, blocks, fmt="cs16", env=None, flags=0, host_ring=0, depth=1,
              churn=None, seed=0, reserve=0):
    """Feed `blocks` to a group holding `plan`'s clients and collect every output.  churn: {block: f(rng,
    live clients) -> (clients to detach, specs to attach)}, applied before that block's submit with up to
    depth - 1 earlier tickets still in flight.  reserve: output samples per block to size the result arenas
    for up front (a growth when clients join drops the results still in the ring, as xlg_reserve says)."""
    for k, v in (env or {}).items():
        monkeypatch.setenv(k, v)
    rng = np.random.default_rng(seed)
    g = pkg.Group(fs, max_in, flags=flags, host_ring=host_ring)
    if reserve:
        g.reserve(reserve)
    clients = [Client(g, rng, s, fmt, 0) for s in plan]
    pending = []

    def collect(b, t):
        g.wait(t)
        for c in clients:
            if c.first <= b and (c.last is None or b < c.last):
                y = g.read_output(t, c.cid) if flags & pkg.XLG_OUT_DEVICE else g.output(t, c.cid)
                c.got.append(np.array(y, copy=True))
                if c.last is None:
                    c.kinds[b] = g.client_info(c.cid)[1]

    for b, x in enumerate(blocks):
        if churn and b in churn:
            gone, specs = churn[b](rng, [c for c in clients if c.last is None])
            for c in gone:
                g.remove_client(c.cid)
                c.last = b
            clients += [Client(g, rng, s, fmt, b) for s in specs]
        pending.append((b, g.submit(fmt, x)))
        if len(pending) >= depth:
            collect(*pending.pop(0))
    while pending:
        collect(*pending.pop(0))
    g.close()
    return clients


def check(clients, blocks, fmt, fs, max_in, renorm=True, what=""):
    """Every output of every client: dyadic ones against the float64 sums, one-hot ones against the strict
    oracle on the stuffed stream (never given T < M: its history bookkeeping underflows there)."""
    def one(c):
        seen = blocks[c.first:c.last]
        if c.center is None:
            ref = ref_f64(c.taps, c.M, fmt, seen) if c.L == 0 else ref_rational_f64(c.taps, c.L, c.M, fmt, seen)
            step = grid_step(c.taps, fmt)
        else:
            assert c.T >= c.M
            o = po.OracleFilter(c.M, c.taps, c.center, c.Lr * fs, c.Lr * max_in)
            ref = [o.process_cf32("cs16", stuff(fmt, x, c.Lr), renorm=renorm) for x in seen]
            o.close()
            step = None
        try:
            assert_exact(c.got, ref, f"{what} {c.label()}", c.T, c.M, step)
        except AssertionError as e:
            return str(e)
        return None

    with ThreadPoolExecutor(max_workers=8) as ex:
        errors = [e for e in ex.map(one, clients) if e]
    assert not errors, f"{len(errors)} clients differ:\n" + "\n".join(errors[:4])


def kinds_of(clients, pick=lambda c: True):
    return {k for c in clients if pick(c) for k in c.kinds.values()}


# ---------------------------------------------------------------------------
# wide interpolations: one class of 8 clients per spec
# ---------------------------------------------------------------------------
WIDE = [  # (L, M, T), expected kind with the tiled rational path on
    ((16, 15, 97), TILED),         # L = 16, the drop-in span boundary
    ((17, 16, 200), TILED),        # L just above it
    ((36, 35, 300), TILED),        # exactly T_MAX_CLASSES = 36 branch classes
    ((37, 36, 300), GENERIC),      # one branch over the class budget
    ((6, 256, 400), GENERIC),      # gcd(L, M) = 2
    ((4, 2, 9), GENERIC),          # gcd(L, M) = 2 and L > M
    ((160, 147, 1000), GENERIC),   # 48 kHz from 44.1 kHz: L > M, L > 36
    ((147, 160, 1000), GENERIC),   # L > 36 with L < M
    ((441, 20480, 2000), GENERIC),  # 44.1 kHz from 2.048 Msps: T < M, every block fewer outputs than L
    ((17, 16, 5), TILED),          # T < L: most branches empty
]


@pytest.mark.parametrize("tile", [True, False], ids=["poly_tile", "poly_generic"])
@pytest.mark.parametrize("i", range(len(WIDE)), ids=["L{}_M{}_T{}".format(*s) for s, _ in WIDE])
def test_wide_interpolations(pkg, monkeypatch, i, tile):
    (L, M, T), want = WIDE[i]
    fmt = ("cu8", "cs8", "cs16")[i % 3]
    fs, max_in = 2048000, 16384
    rng = np.random.default_rng(100 + i)
    blocks = [exact_input(rng, fmt, n) for n in SMALL]
    cl = run_group(pkg, monkeypatch, fs, max_in, [(L, M, T, None)] * 8, blocks, fmt=fmt,
                   env=None if tile else POLY_GENERIC, seed=i)
    assert kinds_of(cl) == {want if tile else GENERIC}
    check(cl, blocks, fmt, fs, max_in, what=f"L={L} M={M} T={T} {fmt}")
    if L == 441:
        assert max(len(y) for y in cl[0].got) < L


def test_poly_class_budget(pkg, monkeypatch):
    """8 clients of 13/12 and 8 of 25/24 need 13 + 25 = 38 > 36 branch classes: the first bucket (L = 13)
    is tiled, L = 25 runs on the generic kernel -- until the L = 13 class leaves mid-stream (tickets in
    flight), after which L = 25 fits and is tiled."""
    fs, max_in, fmt = 2016000, 16384, "cu8"
    rng = np.random.default_rng(7)
    sizes = [16384, 16384, 7001, 16384, 2, 16384, 0, 16384, 16383, 16384, 16384, 16384, 16384]
    blocks = [exact_input(rng, fmt, n) for n in sizes]
    cut = 6
    churn = {cut: lambda r, live: ([c for c in live if c.L == 13], [])}
    cl = run_group(pkg, monkeypatch, fs, max_in, [(13, 12, 100, None)] * 8 + [(25, 24, 100, None)] * 8, blocks,
                   fmt=fmt, depth=pkg.XLG_SLOTS, churn=churn, seed=8)
    k13 = kinds_of(cl, lambda c: c.L == 13)
    before = {k for c in cl if c.L == 25 for b, k in c.kinds.items() if b < cut - pkg.XLG_SLOTS}
    after = {k for c in cl if c.L == 25 for b, k in c.kinds.items() if b >= cut}
    assert k13 == {TILED} and before == {GENERIC} and after == {TILED}, (k13, before, after)
    check(cl, blocks, fmt, fs, max_in, what="class budget")


# ---------------------------------------------------------------------------
# the rational phase harness: branch-one-hot taps, real cs16 stream, any centre
# ---------------------------------------------------------------------------
PHASE_SPECS = [((3, 128, 385), 8), ((7, 320, 431), 8), ((17, 16, 200), 8), ((6, 256, 401), 2), ((160, 147, 1000), 2)]


def swap_one(rng, live, fs):
    """One client leaves, one of the same (L, M, T) with new taps and centre joins."""
    c = live[int(rng.integers(0, len(live)))]
    return [c], [(c.L, c.M, c.T, int(rng.integers(-fs // 2 + 30000, fs // 2 - 30000)))]


def phase_harness(pkg, monkeypatch, n_blocks, env=None, flags=0, depth=1, seed=0):
    fs, max_in = 2048000, 16384
    rng = np.random.default_rng(seed)
    band = fs // 2 - 30000
    plan = [(L, M, T, int(rng.integers(-band, band))) for (L, M, T), n in PHASE_SPECS for _ in range(n)]
    sizes = [int(rng.choice([max_in, max_in, max_in - 2, int(rng.integers(0, max_in // 2)) * 2, 2]))
             for _ in range(n_blocks)]
    blocks = [real_grid_input(rng, n) for n in sizes]
    churn = {b: (lambda r, live: swap_one(r, live, fs)) for b in range(n_blocks) if b % 37 == 20}
    cl = run_group(pkg, monkeypatch, fs, max_in, plan, blocks, env=env, flags=flags, depth=depth, churn=churn,
                   seed=seed + 1, reserve=sum(outputs_per_block(s, max_in) for s in plan))
    check(cl, blocks, "cs16", fs, max_in, renorm=not flags & pkg.XLG_NO_RENORM, what=f"{env} flags={flags}")
    return kinds_of(cl)


PHASE_VARIANTS = {"no_renorm": ({}, "XLG_NO_RENORM", 1), "no_speculation": ({"XLATING_B200_SPECULATE": "0"}, 0, 1),
                  "partition": ({"XLATING_B200_PARTITION": "1"}, "XLG_SM_PARTITION", 1),
                  "poly_generic": (POLY_GENERIC, 0, 1), "in_flight": ({}, 0, "XLG_SLOTS")}


def test_rational_phase_harness(pkg, monkeypatch):
    assert phase_harness(pkg, monkeypatch, 300, seed=30) == {GENERIC, TILED}


@pytest.mark.parametrize("variant", list(PHASE_VARIANTS))
def test_rational_phase_harness_variants(pkg, monkeypatch, variant):
    env, flag, depth = PHASE_VARIANTS[variant]
    flags = getattr(pkg, flag) if flag else 0
    depth = getattr(pkg, depth) if isinstance(depth, str) else depth
    kinds = phase_harness(pkg, monkeypatch, 60, env=env, flags=flags, depth=depth, seed=31)
    assert kinds == ({GENERIC} if variant == "poly_generic" else {GENERIC, TILED})


# ---------------------------------------------------------------------------
# randomised mixed populations
# ---------------------------------------------------------------------------
RSPECS = [(3, 128, 97), (5, 4, 3), (2, 1, 9), (5, 3, 40), (7, 320, 431), (16, 15, 97), (17, 16, 200), (36, 35, 300),
          (37, 36, 300), (6, 256, 400), (4, 2, 9), (160, 147, 1000), (147, 160, 1000), (441, 20480, 2000),
          (17, 16, 5), (3, 128, 385)]
TILEABLE = [(3, 128, 97), (5, 3, 40), (7, 320, 431), (16, 15, 97), (17, 16, 200), (36, 35, 300), (17, 16, 5)]
ISPECS = [(42, 505), (21, 253), (8, 97), (5, 40), (1, 1)]
MIXED_VARIANTS = ["sm_partition", "no_renorm", "out_device", "host_ring"]


def mixed_plan(rng, fs):
    band = fs // 2 - 60000

    def centre(T, M, L):  # one-hot where the oracle may run (T >= M) and the stuffed stream stays short
        return int(rng.integers(-band, band)) if T >= M and L <= 17 and rng.integers(0, 2) else None

    plan = []
    D, T = ISPECS[int(rng.integers(0, 3))]
    plan += [(0, D, T, centre(T, D, 1)) for _ in range(8)]  # a tiled integer class
    for _ in range(int(rng.integers(2, 7))):
        D, T = ISPECS[int(rng.integers(0, len(ISPECS)))]
        plan.append((0, D, T, centre(T, D, 1)))
    L, M, T = TILEABLE[int(rng.integers(0, len(TILEABLE)))]
    plan += [(L, M, T, centre(T, M, L)) for _ in range(int(rng.integers(8, 13)))]  # a tiled rational class
    L, M, T = [(37, 36, 300), (6, 256, 400), (441, 20480, 2000)][int(rng.integers(0, 3))]
    plan.append((L, M, T, centre(T, M, L)))  # never tiled
    for _ in range(int(rng.integers(3, 9))):
        L, M, T = RSPECS[int(rng.integers(0, len(RSPECS)))]
        plan.append((L, M, T, centre(T, M, L)))
    return plan


@pytest.mark.parametrize("seed", range(12))
def test_random_mixed_populations(pkg, monkeypatch, seed):
    rng = np.random.default_rng(1000 + seed)
    fs = int(rng.choice([2016000, 2048000, 2400000]))
    max_in = int(rng.choice([16384, 32768, 65536]))
    plan = mixed_plan(rng, fs)
    assert all(max(L, 1) * fs <= 0xFFFFFFFF and max(L, 1) * max_in // 2 < 2 ** 31 for L, _, _, _ in plan)
    choices = [max_in, max_in, max_in - 2, 0, 2, 7, int(rng.integers(1, max_in // 2)) * 2 + 1]
    sizes = [int(rng.choice(choices)) for _ in range(14)]
    blocks = [real_grid_input(rng, n) for n in sizes]
    b1, b2 = sorted(rng.choice(np.arange(2, 13), 2, replace=False).tolist())

    def churn(r, live):
        gone = [live[i] for i in r.choice(len(live), int(r.integers(1, 4)), replace=False)]
        new = mixed_plan(r, fs)
        return gone, [new[i] for i in r.choice(len(new), int(r.integers(1, 10)), replace=False)]

    depth = int(rng.integers(1, pkg.XLG_SLOTS + 1))
    variant = MIXED_VARIANTS[seed % len(MIXED_VARIANTS)]
    flags, env, host_ring = 0, None, 0
    if variant == "sm_partition":
        flags, env = pkg.XLG_SM_PARTITION, {"XLATING_B200_PARTITION": "1"}
    elif variant == "no_renorm":
        flags = pkg.XLG_NO_RENORM
    elif variant == "out_device":
        flags = pkg.XLG_OUT_DEVICE
    else:
        host_ring = 12
    worst = max(outputs_per_block((L, M, T, None), max_in) for L, M, T in RSPECS)
    reserve = sum(outputs_per_block(s, max_in) for s in plan) + 2 * 9 * worst  # two churns of up to 9 joins
    cl = run_group(pkg, monkeypatch, fs, max_in, plan, blocks, env=env, flags=flags, host_ring=host_ring,
                   depth=depth, churn={b1: churn, b2: churn}, seed=seed, reserve=reserve)
    check(cl, blocks, "cs16", fs, max_in, renorm=not flags & pkg.XLG_NO_RENORM,
          what=f"seed {seed} fs={fs} max_in={max_in} depth={depth} {variant}")
    # every plan holds a tiled integer class, a tiled rational class and a rational client that is never tiled
    assert {TILED_INT, GENERIC, TILED} <= kinds_of(cl, lambda c: c.first == 0), kinds_of(cl)


# ---------------------------------------------------------------------------
# upsampled positions past 2^32
# ---------------------------------------------------------------------------
def test_upsampled_position_past_2_32(pkg):
    """310 full cu8 blocks into a 441/20480 client: about 4.5e9 upsampled samples, past 2^32.  Reading the
    code shows these positions held in 64 bits everywhere; this guards against a regression to 32 bits,
    not a known bug.  The batch client (kind 3) and a drop-in XlatingFilter.rational, block by block."""
    fs, max_in, fmt = 2048000, 65536, "cu8"
    L, M, T = 441, 20480, 2000
    rng = np.random.default_rng(44)
    taps, dtaps = dyadic_taps(rng, T, fmt), dyadic_taps(rng, T, fmt)
    g = pkg.Group(fs, max_in)
    cid = g.add_client_rational(L, M, taps, 0)
    f = pkg.XlatingFilter.rational(L, M, dtaps, 0, fs, max_in)
    ref, dref = RationalRef(taps, L, M), RationalRef(dtaps, L, M)
    n_blocks = 310
    assert n_blocks * (max_in // 2) * L > 2 ** 32
    step = grid_step(taps, fmt)
    kinds = set()
    try:
        for b in range(n_blocks):
            x = exact_input(rng, fmt, max_in)
            t = g.submit(fmt, x)
            y = f.process_cf32(fmt, x)
            g.wait(t)
            kinds.add(g.client_info(cid)[1])
            assert_exact(g.output(t, cid), ref.feed(fmt, x), f"group block {b}", T, M, step)
            assert_exact(y, dref.feed(fmt, x), f"drop-in block {b}", T, M, grid_step(dtaps, fmt))
    finally:
        f.close()
        g.close()
    assert kinds == {GENERIC} and ref.n * L > 2 ** 32 and ref.k > 0
