"""Client state across hand-overs in the batch ABI, bit for bit at any centre.

The per-filter drop-in engine moves a filter between its private path and its band's group with
XLG_TRACK_STATE: xlg_copy_output(..., state_after) gives the state after a ticket and
xlg_add_client_ex / xlg_add_client_rational_ex continue it in another group.  These tests check that
state against the strict oracle: the history offset to the sample and the oscillator to the bit.

Two kinds of client share each stream (real cs16 on the exact grid, tests/rational.py real_grid_input):
one-hot (integer) and branch-one-hot (rational) taps at centres drawn across the band, where every
accumulator is one rounded product, so the output equals the strict oracle bit for bit with the
oscillator included; and dyadic taps at centre 0, where every partial sum is exact, so every history
sample, and every sample that must read as zero, is checked.
"""
import errno

import numpy as np
import pytest

from exact import assert_exact, dyadic_taps, one_hot_taps
from oracle import pyoracle as po
from rational import branch_one_hot_taps, oracle_filter, real_grid_input, stuff

pytestmark = pytest.mark.gpu
FS, FS5, MAX_IN = 2016000, 61440000, 16384
GENERIC, TILED, LONG, POLY, POLY_TILED = 0, 1, 2, 3, 4


class Client:
    """One client and its strict oracle, which is fed every block the client consumed."""

    def __init__(self, rng, fs, L, M, T, dyadic=False, j=None, renorm=True):
        assert T >= M  # the oracle's history bookkeeping underflows with fewer taps
        self.L, self.M, self.T, self.renorm = L, M, T, renorm
        if dyadic:
            self.taps, self.center = dyadic_taps(rng, T, "cs16"), 0
        else:
            if L == 1:
                j = int(rng.integers(0, T)) if j is None else j
                self.taps = one_hot_taps(T, j, float(rng.choice([0.75, -0.5, 0.3125])))
            else:
                self.taps = branch_one_hot_taps(rng, T, L)
            band = fs // 2 - fs * L // (2 * M) - 1000
            self.center = int(rng.integers(-band, band))
        self.oracle = oracle_filter(po, L, M, self.taps, self.center, fs, MAX_IN)
        self.label = f"L={L} M={M} T={T} centre={self.center}{' dyadic' if dyadic else ''}"
        self.got, self.want, self.kinds = [], [], set()

    def attach(self, g, state=None):
        return g.add_client_rational(self.L, self.M, self.taps, self.center, state=state)

    def feed(self, x):
        self.want.append(self.oracle.process_cf32("cs16", stuff("cs16", x, self.L), renorm=self.renorm))
        return self.want[-1]

    def check_state(self, st, what):
        """hist (upsampled samples for a rational client) and the oscillator's float32 bits equal the oracle's."""
        assert st.hist == self.oracle.history, f"{what}: hist {st.hist} != {self.oracle.history}"
        got = np.array([st.phase_re, st.phase_im], np.float32).view(np.uint32)
        ph = self.oracle.phase
        want = np.array([ph.real, ph.imag], np.float32).view(np.uint32)
        assert np.array_equal(got, want), f"{what}: phase {st.phase_re} {st.phase_im} != {ph}"


# ---------------------------------------------------------------------------
# (a) state_after of every ticket, read up to 15 tickets late
# ---------------------------------------------------------------------------
# lengths that repeat (the speculative pre-pass guesses right) and change (it guesses wrong), empty and
# 2-element calls (samples without outputs), odd lengths.  The group does not report its speculation hits
# and misses: that both happen follows from these lengths, it is not asserted.
SIZES = ([MAX_IN] * 5 + [12346] * 4 + [2, 0, 2] + [MAX_IN] * 3 + [7, 7001, 7001, 7001, MAX_IN, 0]
         + [MAX_IN - 2] * 3 + [MAX_IN] * 6 + [3, MAX_IN, 9999, MAX_IN])
# (L, M, T): a tiled class, a generic class with even T, a polyphase tiled class (kind 4), polyphase generic
BAND_A = [(1, 21, 253)] * 8 + [(1, 42, 200)] * 2 + [(1, 8, 64)] + [(3, 128, 385)] * 8 + [(7, 320, 431)] * 2
BAND_B = [(1, 1280, 1407)] * 9  # split-K at 61.44 Msps
CHURN = {17: (9, (1, 21, 253)), 26: (18, (3, 128, 385))}  # block: (index of the client to remove, spec to add)


def run_state_after(pkg, fs, plan, rng, flags, churn=None, q15_tail=False):
    renorm = not (flags & pkg.XLG_NO_RENORM)
    g = pkg.Group(fs, MAX_IN, flags=pkg.XLG_TRACK_STATE | flags, host_ring=16)
    live, clients = [], []  # [cid, Client] attached now; every client

    def add(spec):
        L, M, T = spec
        c = Client(rng, fs, L, M, T, j=(0, T - 1, None)[len(clients) % 3], renorm=renorm)
        live.append([c.attach(g), c])
        clients.append(c)

    for spec in plan:
        add(spec)
    pending, late = [], 0

    def collect():
        nonlocal late
        t, b, x, members = pending.pop(0)
        late = max(late, len(pending))
        g.wait(t)
        for cid, c in members:
            y, st = g.copy_output(t, cid)
            what = f"flags={flags:#x} block {b} client {cid} {c.label}"
            assert_exact(y, c.feed(x), what, c.T, c.M)
            c.check_state(st, what)
            c.kinds.add(g.client_info(cid)[1])

    for b, n in enumerate(SIZES):
        if churn and b in churn:
            while pending:
                collect()
            i, spec = churn[b]
            g.remove_client(live.pop(i)[0])
            add(spec)
        x = real_grid_input(rng, n)
        pending.append((g.submit("cs16", x), b, x, list(live)))
        if len(pending) == 16:  # ticket t is read after t + 15 was submitted
            collect()
    while pending:
        collect()
    assert late == 15
    if q15_tail:
        t = g.submit("cs16", real_grid_input(rng, MAX_IN), flags=pkg.XLG_PATH_Q15)
        g.wait(t)
        with pytest.raises(ValueError, match=str(-errno.EINVAL)):
            g.copy_output(t, live[0][0])
    g.close()
    return set().union(*(c.kinds for c in clients))


@pytest.mark.parametrize("env,flag", [({}, None), ({"XLATING_B200_SPECULATE": "0"}, None), ({}, "XLG_NO_RENORM")],
                         ids=["default", "no_speculation", "no_renorm"])
def test_state_after_every_ticket(pkg, monkeypatch, env, flag):
    """Every client's state after every ticket equals the oracle's after the same blocks, on every kernel,
    over block lengths that repeat and change (so that speculation should both hit and miss; see SIZES),
    churn, and host-ring entries read 15 tickets late; a Q15 ticket carries no cf32 state (-EINVAL)."""
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    flags = getattr(pkg, flag) if flag else 0
    rng = np.random.default_rng(31)
    kinds = run_state_after(pkg, FS, BAND_A, rng, flags, churn=CHURN)
    assert {GENERIC, TILED, POLY, POLY_TILED} <= kinds
    kinds = run_state_after(pkg, FS5, BAND_B, rng, flags, q15_tail=True)
    assert LONG in kinds


# ---------------------------------------------------------------------------
# (b), (c) a client handed from group to group and back, tickets in flight on both
# ---------------------------------------------------------------------------
HAND_SIZES = [MAX_IN, MAX_IN, 7001, MAX_IN, 2, MAX_IN, 0, MAX_IN, 3, MAX_IN, 12345, MAX_IN, MAX_IN, MAX_IN - 2,
              MAX_IN, MAX_IN, 5, MAX_IN, MAX_IN, MAX_IN, MAX_IN, 9999, MAX_IN]


def run_handoff(pkg, fs, spec, n_others, sizes, cuts, attach_at=0, seed=0):
    """Group A starts with only the continuing clients; group B with `n_others` clients of the same spec.
    Both groups consume every block.  The continuing clients (one one-hot at a nonzero centre that reads
    its deepest history sample, one dyadic at centre 0) are created in A before block `attach_at` and move
    to the other group before every block in `cuts`.  Returns (clients, valid_history of each hand-over)."""
    L, M, T = spec
    rng = np.random.default_rng(seed)
    a = pkg.Group(fs, MAX_IN, flags=pkg.XLG_TRACK_STATE)
    b = pkg.Group(fs, MAX_IN, flags=pkg.XLG_TRACK_STATE)
    for _ in range(n_others):
        Client(rng, fs, L, M, T).attach(b)
    groups = {"A": a, "B": b}
    xs = [Client(rng, fs, L, M, T, j=T - 1), Client(rng, fs, L, M, T, dyadic=True)]
    for c in xs:
        c.kinds = {"A": set(), "B": set()}
        c.state = None
    cids, where, pending = {}, None, {"A": [], "B": []}
    consumed, handed = 0, []

    def collect(name):
        t, blk, members = pending[name].pop(0)
        if not members:
            return  # nothing to read (a client added later may have grown the group's result arenas)
        groups[name].wait(t)
        for c, cid in members:
            y, c.state = groups[name].copy_output(t, cid)
            c.got.append(y)
            c.kinds[name].add(groups[name].client_info(cid)[1])

    for i, n in enumerate(sizes):
        if i == attach_at:
            where = "A"
            cids = {id(c): c.attach(a) for c in xs}
        elif i in cuts:
            src, dst = where, "B" if where == "A" else "A"
            while pending[src]:
                collect(src)
            for c in xs:
                groups[src].remove_client(cids[id(c)])
                c.state.valid_history = consumed
                cids[id(c)] = c.attach(groups[dst], state=c.state)
            handed.append(consumed)
            where = dst
        x = real_grid_input(rng, n)
        if i >= attach_at:
            for c in xs:
                c.feed(x)
            consumed += n // 2
        for name, g in groups.items():
            members = [(c, cids[id(c)]) for c in xs] if name == where else []
            pending[name].append((g.submit("cs16", x), i, members))
            if len(pending[name]) >= 3:
                collect(name)
    for name in groups:
        while pending[name]:
            collect(name)
    a.close()
    b.close()
    for c in xs:
        assert_exact(c.got, c.want, f"continuing client {c.label}, hand-overs at {sorted(cuts)}", T, M)
    return xs, handed


@pytest.mark.parametrize("fs,spec,kind", [(FS, (1, 21, 253), TILED), (FS5, (1, 1280, 1407), LONG),
                                          (FS, (3, 128, 385), POLY_TILED)], ids=["tiled", "split_k", "poly_tiled"])
def test_continuing_client_across_kernels(pkg, fs, spec, kind):
    """A client handed from A (where it is alone with its twin) to B (where 8 others make its class) and
    back every few blocks, after odd, empty and 2-element calls: every output equals the oracle fed the
    whole stream.  In A it runs on the generic kernel of its kind, in B on `kind`."""
    xs, handed = run_handoff(pkg, fs, spec, 8, HAND_SIZES, {2, 5, 8, 12, 16, 19}, seed=spec[2])
    assert len(handed) == 6
    for c in xs:
        assert kind in c.kinds["B"], (c.label, c.kinds)
        if kind != LONG:
            assert c.kinds["A"] == {POLY if spec[0] > 1 else GENERIC}, (c.label, c.kinds)


@pytest.mark.parametrize("spec", [(1, 21, 253), (3, 128, 385)], ids=["integer", "rational"])
def test_continuing_client_with_short_history(pkg, spec):
    """A client attached to A mid-stream is handed to B after 2 samples, before it has T - 1 of its own:
    B has run from the start, and the samples its ring holds from before the attach point must read as
    zero for the client (valid_history < T - 1)."""
    L, M, T = spec
    sizes = [MAX_IN, MAX_IN, 7001, 2, 3, MAX_IN, MAX_IN, 12345, MAX_IN, MAX_IN, MAX_IN, 5, MAX_IN]
    xs, handed = run_handoff(pkg, FS, spec, 8, sizes, {5, 9}, attach_at=3, seed=T)
    assert handed[0] == 2 and handed[0] * L < T - 1
