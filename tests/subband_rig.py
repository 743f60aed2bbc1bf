"""A group driven block by block with tickets in flight, whose sub-band members, bank channels and neighbour
clients are all checked exactly (tests/test_gpu_subband_exact.py, tests/test_gpu_bank_exact.py).

Ordinary sub-band members are checked against the float64 composition (dyadic stimuli) or the strict oracle
(stimuli where every member accumulator is one product); members of bank channels against bank_member_model's
chain (tests/bank_exact.py), on any taps and input, and -- where the channel has a copy member from its first
block -- also against member_model fed the GPU's own rows of that channel, so that a failure shows which stage
is wrong.  Neighbours (dyadic taps at centre 0) are checked against their float64 references.
"""
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from bank_exact import bank_model
from cascade import FloatPath, small_taps
from cascade_rational import f64_composition, stuff
from exact import assert_exact, one_hot_taps, ref_f64, to_complex
from oracle import pyoracle as po
from rational import branch_one_hot_taps, ref_rational_f64
from subband_exact import exact_bound, f64_member, f64_rows, member_consts, member_model

MEMBER = 6  # xlg_client_info kind of a sub-band member
BANK = 7    # xlg_subband_info kind of a bank channel


class Sb:
    """An ordinary sub-band, or (bank set) channel `chan` of a bank; `slot` is its client index."""

    def __init__(self, sid, d1, taps1, centre, first, dyadic, slot, bank=None, chan=None):
        self.sid, self.d1, self.taps1, self.centre, self.first, self.dyadic = sid, d1, taps1, centre, first, dyadic
        self.slot, self.bank, self.chan = slot, bank, chan
        self.last = self.copy = None


class Bank:
    def __init__(self, bid, d1, taps1, first):
        self.bid, self.d1, self.taps1, self.first = bid, d1, np.asarray(taps1, np.float32), first
        self.last = None


class Mb:
    """A member: f64 says it is checked against the float64 composition (dyadic taps at offset 0 on a dyadic
    sub-band), otherwise against the oracle (ordinary sub-bands) or the bank chain (bank channels)."""

    def __init__(self, cid, sb, l2, d2, taps2, offset, first, f64):
        self.cid, self.sb, self.l2, self.d2, self.taps2, self.offset = cid, sb, l2, d2, taps2, offset
        self.first, self.f64, self.last = first, f64, None
        self.got, self.kinds = [], set()

    def label(self):
        where = f"channel {self.sb.chan} of bank {self.sb.bank.bid}" if self.sb.bank else "sub-band"
        return (f"member {self.cid} of {where} {self.sb.sid} L2={self.l2} D2={self.d2} T2={self.taps2.size} "
                f"offset {self.offset} {'f64' if self.f64 else 'model/oracle'} from block {self.first}")


class Nb:
    """A neighbour client with dyadic taps at centre 0: ("i", D, taps), ("r", L, M, taps) or
    ("c", d1, taps1, d2, taps2)."""

    def __init__(self, cid, spec, first):
        self.cid, self.spec, self.first, self.last = cid, spec, first, None
        self.got = []


class Rig:
    """One group fed one block stream; outputs are read `depth` tickets late and churn happens with those
    tickets in flight (`reserve` sizes the result arenas up front so that no re-layout drops them).  The rig
    mirrors the group's client slots (every client takes the lowest free index), which order a bank's channel
    table."""

    def __init__(self, pkg, monkeypatch, fs, max_in, fmt, flags=0, host_ring=0, depth=1, env=None, reserve=0):
        for k, v in (env or {}).items():
            monkeypatch.setenv(k, v)
        self.pkg, self.fs, self.max_in, self.fmt, self.flags, self.depth = pkg, fs, max_in, fmt, flags, depth
        self.g = pkg.Group(fs, max_in, flags=flags, host_ring=host_ring)
        if reserve:
            self.g.reserve(reserve)
        self.blocks, self.sbs, self.mems, self.nbs, self.banks, self.pending = [], [], [], [], [], []
        self.used = set()

    def _slot(self):
        s = 0
        while s in self.used:
            s += 1
        return s

    def _take(self, cid=None):
        s = self._slot()
        assert cid is None or cid == s, (cid, s)  # the mirror of the group's slots
        self.used.add(s)
        return s

    def add_subband(self, d1, taps1, centre, dyadic):
        sid = self.g.add_subband(d1, taps1, centre)
        sb = Sb(sid, d1, taps1, centre, len(self.blocks), dyadic, self._take())
        self.sbs.append(sb)
        return sb

    def remove_subband(self, sb):
        self.g.remove_subband(sb.sid)
        sb.last = len(self.blocks)
        self.used.discard(sb.slot)

    def add_bank(self, d1, taps1):
        bk = Bank(self.g.add_bank(d1, taps1), d1, taps1, len(self.blocks))
        self.banks.append(bk)
        return bk

    def remove_bank(self, bk):
        self.g.remove_bank(bk.bid)
        bk.last = len(self.blocks)

    def add_channel(self, bk, k, copy=False):
        """Channel k of bank bk; copy: with a copy member (taps [1.0], D2 = 1, offset 0) that returns its rows."""
        sid = self.g.add_bank_subband(bk.bid, k)
        sb = Sb(sid, bk.d1, bk.taps1, k * self.fs // (2 * bk.d1), len(self.blocks), False, self._take(), bk, k)
        self.sbs.append(sb)
        if copy:
            sb.copy = self.add_member(sb, 1, 1, np.ones(1, np.float32), 0, False)
        return sb

    def channel_table(self, bk):
        """The bank's channel table in kernel order: its live channels by client slot."""
        return sorted((sb for sb in self.sbs if sb.bank is bk and sb.last is None), key=lambda sb: sb.slot)

    def add_member(self, sb, l2, d2, taps2, offset, f64):
        cid = self.g.add_client_subband(sb.sid, d2, taps2, offset, interp2=l2)
        self._take(cid)
        m = Mb(cid, sb, l2, d2, np.asarray(taps2, np.float32), offset, len(self.blocks), f64)
        self.mems.append(m)
        return m

    def remove_member(self, m):
        self.g.remove_client(m.cid)
        m.last = len(self.blocks)
        self.used.discard(m.cid)

    def add_neighbour(self, spec):
        g = self.g
        if spec[0] == "i":
            cid = g.add_client(spec[1], spec[2], 0)
        elif spec[0] == "r":
            cid = g.add_client_rational(spec[1], spec[2], spec[3], 0)
        else:
            cid = g.add_client_cascade(spec[1], spec[2], 0, spec[3], spec[4])
        self._take(cid)
        nb = Nb(cid, spec, len(self.blocks))
        self.nbs.append(nb)
        return nb

    def remove_neighbour(self, nb):
        self.g.remove_client(nb.cid)
        nb.last = len(self.blocks)
        self.used.discard(nb.cid)

    def live(self, c, b):
        return c.first <= b and (c.last is None or b < c.last)

    def submit(self, x):
        self.blocks.append(x)
        self.pending.append((len(self.blocks) - 1, self.g.submit(self.fmt, x)))
        while len(self.pending) >= self.depth:
            self.collect()

    def read(self, t, cid):
        y = self.g.read_output(t, cid) if self.flags & self.pkg.XLG_OUT_DEVICE else self.g.output(t, cid)
        return np.array(y, copy=True)

    def collect(self):
        b, t = self.pending.pop(0)
        self.g.wait(t)
        for m in self.mems:
            if self.live(m, b):
                m.got.append(self.read(t, m.cid))
                if m.last is None:
                    assert self.g.client_info(m.cid)[1] == MEMBER, m.label()
                    sid, kind, _ = self.g.subband_info(m.cid)
                    assert sid == m.sb.sid, m.label()
                    m.kinds.add(kind)
        for c in self.nbs:
            if self.live(c, b):
                c.got.append(self.read(t, c.cid))

    def flush(self):
        while self.pending:
            self.collect()

    def close(self):
        self.flush()
        self.g.close()

    def kinds(self):
        return set().union(*(m.kinds for m in self.mems))

    def check(self):
        """Every output of every member and neighbour of every block against its exact reference."""
        self.flush()
        renorm = not self.flags & self.pkg.XLG_NO_RENORM
        fs, fmt = self.fs, self.fmt
        sizes = [np.asarray(x).size // 2 for x in self.blocks]

        def rows_of(sb):
            seen = self.blocks[sb.first:sb.last]
            o = po.OracleFilter(sb.d1, sb.taps1, sb.centre, fs, self.max_in)
            rows = [o.process_cf32(fmt, x, renorm=renorm) for x in seen]
            o.close()
            if sb.dyadic:
                r64 = f64_rows(sb.d1, sb.taps1, fs, fmt, seen)
                assert all(np.array_equal(a, b) for a, b in zip(r64, rows)), f"sub-band {sb.sid}: oracle rows"
                return rows, r64
            return rows, None

        def bank_rows(bk):
            # the rows of the bank's channels that have members, from the bank's first block to its last
            chans = sorted({m.sb.chan for m in self.mems if m.sb.bank is bk})
            if not chans:
                return {}
            x = np.concatenate([to_complex(fmt, r) for r in self.blocks]).astype(np.complex64)
            return bank_model(bk.taps1, bk.d1, chans, x, int(sum(sizes[:bk.first])), sizes[bk.first:bk.last])

        ordinary = [sb for sb in self.sbs if sb.bank is None]
        with ThreadPoolExecutor(max_workers=8) as ex:
            rows = dict(zip(ordinary, ex.map(rows_of, ordinary)))
            brows = dict(zip(self.banks, ex.map(bank_rows, self.banks)))

        def one_member(m):
            sb = m.sb
            a = m.first - sb.first
            z = None if m.last is None else m.last - sb.first
            fs1 = fs // sb.d1
            if sb.bank is not None:
                bk = sb.bank
                lo = sb.first - bk.first
                hi = (len(self.blocks) if sb.last is None else sb.last) - bk.first
                rev, inc = member_consts(m.taps2, m.d2, m.offset, m.l2, fs1)
                want = member_model(brows[bk][sb.chan][lo:hi][:z], a, m.l2, m.d2, [rev], [inc], renorm)[0]
                errs = []
                try:
                    assert_exact(m.got, want, m.label() + " (bank chain)", m.taps2.size, m.d2)
                except AssertionError as e:
                    errs.append(str(e))
                c = sb.copy
                if c is not None and c is not m and c.first == sb.first and (c.last is None or (
                        m.last is not None and c.last >= m.last)):
                    own = member_model(c.got[:z], a, m.l2, m.d2, [rev], [inc], renorm)[0]
                    try:
                        assert_exact(m.got, own, m.label() + " (fed the GPU's rows)", m.taps2.size, m.d2)
                    except AssertionError as e:
                        errs.append(str(e))
                return "\n".join(errs) or None
            if m.f64:
                want = f64_member(rows[sb][1][a:z], m.l2, m.d2, m.taps2, fs1)
            else:
                f = FloatPath(m.d2, m.taps2, m.offset, m.l2 * fs1)
                want = [f.process_cf32(stuff(y, m.l2), renorm=renorm) for y in rows[sb][0][a:z]]
            try:
                assert_exact(m.got, want, m.label(), m.taps2.size, m.d2)
            except AssertionError as e:
                return str(e)
            return None

        def one_neighbour(c):
            seen = self.blocks[c.first:c.last]
            s = c.spec
            if s[0] == "i":
                want = ref_f64(s[2], s[1], fmt, seen)
            elif s[0] == "r":
                want = ref_rational_f64(s[3], s[1], s[2], fmt, seen)
            else:
                want = [y.astype(np.complex64) for y in
                        f64_composition(s[1], s[2], 1, s[3], s[4], fs, [to_complex(fmt, x) for x in seen])]
            try:
                assert_exact(c.got, want, f"neighbour {s[0]} {c.cid} from block {c.first}")
            except AssertionError as e:
                return str(e)
            return None

        with ThreadPoolExecutor(max_workers=8) as ex:
            errors = [e for e in list(ex.map(one_member, self.mems)) + list(ex.map(one_neighbour, self.nbs)) if e]
        assert not errors, f"{len(errors)} clients differ:\n" + "\n".join(errors[:6])
        for m in self.mems:
            assert len(m.got) == (len(self.blocks) if m.last is None else m.last) - m.first, m.label()
        return rows


# ---------------------------------------------------------------------------
# stimuli of ordinary sub-bands
# ---------------------------------------------------------------------------
def dyadic_stage_a(rng, d1, T1):
    """Dyadic sub-band taps: 3-bit ones for the short kinds; for the long kind (T1 = 800) 24 taps of +-1/2
    (the first and the last among them), so that long members still fit exact_bound."""
    if T1 < 100:
        return small_taps(rng, T1, 3)
    t = np.zeros(T1, np.float32)
    idx = np.concatenate([[0, T1 - 1], rng.choice(np.arange(1, T1 - 1), 22, replace=False)])
    t[idx] = 0.5 * rng.choice(np.array([-1, 1]), idx.size)
    return t


def dyadic_member(rng, taps1, T2, fmt):
    """Full-length dyadic member taps within exact_bound: 3-bit, 1-bit, or for long members +-1/2 at the first
    and last taps and as many others as the bound leaves."""
    for bits in (3, 2, 1):
        t = small_taps(rng, T2, bits)
        if exact_bound(taps1, t, fmt):
            return t
    t = np.zeros(T2, np.float32)
    t[[0, T2 - 1]] = 0.5
    n = 2
    while True:
        u = t.copy()
        u[rng.choice(np.arange(1, T2 - 1), min(n, T2 - 2), replace=False)] = 0.5
        if not exact_bound(taps1, u, fmt):
            break
        t, n = u, n * 2
    assert exact_bound(taps1, t, fmt) and np.count_nonzero(t) >= 2
    return t * rng.choice(np.array([-1, 1]), T2).astype(np.float32)


def one_hot_member(rng, l2, T2, fs1, any_offset):
    """(taps2, offset) exact on a complex row: offset 0 with one nonzero tap anywhere (branch-one-hot when
    rational), or any offset with the only nonzero tap at taps2[0]."""
    if any_offset:
        return one_hot_taps(T2, 0, float(rng.choice([0.5, -0.75, 0.625]))), int(rng.integers(-fs1 // 2, fs1 // 2))
    if l2 == 1:
        return one_hot_taps(T2, int(rng.integers(0, T2)), float(rng.choice([0.5, -0.75, 0.625]))), 0
    return branch_one_hot_taps(rng, T2, l2), 0


def real_row_member(rng, l2, T2, fs1):
    """(taps2, offset) exact on a real row (a centre-0 sub-band on a real input) at any offset: one nonzero
    tap, or one per branch."""
    t = one_hot_taps(T2, int(rng.integers(0, T2)), 0.5) if l2 == 1 else branch_one_hot_taps(rng, T2, l2)
    return t, int(rng.integers(-fs1 // 2, fs1 // 2))
