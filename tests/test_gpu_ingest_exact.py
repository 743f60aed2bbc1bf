"""Every way a block enters a batch group, bit for bit.

The other exact suites feed pageable numpy arrays.  Here the same blocks also arrive as page-locked host
memory (the library's PinnedBuffer at offsets 0-3 and a torch pin_memory() tensor, with and without
XLG_INPUT_KEEP), as device memory at byte offsets 0, 2, 4 and 8, and as device memory written by a producer
on another stream and published with xlg_wait_stream.  Every buffer that the contract allows to be reused is
overwritten at the earliest moment the contract allows it, so an early return shows up as wrong outputs.

1. The conversion matrix: cu8, cs8 and cs16 on the float and the Q15 path, blocks of 0 to 3 scalars, odd
   complex counts, max_in - 2 and max_in at both stream parities, against the float64 / int64 references on
   dyadic taps, and the one-hot phase harness at random centres against the strict oracle.  A mirror of
   launch_convert's rule (tests/ingest.py) confirms that the vectorised, scalar and Q15 conversions all ran,
   on host and on device blocks, for every format.
2. Every kernel family in one group, in every pipeline variant, fed through every non-pageable mode with
   XLG_SLOTS tickets in flight: bitwise equal to a twin group fed pageable arrays.
3. Ordering contracts, made deterministic by holding the group's streams back behind a bounded sleep kernel.
4. bench.py's three ingest loops, replayed small, every client of every block checked.
5. Refusals: misaligned device blocks, and xlg_input_consumed's answers.
"""
import numpy as np
import pytest

from exact import (assert_exact, dyadic_taps, exact_input, grid_step, one_hot_taps, real_input, ref_f64_many,
                   ref_q15)
from ingest import Q15, SCALAR, VEC, conv_kind, device_offsets
from oracle import pyoracle as po

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

FS, MAX_IN = 2016000, 4096
ITEM = {"cu8": 1, "cs8": 1, "cs16": 2}
# a bounded delay for the group's streams: about 100 ms at the H100's boost clock, 200 ms at 1 GHz
SLEEP_CYCLES = 200_000_000
EINVAL = -22
HOST_MODES = ["pageable", "pageable_odd", "pinned0", "pinned1", "pinned2", "pinned3", "keep_consumed", "keep_wait",
              "torch_pinned"]


def device_modes(fmt):
    return [f"dev{o}" for o in device_offsets(fmt)] + ["dev_stream"]


def all_modes(fmt):
    return HOST_MODES + device_modes(fmt)


def garbage(a):
    """Overwrite a raw block in place with other values (every element changes)."""
    a[...] = ~a


class Feeder:
    """Submits raw blocks to a group through a chosen mode.  Every buffer lives as long as the feeder, and a
    buffer is overwritten with garbage at the earliest moment the contract allows: at once when submit
    returns (pageable, pinned without KEEP), or after xlg_input_consumed / xlg_wait of its ticket (KEEP,
    device), which the feeder calls before the next block it submits (or in flush())."""

    def __init__(self, pkg, g, fmt, max_in, q15=False):
        self.pkg, self.g, self.fmt, self.q15 = pkg, g, fmt, q15
        self.code = pkg.FMT[fmt]
        self.dtype = pkg.NP_DTYPE[fmt]
        nb = max_in * ITEM[fmt] + 16
        self.pageable = np.zeros(nb, np.uint8)
        self.pinned = pkg.PinnedBuffer(nb)
        self.keep = pkg.PinnedBuffer(nb)
        self.torch_pin = torch.zeros(nb, dtype=torch.uint8).pin_memory()
        self.src_pin = torch.zeros(nb, dtype=torch.uint8).pin_memory()
        self.dev = torch.zeros(nb, dtype=torch.uint8, device="cuda")
        self.side, self.other = torch.cuda.Stream(), torch.cuda.Stream()
        self.pending = []  # releases of the previous block's buffer
        self.kernel_ptrs = []  # (mode, n complex, S, pointer the conversion reads or None) per submit
        torch.cuda.current_stream().synchronize()

    def flush(self):
        while self.pending:
            self.pending.pop(0)()

    def _scribble_dev(self):
        with torch.cuda.stream(self.other):
            self.dev.fill_(0x5A)
        self.other.synchronize()

    def submit(self, mode, raw, S):
        """Submit raw (a numpy block of the feeder's format) through mode; S is the stream position on the
        block's path (for the conversion mirror).  Returns the ticket."""
        self.flush()
        g, pkg = self.g, self.pkg
        raw = np.ascontiguousarray(raw, dtype=self.dtype)
        b = raw.view(np.uint8)
        nbytes, n = b.size, raw.size
        flags = pkg.XLG_PATH_Q15 if self.q15 else 0
        kptr = None
        if mode in ("pageable", "pageable_odd"):
            off = 1 if mode == "pageable_odd" else 0
            view = self.pageable[off:off + nbytes]
            view[:] = b
            t = g.submit_ptr(self.code, view.ctypes.data, n, flags)
            garbage(view)
        elif mode.startswith("pinned"):
            off = int(mode[len("pinned"):])
            view = self.pinned.array()[off:off + nbytes]
            view[:] = b
            t = g.submit_ptr(self.code, self.pinned.ptr + off, n, flags)
            garbage(view)
        elif mode in ("keep_consumed", "keep_wait"):
            view = self.keep.array()[:nbytes]
            view[:] = b
            t = g.submit_ptr(self.code, self.keep.ptr, n, flags | pkg.XLG_INPUT_KEEP)
            release = g.input_consumed if mode == "keep_consumed" else g.wait
            self.pending.append(lambda: (release(t), garbage(view)))
        elif mode == "torch_pinned":
            view = self.torch_pin.numpy()[:nbytes]
            view[:] = b
            t = g.submit_ptr(self.code, self.torch_pin.data_ptr(), n, flags)
            garbage(view)
        elif mode.startswith("dev"):
            if mode == "dev_stream":
                off = 0
                self.src_pin.numpy()[:nbytes] = b
                with torch.cuda.stream(self.side):
                    self.dev[:nbytes].copy_(self.src_pin[:nbytes], non_blocking=True)
                g.wait_stream(self.side.cuda_stream)
            else:
                off = int(mode[len("dev"):])
                self.dev[off:off + nbytes].copy_(torch.from_numpy(b.copy()))
                torch.cuda.current_stream().synchronize()
            kptr = self.dev.data_ptr() + off
            t = g.submit_ptr(self.code, kptr, n, flags | pkg.XLG_INPUT_DEVICE)

            def release(t=t):
                g.input_consumed(t)
                self.side.synchronize()
                self._scribble_dev()
            self.pending.append(release)
        else:
            raise ValueError(mode)
        self.kernel_ptrs.append((mode, n // 2, S, kptr))
        return t


def read(g, t, cid, q15=False):
    return g.read_output(t, cid, q15=q15) if g.flags & 0x1 else g.output(t, cid, q15=q15)


def coverage(fmt, q15, kernel_ptrs):
    """{"host": kinds, "device": kinds} of the conversions the schedule ran (blocks with n > 0)."""
    seen = {"host": set(), "device": set()}
    for mode, n, S, ptr in kernel_ptrs:
        if n > 0:
            seen["device" if mode.startswith("dev") else "host"].add(conv_kind(fmt, q15, n, S, ptr))
    return seen


# ---------------------------------------------------------------------------
# 1. the conversion matrix
# ---------------------------------------------------------------------------
# scalars per block: empty, 1 to 3 scalars, odd complex counts, max_in - 2 and max_in; the sum of complex samples
# is odd, so consecutive modes start at alternating stream parities
LENS = [MAX_IN, 0, 2, 6, 1, 3, MAX_IN - 2, 154, 11, MAX_IN, 2002, MAX_IN]
assert sum(n // 2 for n in LENS) % 2 == 1


def matrix_run(pkg, fmt, q15, seed):
    rng = np.random.default_rng(seed)
    g = pkg.Group(FS, MAX_IN)
    specs = [(1, 1), (3, 5), (2, 8), (7, 64)]
    clients = []
    for D, T in specs:
        taps = dyadic_taps(rng, T, fmt, k=15 if q15 else None)
        clients.append((g.add_client(D, taps, 0), D, taps))
    f = Feeder(pkg, g, fmt, MAX_IN, q15)
    schedule = [(m, n) for m in all_modes(fmt) for n in LENS]
    blocks, got, pending, S = [], [[] for _ in clients], [], 0

    def collect():
        t = pending.pop(0)
        g.wait(t)
        for i, (cid, _, _) in enumerate(clients):
            got[i].append(np.array(g.output(t, cid, q15=q15), copy=True))

    for mode, n in schedule:
        x = exact_input(rng, fmt, n)
        blocks.append(x)
        pending.append(f.submit(mode, x, S))
        S += n // 2
        if len(pending) >= 2:
            collect()
    f.flush()
    while pending:
        collect()
    g.close()
    for i, (cid, D, taps) in enumerate(clients):
        if q15:
            ref = ref_q15(taps, D, fmt, blocks)
        else:
            ref = ref_f64_many([taps], D, fmt, blocks)[0]
        # name the mode of the first failing block
        for b, (mode, n) in enumerate(schedule):
            if not np.array_equal(np.asarray(got[i][b]), np.asarray(ref[b])):
                assert_exact(got[i][b:], ref[b:], f"{fmt} q15={q15} client D={D} T={len(taps)}: block {b} via "
                             f"{mode} ({n} scalars)", len(taps), D, None if q15 else grid_step(taps, fmt))
    return coverage(fmt, q15, f.kernel_ptrs)


@pytest.mark.parametrize("fmt", ["cu8", "cs8", "cs16"])
def test_conversion_matrix(pkg, fmt):
    """Every mode, every length class, both stream parities, the float and the Q15 path: exact."""
    cf = matrix_run(pkg, fmt, False, seed=100 + len(fmt))
    qq = matrix_run(pkg, fmt, True, seed=200 + len(fmt))
    for where in ("host", "device"):
        assert cf[where] == {VEC, SCALAR}, (fmt, where, cf[where])
        assert qq[where] == {Q15}, (fmt, where, qq[where])


def test_phase_harness_every_mode(pkg):
    """One-hot taps, real cs16 input, random centres: every mode equals the strict float32 oracle bit for bit
    (the oscillator sees the stream positions every mode advances)."""
    rng = np.random.default_rng(300)
    D, T = 3, 9
    g = pkg.Group(FS, MAX_IN)
    band = FS // 2 - FS // (2 * D)
    live = []
    for i in range(6):
        j = (0, T - 1, int(rng.integers(1, T - 1)))[i % 3]
        center = int(rng.integers(-band, band))
        taps = one_hot_taps(T, j, float(rng.choice([0.75, -0.5, 0.3125])))
        live.append((g.add_client(D, taps, center), po.OracleFilter(D, taps, center, FS, MAX_IN), f"j={j} c={center}"))
    f = Feeder(pkg, g, "cs16", MAX_IN)
    S = 0
    for mode in all_modes("cs16"):
        for n in (MAX_IN, 2, MAX_IN - 2, 154, MAX_IN):
            x = real_input(rng, n)
            t = f.submit(mode, x, S)
            S += n // 2
            g.wait(t)
            for cid, o, label in live:
                assert_exact(g.output(t, cid), o.process_cf32("cs16", x), f"{mode} n={n} {label}")
    f.flush()
    g.close()


# ---------------------------------------------------------------------------
# 2. every kernel family, bitwise against a twin fed pageable arrays
# ---------------------------------------------------------------------------
FS_MIX, MAX_MIX = 2048000, 65536
FS5, MAX5 = 61440000, 131072


def rtaps(rng, n):
    return rng.standard_normal(n).astype(np.float32) / n


def population(pkg, g, rng, kind):
    """(every client id, [(cid, D, dyadic taps)] of the integer clients at centre 0 with an exact reference)."""
    ids, exact = [], []

    def add_exact(D, T, count, fmt):
        for _ in range(count):
            taps = dyadic_taps(rng, T, fmt)
            exact.append((g.add_client(D, taps, 0), D, taps))

    if kind == "mixed":
        # test_gpu_group_spans.py::test_every_span_in_one_group's population, with members on the bank channel,
        # a rational cascade and a rational member
        ids += [g.add_client(64, rtaps(rng, 257), -900000 + 110000 * c) for c in range(16)]
        ids.append(g.add_client(32, rtaps(rng, 101), 300000))
        plan = pkg.rational_plan(FS_MIX, [48000] * 8)
        ids += [g.add_client_rational(p["interp"], p["decim"], p["taps"], p["center"]) for p in plan]
        p = plan[0]
        ids.append(g.add_client_rational(p["interp"], p["decim"], p["taps"][:-3], -p["center"]))
        ids.append(g.add_client_cascade(16, rtaps(rng, 65), 200000, 4, rtaps(rng, 33)))
        ids.append(g.add_client_cascade(16, rtaps(rng, 65), -250000, 5, rtaps(rng, 40), interp2=3))
        sid = g.add_subband(32, rtaps(rng, 129), -400000)
        ids.append(g.add_client_subband(sid, 4, rtaps(rng, 33), 5000))
        ids.append(g.add_client_subband(sid, 5, rtaps(rng, 30), -3000, interp2=2))
        bid = g.add_bank(16, rtaps(rng, 257))
        ids.append(g.add_client_subband(g.add_bank_subband(bid, 3), 4, rtaps(rng, 33), 0))
        add_exact(32, 97, 8, "cu8")  # a tiled class
        add_exact(5, 40, 2, "cu8")   # generic
    else:
        # a split-K long-filter class at 61.44 Msps
        ids += [g.add_client(1280, rtaps(rng, 1407), int(rng.integers(-30000000, 30000000))) for _ in range(8)]
        add_exact(1280, 2561, 8, "cs16")
        add_exact(5, 40, 2, "cs16")
    return ids + [c for c, _, _ in exact], exact


TWIN_VARIANTS = [({}, 0), ({"XLATING_B200_CONV_STREAM": "0"}, 0),
                 ({"XLATING_B200_SPECULATE": "0", "XLATING_B200_CSTREAMS": "1"}, 0),
                 ({"XLATING_B200_PARTITION": "1"}, "XLG_SM_PARTITION"), ({}, "XLG_OUT_DEVICE")]


@pytest.mark.parametrize("kind", ["mixed", "split_k"])
@pytest.mark.parametrize("env,flag", TWIN_VARIANTS,
                         ids=["default", "conv_on_compute_stream", "no_spec_1stream", "partition", "device_out"])
def test_every_family_against_pageable_twin(pkg, monkeypatch, kind, env, flag):
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    flags = getattr(pkg, flag) if flag else 0
    fs, max_in, fmt = (FS_MIX, MAX_MIX, "cu8") if kind == "mixed" else (FS5, MAX5, "cs16")
    a, b = pkg.Group(fs, max_in, flags=flags), pkg.Group(fs, max_in, flags=flags)
    ids, exact = population(pkg, a, np.random.default_rng(400), kind)
    ids_b, _ = population(pkg, b, np.random.default_rng(400), kind)
    assert ids == ids_b
    modes = [m for m in all_modes(fmt) if not m.startswith("pageable")]
    rng = np.random.default_rng(401)
    sizes = [max_in, max_in, max_in - 2, 30002, max_in, 7] * 4
    schedule = [(modes[i % len(modes)], sizes[i % len(sizes)]) for i in range(2 * len(modes))]
    f = Feeder(pkg, a, fmt, max_in)
    blocks, pend, S = [], [], 0
    got = {c: [] for c, _, _ in exact}

    def collect():
        i, ta, tb = pend.pop(0)
        a.wait(ta)
        b.wait(tb)
        for c in ids:
            ya, yb = read(a, ta, c), read(b, tb, c)
            assert_exact(ya, yb, f"{kind} {env} flags={flags}: client {c} kind {a.client_info(c)[1]}, block {i} "
                         f"via {schedule[i][0]}")
            if c in got:
                got[c].append(ya)

    for i, (mode, n) in enumerate(schedule):
        x = exact_input(rng, fmt, n)
        blocks.append(x)
        ta = f.submit(mode, x, S)
        tb = b.submit(fmt, x)
        assert ta == tb
        S += n // 2
        pend.append((i, ta, tb))
        if len(pend) >= pkg.XLG_SLOTS:
            collect()
    f.flush()
    while pend:
        collect()
    kinds = {a.client_info(c)[1] for c in ids}
    a.close()
    b.close()
    assert kinds >= ({0, 1, 3, 4, 5, 6} if kind == "mixed" else {0, 2}), kinds
    by_shape = {}
    for c, D, taps in exact:
        by_shape.setdefault((D, taps.size), []).append((c, taps))
    for (D, T), cs in by_shape.items():
        refs = ref_f64_many([t for _, t in cs], D, fmt, blocks)
        for (c, taps), r in zip(cs, refs):
            assert_exact(got[c], r, f"{kind} {env} flags={flags}: exact client {c} (D={D}, T={T})", T, D,
                         grid_step(taps, fmt))


# ---------------------------------------------------------------------------
# 3. ordering contracts, with the group's streams held back by a sleep on a side stream
# ---------------------------------------------------------------------------
N3 = 2048  # scalars per block


class Rig:
    """A small group of dyadic integer clients at centre 0 whose every output is checked exactly."""

    def __init__(self, pkg, fmt="cu8", flags=0, q15=False, seed=0, max_in=N3):
        self.pkg, self.fmt, self.q15 = pkg, fmt, q15
        self.rng = np.random.default_rng(seed)
        self.g = pkg.Group(FS, max_in, flags=flags)
        self.g.reserve(4 * max_in)  # attaches below must not grow the arenas (results in flight would be lost)
        self.clients = []  # [cid, D, taps, first block index]
        self.blocks, self.tickets = [], []
        self.outs = {}  # ticket -> {cid: output}, read before the ticket's results are recycled
        for D, T in ((1, 1), (3, 5), (7, 64)):
            self.add(D, T)

    def add(self, D, T):
        taps = dyadic_taps(self.rng, T, self.fmt, k=15 if self.q15 else None)
        self.clients.append([self.g.add_client(D, taps, 0), D, taps, len(self.blocks)])

    def block(self, n=N3):
        return exact_input(self.rng, self.fmt, n)

    def submitted(self, x, t):
        """Record that ticket t carries block x (as the stream must see it)."""
        self.blocks.append(np.array(x, copy=True))
        self.tickets.append(t)

    def read_now(self, t):
        self.g.wait(t)
        b = self.tickets.index(t)
        self.outs[t] = {cid: read(self.g, t, cid, q15=self.q15) for cid, _, _, first in self.clients if first <= b}

    def check(self, what, blocks=None):
        """Every output of every client against the reference of `blocks` (default: the recorded ones)."""
        blocks = self.blocks if blocks is None else blocks
        for t in self.tickets:
            if t not in self.outs:
                self.read_now(t)
        for cid, D, taps, first in self.clients:
            got = [self.outs[t][cid] for t in self.tickets[first:]]
            if self.q15:
                ref = ref_q15(taps, D, self.fmt, blocks[first:])
            else:
                ref = ref_f64_many([taps], D, self.fmt, blocks[first:])[0]
            assert_exact(got, ref, f"{what}: client {cid} (D={D}, T={len(taps)})", len(taps), D,
                         None if self.q15 else grid_step(taps, self.fmt))

    def close(self):
        self.g.close()


def hold_back(g):
    """A bounded sleep on a side stream that the group's next submits wait for; returns the stream."""
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(SLEEP_CYCLES)
    g.wait_stream(side.cuda_stream)
    return side


def filler(r):
    """The first submit after a wait_stream: its H2D copy is enqueued before the wait is attached, so it is the
    second submit whose copy the delay holds back."""
    x = r.block()
    r.submitted(x, r.g.submit(r.fmt, x))


@pytest.mark.parametrize("case", ["pageable", "pinned", "keep_consumed", "keep_overwritten"])
def test_host_block_reuse(pkg, case):
    """(a) a pageable block and a pinned one without KEEP overwritten as soon as submit returns, (b) a KEEP
    block overwritten after input_consumed: exact.  (c) The positive control: a KEEP block overwritten at once,
    with neither call, yields the overwritten block's outputs -- the copy really was held back."""
    r = Rig(pkg, seed=500)
    side = hold_back(r.g)
    filler(r)
    x = r.block()
    y = r.block()
    pin = pkg.PinnedBuffer(N3)
    view = pin.array()
    view[:] = x
    if case == "pageable":
        buf = x.copy()
        t = r.g.submit(r.fmt, buf)
        buf[:] = y
    elif case == "pinned":
        t = r.g.submit_ptr(pkg.FMT[r.fmt], pin.ptr, N3)
        view[:] = y
    else:
        t = r.g.submit_ptr(pkg.FMT[r.fmt], pin.ptr, N3, pkg.XLG_INPUT_KEEP)
        if case == "keep_consumed":
            r.g.input_consumed(t)
        view[:] = y
    r.submitted(x, t)
    if case == "keep_overwritten":
        r.check("positive control", blocks=r.blocks[:-1] + [y])
    else:
        r.check(case)
    side.synchronize()
    r.close()
    pin.free()


def device_block(r, x):
    """x in a fresh device buffer, written and finished on the current stream."""
    d = torch.from_numpy(x.view(np.uint8).copy()).cuda()
    torch.cuda.current_stream().synchronize()
    return d


D_CASES = ["direct", "empty_between", "attach_between", "attach_switches_partition", "q15"]
D_ENVS = [{}, {"XLATING_B200_CONV_STREAM": "0"}, {"XLATING_B200_SPECULATE": "0", "XLATING_B200_CSTREAMS": "1"}]


@pytest.mark.parametrize("env", D_ENVS, ids=["default", "conv_on_compute_stream", "no_spec_1stream"])
@pytest.mark.parametrize("case", D_CASES)
def test_device_block_from_side_stream(pkg, monkeypatch, case, env):
    """(d) A device block written on a side stream after a sleep and published with wait_stream: exact
    directly, with an empty block or a client attach (a re-layout) in between, with an attach that switches
    the group between its partitioned and its plain stream sets, and on the Q15 path."""
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    monkeypatch.delenv("XLATING_B200_PARTITION", raising=False)
    part = case == "attach_switches_partition"
    q15 = case == "q15"
    max_in = 131072 if part else N3
    r = Rig(pkg, flags=pkg.XLG_SM_PARTITION if part else 0, q15=q15, seed=600, max_in=max_in)
    if part:
        # FIR-bound: long filters at a high decimation leave the oscillator chain short, so the group declines the
        # partition; the (1, 1) client attached below makes the chain the pacing stage, and the group takes it
        for cid, _, _, _ in r.clients:
            r.g.remove_client(cid)
        r.clients = []
        for c in range(64):
            r.g.add_client(64, rtaps(r.rng, 12001), -900000 + 28000 * c)
        r.add(64, 129)
    path = pkg.XLG_PATH_Q15 if q15 else 0
    n = max_in if part else N3
    x0 = r.block(n)
    r.submitted(x0, r.g.submit(r.fmt, x0, flags=path))
    r.g.wait(r.tickets[-1])
    sms_before = r.g.partition_sms()
    x = r.block(n)
    src = device_block(r, x)
    dst = torch.zeros_like(src)
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        torch.cuda._sleep(SLEEP_CYCLES)
        dst.copy_(src)
    r.g.wait_stream(side.cuda_stream)
    if case == "empty_between":
        r.submitted(x[:0], r.g.submit(r.fmt, x[:0], flags=path))
    elif case in ("attach_between", "attach_switches_partition"):
        r.add(1, 1)
    t = r.g.submit_ptr(pkg.FMT[r.fmt], dst.data_ptr(), n, path | pkg.XLG_INPUT_DEVICE)
    r.submitted(x, t)
    r.check(f"{case} {env}")
    sms_after = r.g.partition_sms()
    side.synchronize()
    r.close()
    if part:
        if sms_before == sms_after == 0:
            pytest.skip("green contexts unavailable: the partition could not be offered")
        assert sms_before == 0 and sms_after > 0, (sms_before, sms_after)


@pytest.mark.parametrize("env", D_ENVS, ids=["default", "conv_on_compute_stream", "no_spec_1stream"])
def test_two_producers_one_block(pkg, monkeypatch, env):
    """(e) Two producers fill the two halves of one device block, the slow one first; wait_stream on both, then
    one submit: the group waits for both streams, not only the last one named."""
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    r = Rig(pkg, seed=700)
    filler(r)
    x = r.block()
    src = device_block(r, x)
    dst = torch.zeros_like(src)
    h = N3 // 2
    slow, fast = torch.cuda.Stream(), torch.cuda.Stream()
    slow.wait_stream(torch.cuda.current_stream())
    fast.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(slow):
        torch.cuda._sleep(SLEEP_CYCLES)
        dst[:h].copy_(src[:h])
    with torch.cuda.stream(fast):
        dst[h:].copy_(src[h:])
    r.g.wait_stream(slow.cuda_stream)
    r.g.wait_stream(fast.cuda_stream)
    t = r.g.submit_ptr(pkg.FMT[r.fmt], dst.data_ptr(), N3, pkg.XLG_INPUT_DEVICE)
    r.submitted(x, t)
    r.check(f"two producers {env}")
    slow.synchronize()
    r.close()


@pytest.mark.parametrize("env", D_ENVS, ids=["default", "conv_on_compute_stream", "no_spec_1stream"])
def test_device_block_reused_after_input_consumed(pkg, monkeypatch, env):
    """(f) A device block whose conversion is held back behind a wait_stream: after input_consumed(t) a kernel
    on an unrelated stream overwrites it, and the ticket's outputs are still those of the original block."""
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    r = Rig(pkg, seed=800)
    filler(r)
    x = r.block()
    d = device_block(r, x)
    side = hold_back(r.g)
    t = r.g.submit_ptr(pkg.FMT[r.fmt], d.data_ptr(), N3, pkg.XLG_INPUT_DEVICE)
    r.g.input_consumed(t)
    other = torch.cuda.Stream()
    with torch.cuda.stream(other):
        d.fill_(0x5A)
    r.submitted(x, t)
    r.check(f"reused after input_consumed {env}")
    other.synchronize()
    side.synchronize()
    r.close()


# ---------------------------------------------------------------------------
# 4. bench.py's ingest loops, small
# ---------------------------------------------------------------------------
def bench_clients(r):
    for D, T in [(42, 129)] * 8 + [(21, 64)] * 8:
        r.add(D, T)


def test_bench_device_ring(pkg):
    """Tier (i): a device ring of blocks submitted at stride offsets (XLG_INPUT_DEVICE, XLG_OUT_DEVICE)."""
    r = Rig(pkg, flags=pkg.XLG_OUT_DEVICE, seed=900, max_in=16384)
    bench_clients(r)
    ring = [r.block(16384) for _ in range(6)]
    dev = torch.from_numpy(np.stack(ring).view(np.uint8).reshape(6, -1)).cuda()
    torch.cuda.current_stream().synchronize()
    stride, base = dev.stride(0), dev.data_ptr()
    pend = []
    for i in range(20):
        b = i % 6
        t = r.g.submit_ptr(pkg.FMT[r.fmt], base + b * stride, 16384, pkg.XLG_INPUT_DEVICE)
        r.submitted(ring[b], t)
        pend.append(t)
        if len(pend) >= pkg.XLG_SLOTS - 1:
            r.read_now(pend.pop(0))
    r.check("tier (i)")
    r.close()


def test_bench_rotating_keep_blocks(pkg):
    """Tier (iii): 8 rotating KEEP pinned blocks, XLG_SLOTS - 1 tickets in flight, each block refilled only after
    the wait of the ticket that read it."""
    r = Rig(pkg, seed=901, max_in=16384)
    bench_clients(r)
    pins = [pkg.PinnedBuffer(16384) for _ in range(8)]
    owner = [None] * 8
    pend = []

    def drain_one():
        t = pend.pop(0)
        r.read_now(t)
        i = owner.index(t)
        owner[i] = None
        garbage(pins[i].array())  # refilled as soon as the ticket that read it is done

    for s in range(24):
        i = s % 8
        assert owner[i] is None
        x = r.block(16384)
        pins[i].array()[:] = x
        t = r.g.submit_ptr(pkg.FMT[r.fmt], pins[i].ptr, 16384, pkg.XLG_INPUT_KEEP)
        owner[i] = t
        r.submitted(x, t)
        pend.append(t)
        if len(pend) >= pkg.XLG_SLOTS - 1:
            drain_one()
    while pend:
        drain_one()
    r.check("tier (iii)")
    r.close()
    for p in pins:
        p.free()


@pytest.mark.parametrize("from_host", [False, True], ids=["from_device", "from_pinned"])
def test_bench_broadcast_leg(pkg, from_host):
    """The broadcast leg at world = 1: XLG_SLOTS device buffers, a non_blocking copy on the current stream,
    wait_stream on it, a device submit; a buffer is refilled after the wait of the ticket that used it."""
    r = Rig(pkg, flags=pkg.XLG_OUT_DEVICE, seed=902, max_in=16384)
    bench_clients(r)
    src_host = np.stack([r.block(16384) for _ in range(5)])
    raw = torch.from_numpy(src_host.view(np.uint8).reshape(5, -1))
    src = raw.pin_memory() if from_host else raw.cuda()
    ring = [torch.empty(src.shape[1], dtype=torch.uint8, device="cuda") for _ in range(pkg.XLG_SLOTS)]
    stream = torch.cuda.current_stream()
    pend = []
    for i in range(17):
        buf = ring[i % len(ring)]
        if len(pend) >= len(ring) - 1:
            r.read_now(pend.pop(0))
        buf.copy_(src[i % 5], non_blocking=True)
        r.g.wait_stream(stream.cuda_stream)
        t = r.g.submit_ptr(pkg.FMT[r.fmt], buf.data_ptr(), 16384, pkg.XLG_INPUT_DEVICE)
        r.submitted(src_host[i % 5], t)
        pend.append(t)
    while pend:
        r.read_now(pend.pop(0))
    r.check("broadcast leg")
    r.close()


# ---------------------------------------------------------------------------
# 5. refusals
# ---------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", ["cu8", "cs8", "cs16"])
def test_misaligned_device_block_is_refused(pkg, fmt):
    """A device block not aligned to one complex sample: -EINVAL before anything is enqueued, no ticket taken,
    and the blocks after it are exact."""
    r = Rig(pkg, fmt=fmt, seed=1000)
    x0 = r.block()
    r.submitted(x0, r.g.submit(fmt, x0))
    d = torch.zeros(N3 * ITEM[fmt] + 16, dtype=torch.uint8, device="cuda")
    torch.cuda.current_stream().synchronize()
    step = 2 * ITEM[fmt]
    for off in range(1, step):
        for n in (N3, 2, 1):
            code = r.g._L.xlg_submit(r.g._h, pkg.FMT[fmt], d.data_ptr() + off, n, pkg.XLG_INPUT_DEVICE)
            assert code == EINVAL, (off, n, code)
    x = r.block()
    d[step:step + x.nbytes].copy_(torch.from_numpy(x.view(np.uint8).copy()))
    torch.cuda.current_stream().synchronize()
    t = r.g.submit_ptr(pkg.FMT[fmt], d.data_ptr() + step, N3, pkg.XLG_INPUT_DEVICE)
    assert t == r.tickets[-1] + 1
    r.submitted(x, t)
    x2 = r.block()
    r.submitted(x2, r.g.submit(fmt, x2))
    r.check(f"after refusals ({fmt})")
    r.close()


def test_input_consumed_answers(pkg):
    """-EINVAL for a ticket not yet submitted (and a negative one), 0 for a recycled ticket, for an empty block
    and for a completed one."""
    r = Rig(pkg, seed=1100)
    L, h = r.g._L, r.g._h
    assert L.xlg_input_consumed(h, 0) == EINVAL
    ts = []
    for n in [N3] * (pkg.XLG_SLOTS + 2) + [0]:
        x = r.block(n)
        ts.append(r.g.submit(r.fmt, x))
        r.submitted(x, ts[-1])
        r.read_now(ts[-1])
    assert L.xlg_input_consumed(h, ts[-1] + 1) == EINVAL
    assert L.xlg_input_consumed(h, -1) == EINVAL
    assert L.xlg_input_consumed(h, ts[0]) == 0  # recycled: its slot serves a later ticket
    assert L.xlg_input_consumed(h, ts[-1]) == 0  # empty block
    assert L.xlg_input_consumed(h, ts[-2]) == 0
    r.check("input_consumed answers")
    r.close()
