"""Cascade clients (xlg_add_client_cascade) on the GPU.

A cascade client is by definition two reference filters in series (include/xlating_group.h): stage A at the
band rate, stage B at centre 0 fed stage A's outputs.  Exact stimuli must equal the float64 composition bit
for bit; a single power-of-two stage-B tap must turn the output into the group's own integer client, taken
every D2-th output and scaled, at any centre; designed taps are held to the 1e-5 contract against
cascade_oracle.  Every test asserts which kernel served stage A (xlg_cascade_info).
"""
import errno

import numpy as np
import pytest

from cascade import cascade_oracle, f64_filter, small_taps
from exact import exact_input, reversed_taps, to_complex
from util import assert_cf32_close, oracle_stream, rand_block

pytestmark = pytest.mark.gpu

GENERIC, TILED, LONG, CASCADE = 0, 1, 2, 5
SLOTS = 4


def run_group(pkg, fs, max_in, fmt, specs, blocks, flags=0, host_ring=0, attach=None, detach=None, depth=1):
    """Drive one group.  specs / attach entries: ("c", d1, taps1, center, d2, taps2) or ("i", d, taps, center).
    Returns per spec: (outputs of the blocks it was attached for, first block, stage-A kinds seen)."""
    g = pkg.Group(fs, max_in, flags=flags, host_ring=host_ring)
    clients = []

    def add(spec, b):
        if spec[0] == "c":
            cid = g.add_client_cascade(spec[1], spec[2], spec[3], spec[4], spec[5])
        else:
            cid = g.add_client(spec[1], spec[2], spec[3])
        clients.append({"spec": spec, "cid": cid, "first": b, "last": None, "got": [], "kinds": set()})

    for sp in specs:
        add(sp, 0)
    pending = []

    def collect(b, t):
        g.wait(t)
        for c in clients:
            if c["first"] <= b and (c["last"] is None or b < c["last"]):
                y = g.read_output(t, c["cid"]) if flags & pkg.XLG_OUT_DEVICE else g.output(t, c["cid"])
                c["got"].append(np.array(y, copy=True))
                if c["spec"][0] == "c" and (c["last"] is None):
                    assert g.client_info(c["cid"])[1] == CASCADE
                    c["kinds"].add(g.cascade_info(c["cid"])[0])
                elif c["last"] is None:
                    c["kinds"].add(g.client_info(c["cid"])[1])

    for b, x in enumerate(blocks):
        if b in (attach or {}) or b in (detach or {}):
            if b in (attach or {}):  # an attach re-lays out the arenas: collect first (detach need not)
                while pending:
                    collect(*pending.pop(0))
            for i in (detach or {}).get(b, []):
                g.remove_client(clients[i]["cid"])
                clients[i]["last"] = b
            for sp in (attach or {}).get(b, []):
                add(sp, b)
        pending.append((b, g.submit(fmt, x)))
        if len(pending) >= depth:
            collect(*pending.pop(0))
    while pending:
        collect(*pending.pop(0))
    g.close()
    return clients


def exact_reference(spec, fmt, fs, blocks):
    _, d1, t1, center, d2, t2 = spec
    assert center == 0
    a = f64_filter(t1, d1, 0, fs, [to_complex(fmt, x) for x in blocks])
    z = f64_filter(t2, d2, 0, fs // d1, a)
    for y in z:  # the stimuli are exact: the float64 result is a float32 number
        assert np.array_equal(y.astype(np.complex64).astype(np.complex128), y)
    return z


# stage A: (D1, T1, taps1 bits), stage B: (D2, T2, taps2 bits), format, max_in, blocks; every partial sum
# is an integer number of steps below 2^24: T1 * A * M1 * T2 * M2 <= 2^24 (A: input magnitude in steps)
EXACT = {
    "generic": (6, 17, 3, 7, 85, 2, "cu8", 8192, True),
    "tiled": (6, 17, 3, 7, 85, 2, "cu8", 8192, False),
    "long": (400, 800, 1, 4, 21, 3, "cs16", 65536, False),
}


@pytest.mark.parametrize("case", list(EXACT))
def test_exact_against_float64_composition(pkg, case):
    d1, T1, b1, d2, T2, b2, fmt, max_in, generic = EXACT[case]
    amax = {"cu8": 255, "cs16": 128}[fmt]
    assert T1 * amax * (2 ** b1 - 1) * T2 * (2 ** b2 - 1) <= 2 ** 24
    rng = np.random.default_rng(len(case))
    fs = 2016000
    specs = [("c", d1, small_taps(rng, T1, b1), 0, d2, small_taps(rng, T2, b2)) for _ in range(8)]
    sizes = [max_in, max_in, 1001, max_in, 7, 0, max_in - 2, 2 * d1 * T2 + 1] + [max_in] * 8 + [333] * 8
    blocks = [exact_input(rng, fmt, n) for n in sizes]
    flags = pkg.XLG_FORCE_GENERIC if generic else 0
    clients = run_group(pkg, fs, max_in, fmt, specs, blocks, flags=flags, depth=SLOTS)
    want_kind = {"generic": GENERIC, "tiled": TILED, "long": LONG}[case]
    for c in clients:
        assert want_kind in c["kinds"] and c["kinds"] <= {GENERIC, want_kind}, c["kinds"]
        if case == "generic":
            assert c["kinds"] == {GENERIC}
        ref = exact_reference(c["spec"], fmt, fs, blocks)
        for b, (y, r) in enumerate(zip(c["got"], ref)):
            assert y.shape == r.shape, (case, b)
            assert np.array_equal(y, r.astype(np.complex64)), (case, b, np.max(np.abs(y - r)))


ANY_CENTRE = {  # fs, fmt, max_in, D1, stage-A rate for the design, flags
    "generic": (2016000, "cu8", 4096, 6, 48000, True),
    "tiled": (2016000, "cu8", 4096, 6, 48000, False),
    "long": (2016000, "cs16", 32768, 400, 2520, False),
}


@pytest.mark.parametrize("case", list(ANY_CENTRE))
def test_any_centre_single_tap_is_the_integer_client(pkg, case):
    """Stage B with one nonzero tap 0.5: the cascade's output k is 0.5 * y[k*D2 + r - (T2 - 1)], y being the
    outputs of the group's own integer client (D1, taps1, centre), r the tap's position in the reversed taps
    and y before the attach zero.  Five centres, 300+ blocks."""
    fs, fmt, max_in, d1, rate, generic = ANY_CENTRE[case]
    taps1 = pkg.create_low_pass_filter(1.0, fs, rate // 2, rate // 5)
    d2, T2 = 5, 24
    centres = [0, -312000, 17, 251001, -1000003]
    specs = []
    for i, ce in enumerate(centres):
        t2 = np.zeros(T2, np.float32)
        t2[(7 * i + 3) % T2] = 0.5
        specs += [("c", d1, taps1, ce, d2, t2), ("i", d1, taps1, ce)]
    rng = np.random.default_rng(11)
    sizes = [int(v) * 2 for v in rng.integers(max_in // 8, max_in // 2 + 1, 310)]
    sizes[5] = 0
    blocks = [rand_block(rng, fmt, n) for n in sizes]
    clients = run_group(pkg, fs, max_in, fmt, specs, blocks, flags=pkg.XLG_FORCE_GENERIC if generic else 0,
                        depth=SLOTS)
    want = {"generic": GENERIC, "tiled": TILED, "long": LONG}[case]
    for c, ci in zip(clients[0::2], clients[1::2]):
        assert want in c["kinds"] and c["kinds"] <= {GENERIC, want}, c["kinds"]
        assert c["kinds"] == ci["kinds"]
        r = int(np.flatnonzero(reversed_taps(c["spec"][5]))[0])
        y = np.concatenate(ci["got"])
        z = np.concatenate(c["got"])
        idx = np.arange(z.size) * d2 + r - (T2 - 1)
        assert idx[-1] < y.size
        want_z = np.where(idx >= 0, y[np.maximum(idx, 0)] * np.float32(0.5), 0).astype(np.complex64)
        assert np.array_equal(z, want_z), (case, c["spec"][3])


def contract(pkg, fs, rate, fmt, n_clients, max_in, sizes, seed, **kw):
    plan = pkg.cascade_plan(fs, [rate] * n_clients)
    specs = [("c", p["d1"], p["taps1"], p["center"], p["d2"], p["taps2"]) for p in plan]
    rng = np.random.default_rng(seed)
    blocks = [rand_block(rng, fmt, n) for n in sizes]
    attach = kw.pop("attach_plan", None)
    if attach is not None:
        kw["attach"] = {b: [("c", p["d1"], p["taps1"], p["center"], p["d2"], p["taps2"])
                            for p in pkg.cascade_plan(fs, [rate] * n)] for b, n in attach.items()}
    clients = run_group(pkg, fs, max_in, fmt, specs, blocks, **kw)
    oracles = [cascade_oracle(c["spec"][1], c["spec"][2], c["spec"][3], c["spec"][4], c["spec"][5], fs, max_in)
               for c in clients]
    outs = [oracle_stream([o], fmt, blocks[c["first"]:c["last"]])[0] for o, c in zip(oracles, clients)]
    for c, ref in zip(clients, outs):
        assert len(c["got"]) == len(ref)
        got, want = np.concatenate(c["got"]), np.concatenate(ref)
        assert [y.size for y in c["got"]] == [y.size for y in ref]
        assert_cf32_close(got, want, f"client {c['cid']} from block {c['first']}")
    return clients


def test_contract_61M_cs16(pkg):
    """The 61.44 Msps cs16 shape (configs[4]) with 8 clients at 48 kHz: 32 x 40, taps 79 / 481."""
    fs, max_in = 61440000, 131072
    sizes = [max_in if b % 7 else 65538 for b in range(300)]
    clients = contract(pkg, fs, 48000, "cs16", 8, max_in, sizes, 1, depth=SLOTS)
    assert all(TILED in c["kinds"] for c in clients)


def test_contract_2M_cu8_ragged_odd(pkg):
    """The 2.016 Msps cu8 shape (configs[1]): 6 x 7, taps 17 / 85, over ragged and odd block lengths."""
    fs, max_in = 2016000, 65536
    rng = np.random.default_rng(2)
    sizes = [max_in if b % 3 else int(v) for b, v in enumerate(rng.integers(0, max_in + 1, 300))]
    clients = contract(pkg, fs, 48000, "cu8", 8, max_in, sizes, 2, depth=SLOTS)
    assert all(c["kinds"] <= {GENERIC, TILED} and TILED in c["kinds"] for c in clients)


def test_contract_history_spans_blocks_ring_wraps(pkg):
    """Blocks so small that a block's stage-A outputs are fewer than stage B's history, XLG_SLOTS tickets in
    flight: stage B reads stage-A outputs of several earlier blocks, and each client's ring wraps a dozen times."""
    fs, max_in = 2016000, 256
    rng = np.random.default_rng(3)
    sizes = [int(v) for v in rng.integers(0, max_in + 1, 320)]
    clients = contract(pkg, fs, 48000, "cu8", 3, max_in, sizes, 3, depth=SLOTS)
    assert all(c["kinds"] == {GENERIC} for c in clients)


def test_contract_attach_and_remove_in_flight(pkg):
    """Clients attached mid-stream (zero history from their attach point) and removed with tickets in flight."""
    fs, max_in = 2016000, 16384
    rng = np.random.default_rng(4)
    sizes = [int(v) for v in rng.integers(1, max_in + 1, 300)]
    clients = contract(pkg, fs, 48000, "cu8", 9, max_in, sizes, 4, depth=SLOTS, attach_plan={97: 8, 180: 2},
                       detach={150: [0, 2, 4], 201: [10]})
    assert {len(c["got"]) for c in clients[:9]} == {150, 300}
    assert any(TILED in c["kinds"] for c in clients)


@pytest.mark.parametrize("mode", ["out_device", "host_ring"])
def test_contract_out_device_and_host_ring(pkg, mode):
    fs, max_in = 2016000, 32768
    rng = np.random.default_rng(5)
    sizes = [int(v) for v in rng.integers(max_in // 2, max_in + 1, 300)]
    if mode == "out_device":
        contract(pkg, fs, 48000, "cu8", 8, max_in, sizes, 5, flags=pkg.XLG_OUT_DEVICE, depth=SLOTS)
    else:
        contract(pkg, fs, 48000, "cu8", 8, max_in, sizes, 6, host_ring=16, depth=12)


def test_mixed_group_is_unchanged_by_cascade_clients(pkg):
    """Integer (tiled, generic), rational (tiled, generic) and cascade clients in one group: the integer and
    rational outputs equal those of the same group without the cascade clients bit for bit, the cascade
    clients meet the contract, and the result copy to the host ends at the last host-visible row."""
    fs, max_in, fmt = 2048000, 65536, "cu8"
    ints = [(64, pkg.create_low_pass_filter(1.0, fs, p["cutoff"], p["tw"]), p["center"])
            for p in pkg.client_plan(fs, [32000] * 8)]
    ints += [(32, pkg.create_low_pass_filter(1.0, fs, 32000, 12800), c) for c in (-500000, 400000)]
    rats = pkg.rational_plan(fs, [48000] * 8 + [96000] * 2)
    cas = pkg.cascade_plan(fs, [32000] * 8)
    rng = np.random.default_rng(7)
    blocks = [rand_block(rng, fmt, max_in if b % 4 else 30001) for b in range(40)]
    res = []
    for with_cascade in (True, False):
        g = pkg.Group(fs, max_in)
        ids = [g.add_client(d, t, c) for d, t, c in ints]
        ids += [g.add_client_rational(p["interp"], p["decim"], p["taps"], p["center"]) for p in rats]
        cids = [g.add_client_cascade(p["d1"], p["taps1"], p["center"], p["d2"], p["taps2"]) for p in cas] \
            if with_cascade else []
        g.profile_enable(True)
        outs, couts, kinds, d2h = [], [], set(), []
        for x in blocks:
            t = g.submit(fmt, x)
            g.wait(t)
            outs.append([g.output(t, c) for c in ids])
            couts.append([g.output(t, c) for c in cids])
            ptrs = [g.output_ptr(t, c) for c in ids + cids]
            base = min(p for p, _ in ptrs)
            d2h.append((g.cascade_profile_read()["d2h_bytes"], max((p - base) + 8 * n for p, n in ptrs),
                        8 * sum(n for _, n in ptrs)))
            kinds |= {g.client_info(c)[1] for c in ids}
        akinds = {g.cascade_info(c)[0] for c in cids}
        g.close()
        res.append((outs, couts, kinds, akinds, d2h))
    assert res[0][2] == res[1][2] == {0, 1, 3, 4}
    assert res[0][3] == {TILED}
    for a, b in zip(res[0][0], res[1][0]):
        for ya, yb in zip(a, b):
            assert np.array_equal(ya.view(np.uint64), yb.view(np.uint64))
    for got_bytes, extent, payload in res[0][4]:
        assert got_bytes == extent and payload <= got_bytes
    for i, p in enumerate(cas):
        o = cascade_oracle(p["d1"], p["taps1"], p["center"], p["d2"], p["taps2"], fs, max_in)
        ref = [o.process_cf32(fmt, x) for x in blocks]
        assert_cf32_close(np.concatenate([c[i] for c in res[0][1]]), np.concatenate(ref), f"cascade {i}")


def test_refusals(pkg, capfd):
    """-EINVAL for a zero decimation or tap count, -ENOTSUP on an XLG_TRACK_STATE group, -ENOTSUP for a Q15
    submit to a group with a cascade client: each logged, nothing enqueued, and the next cf32 submit carries
    on as if the refused calls had not happened."""
    fs, max_in, fmt = 2016000, 16384, "cu8"
    p = pkg.cascade_plan(fs, [48000])[0]
    t1, t2 = p["taps1"], p["taps2"]
    rng = np.random.default_rng(8)
    blocks = [rand_block(rng, fmt, max_in) for _ in range(6)]
    g = pkg.Group(fs, max_in)
    twin = pkg.Group(fs, max_in)
    empty = np.zeros(0, np.float32)
    for args in ((0, t1, 0, 7, t2), (6, t1, 0, 0, t2), (6, empty, 0, 7, t2), (6, t1, 0, 7, empty)):
        with pytest.raises(ValueError) as e:
            g.add_client_cascade(*args)
        assert e.value.args[0] == -errno.EINVAL
        assert "<3>" in capfd.readouterr().err
    tg = pkg.Group(fs, max_in, flags=pkg.XLG_TRACK_STATE)
    with pytest.raises(ValueError) as e:
        tg.add_client_cascade(6, t1, 0, 7, t2)
    assert e.value.args[0] == -errno.ENOTSUP and tg.client_count() == 0
    assert "<3>" in capfd.readouterr().err
    tg.close()
    ids = [grp.add_client_cascade(6, t1, p["center"], 7, t2) for grp in (g, twin)]
    assert g.client_count() == 1
    got, want = [], []
    for b, x in enumerate(blocks):
        if b in (1, 4):
            with pytest.raises(RuntimeError) as e:
                g.submit(fmt, x, flags=pkg.XLG_PATH_Q15)
            assert str(-errno.ENOTSUP) in str(e.value)
            assert "<3>" in capfd.readouterr().err
        t, tt = g.submit(fmt, x), twin.submit(fmt, x)
        assert t == tt == b  # the refused submits took no ticket
        g.wait(t)
        twin.wait(tt)
        got.append(g.output(t, ids[0]))
        want.append(twin.output(tt, ids[1]))
    g.close()
    twin.close()
    for a, b in zip(got, want):
        assert np.array_equal(a.view(np.uint64), b.view(np.uint64))
