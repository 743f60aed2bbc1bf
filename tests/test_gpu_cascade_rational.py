"""Rational cascade clients (xlg_add_client_cascade_rational) on the GPU.

A rational cascade client is by definition stage A, the reference filter at the band rate, followed by stage B,
the reference filter with decimation M2 at L2 * fs / D1 and centre 0 fed the zero-stuffed stage-A stream
(include/xlating_group.h).  Exact stimuli must equal the float64 composition bit for bit; a single stage-B tap
of 0.5 must turn the output into the group's own integer client, picked where the window meets a stage-A
sample, at any centre; designed taps are held to the 1e-5 contract against the composed oracle.
"""
import ctypes as C
import errno

import numpy as np
import pytest

from cascade import small_taps
from cascade_rational import RationalCascadeOracle, f64_composition
from exact import exact_input, reversed_taps, to_complex
from util import assert_cf32_close, oracle_stream, rand_block

pytestmark = pytest.mark.gpu

GENERIC, TILED, LONG, CASCADE = 0, 1, 2, 5
SLOTS = 4


def run_group(pkg, fs, max_in, fmt, specs, blocks, flags=0, host_ring=0, attach=None, detach=None, depth=1):
    """Drive one group.  specs / attach entries: ("c", d1, taps1, center, d2, taps2, l2), ("i", d, taps, center)
    or ("r", interp, decim, taps, center).  Returns per spec: outputs of the blocks it was attached for, first
    block, kernel kinds seen (stage A's for a cascade client)."""
    g = pkg.Group(fs, max_in, flags=flags, host_ring=host_ring)
    clients = []

    def add(spec, b):
        if spec[0] == "c":
            cid = g.add_client_cascade(spec[1], spec[2], spec[3], spec[4], spec[5], interp2=spec[6])
        elif spec[0] == "r":
            cid = g.add_client_rational(spec[1], spec[2], spec[3], spec[4])
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
                if c["last"] is None:
                    if c["spec"][0] == "c":
                        assert g.client_info(c["cid"])[1] == CASCADE
                        c["kinds"].add(g.cascade_info(c["cid"])[0])
                    else:
                        c["kinds"].add(g.client_info(c["cid"])[1])

    for b, x in enumerate(blocks):
        if b in (attach or {}) or b in (detach or {}):
            if b in (attach or {}):  # an attach re-lays out the arenas: collect first
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


# stage A: (D1, T1, taps1 bits), stage B: (L2, M2, T2, taps2 bits), format, max_in, forced generic; every
# partial sum is an integer number of steps below 2^24: T1 * A * M1 * ceil(T2 / L2) * M2 <= 2^24
EXACT = {
    "generic_l2": (6, 17, 3, 2, 7, 85, 2, "cu8", 8192, True),
    "tiled_l3": (6, 17, 3, 3, 7, 85, 2, "cu8", 8192, False),
    "tiled_l12": (6, 17, 3, 12, 5, 120, 2, "cu8", 8192, False),
    "tiled_gcd2": (6, 17, 3, 4, 6, 50, 2, "cu8", 8192, False),
    "long_l3": (400, 800, 1, 3, 4, 21, 3, "cs16", 65536, False),
}


@pytest.mark.parametrize("case", list(EXACT))
def test_exact_against_float64_composition(pkg, case):
    d1, T1, b1, L2, M2, T2, b2, fmt, max_in, generic = EXACT[case]
    amax = {"cu8": 255, "cs16": 128}[fmt]
    assert T1 * amax * (2 ** b1 - 1) * -(-T2 // L2) * (2 ** b2 - 1) <= 2 ** 24
    rng = np.random.default_rng(len(case) + L2)
    fs = 2016000
    specs = [("c", d1, small_taps(rng, T1, b1), 0, M2, small_taps(rng, T2, b2), L2) for _ in range(8)]
    sizes = [max_in, max_in, 1001, max_in, 7, 0, max_in - 2, 2 * d1 * T2 + 1] + [max_in] * 8 + [333] * 8
    blocks = [exact_input(rng, fmt, n) for n in sizes]
    clients = run_group(pkg, fs, max_in, fmt, specs, blocks, flags=pkg.XLG_FORCE_GENERIC if generic else 0,
                        depth=SLOTS)
    want_kind = GENERIC if generic else (LONG if case.startswith("long") else TILED)
    cin = [to_complex(fmt, x) for x in blocks]
    for c in clients:
        assert want_kind in c["kinds"] and c["kinds"] <= {GENERIC, want_kind}, c["kinds"]
        _, _, t1, _, _, t2, _ = c["spec"]
        ref = f64_composition(d1, t1, L2, M2, t2, fs, cin)
        for b, (y, r) in enumerate(zip(c["got"], ref)):
            assert np.array_equal(r.astype(np.complex64).astype(np.complex128), r)  # exact stimuli
            assert y.shape == r.shape, (case, b)
            assert np.array_equal(y, r.astype(np.complex64)), (case, b, np.max(np.abs(y - r)))


@pytest.mark.parametrize("l2,m2", [(3, 7), (4, 10)])
def test_any_centre_single_tap_is_the_integer_client(pkg, l2, m2):
    """Stage B with one nonzero tap 0.5 at reversed position j: output k is 0.5 * y[(w_k + j) / L2] where L2
    divides w_k + j (w_k = k * M2 - (T2 - 1), the upsampled window start) and 0 elsewhere, y being the outputs
    of the group's own integer client (D1, taps1, centre) and zero before the attach.  Five centres, 300+
    blocks, bit for bit."""
    fs, fmt, max_in, d1, rate = 2016000, "cu8", 4096, 6, 48000
    taps1 = pkg.create_low_pass_filter(1.0, fs, rate // 2, rate // 5)
    T2 = 24
    centres = [0, -312000, 17, 251001, -1000003]
    specs = []
    for i, ce in enumerate(centres):
        t2 = np.zeros(T2, np.float32)
        t2[(7 * i + 3) % T2] = 0.5
        specs += [("c", d1, taps1, ce, m2, t2, l2), ("i", d1, taps1, ce)]
    rng = np.random.default_rng(11 + l2)
    sizes = [int(v) * 2 for v in rng.integers(max_in // 8, max_in // 2 + 1, 310)]
    sizes[5] = 0
    sizes[9] = 2
    blocks = [rand_block(rng, fmt, n) for n in sizes]
    clients = run_group(pkg, fs, max_in, fmt, specs, blocks, depth=SLOTS)
    for c, ci in zip(clients[0::2], clients[1::2]):
        assert c["kinds"] == ci["kinds"] and TILED in c["kinds"]
        j = int(np.flatnonzero(reversed_taps(c["spec"][5]))[0])
        y = np.concatenate(ci["got"])
        z = np.concatenate(c["got"])
        u = np.arange(z.size) * m2 - (T2 - 1) + j
        hit = (u % l2 == 0) & (u >= 0)
        idx = np.where(hit, u // l2, 0)
        assert idx.max() < y.size
        want_z = np.where(hit, y[idx] * np.float32(0.5), 0).astype(np.complex64)
        assert np.array_equal(z, want_z), c["spec"][3]


def contract(pkg, fs, rate, fmt, n_clients, max_in, sizes, seed, **kw):
    plan = pkg.cascade_plan(fs, [rate] * n_clients)
    assert all(p["interp2"] > 1 for p in plan)

    def spec(p):
        return ("c", p["d1"], p["taps1"], p["center"], p["d2"], p["taps2"], p["interp2"])

    specs = [spec(p) for p in plan]
    rng = np.random.default_rng(seed)
    blocks = [rand_block(rng, fmt, n) for n in sizes]
    attach = kw.pop("attach_plan", None)
    if attach is not None:
        kw["attach"] = {b: [spec(p) for p in pkg.cascade_plan(fs, [rate] * n)] for b, n in attach.items()}
    clients = run_group(pkg, fs, max_in, fmt, specs, blocks, **kw)
    oracles = [RationalCascadeOracle(s[1], s[2], s[3], s[6], s[4], s[5], fs, max_in)
               for s in (c["spec"] for c in clients)]
    outs = [oracle_stream([o], fmt, blocks[c["first"]:c["last"]])[0] for o, c in zip(oracles, clients)]
    for c, ref in zip(clients, outs):
        assert len(c["got"]) == len(ref)
        assert [y.size for y in c["got"]] == [y.size for y in ref]
        assert_cf32_close(np.concatenate(c["got"]), np.concatenate(ref), f"client {c['cid']} from block {c['first']}")
    return clients


def test_contract_10M_cs16(pkg):
    """10 Msps cs16, 8 clients at 48 kHz: 20 x 12/125, taps 55 / 1505."""
    max_in = 65536
    sizes = [max_in if b % 7 else 30002 for b in range(100)]
    clients = contract(pkg, 10000000, 48000, "cs16", 8, max_in, sizes, 1, depth=SLOTS)
    assert all(TILED in c["kinds"] for c in clients)


def test_contract_20M_cs8(pkg):
    """20 Msps cs8, 8 clients at 48 kHz: 25 x 3/50, taps 65 / 603, ragged and odd blocks."""
    max_in = 65536
    rng = np.random.default_rng(2)
    sizes = [max_in if b % 3 else int(v) for b, v in enumerate(rng.integers(0, max_in + 1, 100))]
    contract(pkg, 20000000, 48000, "cs8", 8, max_in, sizes, 2, depth=SLOTS)


def test_contract_2M_history_spans_blocks_ring_wraps(pkg):
    """2.048 Msps cu8 (8 x 3/16, taps 25 / 193) in blocks so small that a block's stage-A samples are fewer
    than stage B's history, XLG_SLOTS tickets in flight: the rings wrap many times."""
    max_in = 256
    rng = np.random.default_rng(3)
    sizes = [int(v) for v in rng.integers(0, max_in + 1, 320)]
    clients = contract(pkg, 2048000, 48000, "cu8", 3, max_in, sizes, 3, depth=SLOTS)
    assert all(c["kinds"] == {GENERIC} for c in clients)


def test_contract_attach_and_remove_in_flight(pkg):
    max_in = 16384
    rng = np.random.default_rng(4)
    sizes = [int(v) for v in rng.integers(1, max_in + 1, 200)]
    clients = contract(pkg, 2048000, 48000, "cu8", 9, max_in, sizes, 4, depth=SLOTS, attach_plan={67: 8, 120: 2},
                       detach={100: [0, 2, 4], 141: [10]})
    assert {len(c["got"]) for c in clients[:9]} == {100, 200}


@pytest.mark.parametrize("mode", ["out_device", "host_ring"])
def test_contract_out_device_and_host_ring(pkg, mode):
    max_in = 32768
    rng = np.random.default_rng(5)
    sizes = [int(v) for v in rng.integers(max_in // 2, max_in + 1, 120)]
    if mode == "out_device":
        contract(pkg, 2048000, 48000, "cu8", 8, max_in, sizes, 5, flags=pkg.XLG_OUT_DEVICE, depth=SLOTS)
    else:
        contract(pkg, 2048000, 48000, "cu8", 8, max_in, sizes, 6, host_ring=16, depth=12)


def test_neighbours_unchanged_by_rational_cascade_clients(pkg):
    """Integer, rational and integer-cascade clients give the same bits with and without rational cascade
    clients in the group; the rational cascade clients meet the contract, and the result copy to the host ends
    at the last host-visible row."""
    fs, max_in, fmt = 2048000, 65536, "cu8"
    ints = [(64, pkg.create_low_pass_filter(1.0, fs, p["cutoff"], p["tw"]), p["center"])
            for p in pkg.client_plan(fs, [32000] * 8)]
    ints += [(32, pkg.create_low_pass_filter(1.0, fs, 32000, 12800), c) for c in (-500000, 400000)]
    rats = pkg.rational_plan(fs, [48000] * 8 + [96000] * 2)
    icas = pkg.cascade_plan(fs, [32000] * 4)
    rcas = pkg.cascade_plan(fs, [48000] * 8)
    rng = np.random.default_rng(7)
    blocks = [rand_block(rng, fmt, max_in if b % 4 else 30001) for b in range(40)]
    res = []
    for with_rational_cascade in (True, False):
        g = pkg.Group(fs, max_in)
        ids = [g.add_client(d, t, c) for d, t, c in ints]
        ids += [g.add_client_rational(p["interp"], p["decim"], p["taps"], p["center"]) for p in rats]
        ids += [g.add_client_cascade(p["d1"], p["taps1"], p["center"], p["d2"], p["taps2"]) for p in icas]
        cids = [g.add_client_cascade(p["d1"], p["taps1"], p["center"], p["d2"], p["taps2"], interp2=p["interp2"])
                for p in rcas] if with_rational_cascade else []
        g.profile_enable(True)
        outs, couts, d2h = [], [], []
        for x in blocks:
            t = g.submit(fmt, x)
            g.wait(t)
            outs.append([g.output(t, c) for c in ids])
            couts.append([g.output(t, c) for c in cids])
            ptrs = [g.output_ptr(t, c) for c in ids + cids]
            base = min(p for p, _ in ptrs)
            d2h.append((g.cascade_profile_read()["d2h_bytes"], max((p - base) + 8 * n for p, n in ptrs)))
        kinds = {g.client_info(c)[1] for c in ids}
        g.close()
        res.append((outs, couts, kinds, d2h))
    assert res[0][2] == res[1][2] and {0, 1, 3, 4, 5} <= res[0][2]
    for a, b in zip(res[0][0], res[1][0]):
        for ya, yb in zip(a, b):
            assert np.array_equal(ya.view(np.uint64), yb.view(np.uint64))
    for got_bytes, extent in res[0][3]:
        assert got_bytes == extent
    for i, p in enumerate(rcas):
        o = RationalCascadeOracle(p["d1"], p["taps1"], p["center"], p["interp2"], p["d2"], p["taps2"], fs, max_in)
        ref = [o.process_cf32(fmt, x) for x in blocks]
        assert_cf32_close(np.concatenate([c[i] for c in res[0][1]]), np.concatenate(ref), f"cascade {i}")


def test_interp2_one_is_the_integer_cascade(pkg):
    """interp2 = 1 through the rational entry point is xlg_add_client_cascade, bit for bit; stage_b_macs counts
    n2 * ceil(T2 / L2) for the rational clients and n2 * T2 for the integer ones."""
    fs, max_in, fmt = 2016000, 16384, "cu8"
    p = pkg.cascade_plan(fs, [48000])[0]
    q = pkg.cascade_plan(2048000, [48000])[0]
    rng = np.random.default_rng(9)
    blocks = [rand_block(rng, fmt, n) for n in [max_in] * 20 + [7, 0, 333] * 4]
    g = pkg.Group(fs, max_in)
    a = g.add_client_cascade(p["d1"], p["taps1"], p["center"], p["d2"], p["taps2"], interp2=1)
    t1, t2 = (np.ascontiguousarray(t, dtype=np.float32) for t in (p["taps1"], p["taps2"]))
    fp, cid = C.POINTER(C.c_float), C.c_int(-1)
    assert g._L.xlg_add_client_cascade(g._h, p["d1"], t1.ctypes.data_as(fp), t1.size, p["center"], p["d2"],
                                       t2.ctypes.data_as(fp), t2.size, C.byref(cid)) == 0
    r = g.add_client_cascade(q["d1"], q["taps1"], 0, q["d2"], q["taps2"], interp2=q["interp2"])
    g.profile_enable(True)
    g.cascade_profile_read(reset=True)
    macs = 0
    for x in blocks:
        t = g.submit(fmt, x)
        g.wait(t)
        ya, yb = g.output(t, a), g.output(t, cid.value)
        assert np.array_equal(ya.view(np.uint64), yb.view(np.uint64))
        macs += 2 * ya.size * p["taps2"].size + g.output(t, r).size * -(-q["taps2"].size // q["interp2"])
    prof = g.cascade_profile_read()
    g.close()
    assert prof["stage_b_macs"] == macs and prof["stage_b_launches"] == len(blocks)


def test_refusals(pkg, capfd):
    """-EINVAL for interp2 = 0, an upsampled block of 2^31 stage-A samples or more and branches too long for
    the stage-B kernel; -ENOTSUP on an XLG_TRACK_STATE group and for a Q15 submit: each logged, nothing
    enqueued, and the next cf32 submit carries on as if the refused calls had not happened."""
    fs, max_in, fmt = 2048000, 16384, "cu8"
    p = pkg.cascade_plan(fs, [48000])[0]
    t1, t2, d1, l2, m2 = p["taps1"], p["taps2"], p["d1"], p["interp2"], p["d2"]
    rng = np.random.default_rng(8)
    blocks = [rand_block(rng, fmt, max_in) for _ in range(6)]
    g = pkg.Group(fs, max_in)
    twin = pkg.Group(fs, max_in)
    huge = np.full(120001, 1e-3, np.float32)
    for args in ((d1, t1, 0, m2, t2, 0), (d1, t1, 0, 0, t2, l2), (1, t1, 0, m2, t2, 2 ** 19),
                 (d1, t1, 0, m2, huge, 2)):
        with pytest.raises(ValueError) as e:
            g.add_client_cascade(*args[:5], interp2=args[5])
        assert e.value.args[0] == -errno.EINVAL, args[5]
        assert "<3>" in capfd.readouterr().err
    tg = pkg.Group(fs, max_in, flags=pkg.XLG_TRACK_STATE)
    with pytest.raises(ValueError) as e:
        tg.add_client_cascade(d1, t1, 0, m2, t2, interp2=l2)
    assert e.value.args[0] == -errno.ENOTSUP and tg.client_count() == 0
    assert "<3>" in capfd.readouterr().err
    tg.close()
    ids = [grp.add_client_cascade(d1, t1, p["center"], m2, t2, interp2=l2) for grp in (g, twin)]
    assert g.client_count() == 1 and g.client_info(ids[0])[1] == CASCADE
    assert g.cascade_info(ids[0])[2] == t2.size - 1
    got, want = [], []
    for b, x in enumerate(blocks):
        if b in (1, 4):
            with pytest.raises(RuntimeError) as e:
                g.submit(fmt, x, flags=pkg.XLG_PATH_Q15)
            assert str(-errno.ENOTSUP) in str(e.value)
            assert "<3>" in capfd.readouterr().err
        t, tt = g.submit(fmt, x), twin.submit(fmt, x)
        assert t == tt == b
        g.wait(t)
        twin.wait(tt)
        got.append(g.output(t, ids[0]))
        want.append(twin.output(tt, ids[1]))
    g.close()
    twin.close()
    for a, b in zip(got, want):
        assert a.size > 0 and np.array_equal(a.view(np.uint64), b.view(np.uint64))
