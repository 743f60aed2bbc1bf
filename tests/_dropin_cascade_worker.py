"""Worker for tests/test_gpu_dropin_cascade.py: cascade (two-stage) filters of the per-filter drop-in ABI
(create_cascade_frequency_xlating_filter).  Runs in a subprocess because the engine reads its environment
switches (XLATING_B200_STREAM, _OSC, _DROPIN, _LANES, _SHARE) once per process.

usage: _dropin_cascade_worker.py <scenario> [arg]   -> one JSON line, exit code 1 on any error

  exact                   exact stimuli in all three formats over ragged calls that wrap the stage-A ring:
                          integer cascades (odd and even D2), L2 = 2, 3, 12 and gcd(L2, M2) > 1; every output
                          equal to the float64 composition bit for bit
  designed <dir> [lone]   cascade_plan's filters at 2.016, 2.048, 10, 20 and 61.44 Msps, one thread per filter
                          next to integer (cf32 and Q15) and rational filters of the same bands, all meeting at
                          a barrier every call: output counts of the composed oracle and 1e-5 against it, and
                          the bits of the same clients in a Group(flags=XLG_FORCE_GENERIC) fed the same blocks
                          (skipped under XLATING_B200_DROPIN=group); cascade outputs saved to <dir>; lone: one
                          filter alive at a time
  neighbours              overlay on: integer and rational filters of one band on exact stimuli give the same
                          bits with and without cascade filters alive, and still join their band's group
  q15refuse               two refused Q15 calls leave a cascade filter's cf32 stream untouched
  pool <dir> [fresh]      cascade, rational and integer filters created and destroyed interleaved (the cascade
                          arena grows and is reused, filter memory comes from the pool): every cascade filter's
                          calls saved to <dir>; fresh: one filter in a fresh process
"""
import importlib
import json
import os
import sys
import threading

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
from oracle import pyoracle as po  # noqa: E402  (checker)
from cascade import CascadeOracle, f64_filter, small_taps  # noqa: E402
from cascade_rational import RationalCascadeOracle, f64_composition  # noqa: E402
from exact import exact_input, to_complex  # noqa: E402
from rational import oracle_filter, stuff  # noqa: E402
from util import assert_cf32_close, rand_block  # noqa: E402

pkg = importlib.import_module("sdr-server_b200")
MAX_IN = 65536
# full, 30001, 2, 0, 7 and 65534 elements, then full calls that wrap every stage-A ring
RAGGED = [65536, 30001, 2, 0, 7, 65534] + [65536] * 6
GROUP_MODEL = os.environ.get("XLATING_B200_DROPIN") == "group"


def u64(y):
    return np.ascontiguousarray(y).view(np.uint64)


def same_bits(a, b, what):
    assert len(a) == len(b), f"{what}: {len(a)} calls != {len(b)}"
    for i, (x, y) in enumerate(zip(a, b)):
        assert x.shape == y.shape and np.array_equal(u64(x), u64(y)), f"{what}: call {i} differs"


def cascade(p, fs):
    return pkg.XlatingFilter.cascade(p["d1"], p["taps1"], p["center"], p["d2"], p["taps2"], fs, MAX_IN,
                                     interp2=p["interp2"])


def run_threads(workers, n_calls):
    """One thread per worker; worker(b) makes call b.  They meet at a barrier before every call."""
    errors = []
    bar = threading.Barrier(len(workers))

    def loop(w):
        try:
            for b in range(n_calls):
                bar.wait()
                w(b)
        except threading.BrokenBarrierError:
            pass
        except Exception as e:  # noqa: BLE001
            errors.append(repr(e))
            bar.abort()

    ts = [threading.Thread(target=loop, args=(w,)) for w in workers]
    for t in ts:
        t.start()
    for t in ts:
        t.join()
    assert not errors, errors[:3]


# ---- exact stimuli ----
# stage A: D1 = 6, 17 taps of 3 bits; stage B: (L2, M2, T2), taps of 2 bits.  Every partial sum is an integer
# number of grid steps below 2^24: 17 * 255 * 7 * ceil(T2 / L2) * 3 <= 2^24
EXACT_B = [(1, 7, 85), (1, 8, 64), (2, 7, 85), (3, 7, 85), (12, 5, 120), (4, 6, 50)]


def scenario_exact(out):
    rng = np.random.default_rng(5)
    fs, d1 = 2016000, 6
    fmts = ["cu8", "cs8", "cs16"]
    blocks = {f: [exact_input(rng, f, n) for n in RAGGED] for f in fmts}
    filters = []
    for L2, M2, T2 in EXACT_B:
        assert 17 * 255 * 7 * -(-T2 // L2) * 3 <= 2 ** 24
        for fmt in fmts:
            t1, t2 = small_taps(rng, 17, 3), small_taps(rng, T2, 2)
            f = pkg.XlatingFilter.cascade(d1, t1, 0, M2, t2, fs, MAX_IN, interp2=L2)
            filters.append((f, fmt, t1, t2, L2, M2, []))
    for b in range(len(RAGGED)):  # interleaved: consecutive calls of different filters
        for f, fmt, _, _, _, _, got in filters:
            got.append(f.process_cf32(fmt, blocks[fmt][b]))
    wraps = 0
    for f, fmt, t1, t2, L2, M2, got in filters:
        ref = f64_composition(d1, t1, L2, M2, t2, fs, [to_complex(fmt, x) for x in blocks[fmt]])
        for b, (y, r) in enumerate(zip(got, ref)):
            assert np.array_equal(r.astype(np.complex64).astype(np.complex128), r)  # exact stimuli
            assert y.shape == r.shape, (L2, M2, fmt, b)
            assert np.array_equal(y, r.astype(np.complex64)), (L2, M2, fmt, b)
        # the stage-A ring holds a power of two >= ceil((T2 - 1) / L2) + 1 + 5463 samples: 8192
        wraps += sum(len(to_complex(fmt, x)) for x in blocks[fmt]) // d1 > 8192
        f.close()
    out["filters"] = len(filters)
    out["ring_wraps"] = int(wraps)


# ---- designed taps ----
BANDS = [(2016000, [48000], "cu8"), (2048000, [48000, 96000], "cu8"), (10000000, [48000], "cs16"),
         (20000000, [48000], "cs8"), (61440000, [48000, 96000], "cu8")]


def scenario_designed(out, dump, lone=False):
    rng = np.random.default_rng(17)
    jobs = []  # (fs, fmt, kind, spec, blocks)
    for fs, rates, fmt in BANDS:
        blocks = [rand_block(rng, fmt, n) for n in RAGGED]
        for p in pkg.cascade_plan(fs, rates * 2):
            jobs.append((fs, fmt, "c", p, blocks))
        # neighbours of other kinds in the same batches: integer cf32, integer Q15, rational
        p = pkg.client_plan(fs, [48000])[0]
        if not lone:
            taps = pkg.create_low_pass_filter(1.0, fs, p["cutoff"], p["tw"])
            jobs.append((fs, fmt, "i", (p["decimation"], taps, p["center"]), blocks))
            jobs.append((fs, fmt, "q", (p["decimation"], taps, p["center"]), blocks))
            if fs % 48000:
                jobs.append((fs, fmt, "r", pkg.rational_plan(fs, [48000])[0], blocks))
    outs = [[] for _ in jobs]

    def make(j):
        fs, fmt, kind, p, _ = jobs[j]
        if kind == "c":
            return cascade(p, fs)
        if kind == "r":
            return pkg.XlatingFilter.rational(p["interp"], p["decim"], p["taps"], p["center"], fs, MAX_IN)
        return pkg.XlatingFilter(p[0], p[1], p[2], fs, MAX_IN)

    def call(f, j, b):
        fs, fmt, kind, _, blocks = jobs[j]
        x = blocks[b].copy()
        outs[j].append(f.process_q15(fmt, x) if kind == "q" else f.process_cf32(fmt, x))

    if lone:
        for j in range(len(jobs)):
            f = make(j)
            for b in range(len(RAGGED)):
                call(f, j, b)
            f.close()
    else:
        filters = [make(j) for j in range(len(jobs))]
        run_threads([lambda b, j=j: call(filters[j], j, b) for j in range(len(jobs))], len(RAGGED))
        for f in filters:
            f.close()
    # the composed oracle (counts, 1e-5), and the group's cascade clients on the generic kernels (bits)
    kinds = set()
    for j, (fs, fmt, kind, p, blocks) in enumerate(jobs):
        what = f"{kind} {fs} job {j}"
        if kind == "c":
            if p["interp2"] == 1:
                o = CascadeOracle(p["d1"], p["taps1"], p["center"], p["d2"], p["taps2"], fs, MAX_IN)
            else:
                o = RationalCascadeOracle(p["d1"], p["taps1"], p["center"], p["interp2"], p["d2"], p["taps2"], fs,
                                          MAX_IN)
            ref = [o.process_cf32(fmt, x) for x in blocks]
            n_c = sum(jb[2] == "c" for jb in jobs[:j])  # the same name whichever neighbours ran
            np.save(os.path.join(dump, f"c{n_c:02d}.npy"), np.concatenate(outs[j]))
        elif kind == "r":
            o = oracle_filter(po, p["interp"], p["decim"], p["taps"], p["center"], fs, MAX_IN)
            ref = [o.process_cf32("cs16", stuff(fmt, x, p["interp"])) for x in blocks]
        elif kind == "q":
            o = po.OracleFilter(p[0], p[1], p[2], fs, MAX_IN)
            for b, x in enumerate(blocks):
                assert np.array_equal(np.asarray(outs[j][b]).reshape(-1, 2), o.process_q15(fmt, x).reshape(-1, 2)), \
                    (what, b)
            continue
        else:
            o = po.OracleFilter(p[0], p[1], p[2], fs, MAX_IN)
            ref = [o.process_cf32(fmt, x) for x in blocks]
        assert [y.size for y in outs[j]] == [y.size for y in ref], what
        assert_cf32_close(np.concatenate(outs[j]), np.concatenate(ref), what)
        kinds.add(kind)
    if not GROUP_MODEL:
        for fs, _, fmt in BANDS:
            idx = [j for j, jb in enumerate(jobs) if jb[0] == fs and jb[2] == "c"]
            g = pkg.Group(fs, MAX_IN, flags=pkg.XLG_FORCE_GENERIC)
            cids = [g.add_client_cascade(p["d1"], p["taps1"], p["center"], p["d2"], p["taps2"], interp2=p["interp2"])
                    for p in (jobs[j][3] for j in idx)]
            got = {j: [] for j in idx}
            for x in jobs[idx[0]][4]:
                t = g.submit(fmt, x)
                g.wait(t)
                for j, c in zip(idx, cids):
                    got[j].append(np.array(g.output(t, c), copy=True))
            g.close()
            for j in idx:
                same_bits(outs[j], got[j], f"cascade {fs} job {j} against the group")
    if not GROUP_MODEL:
        out["batches"], out["calls"], out["shared"] = pkg.dropin_stats()
    out.update(kinds=sorted(kinds), cascades=sum(j[2] == "c" for j in jobs),
               d2_parity=sorted({(j[3]["interp2"] > 1, j[3]["d2"] % 2) for j in jobs if j[2] == "c"}))


# ---- neighbours under the overlay ----
def scenario_neighbours(out):
    rng = np.random.default_rng(23)
    fs, fmt = 2016000, "cs16"
    n_calls = 24
    blocks = [exact_input(rng, fmt, MAX_IN) for _ in range(n_calls)]
    specs = [("i", 42, small_taps(rng, 97, 3)) for _ in range(4)] + [("r", (2, 7), small_taps(rng, 120, 3))
                                                                     for _ in range(4)]
    plan = pkg.cascade_plan(fs, [48000, 96000])

    def one_run(with_cascades):
        fs_ = [pkg.XlatingFilter(s[1], s[2], 0, fs, MAX_IN) if s[0] == "i" else
               pkg.XlatingFilter.rational(s[1][0], s[1][1], s[2], 0, fs, MAX_IN) for s in specs]
        cs = [cascade(p, fs) for p in plan] if with_cascades else []
        got = [[] for _ in fs_]
        stream = {}

        def worker(i):
            def w(b):
                got[i].append(fs_[i].process_cf32(fmt, blocks[b].copy()))
            return w

        def casc_worker(c):
            return lambda b: c.process_cf32(fmt, blocks[b].copy())

        run_threads([worker(i) for i in range(len(fs_))] + [casc_worker(c) for c in cs], n_calls)
        stream = pkg.dropin_stream_stats()
        for f in fs_ + cs:
            f.close()
        return got, stream

    base, st0 = one_run(False)
    with_c, st1 = one_run(True)
    for i, (a, b) in enumerate(zip(base, with_c)):
        same_bits(a, b, f"neighbour {i} with and without cascade filters")
    for i, s in enumerate(specs):  # exact stimuli: the float64 filter, whichever engine served a call
        if s[0] == "i":
            ref = f64_filter(s[2], s[1], 0, fs, [to_complex(fmt, x) for x in blocks])
        else:
            L, M = s[1]
            ref = f64_filter(s[2], M, 0, L * fs, [to_complex("cs16", stuff(fmt, x, L)) for x in blocks])
        for b, (y, r) in enumerate(zip(base[i], ref)):
            assert y.shape == r.shape and np.array_equal(y, r.astype(np.complex64)), (i, b)
    out["stream"] = {"before": st0, "after": st1}
    out["filters"] = len(specs)


# ---- Q15 refusal ----
def scenario_q15refuse(out):
    rng = np.random.default_rng(29)
    fs, fmt = 10000000, "cs16"
    p = pkg.cascade_plan(fs, [48000])[0]
    blocks = [rand_block(rng, fmt, n) for n in RAGGED]
    a, b = cascade(p, fs), cascade(p, fs)
    ya, yb, refused = [], [], []
    for i, x in enumerate(blocks):
        if i == 2:
            refused.append(len(a.process_q15(fmt, x)))
            refused.append(len(a.process_q15("cu8", np.zeros(100, np.uint8))))
        ya.append(a.process_cf32(fmt, x))
        yb.append(b.process_cf32(fmt, x))
    same_bits(ya, yb, "cascade filter after refused Q15 calls")
    assert sum(y.size for y in ya) > 0
    a.close()
    b.close()
    out["refused"] = refused


# ---- pool and arena reuse ----
def scenario_pool(out, dump, fresh=False):
    rng = np.random.default_rng(31)
    fs, fmt = 61440000, "cu8"
    blocks = [rand_block(rng, fmt, n) for n in (65536, 30001, 65536, 65534)]
    p = pkg.cascade_plan(fs, [48000])[0]
    if fresh:
        f = cascade(p, fs)
        np.savez(os.path.join(dump, "fresh.npz"), **{f"c{b}": f.process_cf32(fmt, x) for b, x in enumerate(blocks)})
        f.close()
        return
    other = pkg.cascade_plan(2048000, [48000])[0]
    rat = pkg.rational_plan(2048000, [48000])[0]
    live = []  # [filter, calls made]
    extra = []

    def call_all(b):
        for e in live:
            if e[1] == b:
                e.append(e[0].process_cf32(fmt, blocks[b]))
                e[1] += 1

    for _ in range(30):
        live.append([cascade(p, fs), 0])
    call_all(0)
    for i in range(70):  # the cascade arena grows under filters that have already run
        live.append([cascade(p, fs), 0])
        if i % 10 == 0:
            extra.append(pkg.XlatingFilter.rational(rat["interp"], rat["decim"], rat["taps"], rat["center"], 2048000,
                                                    MAX_IN))
    call_all(0)
    call_all(1)
    for e in live[::2]:
        e[0].close()
    live = live[1::2]
    for i in range(40):  # pooled memory, arena holes: interleaved with other kinds
        if i % 3 == 0:
            extra.append(pkg.XlatingFilter(64, pkg.create_low_pass_filter(1.0, fs, 24000, 9600), 1000, fs, MAX_IN))
        if i % 4 == 0:
            c = cascade(other, 2048000)
            c.process_cf32(fmt, blocks[0])
            c.close()
        live.append([cascade(p, fs), 0])
    for b in range(len(blocks)):
        call_all(b)
    for e in extra:
        e.close()
    saved = {}
    for i, e in enumerate(live):
        e[0].close()
        saved[f"f{i}"] = np.concatenate(e[2:])
        saved[f"n{i}"] = np.array(e[1])
    np.savez(os.path.join(dump, "pool.npz"), **saved)
    out["filters"] = len(live)


def main():
    out = {"errors": []}
    try:
        sc = sys.argv[1]
        args = sys.argv[2:]
        if sc == "exact":
            scenario_exact(out)
        elif sc == "designed":
            scenario_designed(out, args[0], lone=len(args) > 1 and args[1] == "lone")
        elif sc == "neighbours":
            scenario_neighbours(out)
        elif sc == "q15refuse":
            scenario_q15refuse(out)
        elif sc == "pool":
            scenario_pool(out, args[0], fresh=len(args) > 1 and args[1] == "fresh")
        else:
            raise ValueError(sc)
    except Exception as e:  # noqa: BLE001
        import traceback
        out["errors"].append(traceback.format_exc()[-3000:])
    print(json.dumps(out, default=int))
    sys.exit(1 if out["errors"] else 0)


if __name__ == "__main__":
    main()
