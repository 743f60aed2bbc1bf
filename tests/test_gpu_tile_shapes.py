"""Every thread tile of the tiled kernel computes the same outputs, bit for bit.

The host picks the tile shape (RK outputs x 8 clients per thread, OS sets of warps that each
take 16 * RK outputs) from the client count and the block length; XLATING_B200_TILE pins it.  Every shape forms
the same products and adds them in the same order per accumulator, so the shapes must agree
exactly with each other, and with the oracle within the float tolerance.  The clients cover
the natural input layout (D = 42 and 21), the skewed layout (D = 8), ragged block lengths,
and a class whose members attached at different stream positions (per-subgroup window
offsets inside one CTA).
"""
import numpy as np
import pytest

from oracle import pyoracle as po
from util import assert_cf32_close, rand_block

pytestmark = pytest.mark.gpu

FS, MAX_IN = 2016000, 65536
BLOCKS = [65536, 65536, 30000, 65536, 12346, 65536]
LATE_AFTER = 1  # clients of the second wave attach after this block


def run_shape(pkg, monkeypatch, shape):
    """Every client's output of every block with the tile shape pinned to `shape`."""
    monkeypatch.setenv("XLATING_B200_TILE", shape)
    rng = np.random.default_rng(29)
    early = pkg.client_plan(FS, [48000 if c % 2 == 0 else 96000 for c in range(48)])
    early += pkg.client_plan(FS, [252000] * 8)
    late = pkg.client_plan(FS, [48000] * 16)  # same (D, T) as the early 48 ksps clients, another alignment
    g = pkg.Group(FS, MAX_IN)
    clients = []  # (id, oracle)

    def attach(plan):
        for p in plan:
            taps = pkg.create_low_pass_filter(1.0, FS, p["cutoff"], p["tw"])
            clients.append((g.add_client(p["decimation"], taps, p["center"]),
                            po.OracleFilter(p["decimation"], taps, p["center"], FS, MAX_IN)))

    attach(early)
    outs, kinds = [], set()
    for blk, n in enumerate(BLOCKS):
        x = rand_block(rng, "cu8", n)
        t = g.submit("cu8", x)
        g.wait(t)
        got = {}
        for cid, o in clients:
            y = g.output(t, cid)
            assert_cf32_close(y, o.process_cf32("cu8", x), f"shape {shape} block {blk} client {cid}")
            got[cid] = np.array(y, copy=True)
            kinds.add(g.client_info(cid)[1])
        outs.append(got)
        if blk == LATE_AFTER:
            attach(late)
    g.close()
    assert 1 in kinds  # the tiled kernel ran
    return outs


@pytest.mark.parametrize("shape", ["1641", "1621", "1611"])
def test_tile_shapes_bit_identical(pkg, monkeypatch, shape):
    ref = run_shape(pkg, monkeypatch, "1642")
    got = run_shape(pkg, monkeypatch, shape)
    for blk, (a, b) in enumerate(zip(ref, got)):
        assert a.keys() == b.keys()
        for cid in a:
            assert np.array_equal(a[cid].view(np.uint32), b[cid].view(np.uint32)), (shape, blk, cid)
