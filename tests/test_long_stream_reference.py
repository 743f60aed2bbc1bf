"""The window argument of tests/long_stream.py, checked on streams short enough to reference in one shot.

For every kernel family the fresh reference fed the blocks from window_start's boundary on equals the
reference of the whole stream, block by block, on the ranges after a ragged pair of odd lengths.  A boundary
whose distance from the attach point is not a multiple of the period gives different outputs: the check the
GPU tests make can fail.  The Q15 oscillator is the exception the GPU tests work around: it is never
renormalised, so at centre 0 it decays from 32767 to 0 within 32767 outputs, and only fresh Q15 clients carry
data.  No GPU.
"""
import numpy as np
import pytest

from cascade import small_taps
from exact import assert_exact, dyadic_taps, exact_input, q15_phases, ref_q15
from long_stream import fresh_refs, history, period, window_start
from subband_rig import dyadic_member, dyadic_stage_a

FS, FMT = 2_520_000, "cs16"
NS = 840        # a small block length that every period below divides (lcm 120)
A_ODD = 301     # the ragged pair: 301 + 539 samples


def specs(rng):
    t1 = dyadic_stage_a(rng, 4, 17)
    b1, b2 = small_taps(rng, 13, 2), small_taps(rng, 19, 2)
    return {
        "int": ("int", 6, dyadic_taps(rng, 13, FMT)),
        "int_long": ("int", 8, dyadic_taps(rng, 30, FMT)),
        "rat": ("rat", 3, 8, dyadic_taps(rng, 20, FMT)),
        "casc": ("casc", 4, small_taps(rng, 9, 3), 1, 3, small_taps(rng, 7, 3)),
        "casc_rat": ("casc", 4, small_taps(rng, 9, 3), 3, 5, small_taps(rng, 13, 3)),
        "sub": ("sub", 4, t1, 1, 3, dyadic_member(rng, t1, 7, FMT)),
        "sub_rat": ("sub", 4, t1, 2, 5, dyadic_member(rng, t1, 11, FMT)),
        "bank_k6": ("bank", 3, b1, 1, 2, small_taps(rng, 5, 3)),  # K = 6: not a power of two
        "bank_k8": ("bank", 4, b2, -3, 3, small_taps(rng, 7, 3)),
    }


def stream(rng, n_blocks, pair_at):
    """Raw blocks of NS samples, the one at pair_at replaced by a ragged pair; and their start positions."""
    sizes = [NS] * n_blocks
    sizes[pair_at:pair_at + 1] = [A_ODD, NS - A_ODD]
    blocks = [exact_input(rng, FMT, 2 * n) for n in sizes]
    return blocks, list(np.concatenate([[0], np.cumsum(sizes)]).astype(int))


def test_block_length_is_a_multiple_of_every_period():
    for s in specs(np.random.default_rng(0)).values():
        assert NS % period(s) == 0, s[0]


@pytest.mark.parametrize("name", list(specs(np.random.default_rng(0))))
@pytest.mark.parametrize("attach_block", [0, 3])
def test_window_equals_whole_stream(name, attach_block):
    """A client attached before block attach_block; the ranges after the ragged pair (its second half, whose
    windows straddle its boundary at an odd position) and the last blocks."""
    rng = np.random.default_rng(10 + attach_block)
    spec = specs(rng)[name]
    blocks, starts = stream(rng, 12, 6)
    attach = starts[attach_block]
    whole = fresh_refs([spec], FMT, FS, blocks[attach_block:])[0]
    for c0, c1 in ((7, 9), (8, 11), (11, 13)):
        b = window_start(starts, c0, attach, period(spec), history(spec))
        assert (starts[b] - attach) % period(spec) == 0 and b < c0
        win = fresh_refs([spec], FMT, FS, blocks[b:c1])[0][c0 - b:]
        assert_exact(win, whole[c0 - attach_block:c1 - attach_block], f"{name}: window from block {b} for {c0}..{c1}")


@pytest.mark.parametrize("name", list(specs(np.random.default_rng(0))))
def test_misaligned_boundary_differs(name):
    """Negative control: the boundary inside the ragged pair, an odd distance from the attach point (not a
    multiple of any period here), gives other outputs on the same range."""
    rng = np.random.default_rng(20)
    spec = specs(rng)[name]
    blocks, starts = stream(rng, 12, 6)
    assert (starts[7] - starts[0]) % period(spec) != 0
    whole = fresh_refs([spec], FMT, FS, blocks)[0]
    win = fresh_refs([spec], FMT, FS, blocks[7:11])[0]
    with pytest.raises(AssertionError, match="outputs differ|output shape"):
        assert_exact(win[1:], whole[8:11], name)


def test_q15_oscillator_decays_to_zero():
    """The Q15 oscillator at centre 0 is 32767 - k at output k and 0 from output 32767 on: a Q15 client that
    has run for 32767 outputs returns zeros, whatever its windows read, so the Q15 tests check old clients'
    output counts and fresh clients' data."""
    ph = q15_phases(32770)
    assert list(ph[:3, 0]) == [32767, 32766, 32765]
    assert np.all(ph[32767:] == 0) and ph[32766, 0] == 1
    rng = np.random.default_rng(30)
    taps = dyadic_taps(rng, 9, FMT, k=15)
    blocks = [exact_input(rng, FMT, 2 * NS) for _ in range(3)]
    y = ref_q15(taps, 1, FMT, blocks)
    assert [len(v) for v in y] == [NS] * 3 and np.any(y[0] != 0)
