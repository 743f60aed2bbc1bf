"""The hand-over stimuli see hand-over mistakes: a CPU check, before the GPU tests rely on them.

A client handed from one engine to another carries its state: the history offset and the samples
its next window reaches back to (zero before it was attached), and the oscillator.  Here the strict
oracle plays both engines: one oracle runs up to the cut, a second one is given its state
(OracleFilter.set_state) and runs on.  Given the right state it equals the uninterrupted oracle bit
for bit; given each mistake below it does not, on the specs, centres and stimuli of
tests/test_gpu_handover.py and the drop-in phase scenarios:

* the phase one ulp off, one output behind, not renormalised at the hand-over, or renormalised once
  more after a call without outputs (one-hot taps at nonzero centres; a later rounding can absorb
  some of these at some hand-overs, see test_phase_mistakes_change_later_outputs);
* the history offset one sample off, or one sample too many of real history before the attach point
  (dyadic taps at centre 0).

A rational client is the integer filter at L * fs fed the zero-stuffed stream (tests/rational.py), so
the same model serves it with the state in upsampled samples.
"""
import numpy as np
import pytest

from exact import assert_exact, dyadic_taps, one_hot_taps, oracle_phases, oscillator_increment, to_complex
from oracle import pyoracle as po
from rational import branch_one_hot_taps, oracle_filter, real_grid_input, stuff

FS, MAX_IN = 2016000, 16384
SPECS = [(1, 42, 505), (1, 21, 253), (1, 8, 64), (3, 128, 385)]  # (L, M, T)
CENTRES = [-987654, -312000, 1, 400123]
SIZES = [16384, 7001, 2, 16384, 0, 3, 16384, 12345, 2, 16384, 16384]
PHASE_MUTATIONS = ["phase_ulp", "phase_behind", "no_renorm", "renorm_no_outputs"]
HISTORY_MUTATIONS = ["hist_plus_one", "hist_minus_one", "valid_history_plus_one"]


def handover(spec, taps, center, blocks, attach, cut, mutation=None):
    """A client created before block `attach` and handed over before block `cut`: (outputs after the cut of
    the handed-over oracle, of the uninterrupted one; outputs of the uninterrupted one before the cut)."""
    L, M, T = spec
    fed = [stuff("cs16", b, L) for b in blocks[attach:]]
    k = cut - attach
    whole = oracle_filter(po, L, M, taps, center, FS, MAX_IN)
    want = [whole.process_cf32("cs16", u) for u in fed]
    src = oracle_filter(po, L, M, taps, center, FS, MAX_IN)
    for i, u in enumerate(fed[:k]):
        src.process_cf32("cs16", u, renorm=not (mutation == "no_renorm" and i == k - 1))
    hist, ph = src.history, complex(np.complex64(src.phase))
    # what the client's next window can reach: its own samples, zeros before the attach point
    before = np.concatenate([to_complex("cs16", u) for u in [stuff("cs16", b, L) for b in blocks[:attach]]] +
                            [np.zeros(0)])
    own = np.concatenate([to_complex("cs16", u) for u in fed[:k]] + [np.zeros(0)])
    if mutation == "valid_history_plus_one":  # one more input sample (L upsampled ones) of real history
        assert before.size >= L
        pad = np.concatenate([np.zeros(T + 1), before[-L:]])
    else:
        pad = np.zeros(T + 1 + L)
    x = np.concatenate([pad, own])
    if mutation == "hist_plus_one":
        hist += 1
    elif mutation == "hist_minus_one":
        hist -= 1
    f32 = np.float32
    if mutation == "phase_ulp":  # in the larger component: an ulp of the smaller one can round away
        if abs(ph.real) >= abs(ph.imag):
            ph = complex(np.nextafter(f32(ph.real), f32(np.inf)), ph.imag)
        else:
            ph = complex(ph.real, np.nextafter(f32(ph.imag), f32(np.inf)))
    elif mutation == "phase_behind":
        counts = [len(y) for y in want[:k]]
        assert sum(counts) > 0
        ph = oracle_phases(oscillator_increment(M, center, L * FS), counts)[-1]
    elif mutation == "renorm_no_outputs":
        assert len(want[k - 1]) == 0, "the hand-over must follow a call without outputs"
        mag = f32(np.sqrt(np.float64(f32(ph.real)) ** 2 + np.float64(f32(ph.imag)) ** 2))
        ph = complex(f32(f32(ph.real) / mag), f32(f32(ph.imag) / mag))
    dst = oracle_filter(po, L, M, taps, center, FS, MAX_IN)
    dst.set_state(x[x.size - hist:], ph)
    got = [dst.process_cf32("cs16", u) for u in fed[k:]]
    return got, want[k:], want[:k]


def stimuli(spec, center, seed):
    L, M, T = spec
    rng = np.random.default_rng(seed)
    blocks = [real_grid_input(rng, n) for n in SIZES]
    if center == 0:
        return dyadic_taps(rng, T, "cs16"), blocks
    taps = one_hot_taps(T, T - 1, 0.75) if L == 1 else branch_one_hot_taps(rng, T, L)
    return taps, blocks


# hand-over points: after long, odd and 1-sample calls; (attach, cut) with the client attached mid-stream
CUTS = [(0, 2), (0, 3), (0, 5), (0, 9), (1, 3), (3, 6), (2, 3), (4, 6), (8, 9)]


@pytest.mark.parametrize("spec", SPECS, ids=[f"L{s[0]}M{s[1]}T{s[2]}" for s in SPECS])
def test_right_state_continues_bit_for_bit(spec):
    for center in CENTRES + [0]:
        taps, blocks = stimuli(spec, center, spec[2])
        for attach, cut in CUTS:
            got, want, _ = handover(spec, taps, center, blocks, attach, cut)
            assert sum(len(y) for y in want) > 0
            assert_exact(got, want, f"{spec} centre {center} attach {attach} cut {cut}")


@pytest.mark.parametrize("mutation", PHASE_MUTATIONS)
@pytest.mark.parametrize("spec", SPECS, ids=[f"L{s[0]}M{s[1]}T{s[2]}" for s in SPECS])
def test_phase_mistakes_change_later_outputs(spec, mutation):
    """A later rounding can absorb a phase mistake (an ulp that the next step rounds away, a renormalisation
    that divides by a magnitude already rounding to 1), so not every hand-over shows every mistake: each
    centre must show it at some hand-over, and renormalising an already renormalised phase again must show
    at some centre."""
    seen = {}
    for center in CENTRES:
        taps, blocks = stimuli(spec, center, spec[2])
        seen[center] = 0
        for attach, cut in CUTS:
            good, _, before = handover(spec, taps, center, blocks, attach, cut)
            if mutation == "renorm_no_outputs" and len(before[-1]) > 0:
                continue  # renormalised by the call itself
            if mutation == "phase_behind" and sum(len(y) for y in before) == 0:
                continue  # no output yet: no step to be behind by
            bad, _, _ = handover(spec, taps, center, blocks, attach, cut, mutation)
            seen[center] += any(not np.array_equal(a.view(np.uint64), b.view(np.uint64)) for a, b in zip(bad, good))
    if mutation == "renorm_no_outputs":
        assert sum(seen.values()) > 0, seen
    else:
        assert all(seen.values()), seen


@pytest.mark.parametrize("mutation", HISTORY_MUTATIONS)
@pytest.mark.parametrize("spec", SPECS, ids=[f"L{s[0]}M{s[1]}T{s[2]}" for s in SPECS])
def test_history_mistakes_change_later_outputs(spec, mutation):
    taps, blocks = stimuli(spec, 0, spec[2])
    checked = 0
    for attach, cut in CUTS:
        if mutation == "valid_history_plus_one" and attach == 0:
            continue  # nothing came before the attach point
        _, want, _ = handover(spec, taps, 0, blocks, attach, cut)
        own = sum(np.asarray(b).size // 2 for b in blocks[attach:cut]) * spec[0]
        if mutation == "valid_history_plus_one" and own >= spec[2] - 1:
            continue  # the next window no longer reaches back to the attach point
        bad, _, _ = handover(spec, taps, 0, blocks, attach, cut, mutation)
        with pytest.raises(AssertionError, match="outputs differ|output shape"):
            assert_exact(bad, want, f"{mutation} attach {attach} cut {cut}")
        checked += 1
    assert checked >= 3
