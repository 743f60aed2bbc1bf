"""Helpers of the rational cascade-client tests (xlg_add_client_cascade_rational): the composed oracle and its
float64 counterpart, both built on tests/cascade.py.  No GPU."""
import numpy as np

from cascade import FloatPath, f64_filter
from oracle import pyoracle as po


def stuff(y, L):
    """The zero-stuffed stream u[L*n] = y[n], u[m] = 0 otherwise, of one block."""
    u = np.zeros(len(y) * L, dtype=np.asarray(y).dtype)
    u[::L] = y
    return u


class RationalCascadeOracle:
    """A rational cascade client as two reference filters called block by block: stage A = the oracle filter
    (d1, taps1, center) at fs fed the block, stage B = FloatPath(d2, taps2, centre 0) at l2 * fs / d1 fed the
    zero-stuffed stage-A output of the same block."""

    def __init__(self, d1, taps1, center_freq, l2, d2, taps2, fs, max_input_len):
        self.a = po.OracleFilter(d1, taps1, center_freq, fs, max_input_len)
        self.l2 = l2
        self.b = FloatPath(d2, taps2, 0, l2 * (fs // d1))

    def process_cf32(self, fmt, data, renorm=True):
        return self.b.process_cf32(stuff(self.a.process_cf32(fmt, data, renorm=renorm), self.l2), renorm=renorm)


def f64_composition(d1, taps1, l2, d2, taps2, fs, blocks):
    """Both stages in float64 at centre 0, fed complex blocks; one complex128 array per block."""
    a = f64_filter(taps1, d1, 0, fs, blocks)
    return f64_filter(taps2, d2, 0, l2 * (fs // d1), [stuff(y, l2) for y in a])
