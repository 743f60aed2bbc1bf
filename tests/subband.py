"""Checker of the sub-band tests: a sub-band (include/xlating_group.h, xlg_add_subband) and its members as
reference filters called block by block.  No GPU."""
from cascade import FloatPath
from oracle import pyoracle as po


class SubbandOracle:
    """The sub-band = the oracle filter (d1, taps1, center) at fs fed the block; each member = FloatPath
    (d2, taps2, offset) at fs // d1 fed the sub-band's cf32 outputs of the blocks from the one it was attached
    before (add_member before that block's process_cf32)."""

    def __init__(self, d1, taps1, center_freq, fs, max_input_len):
        self.a = po.OracleFilter(d1, taps1, center_freq, fs, max_input_len)
        self.fs1 = fs // d1
        self.members = {}
        self.rows = []  # the sub-band's outputs, block by block

    def add_member(self, key, d2, taps2, offset):
        self.members[key] = FloatPath(d2, taps2, offset, self.fs1)

    def remove_member(self, key):
        del self.members[key]

    def process_cf32(self, fmt, data, renorm=True):
        """Feeds one block; returns {member key: its cf32 outputs of the block}."""
        y = self.a.process_cf32(fmt, data, renorm=renorm)
        self.rows.append(y)
        return {k: m.process_cf32(y, renorm=renorm) for k, m in self.members.items()}
