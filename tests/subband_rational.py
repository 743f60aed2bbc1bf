"""Checker of the rational sub-band member tests (include/xlating_group.h, xlg_add_client_subband_rational):
SubbandOracle whose members may resample.  No GPU."""
from cascade import FloatPath
from cascade_rational import stuff
from subband import SubbandOracle


class RationalSubbandOracle(SubbandOracle):
    """SubbandOracle whose member (d2, taps2, offset, interp2) is FloatPath (d2, taps2, offset) at
    interp2 * fs // d1 fed the sub-band's cf32 outputs zero-stuffed by interp2 (u[interp2*n] = y[n]), from the
    block it was attached before.  interp2 = 1 is SubbandOracle's member."""

    def __init__(self, d1, taps1, center_freq, fs, max_input_len):
        super().__init__(d1, taps1, center_freq, fs, max_input_len)
        self.interp = {}  # member key -> interp2

    def add_member(self, key, d2, taps2, offset, interp2=1):
        self.members[key] = FloatPath(d2, taps2, offset, interp2 * self.fs1)
        self.interp[key] = interp2

    def remove_member(self, key):
        super().remove_member(key)
        del self.interp[key]

    def process_cf32(self, fmt, data, renorm=True):
        """Feeds one block; returns {member key: its cf32 outputs of the block}."""
        y = self.a.process_cf32(fmt, data, renorm=renorm)
        self.rows.append(y)
        return {k: m.process_cf32(stuff(y, self.interp[k]) if self.interp[k] > 1 else y, renorm=renorm)
                for k, m in self.members.items()}
