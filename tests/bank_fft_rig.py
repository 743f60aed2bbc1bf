"""subband_rig.Rig with FFT banks (xlg_add_bank_fft): their channels' members are checked against
bank_fft_model's rows chained into the member kernels (tests/bank_fft_exact.py), direct banks' as before."""
import numpy as np

import subband_rig
from bank_exact import bank_model
from bank_fft_exact import bank_fft_model
from subband_rig import Bank, Rig

FFT_BANK = 8  # xlg_subband_info kind of an FFT bank channel


class FftRig(Rig):
    def __init__(self, pkg, monkeypatch, *args, **kwargs):
        super().__init__(pkg, monkeypatch, *args, **kwargs)
        self.fft_taps = set()  # id() of the FFT banks' taps arrays: the rig's row model tells the kernels apart by it
        monkeypatch.setattr(subband_rig, "bank_model", self._bank_model)

    def add_bank_fft(self, d1, taps1):
        bk = Bank(self.g.add_bank_fft(d1, taps1), d1, taps1, len(self.blocks))
        bk.fft = True
        self.fft_taps.add(id(bk.taps1))
        self.banks.append(bk)
        return bk

    def _bank_model(self, taps1, d1, chans, x, P, sizes):
        model = bank_fft_model if id(taps1) in self.fft_taps else bank_model
        return model(taps1, d1, chans, x, P, sizes)


def fft_taps(rng, T):
    return (rng.standard_normal(T) / np.sqrt(T)).astype(np.float32)
