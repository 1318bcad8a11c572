"""NumPy restatement of the spectrum widget's two-channel tick (its dual-channel measurement mode).

TEST INFRASTRUCTURE ONLY (see ``oracle/__init__.py``).  Built from the restatements in
``oracle/friture_oracle.py``; all arithmetic float64, like the reference.
"""
from __future__ import annotations

import numpy as np

from .friture_oracle import (SpectrumWidgetOracle, exp_smoothed_value_2d, harmonic_product_spectrum,
                             log_spectrogram, stft_power)


class DualSpectrumWidgetOracle(SpectrumWidgetOracle):
    """Spectrum_Widget.handle_new_data with both of its smoothed columns
    (friture/spectrum.py:141-182, setdualchannels :286-293).  Per tick with realizable frames:
    sp1 from row 0 of floatdata; sp2 from row 1 when dual_channels is set and there are two rows,
    otherwise all zeros -- both smoothed on every tick, so that dispbuffers2 decays by
    (1-alpha)^frames in single mode.  Dual: dB = log(sp2) - log(sp1), no weighting; single:
    dB = log(sp1) + w.  The peak is the arg-max of that dB, the pitch the HPS arg-max of sp1."""

    def __init__(self, fft_size, overlap=0.75, response_time=0.025, weight=None,
                 dual_channels=False):
        super().__init__(fft_size, overlap, response_time, weight)
        self.dual_channels = dual_channels
        self.disp2 = np.zeros(fft_size // 2 + 1)

    def setdualchannels(self, dual_enabled):
        self.dual_channels = dual_enabled          # no state is reset (spectrum.py:286-293)

    def tick_power(self, sp1n, sp2n=None):
        """sp1n, sp2n: [bins, realizable] power of rows 0 and 1 (sp2n None: one row).
        Returns None for a tick without frames (spectrum.py:140), else
        (dB, fmax Hz, fpitch Hz, peak index, pitch index)."""
        if sp1n.shape[1] == 0:
            return None
        dual = self.dual_channels and sp2n is not None
        if not dual:
            sp2n = np.zeros_like(sp1n)              # spectrum.py:142
        sp1 = exp_smoothed_value_2d(self.kernel, self.alpha, sp1n, self.disp)
        sp2 = exp_smoothed_value_2d(self.kernel, self.alpha, sp2n, self.disp2)
        self.disp, self.disp2 = sp1, sp2
        if dual:
            db = log_spectrogram(sp2) - log_spectrogram(sp1)
        else:
            db = log_spectrogram(sp1) + self.w
        i = int(np.argmax(db))
        pitch = int(np.argmax(harmonic_product_spectrum(sp1)))
        return db, self.freq[i], max(self.freq[pitch], 1e-20), i, pitch

    def tick(self, x):
        """x: floatdata of the tick, [rows, T] (or [T] for one row)."""
        x = np.atleast_2d(x)
        sp1n = stft_power(x[0], self.fft_size, self.hop).T
        sp2n = None
        if self.dual_channels and x.shape[0] > 1:
            sp2n = stft_power(x[1], self.fft_size, self.hop).T
        return self.tick_power(sp1n, sp2n)


