"""NumPy restatement of the octave widget's levels on its LIVE filterbank.

TEST INFRASTRUCTURE ONLY (see ``oracle/__init__.py``).  Built from the restatements in
``oracle/friture_oracle.py``; all arithmetic float64, like the reference.
"""
from __future__ import annotations

import numpy as np

from .friture_oracle import (NOCTAVE, SAMPLING_RATE, exp_smoothed_value, fft_bank_state, fir_bank_direct,
                             get_decs, octave_filter_bank_decimation_fft, smoothing_alpha, smoothing_kernel)


class LiveOctaveSpectrumOracle:
    """OctaveSpectrum_Widget.handle_new_data over the LIVE bank the widget actually runs
    (friture/octavespectrum.py:91-121,140-163 around friture/filter.py:136-247): `push` as in
    friture_oracle.OctaveSpectrumOracle, the bank being octave_filter_bank_decimation_fft for
    blocks of at most 1024 samples (the reference's FFT sizes are valid up to there,
    friture/filter_design.py:400-401) and fir_bank_direct, the same convolutions, for longer
    blocks.  One stream keeps to one side of that line: the two forms carry different state."""

    def __init__(self, boct_fir, bdec_fir, response_time=1.0, noctave=NOCTAVE):
        self.boct_fir = np.asarray(boct_fir, dtype=np.float64)
        self.bdec_fir = np.asarray(bdec_fir, dtype=np.float64)
        self.noctave = noctave
        self.bpo, L = self.boct_fir.shape
        self.nbands = noctave * self.bpo
        self.decs = get_decs(self.bpo, noctave)
        self.overlaps = fft_bank_state(self.bpo, L, noctave)
        self.hist = [np.zeros(L - 1) for _ in range(noctave)]
        self.form = None
        self.dispbuffers = [0.0] * self.nbands
        self.set_response_time(response_time)

    def set_response_time(self, response_time):
        """setresponsetime (friture/octavespectrum.py:140-156): new alphas and kernels, the display
        buffers and the filter state are kept."""
        self.alphas = [smoothing_alpha(response_time, SAMPLING_RATE / d) for d in self.decs]
        self.kernels = [smoothing_kernel(a, 2 * 4096 / d) for a, d in zip(self.alphas, self.decs)]

    def filter(self, x):
        form = "fft" if len(x) <= 1024 else "direct"
        if self.form not in (None, form):
            raise ValueError("one stream keeps to blocks of <= 1024 samples or to longer ones")
        self.form = form
        if form == "fft":
            y, _, oo, od = octave_filter_bank_decimation_fft(self.boct_fir, self.bdec_fir, x,
                                                             *self.overlaps, noctave=self.noctave)
            self.overlaps = (oo, od)
        else:
            y, self.hist = fir_bank_direct(self.boct_fir, self.bdec_fir, x, self.hist, self.noctave)
        return y

    def push(self, x):
        """One chunk -> (smoothed band energies[nbands], dB[nbands], y)."""
        y = self.filter(np.asarray(x, dtype=np.float64))
        sp = [exp_smoothed_value(k, a, yy ** 2, old)
              for yy, k, a, old in zip(y, self.kernels, self.alphas, self.dispbuffers)]
        self.dispbuffers = sp
        sp = np.array(sp)
        return sp, 10 * np.log10(sp + 1e-30), y
