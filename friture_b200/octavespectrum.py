"""Numeric part of ``OctaveSpectrum_Widget`` (friture/octavespectrum.py:91-163) for many channels on
the GPU, with the live filterbank's numerics: the 512-tap FIR bank that the widget's
``Octave_Filters.filter()`` runs (friture/filter.py:136-247), then per band
``y**2 -> exp_smoothed_value -> 10*log10(sp + 1e-30) + w``.  One kernel launch per call covers all
of the call's blocks and writes one level vector per channel and block; the band signals never
leave the chip."""
from __future__ import annotations

import numpy as np

from . import _lib
from .octavefilters import Octave_Filters, smoothing_alphas
from .filter_data import NOCTAVE

MAX_BLOCK = 4096   # the live bank's per-launch limit; also keeps every stage's block within the
                   # smoothing kernel of 8192/dec taps (friture/signal/exp_smoothing.py:43-47)


class OctaveSpectrumAnalyzer:
    """Per-block band levels of ``n_channels`` independent streams.  Defaults are the widget's
    (friture/octavespectrum_settings.py:27-30).  ``alphas`` holds the smoothing factor of each
    decimation stage j (rate fs/2^j); the band levels carry over from call to call."""

    def __init__(self, n_channels, bandsperoctave=3, response_time=1.0, weighting=0,
                 n_octaves=NOCTAVE, handle=None):
        self.n_channels = int(n_channels)
        self._n_octaves = n_octaves
        self._handle = handle
        self.filters = None
        self.response_time = response_time
        self.weighting = weighting
        self.setbandsperoctave(bandsperoctave)

    # -- the widget's setters ---------------------------------------------------------------
    def setbandsperoctave(self, bandsperoctave):
        """New filters: filter state and levels restart from zero (octavespectrum.py:158-163)."""
        if self.filters is None:
            self.filters = Octave_Filters(bandsperoctave, mode="fft", n_octaves=self._n_octaves,
                                          handle=self._handle)
        else:
            self.filters.setbandsperoctave(bandsperoctave)
        f = self.filters
        self.bandsperoctave = f.bandsperoctave
        self.nbands = f.nbands
        self.fi, self.flow, self.fhigh, self.f_nominal = f.fi, f.flow, f.fhigh, f.f_nominal
        self._planned = False
        self.setresponsetime(self.response_time)
        self.setweighting(self.weighting)

    def setresponsetime(self, response_time):
        """New smoothing time constant; the levels carry on (octavespectrum.py:140-156)."""
        self.response_time = response_time
        self.alphas = smoothing_alphas(response_time, self._n_octaves)
        self._push_smoothing()

    def setweighting(self, weighting):
        """0 none, 1 / 'A', 2 / 'B', 3 / 'C' (octavespectrum.py:111-118); the levels carry on."""
        key = {0: None, 1: "A", 2: "B", 3: "C", "A": "A", "B": "B", "C": "C"}.get(weighting, False)
        if key is False:
            raise ValueError("weighting must be 0-3 or 'A', 'B', 'C'")
        self.weighting = weighting
        self._w = None if key is None else np.ascontiguousarray(getattr(self.filters, key), dtype=np.float32)
        self._push_smoothing()

    def reset(self):
        """Filter state and levels back to zero."""
        if self._planned:
            self.filters.handle.call("frt_firbank_reset")

    # -- plumbing ----------------------------------------------------------------------------
    def _push_smoothing(self):
        if self._planned:
            self.filters.handle.call("frt_firbank_set_smoothing", _lib._ptr(self.alphas), _lib._ptr(self._w))

    def _ensure_plan(self):
        if not self._planned:
            self.filters._ensure_fir_plan(self.n_channels)
            self._planned = True
            self._push_smoothing()

    # -- one call ----------------------------------------------------------------------------
    def process(self, x, block=512, db=True, stream=None):
        """x: CUDA float32 [C, n_blocks*block], contiguous along time (any row stride).  Returns a
        CUDA float32 tensor [C, n_blocks, nbands]: the widget's output after each block, in dB
        with the weighting when ``db``, else the smoothed linear band energies."""
        import torch
        x, x_stride = _lib.device_rows(self.filters, x, "x")
        C, T = x.shape
        if C != self.n_channels:
            raise ValueError("expected %d channels, got %d" % (self.n_channels, C))
        step = 1 << (self._n_octaves - 1)
        if not isinstance(block, (int, np.integer)) or block <= 0 or block > MAX_BLOCK or block % step:
            raise ValueError("block must be a multiple of %d and at most %d (every decimation stage "
                             "keeps its even samples, friture/signal/decimate.py:41)" % (step, MAX_BLOCK))
        if T == 0 or T % block:
            raise ValueError("T must be a whole, non-zero number of blocks")
        if x_stride < T:
            raise ValueError("x rows must not overlap")
        self._ensure_plan()
        n_blocks = T // block
        with _lib.call_stream(x.device, stream) as sp:
            out = torch.empty((C, n_blocks, self.nbands), dtype=torch.float32, device=x.device)
            self.filters.handle.call("frt_firbank_levels", _lib._ptr(x), x_stride, int(block), int(n_blocks),
                                     _lib._ptr(out), 1 if db else 0, sp)
        return out
