"""Numeric part of ``Delay_Estimator_Widget.handle_new_data`` (friture/delay_estimator.py:87-176)
for many channel pairs on the GPU: two-fold IIR decimation (48 -> 12 kHz), framing with 50 %
overlap and end-index semantics, GCC-PHAT, temporal smoothing, peak pick, delay / distance /
confidence."""
from __future__ import annotations

import numpy as np

from . import _lib, filter_data
from ._lib import Handle
from .audioproc import SAMPLING_RATE
from .correlation import GccPhat, PairGccPhat
from .stream import StreamFramer

DEFAULT_DELAYRANGE = 1   # seconds, friture/delay_estimator.py:31


class Decimator:
    """``decimate_multiple`` (friture/signal/decimate.py:45-71) with carried state for C channels."""

    def __init__(self, n_channels, n_stages=2, device=None):
        import torch
        self.device = torch.device("cuda", _lib.device_index(device))
        self.n_channels = int(n_channels)
        self.n_stages = int(n_stages)
        self.handle = Handle(self.device.index)
        sos = np.ascontiguousarray(filter_data.decimator()[2], dtype=np.float64)
        self.handle.call("frt_decimate_plan", self.n_channels, self.n_stages, _lib._ptr(sos))

    def process(self, x, stream=None):
        import torch
        _lib.check_tensor(self, x, "x")
        with _lib.call_stream(x.device, stream) as sp:
            x, x_stride = _lib.device_rows(self, x.contiguous(), "x")
            C, T = x.shape
            if C != self.n_channels:
                raise ValueError("x must be a CUDA float32 tensor [%d, T]" % self.n_channels)
            if T == 0:
                return x
            if T % 256 != 0:
                raise ValueError("chunk length must be a multiple of 256")
            out = torch.empty((self.n_channels, T >> self.n_stages), dtype=torch.float32, device=x.device)
            self.handle.call("frt_decimate_process", _lib._ptr(x), x_stride, int(T), _lib._ptr(out),
                             int(out.shape[1]), sp)
        return out


class _DelayWidget:
    """What the widget's numeric part shares between the pair and the channel-array estimators: the
    frame geometry of a delay range and the published values."""

    def _setup_range(self, delayrange_s, device):
        import torch
        self.device = torch.device("cuda", _lib.device_index(device))
        self.Ndec = 2                                                    # delay_estimator.py:52
        self.subsampled_sampling_rate = SAMPLING_RATE / 2 ** self.Ndec   # :53
        self.delayrange_s = delayrange_s
        self.length = int(2 * delayrange_s * self.subsampled_sampling_rate)   # :114-115
        self.needed = int(0.5 * self.length)                                 # :116-117
        # a frame and its successor's hop, plus room for a few chunks; the framers grow when a
        # longer chunk arrives (the default capacity, 4 L + 64 hops, is 3.5 GB per pair at 1000 s)
        self.capacity = 2 * self.length + 4096

    def _setup_outputs(self, n_pairs):
        self.delay_ms = np.zeros(n_pairs)
        self.distance_m = np.zeros(n_pairs)
        self.correlation = np.zeros(n_pairs, dtype=int)
        self.Xcorr_extremum = np.zeros(n_pairs)

    def _publish(self, idx, val):
        import torch
        sm = self.gcc._smoothed
        i = idx.cpu().numpy().astype(np.int64)
        v = val.cpu().numpy().astype(np.float64)
        std = torch.std(sm.double(), dim=1, unbiased=False).cpu().numpy()
        time = 2 * self.delayrange_s
        with np.errstate(divide="ignore", invalid="ignore"):
            norm = np.where(std > 0, np.abs(v) / (3 * std), 0.0)           # :146
        delay = 1e3 * i / self.subsampled_sampling_rate                     # :147
        delay = np.where(delay > 1e3 * time / 2., delay - 1e3 * time, delay)   # :150-151
        self.delay_ms = delay
        self.Xcorr_extremum = v
        self.distance_m = delay * 1e-3 * 340.                              # :169-170
        x = (norm > 1.) * (norm - 1.)                                      # :173-176
        x = (0.12 * x) ** 3
        self.correlation = ((x / (1. + x)) * 100).astype(int)


class DelayEstimator(_DelayWidget):
    """Per pair (channel 0 vs channel 1 of each stream): push 48 kHz chunks, get the delay."""

    def __init__(self, n_pairs, delayrange_s=DEFAULT_DELAYRANGE, device=None):
        self._setup_range(delayrange_s, device)
        self.n_pairs = int(n_pairs)
        self.dec0 = Decimator(n_pairs, self.Ndec, self.device)
        self.dec1 = Decimator(n_pairs, self.Ndec, self.device)
        self.fr0 = StreamFramer(n_pairs, self.length, self.needed, self.device, capacity=self.capacity,
                                pre_increment=True)
        self.fr1 = StreamFramer(n_pairs, self.length, self.needed, self.device, capacity=self.capacity,
                                pre_increment=True)
        self.gcc = GccPhat(self.length, handle=self.dec0.handle, fs=self.subsampled_sampling_rate)
        self._setup_outputs(n_pairs)

    def handle_new_data(self, x0, x1):
        """x0, x1: CUDA float32 [n_pairs, n] chunks of the two channels at 48 kHz."""
        d0 = self.dec0.process(x0)
        d1 = self.dec1.process(x1)
        self.fr0.push(d0)
        self.fr1.push(d1)
        v0, r = self.fr0.take()
        v1, _ = self.fr1.take()
        for i in range(r):
            a = v0[:, i * self.needed:i * self.needed + self.length]
            b = v1[:, i * self.needed:i * self.needed + self.length]
            idx, val, xc = self.gcc.estimate(a, b, smooth=True, want_xcorr=False)
            self._publish(idx, val)
        return r


class ArrayDelayEstimator(_DelayWidget):
    """Delays between channels of one multichannel stream: for every entry (i, j) of ``pairs``,
    channel i is the widget's channel 0 and channel j its channel 1.  Push [C, n] chunks at 48 kHz;
    each channel is decimated, framed and transformed once.  ``delay_ms``, ``distance_m``,
    ``correlation`` and ``Xcorr_extremum`` are indexed by pair, as ``DelayEstimator``'s are."""

    def __init__(self, n_channels, pairs, delayrange_s=DEFAULT_DELAYRANGE, device=None):
        self._setup_range(delayrange_s, device)
        self.n_channels = int(n_channels)
        self.dec = Decimator(self.n_channels, self.Ndec, self.device)
        self.fr = StreamFramer(self.n_channels, self.length, self.needed, self.device, capacity=self.capacity,
                               pre_increment=True)
        self.gcc = PairGccPhat(self.length, self.n_channels, pairs, handle=self.dec.handle,
                               fs=self.subsampled_sampling_rate)
        self.n_pairs = self.gcc.n_pairs
        self._setup_outputs(self.n_pairs)

    def handle_new_data(self, x):
        """x: CUDA float32 [n_channels, n] chunk at 48 kHz.  Returns the number of frames run."""
        self.fr.push(self.dec.process(x))
        v, r = self.fr.take()
        for i in range(r):
            idx, val, _ = self.gcc.estimate(v[:, i * self.needed:i * self.needed + self.length], smooth=True)
            self._publish(idx, val)
        return r
