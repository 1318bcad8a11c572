"""Numeric part of ``Delay_Estimator_Widget.handle_new_data`` (friture/delay_estimator.py:87-176)
for many channel pairs on the GPU: two-fold IIR decimation (48 -> 12 kHz), framing with 50 %
overlap and end-index semantics, GCC-PHAT, temporal smoothing, peak pick, delay / distance /
confidence."""
from __future__ import annotations

from typing import NamedTuple

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


class DelayTrack(NamedTuple):
    """Every frame of an estimator's last ``handle_new_data`` call, oldest first.  ``end_index`` [r]:
    the widget's ``old_index`` after the frame (its last sample, in 12 kHz samples since the stream
    began); the others are [r, n_pairs] and mean what the estimator's attributes of the same names
    mean for the last frame."""
    end_index: np.ndarray
    delay_ms: np.ndarray
    distance_m: np.ndarray
    correlation: np.ndarray
    Xcorr_extremum: np.ndarray


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
        self.track = self._track(np.zeros(0, dtype=np.int64), np.zeros((0, n_pairs), dtype=np.int64),
                                 np.zeros((0, n_pairs)), np.zeros((0, n_pairs)))

    def _run_frames(self, r, gcc_frames):
        """Runs the r frames the framer just took with one ``estimate_frames`` call (gcc_frames) and
        publishes them; the framer's old_index has already moved past them."""
        end_index = self._framer.old_index - self.needed * np.arange(r - 1, -1, -1, dtype=np.int64)
        if r == 0:
            self.track = self._track(end_index, np.zeros((0, self.n_pairs), dtype=np.int64),
                                     np.zeros((0, self.n_pairs)), np.zeros((0, self.n_pairs)))
            return
        idx, val, std = gcc_frames()
        self._publish(end_index, idx, val, std)

    def _publish(self, end_index, idx, val, std):
        """idx, val, std: [r, P] per frame (any tensor or array on any device).  The widget's formulas
        (delay_estimator.py:146-176) on every frame; the attributes take the last one."""
        track = self._track(np.asarray(end_index, dtype=np.int64), np.asarray(idx.cpu()).astype(np.int64),
                            np.asarray(val.cpu()).astype(np.float64), np.asarray(std.cpu()).astype(np.float64))
        self.track = track
        if track.end_index.shape[0]:
            self.delay_ms = track.delay_ms[-1]
            self.Xcorr_extremum = track.Xcorr_extremum[-1]
            self.distance_m = track.distance_m[-1]
            self.correlation = track.correlation[-1]

    def _track(self, end_index, i, v, std):
        time = 2 * self.delayrange_s
        with np.errstate(divide="ignore", invalid="ignore"):
            norm = np.where(std > 0, np.abs(v) / (3 * std), 0.0)           # :146
        delay = 1e3 * i / self.subsampled_sampling_rate                     # :147
        delay = np.where(delay > 1e3 * time / 2., delay - 1e3 * time, delay)   # :150-151
        x = (norm > 1.) * (norm - 1.)                                      # :173-176
        x = (0.12 * x) ** 3
        return DelayTrack(end_index=end_index, delay_ms=delay, distance_m=delay * 1e-3 * 340.,   # :169-170
                          correlation=((x / (1. + x)) * 100).astype(int), Xcorr_extremum=v)


class DelayEstimator(_DelayWidget):
    """Per pair (channel 0 vs channel 1 of each stream): push 48 kHz chunks, get the delay.  Each
    ``handle_new_data`` runs all the frames the chunk completes in one library call; ``track`` keeps
    every one of them, and ``delay_ms`` etc. are the last one's."""

    def __init__(self, n_pairs, delayrange_s=DEFAULT_DELAYRANGE, device=None):
        self._setup_range(delayrange_s, device)
        self.n_pairs = int(n_pairs)
        self.dec0 = Decimator(n_pairs, self.Ndec, self.device)
        self.dec1 = Decimator(n_pairs, self.Ndec, self.device)
        self.fr0 = StreamFramer(n_pairs, self.length, self.needed, self.device, capacity=self.capacity,
                                pre_increment=True)
        self.fr1 = StreamFramer(n_pairs, self.length, self.needed, self.device, capacity=self.capacity,
                                pre_increment=True)
        self._framer = self.fr0
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
        self._run_frames(r, lambda: self.gcc.estimate_frames(v0, v1, self.needed, r))
        return r


class ArrayDelayEstimator(_DelayWidget):
    """Delays between channels of one multichannel stream: for every entry (i, j) of ``pairs``,
    channel i is the widget's channel 0 and channel j its channel 1.  Push [C, n] chunks at 48 kHz;
    each channel is decimated, framed and transformed once.  ``delay_ms``, ``distance_m``,
    ``correlation``, ``Xcorr_extremum`` and ``track`` are indexed by pair, as ``DelayEstimator``'s are."""

    def __init__(self, n_channels, pairs, delayrange_s=DEFAULT_DELAYRANGE, device=None):
        self._setup_range(delayrange_s, device)
        self.n_channels = int(n_channels)
        self.dec = Decimator(self.n_channels, self.Ndec, self.device)
        self.fr = StreamFramer(self.n_channels, self.length, self.needed, self.device, capacity=self.capacity,
                               pre_increment=True)
        self._framer = self.fr
        self.gcc = PairGccPhat(self.length, self.n_channels, pairs, handle=self.dec.handle,
                               fs=self.subsampled_sampling_rate)
        self.n_pairs = self.gcc.n_pairs
        self._setup_outputs(self.n_pairs)

    def handle_new_data(self, x):
        """x: CUDA float32 [n_channels, n] chunk at 48 kHz.  Returns the number of frames run."""
        self.fr.push(self.dec.process(x))
        v, r = self.fr.take()
        self._run_frames(r, lambda: self.gcc.estimate_frames(v, self.needed, r))
        return r
