"""Numeric part of the levels widget (``Levels_Widget.handle_new_data``, friture/levels.py:84-131, with
the ballistic peak of friture/ballistic_peak.py and friture/iec.py) and of the long-term levels widget
(``LongLevelWidget.handle_new_data`` and its setters, friture/longlevels.py:150-230) for many channels on
the GPU.  Every channel gets its own meter and its own level history; one call runs all the buffers or
blocks of a chunk in one launch."""
from __future__ import annotations

from typing import NamedTuple

import numpy as np

from . import _lib
from ._lib import Handle
from .audioproc import FRAMES_PER_BUFFER, SAMPLING_RATE
from .stream import StreamFramer

PEAK_DECAY_RATE = 1.0 - 3E-6 / 500.        # friture/ballistic_peak.py:22
LONG_RESPONSE_TIMES = (1, 20)              # seconds, friture/longlevels_settings.py:58-59
LONG_DURATIONS = (5, 3600)                 # seconds, friture/longlevels_settings.py:66-67
LONG_HISTORY = 8192                        # samples kept before old_index: the longest block (rt = 20 s)
RING_LENGTH = 10000                        # the level ring's first length (friture/ringbuffer.py:33)


def gauss(n=11, sigma=1):
    """friture/longlevels.py:45-47, term for term."""
    r = range(-int(n / 2), int(n / 2) + 1)
    return [1 / (sigma * np.sqrt(2 * np.pi)) * np.exp(-float(x) ** 2 / (2 * sigma ** 2)) for x in r]


def _check_rows(x, n_channels, name):
    """x as [C, T] once it is a tensor of n_channels rows, contiguous along time, whose rows do not
    overlap.  Only the layout is checked here, so that these refusals come before any device work."""
    import torch
    if not isinstance(x, torch.Tensor):
        raise ValueError("%s must be a CUDA float32 tensor [%d, T]" % (name, n_channels))
    if x.dim() == 1:
        x = x[None, :]
    if x.dim() != 2 or x.shape[0] != n_channels:
        raise ValueError("%s must be a CUDA float32 tensor [%d, T]" % (name, n_channels))
    C, T = x.shape
    if T > 1 and x.stride(1) != 1:
        raise ValueError("%s must be contiguous along time" % name)
    if C > 1 and T > 0 and x.stride(0) < T:
        raise ValueError("%s has overlapping rows (row stride %d < %d samples)" % (name, x.stride(0), T))
    return x


def grow_ring(ring, offset, length):
    """RingBuffer.grow_if_needed (ringbuffer.py:105-130) on ring [rows, old], a device tensor whose slot
    p % old holds stream position p, after `offset` positions were pushed.  When length > old, the value
    in slot s moves to slot (s + shift) % new of a zeroed ring of new = int(1.5 * length) slots, shift =
    (offset % new - offset % old) % new.  Returns (ring, its length)."""
    import torch
    old = ring.shape[1]
    if length <= old:
        return ring, old
    new = int(1.5 * length)
    shift = (offset % new - offset % old) % new
    grown = torch.zeros((ring.shape[0], new), dtype=ring.dtype, device=ring.device)
    direct = min(old, new - shift)
    grown[:, shift:shift + direct] = ring[:, :direct]
    grown[:, :old - direct] = ring[:, direct:old]
    return grown, new


class LevelTicks(NamedTuple):
    """One column per buffer of the call, CUDA float64 [C, R]: the widget's ``level_rms`` and
    ``level_max`` (dB) and the ballistic ``peak_iec`` after that buffer."""
    level_rms: object
    level_max: object
    peak_iec: object


class LevelsAnalyzer:
    """The peak / RMS meter and its ballistic peak, for each of ``n_channels`` channels.
    ``response_time`` is the RMS smoothing time in seconds (0.3 in the widget; its comments name
    0.025, 0.125 and 1 s as the standard meter settings)."""

    handle = _lib.lazy_handle(lambda self: Handle(_lib.device_index(self._device)))

    def __init__(self, n_channels, response_time=0.3, device=None):
        if int(n_channels) < 1:
            raise ValueError("n_channels must be >= 1")
        if not response_time > 0:
            raise ValueError("response_time must be > 0")
        self.n_channels = int(n_channels)
        self.response_time = response_time
        self._device = device
        self._handle = None
        # levels.py:54-74
        w = 0.65
        n = self.response_time * SAMPLING_RATE
        N = 5 * n
        self.alpha = 1. - (1. - w) ** (1. / (n + 1))
        self.kernel = (1. - self.alpha) ** (np.arange(0, N)[::-1])
        n2 = 0.025 / (25 / 1000.)
        self.alpha2 = 1. - (1. - w) ** (1. / (n2 + 1))
        self._buffer = None       # the planned buffer length

    @property
    def max_buffer(self):
        """The longest buffer: the kernel's length Nk.  A longer one would take exp_smoothed_value's
        truncating branch (exp_smoothing.py:44-46)."""
        return self.kernel.shape[0]

    def _plan(self, buffer):
        if buffer == self._buffer:
            return
        Nk = self.kernel.shape[0]
        tail = np.ascontiguousarray(self.kernel[Nk - buffer:Nk], dtype=np.float64)
        decay = (1.0 - self.alpha) ** buffer                 # exp_smoothing.py:48
        self.handle.call("frt_levels_plan", self.n_channels, int(buffer), _lib._ptr(tail),
                         float(self.alpha), float(decay), float(1. - self.alpha2))
        self._buffer = buffer

    def handle_new_data(self, chunk, buffer=FRAMES_PER_BUFFER, stream=None):
        """chunk: CUDA float32 [C, R*buffer] (or [T] for one channel), any row stride.  Each buffer
        is one call of the widget's handle_new_data.  The result is the same bits however the stream
        is cut into chunks."""
        import torch
        buffer = int(buffer)
        if buffer < 1 or buffer > self.max_buffer:
            raise ValueError("buffer must be in 1..%d (the smoothing kernel's length)" % self.max_buffer)
        x = _check_rows(chunk, self.n_channels, "chunk")
        if x.shape[1] % buffer:
            raise ValueError("chunk length %d is not a whole number of %d-sample buffers"
                             % (x.shape[1], buffer))
        with _lib.call_stream(x.device, stream) as sp:
            x, stride = _lib.device_rows(self, x, "chunk")
            R = x.shape[1] // buffer
            out = [torch.empty((self.n_channels, R), dtype=torch.float64, device=x.device) for _ in range(3)]
            if R:
                self._plan(buffer)
                self.handle.call("frt_levels_process", _lib._ptr(x), stride, R, *(_lib._ptr(o) for o in out), sp)
        return LevelTicks(*out)

    def reset(self):
        """Back to the widget's initial state (levels.py:62-64, ballistic_peak.py:33-35)."""
        if self._buffer is not None:
            self.handle.call("frt_levels_reset")

    def state(self):
        """The carried state, host arrays [C]: old_rms, old_max, peak_iec, decay (the ballistic
        peak's decay factor) and hold (its hold counter).  Waits for the device."""
        C = self.n_channels
        if self._buffer is None:
            return dict(old_rms=np.full(C, 1e-30), old_max=np.full(C, 1e-30), peak_iec=np.zeros(C),
                        decay=np.full(C, PEAK_DECAY_RATE), hold=np.zeros(C, dtype=np.int32))
        s = np.empty((4, C), dtype=np.float64)
        hold = np.empty(C, dtype=np.int32)
        self.handle.call("frt_levels_state", _lib._ptr(s), _lib._ptr(hold))
        return dict(old_rms=s[0], old_max=s[1], peak_iec=s[2], decay=s[3], hold=hold)


class LongLevelTrack(NamedTuple):
    """The blocks one ``handle_new_data`` call completed, oldest first: ``end_index`` [r] host
    int64, the stream index each block ends at (the widget's ``old_index`` when it read the block;
    the first block ends at 0 and is the zeros before the stream); ``level_rms`` CUDA float64 [C, r],
    10 log10(max(level, 1e-150)); ``level`` CUDA float64 [C, r], the linear level."""
    end_index: np.ndarray
    level_rms: object
    level: object


class LongLevelsAnalyzer:
    """The long-term level history of each of ``n_channels`` channels.

    The history is a float32 dB ring per channel with the widget's level ring buffer's layout
    (friture/ringbuffer.py): 10000 values at first, grown to int(1.5 * length) when the plotted
    length outgrows it, at the moment the widget grows it and with the values it keeps.  It takes
    C x ring length x 4 bytes of device memory: at rt = 1 s and a 3600 s duration the length is
    675 000 values and the ring 1 012 500, 4.1 GB at C = 1024.

    A NaN or infinite sample acts as in the widget, whose filters then hold NaN: the channel's levels
    are NaN from that block on, until ``setresptime`` or ``reset``."""

    handle = _lib.lazy_handle(lambda self: Handle(_lib.device_index(self._device)))

    def __init__(self, n_channels, response_time=20, duration=600, level_min=-70, level_max=-20, device=None):
        if int(n_channels) < 1:
            raise ValueError("n_channels must be >= 1")
        self.n_channels = int(n_channels)
        self._device = device
        self._handle = None
        self.level_min = level_min
        self.level_max = level_max
        self.length_seconds = None
        self._plan_ndec = None      # the decimation depth the handle's filter state is planned for
        self.setresptime(response_time)
        self.setduration(duration)
        self.reset()

    # -- the widget's setters ---------------------------------------------------------------
    def setresptime(self, value):
        """longlevels.py:207-224: a new decimation depth and block length; the filter state starts
        again, old_index and the level history are kept."""
        if not LONG_RESPONSE_TIMES[0] <= value <= LONG_RESPONSE_TIMES[1]:
            raise ValueError("response time must be in %g..%g s" % LONG_RESPONSE_TIMES)
        self.response_time = value
        self.Ndec = int(max(0, np.floor((np.log2(self.response_time * SAMPLING_RATE / 100.)))))
        self.needed = int(2 ** self.Ndec)
        self.subsampled_sampling_rate = SAMPLING_RATE / 2 ** (self.Ndec)
        self._restart_filters()
        if getattr(self, "_framer", None) is not None:
            self._framer.set_geometry(self.needed, self.needed)
        if self.length_seconds:
            self.setduration(self.length_seconds)

    def setduration(self, value):
        """longlevels.py:201-205: the plotted length, from the next block on."""
        if not LONG_DURATIONS[0] <= value <= LONG_DURATIONS[1]:
            raise ValueError("duration must be in %g..%g s" % LONG_DURATIONS)
        self.length_seconds = value
        self.length_samples = int(self.length_seconds * self.subsampled_sampling_rate)

    def setmin(self, value):
        self.level_min = value

    def setmax(self, value):
        self.level_max = value

    def reset(self):
        """A new widget with the current settings: no samples, zero filter state, an empty history."""
        self._framer = None
        self._ring = None
        self._ring_len = RING_LENGTH
        self._ring_pos = 0
        self._curve = None
        self._restart_filters()

    def _restart_filters(self):
        """Zero filter state from the next block on: a plan of another depth zeroes it when the next
        block runs; with the planned depth, frt_longlevels_reset zeroes it now."""
        if self._plan_ndec == self.Ndec:
            self.handle.call("frt_longlevels_reset")

    # -- the stream ---------------------------------------------------------------------------
    def take_blocks(self, chunk):
        """The framing of handle_new_data: appends chunk [C, n] (any torch device) and returns
        (blocks, end_index), blocks [C, r*needed] the r blocks it completed back to back (None when
        r == 0) and end_index [r] int64 where each ends (longlevels.py:150-191: the `needed`
        samples that end at old_index, then old_index += needed)."""
        if self._framer is None:
            self._framer = StreamFramer(self.n_channels, self.needed, self.needed, chunk.device,
                                        history=LONG_HISTORY)
        self._framer.push(chunk)
        first = self._framer.old_index
        view, r = self._framer.take()
        return view, first + self.needed * np.arange(r, dtype=np.int64)

    def _plan(self):
        if self._plan_ndec == self.Ndec:
            return
        bdec = np.ascontiguousarray(gauss(11, 2.), dtype=np.float64)           # longlevels.py:56
        bfir = np.ascontiguousarray(gauss(10 * 4 + 1, 2. * 4), dtype=np.float64)   # longlevels.py:213-214
        self.handle.call("frt_longlevels_plan", self.n_channels, self.Ndec, _lib._ptr(bdec), _lib._ptr(bfir))
        self._plan_ndec = self.Ndec

    def _grow_if_needed(self, length):
        self._ring, self._ring_len = grow_ring(self._ring, self._ring_pos, length)

    def handle_new_data(self, chunk, stream=None):
        """chunk: CUDA float32 [C, n] (or [T] for one channel), any row stride and any length.
        Runs every block the chunk completes in one launch and returns their LongLevelTrack."""
        import torch
        x = _check_rows(chunk, self.n_channels, "chunk")
        with _lib.call_stream(x.device, stream) as sp:
            x, _ = _lib.device_rows(self, x, "chunk")
            view, end_index = self.take_blocks(x)
            r = len(end_index)
            level = torch.empty((self.n_channels, r), dtype=torch.float64, device=x.device)
            db = torch.empty_like(level)
            if r == 0:
                return LongLevelTrack(end_index, db, level)
            self._plan()
            if self._ring is None:
                self._ring = torch.zeros((self.n_channels, self._ring_len), dtype=torch.float32, device=x.device)
            stride = _lib._row_stride(view.shape, view.stride(0))
            self.handle.call("frt_longlevels_process", _lib._ptr(view), stride, r, _lib._ptr(level), _lib._ptr(db),
                             _lib._ptr(self._ring), self._ring_len, self._ring_pos, sp)
            self._ring_pos += r
            # longlevels.py:193-199: the curve is taken from the ring after the blocks
            self._grow_if_needed(self.length_samples)
            self._curve = (self.length_samples, self.subsampled_sampling_rate, self.length_seconds,
                           float(self.level_min), float(self.level_max))
        return LongLevelTrack(end_index, db, level)

    def curve(self, stream=None):
        """The curve the widget draws after the last handle_new_data call that completed a block
        (longlevels.py:193-199): (scaled_t host float64 [L], scaled_y CUDA float32 [C, L]), with the
        duration, level range and response time in force at that call.  Before any block, L = 0."""
        import torch
        if self._curve is None:
            return np.zeros(0), None
        L, rate, seconds, lo, hi = self._curve
        scaled_t = (np.arange(L) / rate) / seconds
        with _lib.call_stream(self._ring.device, stream) as sp:
            out = torch.empty((self.n_channels, L), dtype=torch.float32, device=self._ring.device)
            self.handle.call("frt_longlevels_history", _lib._ptr(self._ring), self._ring_len, self._ring_pos,
                             self.n_channels, L, lo, hi, _lib._ptr(out), sp)
        return scaled_t, out
