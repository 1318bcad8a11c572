"""Numeric part of the scope widget (``Scope_Widget.handle_new_data`` and ``set_timerange``,
friture/scope.py:78-148) for many scopes on the GPU.  Every scope reads its own copy of the widget's
ring buffer (friture/ringbuffer.py); one call runs all the 512-sample buffers of a chunk, each one tick
of the widget, in one trigger launch and one curve launch."""
from __future__ import annotations

from typing import NamedTuple

import numpy as np

from . import _lib
from ._lib import Handle
from .audioproc import FRAMES_PER_BUFFER, SAMPLING_RATE
from .levels import RING_LENGTH, _check_rows, grow_ring

SCROLLING_THRESHOLD_MS = 500.0          # friture/scope.py:35
DEFAULT_TIMERANGE = 50                  # friture/scope.py:33, ms
TIMERANGE_MS = (0.1, 10000.0)           # the settings dialog's range (scope.py:174-175)
NOT_DRAWN = np.iinfo(np.int64).min      # window_start of a tick that drew nothing


def scope_width(timerange):
    """scope.py:79-80: the window length in samples, with the widget's two float64 roundings."""
    time = timerange * 1e-3
    return int(time * SAMPLING_RATE)


def is_trigger(timerange):
    """Trigger mode (scope.py:89): timerange <= 500 ms; above it the scope scrolls."""
    return not timerange > SCROLLING_THRESHOLD_MS


def scope_points(timerange):
    """The number of points a tick draws: 2 * (width // 2) in trigger mode, width when scrolling."""
    w = scope_width(timerange)
    return 2 * (w // 2) if is_trigger(timerange) else w


def scope_time(timerange):
    """scaled_t (scope.py:125-127), host float64 [scope_points(timerange)]."""
    w = scope_width(timerange)
    time = (np.arange(scope_points(timerange)) - w // 2) / float(SAMPLING_RATE)
    return (time * 1e3 + timerange / 2.) / timerange


def trigger_level(window):
    """scope.py:105: max * 2 / 3 in float64 of a search window (NaN when it holds one)."""
    return np.asarray(window, dtype=np.float64).max() * 2. / 3.


class ScopeTicks(NamedTuple):
    """One entry per tick of a call: ``end_index`` host int64 [R], the stream index the tick's
    samples end at; ``window_start`` CUDA int64 [S, R], the stream index its drawn window starts at
    (negative when the window reaches into the zeros before the stream), or NOT_DRAWN when the tick
    found no trigger and the scope kept its curve."""
    end_index: np.ndarray
    window_start: object


class ScopeCurve(NamedTuple):
    """The curves the widgets hold: ``scaled_y`` and ``scaled_y2`` (None for one-channel scopes) CUDA
    float32 [S, Lmax], of which row s's first scope_points(timerange[s]) values are its curve;
    ``timerange`` CUDA float64 [S], the range each scope last drew at, NaN if it never drew."""
    scaled_y: object
    scaled_y2: object
    timerange: object


class ScopeAnalyzer:
    """``n_scopes`` scopes, each the widget's numeric state: its ring buffer, time range and curve.

    Each scope models a widget that reads its own ring buffer: 10000 samples at first, grown to
    int(1.5 * length) by the first tick that asks for more, which keeps only what was written since
    the ring last wrapped, as friture/ringbuffer.py does.  (In Friture the ring is the audio buffer
    shared by every widget, which another widget may grow first.)  Per channel the ring takes up to
    720 000 float32 samples at 10 s and the curve up to 480 000, 4.8 MB per channel together; a call
    also stages the window before the chunk and the chunk, up to 480 000 + n samples per channel."""

    handle = _lib.lazy_handle(lambda self: Handle(_lib.device_index(self._device)))

    def __init__(self, n_scopes, two_channels=False, timerange=DEFAULT_TIMERANGE, device=None):
        if int(n_scopes) < 1:
            raise ValueError("n_scopes must be >= 1")
        self.n_scopes = int(n_scopes)
        self.n_channels = 2 if two_channels else 1
        self._device = device
        self._handle = None
        self.set_timerange(timerange)
        self.reset()

    def set_timerange(self, timerange):
        """scope.py:146-148: the time range in ms, from the next tick on."""
        if not TIMERANGE_MS[0] <= timerange <= TIMERANGE_MS[1]:
            raise ValueError("timerange must be in %g..%g ms" % TIMERANGE_MS)
        self.timerange = timerange

    def reset(self):
        """A new widget with the current time range: an empty ring, no curve."""
        self._ring = None             # [S * n_ch, ring_len] float32: slot p % ring_len holds position p
        self._ring_len = RING_LENGTH
        self._offset = 0              # samples pushed
        self._curve = None            # [S * n_ch, Lmax] float32
        self._drawn = None            # [S] float64

    # -- the ring ------------------------------------------------------------------------------
    def _push(self, x):
        """RingBuffer.push (ringbuffer.py:39-61) of x [rows, n]: slot (offset + j) % ring_len."""
        n, L = x.shape[1], self._ring_len
        first = self._offset
        if n > L:
            x, first = x[:, n - L:], first + n - L
        a = first % L
        k = min(L - a, x.shape[1])
        self._ring[:, a:a + k] = x[:, :k]
        self._ring[:, :x.shape[1] - k] = x[:, k:]
        self._offset += n

    def _read(self, length):
        """RingBuffer.data (ringbuffer.py:63-78) without its growth: the views of the ring that hold
        the `length` positions before offset, oldest first."""
        a = (self._offset - length) % self._ring_len
        if a + length <= self._ring_len:
            return [self._ring[:, a:a + length]]
        return [self._ring[:, a:], self._ring[:, :a + length - self._ring_len]]

    # -- the stream ----------------------------------------------------------------------------
    def _rows(self, chunk):
        """chunk as [S * n_ch, n] rows once its layout is checked (before any device work)."""
        import torch
        S, nch = self.n_scopes, self.n_channels
        shape = "[%d, n]" % S if nch == 1 else "[%d, 2, n]" % S
        if not isinstance(chunk, torch.Tensor) or chunk.dim() != (2 if nch == 1 else 3):
            raise ValueError("chunk must be a CUDA float32 tensor %s" % shape)
        if nch == 1:
            return [_check_rows(chunk, S, "chunk")]
        if chunk.shape[1] != 2:
            raise ValueError("chunk must be a CUDA float32 tensor %s" % shape)
        return [_check_rows(chunk[:, k], S, "chunk") for k in range(2)]

    def handle_new_data(self, chunk, buffer=FRAMES_PER_BUFFER, stream=None):
        """chunk: CUDA float32 [S, n], or [S, 2, n] for two-channel scopes, any row stride; n a whole
        number of buffers, each one tick of the widget.  Returns the ticks' ScopeTicks.  The result
        and the curves are the same bits however the stream is cut into chunks."""
        import torch
        buffer = int(buffer)
        if not 1 <= buffer <= RING_LENGTH:
            raise ValueError("buffer must be in 1..%d (the ring buffer's first length)" % RING_LENGTH)
        rows = self._rows(chunk)
        n = rows[0].shape[1]
        if n % buffer:
            raise ValueError("chunk length %d is not a whole number of %d-sample buffers" % (n, buffer))
        for r in rows:
            _lib.check_tensor(self, r, "chunk")
        S, nch, R = self.n_scopes, self.n_channels, n // buffer
        timerange = self.timerange
        width, trigger, points = scope_width(timerange), is_trigger(timerange), scope_points(timerange)
        need = 2 * width if trigger else width
        end_index = self._offset + buffer * np.arange(1, R + 1, dtype=np.int64)
        dev = rows[0].device
        with _lib.call_stream(dev, stream) as sp:
            start = torch.empty((S, R), dtype=torch.int64, device=dev)
            if R == 0:
                return ScopeTicks(end_index, start)
            x = torch.stack(rows, dim=1).reshape(S * nch, n) if nch == 2 else rows[0]
            if self._ring is None:
                self._ring = torch.zeros((S * nch, self._ring_len), dtype=torch.float32, device=dev)
                self._drawn = torch.full((S,), float("nan"), dtype=torch.float64, device=dev)
            if self._curve is None or self._curve.shape[1] < points:
                curve = torch.zeros((S * nch, points), dtype=torch.float32, device=dev)
                if self._curve is not None:
                    curve[:, :self._curve.shape[1]] = self._curve
                self._curve = curve
            if need > self._ring_len:
                # the first tick's data() grows the ring after its buffer is pushed (scope.py:92,97)
                self._push(x[:, :buffer])
                self._ring, self._ring_len = grow_ring(self._ring, self._offset, need)
                x = x[:, buffer:]
                lead = need - buffer
            else:
                lead = need
            origin = self._offset - need
            staged = torch.cat(self._read(need) + [x], dim=1)
            self.handle.call("frt_scope_process", _lib._ptr(staged), staged.shape[1], S, nch, lead, R, buffer,
                             width, int(trigger), origin, _lib._ptr(start), _lib._ptr(self._curve),
                             self._curve.shape[1], float(timerange), _lib._ptr(self._drawn), sp)
            self._push(x)
        return ScopeTicks(end_index, start)

    def curve(self, stream=None):
        """The curves the widgets hold after the last call (ScopeCurve), copies made on the call's
        stream without waiting for it.  Before any tick: all three None."""
        if self._curve is None:
            return ScopeCurve(None, None, None)
        S, nch = self.n_scopes, self.n_channels
        with _lib.call_stream(self._curve.device, stream):
            c = self._curve.view(S, nch, -1)
            y2 = c[:, 1].clone() if nch == 2 else None
            return ScopeCurve(c[:, 0].clone(), y2, self._drawn.clone())
