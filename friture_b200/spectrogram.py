"""The spectrogram widget for many channels, from stream chunks to screen pixels: the numeric part of
``Spectrogram_Widget.handle_new_data`` (friture/spectrogram.py:131-173) with its setters.

Each call frames the stream as the widget does (the frame of ``fft_size`` samples ending at
``old_index``, then ``old_index += fft_size/4``; zeros before the stream starts), transforms every
frame straight to its screen rows (``frt_stft_screen_rows``: the log-power column stays on chip) and
resamples those rows to screen columns with the colour look-up (``SpectrogramDisplay.push_rows``).
The pixels are bit for bit those of ``SpectrogramDisplay.push(audioproc.stft(frames, fft_size/4,
log=True))`` on the same frames, without the full-resolution column going through memory.
"""
from __future__ import annotations

from collections import namedtuple
from ctypes import c_float

from . import _lib
from .audioproc import SAMPLING_RATE
from .display import Mel, SpectrogramDisplay
from .stream import StreamFramer

SpectrogramOutput = namedtuple("SpectrogramOutput", "pixels rows n_frames")
SpectrogramOutput.__doc__ = """One ``handle_new_data`` call: pixels int32 [C, height, n_out]
(0xAARRGGBB), rows float32 [C, n_frames, height] (the frames' unclipped screen values, or None unless
asked for) and the number of frames the call transformed."""


class SpectrogramAnalyzer:
    """``Spectrogram_Widget`` for ``n_channels`` channels on one GPU.  Defaults are the widget's
    (friture/spectrogram_settings.py:27-34, overlap 3/4).

    Setters apply to later calls only and never read device data.  A height change restarts the
    carried column (``SpectrogramDisplay.set_screen``; the reference resamples it instead)."""

    HISTORY = 16384   # samples kept before old_index: the widget's largest FFT size

    def __init__(self, n_channels, fft_size=4096, freqscale=Mel, minfreq=20., maxfreq=SAMPLING_RATE / 2,
                 spec_min=-140., spec_max=0., weighting=0, height=512, width=1024, timerange_s=10.,
                 handle=None):
        self.n_channels = int(n_channels)
        _check_fft_size(fft_size)
        self.display = SpectrogramDisplay(self.n_channels, fft_size=fft_size, freqscale=freqscale,
                                          minfreq=minfreq, maxfreq=maxfreq, spec_min=spec_min,
                                          spec_max=spec_max, weighting=weighting, height=height, width=width,
                                          timerange_s=timerange_s, handle=handle)
        self._framer = None

    @property
    def handle(self):
        return self.display.handle

    @property
    def fft_size(self):
        return self.display.fft_size

    @property
    def hop(self):
        return self.display.fft_size // 4       # spectrogram.py:141, overlap 3/4

    @property
    def old_index(self):
        return self._framer.old_index if self._framer is not None else 0

    # ------------------------------------------------------------------ setters (spectrogram.py:203-257)
    def setfftsize(self, fft_size):
        _check_fft_size(fft_size)
        self.display.set_fftsize(fft_size)
        if self._framer is not None:
            self._framer.set_geometry(fft_size, fft_size // 4)

    def setminfreq(self, freq):
        d = self.display
        d.set_rows(d.scale, freq, d.maxfreq, d.weighting)

    def setmaxfreq(self, freq):
        d = self.display
        d.set_rows(d.scale, d.minfreq, freq, d.weighting)

    def setfreqscale(self, freqscale):
        d = self.display
        d.set_rows(freqscale, d.minfreq, d.maxfreq, d.weighting)

    def setweighting(self, weighting):
        d = self.display
        d.set_rows(d.scale, d.minfreq, d.maxfreq, weighting)

    def setmin(self, value):
        self.display.spec_min = float(value)

    def setmax(self, value):
        self.display.spec_max = float(value)

    def timerangechanged(self, value):
        self.display.timerange_s = value

    def set_screen(self, height, width):
        self.display.set_screen(height, width)

    # ------------------------------------------------------------------ the widget's tick
    def handle_new_data(self, chunk, want_rows=False, stream=None):
        """Push ``chunk`` (CUDA float32 [C, n]) and return the screen columns of every frame that is
        now complete, as a ``SpectrogramOutput``.  A call without a complete frame returns pixels
        [C, height, 0] and leaves the display's state as it was."""
        import torch
        x, _ = _lib.device_rows(self, chunk, "chunk")
        if x.shape[0] != self.n_channels:
            raise ValueError("chunk must have %d channels" % self.n_channels)
        d = self.display
        with _lib.call_stream(x.device, stream) as sp:
            if self._framer is None:
                self._framer = StreamFramer(self.n_channels, self.fft_size, self.hop, x.device,
                                            capacity=2 * self.HISTORY, history=self.HISTORY)
            fr = self._framer
            fr.push(x)
            view, F = fr.take()
            H = d.height
            if F == 0:
                empty = torch.empty((self.n_channels, H, 0), dtype=torch.int32, device=x.device)
                return SpectrogramOutput(empty, None, 0)
            T = d.tables(x.device)
            rows = torch.empty((self.n_channels, F, H), dtype=torch.float32, device=x.device)
            self.handle.call("frt_stft_plan", int(self.fft_size))
            self.handle.call("frt_stft_screen_rows", _lib._ptr(view), int(view.stride(0)), self.n_channels,
                             int(F), int(self.hop), _lib._ptr(T["w"]), c_float(d.spec_min), c_float(d.spec_max),
                             _lib._ptr(T["i0"]), _lib._ptr(T["t"]), int(H), _lib._ptr(rows), int(F * H), int(H),
                             sp)
            pixels = d.push_rows(rows, stream=sp.value)
        return SpectrogramOutput(pixels, rows if want_rows else None, F)


def _check_fft_size(n):
    # the widget offers 32 * 2^k, k = 0..9 (spectrogram_settings.py)
    if n not in [32 << k for k in range(10)]:
        raise ValueError("fft_size must be 32, 64, .., 16384")
