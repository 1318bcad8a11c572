"""What the spectrum and octave widgets draw, for many channels on the GPU: the plotted curve of the
dB vector, its colour intensity and the held peaks (``SpectrumPlotWidget.setdata`` and
``compute_peaks``, friture/spectrumPlotWidget.py:122-200; ``HistPlot.setdata`` and
``compute_peaks``, friture/histplot.py:77-130).

The per-bin work -- the peak state machine carried in float64 from call to call, the vertical
scaling and the intensity -- runs in one CUDA kernel (``frt_plot_curves``, ``csrc/reduce.cu``).
The horizontal edges depend only on the settings and are computed here on the host, once per
settings change, as are the frequency trackers' positions and text and the bar labels' x
positions.

The peak state is reset (peak -500 dB, intensity 0, decay d0) on the first call that computes peaks
and whenever the number of bins changes, as ``compute_peaks`` does when ``len(peak) != len(y)``."""
from __future__ import annotations

from ctypes import c_double
from dataclasses import dataclass
from functools import cached_property

import numpy as np

from . import _lib
from .audioproc import SAMPLING_RATE
from .display import Linear, Logarithmic, Mel

PEAK_DECAY_RATE = 1.0 - 3e-6                               # spectrumPlotWidget.py:19, histplot.py:31
PEAK_DECAY = 20.0 * np.log10(PEAK_DECAY_RATE) * 5000      # d0, the first step of a fall (~ -0.13 dB)


def to_screen(scale, coord_min, coord_max, x):
    """CoordinateTransform.toScreen with length 1 and no borders (plotting/coordinateTransform.py:
    62-83), including the Logarithmic scale's own clipped branch."""
    length, start, end = 1, 0, 0
    if scale is Logarithmic:
        clipped_min = max(1e-20, coord_min)
        clipped_max = max(clipped_min, coord_max)
        if clipped_min == clipped_max:
            return start + 0. * x
        ratio_log = np.log10(clipped_max / clipped_min)
        x = (x < 1e-20) * 1e-20 + (x >= 1e-20) * x
        return np.log10(x / clipped_min) * (length - start - end) / ratio_log + start
    if coord_max == coord_min:
        return start + 0. * x
    trans_x = scale.transform(x)
    trans_min = scale.transform(coord_min)
    trans_max = scale.transform(coord_max)
    return (trans_x - trans_min) * (length - start - end) / (trans_max - trans_min) + start


def frequency_to_note(freq):
    """friture/pitch_tracker_data.py:26-34."""
    if np.isnan(freq) or freq <= 0:
        return ""
    semitone = round(np.log2(freq / 440) * 12) + 9
    octave = int(np.floor(semitone / 12)) + 4
    notes = ["C", "C♯", "D", "D♯", "E", "F", "F♯", "G", "G♯", "A", "A♯", "B"]
    return f'{notes[semitone % 12]}{octave}'


def format_frequency(freq):
    """friture/pitch_tracker_data.py:36-40."""
    if freq < 1000:
        return f'{freq:.0f} Hz ({frequency_to_note(freq)})'
    return f'{freq / 1000:.1f} kHz ({frequency_to_note(freq)})'


@dataclass
class Curves:
    """One call's drawing data.  ``x_left`` / ``x_right`` (host float64 [K], shared by all channels)
    and ``baseline`` are in screen units; ``y``, ``z``, ``peak``, ``z_peak`` are CUDA float32
    tensors [C, K]: the signal curve, its intensity, the peak curve and the peak intensity after the
    call's last dB vector.  ``peak`` and ``z_peak`` are None when peaks are disabled (the widget
    removes its peak curve)."""
    x_left: np.ndarray
    x_right: np.ndarray
    baseline: float
    y: object
    z: object
    peak: object = None
    z_peak: object = None


@dataclass
class SpectrumCurves(Curves):
    """Plus the frequency trackers (spectrumPlotWidget.py:124-134), per channel: the peak and pitch
    frequencies (host float64 [C], Hz) and their screen positions (host float64 [C]).  The trackers'
    text is formatted on first access of ``fmax_text`` / ``fpitch_text`` (about 8 us per channel in
    Python), so a tick whose text nobody reads does not pay for it."""
    fmax_hz: np.ndarray = None
    fpitch_hz: np.ndarray = None
    fmax_x: np.ndarray = None
    fpitch_x: np.ndarray = None

    @cached_property
    def fmax_text(self):
        """spectrumPlotWidget.py:124-127, per channel."""
        return ["%.1f Hz" % f if f < 2e2 else "%d Hz" % np.rint(f) for f in self.fmax_hz]

    @cached_property
    def fpitch_text(self):
        """format_frequency (pitch_tracker_data.py:36-40), per channel."""
        return [format_frequency(f) for f in self.fpitch_hz]


@dataclass
class HistCurves(Curves):
    """Plus the bar labels (histplot.py:98-99): x positions (host float64 [K]) and nominal band
    frequencies; the labels' heights are ``y``."""
    bar_label_x: np.ndarray = None
    bar_label_f: np.ndarray = None


class _PlotState:
    """The vertical range, the pause flag and the float64 peak state [C, K] on the device."""

    def __init__(self, n_channels, spec_min, spec_max, handle):
        self.n_channels = int(n_channels)
        self._handle = handle
        self.paused = False
        self.peak = self.peak_int = self.peak_decay = None
        self._last = None
        self.setspecrange(spec_min, spec_max)

    handle = _lib.shared_handle

    def setspecrange(self, spec_min, spec_max):
        """New vertical range from the next call on; the peak state is kept."""
        if spec_min > spec_max:
            spec_min, spec_max = spec_max, spec_min
        self.spec_min, self.spec_max = spec_min, spec_max

    def pause(self):
        self.paused = True

    def restart(self):
        self.paused = False

    def _run(self, y, peaks):
        """y: CUDA float32 [C, n_steps, K], contiguous along K.  Returns (y, z, peak, z_peak)."""
        import torch
        if not isinstance(y, torch.Tensor) or y.dim() != 3:
            raise ValueError("dB must be a CUDA float32 tensor [C, n_steps, K]")
        C, S, K = y.shape
        if C != self.n_channels or S == 0 or K == 0:
            raise ValueError("expected [%d, n_steps >= 1, K >= 1] dB, got %s" % (self.n_channels, tuple(y.shape)))
        _lib.check_tensor(self, y, "dB")
        if K > 1 and y.stride(2) != 1:
            y = y.contiguous()
        h = self.handle
        dev = y.device
        with _lib.call_stream(dev) as sp:
            out = [torch.empty((C, K), dtype=torch.float32, device=dev) for _ in range(4 if peaks else 2)]
            state = (self.peak, self.peak_int, self.peak_decay)
            reset = peaks and (self.peak is None or self.peak.shape[1] != K)
            if reset:
                # kept aside until the call is accepted: a rejected call must not leave a state of the
                # new size that the next call would read without the reset
                state = tuple(torch.empty((C, K), dtype=torch.float64, device=dev) for _ in range(3))
            st = [_lib._ptr(t) if peaks else None for t in state]
            h.call("frt_plot_curves", _lib._ptr(y), int(y.stride(0)), int(y.stride(1)), int(C), int(S),
                   int(K), c_double(self.spec_min), c_double(self.spec_max), c_double(PEAK_DECAY),
                   1 if peaks else 0, 1 if reset else 0, *st, *[_lib._ptr(t) for t in out],
                   *([None, None] if not peaks else []), sp)
        if reset:
            self.peak, self.peak_int, self.peak_decay = state
        return out + [None] * (4 - len(out))


class SpectrumPlot(_PlotState):
    """``SpectrumPlotWidget`` for ``n_channels`` channels.  Defaults are the spectrum widget's
    (friture/spectrum.py:51-75, spectrum_settings.py:27-35): Mel scale over 20-20000 Hz, -100 to
    -20 dB, peaks on, baseline at the plot bottom."""

    def __init__(self, n_channels, freqscale=Mel, minfreq=20., maxfreq=20000., spec_min=-100.,
                 spec_max=-20., handle=None):
        super().__init__(n_channels, spec_min, spec_max, handle)
        self.scale = freqscale
        self.xmin, self.xmax = minfreq, maxfreq
        self.peaks_enabled = True
        self.data_baseline = False
        self._edges = None

    # -- the widget's setters ---------------------------------------------------------------
    def setfreqscale(self, scale):
        self.scale = scale
        self._edges = None

    def setfreqrange(self, minfreq, maxfreq):
        self.xmin, self.xmax = minfreq, maxfreq
        self._edges = None

    def set_peaks_enabled(self, enabled):
        """While disabled the peak state stays frozen and no peak curve is returned."""
        self.peaks_enabled = bool(enabled)

    def set_baseline_displayUnits(self, baseline=0.):
        """Curves filled down to the plot bottom (the widget's single-channel mode)."""
        self.data_baseline = False

    def set_baseline_dataUnits(self, baseline=0.):
        """Curves filled down to 0 dB (the widget's dual-channel mode)."""
        self.data_baseline = True

    def setdualchannels(self, dual_enabled):
        """Spectrum_Widget.setdualchannels (friture/spectrum.py:286-293): dual mode turns the peaks
        off and fills down to 0 dB; single mode turns them back on over the plot bottom."""
        self.set_peaks_enabled(not dual_enabled)
        if dual_enabled:
            self.set_baseline_dataUnits(0.)
        else:
            self.set_baseline_displayUnits(0.)

    # -- one tick ----------------------------------------------------------------------------
    def edges(self, nbins):
        """Screen x of the bins' left and right edges for ``nbins`` bins of the analyzer's frequency
        axis linspace(0, fs // 2, nbins) (audioproc.py), spectrumPlotWidget.py:144-151."""
        key = (self.scale, self.xmin, self.xmax, nbins)
        if self._edges is None or self._edges[0] != key:
            x = np.linspace(0, SAMPLING_RATE // 2, nbins)
            x_left = np.zeros(x.shape)
            x_right = np.zeros(x.shape)
            x_left[0] = 1e-10
            x_left[1:] = (x[1:] + x[:-1]) / 2.0
            x_right[:-1] = x_left[1:]
            x_right[-1] = float(SAMPLING_RATE / 2)
            self._edges = (key, to_screen(self.scale, self.xmin, self.xmax, x_left),
                           to_screen(self.scale, self.xmin, self.xmax, x_right))
        return self._edges[1], self._edges[2]

    def push(self, db, fmax, fpitch, n_frames=1):
        """``SpectrumAnalyzer.process``'s outputs of one tick: db CUDA float32 [C, K], fmax and
        fpitch [C] Hz.  ``n_frames`` is the tick's frame count: the widget draws only ticks with at
        least one frame (friture/spectrum.py:140), so with 0, as while paused, nothing changes and
        the previous call's curves are returned (None before the first)."""
        if self.paused or n_frames == 0:
            return self._last
        if db.dim() != 2:
            raise ValueError("db must be [C, K]")
        fmax, fpitch = self._trackers(fmax, fpitch)
        return self._publish(self._run(db[:, None, :], self.peaks_enabled), db.shape[1], fmax, fpitch)

    def push_ticks(self, ticks):
        """``SpectrumAnalyzer.process_ticks``'s outputs (a ``SpectrumTicks`` with dB): the widget's
        setdata once per tick, in tick order, in one launch -- the peak state steps through every
        tick.  The curves are those after the last tick, with that tick's frequency trackers: the
        same as one ``push`` per tick.  With no ticks, or while paused, nothing changes and the
        previous call's curves are returned (None before the first)."""
        if self.paused:
            return self._last
        db = ticks.db
        if db is None:
            raise ValueError("the ticks carry no dB (process_ticks was called with want_db=False)")
        if db.dim() != 3:
            raise ValueError("db must be [C, n_ticks, K]")
        if db.shape[1] == 0:
            return self._last
        fmax, fpitch = self._trackers(ticks.fmax_hz[-1], ticks.fpitch_hz[-1])
        return self._publish(self._run(db, self.peaks_enabled), db.shape[2], fmax, fpitch)

    def _trackers(self, fmax, fpitch):
        return (np.broadcast_to(np.asarray(fmax, dtype=np.float64), (self.n_channels,)),
                np.broadcast_to(np.asarray(fpitch, dtype=np.float64), (self.n_channels,)))

    def _publish(self, curves, nbins, fmax, fpitch):
        """The drawing data of one call from its curves and its last tick's frequency trackers."""
        y, z, peak, z_peak = curves
        x_left, x_right = self.edges(nbins)
        baseline = 1.0 - to_screen(Linear, self.spec_min, self.spec_max, 0.0) if self.data_baseline else 1.0
        self._last = SpectrumCurves(
            x_left, x_right, baseline, y, z, peak, z_peak, fmax_hz=fmax, fpitch_hz=fpitch,
            fmax_x=np.asarray(to_screen(self.scale, self.xmin, self.xmax, fmax), dtype=np.float64),
            fpitch_x=np.asarray(to_screen(self.scale, self.xmin, self.xmax, fpitch), dtype=np.float64))
        return self._last


class HistPlot(_PlotState):
    """``HistPlot`` for ``n_channels`` channels, drawing the bands of ``analyzer`` (an
    ``OctaveSpectrumAnalyzer``; its band edges and nominal frequencies are read at every call, so
    ``setbandsperoctave`` on it carries over).  Defaults are the octave widget's
    (friture/octavespectrum_settings.py:25-26): -80 to -20 dB."""

    def __init__(self, n_channels, analyzer, spec_min=-80., spec_max=-20., handle=None):
        super().__init__(n_channels, spec_min, spec_max, handle)
        self.analyzer = analyzer
        self._edges = None

    def edges(self):
        """Screen x of the bands' edges, Logarithmic over 44-22000 Hz (histplot.py:63-67,81-82)."""
        a = self.analyzer
        if self._edges is None or self._edges[0] is not a.flow:
            x_left = to_screen(Logarithmic, 44, 22000, np.asarray(a.flow))
            x_right = to_screen(Logarithmic, 44, 22000, np.asarray(a.fhigh))
            self._edges = (a.flow, x_left, x_right, (x_left + x_right) / 2)
        return self._edges[1:]

    def push(self, db):
        """``OctaveSpectrumAnalyzer.process(..., db=True)``'s [C, n_blocks, nbands]: the widget's
        setdata once per block, in block order (the state steps through every block); the curves
        are those after the last block.  While paused nothing changes and the previous call's
        curves are returned (None before the first)."""
        if self.paused:
            return self._last
        if db.dim() != 3:
            raise ValueError("db must be [C, n_blocks, nbands]")
        x_left, x_right, bar_x = self.edges()
        if len(x_left) != db.shape[2]:
            raise ValueError("db has %d bands, the analyzer %d" % (db.shape[2], len(x_left)))
        y, z, peak, z_peak = self._run(db, True)
        self._last = HistCurves(x_left, x_right, 1., y, z, peak, z_peak, bar_label_x=bar_x,
                                bar_label_f=np.asarray(self.analyzer.f_nominal))
        return self._last
