"""Spectrogram display chain on the GPU (friture/spectrogram.py:161-173): log-power columns ->
weighting + [0,1] scaling -> frequency-axis interpolation to the screen rows -> online linear
resampling along time to the screen columns -> colour look-up (RGB32), for many channels at once.

The frequency scales, the screen-row table and the time resampler's index bookkeeping are host
logic restated from the reference (friture/plotting/frequency_scales.py,
friture/signal/frequency_resampler.py, friture/signal/online_linear_2D_resampler.py); the
per-pixel arithmetic runs in one CUDA kernel (``csrc/reduce.cu``)."""
from __future__ import annotations

import os
from ctypes import c_float
from fractions import Fraction

import numpy as np

from . import _lib
from .audioproc import SAMPLING_RATE, audioproc


# ---- frequency scales (transform / inverse pairs of friture/plotting/frequency_scales.py) ----
class Linear:
    NAME = "Linear"
    transform = staticmethod(lambda f: f)                                   # :69-76
    inverse = staticmethod(lambda v: v)


class Logarithmic:
    NAME = "Logarithmic"
    transform = staticmethod(lambda f: np.log10(f))                         # :144-149
    inverse = staticmethod(lambda v: 10 ** v)


class Octave:
    NAME = "Octave"
    transform = staticmethod(lambda f: np.log2(np.fmax(f, 1e-20)))          # :196-201
    inverse = staticmethod(lambda v: 2 ** v)


class Mel:
    NAME = "Mel"
    transform = staticmethod(lambda f: 2595 * np.log10(1 + f / 700))        # :266-271
    inverse = staticmethod(lambda m: 700 * (10 ** (m / 2595) - 1))


class Erb:
    NAME = "ERB"
    A = 21.33228113095401739888262
    transform = staticmethod(lambda f: Erb.A * np.log10(1 + 0.00437 * f))   # :284-289
    inverse = staticmethod(lambda e: (10 ** (e / Erb.A) - 1) / 0.00437)


SCALES = {0: Linear, 1: Logarithmic, 2: Mel, 3: Erb, 4: Octave}


def screen_rows(freq, scale, minfreq, maxfreq, nsamples):
    """Frequency_Resampler.update_xscale + the index/fraction np.interp would use
    (friture/signal/frequency_resampler.py:44-49,67-83).  Returns (xscaled, i0, t)."""
    xscaled = scale.inverse(np.linspace(scale.transform(minfreq), scale.transform(maxfreq), nsamples))
    xscaled = np.atleast_1d(np.asarray(xscaled, dtype=np.float64))
    freq = np.asarray(freq, dtype=np.float64)
    i0 = np.clip(np.searchsorted(freq, xscaled, side="right") - 1, 0, len(freq) - 2)
    t = np.clip((xscaled - freq[i0]) / (freq[i0 + 1] - freq[i0]), 0.0, 1.0)
    return xscaled, i0.astype(np.int32), t


class OnlineResamplerIndex:
    """Index bookkeeping of Online_Linear_2D_resampler (online_linear_2D_resampler.py:19-97):
    which input column each output column is drawn from and the weight `a` of the previous one."""

    def __init__(self, interp_factor_L=1, decim_factor_M=1):
        self.interp_factor_L = interp_factor_L
        self.decim_factor_M = decim_factor_M
        self.resampling_ratio = float(interp_factor_L) / decim_factor_M
        self.orig_index = 0.
        self.resampled_index = 0.

    def set_ratio(self, interp_factor_L, decim_factor_M):
        if self.interp_factor_L != interp_factor_L or self.decim_factor_M != decim_factor_M:
            self.interp_factor_L = interp_factor_L
            self.decim_factor_M = decim_factor_M
            self.resampling_ratio = float(interp_factor_L) / decim_factor_M
            self.orig_index = 0.
            self.resampled_index = 0.

    def reset(self):
        self.orig_index = 0.
        self.resampled_index = 0.

    def processable(self, m):
        return int(np.ceil((self.orig_index + m - (self.resampled_index + self.resampling_ratio))
                           / self.resampling_ratio))

    def push(self, n_columns):
        """(cols int32[n_out], a float64[n_out]) for a tick of n_columns input columns."""
        cols, avals = [], []
        for j in range(n_columns):
            self.orig_index += 1.
            n = self.processable(0)
            if n <= 0:
                continue
            new_indices = self.resampled_index + self.resampling_ratio * np.arange(1, n + 1, dtype=np.float64)
            a = self.orig_index - new_indices                       # linear_interp.py:50-51
            cols += [j] * n
            avals += list(a)
            self.resampled_index = float(new_indices[-1])
        return np.asarray(cols, dtype=np.int32), np.asarray(avals, dtype=np.float64)


def _upload(arr, device):
    """Host array -> device tensor, ordered on the current stream without blocking the host: a copy
    from pageable memory would first wait for the work already queued on the stream."""
    import torch
    return torch.from_numpy(np.ascontiguousarray(arr)).pin_memory().to(device, non_blocking=True)


def load_lut():
    path = os.path.join(os.path.dirname(os.path.abspath(__file__)), "data", "cmrmap.npz")
    with np.load(path) as d:
        return d["lut"].astype(np.uint32)


class SpectrogramDisplay:
    """Spectrogram_Widget's transform pipeline for C channels.  ``push(db)`` takes the tick's
    log-power columns [C, F, bins] (``audioproc.stft(..., log=True)``) and returns the new screen
    columns as an int32 CUDA tensor [C, height, n_out] holding 0xAARRGGBB words.  ``push_rows(rows)``
    does the same from rows already interpolated to the screen height ([C, F, height],
    ``frt_stft_screen_rows`` with this object's ``tables``)."""

    def __init__(self, n_channels, fft_size=4096, freqscale=Mel, minfreq=20., maxfreq=SAMPLING_RATE / 2,
                 spec_min=-140., spec_max=0., weighting=0, height=512, width=1024, timerange_s=10.,
                 overlap_frac=Fraction(3, 4), handle=None):
        self.n_channels = int(n_channels)
        self._handle = handle
        self.proc = audioproc(handle)          # only for freq / weighting tables (host side)
        self.fft_size = fft_size
        self.proc.fft_size = 0
        self.proc.set_fftsize(fft_size)
        self.freq = self.proc.get_freq_scale()
        self.scale = freqscale
        self.minfreq, self.maxfreq = minfreq, maxfreq
        self.spec_min, self.spec_max = float(spec_min), float(spec_max)
        self.weighting = weighting
        self.height, self.width = int(height), int(width)
        self.timerange_s = timerange_s
        # spectrogram.py:98,166-167: input columns per ms / screen columns per ms
        self.overlap_frac = overlap_frac
        self.sfft_rate_frac = Fraction(SAMPLING_RATE, fft_size) / (Fraction(1) - overlap_frac) / 1000
        self.index = OnlineResamplerIndex()
        self._tables = None
        self._old = None

    handle = _lib.shared_handle

    def set_screen(self, height, width):
        if height != self.height:
            self.height = int(height)
            self._tables = None
            self._old = None                  # (the reference resamples the carried column; we restart it)
            self.index.reset()                # online_linear_2D_resampler.py:46-57
        self.width = int(width)

    def set_fftsize(self, fft_size):
        """Spectrogram_Widget.setfftsize (friture/spectrogram.py:225-238): new bin frequencies and
        weighting tables, and a new input-column rate, which restarts the resampler's index on the
        next push (set_ratio).  The carried column is on the screen grid and is kept."""
        if fft_size != self.fft_size:
            self.fft_size = fft_size
            self.proc.set_fftsize(fft_size)
            self.freq = self.proc.get_freq_scale()
            self.sfft_rate_frac = Fraction(SAMPLING_RATE, fft_size) / (Fraction(1) - self.overlap_frac) / 1000
            self._tables = None

    def set_rows(self, freqscale, minfreq, maxfreq, weighting):
        """Frequency scale, range and weighting (setfreqscale / setminfreq / setmaxfreq /
        setweighting, friture/spectrogram.py:203-249): the screen-row and weighting tables are
        rebuilt on the next push; nothing else is reset."""
        self.scale, self.minfreq, self.maxfreq, self.weighting = freqscale, minfreq, maxfreq, weighting
        self._tables = None

    def tables(self, device):
        """The screen-row table (``i0`` int32, ``t`` float32 [height]), the weighting (``w`` float32
        [bins] or None) and the LUT on ``device``, built for the current settings."""
        self._ensure(device)
        return self._tables

    def _ensure(self, device):
        import torch
        screen_rate_frac = Fraction(max(self.width, 1), int(self.timerange_s * 1000))
        self.index.set_ratio(self.sfft_rate_frac, screen_rate_frac)      # spectrogram.py:166-167
        if self._tables is None:
            _, i0, t = screen_rows(self.freq, self.scale, self.minfreq, self.maxfreq, self.height)
            A, B, C = self.proc.get_freq_weighting()
            w = [None, A, B, C][self.weighting]
            self._tables = {
                "i0": _upload(i0, device),
                "t": _upload(t.astype(np.float32), device),
                "w": None if w is None else _upload(np.asarray(w, dtype=np.float32), device),
                "lut": _upload(load_lut().view(np.int32), device),
            }
        if self._old is None:
            self._old = torch.zeros((self.n_channels, self.height), dtype=torch.float32, device=device)

    def push(self, db, stream=None):
        return self._push("frt_display_columns", db, "db", len(self.freq), stream, lambda T: (
            _lib._ptr(T["w"]), c_float(self.spec_min), c_float(self.spec_max), _lib._ptr(T["i0"]), _lib._ptr(T["t"]),
            int(self.height)))

    def push_rows(self, rows, stream=None):
        """``push`` for rows already on the screen grid: rows [C, F, height] contiguous CUDA float32,
        made with this object's current ``tables`` and dB range."""
        return self._push("frt_display_rows", rows, "rows", self.height, stream, lambda T: ())

    def _push(self, fn, x, name, width, stream, table_args):
        """What push and push_rows share: x [C, F, width] is checked, the time resampler advances by F
        columns and ``fn`` (frt_display_columns or frt_display_rows) draws them, with ``table_args(tables)``
        between the input's shape and the resampler's arguments."""
        import torch
        if x.dim() != 3 or x.shape[0] != self.n_channels or x.shape[2] != width:
            raise ValueError("%s must be [%d, F, %d]" % (name, self.n_channels, width))
        if not x.is_contiguous():
            raise ValueError("%s must be a contiguous CUDA float32 tensor" % name)
        _lib.check_tensor(self, x, name)
        C, F, W = x.shape
        with _lib.call_stream(x.device, stream) as sp:
            self._ensure(x.device)
            cols, a = self.index.push(F)
            n_out = len(cols)
            pixels = torch.empty((C, self.height, n_out), dtype=torch.int32, device=x.device)
            if F == 0:
                return pixels
            cols_d = _upload(cols, x.device) if n_out else None
            a_d = _upload(a.astype(np.float32), x.device) if n_out else None
            self.handle.call(fn, _lib._ptr(x), int(F * W), int(W), int(C), int(F), int(W), *table_args(self._tables),
                             _lib._ptr(cols_d), _lib._ptr(a_d), int(n_out), _lib._ptr(self._old),
                             _lib._ptr(self._tables["lut"]), _lib._ptr(pixels) if n_out else None, sp)
        return pixels
