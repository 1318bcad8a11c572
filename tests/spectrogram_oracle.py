"""Spectrogram_Widget.handle_new_data (friture/spectrogram.py:131-173) and its setters (:203-257) for
one channel over a chunked stream, in float64, composed from the oracle pieces that
tests/test_display_host.py pins against the reference: stft_power, log_spectrogram,
frequency_resample, OnlineLinear2DResamplerOracle and color_transform.

One deviation, shared with SpectrogramAnalyzer and documented there: a height change restarts the
carried column instead of resampling it (Online_Linear_2D_resampler.set_height)."""
from fractions import Fraction

import numpy as np

from oracle import friture_oracle as fo

SAMPLING_RATE = 48000


class SpectrogramWidgetOracle:
    def __init__(self, fft_size=4096, freqscale=None, minfreq=20., maxfreq=SAMPLING_RATE / 2, spec_min=-140.,
                 spec_max=0., weighting=0, height=512, width=1024, timerange_s=10., lut=None):
        from friture_b200.display import Mel, load_lut
        self.fft_size = fft_size
        self.scale = freqscale or Mel
        self.minfreq, self.maxfreq = minfreq, maxfreq
        self.spec_min, self.spec_max = spec_min, spec_max
        self.weighting = weighting
        self.height, self.width = height, width
        self.timerange_s = timerange_s
        self.lut = load_lut() if lut is None else lut
        self.x = np.zeros(0)          # the whole stream so far (RingBuffer with unbounded length)
        self.old_index = 0
        self.res = None               # OnlineLinear2DResamplerOracle
        self.res_LM = None

    # setters: the widget's, each changing only what it changes
    def setfftsize(self, n):
        self.fft_size = n

    def setminfreq(self, f):
        self.minfreq = f

    def setmaxfreq(self, f):
        self.maxfreq = f

    def setfreqscale(self, s):
        self.scale = s

    def setmin(self, v):
        self.spec_min = v

    def setmax(self, v):
        self.spec_max = v

    def setweighting(self, w):
        self.weighting = w

    def timerangechanged(self, v):
        self.timerange_s = v

    def set_screen(self, height, width):
        if height != self.height:
            self.height = height
            self.res = None           # the carried column restarts (see the module docstring)
        self.width = width

    def push(self, chunk):
        """Append ``chunk`` and run one handle_new_data.  Returns (pixels uint32 [H, n_out], screen
        rows [H, F] before the time resampling, F, the resampled values [H, n_out] behind the pixels)."""
        self.x = np.concatenate([self.x, np.asarray(chunk, dtype=np.float64)])
        N, H = self.fft_size, self.height
        hop = N // 4
        realizable = (len(self.x) - self.old_index) // hop
        if realizable <= 0:
            return np.zeros((H, 0), dtype=self.lut.dtype), np.zeros((H, 0)), 0, np.zeros((H, 0))
        # frame i ends at old_index + i*hop (data_indexed); zeros before the stream starts
        start = self.old_index - N
        seg = self.x[max(start, 0):self.old_index + (realizable - 1) * hop]
        seg = np.concatenate([np.zeros(max(-start, 0)), seg])
        spn = fo.stft_power(seg, N, hop).T                         # [bins, F]
        self.old_index += realizable * hop
        freq = np.linspace(0, SAMPLING_RATE // 2, N // 2 + 1)
        A, B, C = fo.weighting_tables(freq)
        w = [np.zeros_like(freq), A, B, C][self.weighting]
        norm = (fo.log_spectrogram(spn) + w[:, None] - self.spec_min) / (self.spec_max - self.spec_min)
        s = self.scale
        xscaled = s.inverse(np.linspace(s.transform(self.minfreq), s.transform(self.maxfreq), H))
        rows = fo.frequency_resample(norm, freq, np.atleast_1d(xscaled))
        LM = (Fraction(SAMPLING_RATE, N) / Fraction(1, 4) / 1000,
              Fraction(max(self.width, 1), int(self.timerange_s * 1000)))
        if self.res is None:
            self.res = fo.OnlineLinear2DResamplerOracle(*LM, H)
        elif LM != self.res_LM:       # set_ratio: the indices restart, the carried column stays
            old = self.res.old_data
            self.res = fo.OnlineLinear2DResamplerOracle(*LM, H)
            self.res.old_data = old
        self.res_LM = LM
        data = self.res.push(rows)
        return fo.color_transform(self.lut, data), rows, realizable, data
