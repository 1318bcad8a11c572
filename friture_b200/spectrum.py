"""Numeric part of ``Spectrum_Widget`` (friture/spectrum.py:125-222) for many channels on the GPU:
framing + ``analyzelive`` per frame, exponential smoothing across the tick's frames, weighting,
dB, peak frequency and harmonic-product-spectrum pitch -- one smoothed column per channel per
tick instead of one column per frame (this is what the display consumes, and it shrinks what a
multi-GPU gather has to move from ``frames x bins`` to ``bins`` per channel).

With ``dual_channels`` (the widget's "Measurement type: Dual-channel", spectrum.py:141-171,286-293)
each channel is a (reference, measurement) pair and the output is the transfer function between
the two."""
from __future__ import annotations

from ctypes import c_float
from dataclasses import dataclass

import numpy as np

from . import _lib
from .audioproc import FRAMES_PER_BUFFER, SAMPLING_RATE, audioproc, frame_count
from .stream import StreamFramer

DEFAULT_FFT_SIZE = 8192        # friture/spectrum_settings.py:27 (2**7 * 32 ... the widget default)
DEFAULT_RESPONSE_TIME = 0.025  # friture/spectrum_settings.py
OVERLAP = 0.75                 # friture/spectrum.py:66
MAX_FRAMES_PER_TICK = 8192     # the frames one tick may smooth (the reference's 8192-tap kernel)
STREAM_HISTORY = 16384         # samples handle_new_data keeps before old_index: the largest FFT size


@dataclass
class SpectrumTicks:
    """``SpectrumAnalyzer.process_ticks``'s and ``handle_new_data``'s outputs, one row per tick: ``db``
    CUDA float32 [C, R, bins] (None when not requested), ``fmax_hz`` and ``fpitch_hz`` host float64
    [R, C].  From ``handle_new_data`` also ``tick`` [R], which buffer of the call each row belongs to,
    and ``n_frames`` [R], the frames it smoothed (None from ``process_ticks``)."""
    db: object
    fmax_hz: np.ndarray
    fpitch_hz: np.ndarray
    tick: np.ndarray = None
    n_frames: np.ndarray = None


class SpectrumAnalyzer:
    def __init__(self, n_channels, fft_size=DEFAULT_FFT_SIZE, overlap=OVERLAP,
                 response_time=DEFAULT_RESPONSE_TIME, weighting=0, handle=None, dual_channels=False):
        self.n_channels = int(n_channels)
        self.proc = audioproc(handle)
        self.overlap = overlap
        self.weighting = weighting
        self.response_time = response_time
        self.dual_channels = bool(dual_channels)
        self._disp = None
        self._disp2 = None
        self._w_dev = None
        self._framer = None      # handle_new_data's stream, created by its first call
        self._pairs = None       # whether that stream is [C, 2, n]
        self.minfreq = 20.       # friture/spectrum_settings.py defaults
        self.maxfreq = SAMPLING_RATE / 2
        self.setfftsize(fft_size)

    # -- the widget's setters ---------------------------------------------------------------
    def setfftsize(self, fft_size):
        self.fft_size = fft_size
        self.proc.set_fftsize(fft_size)
        self.freq = self.proc.get_freq_scale()
        self.hop = int(self.fft_size * (1. - self.overlap))          # spectrum.py:137,155
        self.setresponsetime(self.response_time)
        self.setweighting(self.weighting)
        self._disp = None                                            # update_display_buffers, :224-226
        self._disp2 = None
        if self._framer is not None:                                 # old_index is kept
            self._framer.set_geometry(self.fft_size, self.hop)

    def setresponsetime(self, response_time):
        # spectrum.py:196-218: the newest n = T*fs/hop frames carry 65 % of the weight
        self.response_time = response_time
        w = 0.65
        n = self.response_time * SAMPLING_RATE / (self.fft_size * (1. - self.overlap))
        self.alpha = 1. - (1. - w) ** (1. / (n + 1))

    def setweighting(self, weighting):
        # 0 none, 1 A, 2 B, 3 C (spectrum.py:240-252)
        self.weighting = weighting
        A, B, C = self.proc.get_freq_weighting()
        self.w = [0. * A, A, B, C][weighting]
        self._w_dev = None

    def setdualchannels(self, dual_enabled):
        """spectrum.py:286-293: changes the mode only; both smoothed states are kept."""
        self.dual_channels = bool(dual_enabled)

    def setminfreq(self, minfreq):
        self.setMinMaxFreq(minfreq, self.maxfreq)

    def setmaxfreq(self, maxfreq):
        self.setMinMaxFreq(self.minfreq, maxfreq)

    def setMinMaxFreq(self, minfreq, maxfreq):
        """spectrum.py:228-249: restarts both smoothed states.  The frequency axis stays: the reference's
        audioproc.set_maxfreq only rebuilds it when the FFT size changes (audioproc.py:83-96)."""
        self.minfreq = minfreq
        self.maxfreq = maxfreq
        self._disp = None                                            # update_display_buffers
        self._disp2 = None

    @property
    def old_index(self):
        """The widget's old_index: where the next frame of ``handle_new_data``'s stream ends."""
        return self._framer.old_index if self._framer is not None else 0

    # -- one tick ----------------------------------------------------------------------------
    def process(self, x, stream=None):
        """x: CUDA float32 [C, T] holding the tick's new frames (frame f = x[:, f*hop : f*hop+N]),
        or [C, 2, T], each channel a pair of rows: row 0 the reference, row 1 the measurement
        (the widget's floatdata[0] and floatdata[1]).
        Returns (dB [C, bins] CUDA tensor, fmax [C] Hz, fpitch [C] Hz) after smoothing across
        the frames, with the smoothing state carried from tick to tick.  In dual-channel mode with
        [C, 2, T] input, dB is the transfer function 10 log10(sp2) - 10 log10(sp1), unweighted, and
        fmax its peak; otherwise dB is 10 log10(sp1) + weighting of row 0.  The pitch always comes
        from row 0 (spectrum.py:180)."""
        import torch
        x, dual = self._input(x)
        C = self.n_channels
        nb = self.fft_size // 2 + 1
        nf = frame_count(x.shape[-1], self.fft_size, self.hop)
        dev = x.device
        with _lib.call_stream(dev, stream) as sp:
            rows = x.view(2 * C, x.shape[-1]) if dual else x
            power = self.proc.stft(rows, hop=self.hop, log=False, stream=stream)
            self._states(dev, dual)
            db = torch.empty((C, nb), dtype=torch.float32, device=dev)
            imax = torch.empty(C, dtype=torch.int32, device=dev)
            ipitch = torch.empty(C, dtype=torch.int32, device=dev)
            h = self.proc.handle
            if dual:
                # power [2C, nf, nb]: pair c's reference at row 2c, its measurement at row 2c + 1
                p1 = power.data_ptr() if nf else 0
                p2 = p1 + 4 * nf * nb if nf else 0
                h.call("frt_spectrum_reduce_dual", _lib._ptr(p1), _lib._ptr(p2), int(2 * nf * nb), int(nb), int(C),
                       int(nf), int(nb), c_float(self.alpha), _lib._ptr(self._disp), _lib._ptr(self._disp2),
                       _lib._ptr(db), _lib._ptr(imax), _lib._ptr(ipitch), sp)
            else:
                h.call("frt_spectrum_reduce", _lib._ptr(power), int(nf * nb), int(nb), int(C), int(nf), int(nb),
                       c_float(self.alpha), _lib._ptr(self._disp),
                       _lib._ptr(self._w_dev) if self.weighting else None, _lib._ptr(db), _lib._ptr(imax),
                       _lib._ptr(ipitch), sp)
                self._decay_unfilled([nf])
            return (db,) + self._indices_to_hz(imax, ipitch)

    def _input(self, x):
        """x as [C, T] or [C, 2, T] and whether it runs in dual mode; [C, 2, T] outside dual mode is
        its reference rows."""
        if x.dim() == 1:
            x = x[None, :]
        if x.dim() not in (2, 3) or (x.dim() == 3 and x.shape[1] != 2):
            raise ValueError("expected [C, T] or [C, 2, T] input, got %s" % (tuple(x.shape),))
        if x.shape[0] != self.n_channels:
            raise ValueError("expected %d channels" % self.n_channels)
        if x.dim() == 3 and self.dual_channels:
            return x, True
        return (x[:, 0] if x.dim() == 3 else x), False

    def default_frames_per_tick(self):
        """The frames of one tick of the widget's feed: one 512-sample buffer per tick
        (friture/audiobackend.py:32), at least one frame."""
        return max(1, FRAMES_PER_BUFFER // self.hop)

    def tick_geometry(self, n_samples, frames_per_tick=None):
        """(frames_per_tick, ticks) of a ``process_ticks`` call over ``n_samples`` samples per row;
        raises FrtValueError unless the frames are a whole number of ticks of 1..8192 frames."""
        g = self.default_frames_per_tick() if frames_per_tick is None else frames_per_tick
        if isinstance(g, (bool, np.bool_)) or not isinstance(g, (int, np.integer)) or \
                not 1 <= g <= MAX_FRAMES_PER_TICK:
            raise _lib.FrtValueError(_lib.FRT_EINVAL, "frames_per_tick must be an integer in 1..%d, got %r"
                                     % (MAX_FRAMES_PER_TICK, frames_per_tick))
        nf = frame_count(n_samples, self.fft_size, self.hop)
        if nf % g:
            raise _lib.FrtValueError(_lib.FRT_EINVAL, "%d frames are not a whole number of %d-frame ticks"
                                     % (nf, g))
        return int(g), nf // g

    # -- many ticks --------------------------------------------------------------------------
    def process_ticks(self, x, frames_per_tick=None, want_db=True, stream=None):
        """R = frames / frames_per_tick consecutive ticks in one call: x as for ``process``, holding
        the frames of all of them (tick r is x[..., r*g*hop : (r+1)*g*hop + N - hop] for g =
        frames_per_tick, by default the widget's feed, ``default_frames_per_tick()``).  Returns a
        ``SpectrumTicks`` with every tick's row: the same bits as R ``process`` calls on those
        slices, and the same carried states afterwards.  One STFT launch, one reduction call and
        one read of each index array for all R ticks."""
        import torch
        x, dual = self._input(x)
        g, R = self.tick_geometry(x.shape[-1], frames_per_tick)
        C = self.n_channels
        nb = self.fft_size // 2 + 1
        nf = g * R
        dev = x.device
        with _lib.call_stream(dev, stream) as sp:
            rows = x.view(2 * C, x.shape[-1]) if dual else x
            power = self.proc.stft(rows, hop=self.hop, log=False, stream=stream)
            self._states(dev, dual)
            db = torch.empty((C, R, nb), dtype=torch.float32, device=dev) if want_db else None
            imax = torch.empty((R, C), dtype=torch.int32, device=dev)
            ipitch = torch.empty((R, C), dtype=torch.int32, device=dev)
            if R:
                h = self.proc.handle
                if dual:
                    # power [2C, nf, nb]: pair c's reference at row 2c, its measurement at row 2c + 1
                    p1 = power.data_ptr()
                    h.call("frt_spectrum_reduce_dual_ticks", _lib._ptr(p1), _lib._ptr(p1 + 4 * nf * nb),
                           int(2 * nf * nb), int(nb), int(C), g, int(R), int(nb), c_float(self.alpha),
                           _lib._ptr(self._disp), _lib._ptr(self._disp2), _lib._ptr(db), _lib._ptr(imax),
                           _lib._ptr(ipitch), sp)
                else:
                    h.call("frt_spectrum_reduce_ticks", _lib._ptr(power), int(nf * nb), int(nb), int(C), g,
                           int(R), int(nb), c_float(self.alpha), _lib._ptr(self._disp),
                           _lib._ptr(self._w_dev) if self.weighting else None, _lib._ptr(db),
                           _lib._ptr(imax), _lib._ptr(ipitch), sp)
                    self._decay_unfilled([g] * R)
            return SpectrumTicks(db, *self._indices_to_hz(imax, ipitch))

    # -- the widget's stream ----------------------------------------------------------------------
    def handle_new_data(self, chunk, buffer=None, want_db=True, stream=None):
        """``Spectrum_Widget.handle_new_data`` (friture/spectrum.py:125-184) over a stream pushed in
        chunks: CUDA float32 [C, n], or [C, 2, n] with row 0 the reference and row 1 the measurement;
        the first chunk's shape fixes the stream's.  Frames of ``fft_size`` samples end at
        ``old_index``, which then advances by the hop (zeros before the stream starts).  ``buffer=None``:
        the chunk is one widget tick; ``buffer=b``: it is n/b ticks of b samples each, the same bits as
        n/b calls.  Returns a ``SpectrumTicks`` with one row per tick that had frames (the widget draws
        nothing on the others), ``tick`` and ``n_frames`` saying which and how many.  Each frame's power
        column goes straight into the smoothing on chip (``frt_spectrum_frames``); the rows, indices
        and states are the same bits as ``process`` on the frames each tick cut.  Refusals happen
        before the stream or the states change."""
        import torch
        _lib.check_tensor(self.proc, chunk, "chunk")
        if chunk.dim() not in (2, 3) or (chunk.dim() == 3 and chunk.shape[1] != 2):
            raise ValueError("chunk must be [C, n] or [C, 2, n], got %s" % (tuple(chunk.shape),))
        if chunk.shape[0] != self.n_channels:
            raise ValueError("chunk must have %d channels" % self.n_channels)
        pairs = chunk.dim() == 3
        if self._pairs is not None and pairs != self._pairs:
            raise ValueError("the stream is %s; this chunk is not" % ("[C, 2, n]" if self._pairs else "[C, n]"))
        ends, ticks = self.stream_ticks(chunk.shape[-1], buffer)
        C = self.n_channels
        rows_in = 2 * C if pairs else C
        x = chunk.reshape(rows_in, chunk.shape[-1])
        dual = pairs and self.dual_channels
        nb = self.fft_size // 2 + 1
        dev = chunk.device
        with _lib.call_stream(dev, stream) as sp:
            if self._framer is None:
                self._framer = StreamFramer(rows_in, self.fft_size, self.hop, dev, capacity=2 * STREAM_HISTORY,
                                            history=STREAM_HISTORY)
                self._pairs = pairs
            fr = self._framer
            fr.push(x)
            view, F = fr.take()
            R = len(ends)
            db = torch.empty((C, R, nb), dtype=torch.float32, device=dev) if want_db else None
            imax = torch.empty((R, C), dtype=torch.int32, device=dev)
            ipitch = torch.empty((R, C), dtype=torch.int32, device=dev)
            if F:
                self._states(dev, dual)
                # the tick ends go up from pinned memory without waiting for the stream
                ends_host = torch.from_numpy(ends.astype(np.int32))
                if dev.type == "cuda":
                    ends_host = ends_host.pin_memory()
                ends_dev = ends_host.to(dev, non_blocking=True)
                h = self.proc.handle
                h.call("frt_stft_plan", int(self.fft_size))
                pitch = int(view.stride(0))
                db_strides = (int(R * nb), int(nb))
                if dual:
                    p1 = view.data_ptr()
                    h.call("frt_spectrum_frames_dual", _lib._ptr(p1), _lib._ptr(p1 + 4 * pitch), 2 * pitch, C,
                           int(F), int(self.hop), _lib._ptr(ends_dev), int(R), c_float(self.alpha),
                           _lib._ptr(self._disp), _lib._ptr(self._disp2), _lib._ptr(db), *db_strides,
                           _lib._ptr(imax), _lib._ptr(ipitch), sp)
                else:
                    # [C, 2, n]: the reference rows only
                    h.call("frt_spectrum_frames", _lib._ptr(view), 2 * pitch if pairs else pitch, C, int(F),
                           int(self.hop), _lib._ptr(ends_dev), int(R), c_float(self.alpha),
                           _lib._ptr(self._disp), _lib._ptr(self._w_dev) if self.weighting else None,
                           _lib._ptr(db), *db_strides, _lib._ptr(imax), _lib._ptr(ipitch), sp)
                    self._decay_unfilled(np.diff(ends, prepend=0))
            return SpectrumTicks(db, *self._indices_to_hz(imax, ipitch), ticks, np.diff(ends, prepend=0))

    def stream_ticks(self, n, buffer=None):
        """(ends, ticks) of a ``handle_new_data`` call of n samples per row: the frame index at which
        each tick with frames ends (counted from the call's first frame) and which buffer of the call
        it is, from the widget's framing (friture/spectrum.py:128-155); nothing changes.  Raises
        FrtValueError for a buffer that does not divide n or a tick of more than 8192 frames."""
        n = int(n)
        if buffer is not None and (isinstance(buffer, (bool, np.bool_)) or
                                   not isinstance(buffer, (int, np.integer)) or buffer < 1):
            raise _lib.FrtValueError(_lib.FRT_EINVAL, "buffer must be a positive integer, got %r" % (buffer,))
        b = n if buffer is None else int(buffer)
        if n == 0:
            return np.zeros(0, np.int64), np.zeros(0, np.int64)
        if n % b:
            raise _lib.FrtValueError(_lib.FRT_EINVAL, "%d samples are not a whole number of %d-sample buffers"
                                     % (n, b))
        offset = self._framer.offset if self._framer is not None else 0
        # old_index advances by whole hops while offset - old_index >= hop, so after buffer t the frames
        # cut so far are floor((offset_t - old_index) / hop)
        avail = offset + b * np.arange(1, n // b + 1, dtype=np.int64) - self.old_index
        cum = np.maximum(avail, 0) // self.hop
        per = np.diff(cum, prepend=0)
        if per.max() > MAX_FRAMES_PER_TICK:
            raise _lib.FrtValueError(_lib.FRT_EINVAL, "a tick of %d frames exceeds the reference's %d-tap kernel"
                                     % (per.max(), MAX_FRAMES_PER_TICK))
        ticks = np.flatnonzero(per)
        return cum[ticks], ticks

    def _states(self, dev, dual):
        """The carried smoothed states, zeros after a restart (the widget's update_display_buffers), and
        outside dual mode the weighting on the device: whatever of them the coming tick reads and does
        not have yet."""
        import torch
        nb = self.fft_size // 2 + 1
        if self._disp is None:
            self._disp = torch.zeros((self.n_channels, nb), dtype=torch.float32, device=dev)
        if dual and self._disp2 is None:
            self._disp2 = torch.zeros((self.n_channels, nb), dtype=torch.float32, device=dev)
        if not dual and self._w_dev is None:
            self._w_dev = torch.from_numpy(np.ascontiguousarray(self.w, dtype=np.float32)).to(dev)

    def _decay_unfilled(self, frames):
        """Single-mode ticks of the given frame counts on a kept second state: the widget smooths an
        all-zero second column on every tick it does not fill (spectrum.py:142,158-159), so
        dispbuffers2 *= (1-alpha)^frames, rounded once per tick; a tick without frames smooths nothing."""
        if self._disp2 is not None:
            for n in frames:
                if n:
                    self._disp2.mul_((1. - self.alpha) ** int(n))

    def _indices_to_hz(self, imax, ipitch):
        # on the call's stream, which is current: the reads wait for the kernel that writes them
        fmax = self.freq[imax.cpu().numpy()]
        fpitch = np.maximum(self.freq[ipitch.cpu().numpy()], 1e-20)     # spectrum.py:181
        return fmax, fpitch
