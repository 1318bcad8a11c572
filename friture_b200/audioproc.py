"""Drop-in for ``friture.audioproc.audioproc`` (friture/audioproc.py:27-96) on the GPU.

Same call surface as the reference class -- ``analyzelive``, ``set_fftsize``, ``set_maxfreq``,
``get_freq_scale``, ``get_freq_weighting`` and the attributes ``window, freq, A, B, C, fft_size,
size_sq, maxfreq`` -- plus batched device entry points (``stft`` / ``stft_host``) over an
independent-channel axis, which the reference does not have (it processes one frame of one
channel per call, friture/spectrogram.py:149-159).

The arithmetic runs in float32 in the fused CUDA kernel of ``csrc/stft.cu``; the single-frame
shim returns float64 NumPy like the reference.
"""
from __future__ import annotations

import logging

import numpy as np

from . import _lib
from ._lib import STFT_LOGPOWER, STFT_POWER
from .weighting import abc_weighting

SAMPLING_RATE = 48000      # friture/audiobackend.py:31
FRAMES_PER_BUFFER = 512    # friture/audiobackend.py:32


def frame_count(n_samples: int, n_fft: int, hop: int) -> int:
    """Whole frames in a stream of ``n_samples`` (first frame = samples [0, n_fft))."""
    if n_samples < n_fft:
        return 0
    return (n_samples - n_fft) // hop + 1


class audioproc():
    """GPU-backed ``audioproc``.  ``handle`` selects the GPU (default: current torch device)."""

    def __init__(self, handle=None):
        self.logger = logging.getLogger(__name__)
        self._handle = handle
        # same initial attribute values as friture/audioproc.py:29-40
        self.freq = np.linspace(0, SAMPLING_RATE / 2, 10)
        self.A = 0. * self.freq
        self.B = 0. * self.freq
        self.C = 0. * self.freq
        self.maxfreq = 1.
        self.window = np.arange(0, 1)
        self.size_sq = 1.
        self.fft_size = 10

    # ------------------------------------------------------------------ plumbing
    handle = _lib.shared_handle

    def _ensure_plan(self):
        self.handle.call("frt_stft_plan", int(self.fft_size))

    # ------------------------------------------------------------------ reference surface
    def analyzelive(self, samples):
        """|rfft(samples*window)|^2 / N^2 for one frame (friture/audioproc.py:42-50)."""
        samples = np.asarray(samples)
        if samples.ndim != 1 or samples.shape[0] != self.fft_size:
            # the reference fails with a NumPy broadcast error on a length mismatch
            raise ValueError("operands could not be broadcast together with shapes (%s) (%d,)"
                             % (",".join(str(s) for s in samples.shape), self.fft_size))
        out = self.stft_host(samples[None, :], hop=self.fft_size, log=False)
        return out[0, 0].astype(np.float64)

    def norm_square(self, fft):
        return (fft * fft.conjugate()).real / self.size_sq

    def set_fftsize(self, fft_size):
        if fft_size != self.fft_size:
            self.fft_size = fft_size
            self._refresh()

    def set_maxfreq(self, maxfreq):
        if maxfreq != self.maxfreq:
            self.maxfreq = maxfreq
            self._refresh()

    def get_freq_scale(self):
        return self.freq

    def get_freq_weighting(self):
        return self.A, self.B, self.C

    def _refresh(self):
        # the three updates the reference runs on every size / range change (audioproc.py:52-66)
        self.update_freq_cache()
        self.update_window()
        self.update_size()

    def update_size(self):
        self.size_sq = float(self.fft_size) ** 2

    def update_window(self):
        # symmetric Hann 0.5*(1 - cos(2*pi*n/(N-1))), friture/audioproc.py:76-81; the device plan
        # builds the same window in float64 and rounds it to float32, `window` exposes float64
        n = np.arange(self.fft_size)
        self.window = 0.5 * (1. - np.cos(2 * np.pi * n / (self.fft_size - 1)))
        self.logger.info("audioproc: updating window")

    def update_freq_cache(self):
        # bin frequencies and A/B/C weighting tables, friture/audioproc.py:83-96
        nbins = self.fft_size // 2 + 1
        if len(self.freq) != nbins:
            self.logger.info("audioproc: updating self.freq cache")
            self.freq = np.linspace(0, SAMPLING_RATE // 2, nbins)
            self.A, self.B, self.C = abc_weighting(self.freq, eps=1e-50)

    # ------------------------------------------------------------------ batched extensions
    def stft(self, x, hop, log=True, out=None, stream=None):
        """Batched STFT on device tensors.

        x: CUDA float32 tensor [C, T] (last dim contiguous).  Frame f of channel c is
        ``x[c, f*hop : f*hop + fft_size]`` -- one ``analyzelive`` call of the reference each
        (friture/spectrogram.py:149-159 with ``hop = int(fft_size*(1-overlap))``).
        Returns a CUDA float32 tensor [C, frames, fft_size//2+1]: power, or
        ``10*log10(power+1e-30)`` (friture/spectrogram.py:119-125) when ``log``.
        """
        import torch
        x, x_stride = _lib.device_rows(self, x, "x")
        C, T = x.shape
        nf = frame_count(T, self.fft_size, hop)
        nb = self.fft_size // 2 + 1
        if out is not None and (not isinstance(out, torch.Tensor) or out.device != x.device
                                or tuple(out.shape) != (C, nf, nb) or out.dtype != torch.float32
                                or not out.is_contiguous()):
            raise ValueError("out must be a contiguous float32 tensor of shape %s on %s" % ((C, nf, nb), x.device))
        with _lib.call_stream(x.device, stream) as sp:
            if out is None:
                out = torch.empty((C, nf, nb), dtype=torch.float32, device=x.device)
            if C == 0 or nf == 0:
                return out
            self._ensure_plan()
            self.handle.call("frt_stft_process", _lib._ptr(x), x_stride, int(C), int(nf),
                             int(hop), _lib._ptr(out), int(nf * nb), int(nb),
                             STFT_LOGPOWER if log else STFT_POWER, sp)
        return out

    def stft_host(self, x, hop, log=True, out=None):
        """Same with host buffers: float32 NumPy arrays or CPU torch tensors (pinned memory gives
        full PCIe speed).  H2D copy, kernel and D2H copy are pipelined inside the C call."""
        is_torch = hasattr(x, "data_ptr")
        if not is_torch:
            x = np.ascontiguousarray(x, dtype=np.float32)
        x, x_stride = _lib.host_rows(x)
        C, T = x.shape
        nf = frame_count(T, self.fft_size, hop)
        nb = self.fft_size // 2 + 1
        if out is not None:
            _lib.check_host_out(out, (C, nf, nb), "out")
        else:
            if is_torch:
                import torch
                out = torch.empty((C, nf, nb), dtype=torch.float32, pin_memory=x.is_pinned())
            else:
                out = np.empty((C, nf, nb), dtype=np.float32)
        if C == 0 or nf == 0:
            return out
        self._ensure_plan()
        self.handle.call("frt_stft_process_host", _lib._ptr(x), x_stride, int(C), int(T), int(hop),
                         _lib._ptr(out), STFT_LOGPOWER if log else STFT_POWER)
        return out


# CamelCase alias used by BASELINE.json's prose (the reference class is lower-case)
AudioProc = audioproc
