"""Drop-in for ``friture.signal.correlation.generalized_cross_correlation``
(friture/signal/correlation.py:24-43) and a batched delay estimator with the smoothing and peak
pick of ``Delay_Estimator_Widget.handle_new_data`` (friture/delay_estimator.py:129-152)."""
from __future__ import annotations

import numpy as np

from . import _lib


def generalized_cross_correlation(d0, d1, handle=None):
    """GCC-PHAT of one pair: float64 NumPy in, float64 ``Xcorr`` out -- ``len(d0)`` values, or
    ``len(d0) - 1`` for an odd length, like the reference's ``irfft``.  Unlike the reference the
    inputs are left untouched (it subtracts the means in place)."""
    import torch
    d0 = np.ascontiguousarray(d0, dtype=np.float32)
    d1 = np.ascontiguousarray(d1, dtype=np.float32)
    if d0.ndim != 1 or d0.shape != d1.shape:
        raise ValueError("d0 and d1 must be 1-D arrays of the same length")
    est = GccPhat(d0.shape[0], handle=handle)
    dev = torch.device("cuda", est.handle.device)
    _, _, x = est.estimate(torch.from_numpy(d0).to(dev)[None, :], torch.from_numpy(d1).to(dev)[None, :],
                           smooth=False, want_xcorr=True)
    return x[0].cpu().numpy().astype(np.float64)


class GccPhat:
    """Batched GCC-PHAT over independent channel pairs, for every frame length the delay widget
    offers (4 .. 24 000 000 samples, odd or even).  ``estimate`` returns
    (index of max |Xs|, Xs at that index, Xcorr or None); with ``smooth`` the handle keeps
    ``Xs = 0.3*X + 0.7*Xs_prev`` per pair across calls like the widget's ``old_Xcorr``.  For an odd
    length Xcorr and the smoothed buffer hold ``length - 1`` samples, like the reference's
    ``irfft``."""

    def __init__(self, length, handle=None, fs=12000.0):
        self.length = int(length)
        self.out_length = self.length - (self.length & 1)   # samples of Xcorr and of the smoothed buffer
        self.fs = fs                      # 48 kHz / 2**Ndec, delay_estimator.py:53-54
        self._handle = handle
        self._smoothed = None
        self._have_prev = False

    handle = _lib.shared_handle

    def reset(self):
        self._smoothed = None
        self._have_prev = False

    def estimate(self, d0, d1, smooth=True, want_xcorr=False, stream=None):
        _lib.check_tensor(self, d0, "d0")
        with _lib.call_stream(d0.device, stream) as sp:
            d0, _ = _lib.device_rows(self, d0.contiguous(), "d0")
            d1, _ = _lib.device_rows(self, d1.contiguous(), "d1")
            if d0.shape != d1.shape:
                raise ValueError("d0, d1 must be CUDA float32 tensors of the same shape [P, L]")
            P, L = d0.shape
            if L != self.length:
                raise ValueError("frame length %d != planned %d" % (L, self.length))
            return self._call("frt_gcc_phat", P, d0.device, smooth, want_xcorr, sp,
                              _lib._ptr(d0), _lib._ptr(d1), int(L), int(P))

    def _call(self, symbol, P, device, smooth, want_xcorr, sp, *inputs, after_plan=None):
        """Plans the length, runs ``after_plan()`` if given, makes the outputs of P pairs and calls
        ``symbol(*inputs, xcorr, smoothed, have_prev, idx, val, stream)``; returns (idx, val, xcorr or
        None)."""
        import torch
        self.handle.call("frt_gcc_plan", self.length)
        if after_plan is not None:
            after_plan()
        Lo = self.out_length
        idx = torch.empty(P, dtype=torch.int32, device=device)
        val = torch.empty(P, dtype=torch.float32, device=device)
        xc = torch.empty((P, Lo), dtype=torch.float32, device=device) if want_xcorr else None
        sm = None
        have_prev = 0
        if smooth:
            if self._smoothed is None or tuple(self._smoothed.shape) != (P, Lo):
                self._smoothed = torch.zeros((P, Lo), dtype=torch.float32, device=device)
                self._have_prev = False
            sm = self._smoothed
            # 2 = per pair: a pair whose frames have all been silent so far has no previous smoothed
            # frame (the kernel marks it), like old_Xcorr = None in the widget
            have_prev = 2 if self._have_prev else 0
        self.handle.call(symbol, *inputs, _lib._ptr(xc), _lib._ptr(sm), have_prev, _lib._ptr(idx), _lib._ptr(val),
                         sp)
        if smooth:
            self._have_prev = True
        return idx, val, xc

    def estimate_frames(self, d0, d1, hop, n_frames, stream=None):
        """``estimate`` over ``n_frames`` frames of every pair in one library call, smoothing on: frame f
        of pair p is ``d0[p, f*hop : f*hop + length]`` (and the same of ``d1``).  d0, d1: CUDA float32
        [P, T], contiguous along time, T >= (n_frames - 1) * hop + length; strided views such as a
        framer's buffer rows are passed as they are, overlapping frames are not copied.  Returns
        (idx [F, P] int32, val [F, P] float32, std [F, P] float64), std being the population standard
        deviation of each frame's smoothed row.  idx, val and the smoothing state are the same bits as
        ``estimate`` called frame by frame."""
        _lib.check_tensor(self, d0, "d0")
        with _lib.call_stream(d0.device, stream) as sp:
            d0, s0 = _lib.device_rows(self, d0, "d0")
            d1, s1 = _lib.device_rows(self, d1, "d1")
            if d0.shape != d1.shape:
                raise ValueError("d0, d1 must be CUDA float32 tensors of the same shape [P, T]")
            if s0 != s1:   # one row stride for both inputs
                d0, s0 = _lib.device_rows(self, d0.contiguous(), "d0")
                d1, s1 = _lib.device_rows(self, d1.contiguous(), "d1")
            P = d0.shape[0]
            return self._call_frames("frt_gcc_phat_frames", P, d0, hop, n_frames, sp,
                                     _lib._ptr(d0), _lib._ptr(d1), s0, int(hop), int(n_frames), int(P))

    def _frame_geometry(self, T, hop, n_frames):
        hop, n_frames = int(hop), int(n_frames)
        if n_frames < 0:
            raise ValueError("n_frames must be >= 0")
        if n_frames > 1 and hop < 1:
            raise ValueError("hop must be >= 1")
        if n_frames > 0 and T < (n_frames - 1) * hop + self.length:
            raise ValueError("%d frames of %d samples at hop %d need %d samples per row, got %d"
                             % (n_frames, self.length, hop, (n_frames - 1) * hop + self.length, T))

    def _call_frames(self, symbol, P, x, hop, n_frames, sp, *inputs, after_plan=None):
        """The frames twin of ``_call``: ``symbol(*inputs, smoothed, have_prev, idx, val, std, stream)``
        with the smoothing state of P pairs; returns (idx, val, std), each [n_frames, P]."""
        import torch
        self._frame_geometry(x.shape[1], hop, n_frames)
        self.handle.call("frt_gcc_plan", self.length)
        if after_plan is not None:
            after_plan()
        F, device = int(n_frames), x.device
        idx = torch.empty((F, P), dtype=torch.int32, device=device)
        val = torch.empty((F, P), dtype=torch.float32, device=device)
        std = torch.empty((F, P), dtype=torch.float64, device=device)
        if F == 0 or P == 0:
            return idx, val, std
        if self._smoothed is None or tuple(self._smoothed.shape) != (P, self.out_length):
            self._smoothed = torch.zeros((P, self.out_length), dtype=torch.float32, device=device)
            self._have_prev = False
        self.handle.call(symbol, *inputs, _lib._ptr(self._smoothed), 2 if self._have_prev else 0, _lib._ptr(idx),
                         _lib._ptr(val), _lib._ptr(std), sp)
        self._have_prev = True
        return idx, val, std

    def delay_ms(self, idx):
        """Index -> delay in ms, wrapped to +-L/2 (delay_estimator.py:147-152)."""
        d = 1e3 * idx.to("cpu").double().numpy() / self.fs
        span = 1e3 * self.length / self.fs
        return np.where(d > span / 2.0, d - span, d)


class PairGccPhat(GccPhat):
    """GCC-PHAT between channels of one multichannel frame: ``estimate(x)`` takes x [C, L] and
    correlates, for every entry (i, j) of ``pairs``, channel i (the widget's channel 0) with
    channel j.  Each channel is transformed once however many pairs it is in.  Outputs, smoothing
    state, ``reset`` and ``delay_ms`` are those of ``GccPhat``, indexed by pair.  With the pairs
    (0, 1), (2, 3), ... the results are the same bits as ``GccPhat.estimate(x[0::2], x[1::2])``."""

    def __init__(self, length, n_channels, pairs, handle=None, fs=12000.0):
        super().__init__(length, handle=handle, fs=fs)
        self.n_channels = int(n_channels)
        if self.n_channels < 1:
            raise ValueError("n_channels must be >= 1")
        p = np.asarray(pairs)
        if p.size == 0:
            p = np.zeros((0, 2), dtype=np.int32)
        if p.ndim != 2 or p.shape[1] != 2 or not np.issubdtype(p.dtype, np.integer):
            raise ValueError("pairs must be integer (i, j) pairs, shape [P, 2]")
        if p.size and (p.min() < 0 or p.max() >= self.n_channels):
            raise ValueError("pair channels must lie in 0 .. %d" % (self.n_channels - 1))
        self.pairs = np.ascontiguousarray(p, dtype=np.int32)
        self.n_pairs = self.pairs.shape[0]
        self._table = object()   # identifies this object's table on the handle

    def _sync_table(self):
        """Give the handle this object's pair table unless it already holds it: another object on
        the same handle may have set its own since."""
        h = self.handle
        if getattr(h, "_gcc_pairs_table", None) is not self._table:
            h.call("frt_gcc_set_pairs", self.n_channels, _lib._ptr(self.pairs), self.n_pairs)
            h._gcc_pairs_table = self._table

    def estimate(self, x, smooth=True, want_xcorr=False, stream=None):
        """x: CUDA float32 [C, L], any row stride.  Returns (idx [P], val [P], xcorr [P, L'] or None)."""
        _lib.check_tensor(self, x, "x")
        with _lib.call_stream(x.device, stream) as sp:
            if x.dim() == 2 and x.shape[1] > 0 and x.stride(1) != 1:
                x = x.contiguous()
            x, x_stride = _lib.device_rows(self, x, "x")
            C, L = x.shape
            if C != self.n_channels:
                raise ValueError("x has %d channels, the pair table %d" % (C, self.n_channels))
            if L != self.length:
                raise ValueError("frame length %d != planned %d" % (L, self.length))
            return self._call("frt_gcc_phat_pairs", self.n_pairs, x.device, smooth, want_xcorr, sp,
                              _lib._ptr(x), x_stride, after_plan=self._sync_table)

    def estimate_frames(self, x, hop, n_frames, stream=None):
        """``estimate`` over ``n_frames`` frames in one library call, smoothing on: frame f of channel c
        is ``x[c, f*hop : f*hop + length]``.  x: CUDA float32 [C, T], contiguous along time, any row
        stride (a framer's buffer rows as they are).  Returns (idx, val, std), each [F, P], as
        ``GccPhat.estimate_frames``; the same bits as ``estimate`` called frame by frame."""
        _lib.check_tensor(self, x, "x")
        with _lib.call_stream(x.device, stream) as sp:
            x, x_stride = _lib.device_rows(self, x, "x")
            if x.shape[0] != self.n_channels:
                raise ValueError("x has %d channels, the pair table %d" % (x.shape[0], self.n_channels))
            return self._call_frames("frt_gcc_phat_pairs_frames", self.n_pairs, x, hop, n_frames, sp,
                                     _lib._ptr(x), x_stride, int(hop), int(n_frames),
                                     after_plan=self._sync_table)
