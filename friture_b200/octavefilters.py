"""Drop-in for ``friture.octavefilters.Octave_Filters`` (friture/octavefilters.py:37-158) on the GPU.

Same call surface -- ``Octave_Filters(bandsperoctave)``, ``filter(x) -> (y, dec)``, ``get_decs()``,
``setbandsperoctave(bpo)`` and the attributes ``fi, flow, fhigh, f_nominal, A, B, C, nbands,
bandsperoctave, bdec, adec, boct, aoct`` -- plus batched device entry points over an
independent-channel axis (``filter_batch`` / ``energies_batch``) that fuse the octave widget's
``y**2 -> exp_smoothed_value -> 10*log10`` (friture/octavespectrum.py:101-121) behind the bank.

Numerics: the reference has two implementations of the same IIR designs, the live FFT
overlap-add with 512-tap FIR approximations (friture/filter.py:136-247) and the IIR bank
``octave_filter_bank_decimation`` (friture/filter.py:86-118) that its own tests check against
(friture/test/test_octave_filters.py:21-35).  The GPU kernel runs the IIR designs themselves (as
float32 second-order sections), so it matches the IIR bank to ~1e-6 and the live FFT path to the
~5e-4 by which the reference's two paths differ from each other.
"""
from __future__ import annotations

from ctypes import c_int64, byref

import numpy as np

from . import _lib, filter_data
from ._lib import Handle
from .audioproc import SAMPLING_RATE
from .filter_data import NOCTAVE
from .weighting import abc_weighting

FIR_LENGTH = 512   # friture/octavefilters.py:35 (kept for attribute parity; unused by the IIR kernel)
MAX_BLOCK = 8192   # exp_smoothed_value drops history beyond its 8192/dec-tap kernel
                   # (friture/signal/exp_smoothing.py:43-47, octavespectrum.py:152)


def octave_frequencies(total_bands_count, bands_per_octave):
    """Centre and edge frequencies (friture/filter.py:39-54)."""
    f0 = 1000.
    b = 1. / bands_per_octave
    imax = total_bands_count // 2
    if total_bands_count % 2 == 0:
        i = np.arange(-imax, imax)
    else:
        i = np.arange(-imax, imax + 1)
    fi = f0 * 2 ** (i * b)
    f_low = fi * np.sqrt(2 ** (-b))
    f_high = fi * np.sqrt(2 ** b)
    return fi, f_low, f_high


def smoothing_alphas(response_time, n_octaves=NOCTAVE, fs=SAMPLING_RATE):
    """alpha per stage j (rate fs/2^j): the newest n = T*fs/dec samples carry 65 % of the weight
    (friture/octavespectrum.py:140-154)."""
    w = 0.65
    return np.array([1. - (1. - w) ** (1. / (response_time * fs / 2 ** j + 1))
                     for j in range(n_octaves)], dtype=np.float64)


def bank_block_ok(block, n_octaves):
    """Whether the IIR filterbank takes blocks of ``block`` samples with ``n_octaves`` octaves
    (csrc/bank.cu, bank_route): a multiple of 256 samples, and the longest of the 1024, 512 and
    256-sample tiles that divides it still even at the last of the halving stages."""
    if block <= 0 or block % 256:
        return False
    tile = next(t for t in (1024, 512, 256) if block % t == 0)
    return (tile >> (n_octaves - 1)) >= 1


def check_bank_block(block, n_octaves):
    """ValueError unless the IIR filterbank takes blocks of ``block`` samples (bank_block_ok)."""
    if not bank_block_ok(block, n_octaves):
        raise ValueError("the filterbank takes no %d-sample blocks at %d octaves: a block must be a multiple "
                         "of 256 samples whose longest tile of 1024, 512 or 256 that divides it holds at least "
                         "%d samples (every decimation stage needs an even length, friture/signal/decimate.py:41)"
                         % (block, n_octaves, 1 << (n_octaves - 1)))


def ragged_layout(n_samples, bpo, n_octaves=NOCTAVE):
    """(offsets, lengths) of the bands in the kernel's concatenated y layout, band k = 0..nbands-1
    (k = (n_octaves-1-j)*bpo + i, friture/filter.py:104-109)."""
    lengths = [n_samples >> (n_octaves - 1 - k // bpo) for k in range(n_octaves * bpo)]
    offsets = np.concatenate([[0], np.cumsum(lengths)[:-1]]).astype(np.int64)
    return offsets, lengths


class Octave_Filters():
    """GPU-backed ``Octave_Filters``.  Every instance owns its filter state, like the reference
    (friture/octavefilters.py:50-56); ``device`` selects the GPU."""

    FIR_LENGTH = FIR_LENGTH

    def __init__(self, bandsperoctave, device=None, n_octaves=NOCTAVE, response_time=1.0, handle=None,
                 mode="iir"):
        self.bdec, self.adec, self._sos_dec = filter_data.decimator()
        self.bdec = np.array(self.bdec)
        self.adec = np.array(self.adec)
        self._device = device
        self._handle = handle      # share a handle (one GPU context) with other objects, or own one
        self._n_octaves = n_octaves
        self._response_time = response_time
        self._plan_key = None
        self._weighting = None
        # "iir": the reference's IIR designs themselves (the bank its own tests check against,
        # friture/filter.py:86-118) -- fused energies, the throughput path.  "fft": the numerics of
        # the reference's live filter(), 512-tap FIR approximations run by FFT overlap-add
        # (friture/filter.py:136-247), computed as exact FIR convolutions; band outputs only.
        if mode not in ("iir", "fft"):
            raise ValueError("mode must be 'iir' or 'fft'")
        self._mode = mode
        self._fir_key = None
        self.setbandsperoctave(bandsperoctave)

    # ------------------------------------------------------------------ reference surface
    def filter(self, floatdata):
        """One chunk of one channel -> (y, dec): ``y[k]`` float64 array of length len(x)/dec[k]
        (friture/octavefilters.py:49-58)."""
        x = np.ascontiguousarray(floatdata, dtype=np.float32)
        if x.ndim != 1:
            raise ValueError("filter expects a 1-D array")
        if x.shape[0] == 0:
            raise Exception("Filter input is too small")   # friture/signal/decimate.py:33-34
        import torch
        dev = torch.device("cuda", self.handle.device)
        if self._mode == "fft" and x.shape[0] > 4096:
            raise ValueError("fft mode: at most 4096 samples per call (the reference's live path is "
                             "valid up to 1024, friture/filter_design.py:400-401)")
        y, _ = self.filter_batch(torch.from_numpy(x).to(dev)[None, :], block=x.shape[0],
                                 energies=False, want_y=True)
        ylist = [v[0].cpu().numpy().astype(np.float64) for v in y]
        return ylist, self.get_decs_by_band()

    def get_decs(self):
        # friture/octavefilters.py:60-63
        return [2 ** j for j in range(0, self._n_octaves)[::-1] for i in range(0, self.bandsperoctave)]

    def get_decs_by_band(self):
        """dec list as returned by filter(): dec[k] = 2^j for band k (friture/filter.py:108)."""
        return self.get_decs()

    def setbandsperoctave(self, bandsperoctave):
        # friture/octavefilters.py:65-121
        boct, aoct, sos = filter_data.bands(bandsperoctave)
        self.bandsperoctave = bandsperoctave
        self.nbands = self._n_octaves * self.bandsperoctave
        self.fi, self.flow, self.fhigh = octave_frequencies(self.nbands, self.bandsperoctave)
        self.boct = [np.array(f) for f in boct]
        self.aoct = [np.array(f) for f in aoct]
        self._sos_band = np.ascontiguousarray(sos, dtype=np.float64)
        self.A, self.B, self.C = abc_weighting(self.fi)     # friture/octavefilters.py:76-82
        self._weighting = None
        self._plan_key = None   # new filters -> state restarts from zero (octavefilters.py:151-158)
        self._fir_key = None
        self.f_nominal = self._nominal_labels()

    def _nominal_labels(self):
        # friture/octavefilters.py:84-121
        bpo = self.bandsperoctave
        if bpo == 1:
            return ["%.1fk" % (f / 1000) if f >= 10000
                    else "%.2fk" % (f / 1000) if f >= 1000
                    else "%d" % (f)
                    for f in self.fi]
        basis = filter_data.renard({3: 10, 6: 20, 12: 40, 24: 80}[bpo])
        hits = np.where(self.fi == 1000.)[0]
        if len(hits) == 0:     # even band counts (n_octaves = 10): no exact 1 kHz band
            return ["%g" % f for f in self.fi]
        i = hits[0]
        labels = []
        k = 0
        while len(labels) < len(self.fi) - i:
            labels += ["{0:.{width}f}k".format(10 ** k * f, width=2 - k) for f in basis]
            k += 1
        labels = labels[:len(self.fi) - i]
        k = 0
        while len(labels) < len(self.fi):
            labels = ["%d" % (10 ** (2 - k) * f) for f in basis] + labels
            k += 1
        return labels[-len(self.fi):]

    # ------------------------------------------------------------------ plumbing
    handle = _lib.lazy_handle(lambda self: Handle(_lib.device_index(self._device)))

    def set_response_time(self, response_time):
        """Smoothing time constant of the fused exponential RMS (octavespectrum.py:140-156);
        changing it restarts the state, as the widget does."""
        if response_time != self._response_time:
            self._response_time = response_time
            self._plan_key = None

    def reset(self):
        if self._plan_key is not None:
            self.handle.call("frt_bank_reset")
        if self._fir_key is not None:
            self.handle.call("frt_firbank_reset")

    def _ensure_fir_plan(self, n_channels):
        key = (n_channels, self.bandsperoctave, self._n_octaves)
        if key == self._fir_key:
            return
        boct_fir, bdec_fir = filter_data.fir_taps(self.bandsperoctave)
        boct_fir = np.ascontiguousarray(boct_fir, dtype=np.float64)
        bdec_fir = np.ascontiguousarray(bdec_fir, dtype=np.float64)
        self.handle.call("frt_firbank_plan", int(n_channels), int(self.bandsperoctave), int(self._n_octaves),
                         int(boct_fir.shape[1]), _lib._ptr(boct_fir), _lib._ptr(bdec_fir))
        self._fir_key = key

    def _filter_batch_fir(self, x, x_stride, block, sp):
        """Live-path numerics: band outputs of x [C, n_blocks*block] (row stride ``x_stride``),
        block by block, on the stream ``sp``, which is current."""
        import torch
        C, T = x.shape
        if block > 4096 or block % (1 << (self._n_octaves - 1)):
            raise ValueError("fft mode: block must be a multiple of %d and at most 4096"
                             % (1 << (self._n_octaves - 1)))
        self._ensure_fir_plan(C)
        offsets, lengths = ragged_layout(block, self.bandsperoctave, self._n_octaves)
        ystride = int(offsets[-1] + lengths[-1])
        parts = []
        for b in range(T // block):
            ybuf = torch.empty((C, ystride), dtype=torch.float32, device=x.device)
            xb = x[:, b * block:(b + 1) * block]
            self.handle.call("frt_firbank_process", _lib._ptr(xb), x_stride,
                             int(block), _lib._ptr(ybuf), ystride, sp)
            parts.append(ybuf)
        return [torch.cat([p[:, int(o):int(o) + int(n)] for p in parts], dim=1)
                for o, n in zip(offsets, lengths)]

    def set_weighting(self, weighting):
        """dB offsets added to the dB energies (``db=True``), as the octave widget does
        (friture/octavespectrum.py:108-121): None / 0 = none, 'A' / 'B' / 'C' or 1 / 2 / 3 = the
        reference's tables (friture/octavefilters.py:76-82), or an array of nbands values."""
        if weighting is None or (isinstance(weighting, (int, np.integer)) and weighting == 0):
            w = None
        elif isinstance(weighting, str) or isinstance(weighting, (int, np.integer)):
            key = {"A": "A", "B": "B", "C": "C", 1: "A", 2: "B", 3: "C"}[weighting]
            w = np.asarray(getattr(self, key), dtype=np.float32)
        else:
            w = np.ascontiguousarray(weighting, dtype=np.float32)
            if w.shape != (self.nbands,):
                raise ValueError("weighting must have nbands = %d values" % self.nbands)
        self._weighting = w
        if self._plan_key is not None:
            self.handle.call("frt_bank_set_weighting", _lib._ptr(self._weighting))

    def _ensure_plan(self, n_channels):
        key = (n_channels, self.bandsperoctave, self._n_octaves, self._response_time)
        if key == self._plan_key:
            return
        alphas = smoothing_alphas(self._response_time, self._n_octaves)
        sos_dec = np.ascontiguousarray(self._sos_dec, dtype=np.float64)
        self.handle.call("frt_bank_plan", int(n_channels), int(self.bandsperoctave),
                         int(self._n_octaves), _lib._ptr(self._sos_band), _lib._ptr(sos_dec),
                         _lib._ptr(alphas))
        self._plan_key = key
        self.alphas = alphas
        if self._weighting is not None:
            self.handle.call("frt_bank_set_weighting", _lib._ptr(self._weighting))

    # ------------------------------------------------------------------ batched extensions
    def filter_batch(self, x, block, energies=True, want_y=False, db=False, stream=None):
        """x: CUDA float32 [C, n_blocks*block].  Returns (y, e):
        y  list of nbands CUDA tensors [C, T >> j] (views into one buffer) when ``want_y``;
        e  CUDA tensor [C, n_blocks, nbands]: the smoothed band energies after each block -- what
           OctaveSpectrum_Widget.handle_new_data computes per chunk (octavespectrum.py:101-107) --
           in dB (10*log10(e+1e-30), octavespectrum.py:119-120) when ``db``.
        Filter and smoothing state carry over from call to call."""
        import torch
        x, x_stride = _lib.device_rows(self, x, "x")
        C, T = x.shape
        if T == 0 or C == 0:
            raise Exception("Filter input is too small")
        if block <= 0 or T % block != 0:
            raise ValueError("T must be a whole number of blocks")
        check_bank_block(block, self._n_octaves)
        if energies and block > MAX_BLOCK:
            raise ValueError("block > %d: the reference's smoothing kernel is shorter than the "
                             "block (exp_smoothing.py:43-47)" % MAX_BLOCK)
        n_blocks = T // block
        if self._mode == "fft" and energies:
            raise ValueError("fft mode gives the band outputs only (energies=False, want_y=True)")
        with _lib.call_stream(x.device, stream) as sp:
            if self._mode == "fft":
                return self._filter_batch_fir(x, x_stride, block, sp), None
            self._ensure_plan(C)
            e = None
            if energies:
                e = torch.empty((C, n_blocks, self.nbands), dtype=torch.float32, device=x.device)
            ybuf = None
            ystride = 0
            if want_y:
                offsets, lengths = ragged_layout(T, self.bandsperoctave, self._n_octaves)
                ystride = int(offsets[-1] + lengths[-1])
                ybuf = torch.empty((C, ystride), dtype=torch.float32, device=x.device)
            self.handle.call("frt_bank_process", _lib._ptr(x), x_stride, int(block),
                             int(n_blocks), _lib._ptr(e), _lib._ptr(ybuf), ystride, 1 if db else 0, sp)
            y = None
            if want_y:
                y = [ybuf[:, int(o):int(o) + int(n)] for o, n in zip(offsets, lengths)]
        return y, e

    def energies_batch(self, x, block, db=False):
        """Smoothed band energies only (the fused fast path): [C, n_blocks, nbands]."""
        return self.filter_batch(x, block, energies=True, want_y=False, db=db)[1]

    # ------------------------------------------------------------------ state checkpoint
    def get_state(self):
        """(z, ema) NumPy copies of the filter / smoothing state (for resume tests)."""
        if self._plan_key is None:
            raise _lib.FrtError(_lib.FRT_ESTATE, "no filterbank state yet")
        nz, ne = c_int64(), c_int64()
        self.handle.call("frt_bank_state_size", byref(nz), byref(ne))
        z = np.empty(nz.value, dtype=np.float32)
        e = np.empty(ne.value, dtype=np.float32)
        self.handle.call("frt_bank_get_state", _lib._ptr(z), _lib._ptr(e))
        return z, e

    def set_state(self, z, e):
        z = np.ascontiguousarray(z, dtype=np.float32)
        e = np.ascontiguousarray(e, dtype=np.float32)
        nz, ne = c_int64(), c_int64()
        self.handle.call("frt_bank_state_size", byref(nz), byref(ne))
        if z.size != nz.value or e.size != ne.value:
            raise ValueError("state size mismatch")
        self.handle.call("frt_bank_set_state", _lib._ptr(z), _lib._ptr(e))


# CamelCase alias used by BASELINE.json's prose (the reference class is Octave_Filters)
OctaveFilters = Octave_Filters

