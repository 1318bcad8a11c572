"""Batched per-hop analysis of many independent channels: the spectrogram column and the
fractional-octave band levels that the reference's widgets compute from the same chunk of new
samples (``Spectrogram_Widget.handle_new_data``, friture/spectrogram.py:131-169 ->
``audioproc.analyzelive`` + ``log_spectrogram``; ``OctaveSpectrum_Widget.handle_new_data``,
friture/octavespectrum.py:91-121 -> ``Octave_Filters.filter``, ``y**2``, ``exp_smoothed_value``,
``10*log10`` + weighting).  This is BASELINE.json configs[4]'s unit of work: per channel and hop one
log-power column and one band vector.

``ChannelAnalyzer`` owns one handle with both plans; ``process`` works on device tensors,
``process_host`` on pinned host buffers
(H2D, kernels and D2H pipelined inside the C call), ``process_sharded`` adds the north-star's final
all-gather of the spectrogram columns over the ranks of a torch.distributed group, issued per
frame chunk on a side stream so that the link time hides behind the filterbank.
"""
from __future__ import annotations

import numpy as np

from . import _lib
from ._lib import Handle
from .audioproc import audioproc, frame_count
from .octavefilters import Octave_Filters, bank_block_ok, check_bank_block  # noqa: F401 (bank_block_ok: kept importable from here)


class ChannelAnalyzer:
    def __init__(self, n_channels, fft_size=2048, hop=1024, bandsperoctave=3, n_octaves=10,
                 response_time=1.0, weighting=None, device=None):
        import torch
        self.device = torch.device("cuda", _lib.device_index(device))
        self.handle = Handle(self.device.index)
        self.n_channels = int(n_channels)
        self.fft_size, self.hop = int(fft_size), int(hop)
        check_bank_block(self.hop, n_octaves)   # the hop is the filterbank's block
        self.nbins = self.fft_size // 2 + 1
        self.proc = audioproc(self.handle)
        self.proc.set_fftsize(self.fft_size)
        self.bank = Octave_Filters(bandsperoctave, n_octaves=n_octaves, response_time=response_time,
                                   handle=self.handle)
        if weighting is not None:
            self.bank.set_weighting(weighting)
        self.nbands = self.bank.nbands
        self._streams = None

    # ------------------------------------------------------------------ shapes
    def frames(self, n_samples):
        return frame_count(n_samples, self.fft_size, self.hop)

    def blocks(self, n_samples):
        if n_samples % self.hop:
            raise ValueError("the stream must be a whole number of hops")
        return n_samples // self.hop

    def _side_streams(self):
        import torch
        if self._streams is None:
            self._streams = [torch.cuda.Stream(self.device) for _ in range(3)]
        return self._streams

    # ------------------------------------------------------------------ device path
    def process(self, x, spec=None, bands=None, overlap=False):
        """x: CUDA float32 [C, n_samples] (n_samples % hop == 0).  Returns (spec [C, F, nbins]
        log-power columns, bands [C, n_samples/hop, nbands] smoothed band levels in dB).  Filter
        and smoothing state carry over from call to call (a stream can be fed in pieces; the
        spectrogram frames of a piece are those that lie inside it).

        The two kernels run back to back on the current stream.  `overlap=True` puts them on two
        streams; that is SLOWER than back to back: the
        persistent 16-warp CTAs of the HBM-bound STFT kernel squeeze onto SMs next to the
        latency-bound one-warp CTAs of the filterbank and starve them of issue slots."""
        import torch
        C, T = x.shape
        F, B = self.frames(T), self.blocks(T)
        if spec is None:
            spec = torch.empty((C, F, self.nbins), dtype=torch.float32, device=x.device)
        elif (not isinstance(spec, torch.Tensor) or spec.device != x.device or spec.dtype != torch.float32
              or tuple(spec.shape) != (C, F, self.nbins) or not spec.is_contiguous()):
            raise ValueError("spec must be a contiguous float32 tensor of shape %s on %s"
                             % ((C, F, self.nbins), x.device))
        if bands is None:
            bands = torch.empty((C, B, self.nbands), dtype=torch.float32, device=x.device)
        self._check_bands(x, bands)     # both outputs are checked before either kernel is queued
        if not overlap:
            self.proc.stft(x, hop=self.hop, log=True, out=spec)
            self._bank(x, bands)
            return spec, bands
        cur = torch.cuda.current_stream(x.device)
        s_stft, s_bank, _ = self._side_streams()
        s_stft.wait_stream(cur)
        s_bank.wait_stream(cur)
        with torch.cuda.stream(s_bank):
            self._bank(x, bands)
        with torch.cuda.stream(s_stft):
            self.proc.stft(x, hop=self.hop, log=True, out=spec)
        cur.wait_stream(s_stft)
        cur.wait_stream(s_bank)
        return spec, bands

    def _check_bands(self, x, bands):
        """The bank writes channel c, block b of every channel at bands + c*stride(0) + b*nbands."""
        x, _ = _lib.device_rows(self, x, "x")
        C, T = x.shape
        B = self.blocks(T)
        _lib.check_tensor(self, bands, "bands")
        if (bands.device != x.device or bands.dim() != 3 or tuple(bands.shape) != (C, B, self.nbands)
                or (B > 0 and bands.stride(2) != 1) or (B > 1 and bands.stride(1) != self.nbands)):
            raise ValueError("bands must be [C, n_samples/hop, nbands] = %s on %s, with stride(2) == 1 and "
                             "stride(1) == nbands" % ((C, B, self.nbands), x.device))

    def _bank(self, x, bands):
        self._check_bands(x, bands)
        x, x_stride = _lib.device_rows(self, x, "x")
        C, B = x.shape[0], bands.shape[1]
        self.bank._ensure_plan(C)
        with _lib.call_stream(x.device) as sp:
            self.handle.call("frt_bank_process_strided", _lib._ptr(x), x_stride, int(self.hop), int(B),
                             _lib._ptr(bands), int(bands.stride(0)), 1, sp)

    # ------------------------------------------------------------------ host path
    def process_host(self, x_host, spec_host=None, bands_host=None):
        """x_host: CPU float32 tensor / array [C, n_samples] (pinned memory for full PCIe speed).
        Outputs are written into the given CPU tensors (allocated pinned when omitted)."""
        import torch
        if getattr(x_host, "ndim", None) != 2:
            raise ValueError("x_host must be [C, n_samples]")
        x_host, x_stride = _lib.host_rows(x_host, "x_host")
        C, T = x_host.shape
        F, B = self.frames(T), self.blocks(T)
        if spec_host is None:
            spec_host = torch.empty((C, F, self.nbins), dtype=torch.float32, pin_memory=True)
        if bands_host is None:
            bands_host = torch.empty((C, B, self.nbands), dtype=torch.float32, pin_memory=True)
        _lib.check_host_out(spec_host, (C, F, self.nbins), "spec_host")
        _lib.check_host_out(bands_host, (C, B, self.nbands), "bands_host")
        self.proc._ensure_plan()
        self.bank._ensure_plan(C)
        self.handle.call("frt_combined_process_host", _lib._ptr(x_host), x_stride, int(C), int(T),
                         int(self.hop), _lib._ptr(spec_host), _lib._ptr(bands_host), int(self.nbands), 1)
        return spec_host, bands_host

    def close(self):
        """Release the peer-memory gather buffers (collective: every rank of the group must call it).
        Only needed when an analyzer that used `process_sharded(transport="peer")` is dropped long
        before the process ends; the buffers are otherwise freed with the process."""
        pg = getattr(self, "peer_gather", None)
        if pg is not None:
            pg.close()
            self.peer_gather = None
            self._pg_key = None

    # ------------------------------------------------------------------ multi-GPU path
    def process_sharded(self, x, gathered=None, spec_chunks=None, bands=None, n_chunks=8, group=None,
                        transport="peer", engine="auto"):
        """This rank's channels x [C, n_samples] plus the north-star's final all-gather of the
        spectrogram columns.  The columns are produced in `n_chunks` frame chunks; each chunk is on
        its way to the other GPUs while the next one is transformed, and all of that hides behind
        the filterbank kernel, which dominates the step: the step costs max(compute, link), not
        their sum.  The (short, HBM-bound) transforms run first, the (long, latency-bound)
        filterbank after them; the two compute kernels are NOT run side by side (see process()).

        transport="peer"  one-hop pushes into the peers' IPC-opened buffers over NVLink (friture_b200/peer.py):
                          copy engines up to 4 GPUs, a small copy kernel above (engine="ce"|"kernel").  The gathered array [n_chunks, world, C, F/n_chunks, nbins]
                          belongs to the analyzer (`self.peer_gather.gathered`); call
                          `self.peer_gather.wait_all()` before reading other ranks' columns.
        transport="nccl"  torch.distributed all_gather_into_tensor per chunk on a side stream into
                          `gathered` [n_chunks, world*C, F/n_chunks, nbins].
        Returns (spec_chunks, bands, gathered)."""
        import torch
        import torch.distributed as dist
        C, T = x.shape
        _, x_stride = _lib.device_rows(self, x, "x")
        F, B = self.frames(T), self.blocks(T)
        if F % n_chunks:
            raise ValueError("frames (%d) must divide into %d chunks" % (F, n_chunks))
        fc = F // n_chunks
        if bands is None:
            bands = torch.empty((C, B, self.nbands), dtype=torch.float32, device=x.device)
        self._check_bands(x, bands)
        cur = torch.cuda.current_stream(x.device)
        s_stft, s_bank, s_comm = self._side_streams()
        for s in (s_stft, s_bank, s_comm):
            s.wait_stream(cur)
        self.proc._ensure_plan()
        pg = None
        if transport == "peer":
            key = (n_chunks, C, fc, engine)
            if getattr(self, "_pg_key", None) != key:
                if getattr(self, "peer_gather", None) is not None:
                    self.peer_gather.close()
                from .peer import PeerGather
                self.peer_gather = PeerGather(self.handle, n_chunks, (C, fc, self.nbins), group=group, engine=engine)
                self._pg_key = key
            pg = self.peer_gather
            gathered = pg.gathered
        elif transport == "nccl":
            if spec_chunks is None:
                spec_chunks = torch.empty((n_chunks, C, fc, self.nbins), dtype=torch.float32, device=x.device)
        else:
            raise ValueError("transport must be 'peer' or 'nccl'")
        for i in range(n_chunks):
            dst = pg.local(i) if pg is not None else spec_chunks[i]
            with torch.cuda.stream(s_stft), _lib.call_stream(x.device) as sp:
                xi = x[:, i * fc * self.hop: (i * fc + fc - 1) * self.hop + self.fft_size]
                self.handle.call("frt_stft_process", _lib._ptr(xi), x_stride, int(C), int(fc),
                                 int(self.hop), _lib._ptr(dst), int(fc * self.nbins),
                                 int(self.nbins), _lib.STFT_LOGPOWER, sp)
            if pg is not None:
                pg.push(i, s_stft)
            else:
                s_comm.wait_stream(s_stft)
                with torch.cuda.stream(s_comm):
                    dist.all_gather_into_tensor(gathered[i], spec_chunks[i], group=group)
        s_bank.wait_stream(s_stft)
        with torch.cuda.stream(s_bank):
            self._bank(x, bands)
        cur.wait_stream(s_bank)
        cur.wait_stream(s_stft)
        cur.wait_stream(s_comm)
        if pg is not None:
            pg.join(cur)
            spec_chunks = gathered[:, pg.rank]
        return spec_chunks, bands, gathered
