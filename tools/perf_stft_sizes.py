#!/usr/bin/env python
"""Throughput of the STFT kernels at the widgets' FFT sizes, 75 % overlap, 256 channels x 64 Ki samples
(the configuration of bench.py's stft_<N>_overlap75 extras)."""
import os
import sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
from friture_b200 import audioproc  # noqa: E402

PEAK = 3350.0     # H100 SXM data sheet, HBM3 GB/s
x = torch.randn(256, 64 * 1024, device="cuda") * 0.1
for n in (64, 256, 512, 1024, 2048, 4096, 8192, 16384):
    for hop in (n // 4, n // 2):
        p = audioproc()
        p.set_fftsize(n)
        F = (x.shape[1] - n) // hop + 1
        out = torch.empty((256, F, n // 2 + 1), device="cuda")
        p.stft(x, hop=hop, out=out)
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(5):
            p.stft(x, hop=hop, out=out)
        e1.record()
        torch.cuda.synchronize()
        ms = e0.elapsed_time(e1) / 5
        byts = 256 * F * (hop * 4 + (n // 2 + 1) * 4)
        print("N=%5d hop=%5d: %8.3f ms  %.3e spectra/s  %6.0f GB/s algorithmic = %.1f %% of %.0f"
              % (n, hop, ms, 256 * F / ms * 1e3, byts / ms / 1e6, byts / ms / 1e6 / PEAK * 100, PEAK),
              flush=True)
        del out
