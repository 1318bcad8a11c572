#!/usr/bin/env python
"""Minimal run of every kernel for `compute-sanitizer --tool memcheck --target-processes all`."""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from friture_b200 import audioproc
from friture_b200.octavefilters import Octave_Filters
from friture_b200.correlation import GccPhat
from friture_b200.spectrum import SpectrumAnalyzer
from friture_b200.display import SpectrogramDisplay
from friture_b200.delay import Decimator
torch.manual_seed(0)
p = audioproc()
for n in (2048, 4096, 8192, 16384, 64):
    p.set_fftsize(n)
    x = torch.randn(2, n + 2 * (n // 2), device="cuda") * 0.1
    p.stft(x, hop=n // 2, log=True)
    p.stft(x[:, 1:], hop=n // 2, log=False)
for block in (256, 512, 1024):      # 256 / 512: the three-warp scan kernel, 1024: the one-warp kernel
    Octave_Filters(3).filter_batch(torch.randn(2, block, device="cuda") * 0.1, block=block, want_y=True, db=True)
    Octave_Filters(3).energies_batch(torch.randn(2, block, device="cuda") * 0.1, block=block)
g = GccPhat(1000)
d0 = torch.randn(2, 1000, device="cuda")
g.estimate(d0, torch.roll(d0, 5, 1), smooth=True, want_xcorr=True)
g.estimate(d0, torch.roll(d0, 5, 1), smooth=True)
an = SpectrumAnalyzer(2, fft_size=2048, response_time=0.125, weighting=1)
db, _, _ = an.process(torch.randn(2, 2048 + 3 * 512, device="cuda") * 0.1)
p.set_fftsize(2048)
cols = p.stft(torch.randn(2, 2048 + 4 * 512, device="cuda") * 0.1, hop=512, log=True)
SpectrogramDisplay(2, fft_size=2048, height=64, width=800).push(cols)
Decimator(2, 2).process(torch.randn(2, 512, device="cuda"))
torch.cuda.synchronize()
print("sanitize_min done")
