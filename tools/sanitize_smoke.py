#!/usr/bin/env python
"""Small run of every kernel for compute-sanitizer (memcheck / racecheck / synccheck):
    compute-sanitizer --tool memcheck python tools/sanitize_smoke.py"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from friture_b200 import audioproc
from friture_b200.octavefilters import Octave_Filters
from friture_b200.correlation import GccPhat

torch.manual_seed(0)
p = audioproc()
# every STFT instance once: all ten sizes x both modes x 16-, 8- and 4-byte aligned frames (first
# sample at float offset 0, 2, 1 of a 16-byte aligned buffer whose row stride is a multiple of 4)
for n in (32, 64, 128, 256, 512, 1024, 2048, 4096, 8192, 16384):
    p.set_fftsize(n)
    T = n + 5 * (n // 2)
    x = torch.randn(3, T + 4, device="cuda") * 0.1
    for off in (0, 2, 1):
        for log in (False, True):
            p.stft(x[:, off:off + T], hop=n // 2, log=log)
p.set_fftsize(2048)
p.stft_host(x[:, :2048 * 3].cpu().numpy(), hop=1024)
for block in (256, 512, 1024):      # 256 / 512: the three-warp scan kernel, 1024: the one-warp kernel
    bank = Octave_Filters(3)
    x = torch.randn(3, 2 * block, device="cuda") * 0.1
    bank.filter_batch(x, block=block, want_y=True, db=True)
bank = Octave_Filters(24, n_octaves=10)
bank.energies_batch(torch.randn(2, 1024, device="cuda"), block=512)
g = GccPhat(6000)
d0 = torch.randn(3, 6000, device="cuda")
g.estimate(d0, torch.roll(d0, 5, 1), smooth=True, want_xcorr=True)
g.estimate(d0, torch.roll(d0, 5, 1), smooth=True)
torch.cuda.synchronize()
print("sanitize_smoke done")
