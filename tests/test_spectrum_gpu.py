"""GPU parity: the spectrum widget's per-tick reductions (smoothing across frames, weighting, dB,
peak, harmonic product spectrum) vs the CPU oracle (friture/spectrum.py:125-222)."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from parity import assert_logpower_parity  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("fft_size,weighting", [(2048, 0), (8192, 1), (1024, 3)])
def test_spectrum_ticks(fft_size, weighting):
    import torch
    from friture_b200.spectrum import SpectrumAnalyzer
    from oracle import friture_oracle as fo
    C = 3
    rng = np.random.default_rng(fft_size)
    hop = fft_size // 4
    t = np.arange(fft_size + 9 * hop) / 48000.0
    ticks = []
    for k in range(3):
        x = rng.standard_normal((C, len(t))) * 0.05
        for c in range(C):
            f0 = 220.0 * (c + 1)
            x[c] += sum(0.3 / h * np.sin(2 * np.pi * f0 * h * t + k) for h in (1, 2, 3))
        ticks.append(x.astype(np.float32))
    an = SpectrumAnalyzer(C, fft_size=fft_size, response_time=0.125, weighting=weighting)
    A, B, Cw = fo.weighting_tables(np.linspace(0, 24000, fft_size // 2 + 1))
    w = [None, A, B, Cw][weighting]
    orcs = [fo.SpectrumWidgetOracle(fft_size, response_time=0.125, weight=w) for _ in range(C)]
    w32 = np.asarray(an.w, dtype=np.float32).astype(np.float64) if weighting else 0.0
    for x in ticks:
        db, fmax, fpitch = an.process(torch.from_numpy(x).cuda())
        db = db.cpu().numpy().astype(np.float64)
        for c in range(C):
            rdb, rfmax, rfpitch, ri, rp = orcs[c].tick(x[c])
            # take off the weight table the kernel was given (A is -998 dB at 0 Hz), then judge the
            # smoothed power's dB
            assert_logpower_parity(db[c] - w32, fo.log_spectrogram(orcs[c].disp), min_frac=0.0,
                                   strict=False, floor_db=40.0)
            assert fmax[c] == rfmax
            assert fpitch[c] == rfpitch
    assert abs(an.alpha - orcs[0].alpha) < 1e-15


def test_smoothing_state_carries_and_resets():
    import torch
    from friture_b200.spectrum import SpectrumAnalyzer
    x = (torch.randn(2, 2048 + 3 * 512) * 0.1).cuda()
    an = SpectrumAnalyzer(2, fft_size=2048, response_time=1.0)
    a1, _, _ = an.process(x)
    a2, _, _ = an.process(x)
    assert not torch.equal(a1, a2)            # history matters
    an.setfftsize(2048)                       # settings change restarts the buffers (spectrum.py:224-226)
    a3, _, _ = an.process(x)
    assert torch.equal(a1, a3)
