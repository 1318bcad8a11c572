"""CPU: the host logic of ``SpectrumAnalyzer.process_ticks`` -- the tick geometry, the default frames per
tick at every FFT size, and the refusals that come before any library call -- and the checks of
``SpectrumPlot.push_ticks`` that need no GPU."""
import numpy as np
import pytest
import torch

from friture_b200._lib import FrtValueError
from friture_b200.plotcurves import SpectrumPlot
from friture_b200.spectrum import SpectrumAnalyzer, SpectrumTicks

FFT_SIZES = [2 ** k for k in range(5, 15)]


class RecordingHandle:
    """Stands in for a Handle: records the calls instead of making them."""

    def __init__(self):
        self.calls = []

    def call(self, name, *args):
        self.calls.append((name, args))


def analyzer(N, C=2, dual=False):
    h = RecordingHandle()
    return SpectrumAnalyzer(C, fft_size=N, handle=h, dual_channels=dual), h


@pytest.mark.parametrize("N", FFT_SIZES)
def test_default_frames_per_tick_is_one_buffer(N):
    """The widget draws once per 512-sample buffer (audiobackend.py:32): 512 / hop frames, at least one."""
    a, _ = analyzer(N)
    assert a.hop == N // 4
    want = {32: 64, 64: 32, 128: 16, 256: 8, 512: 4, 1024: 2}.get(N, 1)
    assert a.default_frames_per_tick() == want
    g, R = a.tick_geometry(R_samples(a, want, 5))
    assert (g, R) == (want, 5)


def R_samples(a, g, R):
    """Samples per row that hold R ticks of g frames: the last tick's frames end at the last sample."""
    return R * g * a.hop + a.fft_size - a.hop


@pytest.mark.parametrize("N", [32, 1024, 16384])
@pytest.mark.parametrize("g", [1, 2, 16, 8192])
def test_tick_geometry(N, g):
    a, _ = analyzer(N)
    for R in (0, 1, 7, 64):
        assert a.tick_geometry(R_samples(a, g, R), g) == (g, R)
        # samples past the last whole frame change nothing
        assert a.tick_geometry(R_samples(a, g, R) + a.hop - 1, g) == (g, R)
    # tick r of a call is x[..., r*g*hop : (r+1)*g*hop + N - hop]: g frames each, tiling the call's frames
    for r in range(3):
        lo, hi = r * g * a.hop, (r + 1) * g * a.hop + N - a.hop
        assert (hi - lo - N) // a.hop + 1 == g
    assert a.tick_geometry(N - 1, g) == (g, 0)


@pytest.mark.parametrize("g", [0, -1, 8193, 2.0, True, "2", None])
def test_bad_frames_per_tick_is_refused_before_any_call(g):
    a, h = analyzer(1024)
    x = torch.zeros(2, R_samples(a, 2, 4))
    if g is None:               # the default is fine
        assert a.tick_geometry(x.shape[1]) == (2, 4)
        return
    with pytest.raises(FrtValueError):
        a.process_ticks(x, frames_per_tick=g)
    assert h.calls == [] and a._disp is None


@pytest.mark.parametrize("dual", [False, True])
def test_frames_not_whole_ticks_are_refused_before_any_call(dual):
    a, h = analyzer(256, C=3, dual=dual)
    T = 10 * a.hop + 256 - a.hop                    # 10 frames
    x = torch.zeros((3, 2, T) if dual else (3, T))
    for g in (3, 4, 6, 7, 11):
        with pytest.raises(FrtValueError):
            a.process_ticks(x, frames_per_tick=g)
    with pytest.raises(FrtValueError):
        a.process_ticks(x)                          # 8 frames per tick by default at N = 256
    assert h.calls == [] and a._disp is None and a._disp2 is None


def test_bad_shapes_are_refused_before_any_call():
    a, h = analyzer(1024, C=2)
    for x in (torch.zeros(3, 2048), torch.zeros(2, 3, 2048), torch.zeros(2, 1, 1, 2048)):
        with pytest.raises(ValueError):
            a.process_ticks(x)
    assert h.calls == []


def test_push_ticks_checks():
    p = SpectrumPlot(2, handle=RecordingHandle())
    fm = np.zeros((3, 2))
    with pytest.raises(ValueError):
        p.push_ticks(SpectrumTicks(None, fm, fm))            # no dB was asked for
    with pytest.raises(ValueError):
        p.push_ticks(SpectrumTicks(torch.zeros(2, 513), fm, fm))
    assert p.push_ticks(SpectrumTicks(torch.zeros(2, 0, 513), fm[:0], fm[:0])) is None
    p.pause()
    assert p.push_ticks(SpectrumTicks(torch.zeros(2, 3, 513), fm, fm)) is None
    assert p._handle.calls == []
