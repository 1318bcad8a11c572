"""CPU: the host logic of the delay estimators' per-frame track -- the widget's formulas on every
frame of a call, the frame end indices, the last frame published as the attributes -- and the
argument checks of estimate_frames that need no GPU."""
import numpy as np
import pytest
import torch

from friture_b200.correlation import GccPhat, PairGccPhat
from friture_b200.delay import DelayTrack, _DelayWidget


class _Framer:
    old_index = 0


def widget(delayrange_s=1.0, n_pairs=3):
    w = _DelayWidget.__new__(_DelayWidget)
    w.delayrange_s = delayrange_s
    w.subsampled_sampling_rate = 12000.0
    w.length = int(2 * delayrange_s * 12000)
    w.needed = int(0.5 * w.length)
    w.n_pairs = n_pairs
    w._framer = _Framer()
    w._setup_outputs(n_pairs)
    return w


def one_frame(i, v, std, delayrange_s):
    """The widget's formulas (delay_estimator.py:146-176) on one frame, as _publish ran them per frame."""
    time = 2 * delayrange_s
    with np.errstate(divide="ignore", invalid="ignore"):
        norm = np.where(std > 0, np.abs(v) / (3 * std), 0.0)
    delay = 1e3 * i / 12000.0
    delay = np.where(delay > 1e3 * time / 2., delay - 1e3 * time, delay)
    x = (norm > 1.) * (norm - 1.)
    x = (0.12 * x) ** 3
    return delay, delay * 1e-3 * 340., ((x / (1. + x)) * 100).astype(int), v


def test_track_rows_are_the_per_frame_formulas():
    rng = np.random.default_rng(0)
    w = widget(0.5, 4)
    r = 6
    idx = torch.from_numpy(rng.integers(0, w.length, (r, 4)).astype(np.int32))
    val = torch.from_numpy((rng.standard_normal((r, 4)) * 0.05).astype(np.float32))
    std = torch.from_numpy(np.abs(rng.standard_normal((r, 4))) * 1e-3)
    std[2, 1] = 0.0                                            # a silent frame
    w._framer.old_index = 10 * w.needed
    w._run_frames(r, lambda: (idx, val, std))
    t = w.track
    assert isinstance(t, DelayTrack)
    assert list(t.end_index) == [w.needed * k for k in range(5, 11)]
    for f in range(r):
        want = one_frame(idx[f].numpy().astype(np.int64), val[f].numpy().astype(np.float64), std[f].numpy(), 0.5)
        for got, exp in zip((t.delay_ms[f], t.distance_m[f], t.correlation[f], t.Xcorr_extremum[f]), want):
            assert np.array_equal(got, exp)
    assert t.correlation[2, 1] == 0
    assert np.array_equal(w.delay_ms, t.delay_ms[-1]) and np.array_equal(w.correlation, t.correlation[-1])
    assert np.array_equal(w.distance_m, t.distance_m[-1]) and np.array_equal(w.Xcorr_extremum, t.Xcorr_extremum[-1])


def test_a_call_without_frames_keeps_the_published_values():
    w = widget()
    w._framer.old_index = 4 * w.needed
    w._run_frames(2, lambda: (torch.tensor([[10, 20, 30], [40, 50, 60]], dtype=torch.int32),
                              torch.full((2, 3), 0.5), torch.full((2, 3), 0.01, dtype=torch.float64)))
    before = w.delay_ms.copy()
    w._run_frames(0, lambda: pytest.fail("no frames: no library call"))
    assert w.track.end_index.shape == (0,) and w.track.delay_ms.shape == (0, 3)
    assert np.array_equal(w.delay_ms, before)


def test_estimate_frames_checks_without_gpu():
    g = GccPhat(2400)
    with pytest.raises(ValueError):
        g.estimate_frames(np.zeros((1, 4800), np.float32), np.zeros((1, 4800), np.float32), 1200, 3)
    with pytest.raises(ValueError):
        g.estimate_frames(torch.zeros((1, 4800)), torch.zeros((1, 4800)), 1200, 3)
    with pytest.raises(ValueError):
        PairGccPhat(2400, 2, [(0, 1)]).estimate_frames(torch.zeros((2, 4800)), 1200, 3)
    with pytest.raises(ValueError, match="need 4800 samples"):
        g._frame_geometry(4799, 1200, 3)
    with pytest.raises(ValueError):
        g._frame_geometry(4800, 0, 3)
    with pytest.raises(ValueError):
        g._frame_geometry(4800, 1200, -1)
    g._frame_geometry(2400, 0, 1)
    g._frame_geometry(0, 1200, 0)
