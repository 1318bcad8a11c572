"""CPU: the levels and long-term levels analyzers refuse bad calls with ValueError before any device
work (no handle is created), and the long-term widget frames its blocks as the reference does
(friture/longlevels.py:150-191): each block is the `needed` samples that end at old_index, the first
one the zeros before the stream, and setresptime keeps old_index."""
import numpy as np
import pytest
import torch

from friture_b200.levels import LevelsAnalyzer, LongLevelsAnalyzer


def overlapping(C, T):
    return torch.zeros(C * T).as_strided((C, T), (T // 2, 1))


@pytest.mark.parametrize("n", [0, -1])
def test_channel_count_refused(n):
    with pytest.raises(ValueError):
        LevelsAnalyzer(n)
    with pytest.raises(ValueError):
        LongLevelsAnalyzer(n)


@pytest.mark.parametrize("make", [lambda: torch.zeros(3, 1024), lambda: torch.zeros(1, 1024),
                                  lambda: torch.zeros(2, 2, 512), lambda: np.zeros((2, 1024), np.float32)])
def test_wrong_channels_or_shape_refused(make):
    for a in (LevelsAnalyzer(2), LongLevelsAnalyzer(2)):
        with pytest.raises(ValueError):
            a.handle_new_data(make())
        assert a._handle is None


@pytest.mark.parametrize("T,buffer", [(500, 512), (1000, 512), (1024, 1000), (7, 2)])
def test_partial_buffers_refused(T, buffer):
    a = LevelsAnalyzer(2)
    with pytest.raises(ValueError, match="whole number"):
        a.handle_new_data(torch.zeros(2, T), buffer=buffer)
    assert a._handle is None


def test_buffer_longer_than_kernel_refused():
    a = LevelsAnalyzer(1, response_time=0.001)       # Nk = 5 * 48 = 240 taps
    assert a.max_buffer == 240
    for buffer in (241, 512, 0, -3):
        with pytest.raises(ValueError, match="buffer"):
            a.handle_new_data(torch.zeros(1, 4 * 512), buffer=buffer)
    assert a._handle is None
    assert LevelsAnalyzer(1).max_buffer == 72000     # the widget's 0.3 s: 5 * 14400


@pytest.mark.parametrize("rt", [0.0, -0.3])
def test_meter_response_time_refused(rt):
    with pytest.raises(ValueError):
        LevelsAnalyzer(1, response_time=rt)


def test_overlapping_rows_refused():
    for a in (LevelsAnalyzer(2), LongLevelsAnalyzer(2)):
        with pytest.raises(ValueError, match="overlapping"):
            a.handle_new_data(overlapping(2, 1024))
        assert a._handle is None


@pytest.mark.parametrize("rt", [0.5, 0.999, 20.001, 60])
def test_long_response_time_refused(rt):
    with pytest.raises(ValueError):
        LongLevelsAnalyzer(1, response_time=rt)
    a = LongLevelsAnalyzer(1)
    with pytest.raises(ValueError):
        a.setresptime(rt)
    assert a.response_time == 20 and a.Ndec == 13


@pytest.mark.parametrize("d", [4, 4.99, 3600.5, 7200])
def test_duration_refused(d):
    with pytest.raises(ValueError):
        LongLevelsAnalyzer(1, duration=d)
    a = LongLevelsAnalyzer(1)
    with pytest.raises(ValueError):
        a.setduration(d)
    assert a.length_seconds == 600


@pytest.mark.parametrize("rt,ndec", [(1, 8), (2, 9), (3, 10), (5, 11), (10, 12), (17, 12), (18, 13), (20, 13)])
def test_decimation_depth(rt, ndec):
    a = LongLevelsAnalyzer(1, response_time=rt, duration=3600)
    assert a.Ndec == ndec and a.needed == 2 ** ndec
    assert a.length_samples == int(3600 * 48000 / 2 ** ndec)


def test_framing():
    a = LongLevelsAnalyzer(2, response_time=1)
    x = torch.arange(1, 6001, dtype=torch.float32).repeat(2, 1)
    x[1] *= -1
    v, e = a.take_blocks(x[:, :300])               # offset 300, old_index 0: the zero block
    assert e.tolist() == [0] and torch.equal(v, torch.zeros(2, 256))
    v, e = a.take_blocks(x[:, 300:900])            # available 644: blocks ending at 256 and 512
    assert e.tolist() == [256, 512] and torch.equal(v, x[:, :512])
    a.setresptime(3)                               # 1024-sample blocks; old_index 768 is kept
    v, e = a.take_blocks(x[:, 900:1500])           # available 732: no block
    assert v is None and e.tolist() == []
    v, e = a.take_blocks(x[:, 1500:3000])          # available 2232: blocks ending at 768 and 1792
    assert e.tolist() == [768, 1792]
    want = torch.cat([torch.zeros(2, 256), x[:, :1792]], dim=1)
    assert torch.equal(v, want)
    a.setresptime(1)
    v, e = a.take_blocks(x[:, 3000:3001])          # old_index 2816, offset 3001: none
    assert e.tolist() == []
    v, e = a.take_blocks(x[:, 3001:3100])          # offset 3100: one block ending at 2816
    assert e.tolist() == [2816] and torch.equal(v, x[:, 2560:2816])


def test_curve_before_any_block():
    t, y = LongLevelsAnalyzer(3).curve()
    assert t.shape == (0,) and y is None
