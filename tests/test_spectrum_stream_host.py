"""CPU: the host side of ``SpectrumAnalyzer.handle_new_data`` -- where the widget's ticks end for the
buffer sizes a host feeds and across an FFT-size change in mid-stream, and that every refusal comes
before any library call and leaves the stream and the states as they were.  The library is replaced by
a recording handle; the stream lives in CPU tensors."""
import contextlib
import ctypes
from math import floor

import numpy as np
import pytest
import torch

from friture_b200 import _lib
from friture_b200.spectrum import SpectrumAnalyzer


class RecordingHandle:
    """Stands in for a Handle: records the calls, with the tick ends the call was given, and leaves
    index 0 in every index output."""

    def __init__(self):
        self.calls = []

    def call(self, name, *args):
        rec = {"name": name}
        if name.startswith("frt_spectrum_frames"):
            dual = name.endswith("_dual")
            ends_p, R = args[5 + dual], args[6 + dual]
            rec["ends"] = list((ctypes.c_int * R).from_address(ends_p.value)) if R else []
            rec["frames"] = args[3 + dual]
            C = args[2 + dual]
            for p in args[-3:-1]:
                ctypes.memset(p.value, 0, 4 * R * C)
        self.calls.append(rec)


@pytest.fixture(autouse=True)
def host_tensors(monkeypatch):
    monkeypatch.setattr(_lib, "check_tensor", lambda owner, x, name: None)
    monkeypatch.setattr(_lib, "call_stream", lambda device, stream=None: contextlib.nullcontext(None))


def analyzer(N, C=2, dual=False):
    h = RecordingHandle()
    return SpectrumAnalyzer(C, fft_size=N, handle=h, dual_channels=dual), h


class WidgetFraming:
    """friture/spectrum.py:126-155 by the letter: which ticks draw and with how many frames."""

    def __init__(self, N):
        self.N, self.offset, self.old_index = N, 0, 0

    def tick(self, n):
        self.offset += n
        available = self.offset - self.old_index
        needed = self.N * (1. - 0.75)
        realizable = int(floor(available / needed))
        self.old_index += realizable * int(needed)
        return realizable


def run_stream(a, h, w, chunks, buffer):
    """Feed the chunks; check each call's rows against the widget's framing."""
    for n in chunks:
        per = [w.tick(buffer) for _ in range(n // buffer)] if buffer else [w.tick(n)]
        h.calls.clear()
        out = a.handle_new_data(torch.zeros(a.n_channels, n), buffer=buffer)
        want_ticks = [i for i, r in enumerate(per) if r]
        assert list(out.tick) == want_ticks
        assert list(out.n_frames) == [per[i] for i in want_ticks]
        assert out.db.shape == (a.n_channels, len(want_ticks), a.fft_size // 2 + 1)
        assert out.fmax_hz.shape == out.fpitch_hz.shape == (len(want_ticks), a.n_channels)
        frames = [c for c in h.calls if c["name"] == "frt_spectrum_frames"]
        if want_ticks:
            assert len(frames) == 1 and frames[0]["ends"] == list(np.cumsum(out.n_frames))
            assert frames[0]["frames"] == sum(per)
        else:
            assert frames == []
        assert a.old_index == w.old_index


@pytest.mark.parametrize("N", [32, 2048, 8192, 16384])
@pytest.mark.parametrize("buffer", [512, 480, 1000])
def test_tick_ends_follow_the_widget(N, buffer):
    a, h = analyzer(N)
    w = WidgetFraming(N)
    run_stream(a, h, w, [buffer * k for k in (1, 3, 1, 7, 2, 40)], buffer)
    run_stream(a, h, w, [buffer, 2 * buffer, 5 * buffer], None)   # one tick per call


@pytest.mark.parametrize("sizes", [(1024, 8192, 256), (16384, 32, 4096)])
def test_fft_size_change_in_mid_stream_keeps_old_index(sizes):
    a, h = analyzer(sizes[0])
    w = WidgetFraming(sizes[0])
    for N in sizes:
        a.setfftsize(N)
        w.N = N
        assert a._framer is None or a._framer.frame_len == N
        run_stream(a, h, w, [512 * k for k in (1, 2, 9, 1)], 512)
        run_stream(a, h, w, [480, 1000, 4097], None)


def test_no_frame_calls_and_empty_chunks():
    a, h = analyzer(8192)
    out = a.handle_new_data(torch.zeros(2, 0))
    assert out.db.shape == (2, 0, 4097) and len(out.tick) == 0 and h.calls == []
    out = a.handle_new_data(torch.zeros(2, 2047))
    assert out.fmax_hz.shape == (0, 2) and h.calls == [] and a.old_index == 0
    out = a.handle_new_data(torch.zeros(2, 1), want_db=False)
    assert out.db is None and list(out.n_frames) == [1] and a.old_index == 2048


def state(a):
    fr = a._framer
    return (fr.offset, fr.old_index, fr.frame_len) if fr is not None else None, a._disp, a._disp2, a._pairs


@pytest.mark.parametrize("dual", [False, True])
def test_refusals_come_before_any_call(dual):
    a, h = analyzer(32, C=3, dual=dual)
    shape = (lambda n: (3, 2, n)) if dual else (lambda n: (3, n))
    a.handle_new_data(torch.zeros(shape(100)), buffer=10)
    h.calls.clear()
    before = state(a)
    bad = [
        (torch.zeros(shape(100)), dict(buffer=0)),
        (torch.zeros(shape(100)), dict(buffer=-5)),
        (torch.zeros(shape(100)), dict(buffer=2.0)),
        (torch.zeros(shape(100)), dict(buffer=True)),
        (torch.zeros(shape(100)), dict(buffer=7)),               # 100 is not whole 7-sample buffers
        (torch.zeros(shape(8 * 8193)), {}),                      # one tick of 8193 frames (hop 8)
        (torch.zeros((3, 100) if dual else (3, 2, 100)), {}),    # the other shape than the stream's
        (torch.zeros(shape(100))[:2], {}),                       # channels
        (torch.zeros((3, 3, 100)), {}),
        (torch.zeros(3, 2, 2, 100), {}),
    ]
    for x, kw in bad:
        with pytest.raises(ValueError):
            a.handle_new_data(x, **kw)
        assert h.calls == [] and state(a) == before
    # 8192 frames in one tick is the limit, not past it
    out = a.handle_new_data(torch.zeros(shape(8 * 8192)))
    assert list(out.n_frames) == [8192]


def test_setters():
    a, h = analyzer(4096)
    a.handle_new_data(torch.zeros(2, 5000))
    freq = a.freq
    a._disp, a._disp2 = torch.ones(2, 2049), torch.ones(2, 2049)
    a.setminfreq(100.)
    assert a._disp is None and a._disp2 is None and a.minfreq == 100.
    a._disp = torch.ones(2, 2049)
    a.setMinMaxFreq(30., 1000.)
    assert a._disp is None and (a.minfreq, a.maxfreq) == (30., 1000.)
    a.setmaxfreq(2000.)
    assert a.maxfreq == 2000. and a.freq is freq
    oi = a.old_index
    a.setfftsize(512)
    assert a.old_index == oi and a._framer.hop == 128 and a._framer.frame_len == 512
