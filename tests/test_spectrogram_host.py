"""CPU: the spectrogram widget's oracle against the pinned pieces, StreamFramer's history and
geometry change against a plain NumPy ring, and SpectrogramAnalyzer's host bookkeeping."""
from fractions import Fraction

import numpy as np
import pytest
import torch

from oracle import friture_oracle as fo
from spectrogram_oracle import SpectrogramWidgetOracle


def tone(n, seed=0):
    g = np.random.default_rng(seed)
    t = np.arange(n)
    return 0.5 * np.sin(2 * np.pi * 1000.5 * t / 48000) + 0.01 * g.standard_normal(n)


def test_oracle_composes_the_pinned_pieces():
    """One chunk holding several frames: the oracle equals the chain written out by hand, and
    chunking the same stream changes nothing but how the frames fall into calls."""
    from friture_b200.display import Linear
    N, H = 256, 20
    x = tone(N + 7 * 64 + 10)
    o = SpectrogramWidgetOracle(fft_size=N, freqscale=Linear, minfreq=100., maxfreq=20000., weighting=1,
                                height=H, width=500, timerange_s=2.)
    pix, rows, F, _ = o.push(x)
    assert F == len(x) // 64 and o.old_index == F * 64
    padded = np.concatenate([np.zeros(N), x])
    sp = fo.stft_power(padded[:N + (F - 1) * 64], N, 64).T
    freq = np.linspace(0, 24000, N // 2 + 1)
    A, _, _ = fo.weighting_tables(freq)
    norm = (fo.log_spectrogram(sp) + A[:, None] + 140.) / 140.
    want_rows = fo.frequency_resample(norm, freq, np.linspace(100., 20000., H))
    assert np.allclose(rows, want_rows, rtol=0, atol=1e-12)
    LM = Fraction(48000, N) * 4 / 1000, Fraction(500, 2000)
    want = fo.color_transform(o.lut, fo.OnlineLinear2DResamplerOracle(*LM, H).push(want_rows))
    assert np.array_equal(pix, want)

    o2 = SpectrogramWidgetOracle(fft_size=N, freqscale=Linear, minfreq=100., maxfreq=20000., weighting=1,
                                 height=H, width=500, timerange_s=2.)
    parts = [o2.push(c) for c in np.array_split(x, [5, 70, 71, 300])]
    assert sum(p[2] for p in parts) == F
    assert np.allclose(np.concatenate([p[1] for p in parts], axis=1), rows, rtol=0, atol=1e-12)
    assert np.array_equal(np.concatenate([p[0] for p in parts], axis=1), pix)


def test_oracle_setters_reset_what_the_widget_resets():
    N = 128
    o = SpectrogramWidgetOracle(fft_size=N, height=8, width=300, timerange_s=1.)
    o.push(tone(1000))
    res = o.res
    o.setmin(-100.)
    o.setweighting(2)
    o.push(tone(64, 1))
    assert o.res is res                       # same ratio: the resampler carries on
    o.setfftsize(256)
    o.push(tone(64, 2))
    assert o.res is not res and o.res.orig_index > 0   # new ratio: the indices restarted
    old = o.res.old_data.copy()
    o.set_screen(8, 600)                       # a width change is a ratio change too
    o.push(np.zeros(0))
    o.set_screen(9, 600)
    assert o.res is None
    _, rows, F, _ = o.push(tone(64, 3))
    assert F == 1 and rows.shape == (9, 1) and o.res.old_data.shape == (9,)
    assert old.shape == (8,)


# ---------------------------------------------------------------------------------------------
# StreamFramer: history and set_geometry against a NumPy ring


def ring_frames(stream, start, N, hop, F):
    """Frame f = the N samples from start + f*hop of a zero-prefixed stream."""
    padded = np.concatenate([np.zeros(16384), stream])
    return [padded[16384 + start + f * hop: 16384 + start + f * hop + N] for f in range(F)]


def test_framer_defaults_unchanged():
    from friture_b200.stream import StreamFramer
    f = StreamFramer(2, 256, 64, "cpu")
    assert f.history == 256 and f.capacity == 4 * 256 + 64 * 64
    assert f._base == -256 and f._fill == 256 and f.old_index == 0


@pytest.mark.parametrize("chunks", [[1] * 50 + [3000, 17, 5000], [4096] * 8, [100000]])
def test_framer_history_and_geometry(chunks):
    from friture_b200.stream import StreamFramer
    g = np.random.default_rng(5)
    C = 2
    fr = StreamFramer(C, 512, 128, "cpu", capacity=1000, history=4096)
    stream = np.zeros((C, 0), dtype=np.float32)
    geoms = [(512, 128), (4096, 1024), (64, 16), (2048, 512), (4096, 1024), (32, 8)]
    for i, n in enumerate(chunks):
        x = g.standard_normal((C, n)).astype(np.float32)
        stream = np.concatenate([stream, x], axis=1)
        fr.push(torch.from_numpy(x))
        N, hop = fr.frame_len, fr.hop
        before = fr.old_index
        view, F = fr.take()
        assert F == max((stream.shape[1] - before) // hop, 0)
        for c in range(C):
            want = ring_frames(stream[c], before - N, N, hop, F)
            for f in range(F):
                assert np.array_equal(view[c, f * hop:f * hop + N].numpy(), want[f]), (i, c, f)
        fr.set_geometry(*geoms[i % len(geoms)])
    with pytest.raises(ValueError):
        fr.set_geometry(8192, 2048)


# ---------------------------------------------------------------------------------------------
# SpectrogramAnalyzer's host bookkeeping (no GPU: the framer and the index only)


def test_analyzer_defaults_and_setters():
    from friture_b200.display import Erb, Mel
    from friture_b200.spectrogram import SpectrogramAnalyzer
    a = SpectrogramAnalyzer(3)
    d = a.display
    assert (a.fft_size, a.hop, d.scale, d.minfreq, d.maxfreq) == (4096, 1024, Mel, 20., 24000.)
    assert (d.spec_min, d.spec_max, d.weighting, d.height, d.width, d.timerange_s) == (-140., 0., 0, 512, 1024, 10.)
    d.index.orig_index, d.index.resampled_index = 5., 4.
    d._tables = {"dummy": 1}
    for setter, arg in [("setmin", -120.), ("setmax", -10.), ("timerangechanged", 5.)]:
        getattr(a, setter)(arg)
        assert d._tables == {"dummy": 1} and d.index.orig_index == 5.
    assert (d.spec_min, d.spec_max, d.timerange_s) == (-120., -10., 5.)
    for setter, arg in [("setminfreq", 50.), ("setmaxfreq", 12000.), ("setfreqscale", Erb), ("setweighting", 3)]:
        d._tables = {"dummy": 1}
        getattr(a, setter)(arg)
        assert d._tables is None and d.index.orig_index == 5.     # the tables only
    assert (d.minfreq, d.maxfreq, d.scale, d.weighting) == (50., 12000., Erb, 3)
    d._old = "carried"
    a.setfftsize(1024)
    assert a.fft_size == 1024 and a.hop == 256 and len(d.freq) == 513 and d._old == "carried"
    assert d.sfft_rate_frac == Fraction(48000, 1024) * 4 / 1000
    a.set_screen(512, 2048)
    assert d._old == "carried" and d.width == 2048
    a.set_screen(300, 2048)
    assert d._old is None and d.index.orig_index == 0. and d.height == 300
    with pytest.raises(ValueError):
        a.setfftsize(1000)
    with pytest.raises(ValueError):
        SpectrogramAnalyzer(1, fft_size=32768)


def test_analyzer_frames_per_call():
    """The framer the analyzer builds: frames per call and old_index across a mid-stream fft-size
    change, as the widget's framing loop gives them."""
    from friture_b200.stream import StreamFramer
    from friture_b200.spectrogram import SpectrogramAnalyzer
    fr = StreamFramer(1, 4096, 1024, "cpu", capacity=2 * SpectrogramAnalyzer.HISTORY,
                      history=SpectrogramAnalyzer.HISTORY)
    counts = []
    for n, size in [(1000, None), (100, None), (5000, 16384), (3000, None), (700, 256), (0, None)]:
        if size:
            fr.set_geometry(size, size // 4)
        fr.push(torch.zeros(1, n))
        counts.append(fr.take()[1])
    # 1000 < hop; 1100 -> 1 frame (old_index 1024); +5000 = 6100 at hop 4096 -> 1 (5120);
    # +3000 = 9100 -> 0; +700 = 9800 at hop 64 -> 73 (9792); +0 -> 0
    assert counts == [0, 1, 1, 0, 73, 0] and fr.old_index == 9792
