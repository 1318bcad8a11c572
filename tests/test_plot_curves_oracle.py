"""CPU: the spectrum and octave widgets' plotted curves and peak hold.

- The float64 restatement ``oracle.plot_curves.PlotCurvesOracle`` reproduces the reference's curves
  in tests/golden/plot_curves.npz bit for bit, and its final peak state.
- ``friture_b200.plotcurves``' host side (the x edges on every frequency scale, the baseline, the
  frequency trackers) reproduces the fixture's.
- Where the reference tree exists: the fixture is what the unmodified widgets compute now, and the
  restatement matches them on fresh random inputs and settings.
- ``SpectrumPlot`` / ``HistPlot`` argument checks and setter semantics that need no GPU."""
import os

import numpy as np
import pytest

from oracle.plot_curves import D0, PlotCurvesOracle, fixture_ticks

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "plot_curves.npz")
SPECTRUM_CASES = ["mel", "lin", "log", "log0", "erb", "oct"]
OCTAVE_CASES = ["hist3", "hist24"]


@pytest.fixture(scope="module")
def gold():
    with np.load(GOLD) as d:
        return {k: d[k] for k in d.files}


def reference_or_skip():
    from oracle import ref_import
    if not ref_import.available():
        pytest.skip("reference tree not present")
    from oracle.plot_curves import reference_widgets
    return reference_widgets()


def scale_of(name):
    from friture_b200 import display
    return {s.NAME: s for s in display.SCALES.values()}[name]


@pytest.mark.parametrize("case", SPECTRUM_CASES + OCTAVE_CASES)
def test_oracle_reproduces_fixture(gold, case):
    o = PlotCurvesOracle()
    for d in fixture_ticks(gold, case):
        if d["paused"]:
            continue
        o.setspecrange(d["spec_min"], d["spec_max"])
        sy, z, sp, zp = o.setdata(d["y"], peaks=d["peaks"])
        assert np.array_equal(sy, d["sy"]) and np.array_equal(z, d["z"]), d["t"]
        if d["peaks"]:
            assert np.array_equal(sp, d["speak"]) and np.array_equal(zp, d["zpeak"]), d["t"]
    for n, a in (("peak", o.peak), ("peak_int", o.peak_int), ("decay", o.peak_decay)):
        assert np.array_equal(a, gold[case + "_" + n])


def test_fixture_covers_the_state_machine(gold):
    """Holds of 64 ticks, falls of 40+ ticks, re-rises during a fall, ties, the reset."""
    o = PlotCurvesOracle(-100, -20)
    longest_fall = ties = rerise = 0
    fall = None
    for d in fixture_ticks(gold, "mel"):
        if d["paused"] or not d["peaks"]:
            continue
        y = d["y"].astype(np.float64)
        if o.peak.shape == y.shape:
            ties += int(np.sum(o.peak == y))
            rerise += int(np.sum((o.peak < y) & (o.peak_int < 0.2)))
        o.setdata(y)
        falling = o.peak_decay < D0
        fall = np.where(falling, (0 if fall is None or fall.shape != y.shape else fall) + 1, 0)
        longest_fall = max(longest_fall, int(fall.max()))
    assert longest_fall > 40 and ties > 100 and rerise > 100
    assert np.any(np.diff(gold["mel_K"]) != 0)


@pytest.mark.parametrize("case", SPECTRUM_CASES)
def test_spectrum_host_side_matches_fixture(gold, case):
    from friture_b200.plotcurves import SpectrumPlot, format_frequency, to_screen
    from friture_b200 import display
    scale, fmin, fmax = gold[case + "_settings"]
    p = SpectrumPlot(1, freqscale=scale_of(scale), minfreq=int(fmin), maxfreq=int(fmax))
    xl, xr = p.edges(int(gold[case + "_K"][-1]))
    assert np.array_equal(xl, gold[case + "_xl"]) and np.array_equal(xr, gold[case + "_xr"])
    for d in fixture_ticks(gold, case):
        if d["paused"]:
            continue
        p.setspecrange(d["spec_min"], d["spec_max"])
        base = 1.0 - to_screen(display.Linear, p.spec_min, p.spec_max, 0.0) if d["data_baseline"] else 1.0
        assert base == d["baseline"]
        t = d["t"]
        assert float(to_screen(p.scale, p.xmin, p.xmax, d["fmax"])) == gold[case + "_fmax_x"][t]
        assert float(to_screen(p.scale, p.xmin, p.xmax, d["fpitch"])) == gold[case + "_fpitch_x"][t]
        assert format_frequency(d["fpitch"]) == gold[case + "_fpitch_text"][t]
    # push() places the trackers of all channels with one call each and formats their text on demand
    from friture_b200.plotcurves import SpectrumCurves
    drawn = gold[case + "_ctrl"][:, 2] == 0
    fmax_hz, fpitch_hz = gold[case + "_fmax"][drawn], gold[case + "_fpitch"][drawn]
    c = SpectrumCurves(xl, xr, 1.0, None, None, fmax_hz=fmax_hz, fpitch_hz=fpitch_hz,
                       fmax_x=to_screen(p.scale, p.xmin, p.xmax, fmax_hz),
                       fpitch_x=to_screen(p.scale, p.xmin, p.xmax, fpitch_hz))
    assert np.array_equal(c.fmax_x, gold[case + "_fmax_x"][drawn])
    assert np.array_equal(c.fpitch_x, gold[case + "_fpitch_x"][drawn])
    assert c.fmax_text == list(gold[case + "_fmax_text"][drawn])
    assert c.fpitch_text == list(gold[case + "_fpitch_text"][drawn])


@pytest.mark.parametrize("case", OCTAVE_CASES)
def test_octave_host_side_matches_fixture(gold, case):
    from friture_b200.octavespectrum import OctaveSpectrumAnalyzer
    from friture_b200.plotcurves import HistPlot
    bpo = int(gold[case + "_settings"][0])
    an = OctaveSpectrumAnalyzer(1, bandsperoctave=1 if case == "hist3" else bpo)   # hist3 ends on bpo 1
    xl, xr, bar_x = HistPlot(1, an).edges()
    assert np.array_equal(xl, gold[case + "_xl"]) and np.array_equal(xr, gold[case + "_xr"])
    assert np.array_equal(bar_x, (xl + xr) / 2)
    an.setbandsperoctave(bpo)
    assert np.array_equal(np.asarray(an.f_nominal), gold[case + "_f_nominal"])


def test_fixture_is_what_the_reference_computes(gold):
    reference_or_skip()
    from oracle.make_golden_plot import generate
    fresh = generate()
    assert sorted(fresh) == sorted(gold)
    for k, v in fresh.items():
        assert np.array_equal(np.asarray(v), gold[k]), k


@pytest.mark.parametrize("seed", range(4))
def test_oracle_matches_unmodified_widgets(seed):
    """Random K, ranges (swapped, empty), steps and settings, spectrum and octave widget."""
    spw, hp, fscales = reference_or_skip()
    from oracle.plot_curves import curve_arrays
    from friture_b200.plotcurves import SpectrumPlot
    rng = np.random.default_rng(seed)
    K = int(rng.choice([17, 33, 257, 1025]))
    w = spw.SpectrumPlotWidget(None)
    w.set_peaks_enabled(True)
    scale = fscales.ALL[seed % len(fscales.ALL)]
    w.setfreqscale(scale)
    w.setfreqrange(20 * seed, 20000)
    h = hp.HistPlot(None)
    o, oh = PlotCurvesOracle(), PlotCurvesOracle()
    x = np.linspace(0, 24000, K)
    fl = np.geomspace(40, 16000, 30)
    ranges = [(-100, -20), (0, -140), (-60, -60), (-120.5, 3.25)]
    for t in range(150):
        sm, sM = ranges[(t // 40) % len(ranges)]
        for ww in (w, h, o, oh):
            ww.setspecrange(sm, sM)
        y = (-80 + 20 * rng.standard_normal(K) * (rng.random() < 0.3)).astype(np.float32).astype(np.float64)
        yh = (-70 + 15 * rng.standard_normal(30) * (rng.random() < 0.2)).astype(np.float32).astype(np.float64)
        w.setdata(x, y, 1000., 440.)
        h.setdata(fl, fl * 1.2, fl * 1.1, yh)
        for ww, oo, yy in ((w, o, y), (h, oh, yh)):
            r = oo.setdata(yy)
            got = curve_arrays(ww._curve_signal)[2:4] + curve_arrays(ww._curve_peak)[2:4]
            for a, b in zip(got, r):
                assert np.array_equal(a, b), t
    p = SpectrumPlot(1, freqscale=scale_of(scale.NAME), minfreq=20 * seed, maxfreq=20000)
    xl, xr = p.edges(K)
    assert np.array_equal(xl, curve_arrays(w._curve_signal)[0])
    assert np.array_equal(xr, curve_arrays(w._curve_signal)[1])


def test_plot_setters_without_gpu():
    import torch
    from friture_b200.octavespectrum import OctaveSpectrumAnalyzer
    from friture_b200.plotcurves import PEAK_DECAY, HistPlot, SpectrumPlot
    assert PEAK_DECAY == D0 and -0.131 < D0 < -0.130
    p = SpectrumPlot(2)
    assert (p.spec_min, p.spec_max, p.peaks_enabled, p.data_baseline) == (-100., -20., True, False)
    p.setspecrange(0, -140)
    assert (p.spec_min, p.spec_max) == (-140, 0)
    p.setdualchannels(True)
    assert not p.peaks_enabled and p.data_baseline
    p.setdualchannels(False)
    assert p.peaks_enabled and not p.data_baseline
    p.pause()
    assert p.push(None, 0., 0.) is None         # paused before any data: nothing to show
    p.restart()
    assert p.push(None, 0., 0., n_frames=0) is None
    for bad in (torch.zeros((2, 33)), torch.zeros((2, 33), dtype=torch.float64), torch.zeros((3, 1, 33)),
                np.zeros((2, 1, 33), np.float32)):
        with pytest.raises(ValueError):
            p._run(bad, True)
    h = HistPlot(2, OctaveSpectrumAnalyzer(2))
    assert (h.spec_min, h.spec_max) == (-80., -20.)
    with pytest.raises(ValueError):
        h.push(torch.zeros((2, 1, 28)))             # 27 bands at bpo 3
    assert p._handle is None and h._handle is None  # nothing above needed a GPU
