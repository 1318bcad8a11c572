"""The spectrum and octave widgets' plotted curves and peak hold on the GPU (``frt_plot_curves``,
``csrc/reduce.cu``, behind ``friture_b200.plotcurves.SpectrumPlot`` and ``HistPlot``).

The reference is ``oracle.plot_curves.PlotCurvesOracle``, the float64 restatement of
SpectrumPlotWidget.setdata / HistPlot.setdata and compute_peaks that the CPU tests hold bit for bit
to the unmodified widgets.  Fed the same float32 dB vectors, the kernel must match it exactly: the
float64 peak state (peak, intensity, decay) bit for bit, and the four float32 curves equal to the
reference's float64 curves rounded once to float32."""
import numpy as np
import pytest

from oracle.plot_curves import D0, PlotCurvesOracle, fixture_ticks

pytestmark = pytest.mark.gpu

SPECTRUM_BINS = [2 ** k + 1 for k in range(4, 14)]          # N = 32 ... 16384: 17 ... 8193 bins
RANGES = [(-100, -20), (0, -140), (-60, -60), (-120.5, 3.25), (-80, -20)]


def torch_():
    import torch
    return torch


def db_stack(rng, C, S, K):
    """float32 dB [C, S, K]: channel 0 silence (-300 dB), channel 1 constant, the others noisy with
    bursts, quiet stretches and exact repeats of the previous step."""
    y = -85 + 6 * rng.standard_normal((C, S, K))
    burst = rng.random((C, S, K)) < 0.02
    y[burst] = rng.uniform(-60, -10, burst.sum())
    if S > 3:
        y[:, 2] = y[:, 1]                      # ties
    if S > 120:
        y[:, 40:110] = -250.                   # a hold, then a long fall
    y[0] = -300.
    if C > 1:
        y[1] = -42.5
    return y.astype(np.float32)


def check(res, orc, ref, peaks=True):
    """Kernel outputs (y, z, peak, z_peak) and the plot's state against the oracle's."""
    names = ("y", "z", "peak", "z_peak")
    for n, got, want in zip(names, res, ref):
        if want is None:
            assert got is None, n
            continue
        got = got.cpu().numpy()
        assert np.array_equal(got, np.asarray(want, dtype=np.float32)), n


def check_state(plot, orc):
    for got, want in ((plot.peak, orc.peak), (plot.peak_int, orc.peak_int), (plot.peak_decay, orc.peak_decay)):
        assert np.array_equal(got.cpu().numpy(), want)


def step_oracle(orc, y, peaks=True):
    """The widget's setdata once per step of y [C, S, K]; returns the last call's curves."""
    for s in range(y.shape[1]):
        r = orc.setdata(y[:, s].astype(np.float64), peaks=peaks)
    return r


def plot_state(C):
    from friture_b200.plotcurves import _PlotState
    return _PlotState(C, -100, -20, None)


@pytest.mark.parametrize("K", SPECTRUM_BINS)
def test_spectrum_bin_counts(K):
    torch = torch_()
    from friture_b200.plotcurves import SpectrumPlot
    rng = np.random.default_rng(K)
    C = 5
    p = SpectrumPlot(C)
    orc = PlotCurvesOracle(-100, -20)
    y = db_stack(rng, C, 12, K)
    for t in range(12):
        sm, sM = RANGES[t % len(RANGES)]
        p.setspecrange(sm, sM)
        orc.setspecrange(sm, sM)
        res = p.push(torch.from_numpy(y[:, t]).cuda(), np.full(C, 1000.), np.full(C, 440.))
        check((res.y, res.z, res.peak, res.z_peak), orc, orc.setdata(y[:, t].astype(np.float64)))
    check_state(p, orc)


@pytest.mark.parametrize("n_octaves", [9, 10])
@pytest.mark.parametrize("bpo", range(1, 25))
def test_octave_band_counts_and_steps(bpo, n_octaves):
    """K = bpo * n_octaves bands; pushes of 1, 7 and 230 steps."""
    torch = torch_()
    K = bpo * n_octaves
    rng = np.random.default_rng(100 * bpo + n_octaves)
    C = 4
    st = plot_state(C)
    orc = PlotCurvesOracle(-100, -20)
    for i, S in enumerate((1, 7, 230)):
        sm, sM = RANGES[(bpo + i) % len(RANGES)]
        st.setspecrange(sm, sM)
        orc.setspecrange(sm, sM)
        y = db_stack(rng, C, S, K)
        res = st._run(torch.from_numpy(y).cuda(), True)
        check(res, orc, step_oracle(orc, y))
    check_state(st, orc)


def test_more_channels_than_sms_and_strides():
    """2 * SMs + 5 channels at 4097 bins, and a strided stack (a step stride past K, a channel
    stride past S * step stride) through the C ABI."""
    torch = torch_()
    from ctypes import c_double
    from friture_b200 import _lib
    from friture_b200.plotcurves import PEAK_DECAY
    h = _lib.default_handle()
    C, S, K = 2 * h.sm_count + 5, 3, 4097
    rng = np.random.default_rng(7)
    y = db_stack(rng, C, S, K)
    st = plot_state(C)
    orc = PlotCurvesOracle(-100, -20)
    res = st._run(torch.from_numpy(y).cuda(), True)
    check(res, orc, step_oracle(orc, y))
    check_state(st, orc)
    # strided: [C, S, K] inside a NaN-padded [C, S + 1, K + 7] buffer
    buf = torch.full((C, S + 1, K + 7), float("nan"), dtype=torch.float32, device="cuda")
    y2 = db_stack(rng, C, S, K)
    buf[:, :S, :K] = torch.from_numpy(y2).cuda()
    out = [torch.empty((C, K), dtype=torch.float32, device="cuda") for _ in range(4)]
    h.call("frt_plot_curves", _lib._ptr(buf), (S + 1) * (K + 7), K + 7, C, S, K, c_double(-100.),
           c_double(-20.), c_double(PEAK_DECAY), 1, 0, _lib._ptr(st.peak), _lib._ptr(st.peak_int),
           _lib._ptr(st.peak_decay), *[_lib._ptr(t) for t in out], _lib.current_stream_ptr())
    check(out, orc, step_oracle(orc, y2))
    check_state(st, orc)


def test_rejected_arguments():
    torch = torch_()
    from ctypes import c_double
    from friture_b200 import _lib
    h = _lib.default_handle()
    y = torch.zeros((2, 3, 5), dtype=torch.float32, device="cuda")
    o = [torch.empty((2, 5), dtype=torch.float32, device="cuda") for _ in range(4)]
    s = [torch.empty((2, 5), dtype=torch.float64, device="cuda") for _ in range(3)]
    good = [y, 15, 5, 2, 3, 5, c_double(-100.), c_double(-20.), c_double(D0), 1, 1, *s, *o]
    bad = {4: 0, 5: 0, 2: -5, 1: -15, 6: c_double(0.), 9: 1}
    for i, v in bad.items():
        args = list(good)
        args[i] = v
        if i == 9:
            args[9 + 3] = None                   # peaks on with no peak-state buffer
        with pytest.raises(ValueError):
            h.call("frt_plot_curves", *[_lib._ptr(a) if isinstance(a, torch.Tensor) else a for a in args],
                   _lib.current_stream_ptr())
    with pytest.raises(ValueError):
        plot_state(2)._run(torch.zeros((2, 0, 5), dtype=torch.float32, device="cuda"), True)


def test_rejected_call_keeps_the_pending_reset():
    """A call rejected after the bin count changed leaves no state of the new size behind: the next
    good call still starts from the reset (-500, 0, d0), not from unwritten memory."""
    torch = torch_()
    from friture_b200 import _lib
    from friture_b200.plotcurves import SpectrumPlot
    rng = np.random.default_rng(13)
    C = 3
    h = _lib.default_handle()

    class Rejecting:                       # the handle, with one call refused by the C side
        sm_count = h.sm_count
        check_device = staticmethod(h.check_device)

        def call(self, name, *args):
            raise _lib.FrtValueError(_lib.FRT_EINVAL, "refused")

    p = SpectrumPlot(C)
    f = np.full(C, 1000.)
    y0 = db_stack(rng, C, 1, 65)[:, 0]
    p.push(torch.from_numpy(y0).cuda(), f, f)
    y1 = db_stack(rng, C, 2, 129)
    p._handle = Rejecting()
    with pytest.raises(ValueError):
        p.push(torch.from_numpy(y1[:, 0]).cuda(), f, f)
    assert p.peak.shape == (C, 65)
    p._handle = h
    r = p.push(torch.from_numpy(y1[:, 1]).cuda(), f, f)
    fresh = PlotCurvesOracle(-100, -20)
    check((r.y, r.z, r.peak, r.z_peak), fresh, fresh.setdata(y1[:, 1].astype(np.float64)))
    check_state(p, fresh)


def test_broadcast_input():
    """One dB vector for every channel as a stride-0 view, read without a copy."""
    torch = torch_()
    rng = np.random.default_rng(17)
    C, S, K = 5, 4, 257
    y = db_stack(rng, 3, S, K)[2]
    st = plot_state(C)
    orc = PlotCurvesOracle(-100, -20)
    res = st._run(torch.from_numpy(y).cuda().expand(C, S, K), True)
    check(res, orc, step_oracle(orc, np.broadcast_to(y, (C, S, K))))
    check_state(st, orc)


def test_one_push_equals_many():
    """One push of n blocks gives the same bits as n pushes of one block."""
    torch = torch_()
    rng = np.random.default_rng(3)
    C, S, K = 6, 150, 216
    y = torch.from_numpy(db_stack(rng, C, S, K)).cuda()
    a, b = plot_state(C), plot_state(C)
    ra = a._run(y, True)
    for s in range(S):
        rb = b._run(y[:, s:s + 1], True)
    for x, z in zip(ra, rb):
        assert torch.equal(x, z)
    for x, z in ((a.peak, b.peak), (a.peak_int, b.peak_int), (a.peak_decay, b.peak_decay)):
        assert torch.equal(x, z)


def test_spectrum_setters():
    """Pause, peaks off and on (state frozen), the dual-channel baseline, a K change resetting the
    state, a range change rescaling the curves without touching the state."""
    torch = torch_()
    from friture_b200.plotcurves import SpectrumPlot, to_screen
    from friture_b200 import display
    rng = np.random.default_rng(11)
    C, K = 3, 257
    y = db_stack(rng, C, 40, K)
    p = SpectrumPlot(C)
    orc = PlotCurvesOracle(-100, -20)
    f = np.full(C, 1000.)
    push = lambda t, **k: p.push(torch.from_numpy(y[:, t]).cuda(), f, f, **k)   # noqa: E731
    for t in range(5):
        r = push(t)
        orc.setdata(y[:, t].astype(np.float64))
    p.pause()
    assert push(5) is r
    p.restart()
    assert push(5, n_frames=0) is r
    state = [x.clone() for x in (p.peak, p.peak_int, p.peak_decay)]
    p.setdualchannels(True)
    r = push(6)
    assert r.peak is None and r.z_peak is None
    assert r.baseline == 1.0 - to_screen(display.Linear, -100, -20, 0.0) and r.baseline != 1.0
    check((r.y, r.z, None, None), orc, orc.setdata(y[:, 6].astype(np.float64), peaks=False))
    for a, b in zip(state, (p.peak, p.peak_int, p.peak_decay)):
        assert torch.equal(a, b)                  # frozen while peaks are off
    p.setdualchannels(False)
    r = push(7)
    assert r.baseline == 1.0
    check((r.y, r.z, r.peak, r.z_peak), orc, orc.setdata(y[:, 7].astype(np.float64)))
    # a new range rescales the next curves; the state steps on as before
    p.setspecrange(-20, -140)
    orc.setspecrange(-20, -140)
    r = push(8)
    check((r.y, r.z, r.peak, r.z_peak), orc, orc.setdata(y[:, 8].astype(np.float64)))
    check_state(p, orc)
    # a K change resets: peak -500, intensity 0, decay d0 before the first step
    y2 = db_stack(rng, C, 1, 513)[:, 0]
    r = p.push(torch.from_numpy(y2).cuda(), f, f)
    fresh = PlotCurvesOracle(-20, -140)
    check((r.y, r.z, r.peak, r.z_peak), fresh, fresh.setdata(y2.astype(np.float64)))
    check_state(p, fresh)
    assert r.x_left.shape == (513,)


def test_octave_setters():
    torch = torch_()
    from friture_b200.octavespectrum import OctaveSpectrumAnalyzer
    from friture_b200.plotcurves import HistPlot
    an = OctaveSpectrumAnalyzer(2)
    h = HistPlot(2, an)
    orc = PlotCurvesOracle(-80, -20)
    rng = np.random.default_rng(5)
    y = db_stack(rng, 2, 10, an.nbands)
    r = h.push(torch.from_numpy(y).cuda())
    check((r.y, r.z, r.peak, r.z_peak), orc, step_oracle(orc, y))
    h.pause()
    assert h.push(torch.from_numpy(y).cuda()) is r
    h.restart()
    an.setbandsperoctave(6)
    y = db_stack(rng, 2, 4, an.nbands)
    r = h.push(torch.from_numpy(y).cuda())
    fresh = PlotCurvesOracle(-80, -20)
    check((r.y, r.z, r.peak, r.z_peak), fresh, step_oracle(fresh, y))
    check_state(h, fresh)
    assert np.array_equal(r.bar_label_f, an.f_nominal) and r.bar_label_x.shape == (an.nbands,)


@pytest.mark.parametrize("case", ["mel", "lin", "log", "log0", "erb", "oct", "hist3", "hist24"])
def test_golden_fixture(golden_dir, case):
    """tests/golden/plot_curves.npz, made with the unmodified widgets, reproduced bit for bit on
    three identical channels."""
    import os
    torch = torch_()
    from friture_b200.octavespectrum import OctaveSpectrumAnalyzer
    from friture_b200.plotcurves import HistPlot, SpectrumPlot
    from friture_b200 import display
    with np.load(os.path.join(golden_dir, "plot_curves.npz")) as d:
        g = {k: d[k] for k in d.files}
    C = 3
    if case.startswith("hist"):
        an = OctaveSpectrumAnalyzer(C, bandsperoctave=int(g[case + "_settings"][0]))
        p = HistPlot(C, an)
    else:
        scale, fmin, fmax = g[case + "_settings"]
        p = SpectrumPlot(C, freqscale={s.NAME: s for s in display.SCALES.values()}[scale],
                         minfreq=int(fmin), maxfreq=int(fmax))
    r = None
    for d in fixture_ticks(g, case):
        p.setspecrange(d["spec_min"], d["spec_max"])
        p.pause() if d["paused"] else p.restart()
        y = torch.from_numpy(np.tile(d["y"], (C, 1))).cuda()
        if case.startswith("hist"):
            if len(d["y"]) != an.nbands:
                an.setbandsperoctave(1)
            r = p.push(y[:, None, :])
        else:
            p.set_peaks_enabled(d["peaks"])
            p.set_baseline_dataUnits(0.) if d["data_baseline"] else p.set_baseline_displayUnits(0.)
            r = p.push(y, d["fmax"], d["fpitch"])
            t = d["t"]
            assert np.all(r.fmax_x == g[case + "_fmax_x"][t]) and np.all(r.fpitch_x == g[case + "_fpitch_x"][t])
            assert r.fmax_text == [g[case + "_fmax_text"][t]] * C
            assert r.fpitch_text == [g[case + "_fpitch_text"][t]] * C
        assert r.baseline == d["baseline"]
        want = [d["sy"], d["z"]] + ([d["speak"], d["zpeak"]] if d["peaks"] else [None, None])
        for got, w in zip((r.y, r.z, r.peak, r.z_peak), want):
            if w is not None:
                assert np.array_equal(got.cpu().numpy(), np.tile(w.astype(np.float32), (C, 1))), d["t"]
    for n, a in (("peak", p.peak), ("peak_int", p.peak_int), ("decay", p.peak_decay)):
        assert np.array_equal(a.cpu().numpy(), np.tile(g[case + "_" + n], (C, 1)))
    assert np.array_equal(r.x_left, g[case + "_xl"]) and np.array_equal(r.x_right, g[case + "_xr"])


def test_end_to_end_spectrum():
    """SpectrumAnalyzer -> SpectrumPlot over ticks of 0, 1 and several frames: the curves equal the
    oracle fed the analyzer's own dB bits, on the ticks the widget draws."""
    torch = torch_()
    from friture_b200.audioproc import frame_count
    from friture_b200.plotcurves import SpectrumPlot
    from friture_b200.spectrum import SpectrumAnalyzer
    C, N = 3, 1024
    an = SpectrumAnalyzer(C, fft_size=N, weighting=1)
    p = SpectrumPlot(C)
    orc = PlotCurvesOracle(-100, -20)
    rng = np.random.default_rng(9)
    last = None
    for i, T in enumerate((N + 3 * 256, N - 1, N, N + 7 * 256, 200, N + 256)):
        x = torch.from_numpy((rng.standard_normal((C, T)) * 10 ** (-i % 3)).astype(np.float32)).cuda()
        nf = frame_count(T, N, an.hop)
        db, fmax, fpitch = an.process(x)
        r = p.push(db, fmax, fpitch, n_frames=nf)
        if nf == 0:
            assert r is last
            continue
        check((r.y, r.z, r.peak, r.z_peak), orc, orc.setdata(db.cpu().numpy().astype(np.float64)))
        assert r.fmax_x.shape == (C,) and len(r.fpitch_text) == C
        last = r
    check_state(p, orc)


@pytest.mark.parametrize("bpo", [3, 24])
def test_end_to_end_octave(bpo):
    """OctaveSpectrumAnalyzer -> HistPlot, 8 blocks per call: the oracle steps through every block."""
    torch = torch_()
    from friture_b200.octavespectrum import OctaveSpectrumAnalyzer
    from friture_b200.plotcurves import HistPlot
    C = 3
    an = OctaveSpectrumAnalyzer(C, bandsperoctave=bpo, response_time=0.125)
    p = HistPlot(C, an)
    orc = PlotCurvesOracle(-80, -20)
    rng = np.random.default_rng(bpo)
    for i in range(3):
        x = torch.from_numpy((rng.standard_normal((C, 8 * 512)) * 0.1 ** i).astype(np.float32)).cuda()
        db = an.process(x, block=512)
        r = p.push(db)
        check((r.y, r.z, r.peak, r.z_peak), orc, step_oracle(orc, db.cpu().numpy()))
    check_state(p, orc)
