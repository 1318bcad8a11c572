"""The spectrum widget's reductions and the spectrogram display kernel at every setting the widgets
offer.

``frt_spectrum_reduce`` (``csrc/reduce.cu``, behind ``friture_b200.spectrum.SpectrumAnalyzer``)
smooths the tick's power frames into the carried state (the widget's ``dispbuffers1``), then forms
dB + weighting, the peak and the harmonic-product pitch (friture/spectrum.py:125-222).  It is fed
float32 power arrays made here, so it is judged apart from the STFT, at all ten FFT sizes x five
response times x four weightings, for as many frames as the smoothing needs to reach steady state
(3 / alpha).  The float64 reference smooths the same float32 values with the oracle's block form.

Bounds:
- carried state: within STATE_TOL of its peak, after every tick, every channel;
- dB: ``parity.assert_logpower_parity`` on every bin, after the float32 weight table is taken off;
- peak and pitch: each index points at a near-maximum of the float64 reference (NEAR_DB, NEAR_HPS),
  and exact ties go to the first index, as ``numpy.argmax`` does.

``frt_display_columns`` (behind ``friture_b200.display.SpectrogramDisplay``) is compared with the
float64 chain of friture/spectrogram.py:161-173: scaling, ``np.interp`` onto the screen rows, the
online linear time resampler and the colour look-up.  Every pixel must be the LUT entry of a value
within PIX_TOL of the oracle's.

The CPU tests (no mark) check that these bounds catch plausible bugs: float32 smoothing with a
rounded 1 - alpha, a float32 harmonic product, and two display bugs."""
import os
import sys
from ctypes import c_float
from fractions import Fraction

import numpy as np
import pytest

from oracle import friture_oracle as fo

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from parity import TOL, assert_logpower_parity  # noqa: E402

FS = 48000
FFT_SIZES = [2 ** k for k in range(5, 15)]           # 32 .. 16384, the widget's choices
RESPONSE_TIMES = [0.025, 0.125, 0.3, 1.0, 5.0]
WEIGHTINGS = [0, 1, 2, 3]                             # none, A, B, C
MAX_FRAMES = 8192                                     # frames per call the ABI accepts
TICK_CYCLE = [1, 0, 7, 64, MAX_FRAMES]                # frames per tick, repeated
FRAME_CAP = 90000                                     # above 3 / alpha at N = 32, T = 5 s

STATE_TOL = 1e-5     # carried smoothed power, relative to the channel's peak
NEAR_DB = TOL        # peak: ref_db[i] >= max(ref_db) - NEAR_DB * max(|ref_db|, 1)
NEAR_HPS = 1e-4      # pitch: hps[p] >= (1 - NEAR_HPS) * max(hps)
PIX_TOL = 1e-5       # display: pixel = lut[int(v' * 255)] with |v' - v| <= PIX_TOL


# --------------------------------------------------------------------------- spectrum references
def widget_alpha(fft_size, response_time):
    """SpectrumAnalyzer.setresponsetime (friture/spectrum.py:196-218), same operation order."""
    n = response_time * FS / (fft_size * (1. - 0.75))
    return 1. - (1. - 0.65) ** (1. / (n + 1))


def weight_table(fft_size, weighting):
    """The float64 weighting of friture/audioproc.py:83-96 (zeros for none)."""
    freq = np.linspace(0, FS // 2, fft_size // 2 + 1)
    A, B, C = fo.weighting_tables(freq)
    return [np.zeros_like(freq), A, B, C][weighting]


def weight_table_f32(fft_size, weighting):
    """The float32 table SpectrumAnalyzer hands the kernel."""
    from friture_b200.weighting import abc_weighting
    freq = np.linspace(0, FS // 2, fft_size // 2 + 1)
    A, B, C = abc_weighting(freq, eps=1e-50)
    return np.asarray([0. * A, A, B, C][weighting], dtype=np.float32)


class WidgetModel:
    """Spectrum_Widget.handle_new_data's numeric part and its setters (friture/spectrum.py:125-282)
    for C channels, on given power frames.  A tick without frames is skipped, as the widget does
    (spectrum.py:140)."""

    def __init__(self, n_channels, fft_size, response_time, weighting=0):
        self.C = n_channels
        self.response_time = response_time
        self.weighting = weighting
        self.setfftsize(fft_size)

    def setfftsize(self, fft_size):
        self.fft_size = fft_size
        self.hop = int(fft_size * (1. - 0.75))
        self.freq = np.linspace(0, FS // 2, fft_size // 2 + 1)
        self.disp = np.zeros((self.C, fft_size // 2 + 1))     # update_display_buffers
        self.setweighting(self.weighting)
        self.setresponsetime(self.response_time)

    def setresponsetime(self, response_time):
        self.response_time = response_time
        self.alpha = widget_alpha(self.fft_size, response_time)
        self.kernel = fo.smoothing_kernel(self.alpha, 2 * 4096)

    def setweighting(self, weighting):
        self.weighting = weighting
        self.w = weight_table(self.fft_size, weighting)

    def tick(self, power):
        """power [C, F, bins] (float64).  Returns False for a skipped tick."""
        if power.shape[1] == 0:
            return False
        for c in range(self.C):
            self.disp[c] = fo.exp_smoothed_value_2d(self.kernel, self.alpha, power[c].T, self.disp[c])
        return True

    def db(self, c):
        return fo.log_spectrogram(self.disp[c]) + self.w

    def hps(self, c):
        return fo.harmonic_product_spectrum(self.disp[c])


def tick_sizes(total):
    """TICK_CYCLE repeated until `total` frames, the last tick cut short."""
    out, done, k = [], 0, 0
    while done < total:
        m = min(TICK_CYCLE[k % len(TICK_CYCLE)], total - done)
        out.append(m)
        done += m
        k += 1
    return out


def case_frames(fft_size, response_time):
    return min(int(np.ceil(3. / widget_alpha(fft_size, response_time))), FRAME_CAP)


def channel_envelopes(n_channels, nbins):
    """Mean power per bin, about 100 dB from the strongest to the weakest bin: a tilt whose top sits
    at a different bin in each channel, channels 40 dB apart in level."""
    u = np.arange(nbins) / (nbins - 1)
    env = []
    for c in range(n_channels):
        top = (0.1 + 0.37 * c) % 1.0
        env.append(1e-2 * 10.0 ** (-4 * c) * 10.0 ** (-10.0 * np.abs(u - top) / max(top, 1 - top)))
    return np.stack(env)


def stationary_frames(rng, env, n_frames):
    """[C, F, bins] float32: the envelope times exponential (chi-squared, 2 dof) fluctuations, the
    statistics of |X|^2 of noise."""
    return (env[:, None, :] * rng.exponential(size=(env.shape[0], n_frames, env.shape[1]))).astype(np.float32)


def state_ratio(got, ref):
    """max|got - ref| over STATE_TOL x peak (inf when a zero state is not reproduced exactly)."""
    err = float(np.max(np.abs(np.asarray(got, np.float64) - ref)))
    peak = float(np.max(np.abs(ref)))
    if peak == 0.0:
        return 0.0 if err == 0.0 else np.inf
    return err / (STATE_TOL * peak)


def pitch_near_max(hps, p):
    return hps[p] >= (1. - NEAR_HPS) * np.max(hps)


def peak_near_max(ref_db, i):
    return ref_db[i] >= np.max(ref_db) - NEAR_DB * max(float(np.max(np.abs(ref_db))), 1.0)


def check_outputs(label, model, w32, disp, db, imax, ipitch):
    """Carried state, dB, peak and pitch of every channel against the model after a tick.
    Returns the worst state ratio."""
    worst = 0.0
    for c in range(model.C):
        lab = "%s ch %d" % (label, c)
        r = state_ratio(disp[c], model.disp[c])
        worst = max(worst, r)
        assert r <= 1.0, "%s: state error %.3g of its peak (bound %g)" % (lab, r * STATE_TOL, STATE_TOL)
        assert_logpower_parity(db[c].astype(np.float64) - w32, fo.log_spectrogram(model.disp[c]),
                               min_frac=0.0, strict=True)
        ref_db, hps = model.db(c), model.hps(c)
        assert peak_near_max(ref_db, int(imax[c])), (lab, int(imax[c]), int(np.argmax(ref_db)))
        assert pitch_near_max(hps, int(ipitch[c])), (lab, int(ipitch[c]), int(np.argmax(hps)))
    return worst


def harmonic_signal(fft_size, seed=1):
    """A 220 Hz tone with two harmonics plus noise, ten frames long."""
    rng = np.random.default_rng(seed)
    hop = fft_size // 4
    t = np.arange(fft_size + 9 * hop) / float(FS)
    return sum(0.3 / h * np.sin(2 * np.pi * 220.0 * h * t) for h in (1, 2, 3)) + 0.05 * rng.standard_normal(len(t))


QUIET_SIZES = [1024, 2048, 8192]
QUIET_SCALES = [1.0, 1e-3, 1e-5, 3e-6, 1e-6, 0.0]


def quiet_power(fft_size):
    """[len(QUIET_SCALES), 10, bins] float32 power of the harmonic signal at each scale."""
    x = harmonic_signal(fft_size)
    out = []
    for s in QUIET_SCALES:
        xs = (x * s).astype(np.float32).astype(np.float64)
        out.append(fo.stft_power_batch(xs[None], fft_size, fft_size // 4)[0])
    return np.stack(out).astype(np.float32)


# --------------------------------------------------------------------------- float32 replicas
def replica_smooth(power, s, alpha, form):
    """One tick of the kernel's smoothing, restated in numpy for one float32 arithmetic form:
    'rounded' s = fmaf(alpha, x, (1 - alpha) * s) with 1 - alpha rounded to float32, 'complement'
    s = fmaf(alpha, x - s, s), 'double' s + alpha (x - s) in float64, rounded once per tick."""
    a32 = np.float32(alpha)
    if form == "double":
        s64 = s.astype(np.float64)
        for f in range(power.shape[1]):
            s64 = s64 + float(a32) * (power[:, f].astype(np.float64) - s64)
        return s64.astype(np.float32)
    om = np.float32(1.0) - a32
    for f in range(power.shape[1]):
        x = power[:, f]
        if form == "rounded":
            s = (float(a32) * x.astype(np.float64) + (om * s).astype(np.float64)).astype(np.float32)
        else:
            s = (float(a32) * (x - s).astype(np.float64) + s.astype(np.float64)).astype(np.float32)
    return s


def replica_worst_state(fft_size, response_time, form):
    """Worst state ratio of a replica over the same input and ticks as test_reduce_grid."""
    nb = fft_size // 2 + 1
    rng = np.random.default_rng([fft_size, int(response_time * 1000)])
    env = channel_envelopes(2, nb)
    model = WidgetModel(2, fft_size, response_time)
    s = np.zeros((2, nb), dtype=np.float32)
    worst = 0.0
    for F in tick_sizes(case_frames(fft_size, response_time)):
        p = stationary_frames(rng, env, F)
        model.tick(p.astype(np.float64))
        s = replica_smooth(p, s, model.alpha, form)
        worst = max(worst, max(state_ratio(s[c], model.disp[c]) for c in range(2)))
    return worst


# --------------------------------------------------------------------------- CPU: references, bounds
@pytest.mark.parametrize("fft_size", FFT_SIZES)
def test_weight_tables_match_oracle(fft_size):
    """The float32 tables the analyzer passes are the oracle's A/B/C weighting rounded to float32."""
    for wi in WEIGHTINGS:
        ref = weight_table(fft_size, wi)
        got = weight_table_f32(fft_size, wi).astype(np.float64)
        assert np.all(np.abs(got - ref) <= np.spacing(np.abs(ref).astype(np.float32))), wi


def test_tick_schedule_reaches_steady_state():
    """Every case runs 3 / alpha frames uncapped; the longest is N = 32, T = 5 s."""
    worst = max(3. / widget_alpha(N, T) for N in FFT_SIZES for T in RESPONSE_TIMES)
    assert 80000 < worst < FRAME_CAP
    assert sum(tick_sizes(20000)) == 20000 and MAX_FRAMES in tick_sizes(20000)
    assert tick_sizes(6)[:2] == [1, 0]


@pytest.mark.parametrize("fft_size,response_time", [(32, 0.125), (256, 1.0)])
def test_state_bound_catches_rounded_complement(fft_size, response_time):
    """float32 smoothing with 1 - alpha rounded to float32 drifts past STATE_TOL; the complement
    form and the per-tick double accumulation the kernel uses stay inside it."""
    rounded = replica_worst_state(fft_size, response_time, "rounded")
    complement = replica_worst_state(fft_size, response_time, "complement")
    double = replica_worst_state(fft_size, response_time, "double")
    print("N=%d T=%g state ratio: rounded %.2f complement %.3f double %.4f"
          % (fft_size, response_time, rounded, complement, double))
    assert rounded > 1.0
    assert complement < 0.5
    assert double < 0.05


@pytest.mark.parametrize("fft_size", QUIET_SIZES)
def test_quiet_cases_have_clear_winners_and_catch_float32_products(fft_size):
    """The harmonic signal's peak and pitch are clear winners at every scale, so the GPU test can
    ask for the exact index; a float32 harmonic product underflows at scale 1e-6 and fails the
    pitch check."""
    power = quiet_power(fft_size)
    alpha = widget_alpha(fft_size, 0.125)
    for j, scale in enumerate(QUIET_SCALES[:-1]):
        model = WidgetModel(1, fft_size, 0.125)
        model.tick(power[j:j + 1].astype(np.float64))
        hps = np.sort(model.hps(0))
        ref_db = np.sort(model.db(0))
        assert hps[-2] < (1. - 10 * NEAR_HPS) * hps[-1], scale
        assert ref_db[-1] - ref_db[-2] > 10 * NEAR_DB * np.max(np.abs(ref_db)), scale
        if scale == 1e-6:
            sp32 = replica_smooth(power[j:j + 1], np.zeros((1, power.shape[2]), np.float32), alpha,
                                 "double")[0]
            h = sp32.shape[0] // 3
            prod32 = sp32[:h] * sp32[::2][:h] * sp32[::3][:h]
            assert prod32.dtype == np.float32
            assert not pitch_near_max(model.hps(0), int(np.argmax(prod32)))


# --------------------------------------------------------------------------- GPU: frt_spectrum_reduce
def padded_power(power, pad_f=3, pad_c=5):
    """[C, F, bins] -> NaN-padded device buffer with stride_f = bins + pad_f and
    stride_c = F * stride_f + pad_c.  Returns (buffer, stride_c, stride_f)."""
    import torch
    C, F, nb = power.shape
    sf = nb + pad_f
    sc = F * sf + pad_c
    buf = np.full((C, sc), np.nan, dtype=np.float32)
    buf[:, :F * sf].reshape(C, F, sf)[:, :, :nb] = power
    return torch.from_numpy(buf).cuda(), sc, sf


class ReduceBuffers:
    def __init__(self, C, nb, w32):
        import torch
        self.disp = torch.zeros((C, nb), dtype=torch.float32, device="cuda")
        self.db = torch.empty((C, nb), dtype=torch.float32, device="cuda")
        self.imax = torch.empty(C, dtype=torch.int32, device="cuda")
        self.ipitch = torch.empty(C, dtype=torch.int32, device="cuda")
        self.w = None if w32 is None else torch.from_numpy(w32).cuda()

    def run(self, h, power, alpha):
        """One call over power [C, F, bins] (host float32); returns the outputs on the host."""
        from friture_b200 import _lib
        C, F, nb = power.shape
        buf, sc, sf = padded_power(power) if F else (None, 0, nb)
        h.call("frt_spectrum_reduce", _lib._ptr(buf), sc, sf, C, F, nb, c_float(alpha),
               _lib._ptr(self.disp), _lib._ptr(self.w), _lib._ptr(self.db), _lib._ptr(self.imax),
               _lib._ptr(self.ipitch), _lib.current_stream_ptr())
        return (self.disp.cpu().numpy(), self.db.cpu().numpy(), self.imax.cpu().numpy(),
                self.ipitch.cpu().numpy())


@pytest.mark.gpu
@pytest.mark.parametrize("weighting", WEIGHTINGS)
@pytest.mark.parametrize("response_time", RESPONSE_TIMES)
@pytest.mark.parametrize("fft_size", FFT_SIZES)
def test_reduce_grid(fft_size, response_time, weighting):
    """Two channels of stationary power for 3 / alpha frames in ticks of 1, 0, 7, 64 and 8192
    frames, rows padded with NaN; every output checked after every tick."""
    from friture_b200 import _lib
    h = _lib.default_handle()
    nb = fft_size // 2 + 1
    rng = np.random.default_rng([fft_size, int(response_time * 1000)])
    env = channel_envelopes(2, nb)
    model = WidgetModel(2, fft_size, response_time, weighting)
    w32 = weight_table_f32(fft_size, weighting)
    bufs = ReduceBuffers(2, nb, w32 if weighting else None)
    sizes = tick_sizes(case_frames(fft_size, response_time))
    worst = 0.0
    for t, F in enumerate(sizes):
        p = stationary_frames(rng, env, F)
        model.tick(p.astype(np.float64))
        out = bufs.run(h, p, model.alpha)
        label = "N=%d T=%g w=%d tick %d (%d frames)" % (fft_size, response_time, weighting, t, F)
        worst = max(worst, check_outputs(label, model, w32 if weighting else 0.0, *out))
    print("N=%d T=%g w=%d: %d frames in %d ticks, worst state ratio %.4f"
          % (fft_size, response_time, weighting, sum(sizes), len(sizes), worst))


@pytest.mark.gpu
@pytest.mark.parametrize("fft_size", [32, 1024, 16384])
@pytest.mark.parametrize("many", [False, True])
def test_reduce_channels_and_layout(fft_size, many):
    """2 * SM + 5 channels (every CTA slot reused) or one, levels 70 dB apart, NaN-padded rows.
    Each channel carries a peak 20 dB above its floor at its own bin, so a channel mix-up moves
    the peak index."""
    from friture_b200 import _lib
    h = _lib.default_handle()
    C = 2 * h.sm_count + 5 if many else 1
    nb = fft_size // 2 + 1
    rng = np.random.default_rng([fft_size, C])
    env = np.stack([10.0 ** (-(c % 8)) * (0.01 + np.zeros(nb)) for c in range(C)])
    peak = (7 * np.arange(C) + 1) % nb
    env[np.arange(C), peak] *= 100.0
    w32 = weight_table_f32(fft_size, 0)
    model = WidgetModel(C, fft_size, 0.125)
    bufs = ReduceBuffers(C, nb, None)
    for t, F in enumerate([3, 0, 17, 1]):
        p = stationary_frames(rng, env, F)
        p[np.arange(C), :, peak] = env[np.arange(C), peak][:, None]    # no fluctuation at the peak
        model.tick(p.astype(np.float64))
        disp, db, imax, ipitch = bufs.run(h, p, model.alpha)
        check_outputs("C=%d N=%d tick %d" % (C, fft_size, t), model, w32, disp, db, imax, ipitch)
        assert np.array_equal(imax, peak), "C=%d N=%d tick %d" % (C, fft_size, t)


@pytest.mark.gpu
@pytest.mark.parametrize("fft_size", QUIET_SIZES)
def test_reduce_quiet_inputs(fft_size):
    """The harmonic signal at scales 1 .. 1e-6 and silence, one channel each, one tick: the pitch
    is the reference's index at every scale; silence gives -300 dB, peak 0 and pitch 0."""
    from friture_b200 import _lib
    h = _lib.default_handle()
    power = quiet_power(fft_size)
    C, F, nb = power.shape
    model = WidgetModel(C, fft_size, 0.125)
    model.tick(power.astype(np.float64))
    bufs = ReduceBuffers(C, nb, None)
    disp, db, imax, ipitch = bufs.run(h, power, model.alpha)
    for c, scale in enumerate(QUIET_SCALES):
        label = "N=%d scale %g" % (fft_size, scale)
        if scale == 0.0:
            assert not np.any(disp[c]), label
            assert np.all(np.abs(db[c] + 300.0) < 300.0 * TOL), label
            assert imax[c] == 0 and ipitch[c] == 0, label
            continue
        assert state_ratio(disp[c], model.disp[c]) <= 1.0, label
        assert_logpower_parity(db[c], model.db(c), min_frac=0.0, strict=True)
        assert int(ipitch[c]) == int(np.argmax(model.hps(c))), (label, int(ipitch[c]))
        assert int(imax[c]) == int(np.argmax(model.db(c))), (label, int(imax[c]))


@pytest.mark.gpu
@pytest.mark.parametrize("weighting", [0, 1])
def test_reduce_exact_ties_pick_first_index(weighting):
    """Two equal peaks in far-apart bins (different warps) and two equal harmonic products: the
    first index wins both arg-maxes, as numpy.argmax does."""
    from friture_b200 import _lib
    h = _lib.default_handle()
    fft_size = 4096
    nb = fft_size // 2 + 1
    rng = np.random.default_rng(5)
    p = (1e-6 * rng.exponential(size=(1, 4, nb))).astype(np.float32)
    p[:, :, [40, 80, 120, 300, 600, 900]] = np.float32(0.25)     # HPS tie at k = 40 and k = 300
    model = WidgetModel(1, fft_size, 0.3, weighting)
    w32 = weight_table_f32(fft_size, weighting)
    if weighting:                                               # dB tie after weighting: equal w
        w32[[1500, 1900]] = w32[1500]
        model.w = w32.astype(np.float64)
        p[:, :, [1500, 1900]] = np.float32(100.0)
    model.tick(p.astype(np.float64))
    bufs = ReduceBuffers(1, nb, w32 if weighting else None)
    disp, db, imax, ipitch = bufs.run(h, p, model.alpha)
    ref_db = model.db(0)
    assert np.sum(ref_db == ref_db.max()) >= 2 and np.sum(model.hps(0) == model.hps(0).max()) == 2
    assert int(imax[0]) == int(np.argmax(ref_db)) == (1500 if weighting else 40)
    assert int(ipitch[0]) == int(np.argmax(model.hps(0))) == 40
    assert db[0, 1500] == db[0, 1900] if weighting else db[0, 40] == db[0, 900]


@pytest.mark.gpu
def test_reduce_rejected_arguments_leave_handle_usable():
    """nbins < 3, more than 8192 frames, alpha outside (0, 1] and NULL buffers raise
    FrtValueError; a valid call afterwards gives the same results as before them."""
    import torch
    from friture_b200 import _lib
    from friture_b200._lib import FrtValueError
    h = _lib.default_handle()
    nb, F = 129, 5
    rng = np.random.default_rng(9)
    p = stationary_frames(rng, channel_envelopes(2, nb), F)
    alpha = widget_alpha(256, 0.125)
    first = ReduceBuffers(2, nb, None).run(h, p, alpha)
    big = torch.zeros((1, MAX_FRAMES + 1, 3), device="cuda")
    b = ReduceBuffers(2, nb, None)
    buf, sc, sf = padded_power(p)
    ptr, cur = _lib._ptr, _lib.current_stream_ptr()

    def call(power, stride_c, stride_f, C, nf, nbins, a, disp=b.disp, db=b.db, im=b.imax, ip=b.ipitch):
        h.call("frt_spectrum_reduce", ptr(power), stride_c, stride_f, C, nf, nbins, c_float(a),
               ptr(disp), None, ptr(db), ptr(im), ptr(ip), cur)

    bad = [
        lambda: call(buf, sc, sf, 2, F, 2, alpha),
        lambda: call(big, (MAX_FRAMES + 1) * 3, 3, 1, MAX_FRAMES + 1, 3, alpha),
        lambda: call(buf, sc, sf, 2, F, nb, 0.0),
        lambda: call(buf, sc, sf, 2, F, nb, -0.5),
        lambda: call(buf, sc, sf, 2, F, nb, 1.5),
        lambda: call(buf, sc, sf, 2, F, nb, float("nan")),
        lambda: call(None, sc, sf, 2, F, nb, alpha),
        lambda: call(buf, sc, sf, 2, F, nb, alpha, disp=None),
        lambda: call(buf, sc, sf, 2, F, nb, alpha, db=None),
        lambda: call(buf, sc, sf, 2, F, nb, alpha, im=None),
        lambda: call(buf, sc, sf, 2, F, nb, alpha, ip=None),
    ]
    for k, f in enumerate(bad):
        with pytest.raises(FrtValueError):
            f()
        assert not torch.any(b.disp), k                  # nothing ran
    again = ReduceBuffers(2, nb, None).run(h, p, alpha)
    for x, y in zip(first, again):
        assert np.array_equal(x, y)
    call(big, (MAX_FRAMES + 1) * 3, 3, 1, MAX_FRAMES, 3, 1.0)   # 8192 frames are accepted


# --------------------------------------------------------------------------- GPU: SpectrumAnalyzer
E2E_SIZES = [32, 256, 1024, 8192, 16384]


def e2e_stream(fft_size, n_frames, C=3, seed=0):
    """[C, samples] float32 for n_frames frames: channel c is a tone with two harmonics at its own
    pitch and level, plus noise."""
    rng = np.random.default_rng([fft_size, seed])
    hop = fft_size // 4
    n = fft_size + (n_frames - 1) * hop
    t = np.arange(n) / float(FS)
    x = 0.02 * rng.standard_normal((C, n))
    for c in range(C):
        f0 = [220.0, 1375.0, 5050.0][c % 3] * (1 + 0.01 * c)
        x[c] += sum(0.3 / k * np.sin(2 * np.pi * f0 * k * t + c) for k in (1, 2, 3))
        x[c] *= 10.0 ** (-2 * c)
    return x.astype(np.float32)


def analyzer_indices(an, fmax, fpitch):
    return np.searchsorted(an.freq, fmax), np.where(fpitch <= 1e-20, 0, np.searchsorted(an.freq, fpitch))


def check_analyzer(label, an, model, db, fmax, fpitch, dbtol_floor=40.0):
    """The analyzer's state, dB, peak and pitch against the model, STFT included (floor-aware dB)."""
    import torch
    disp = an._disp.cpu().numpy()
    db = db.cpu().numpy().astype(np.float64)
    w32 = np.asarray(an.w, dtype=np.float32).astype(np.float64)
    imax, ipitch = analyzer_indices(an, fmax, fpitch)
    assert torch.is_tensor(an._disp)
    worst = 0.0
    for c in range(model.C):
        lab = "%s ch %d" % (label, c)
        r = state_ratio(disp[c], model.disp[c])
        worst = max(worst, r)
        assert r <= 1.0, "%s: state error %.3g of its peak" % (lab, r * STATE_TOL)
        assert_logpower_parity(db[c] - w32, fo.log_spectrogram(model.disp[c]), min_frac=0.0,
                               strict=False, floor_db=dbtol_floor)
        assert peak_near_max(model.db(c), int(imax[c])), lab
        assert pitch_near_max(model.hps(c), int(ipitch[c])), lab
    return worst


@pytest.mark.gpu
@pytest.mark.parametrize("response_time", [0.125, 5.0])
@pytest.mark.parametrize("fft_size", E2E_SIZES)
def test_analyzer_end_to_end(fft_size, response_time):
    """Three channels through the real STFT for 3 / alpha frames, in ticks of 1, 0, 7, 64 and 8192
    frames; a tick shorter than one frame leaves every output and the state as they were."""
    import torch
    from friture_b200.spectrum import SpectrumAnalyzer
    weighting = E2E_SIZES.index(fft_size) % 4
    an = SpectrumAnalyzer(3, fft_size=fft_size, response_time=response_time, weighting=weighting)
    model = WidgetModel(3, fft_size, response_time, weighting)
    assert an.alpha == model.alpha and an.hop == model.hop and np.array_equal(an.freq, model.freq)
    total = case_frames(fft_size, response_time)
    x = e2e_stream(fft_size, total)
    power = fo.stft_power_batch(x.astype(np.float64), fft_size, model.hop)    # [C, frames, bins]
    hop, pos, worst, last = model.hop, 0, 0.0, None
    for t, F in enumerate(tick_sizes(total)):
        label = "N=%d T=%g tick %d (%d frames)" % (fft_size, response_time, t, F)
        if F == 0:
            before = an._disp.clone()
            db, fmax, fpitch = an.process(torch.from_numpy(x[:, pos * hop:pos * hop + fft_size - 1].copy()).cuda())
            assert not model.tick(power[:, :0])
            assert torch.equal(an._disp, before), label
            if last is not None:
                assert torch.equal(db, last[0]) and np.array_equal(fmax, last[1]), label
                assert np.array_equal(fpitch, last[2]), label
            continue
        seg = x[:, pos * hop:(pos + F - 1) * hop + fft_size]
        db, fmax, fpitch = an.process(torch.from_numpy(np.ascontiguousarray(seg)).cuda())
        model.tick(power[:, pos:pos + F])
        pos += F
        worst = max(worst, check_analyzer(label, an, model, db, fmax, fpitch))
        last = (db.clone(), fmax.copy(), fpitch.copy())
    print("analyzer N=%d T=%g w=%d: %d frames, worst state ratio %.4f"
          % (fft_size, response_time, weighting, total, worst))


@pytest.mark.gpu
def test_analyzer_setters_follow_reference():
    """setresponsetime and setweighting keep the smoothed state and change alpha / the table;
    setfftsize restarts the state (friture/spectrum.py:196-282)."""
    import torch
    from friture_b200.spectrum import SpectrumAnalyzer
    an = SpectrumAnalyzer(3, fft_size=1024, response_time=0.125, weighting=0)
    model = WidgetModel(3, 1024, 0.125, 0)

    def run(n_ticks, seed):
        x = e2e_stream(model.fft_size, 20 * n_ticks, seed=seed)
        power = fo.stft_power_batch(x.astype(np.float64), model.fft_size, model.hop)
        for k in range(n_ticks):
            seg = x[:, 20 * k * model.hop:(20 * k + 19) * model.hop + model.fft_size]
            db, fmax, fpitch = an.process(torch.from_numpy(np.ascontiguousarray(seg)).cuda())
            model.tick(power[:, 20 * k:20 * k + 20])
            check_analyzer("N=%d T=%g w=%d tick %d" % (model.fft_size, model.response_time,
                                                       model.weighting, k), an, model, db, fmax, fpitch)

    run(3, 1)
    kept = an._disp.clone()
    an.setresponsetime(1.0)
    model.setresponsetime(1.0)
    assert an.alpha == model.alpha and torch.equal(an._disp, kept)
    run(2, 2)
    an.setweighting(2)
    model.setweighting(2)
    run(2, 3)
    an.setfftsize(2048)
    model.setfftsize(2048)
    assert an._disp is None and an.alpha == model.alpha and an.hop == model.hop
    run(2, 4)


# --------------------------------------------------------------------------- display references
DISPLAY_FFT = 2048
DISPLAY_TICKS = [5, 0, 1, 9, 37]
NEW_HEIGHT_AT = 3                         # set_screen(new height) before this tick
SPEC_MIN, SPEC_MAX = -140.0, 0.0
MINFREQ, MAXFREQ = 5.0, FS / 2            # below freq[1] (23.4 Hz) and at Nyquist
# (height, new height, width) over a 10 s time range: 1800 px draws ~1.9 columns per input column,
# 300 px ~0.32, so that some ticks draw none
GEOMETRIES = {"upsampling": (120, 97, 1800), "decimating": (77, 131, 300)}


def display_db(C, F, nb, tick, seed=0):
    """[C, F, bins] float32 dB columns, each channel its own pattern, spanning below SPEC_MIN and
    above SPEC_MAX so that both ends clip."""
    rng = np.random.default_rng([C, tick, seed])
    u = np.arange(nb) / (nb - 1)
    f = np.arange(F)[:, None]
    out = []
    for c in range(C):
        base = -60.0 - 90.0 * u + 40.0 * np.sin(2 * np.pi * (3 + 2 * c) * u + 0.3 * f + c)
        out.append(base + 8.0 * rng.standard_normal((F, nb)))
    return np.stack(out).astype(np.float32)


class DisplayOracle:
    """friture/spectrogram.py:161-173 per channel in float64: (dB + w - min) / (max - min),
    Frequency_Resampler (np.interp), Online_Linear_2D_resampler; values before clipping."""

    def __init__(self, C, scale, weighting, height, width):
        self.C = C
        self.scale = scale
        self.freq = np.linspace(0, FS // 2, DISPLAY_FFT // 2 + 1)
        self.w = weight_table(DISPLAY_FFT, weighting)
        self.sfft_rate = Fraction(FS, DISPLAY_FFT) / (Fraction(1) - Fraction(3, 4)) / 1000
        self.width = width
        self.set_height(height)

    def set_height(self, height):
        from friture_b200.display import screen_rows
        self.height = height
        self.xscaled, _, _ = screen_rows(self.freq, self.scale, MINFREQ, MAXFREQ, height)
        screen_rate = Fraction(self.width, 10 * 1000)
        self.res = [fo.OnlineLinear2DResamplerOracle(self.sfft_rate, screen_rate, height)
                    for _ in range(self.C)]

    def push(self, db):
        out = []
        for c in range(self.C):
            norm = (db[c].astype(np.float64).T + self.w[:, None] - SPEC_MIN) / (SPEC_MAX - SPEC_MIN)
            out.append(self.res[c].push(fo.frequency_resample(norm, self.freq, self.xscaled)))
        return np.stack(out)


def pixel_mismatch(px, v, lut):
    """Pixels that are not lut[int(v' * 255)] for any v' within PIX_TOL of clip(v, 0, 1)."""
    vc = np.clip(v, 0.0, 1.0)
    lo = (np.clip(vc - PIX_TOL, 0.0, 1.0) * 255).astype(np.intp)
    hi = (np.clip(vc + PIX_TOL, 0.0, 1.0) * 255).astype(np.intp)
    return ~((px == lut[lo]) | (px == lut[hi]))


def display_kernel_model(db, w32, i0, t, cols, a, old, bug=None):
    """display_kernel's per-pixel arithmetic in float64 on the host tables (row i0 / t, output
    column / weight).  bug='left bins' interpolates between bins i0-1 and i0; bug='old from
    channel 0' takes every channel's carried column from channel 0.  Returns (v, new old)."""
    S = (db.astype(np.float64) + w32 - SPEC_MIN) / (SPEC_MAX - SPEC_MIN)       # [C, F, bins]
    lo, hi = (np.maximum(i0 - 1, 0), i0) if bug == "left bins" else (i0, i0 + 1)
    rows = S[:, :, lo] * (1.0 - t) + S[:, :, hi] * t                          # [C, F, height]
    if bug == "old from channel 0":
        old = np.broadcast_to(old[:1], old.shape)
    prev = np.where((cols > 0)[None, :, None], rows[:, np.maximum(cols - 1, 0)], old[:, None, :])
    v = rows[:, cols] * (1.0 - a)[None, :, None] + prev * a[None, :, None]
    return v.transpose(0, 2, 1), rows[:, -1]


def display_model_run(C, scale, weighting, geometry, bug=None):
    """The tick sequence through the host tables and display_kernel_model, against the oracle.
    Yields (tick, oracle v, model v) per tick with frames."""
    from friture_b200.display import OnlineResamplerIndex, screen_rows
    height, new_height, width = GEOMETRIES[geometry]
    orc = DisplayOracle(C, scale, weighting, height, width)
    w32 = weight_table_f32(DISPLAY_FFT, weighting).astype(np.float64)
    index = OnlineResamplerIndex()
    index.set_ratio(orc.sfft_rate, Fraction(width, 10 * 1000))
    nb = DISPLAY_FFT // 2 + 1
    old = np.zeros((C, height))
    for k, F in enumerate(DISPLAY_TICKS):
        if k == NEW_HEIGHT_AT:
            orc.set_height(new_height)
            index.reset()
            height, old = new_height, np.zeros((C, new_height))
        _, i0, t = screen_rows(orc.freq, scale, MINFREQ, MAXFREQ, height)
        db = display_db(C, F, nb, k)
        cols, a = index.push(F)
        if F == 0:
            continue
        v_ref = orc.push(db)
        v, old = display_kernel_model(db, w32, i0, t, cols, a, old, bug)
        yield k, v_ref, v


SCALE_IDS = [0, 1, 2, 3, 4]


@pytest.mark.parametrize("geometry", sorted(GEOMETRIES))
@pytest.mark.parametrize("scale_id", SCALE_IDS)
def test_display_model_matches_oracle_and_bugs_fail(scale_id, geometry):
    """The host tables with the kernel's arithmetic meet the pixel check; interpolating between
    bins i0-1 and i0 fails it; the channels' pixels differ, so a channel mix-up would show."""
    from friture_b200.display import SCALES, load_lut
    lut = load_lut()
    scale = SCALES[scale_id]
    n_out = 0
    for k, v_ref, v in display_model_run(3, scale, 1, geometry):
        assert v.shape == v_ref.shape
        n_out += v.shape[2]
        assert not pixel_mismatch(lut[(np.clip(v, 0, 1) * 255).astype(np.intp)], v_ref, lut).any(), k
        px = fo.color_transform(lut, v_ref)
        if v.shape[2]:
            assert not np.array_equal(px[0], px[1]) and not np.array_equal(px[1], px[2])
    assert n_out > 0
    bad = sum(int(pixel_mismatch(lut[(np.clip(v, 0, 1) * 255).astype(np.intp)], v_ref, lut).sum())
              for _, v_ref, v in display_model_run(3, scale, 0, geometry, bug="left bins"))
    assert bad > 0


@pytest.mark.parametrize("geometry", sorted(GEOMETRIES))
def test_display_check_catches_old_column_of_channel_0(geometry):
    from friture_b200.display import SCALES, load_lut
    lut = load_lut()
    bad = 0
    for _, v_ref, v in display_model_run(3, SCALES[2], 0, geometry, bug="old from channel 0"):
        bad += int(pixel_mismatch(lut[(np.clip(v, 0, 1) * 255).astype(np.intp)], v_ref, lut).sum())
    assert bad > 0


def test_display_geometries_draw_and_skip():
    """The upsampling geometry draws more columns than it reads; the decimating one has ticks that
    draw nothing."""
    from friture_b200.display import SCALES
    counts = {}
    for g in GEOMETRIES:
        counts[g] = [(k, v.shape[2]) for k, _, v in display_model_run(1, SCALES[0], 0, g)]
    up = counts["upsampling"]
    assert sum(n for _, n in up) > sum(DISPLAY_TICKS)
    assert any(n == 0 for _, n in counts["decimating"])


# --------------------------------------------------------------------------- GPU: display
@pytest.mark.gpu
@pytest.mark.parametrize("C", [3, 1])
@pytest.mark.parametrize("weighting", [0, 1])
@pytest.mark.parametrize("geometry", sorted(GEOMETRIES))
@pytest.mark.parametrize("scale_id", SCALE_IDS)
def test_display_vs_oracle(scale_id, geometry, weighting, C):
    """Every pixel of every tick against the float64 chain; the height changes before the fourth
    tick, where both restart the time resampler."""
    import torch
    from friture_b200.display import SCALES, SpectrogramDisplay, load_lut
    lut = load_lut()
    scale = SCALES[scale_id]
    height, new_height, width = GEOMETRIES[geometry]
    disp = SpectrogramDisplay(C, fft_size=DISPLAY_FFT, freqscale=scale, minfreq=MINFREQ,
                              maxfreq=MAXFREQ, spec_min=SPEC_MIN, spec_max=SPEC_MAX,
                              weighting=weighting, height=height, width=width, timerange_s=10.)
    orc = DisplayOracle(C, scale, weighting, height, width)
    nb = DISPLAY_FFT // 2 + 1
    for k, F in enumerate(DISPLAY_TICKS):
        if k == NEW_HEIGHT_AT:
            disp.set_screen(new_height, width)
            orc.set_height(new_height)
        db = display_db(C, F, nb, k)
        px = disp.push(torch.from_numpy(db).cuda()).cpu().numpy().view(np.uint32)
        if F == 0:
            assert px.shape[2] == 0
            continue
        v = orc.push(db)
        assert px.shape == v.shape, (k, px.shape, v.shape)
        bad = pixel_mismatch(px, v, lut)
        assert not bad.any(), "tick %d: %d wrong pixels, first at %s" % (k, bad.sum(), np.argwhere(bad)[0])


@pytest.mark.gpu
def test_display_abi_strided_columns():
    """frt_display_columns on NaN-padded columns (stride_f > bins, stride_c > F * stride_f), two
    ticks: pixels against the float64 chain and the carried column against the last input column."""
    import torch
    from friture_b200 import _lib
    from friture_b200.display import SCALES, OnlineResamplerIndex, load_lut, screen_rows
    h = _lib.default_handle()
    lut = load_lut()
    C, height, width = 2, 90, 1800
    orc = DisplayOracle(C, SCALES[3], 1, height, width)
    _, i0, t = screen_rows(orc.freq, SCALES[3], MINFREQ, MAXFREQ, height)
    index = OnlineResamplerIndex()
    index.set_ratio(orc.sfft_rate, Fraction(width, 10 * 1000))
    w_d = torch.from_numpy(weight_table_f32(DISPLAY_FFT, 1)).cuda()
    i0_d, t_d = torch.from_numpy(i0).cuda(), torch.from_numpy(t.astype(np.float32)).cuda()
    lut_d = torch.from_numpy(lut.view(np.int32)).cuda()
    old = torch.zeros((C, height), dtype=torch.float32, device="cuda")
    nb = DISPLAY_FFT // 2 + 1
    for k, F in enumerate([6, 11]):
        db = display_db(C, F, nb, k, seed=7)
        buf, sc, sf = padded_power(db, pad_f=5, pad_c=9)
        cols, a = index.push(F)
        n_out = len(cols)
        px = torch.empty((C, height, n_out), dtype=torch.int32, device="cuda")
        cols_d = torch.from_numpy(cols).cuda()
        a_d = torch.from_numpy(a.astype(np.float32)).cuda()
        h.call("frt_display_columns", _lib._ptr(buf), sc, sf, C, F, nb, _lib._ptr(w_d),
               c_float(SPEC_MIN), c_float(SPEC_MAX), _lib._ptr(i0_d), _lib._ptr(t_d), height,
               _lib._ptr(cols_d), _lib._ptr(a_d), n_out, _lib._ptr(old), _lib._ptr(lut_d),
               _lib._ptr(px), _lib.current_stream_ptr())
        v = orc.push(db)
        assert n_out > 0 and px.shape == v.shape
        assert not pixel_mismatch(px.cpu().numpy().view(np.uint32), v, lut).any(), k
        carried = old.cpu().numpy().astype(np.float64)
        for c in range(C):
            assert np.max(np.abs(carried[c] - orc.res[c].old_data)) <= PIX_TOL, (k, c)
