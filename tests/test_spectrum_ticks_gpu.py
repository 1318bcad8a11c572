"""GPU: ``SpectrumAnalyzer.process_ticks`` and ``SpectrumPlot.push_ticks`` -- every tick of a call in
one STFT launch and one reduction call (``frt_spectrum_reduce_ticks`` / ``_dual_ticks``,
``csrc/reduce.cu``), and every tick's curves stepped in one ``frt_plot_curves`` launch.

The main check is bit identity: R ticks in one call give the same dB rows, peak and pitch
frequencies, and carried states (``_disp``, ``_disp2``) as R ``process`` calls on the tick slices
``x[..., r*g*hop : (r+1)*g*hop + N - hop]``, and ``push_ticks`` the same curves and float64 peak state
as R ``push`` calls.  The rows are also held to the oracle bounds of ``test_widget_reductions_gpu``
and ``test_spectrum_dual_gpu``, and to the unmodified reference's dual / single ticks of
``tests/golden/spectrum_dual.npz``."""
import os
import sys
from ctypes import c_float

import numpy as np
import pytest
import torch

from friture_b200 import _lib
from friture_b200.plotcurves import SpectrumPlot
from friture_b200.spectrum import SpectrumAnalyzer, SpectrumTicks

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_spectrum_dual_gpu import (  # noqa: E402
    check_dual_analyzer, check_single_analyzer, dual_failures, dual_oracles, fixture_cases, pair_curves,
    pair_frames, segment, tick_oracles)
from test_stream_order_gpu import WAYS, check, side, signal  # noqa: E402,F401
from parity import assert_logpower_parity  # noqa: E402
from test_widget_reductions_gpu import (  # noqa: E402
    FFT_SIZES, WidgetModel, analyzer_indices, channel_envelopes, check_analyzer, e2e_stream, peak_near_max,
    pitch_near_max, weight_table)

pytestmark = pytest.mark.gpu

BUDGET = 256 << 20      # the library's state-row budget per group of ticks (reduce.cu)


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def stream(C, dual, T, seed):
    """[C, T] or [C, 2, T] noise with a tone, each channel at its own level (60 dB span)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    shape = (C, 2, T) if dual else (C, T)
    x = torch.randn(shape, generator=g, device="cuda") * 0.02
    t = torch.arange(T, device="cuda", dtype=torch.float32) / 48000.0
    f0 = 220.0 * (1.0 + torch.arange(C, device="cuda", dtype=torch.float32) % 17)
    tone = 0.3 * torch.sin(2 * np.pi * f0[:, None] * t[None, :])
    if dual:
        x[:, 0] += tone
        x[:, 1] += 0.5 * tone
    else:
        x += tone
    level = 10.0 ** (-3.0 * (torch.arange(C, device="cuda", dtype=torch.float32) % 3))
    return (x * level.view((C,) + (1,) * (x.dim() - 1))).contiguous()


def tick_slice(x, an, g, r):
    return x[..., r * g * an.hop:(r + 1) * g * an.hop + an.fft_size - an.hop]


def bits(t):
    return t.contiguous().view(torch.int32)


def same_state(a, b, label):
    for name in ("_disp", "_disp2"):
        sa, sb = getattr(a, name), getattr(b, name)
        assert (sa is None) == (sb is None), (label, name)
        if sa is not None:
            assert torch.equal(bits(sa), bits(sb)), (label, name)


def per_tick(an, x, g, R):
    """R process calls on the tick slices: dB [C, R, bins], fmax and fpitch [R, C]."""
    out = [an.process(tick_slice(x, an, g, r)) for r in range(R)]
    return (torch.stack([o[0] for o in out], 1), np.stack([o[1] for o in out]),
            np.stack([o[2] for o in out]))


def same_as_per_tick(a, b, x, g, R, label):
    """a.process_ticks(x) against R b.process calls, rows and states bit for bit."""
    got = a.process_ticks(x, frames_per_tick=g)
    assert isinstance(got, SpectrumTicks) and got.db.shape == (a.n_channels, R, a.fft_size // 2 + 1), label
    db, fmax, fpitch = per_tick(b, x, g, R)
    assert torch.equal(bits(got.db), bits(db)), label
    assert got.fmax_hz.dtype == np.float64 and got.fmax_hz.shape == (R, a.n_channels), label
    assert np.array_equal(got.fmax_hz, fmax) and np.array_equal(got.fpitch_hz, fpitch), label
    same_state(a, b, label)
    return got


def pair(C, N, T, weighting, dual):
    return [SpectrumAnalyzer(C, fft_size=N, response_time=T, weighting=weighting, dual_channels=dual)
            for _ in range(2)]


def grid_cases():
    """Every FFT size; response times 0.025, 1 and 5 s; weighting none and A; single and dual; C in
    {1, 3, 2 SMs + 5}; R in {1, 7, 64}; frames_per_tick in {1, 2, 16} -- each value several times."""
    cases = []
    for i, N in enumerate(FFT_SIZES):
        for j in range(2):
            k = 2 * i + j
            cases.append((N, [0.025, 1.0, 5.0][k % 3], k % 2, (k // 2) % 2 == 1, ["1", "3", "big"][(i + 2 * j) % 3],
                          [1, 7, 64][(k // 3) % 3], [1, 2, 16][(k + 2 * i) % 3]))
    return cases


@pytest.mark.parametrize("N,T,weighting,dual,C,R,g", grid_cases())
def test_ticks_are_process_calls_bit_for_bit(N, T, weighting, dual, C, R, g):
    C = {"1": 1, "3": 3, "big": 2 * sms() + 5}[C]
    if N >= 8192 and C > 3:
        R = min(R, 7)      # the per-tick route's inputs stay below a gigabyte
    a, b = pair(C, N, T, weighting, dual)
    lead = stream(C, dual, N + 2 * a.hop, 1)       # a non-zero state to start from
    a.process(lead)
    b.process(lead)
    x = stream(C, dual, R * g * a.hop + N - a.hop, 2)
    same_as_per_tick(a, b, x, g, R, (N, T, weighting, dual, C, R, g))


@pytest.mark.parametrize("dual", [False, True])
def test_ticks_in_several_workspace_groups(dual):
    """Enough channel-bins per tick that the call runs in groups of ticks."""
    C, N, R = 2 * sms() + 5, 16384, 40
    per_tick = (2 if dual else 1) * C * (N // 2 + 1) * 4
    assert BUDGET // per_tick < R
    a, b = pair(C, N, 1.0, 1, dual)
    x = stream(C, dual, R * a.hop + N - a.hop, 3)
    same_as_per_tick(a, b, x, 1, R, "groups")


@pytest.mark.parametrize("dual", [False, True])
@pytest.mark.parametrize("N", [32, 1024, 8192])
def test_one_call_is_any_chunking(N, dual):
    """70 ticks in one call, and in calls of 1, 5 and 64 ticks: the same bits."""
    C = 3
    a, b = pair(C, N, 0.3, 1, dual)
    g = a.default_frames_per_tick()
    x = stream(C, dual, 70 * g * a.hop + N - a.hop, 4)
    whole = a.process_ticks(x, want_db=True)
    rows, r0 = [], 0
    for n in (1, 5, 64):
        part = x[..., r0 * g * b.hop:(r0 + n) * g * b.hop + N - b.hop]
        rows.append(b.process_ticks(part))
        r0 += n
    assert torch.equal(bits(whole.db), bits(torch.cat([t.db for t in rows], 1)))
    assert np.array_equal(whole.fmax_hz, np.concatenate([t.fmax_hz for t in rows]))
    assert np.array_equal(whole.fpitch_hz, np.concatenate([t.fpitch_hz for t in rows]))
    same_state(a, b, "chunking")


def test_default_frames_per_tick_is_the_widgets_feed():
    """One tick per 512-sample buffer: 512 / hop frames at N <= 1024, one frame above."""
    for N in FFT_SIZES:
        a, b = pair(1, N, 0.125, 0, False)
        g = a.default_frames_per_tick()
        assert g == max(1, 512 // (N // 4))
        x = stream(1, False, 9 * g * a.hop + N - a.hop, 5)
        same_as_per_tick(a, b, x, g, 9, N)


def test_without_db():
    a, b = pair(3, 2048, 0.125, 1, False)
    x = stream(3, False, 12 * a.hop + 2048 - a.hop, 6)
    got = a.process_ticks(x, want_db=False)
    want = b.process_ticks(x)
    assert got.db is None
    assert np.array_equal(got.fmax_hz, want.fmax_hz) and np.array_equal(got.fpitch_hz, want.fpitch_hz)
    same_state(a, b, "no dB")


def test_no_whole_tick_does_nothing():
    a, b = pair(2, 1024, 0.125, 0, False)
    a.process(stream(2, False, 4096, 7))
    b.process(stream(2, False, 4096, 7))
    n = a.proc.handle.launch_count
    got = a.process_ticks(stream(2, False, 1023, 8))
    assert got.db.shape == (2, 0, 513) and got.fmax_hz.shape == (0, 2) and got.fpitch_hz.shape == (0, 2)
    assert a.proc.handle.launch_count == n
    same_state(a, b, "empty")


# --------------------------------------------------------------------------- edge cases
@pytest.mark.parametrize("dual", [False, True])
def test_silence(dual):
    a, b = pair(3, 512, 0.125, 1, dual)
    x = torch.zeros((3, 2, 20 * 128 + 384) if dual else (3, 20 * 128 + 384), device="cuda")
    got = same_as_per_tick(a, b, x, 4, 5, "silence")
    assert np.all(got.fpitch_hz == 1e-20)
    if dual:
        assert np.all(got.fmax_hz == 0.0) and torch.all(got.db == 0.0)


def reduce_per_tick(h, power, g, R, alpha, disp, weight=None):
    """R frt_spectrum_reduce calls, one per tick of g frames: dB [C, R, nb], indices [R, C] each."""
    C, _, nb = power.shape
    db = torch.empty((C, R, nb), device="cuda")
    imax = torch.empty((R, C), dtype=torch.int32, device="cuda")
    ipitch = torch.empty((R, C), dtype=torch.int32, device="cuda")
    for r in range(R):
        out = torch.empty((C, nb), device="cuda")
        h.call("frt_spectrum_reduce", _lib._ptr(power[:, r * g:].data_ptr()), power.stride(0), power.stride(1), C,
               g, nb, c_float(alpha), _lib._ptr(disp), _lib._ptr(weight), _lib._ptr(out), _lib._ptr(imax[r]),
               _lib._ptr(ipitch[r]), _lib.current_stream_ptr())
        db[:, r] = out
    return db, imax, ipitch


def test_exact_ties_go_to_the_first_bin():
    """Power equal at bins 10 and 20 above a flat floor: the dB tie goes to bin 10, as numpy.argmax
    does, in both routes; a flat row ties every harmonic product and its pitch is bin 0."""
    h = _lib.default_handle()
    C, g, R, nb = 3, 2, 6, 257
    power = torch.ones((C, g * R, nb), device="cuda")
    power[0, :, 10] = power[0, :, 20] = 5.0
    power[1, :, 40] = power[1, :, 41] = 3.0
    d_a, d_b = torch.zeros((C, nb), device="cuda"), torch.zeros((C, nb), device="cuda")
    db = torch.empty((C, R, nb), device="cuda")
    imax = torch.empty((R, C), dtype=torch.int32, device="cuda")
    ipitch = torch.empty((R, C), dtype=torch.int32, device="cuda")
    h.call("frt_spectrum_reduce_ticks", _lib._ptr(power), power.stride(0), power.stride(1), C, g, R, nb,
           c_float(0.3), _lib._ptr(d_a), None, _lib._ptr(db), _lib._ptr(imax), _lib._ptr(ipitch),
           _lib.current_stream_ptr())
    want = reduce_per_tick(h, power, g, R, 0.3, d_b)
    assert torch.equal(bits(db), bits(want[0])) and torch.equal(bits(d_a), bits(d_b))
    assert torch.equal(imax, want[1]) and torch.equal(ipitch, want[2])
    assert torch.all(imax[:, 0] == 10) and torch.all(imax[:, 1] == 40) and torch.all(imax[:, 2] == 0)
    assert torch.all(ipitch[:, 2] == 0)


def test_single_dual_toggles_between_calls():
    """dual -> single -> dual, and single ticks decaying the second state tick by tick."""
    C, N = 3, 1024
    a, b = pair(C, N, 0.3, 1, True)
    for t, dual in enumerate([True, False, True, False, False, True]):
        a.setdualchannels(dual)
        b.setdualchannels(dual)
        g = 1 + t % 3
        R = 3 + t
        x = stream(C, True, R * g * a.hop + N - a.hop, 20 + t)
        same_as_per_tick(a, b, x, g, R, ("toggle", t, dual))
    assert a._disp2 is not None


# --------------------------------------------------------------------------- oracle
@pytest.mark.parametrize("N,T", [(32, 5.0), (1024, 0.125), (8192, 1.0)])
def test_rows_follow_the_widget_oracle(N, T):
    """Single mode through the real STFT: every row against the widget restated in float64, ticked
    per tick, with check_analyzer's bounds (the dB floor-aware, peak and pitch at near-maxima); the
    carried state after the call within STATE_TOL."""
    from oracle import friture_oracle as fo
    C, weighting = 3, 1
    an = SpectrumAnalyzer(C, fft_size=N, response_time=T, weighting=weighting)
    model = WidgetModel(C, N, T, weighting)
    g = an.default_frames_per_tick()
    R = 48
    x = e2e_stream(N, R * g, C=C)
    power = fo.stft_power_batch(x.astype(np.float64), N, model.hop)
    ticks = an.process_ticks(torch.from_numpy(x).cuda())
    w32 = np.asarray(an.w, dtype=np.float32).astype(np.float64)
    db = ticks.db.cpu().numpy().astype(np.float64)
    for r in range(R):
        model.tick(power[:, r * g:(r + 1) * g])
        imax, ipitch = analyzer_indices(an, ticks.fmax_hz[r], ticks.fpitch_hz[r])
        for c in range(C):
            lab = (N, T, r, c)
            assert_logpower_parity(db[c, r] - w32, fo.log_spectrogram(model.disp[c]), min_frac=0.0, strict=False,
                                   floor_db=40.0)
            assert peak_near_max(model.db(c), int(imax[c])), lab
            assert pitch_near_max(model.hps(c), int(ipitch[c])), lab
    check_analyzer("after the call", an, model, ticks.db[:, -1], ticks.fmax_hz[-1], ticks.fpitch_hz[-1])


@pytest.mark.parametrize("N,T", [(256, 5.0), (8192, 0.125)])
def test_dual_rows_follow_the_dual_oracle(N, T):
    """frt_spectrum_reduce_dual_ticks on float32 power, the oracle ticked on the same values: every
    row's transfer function, peak and pitch within test_spectrum_dual_gpu's bounds, both states after
    the call within STATE_TOL."""
    C, g, R = 3, 3, 20
    nb = N // 2 + 1
    rng = np.random.default_rng([N, 11])
    p1, p2 = pair_frames(rng, channel_envelopes(C, nb), pair_curves(C, nb), R * g)
    orcs = dual_oracles(C, N, T)
    an = SpectrumAnalyzer(C, fft_size=N, response_time=T, dual_channels=True)
    d1 = torch.zeros((C, nb), device="cuda")
    d2 = torch.zeros((C, nb), device="cuda")
    db = torch.empty((C, R, nb), device="cuda")
    imax = torch.empty((R, C), dtype=torch.int32, device="cuda")
    ipitch = torch.empty((R, C), dtype=torch.int32, device="cuda")
    t1, t2 = torch.from_numpy(p1).cuda(), torch.from_numpy(p2).cuda()
    an.proc.handle.call("frt_spectrum_reduce_dual_ticks", _lib._ptr(t1), _lib._ptr(t2), R * g * nb, nb, C, g,
                        R, nb, c_float(an.alpha), _lib._ptr(d1), _lib._ptr(d2), _lib._ptr(db), _lib._ptr(imax),
                        _lib._ptr(ipitch), _lib.current_stream_ptr())
    db, imax, ipitch = db.cpu().numpy(), imax.cpu().numpy(), ipitch.cpu().numpy()
    for r in range(R):
        tick_oracles(orcs, p1[:, r * g:(r + 1) * g], p2[:, r * g:(r + 1) * g])
        last = r == R - 1
        for c, o in enumerate(orcs):
            s1 = d1[c].cpu().numpy() if last else o.disp
            s2 = d2[c].cpu().numpy() if last else o.disp2
            bad = dual_failures(o, s1, s2, db[c, r], imax[r, c], ipitch[r, c])
            assert not bad, (N, T, r, c, bad)


def test_reference_fixture_through_process_ticks(golden_dir):
    """The unmodified reference's dual -> single -> dual ticks, each a process_ticks call of one tick
    of its frame count, with test_spectrum_dual_gpu's bounds."""
    from oracle.spectrum_dual import DualSpectrumWidgetOracle
    d = np.load(os.path.join(golden_dir, "spectrum_dual.npz"))
    x = d["x"][None]
    for key, N, T in fixture_cases(d):
        an = SpectrumAnalyzer(1, fft_size=N, response_time=T, weighting=1)
        pos = 0
        for t, (F, dual) in enumerate(zip(d["frames_" + key], d["dual_" + key])):
            an.setdualchannels(bool(dual))
            ticks = an.process_ticks(segment(x, pos, int(F), an.hop, N), frames_per_tick=int(F))
            pos += int(F)
            assert ticks.db.shape[1] == 1
            o = DualSpectrumWidgetOracle(N, response_time=T, weight=weight_table(N, 1))
            o.disp, o.disp2 = d["sp1_" + key][t], d["sp2_" + key][t]
            check = check_dual_analyzer if dual else check_single_analyzer
            check("%s tick %d" % (key, t), an, [o], ticks.db[:, 0], ticks.fmax_hz[0], ticks.fpitch_hz[0])


# --------------------------------------------------------------------------- plot
@pytest.mark.parametrize("peaks", [True, False])
@pytest.mark.parametrize("dual", [False, True])
def test_push_ticks_is_push_per_tick(dual, peaks):
    C, N, R = 5, 1024, 23
    an = SpectrumAnalyzer(C, fft_size=N, weighting=1, dual_channels=dual)
    x = stream(C, dual, R * 2 * an.hop + N - an.hop, 30)
    ticks = an.process_ticks(x)
    R = ticks.db.shape[1]
    pa, pb = SpectrumPlot(C), SpectrumPlot(C)
    for p in (pa, pb):
        p.setdualchannels(dual)
        p.set_peaks_enabled(peaks)
    first = ticks.db[:, 0].clone()
    pa.push(first, ticks.fmax_hz[0], ticks.fpitch_hz[0])     # a state to continue from
    pb.push(first, ticks.fmax_hz[0], ticks.fpitch_hz[0])
    got = pa.push_ticks(ticks)
    for r in range(R):
        want = pb.push(ticks.db[:, r], ticks.fmax_hz[r], ticks.fpitch_hz[r])
    for f in ("y", "z", "peak", "z_peak"):
        g, w = getattr(got, f), getattr(want, f)
        assert (g is None) == (w is None) and (g is None) == (not peaks and f in ("peak", "z_peak")), f
        if g is not None:
            assert torch.equal(bits(g), bits(w)), f
    for f in ("x_left", "x_right", "fmax_hz", "fpitch_hz", "fmax_x", "fpitch_x"):
        assert np.array_equal(getattr(got, f), getattr(want, f)), f
    assert got.baseline == want.baseline and got.fmax_text == want.fmax_text
    if peaks:
        for f in ("peak", "peak_int", "peak_decay"):
            assert torch.equal(getattr(pa, f).view(torch.int64), getattr(pb, f).view(torch.int64)), f
    pa.pause()
    assert pa.push_ticks(ticks) is got
    pa.restart()
    empty = SpectrumTicks(ticks.db[:, :0], ticks.fmax_hz[:0], ticks.fpitch_hz[:0])
    assert pa.push_ticks(empty) is got
    with pytest.raises(ValueError):
        pa.push_ticks(SpectrumTicks(None, ticks.fmax_hz, ticks.fpitch_hz))


# --------------------------------------------------------------------------- refusals
def ticks_args(C=2, nb=513, g=2, R=3, alpha=0.5, dual=False):
    """A valid argument list for frt_spectrum_reduce_ticks / _dual_ticks, with its buffers."""
    p = torch.ones((C, g * R, nb), device="cuda")
    d1, d2 = torch.zeros((C, nb), device="cuda"), torch.zeros((C, nb), device="cuda")
    db = torch.full((C, R, nb), 7.0, device="cuda")
    imax = torch.full((R, C), -1, dtype=torch.int32, device="cuda")
    ip = torch.full((R, C), -1, dtype=torch.int32, device="cuda")
    keep = (p, d1, d2, db, imax, ip)
    st = _lib.current_stream_ptr()
    if dual:
        args = [_lib._ptr(p), _lib._ptr(p), g * R * nb, nb, C, g, R, nb, c_float(alpha), _lib._ptr(d1),
                _lib._ptr(d2), _lib._ptr(db), _lib._ptr(imax), _lib._ptr(ip), st]
    else:
        args = [_lib._ptr(p), g * R * nb, nb, C, g, R, nb, c_float(alpha), _lib._ptr(d1), None, _lib._ptr(db),
                _lib._ptr(imax), _lib._ptr(ip), st]
    return args, keep


SINGLE_BAD = {"channels": (3, -1), "frames_per_tick 0": (4, 0), "frames_per_tick 8193": (4, 8193),
              "ticks": (5, -1), "bins": (6, 2), "alpha 0": (7, c_float(0.0)), "alpha > 1": (7, c_float(1.5)),
              "alpha < 0": (7, c_float(-0.5)), "alpha NaN": (7, c_float(float("nan"))), "power": (0, None), "disp": (8, None), "fmax": (11, None), "pitch": (12, None),
              "bins too large": (6, 60000)}
DUAL_BAD = {"pairs": (4, -1), "frames_per_tick 0": (5, 0), "frames_per_tick 8193": (5, 8193),
            "ticks": (6, -1), "bins": (7, 2), "alpha": (8, c_float(-0.1)), "power1": (0, None),
            "power2": (1, None), "disp1": (9, None), "disp2": (10, None), "fmax": (12, None),
            "pitch": (13, None)}


@pytest.mark.parametrize("dual,name", [(False, k) for k in SINGLE_BAD] + [(True, k) for k in DUAL_BAD])
def test_refusals_run_nothing_and_keep_the_handle(dual, name):
    h = _lib.default_handle()
    fn = "frt_spectrum_reduce_dual_ticks" if dual else "frt_spectrum_reduce_ticks"
    args, keep = ticks_args(dual=dual)
    i, v = (DUAL_BAD if dual else SINGLE_BAD)[name]
    bad = list(args)
    bad[i] = v
    torch.cuda.synchronize()
    n = h.launch_count
    with pytest.raises(_lib.FrtValueError):
        h.call(fn, *bad)
    torch.cuda.synchronize()
    assert h.launch_count == n
    _, d1, d2, db, imax, ip = keep
    assert torch.all(db == 7.0) and torch.all(imax == -1) and torch.all(d1 == 0) and torch.all(d2 == 0)
    h.call(fn, *args)                      # the handle still works
    torch.cuda.synchronize()
    assert torch.all(imax >= 0) and torch.all(ip >= 0) and h.launch_count == n + 2


def test_zero_ticks_or_channels_do_nothing():
    h = _lib.default_handle()
    for i, name in ((3, "channels"), (5, "ticks")):
        args, keep = ticks_args()
        args[i] = 0
        args[0] = None            # no buffer is looked at
        n = h.launch_count
        h.call("frt_spectrum_reduce_ticks", *args)
        assert h.launch_count == n, name


def test_analyzer_refusals_leave_it_usable():
    a, b = pair(2, 1024, 0.125, 0, False)
    x = stream(2, False, 6 * 256 + 768, 40)
    n = a.proc.handle.launch_count
    for g in (0, 8193, 4, 2.0, True):          # 6 frames: not whole 4-frame ticks
        with pytest.raises(_lib.FrtValueError):
            a.process_ticks(x, frames_per_tick=g)
    assert a.proc.handle.launch_count == n and a._disp is None
    same_as_per_tick(a, b, x, 3, 2, "after refusals")


# --------------------------------------------------------------------------- stream order
@pytest.mark.parametrize("way", WAYS)
@pytest.mark.parametrize("dual", [False, True])
def test_stream_order(side, dual, way):
    """Queued behind a hold on NaN-poisoned inputs: the same ticks as a synchronised run."""
    C, N, g, R = 3, 1024, 2, 9
    T = R * g * (N // 4) + N - N // 4

    def make():
        return SpectrumAnalyzer(C, fft_size=N, weighting=1, dual_channels=dual)

    def warm(a, kw):
        a.process_ticks(signal((C, 2, T) if dual else (C, T), 50), frames_per_tick=g, **kw)

    def run(a, x, kw):
        return a.process_ticks(x, frames_per_tick=g, **kw)

    def run_plot(a, x, kw):
        return a.process_ticks(x, frames_per_tick=g, **kw).fmax_hz

    shape = (C, 2, T) if dual else (C, T)
    check(make, [(run, signal(shape, 51)), (run_plot, signal(shape, 52))], way, side, warm=warm)
