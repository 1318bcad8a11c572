"""The spectrum widget's dual-channel measurement mode: the transfer function between a reference and
a measurement channel, for many pairs at once.

``frt_spectrum_reduce_dual`` (``csrc/reduce.cu``, behind ``SpectrumAnalyzer(dual_channels=True)``)
smooths both power stacks of a pair into the carried states (the widget's ``dispbuffers1`` and
``dispbuffers2``), then forms 10 log10(sp2 + 1e-30) - 10 log10(sp1 + 1e-30), its arg-max and the
harmonic-product arg-max of sp1 (friture/spectrum.py:141-182).  The float64 reference is
``oracle.spectrum_dual.DualSpectrumWidgetOracle`` on the same float32 power values.

Bounds, after every tick:
- both carried states within STATE_TOL of their peaks;
- the transfer function within TOL * max(max|ref|, 1) on every bin;
- the peak index at a near-maximum of the reference's transfer function, and db[imax] == max(db);
- the pitch index at a near-maximum of the reference's harmonic product of sp1.

The CPU tests (no mark) check the oracle against a fixture made with the unmodified reference, and
that these bounds reject swapped channels, weighting in dual mode, the pitch taken from sp2, and
the difference formed from float32 dB values or a float32 ratio."""
import os
import sys
from ctypes import c_float

import numpy as np
import pytest

from oracle import friture_oracle as fo
from oracle.spectrum_dual import DualSpectrumWidgetOracle

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from parity import TOL, assert_logpower_parity  # noqa: E402
from test_widget_reductions_gpu import (  # noqa: E402
    E2E_SIZES, FFT_SIZES, MAX_FRAMES, RESPONSE_TIMES, analyzer_indices, case_frames,
    channel_envelopes, e2e_stream, padded_power, peak_near_max, pitch_near_max, state_ratio,
    stationary_frames, tick_sizes, weight_table, weight_table_f32, widget_alpha)

FIR = np.array([0.6, -0.3, 0.2, -0.1, 0.05])   # measurement = FIR(reference) delayed, plus noise
DELAY = 23


# --------------------------------------------------------------------------- references
def dual_oracles(C, fft_size, response_time, weighting=0, dual=True):
    return [DualSpectrumWidgetOracle(fft_size, response_time=response_time,
                                     weight=weight_table(fft_size, weighting), dual_channels=dual)
            for _ in range(C)]


def tick_oracles(orcs, p1, p2):
    """p1, p2: [C, F, bins] power of the pairs' rows 0 and 1 (p2 None: one row)."""
    for c, o in enumerate(orcs):
        o.tick_power(p1[c].T.astype(np.float64), None if p2 is None else p2[c].T.astype(np.float64))


def transfer_db(s1, s2):
    """10 log10(s2 + 1e-30) - 10 log10(s1 + 1e-30) in float64 (spectrum.py:169)."""
    return (fo.log_spectrogram(np.asarray(s2, np.float64)) -
            fo.log_spectrogram(np.asarray(s1, np.float64)))


def dual_failures(orc, disp1, disp2, db, imax, ipitch):
    """The bounds of one pair against its oracle; returns the names of the ones that fail."""
    ref = transfer_db(orc.disp, orc.disp2)
    bad = []
    if state_ratio(disp1, orc.disp) > 1.0:
        bad.append("state 1")
    if state_ratio(disp2, orc.disp2) > 1.0:
        bad.append("state 2")
    err = np.abs(np.asarray(db, np.float64) - ref)
    if not np.all(err < TOL * max(float(np.max(np.abs(ref))), 1.0)):
        bad.append("dB")
    if not (peak_near_max(ref, int(imax)) and db[int(imax)] == np.max(db)):
        bad.append("peak")
    if not pitch_near_max(fo.harmonic_product_spectrum(orc.disp), int(ipitch)):
        bad.append("pitch")
    return bad


def check_pairs(label, orcs, disp1, disp2, db, imax, ipitch):
    """Every pair's bounds; returns (worst state ratio, worst dB error over max(max|ref|, 1))."""
    worst = (0.0, 0.0)
    for c, o in enumerate(orcs):
        bad = dual_failures(o, disp1[c], disp2[c], db[c], imax[c], ipitch[c])
        assert not bad, "%s pair %d: %s (state ratios %.3g %.3g)" % (
            label, c, bad, state_ratio(disp1[c], o.disp), state_ratio(disp2[c], o.disp2))
        ref = transfer_db(o.disp, o.disp2)
        rel = float(np.max(np.abs(db[c] - ref)) / max(float(np.max(np.abs(ref))), 1.0))
        worst = (max(worst[0], state_ratio(disp1[c], o.disp), state_ratio(disp2[c], o.disp2)),
                 max(worst[1], rel))
    return worst


def pair_curves(C, nb):
    """Per pair a transfer curve spanning about +-40 dB, each with its own shape."""
    u = np.arange(nb) / (nb - 1)
    return np.stack([40.0 * np.sin(2 * np.pi * (1.0 + 0.5 * c) * u + 0.7 * c) for c in range(C)])


def pair_frames(rng, env, H, F):
    """[C, F, bins] float32 reference and measurement power: the envelope times independent
    chi-squared fluctuations, the measurement's mean shaped by the transfer curve H (dB)."""
    return stationary_frames(rng, env, F), stationary_frames(rng, env * 10.0 ** (H / 10.0), F)


# --------------------------------------------------------------------------- float32 replicas
def replica_dual(s1, s2, bug=None, w32=None):
    """The kernel's output arithmetic on float32 states s1, s2 [bins], restated in numpy, with one
    of the bugs: 'swap' (channels swapped), 'weighting' (the table added in dual mode),
    'hps_sp2' (pitch from the measurement), 'f32_ratio' (log of a float32 ratio), 'f32_db'
    (difference of two float32 dB values).  Returns (db float32, imax, ipitch)."""
    s1 = np.asarray(s1, np.float32)
    s2 = np.asarray(s2, np.float32)
    if bug == "swap":
        s1, s2 = s2, s1
    with np.errstate(over="ignore", divide="ignore"):
        if bug == "f32_ratio":
            db = (10.0 * np.log10((s2 + np.float32(1e-30)) / (s1 + np.float32(1e-30)))).astype(np.float32)
        elif bug == "f32_db":
            db = (10.0 * np.log10(s2.astype(np.float64) + 1e-30)).astype(np.float32) - \
                 (10.0 * np.log10(s1.astype(np.float64) + 1e-30)).astype(np.float32)
        else:
            db = (10.0 * np.log10((s2.astype(np.float64) + 1e-30) /
                                  (s1.astype(np.float64) + 1e-30))).astype(np.float32)
    if bug == "weighting":
        db = db + w32
    hsrc = s2 if bug == "hps_sp2" else s1
    return db, int(np.argmax(db)), int(np.argmax(fo.harmonic_product_spectrum(hsrc.astype(np.float64))))


def replica_states(p1, p2, s1, s2, alpha):
    """One tick of the kernel's smoothing (s + alpha (x - s) in double, rounded once per tick)."""
    a = float(np.float32(alpha))
    s1, s2 = s1.astype(np.float64), s2.astype(np.float64)
    for f in range(p1.shape[0]):
        s1 = s1 + a * (p1[f].astype(np.float64) - s1)
        s2 = s2 + a * (p2[f].astype(np.float64) - s2)
    return s1.astype(np.float32), s2.astype(np.float32)


# --------------------------------------------------------------------------- CPU: fixture, bounds
def fixture_cases(d):
    for key in sorted(k[len("alpha_"):] for k in d.files if k.startswith("alpha_")):
        N = int(key.split("_")[0][1:])
        T = int(key.split("_t")[1]) / 1000.0
        yield key, N, T


def test_oracle_matches_reference_fixture(golden_dir):
    """DualSpectrumWidgetOracle (A weighting) against the unmodified reference's ticks: every
    dual / single tick's dB, peak, pitch and both states to 1e-12."""
    d = np.load(os.path.join(golden_dir, "spectrum_dual.npz"))
    x = d["x"].astype(np.float64)
    n_cases = 0
    for key, N, T in fixture_cases(d):
        o = DualSpectrumWidgetOracle(N, response_time=T, weight=weight_table(N, 1))
        assert o.alpha == d["alpha_" + key]
        pos = 0
        for t, (F, dual) in enumerate(zip(d["frames_" + key], d["dual_" + key])):
            o.setdualchannels(bool(dual))
            db, _, _, i, p = o.tick(x[:, pos * o.hop:(pos + F - 1) * o.hop + N])
            pos += int(F)
            ref_db = d["db_" + key][t]
            assert np.max(np.abs(db - ref_db)) <= 1e-12 * max(np.max(np.abs(ref_db)), 1.0), (key, t)
            for s, name in ((o.disp, "sp1_"), (o.disp2, "sp2_")):
                ref = d[name + key][t]
                assert np.max(np.abs(s - ref)) <= 1e-12 * np.max(np.abs(ref)), (key, t, name)
            assert i == d["imax_" + key][t] and p == d["ipitch_" + key][t], (key, t)
        assert list(d["dual_" + key]).count(False) > 0 and d["dual_" + key][-1]
        n_cases += 1
    assert n_cases == 4


def grid_case_states(fft_size, response_time, n_ticks=12):
    """A few ticks of the kernel-grid input through replica_states, with the oracles alongside."""
    nb = fft_size // 2 + 1
    rng = np.random.default_rng([fft_size, int(response_time * 1000), 7])
    env, H = channel_envelopes(2, nb), pair_curves(2, nb)
    orcs = dual_oracles(2, fft_size, response_time)
    s1 = np.zeros((2, nb), np.float32)
    s2 = np.zeros((2, nb), np.float32)
    for F in tick_sizes(case_frames(fft_size, response_time))[:n_ticks]:
        p1, p2 = pair_frames(rng, env, H, F)
        tick_oracles(orcs, p1, p2)
        for c in range(2):
            s1[c], s2[c] = replica_states(p1[c], p2[c], s1[c], s2[c], orcs[c].alpha)
    return orcs, s1, s2


@pytest.mark.parametrize("fft_size,response_time", [(256, 0.125), (8192, 0.3)])
def test_bounds_reject_plausible_bugs(fft_size, response_time):
    """The kernel's arithmetic meets every bound on the grid's input; swapped channels, the
    weighting applied in dual mode and the pitch taken from sp2 each fail one."""
    orcs, s1, s2 = grid_case_states(fft_size, response_time)
    w32 = weight_table_f32(fft_size, 1)
    for c, o in enumerate(orcs):
        assert not dual_failures(o, s1[c], s2[c], *replica_dual(s1[c], s2[c])), c
    for bug, check in (("swap", "dB"), ("weighting", "dB"), ("hps_sp2", "pitch")):
        fails = [dual_failures(o, s1[c], s2[c], *replica_dual(s1[c], s2[c], bug, w32))
                 for c, o in enumerate(orcs)]
        assert any(check in f for f in fails), (bug, fails)


def test_float32_forms_of_the_difference_fail():
    """A float32 ratio overflows to inf on a silent reference against a measurement at 1e10; two
    float32 dB values near -160 dB, subtracted, miss the 1e-5 dB bound of a transfer function
    near 0 dB.  The double form meets both."""
    nb = 513
    o = dual_oracles(1, 1024, 0.125)[0]
    o.disp, o.disp2 = np.zeros(nb), np.full(nb, 1e10)
    s1, s2 = np.zeros(nb, np.float32), np.full(nb, 1e10, np.float32)
    db, _, _ = replica_dual(s1, s2, "f32_ratio")
    assert np.isinf(db).all()
    assert "dB" in dual_failures(o, s1, s2, db, 0, 0)
    assert not dual_failures(o, s1, s2, *replica_dual(s1, s2))

    rng = np.random.default_rng(3)
    s1 = (1e-16 * (1 + rng.random(nb))).astype(np.float32)
    s2 = (s1.astype(np.float64) * (1 + 1e-6 * rng.standard_normal(nb))).astype(np.float32)
    o.disp, o.disp2 = s1.astype(np.float64), s2.astype(np.float64)
    ref = transfer_db(s1, s2)
    assert np.max(np.abs(ref)) < 1.0                      # the bound is 1e-5 dB absolute
    assert "dB" in dual_failures(o, s1, s2, *replica_dual(s1, s2, "f32_db"))
    assert not dual_failures(o, s1, s2, *replica_dual(s1, s2))


def test_oracle_single_mode_decays_second_state():
    """Single-mode ticks smooth an all-zero second column: dispbuffers2 * (1-alpha)^frames, and the
    dual ticks after them resume from it (spectrum.py:142,158-159)."""
    x = e2e_stream(256, 40, C=1)[0].astype(np.float64)
    xx = np.stack([x, 0.5 * x])
    o = DualSpectrumWidgetOracle(256, response_time=0.3, dual_channels=True)
    o.tick(xx[:, :256 + 9 * 64])
    kept = o.disp2.copy()
    o.setdualchannels(False)
    assert o.tick(xx[:, 640:640 + 256 + 6 * 64])[3] == int(np.argmax(fo.log_spectrogram(o.disp)))
    assert np.allclose(o.disp2, kept * (1 - o.alpha) ** 7, rtol=1e-14, atol=0)
    assert o.tick(xx[:, :100]) is None                    # no frame: nothing changes
    o.setdualchannels(True)
    db, _, _, _, _ = o.tick(xx[:, 1088:1088 + 256 + 3 * 64])
    assert np.allclose(db, transfer_db(o.disp, o.disp2), rtol=0, atol=1e-12)


# --------------------------------------------------------------------------- GPU: the C ABI
class DualBuffers:
    def __init__(self, C, nb):
        import torch
        self.disp1 = torch.zeros((C, nb), dtype=torch.float32, device="cuda")
        self.disp2 = torch.zeros((C, nb), dtype=torch.float32, device="cuda")
        self.db = torch.empty((C, nb), dtype=torch.float32, device="cuda")
        self.imax = torch.empty(C, dtype=torch.int32, device="cuda")
        self.ipitch = torch.empty(C, dtype=torch.int32, device="cuda")

    def run(self, h, p1, p2, alpha):
        """One call over p1, p2 [C, F, bins] (host float32), interleaved as the analyzer's STFT
        leaves them (pair c's rows at 2c and 2c + 1), NaN-padded.  Returns host outputs."""
        from friture_b200 import _lib
        C, F, nb = p1.shape
        if F:
            buf, sc, sf = padded_power(np.stack([p1, p2], axis=1).reshape(2 * C, F, nb))
            b1, b2 = buf.data_ptr(), buf.data_ptr() + 4 * sc
        else:
            b1, b2, sc, sf = 0, 0, 0, nb
        h.call("frt_spectrum_reduce_dual", _lib._ptr(b1), _lib._ptr(b2), 2 * sc, sf, C, F, nb,
               c_float(alpha), _lib._ptr(self.disp1), _lib._ptr(self.disp2), _lib._ptr(self.db),
               _lib._ptr(self.imax), _lib._ptr(self.ipitch), _lib.current_stream_ptr())
        return tuple(t.cpu().numpy() for t in (self.disp1, self.disp2, self.db, self.imax, self.ipitch))


@pytest.mark.gpu
@pytest.mark.parametrize("response_time", RESPONSE_TIMES)
@pytest.mark.parametrize("fft_size", FFT_SIZES)
def test_dual_reduce_grid(fft_size, response_time):
    """Two pairs, each a +-40 dB transfer curve times independent chi-squared fluctuations, for
    3 / alpha frames in ticks of 1, 0, 7, 64 and 8192 frames, rows padded with NaN; every output
    checked after every tick."""
    from friture_b200 import _lib
    h = _lib.default_handle()
    nb = fft_size // 2 + 1
    rng = np.random.default_rng([fft_size, int(response_time * 1000), 2])
    env, H = channel_envelopes(2, nb), pair_curves(2, nb)
    orcs = dual_oracles(2, fft_size, response_time)
    bufs = DualBuffers(2, nb)
    sizes = tick_sizes(case_frames(fft_size, response_time))
    worst = (0.0, 0.0)
    for t, F in enumerate(sizes):
        p1, p2 = pair_frames(rng, env, H, F)
        tick_oracles(orcs, p1, p2)
        out = bufs.run(h, p1, p2, orcs[0].alpha)
        label = "N=%d T=%g tick %d (%d frames)" % (fft_size, response_time, t, F)
        worst = tuple(map(max, worst, check_pairs(label, orcs, *out)))
    print("dual N=%d T=%g: %d frames in %d ticks, worst state ratio %.4f, worst dB error %.3g"
          % (fft_size, response_time, sum(sizes), len(sizes), worst[0], worst[1]))


@pytest.mark.gpu
@pytest.mark.parametrize("fft_size", [32, 1024, 16384])
def test_dual_reduce_edge_cases(fft_size):
    """Identical channels, both silent, a silent reference against 1e10, a silent measurement, and
    exact ties in far-apart bins, one pair each, two ticks."""
    from friture_b200 import _lib
    h = _lib.default_handle()
    nb = fft_size // 2 + 1
    rng = np.random.default_rng([fft_size, 11])
    base = stationary_frames(rng, channel_envelopes(1, nb), 9)[0]          # [F, bins]
    z = np.zeros_like(base)
    loud = (1e10 * rng.exponential(size=base.shape)).astype(np.float32)
    tie1 = (1e-6 * rng.exponential(size=base.shape)).astype(np.float32)
    k = [1, 2, 3, nb // 3 - 1, 2 * (nb // 3 - 1), 3 * (nb // 3 - 1)]       # HPS tie at 1 and nb//3-1
    tie1[:, k] = np.float32(0.25)
    tie2 = (tie1 * 1e-2 * rng.exponential(size=base.shape)).astype(np.float32)
    far = [nb // 2 + 1, nb - 2]                                            # dB tie, far apart
    assert not set(far) & set(k)
    tie1[:, far] = np.float32(1e-6)
    tie2[:, far] = np.float32(1.0)
    p1 = np.stack([base, z, z, base, tie1])
    p2 = np.stack([base, z, loud, z, tie2])
    orcs = dual_oracles(5, fft_size, 0.125)
    bufs = DualBuffers(5, nb)
    for t, F in enumerate([4, 5]):
        sl = slice(0, 4) if t == 0 else slice(4, 9)
        tick_oracles(orcs, p1[:, sl], p2[:, sl])
        disp1, disp2, db, imax, ipitch = bufs.run(h, p1[:, sl], p2[:, sl], orcs[0].alpha)
        check_pairs("N=%d tick %d" % (fft_size, t), orcs, disp1, disp2, db, imax, ipitch)
        assert np.array_equal(db[0], np.zeros(nb, np.float32)) and imax[0] == 0
        assert np.array_equal(db[1], np.zeros(nb, np.float32)) and imax[1] == 0 and ipitch[1] == 0
        assert np.all(np.isfinite(db[2])) and np.min(db[2]) > 300.0
        dB1 = 10.0 * np.log10(disp1[3].astype(np.float64) + 1e-30)
        assert np.max(np.abs(db[3] - (-300.0 - dB1))) < TOL * np.max(np.abs(-300.0 - dB1))
        ref = transfer_db(orcs[4].disp, orcs[4].disp2)
        assert db[4, far[0]] == db[4, far[1]] == db[4].max() and imax[4] == far[0] == np.argmax(ref)
        hps = fo.harmonic_product_spectrum(orcs[4].disp)
        assert np.sum(hps == hps.max()) == 2 and ipitch[4] == 1 == np.argmax(hps)


@pytest.mark.gpu
@pytest.mark.parametrize("fft_size", [32, 1024, 16384])
def test_dual_reduce_many_pairs(fft_size):
    """2 * SM + 5 pairs, each with a transfer peak 50 dB up at its own bin, so that a mix-up
    between pairs moves the peak index; the carried states are bit-identical to those of
    frt_spectrum_reduce over the same 2P channels."""
    import torch
    from friture_b200 import _lib
    h = _lib.default_handle()
    C = 2 * h.sm_count + 5
    nb = fft_size // 2 + 1
    rng = np.random.default_rng([fft_size, C, 3])
    env = np.stack([10.0 ** (-(c % 8)) * (0.01 + np.zeros(nb)) for c in range(C)])
    peak = (7 * np.arange(C) + 1) % nb
    orcs = dual_oracles(C, fft_size, 0.125)
    bufs = DualBuffers(C, nb)
    single = torch.zeros((2 * C, nb), dtype=torch.float32, device="cuda")
    scratch = [torch.empty((2 * C, nb), dtype=torch.float32, device="cuda")] + \
              [torch.empty(2 * C, dtype=torch.int32, device="cuda") for _ in range(2)]
    for t, F in enumerate([3, 0, 17, 1]):
        p1, p2 = stationary_frames(rng, env, F), stationary_frames(rng, env, F)
        p1[np.arange(C), :, peak] = env[np.arange(C), peak][:, None]
        p2[np.arange(C), :, peak] = 1e5 * env[np.arange(C), peak][:, None]
        tick_oracles(orcs, p1, p2)
        disp1, disp2, db, imax, ipitch = bufs.run(h, p1, p2, orcs[0].alpha)
        check_pairs("C=%d N=%d tick %d" % (C, fft_size, t), orcs, disp1, disp2, db, imax, ipitch)
        assert np.array_equal(imax, peak), "C=%d N=%d tick %d" % (C, fft_size, t)
        both = np.stack([p1, p2], axis=1).reshape(2 * C, F, nb)
        pw = torch.from_numpy(both).cuda() if F else None
        h.call("frt_spectrum_reduce", _lib._ptr(pw), F * nb, nb, 2 * C, F, nb, c_float(orcs[0].alpha),
               _lib._ptr(single), None, _lib._ptr(scratch[0]), _lib._ptr(scratch[1]),
               _lib._ptr(scratch[2]), _lib.current_stream_ptr())
        s = single.cpu().numpy()
        assert np.array_equal(s[0::2], disp1) and np.array_equal(s[1::2], disp2)


@pytest.mark.gpu
def test_dual_reduce_rejected_arguments_leave_handle_usable():
    """nbins < 3, more than 8192 frames, alpha outside (0, 1] or NaN and every NULL buffer
    (power2 and disp2 included) raise FrtValueError and run nothing; a valid call afterwards gives
    the same results as before them; no pairs is a no-op."""
    import torch
    from friture_b200 import _lib
    from friture_b200._lib import FrtValueError
    h = _lib.default_handle()
    nb, F = 129, 5
    rng = np.random.default_rng(9)
    env = channel_envelopes(2, nb)
    p1, p2 = pair_frames(rng, env, pair_curves(2, nb), F)
    alpha = widget_alpha(256, 0.125)
    first = DualBuffers(2, nb).run(h, p1, p2, alpha)
    big = torch.zeros((2, MAX_FRAMES + 1, 3), device="cuda")
    b = DualBuffers(2, nb)
    buf, sc, sf = padded_power(np.stack([p1, p2], axis=1).reshape(4, F, nb))
    b1, b2 = buf.data_ptr(), buf.data_ptr() + 4 * sc
    ptr, cur = _lib._ptr, _lib.current_stream_ptr()

    def call(q1, q2, stride_c, stride_f, C, nf, nbins, a, d1=b.disp1, d2=b.disp2, db=b.db,
             im=b.imax, ip=b.ipitch):
        h.call("frt_spectrum_reduce_dual", ptr(q1), ptr(q2), stride_c, stride_f, C, nf, nbins,
               c_float(a), ptr(d1), ptr(d2), ptr(db), ptr(im), ptr(ip), cur)

    bp = big.data_ptr()
    bad = [
        lambda: call(b1, b2, 2 * sc, sf, 2, F, 2, alpha),
        lambda: call(bp, bp + 4 * (MAX_FRAMES + 1) * 3, 2 * (MAX_FRAMES + 1) * 3, 3, 1, MAX_FRAMES + 1, 3, alpha),
        lambda: call(b1, b2, 2 * sc, sf, 2, F, nb, 0.0),
        lambda: call(b1, b2, 2 * sc, sf, 2, F, nb, -0.5),
        lambda: call(b1, b2, 2 * sc, sf, 2, F, nb, 1.5),
        lambda: call(b1, b2, 2 * sc, sf, 2, F, nb, float("nan")),
        lambda: call(b1, b2, 2 * sc, sf, -1, F, nb, alpha),
        lambda: call(None, b2, 2 * sc, sf, 2, F, nb, alpha),
        lambda: call(b1, None, 2 * sc, sf, 2, F, nb, alpha),
        lambda: call(b1, b2, 2 * sc, sf, 2, F, nb, alpha, d1=None),
        lambda: call(b1, b2, 2 * sc, sf, 2, F, nb, alpha, d2=None),
        lambda: call(b1, b2, 2 * sc, sf, 2, F, nb, alpha, db=None),
        lambda: call(b1, b2, 2 * sc, sf, 2, F, nb, alpha, im=None),
        lambda: call(b1, b2, 2 * sc, sf, 2, F, nb, alpha, ip=None),
    ]
    launches = h.launch_count
    for k, f in enumerate(bad):
        with pytest.raises(FrtValueError):
            f()
        assert not torch.any(b.disp1) and not torch.any(b.disp2), k      # nothing ran
    call(None, None, 0, 0, 0, F, nb, alpha, d1=None, d2=None)             # no pairs: nothing to do
    assert h.launch_count == launches
    again = DualBuffers(2, nb).run(h, p1, p2, alpha)
    for x, y in zip(first, again):
        assert np.array_equal(x, y)
    call(bp, bp + 4 * (MAX_FRAMES + 1) * 3, 2 * (MAX_FRAMES + 1) * 3, 3, 1, MAX_FRAMES, 3, 1.0)


# --------------------------------------------------------------------------- GPU: SpectrumAnalyzer
def pair_stream(fft_size, n_frames, C=3, seed=0):
    """[C, 2, samples] float32: row 0 the e2e stream, row 1 that through FIR, delayed by DELAY
    samples, plus independent noise 30 dB below the channel's level."""
    x0 = e2e_stream(fft_size, n_frames, C=C, seed=seed).astype(np.float64)
    rng = np.random.default_rng([fft_size, seed, 5])
    n = x0.shape[1]
    x1 = np.zeros_like(x0)
    for c in range(C):
        x1[c, DELAY:] = np.convolve(x0[c], FIR)[:n - DELAY]
        x1[c] += 10.0 ** (-2 * c) * 0.02 * 10 ** (-1.5) * rng.standard_normal(n)
    return np.stack([x0, x1], axis=1).astype(np.float32)


def stream_power(x, fft_size, hop):
    """[C, 2, samples] -> float64 power of rows 0 and 1, [C, frames, bins] each."""
    C = x.shape[0]
    p = fo.stft_power_batch(x.reshape(2 * C, -1).astype(np.float64), fft_size, hop)
    return p[0::2], p[1::2]


worst_db = [0.0]      # worst dB error of the analyzer tests, over max(max|ref|, 1), for the report


def check_dual_analyzer(label, an, orcs, db, fmax, fpitch):
    """Both states within STATE_TOL of the model's peaks; the dB within TOL * max(max|ref|, 1) of
    the float64 log-difference of the analyzer's own float32 states; the peak at a near-maximum of
    that, the pitch at a near-maximum of the model's harmonic product of sp1."""
    d1, d2 = an._disp.cpu().numpy(), an._disp2.cpu().numpy()
    db = db.cpu().numpy()
    imax, ipitch = analyzer_indices(an, fmax, fpitch)
    worst = 0.0
    for c, o in enumerate(orcs):
        lab = "%s pair %d" % (label, c)
        r = max(state_ratio(d1[c], o.disp), state_ratio(d2[c], o.disp2))
        worst = max(worst, r)
        assert r <= 1.0, (lab, r * 1e-5)
        own = transfer_db(d1[c], d2[c])
        worst_db[0] = max(worst_db[0], float(np.max(np.abs(db[c] - own)) / max(float(np.max(np.abs(own))), 1.0)))
        assert np.all(np.abs(db[c] - own) < TOL * max(float(np.max(np.abs(own))), 1.0)), lab
        assert peak_near_max(own, int(imax[c])) and db[c, imax[c]] == db[c].max(), lab
        assert pitch_near_max(fo.harmonic_product_spectrum(o.disp), int(ipitch[c])), lab
    return worst


def check_single_analyzer(label, an, orcs, db, fmax, fpitch):
    """A single-mode tick: state 1 and the weighted dB as check_analyzer does, state 2 decayed."""
    d1 = an._disp.cpu().numpy()
    db = db.cpu().numpy().astype(np.float64)
    w32 = np.asarray(an.w, dtype=np.float32).astype(np.float64)
    imax, ipitch = analyzer_indices(an, fmax, fpitch)
    for c, o in enumerate(orcs):
        lab = "%s ch %d" % (label, c)
        assert state_ratio(d1[c], o.disp) <= 1.0, lab
        if an._disp2 is not None:
            assert state_ratio(an._disp2.cpu().numpy()[c], o.disp2) <= 1.0, lab
        assert_logpower_parity(db[c] - w32, fo.log_spectrogram(o.disp), min_frac=0.0, strict=False,
                               floor_db=40.0)
        assert peak_near_max(fo.log_spectrogram(o.disp) + o.w, int(imax[c])), lab
        assert pitch_near_max(fo.harmonic_product_spectrum(o.disp), int(ipitch[c])), lab


def segment(x, pos, F, hop, fft_size):
    """The tick's samples for F frames from frame pos (F = 0: one sample short of a frame)."""
    import torch
    end = (pos + F - 1) * hop + fft_size if F else pos * hop + fft_size - 1
    return torch.from_numpy(np.ascontiguousarray(x[..., pos * hop:end])).cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("response_time", [0.125, 5.0])
@pytest.mark.parametrize("fft_size", E2E_SIZES)
def test_dual_analyzer_end_to_end(fft_size, response_time):
    """Three pairs through the real STFT for 3 / alpha frames, in ticks of 1, 0, 7, 64 and 8192
    frames: one STFT over the 2C rows, one dual reduce over the C pairs."""
    import torch
    from friture_b200.spectrum import SpectrumAnalyzer
    an = SpectrumAnalyzer(3, fft_size=fft_size, response_time=response_time, dual_channels=True)
    orcs = dual_oracles(3, fft_size, response_time)
    hop = an.hop
    total = case_frames(fft_size, response_time)
    x = pair_stream(fft_size, total)
    p1, p2 = stream_power(x, fft_size, hop)
    pos, worst, last = 0, 0.0, None
    for t, F in enumerate(tick_sizes(total)):
        label = "N=%d T=%g tick %d (%d frames)" % (fft_size, response_time, t, F)
        before = None if an._disp2 is None else (an._disp.clone(), an._disp2.clone())
        db, fmax, fpitch = an.process(segment(x, pos, F, hop, fft_size))
        if F == 0:
            assert torch.equal(an._disp, before[0]) and torch.equal(an._disp2, before[1]), label
            assert torch.equal(db, last[0]) and np.array_equal(fmax, last[1]), label
            continue
        tick_oracles(orcs, p1[:, pos:pos + F], p2[:, pos:pos + F])
        pos += F
        worst = max(worst, check_dual_analyzer(label, an, orcs, db, fmax, fpitch))
        last = (db.clone(), fmax.copy(), fpitch.copy())
    print("dual analyzer N=%d T=%g: %d frames, worst state ratio %.4f, worst dB error so far %.3g"
          % (fft_size, response_time, total, worst, worst_db[0]))


@pytest.mark.gpu
@pytest.mark.parametrize("fft_size", E2E_SIZES)
def test_dual_analyzer_exact_half_gain(fft_size):
    """x1 = 0.5 x0 exactly: the float32 powers scale by 0.25 exactly, so every bin with
    sp1 > 1e-20 shows 10 log10(0.25) within 1e-5 dB."""
    import torch
    from friture_b200.spectrum import SpectrumAnalyzer
    x0 = e2e_stream(fft_size, 12)
    x = np.stack([x0, x0 * np.float32(0.5)], axis=1)
    an = SpectrumAnalyzer(3, fft_size=fft_size, response_time=0.125, dual_channels=True)
    for k in range(2):
        db, _, _ = an.process(torch.from_numpy(np.ascontiguousarray(x[..., k * 5 * an.hop:])).cuda())
        s1 = an._disp.cpu().numpy()
        sel = s1 > 1e-20
        assert sel.sum() > 0.5 * sel.size
        assert np.max(np.abs(db.cpu().numpy()[sel] - 10.0 * np.log10(0.25))) <= 1e-5, (fft_size, k)


@pytest.mark.gpu
def test_dual_analyzer_toggle_and_reset():
    """dual -> single ([C, 2, T] and [C, T] ticks) -> dual, A weighting set: the single ticks
    weight sp1 and decay sp2 by (1-alpha)^frames, the dual ticks resume from the decayed state
    and ignore the weighting; setresponsetime and setweighting keep both states; setfftsize
    resets both."""
    import torch
    from friture_b200.spectrum import SpectrumAnalyzer
    an = SpectrumAnalyzer(3, fft_size=1024, response_time=0.125, weighting=1, dual_channels=True)
    orcs = dual_oracles(3, 1024, 0.125, weighting=1)

    def run(x, schedule, seed_label):
        hop = an.hop
        p1, p2 = stream_power(x, an.fft_size, hop)
        pos = 0
        for t, (F, form) in enumerate(schedule):
            label = "%s tick %d (%s, %d frames)" % (seed_label, t, form, F)
            seg = segment(x, pos, F, hop, an.fft_size)
            if form == "single rows":
                seg = seg[:, 0].contiguous()
            db, fmax, fpitch = an.process(seg)
            tick_oracles(orcs, p1[:, pos:pos + F], p2[:, pos:pos + F] if form == "pairs" else None)
            pos += F
            if an.dual_channels and form == "pairs":
                check_dual_analyzer(label, an, orcs, db, fmax, fpitch)
            else:
                check_single_analyzer(label, an, orcs, db, fmax, fpitch)

    x = pair_stream(1024, 80, seed=1)
    run(x, [(5, "pairs"), (9, "pairs")], "dual")
    an.setdualchannels(False)
    for o in orcs:
        o.setdualchannels(False)
    run(x[..., 14 * an.hop:], [(6, "pairs"), (11, "single rows"), (3, "pairs")], "single")
    an.setdualchannels(True)
    for o in orcs:
        o.setdualchannels(True)
    run(x[..., 34 * an.hop:], [(4, "single rows"), (7, "pairs"), (2, "pairs")], "dual again")
    kept = (an._disp.clone(), an._disp2.clone())
    an.setresponsetime(1.0)
    an.setweighting(2)
    assert torch.equal(an._disp, kept[0]) and torch.equal(an._disp2, kept[1])
    an.setfftsize(2048)
    assert an._disp is None and an._disp2 is None
    orcs[:] = dual_oracles(3, 2048, 1.0, weighting=2)
    run(pair_stream(2048, 30, seed=2), [(9, "pairs"), (12, "pairs")], "after setfftsize")


@pytest.mark.gpu
def test_dual_analyzer_matches_reference_fixture(golden_dir):
    """The analyzer (A weighting) through the unmodified reference's dual -> single -> dual ticks:
    both states within STATE_TOL of the fixture's, the dual dB within the bound of the analyzer's
    own states, the peak and the pitch at near-maxima."""
    import torch
    from friture_b200.spectrum import SpectrumAnalyzer
    d = np.load(os.path.join(golden_dir, "spectrum_dual.npz"))
    x = d["x"][None]                                               # one pair, [1, 2, T]
    for key, N, T in fixture_cases(d):
        an = SpectrumAnalyzer(1, fft_size=N, response_time=T, weighting=1)
        assert an.alpha == d["alpha_" + key]
        pos = 0
        for t, (F, dual) in enumerate(zip(d["frames_" + key], d["dual_" + key])):
            an.setdualchannels(bool(dual))
            db, fmax, fpitch = an.process(segment(x, pos, int(F), an.hop, N))
            pos += int(F)
            label = "%s tick %d" % (key, t)
            o = DualSpectrumWidgetOracle(N, response_time=T, weight=weight_table(N, 1))
            o.disp, o.disp2 = d["sp1_" + key][t], d["sp2_" + key][t]
            if dual:
                check_dual_analyzer(label, an, [o], db, fmax, fpitch)
            else:
                check_single_analyzer(label, an, [o], db, fmax, fpitch)
