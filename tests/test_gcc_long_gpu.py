"""GCC-PHAT's Bluestein route (friture_b200/csrc/gcc_long.cu), which GccPhat runs at the delay
widget's lengths the shared-memory kernel rejects, odd lengths included (Xcorr then has L-1
samples, like the reference's irfft), against the float64 oracle with the bound of
test_gcc_lengths_gpu: at most K = 20 times the error of the float32 restatement
(gcc_long_model.gcc_f32_any), plus 1e-7."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import gcc_long_model as gm  # noqa: E402
from test_gcc_lengths_gpu import (ABS_FLOOR, BLUESTEIN_LAUNCHES, K, PAIR_KINDS, SMEM_LAUNCHES,  # noqa: E402
                                  DelayPipelineModel, assert_route, assert_within, error_bound,
                                  length_cases, shift_recoverable, smooth_f32, smooth_f64)

from oracle import friture_oracle as fo  # noqa: E402

FS = 12000.0
# every widget range 0.7 .. 5.0 s the shared-memory kernel rejects (all but 0.8, 0.9 and 1.0 s)
WIDGET = [int(2 * (r / 10) * FS) for r in range(7, 51) if r not in (8, 9, 10)]
EXTRA = [28800,        # 2^7 3^2 5^2: 5-smooth, but too long for the shared memory
         240000, 2400000,
         16759199,     # 698.3 s: a prime length
         24000000]     # 1000 s, the widget's longest range
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda()


def group_size(L):
    """Pairs per workspace group (include/frt.h): 2 GiB over about 8 M + 8 (L'/2+1) bytes a pair."""
    M = 1 << gm.fft_log2(L)
    return (2 << 30) // (8 * M + 8 * (gm.out_length(L) // 2 + 1) + 4096)


def check_frames(est, L, frames, label, pairs=range(8)):
    """Run est over frames [(d0, d1)] with smoothing; check Xcorr, the smoothed buffer, the index
    and the value of the given pairs against the oracle after every frame."""
    old64, old32 = [None] * 8, [None] * 8
    worst = 0.0
    for f, (d0, d1, shifts) in enumerate(frames):
        idx, val, xc = est.estimate(cuda(d0), cuda(d1), smooth=True, want_xcorr=True)
        idx, val, xc = idx.cpu().numpy(), val.cpu().numpy(), xc.cpu().numpy()
        sm = est._smoothed.cpu().numpy()
        assert xc.shape == (8, gm.out_length(L)) and sm.shape == xc.shape
        for p in pairs:
            lab = "%s frame %d %s" % (label, f, PAIR_KINDS[p])
            x64, x32 = gm.gcc_f64(d0[p], d1[p]), gm.gcc_f32_any(d0[p], d1[p])
            s64, s32 = smooth_f64(x64, old64[p]), smooth_f32(x32, old32[p])
            old64[p], old32[p] = s64, s32
            worst = max(worst, assert_within(xc[p], x64, x32, lab + " xcorr"))
            worst = max(worst, assert_within(sm[p], s64, s32, lab + " smoothed"))
            i, v, _ = fo.delay_peak(s64)
            assert int(idx[p]) == i, (lab, int(idx[p]), i)
            if f == 0 and shift_recoverable(L, shifts[p]) and L % 2 == 0:
                assert i == shifts[p], lab
            assert abs(float(val[p]) - v) <= error_bound(s64, s32), lab
    print("%s: worst ratio %.2f" % (label, worst))


@pytest.mark.gpu
@pytest.mark.parametrize("L", WIDGET + EXTRA)
def test_long_length_vs_oracle(L):
    from friture_b200.correlation import GccPhat
    est = GccPhat(L)
    assert_route(est, BLUESTEIN_LAUNCHES)
    if L < 1000000:
        check_frames(est, L, [length_cases(L, seed=s) for s in range(2)], "L=%d" % L)
    else:
        # the float64 references take minutes at these lengths (the prime one most): one frame, and
        # the kinds shift 0, shift L/2, random shift and inverted checked of the eight computed
        check_frames(est, L, [length_cases(L)], "L=%d" % L, pairs=(0, 3, 5, 6))


@pytest.mark.gpu
def test_routes_alternate_on_one_handle():
    """A shared-memory and a Bluestein estimator alternate on one handle for three rounds: each
    call runs its own route and gives the same bits as on a fresh handle, so the handle follows
    the route of the last plan call and keeps both plans."""
    import torch
    from friture_b200._lib import Handle
    from friture_b200.correlation import GccPhat
    cases = []
    for L, launches in ((2400, SMEM_LAUNCHES), (16800, BLUESTEIN_LAUNCHES)):
        d0, d1, _ = length_cases(L)
        a, b = cuda(d0), cuda(d1)
        fresh = Handle(0)
        want = GccPhat(L, handle=fresh).estimate(a, b, smooth=False, want_xcorr=True)
        fresh.close()
        cases.append((L, launches, a, b, want))
    h = Handle(0)
    ests = {L: GccPhat(L, handle=h) for L, _, _, _, _ in cases}
    for r in range(3):
        for L, launches, a, b, want in cases:
            n = h.launch_count
            got = ests[L].estimate(a, b, smooth=False, want_xcorr=True)
            assert h.launch_count - n == launches, (r, L)
            assert all(torch.equal(x, y) for x, y in zip(got, want)), (r, L)


@pytest.mark.gpu
def test_long_same_bits_alone_in_groups_and_again():
    """One pair gives the same bits alone, as the first and the last of more pairs than one
    workspace group holds, and on a second call."""
    import torch
    from friture_b200.correlation import GccPhat
    L = 2400000
    P = group_size(L) + 2
    rng = np.random.default_rng(5)
    base = rng.standard_normal(L).astype(np.float32)
    a = torch.from_numpy(base).cuda()
    b = torch.roll(a, 12345) + 0.1 * torch.from_numpy(rng.standard_normal(L).astype(np.float32)).cuda()
    d0 = torch.randn(P, L, device="cuda")
    d1 = torch.randn(P, L, device="cuda")
    d0[0], d1[0], d0[P - 1], d1[P - 1] = a, b, a, b
    est = GccPhat(L)
    i1, v1, x1 = est.estimate(a[None], b[None], smooth=False, want_xcorr=True)
    iP, vP, xP = est.estimate(d0, d1, smooth=False, want_xcorr=True)
    i2, v2, x2 = est.estimate(a[None], b[None], smooth=False, want_xcorr=True)
    assert int(i1[0]) == 12345
    for i, v, x in ((iP[0], vP[0], xP[0]), (iP[P - 1], vP[P - 1], xP[P - 1]), (i2[0], v2[0], x2[0])):
        assert int(i) == int(i1[0]) and float(v) == float(v1[0])
        assert torch.equal(x, x1[0])


@pytest.mark.gpu
@pytest.mark.parametrize("L", [55199, 28800])
def test_long_silence_and_previous_frame_modes(L):
    """Six pairs, rows L+3 floats apart, four calls with silent pairs and have_prev = 0, 2, 2, 1,
    checked after each call against delay_estimator.py:129-142: raw Xcorr, smoothed buffer, index,
    value, and the "no previous frame" marker (NaN in slot 0)."""
    import torch
    from friture_b200 import _lib
    P, Lp, stride, FILL = 6, gm.out_length(L), L + 3, 7.0
    calls = [(0, {0: "zero", 3: "const0"}),
             (2, {0: "const", 1: "const1"}),      # 3 gets its first real frame; 1 goes silent
             (2, {2: "zero"}),                    # 0 gets its first real frame
             (1, {5: "const"})]
    rng = np.random.default_rng(L + 1)
    h = _lib.Handle(0)
    h.call("frt_gcc_plan", L)
    d0s = torch.full((P, stride), float("nan"), device="cuda")   # the padding must never be read
    d1s = torch.full((P, stride), float("nan"), device="cuda")
    xc = torch.empty((P, Lp), device="cuda")
    sm = torch.full((P, Lp), FILL, device="cuda")
    idx = torch.empty(P, dtype=torch.int32, device="cuda")
    val = torch.empty(P, dtype=torch.float32, device="cuda")
    old64, old32 = [None] * P, [None] * P
    for c, (have_prev, silent) in enumerate(calls):
        shifts = rng.integers(0, L, P)
        a = rng.standard_normal((P, L))
        b = np.stack([np.roll(a[p], shifts[p]) for p in range(P)]) + 0.1 * rng.standard_normal((P, L))
        for p, kind in silent.items():
            if kind in ("zero", "const"):
                a[p] = b[p] = 0.0 if kind == "zero" else 0.25
            elif kind == "const0":
                a[p] = 0.25
            else:
                b[p] = 0.25
        a, b = a.astype(np.float32), b.astype(np.float32)
        d0s[:, :L] = cuda(a)
        d1s[:, :L] = cuda(b)
        sm_before = sm.clone()
        h.call("frt_gcc_phat", _lib._ptr(d0s), _lib._ptr(d1s), stride, P, _lib._ptr(xc),
               _lib._ptr(sm), have_prev, _lib._ptr(idx), _lib._ptr(val), _lib.current_stream_ptr())
        torch.cuda.synchronize()
        g_xc, g_sm, g_idx, g_val = xc.cpu().numpy(), sm.cpu().numpy(), idx.cpu().numpy(), val.cpu().numpy()
        for p in range(P):
            label = "L=%d call %d pair %d" % (L, c + 1, p)
            if p in silent:
                assert g_idx[p] == 0 and g_val[p] == 0.0, label
                assert not np.any(g_xc[p]), label
                if old64[p] is None:
                    assert np.isnan(g_sm[p, 0]) and np.all(g_sm[p, 1:] == FILL), label
                else:
                    assert torch.equal(sm[p], sm_before[p]), label
                continue
            x64, x32 = gm.gcc_f64(a[p], b[p]), gm.gcc_f32_any(a[p], b[p])
            s64, s32 = smooth_f64(x64, old64[p]), smooth_f32(x32, old32[p])
            old64[p], old32[p] = s64, s32
            assert_within(g_xc[p], x64, x32, label + " xcorr")
            assert_within(g_sm[p], s64, s32, label + " smoothed")
            i, v, _ = fo.delay_peak(s64)
            assert g_idx[p] == i, label
            assert abs(float(g_val[p]) - v) <= error_bound(s64, s32), label
    assert all(o is not None for o in old64)


@pytest.mark.gpu
def test_long_golden_from_reference():
    """tests/golden/gcc_long.npz (oracle/make_golden_gcc_long.py): the unmodified reference's
    generalized_cross_correlation plus the widget's smoothing and peak pick over two frames at
    16800, 55199 (odd) and 240000, kept at every 61st index and around the peak."""
    from friture_b200.correlation import GccPhat
    from oracle.make_golden_gcc_long import golden_frames
    with np.load(os.path.join(GOLD, "gcc_long.npz")) as g:
        for L in (16800, 55199, 240000):
            (a0, a1), (b0, b1) = golden_frames(L)
            idx = g["index_%d" % L]
            est = GccPhat(L)
            ia, va, xa = est.estimate(cuda(a0[None]), cuda(a1[None]), smooth=True, want_xcorr=True)
            ib, vb, _ = est.estimate(cuda(b0[None]), cuda(b1[None]), smooth=True)
            assert xa.shape[1] == int(g["n_out_%d" % L])
            xa32 = gm.gcc_f32_any(a0, a1)
            s32 = smooth_f32(gm.gcc_f32_any(b0, b1), xa32)
            assert_within(xa[0].cpu().numpy()[idx], g["xcorr_%d" % L], xa32[idx], "golden L=%d frame 1" % L)
            sm = g["smoothed_%d" % L]
            assert_within(est._smoothed[0].cpu().numpy()[idx], sm, s32[idx], "golden L=%d frame 2 smoothed" % L)
            assert [int(ia[0]), int(ib[0])] == list(g["argmax_%d" % L])
            peak = int(np.searchsorted(idx, int(ib[0])))
            assert abs(float(vb[0]) - sm[peak]) <= error_bound(sm, s32[idx])


class OddAwarePipelineModel(DelayPipelineModel):
    """DelayPipelineModel with the reference's default irfft length in the float32 restatement."""

    def _frame(self, p, f0, f1):
        s64 = smooth_f64(gm.gcc_f64(f0, f1), self.old64[p])
        s32 = smooth_f32(gm.gcc_f32_any(f0, f1), self.old32[p])
        self.old64[p], self.old32[p] = s64, s32
        i = int(np.argmax(np.abs(s64)))
        v = float(s64[i])
        norm = abs(v) / (3 * np.std(s64))
        delay = 1e3 * float(i) / self.fs
        if delay > 1e3 * self.time / 2.:
            delay -= 1e3 * self.time
        x = (norm > 1.) * (norm - 1.)
        x = (0.12 * x) ** 3
        return delay, v, error_bound(s64, s32), (x / (1. + x)) * 100


@pytest.mark.gpu
@pytest.mark.parametrize("delayrange_s, L", [(0.7, 16800), (1.1, 26400), (2.3, 55199), (10.0, 240000)])
def test_delay_estimator_on_long_route(delayrange_s, L):
    """Three pairs: x1 lagging x0, x1 leading x0 (the wrap of delay_estimator.py:150-151), and a
    lag near the edge of the range; chunks of about a sixteenth of a hop, then twice that."""
    import torch
    from friture_b200.delay import DelayEstimator
    fs = 48000
    lags = [4 * round(f * delayrange_s * fs / 4) for f in (0.37, -0.23, 0.85)]
    model = OddAwarePipelineModel(3, delayrange_s)
    est = DelayEstimator(3, delayrange_s=delayrange_s)
    assert est.length == model.L == L
    assert_route(est.gcc, BLUESTEIN_LAUNCHES)
    hop48 = 4 * model.hop
    c1 = 512 * max(1, hop48 // (512 * 16))
    n1 = -(-5 * hop48 // c1)
    n2 = -(-5 * hop48 // (2 * c1))
    n = c1 * n1 + 2 * c1 * n2
    rng = np.random.default_rng(L)
    M = max(abs(d) for d in lags)
    base = 0.1 * rng.standard_normal(n + 2 * M)
    x0 = np.tile(base[M:M + n], (3, 1))
    x1 = np.stack([base[M - d:M - d + n] for d in lags]) + 0.01 * rng.standard_normal((3, n))
    x0, x1 = x0.astype(np.float32), x1.astype(np.float32)
    pos, frames, worst = 0, 0, 0.0
    for m in [c1] * n1 + [2 * c1] * n2:
        a, b = x0[:, pos:pos + m], x1[:, pos:pos + m]
        pos += m
        r = est.handle_new_data(cuda(a), cuda(b))
        r_ref, out = model.push(a.astype(np.float64), b.astype(np.float64))
        assert r == r_ref
        if r == 0:
            continue
        frames += r
        for p, (delay, v, bound, conf) in enumerate(out):
            label = "range %.1f frame %d pair %d" % (delayrange_s, frames, p)
            assert est.delay_ms[p] == delay, label
            dv = abs(float(est.Xcorr_extremum[p]) - v)
            assert dv <= bound, label
            worst = max(worst, dv * K / max(bound - ABS_FLOOR, 1e-30))
            if abs(conf - round(conf)) < 1e-6:
                assert abs(int(est.correlation[p]) - int(conf)) <= 1, label
            else:
                assert int(est.correlation[p]) == int(conf), label
    print("range %.1f: %d frames, worst extremum ratio %.2f" % (delayrange_s, frames, worst))
    assert frames >= 9
    # for odd L the L-1 point inverse stretches lags by L/(L-1): within two samples
    truth = [1e3 * d / fs for d in lags]
    assert np.allclose(est.delay_ms, truth, atol=(2 if L % 2 else 1) * 1e3 / 12000.0 + 1e-9)
    assert torch.isfinite(est.gcc._smoothed).all()
