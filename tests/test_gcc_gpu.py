"""GPU parity: GCC-PHAT delay estimation vs the CPU oracle and the reference golden vectors
(friture/signal/correlation.py:24-43; friture/delay_estimator.py:129-152)."""
import os
import sys

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
ABS_TOL = 1e-4   # SURVEY 8d #4: identical arg-max, Xcorr within 1e-4 absolute


def load(name):
    with np.load(os.path.join(GOLD, name)) as d:
        return {k: d[k] for k in d.files}


def test_golden_pair_and_smoothing():
    import torch
    from friture_b200.correlation import GccPhat, generalized_cross_correlation
    g = load("gcc_phat.npz")
    x = generalized_cross_correlation(g["d0"], g["d1"])
    assert x.dtype == np.float64 and x.shape == (24000,)
    assert np.max(np.abs(x - g["xcorr"])) < ABS_TOL
    assert int(np.argmax(np.abs(x))) == int(g["argmax"]) == 137
    est = GccPhat(24000)
    d = lambda k: torch.from_numpy(g[k]).cuda()[None, :]
    i1, v1, x1 = est.estimate(d("d0"), d("d1"), want_xcorr=True)
    i2, v2, x2 = est.estimate(d("d0b"), d("d1b"), want_xcorr=True)
    assert int(i1[0]) == 137 and int(i2[0]) == int(g["argmax_b"])
    assert abs(float(v1[0]) - g["xcorr"][137]) < ABS_TOL
    assert abs(float(v2[0]) - g["smoothed_b"][int(g["argmax_b"])]) < ABS_TOL
    assert np.max(np.abs(x2[0].cpu().numpy() - g["xcorr_b"])) < ABS_TOL
    assert np.max(np.abs(est._smoothed[0].cpu().numpy() - g["smoothed_b"])) < ABS_TOL
    assert abs(est.delay_ms(i1)[0] - 1e3 * 137 / 12000.0) < 1e-9


@pytest.mark.parametrize("L", [24000, 12000, 4096, 1000, 6000])
def test_batch_vs_oracle(L):
    import torch
    from friture_b200.correlation import GccPhat
    from oracle import friture_oracle as fo
    rng = np.random.default_rng(L)
    P = 5
    d0 = rng.standard_normal((P, L)).astype(np.float32)
    shifts = [3, L // 7, L // 2 - 1, L - 5, 0]
    d1 = np.stack([np.roll(d0[p], shifts[p]) * (-1 if p == 1 else 1)
                   + 0.1 * rng.standard_normal(L) for p in range(P)]).astype(np.float32)
    est = GccPhat(L)
    idx, val, xc = est.estimate(torch.from_numpy(d0).cuda(), torch.from_numpy(d1).cuda(),
                                smooth=False, want_xcorr=True)
    xc = xc.cpu().numpy()
    for p in range(P):
        ref = fo.generalized_cross_correlation(d0[p], d1[p])
        assert np.max(np.abs(xc[p] - ref)) < ABS_TOL
        i, v, _ = fo.delay_peak(ref)
        assert int(idx[p]) == i == shifts[p]
        assert abs(float(val[p]) - v) < ABS_TOL
    assert float(val[1]) < 0      # inverted polarity shows in the sign of the extremum


def test_constant_input_inputs_untouched_and_short_frame_refused():
    import torch
    from friture_b200.correlation import GccPhat
    L = 4096
    d0 = torch.zeros(2, L).cuda()
    d1 = torch.randn(2, L).cuda()
    d1c = d1.clone()
    idx, val, xc = GccPhat(L).estimate(d0, d1, smooth=False, want_xcorr=True)
    assert idx.tolist() == [0, 0] and val.tolist() == [0.0, 0.0]      # delay_estimator.py:164-167
    assert torch.equal(d1, d1c)
    with pytest.raises(ValueError):
        GccPhat(3).estimate(torch.zeros(1, 3).cuda(), torch.zeros(1, 3).cuda())


def test_config4_sample_4096_pairs():
    """BASELINE config #4 geometry on a bounded sample: known integer delays are recovered."""
    import torch
    from friture_b200.correlation import GccPhat
    L, P = 24000, 64
    g = torch.Generator().manual_seed(4)
    d0 = torch.randn(P, L, generator=g)
    k = torch.randint(0, L, (P,), generator=g)
    d1 = torch.stack([torch.roll(d0[p], int(k[p])) for p in range(P)]) + 0.1 * torch.randn(P, L, generator=g)
    idx, val, _ = GccPhat(L).estimate(d0.cuda(), d1.cuda(), smooth=False)
    assert torch.equal(idx.cpu().long(), k)


def test_silent_pairs_keep_no_smoothing_state():
    """A pair whose first frames are silent has no previous smoothed frame (old_Xcorr is None in the
    widget, delay_estimator.py:129-139): its first real frame is used unsmoothed, the later ones are
    blended; a silent frame in between leaves the state alone.  Two estimators with different frame
    lengths share the device (the kernel's shared-memory limit is set per launch)."""
    import torch
    from friture_b200.correlation import GccPhat
    from oracle import friture_oracle as fo
    rng = np.random.default_rng(5)
    L = 4096
    frames = []
    for k in range(3):
        d0 = rng.standard_normal((2, L))
        d1 = np.roll(d0, 40 + k, axis=1) + 0.1 * rng.standard_normal((2, L))
        frames.append((d0, d1))
    est = GccPhat(L)
    other = GccPhat(24000)                              # lowers / raises the per-device smem limit
    big = torch.randn(1, 24000, device="cuda")
    cuda = lambda a: torch.from_numpy(a.astype(np.float32)).cuda()
    # call 1: pair 0 silent, pair 1 real
    d0, d1 = frames[0]
    a0, a1 = d0.copy(), d1.copy()
    a0[0] = 0.25
    i, v, _ = est.estimate(cuda(a0), cuda(a1), smooth=True)
    other.estimate(big, big, smooth=False)
    assert int(i[0]) == 0 and float(v[0]) == 0.0
    old1 = fo.generalized_cross_correlation(a0[1].astype(np.float32).astype(np.float64),
                                            a1[1].astype(np.float32).astype(np.float64))
    # call 2: both real -> pair 0 unsmoothed (first valid frame), pair 1 blended with call 1
    d0, d1 = frames[1]
    i, v, _ = est.estimate(cuda(d0), cuda(d1), smooth=True)
    x0 = fo.generalized_cross_correlation(d0[0].astype(np.float32).astype(np.float64),
                                          d1[0].astype(np.float32).astype(np.float64))
    x1 = fo.generalized_cross_correlation(d0[1].astype(np.float32).astype(np.float64),
                                          d1[1].astype(np.float32).astype(np.float64))
    s1 = 0.3 * x1 + 0.7 * old1
    assert int(i[0]) == int(np.argmax(np.abs(x0))) and abs(float(v[0]) - x0[int(i[0])]) < ABS_TOL
    assert int(i[1]) == int(np.argmax(np.abs(s1))) and abs(float(v[1]) - s1[int(i[1])]) < ABS_TOL
    assert torch.isfinite(est._smoothed).all()
    # call 3: pair 1 silent -> its state stays; pair 0 blended with call 2
    d0, d1 = frames[2]
    a0, a1 = d0.copy(), d1.copy()
    a1[1] = -1.0
    est.estimate(cuda(a0), cuda(a1), smooth=True)
    assert np.max(np.abs(est._smoothed[1].cpu().numpy() - s1)) < ABS_TOL
    x0c = fo.generalized_cross_correlation(a0[0].astype(np.float32).astype(np.float64),
                                           a1[0].astype(np.float32).astype(np.float64))
    assert np.max(np.abs(est._smoothed[0].cpu().numpy() - (0.3 * x0c + 0.7 * x0))) < ABS_TOL
