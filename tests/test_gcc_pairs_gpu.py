"""GPU: GCC-PHAT between channel pairs of one multichannel frame (frt_gcc_set_pairs /
frt_gcc_phat_pairs, PairGccPhat, ArrayDelayEstimator) on both routes: the shared-memory kernels at
L = 2 400 and 24 000, the Bluestein transforms at 16 800, 55 199 (odd) and 240 000.

The channels 2k and 2k+1 share one complex transform, so the table (0, 1), (2, 3), ... gives the
same bits as frt_gcc_phat on the rows x[0::2], x[1::2]; any other table is checked against the
float64 oracle with the criterion of test_gcc_gpu (Xcorr and value within 1e-4, the same arg-max)."""
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_stream_order_gpu import check, side, signal  # noqa: E402,F401

from oracle import friture_oracle as fo  # noqa: E402

pytestmark = pytest.mark.gpu
ABS_TOL = 1e-4
LENGTHS = [2400, 24000, 16800, 55199, 240000]


def out_len(L):
    return L - (L & 1)


def planted(C, L, seed, shifts=None):
    """C channels: one noise source delayed by an integer shift per channel, plus a little noise."""
    rng = np.random.default_rng(seed)
    s = rng.standard_normal(L)
    if shifts is None:
        shifts = rng.integers(0, L // 3, C)
    x = np.stack([np.roll(s, int(k)) + 0.1 * rng.standard_normal(L) for k in shifts])
    return x.astype(np.float32), shifts


def cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda()


def assert_close(got_idx, got_val, got_x, ref_x, old, label):
    """One pair against the oracle: Xcorr within ABS_TOL, the smoothed peak's index and value."""
    if got_x is not None:
        assert np.max(np.abs(got_x - ref_x)) < ABS_TOL, label
    i, v, sm = fo.delay_peak(ref_x, old)
    assert int(got_idx) == i, (label, int(got_idx), i)
    assert abs(float(got_val) - v) < ABS_TOL, label
    return sm


def all_pairs(n):
    return [(i, j) for i in range(n) for j in range(i + 1, n)]


@pytest.mark.parametrize("L", LENGTHS)
def test_packed_table_same_bits_as_pair_rows(L):
    """Table (0,1), (2,3), (4,5) on 7 channels (the seventh in no pair, packed with zeros): the same
    bits as GccPhat on x[0::2], x[1::2] in idx, val, Xcorr and the smoothed buffer, over three
    frames with smoothing (have_prev 0, then 2); channel 3 is constant in the second frame."""
    from friture_b200.correlation import GccPhat, PairGccPhat
    C = 7
    pair_est = PairGccPhat(L, C, [(0, 1), (2, 3), (4, 5)])
    rows_est = GccPhat(L)
    for f in range(3):
        x, _ = planted(C, L, 100 + f)
        if f == 1:
            x[3] = 0.5
        xd = cuda(x)
        got = pair_est.estimate(xd, want_xcorr=True)
        want = rows_est.estimate(xd[0:6:2], xd[1:6:2], want_xcorr=True)
        for g, w, name in zip(got, want, ("idx", "val", "xcorr")):
            assert torch.equal(g, w), (L, f, name)
        assert torch.equal(pair_est._smoothed, rows_est._smoothed), (L, f)
        if f == 1:
            assert int(got[0][1]) == 0 and float(got[1][1]) == 0.0


@pytest.mark.parametrize("L", LENGTHS)
def test_all_pairs_vs_oracle(L):
    """All pairs of channels 0..8 of an 11-channel frame, the reversed pairs (3, 1) and (8, 0), the
    pair (4, 4), (0, 1) a second time; channels 9 and 10 in no pair.  Two frames with smoothing."""
    from friture_b200.correlation import PairGccPhat
    C = 11
    pairs = all_pairs(9) + [(3, 1), (8, 0), (4, 4), (0, 1)]
    est = PairGccPhat(L, C, pairs)
    old = [None] * len(pairs)
    for f in range(2):
        x, shifts = planted(C, L, 200 + f)
        idx, val, xc = est.estimate(cuda(x), want_xcorr=True)
        assert xc.shape == (len(pairs), out_len(L))
        idx, val, xcn = idx.cpu().numpy(), val.cpu().numpy(), xc.cpu().numpy()
        sm = est._smoothed.cpu().numpy()
        for p, (i, j) in enumerate(pairs):
            ref = fo.generalized_cross_correlation(x[i].astype(np.float64), x[j].astype(np.float64))
            old[p] = assert_close(idx[p], val[p], xcn[p], ref, old[p], (L, f, i, j))
            assert np.max(np.abs(sm[p] - old[p])) < ABS_TOL, (L, f, i, j)
            if f == 0 and i != j and L % 2 == 0:
                assert int(idx[p]) == (shifts[j] - shifts[i]) % L, (L, i, j)
        # the repeated pair gives the same bits as its first entry
        first = pairs.index((0, 1))
        assert torch.equal(xc[first], xc[-1]) and idx[first] == idx[-1] and val[first] == val[-1]


@pytest.mark.parametrize("L", LENGTHS)
def test_constant_channels_keep_their_pairs_state(L):
    """A pair touching a constant channel gives (0, 0) and leaves its smoothing row untouched, as
    test_gcc_gpu.test_silent_pairs_keep_no_smoothing_state checks for frt_gcc_phat: its first real
    frame is used unsmoothed, the later ones blended."""
    from friture_b200.correlation import PairGccPhat
    C = 5
    pairs = [(0, 1), (1, 2), (0, 2), (3, 4), (2, 3)]
    est = PairGccPhat(L, C, pairs)
    frames = [planted(C, L, 300 + f)[0] for f in range(3)]
    frames[0][1] = 0.25          # frame 0: channel 1 constant, channel 4 all zeros
    frames[0][4] = 0.0
    frames[2][2] = -1.0          # frame 2: channel 2 constant
    ref = lambda x, i, j: fo.generalized_cross_correlation(x[i].astype(np.float64), x[j].astype(np.float64))
    old = [None] * len(pairs)
    for f, x in enumerate(frames):
        before = est._smoothed.clone() if est._smoothed is not None else None
        idx, val, xc = est.estimate(cuda(x), want_xcorr=True)
        idx, val, xcn = idx.cpu().numpy(), val.cpu().numpy(), xc.cpu().numpy()
        for p, (i, j) in enumerate(pairs):
            silent = (f == 0 and (1 in (i, j) or 4 in (i, j))) or (f == 2 and 2 in (i, j))
            if silent:
                assert idx[p] == 0 and val[p] == 0.0 and not xcn[p].any(), (L, f, p)
                if before is not None:
                    assert torch.equal(est._smoothed[p], before[p]), (L, f, p)
                continue
            old[p] = assert_close(idx[p], val[p], xcn[p], ref(x, i, j), old[p], (L, f, p))
            assert np.max(np.abs(est._smoothed[p].cpu().numpy() - old[p])) < ABS_TOL, (L, f, p)


def test_bluestein_groups_all_pairs_of_ten_channels():
    """L = 2 400 000 (100 s), 10 channels, all 45 pairs: the pairs' transforms run in two workspace
    groups.  Every pair against the oracle at 4 096 sampled indices and at its peak."""
    from friture_b200.correlation import PairGccPhat
    L, C = 2400000, 10
    pairs = all_pairs(C)
    x, shifts = planted(C, L, 400)
    est = PairGccPhat(L, C, pairs)
    idx, val, xc = est.estimate(cuda(x), smooth=False, want_xcorr=True)
    idx, val = idx.cpu().numpy(), val.cpu().numpy()
    at = np.sort(np.random.default_rng(401).choice(L, 4096, replace=False))
    for p, (i, j) in enumerate(pairs):
        ref = fo.generalized_cross_correlation(x[i].astype(np.float64), x[j].astype(np.float64))
        got = xc[p, torch.from_numpy(at).cuda()].cpu().numpy()
        assert np.max(np.abs(got - ref[at])) < ABS_TOL, (i, j)
        k = int(np.argmax(np.abs(ref)))
        assert int(idx[p]) == k == (shifts[j] - shifts[i]) % L, (i, j)
        assert abs(float(val[p]) - ref[k]) < ABS_TOL, (i, j)


def test_odd_last_channel_joins_its_bluestein_group():
    """L = 240 000, table (0, 1), (2, 3), (4, 5): a call on 7 channels launches as many kernels as a
    call on 8, because the odd last channel's pack runs in the same workspace group as the others."""
    from friture_b200 import _lib
    from friture_b200.correlation import PairGccPhat
    L = 240000
    h = _lib.Handle(0)
    launches = []
    for C in (7, 8):
        est = PairGccPhat(L, C, [(0, 1), (2, 3), (4, 5)], handle=h)
        x = cuda(planted(C, L, 600)[0])
        est.estimate(x, smooth=False)                 # plans and sets the table
        n = h.launch_count
        est.estimate(x, smooth=False)
        launches.append(h.launch_count - n)
    assert launches[0] == launches[1], launches
    h.close()


@pytest.mark.parametrize("L", [2400, 16800])
def test_refused_calls_then_a_good_one(L):
    """Each refused call returns its code and changes nothing: a following call is still right."""
    from friture_b200 import _lib
    from friture_b200.correlation import PairGccPhat
    h = _lib.Handle(0)
    lib, hh = h._lib, h._h
    C = 4
    x, _ = planted(C, L, 500)
    xd = cuda(x)
    idx = torch.empty(2, dtype=torch.int32, device="cuda")
    val = torch.empty(2, device="cuda")
    stream = _lib.current_stream_ptr()

    def run(stride=L):
        return lib.frt_gcc_phat_pairs(hh, _lib._ptr(xd), stride, None, None, 0, _lib._ptr(idx), _lib._ptr(val),
                                      stream)

    def table(pairs, n_channels=C):
        t = np.ascontiguousarray(pairs, dtype=np.int32)
        return lib.frt_gcc_set_pairs(hh, n_channels, _lib._ptr(t), len(pairs))

    assert run() == _lib.FRT_ESTATE                  # no table, no plan
    assert table([(0, 1), (2, 3)]) == _lib.FRT_OK
    assert run() == _lib.FRT_ESTATE                  # no plan
    assert lib.frt_gcc_plan(hh, L) == _lib.FRT_OK
    assert table([(0, 4), (1, 2)]) == _lib.FRT_EINVAL
    assert table([(0, 1), (-1, 2)]) == _lib.FRT_EINVAL
    assert table([(0, 1)], n_channels=0) == _lib.FRT_EINVAL
    assert run(stride=L - 1) == _lib.FRT_EINVAL
    assert run() == _lib.FRT_OK                      # the table (0, 1), (2, 3) is still in place
    want = PairGccPhat(L, C, [(0, 1), (2, 3)]).estimate(xd, smooth=False)
    torch.cuda.synchronize()
    assert torch.equal(idx, want[0]) and torch.equal(val, want[1])
    assert table([]) == _lib.FRT_OK                  # an empty table: a call does nothing
    idx.fill_(-7)
    assert run(stride=L - 1) == _lib.FRT_EINVAL      # but a short stride is still refused
    assert run() == _lib.FRT_OK
    # frt_gcc_phat with no pairs returns before it checks the stride
    assert lib.frt_gcc_phat(hh, _lib._ptr(xd), _lib._ptr(xd), L - 1, 0, None, None, 0, None, None,
                            stream) == _lib.FRT_OK
    torch.cuda.synchronize()
    assert idx.tolist() == [-7, -7]
    h.close()


# ---------------------------------------------------------------------------------------------
# stream order (INTEGRATION.md, "Streams"), in the manner of test_stream_order_gpu

class TwoTables:
    """Two PairGccPhat on one handle with different tables: each call of one sets its table again."""

    def __init__(self, L, C):
        from friture_b200 import _lib
        from friture_b200.correlation import PairGccPhat
        self.h = _lib.Handle(0)
        self.a = PairGccPhat(L, C, [(0, 1), (2, 1), (3, 3)], handle=self.h)
        self.b = PairGccPhat(L, C, [(1, 0), (0, 2)], handle=self.h)


def rows_apart(C, L, seed):
    return signal((C, L + 3), seed)[:, :L]           # rows L + 3 floats apart


@pytest.mark.parametrize("way", ["current", "explicit"])
@pytest.mark.parametrize("L", [2400, 16800])
def test_pair_calls_in_stream_order(side, L, way):
    from friture_b200.correlation import PairGccPhat
    C = 5

    def est(g, x, kw):
        return g.estimate(x, want_xcorr=True, **kw)

    check(lambda: PairGccPhat(L, C, [(0, 1), (2, 1), (3, 3), (4, 0)]),
          [(est, rows_apart(C, L, 31 + i)) for i in range(3)], way, side,
          warm=lambda g, kw: est(g, rows_apart(C, L, 30), kw))


@pytest.mark.parametrize("way", ["current", "explicit"])
@pytest.mark.parametrize("L", [2400, 16800])
def test_table_switches_wait_for_queued_calls(side, L, way):
    """Two estimators with different tables alternate on one handle: each call sets its table again
    (frt_gcc_set_pairs), which must not change the table under the other's queued call."""
    C = 5

    def run_a(o, x, kw):
        return o.a.estimate(x, want_xcorr=True, **kw)

    def run_b(o, x, kw):
        return o.b.estimate(x, want_xcorr=True, **kw)

    check(lambda: TwoTables(L, C), [(run_a, rows_apart(C, L, 41)), (run_b, rows_apart(C, L, 42)),
                                    (run_a, rows_apart(C, L, 43))],
          way, side, warm=lambda o, kw: (run_a(o, rows_apart(C, L, 44), kw), run_b(o, rows_apart(C, L, 45), kw)))


def test_array_delay_estimator_in_stream_order(side):
    from friture_b200.delay import ArrayDelayEstimator
    C, n = 4, 18432      # 0.5 s range: 6000-sample hops at 12 kHz; four chunks give three frames

    def push(e, x, kw):
        r = e.handle_new_data(x)
        return r, e.delay_ms.copy(), e.Xcorr_extremum.copy(), e.correlation.copy()

    def chunk(seed):
        a = signal((2, n), seed)
        return torch.cat([a, torch.roll(a, 40, dims=1) + 0.05 * signal((2, n), seed + 100)])

    got, _ = check(lambda: ArrayDelayEstimator(C, [(0, 2), (1, 3), (0, 3)], delayrange_s=0.5),
                   [(push, chunk(40 + i)) for i in range(4)], "current", side,
                   warm=lambda e, kw: push(e, chunk(39), kw))
    assert sum(r[0] for r in got) == 3


# ---------------------------------------------------------------------------------------------

@pytest.mark.parametrize("delayrange_s", [0.5, 1.4])
def test_array_estimator_matches_pair_estimator(delayrange_s):
    """Interleaved channels with pairs (2p, 2p+1) publish the same values as DelayEstimator on the
    two channels as separate tensors, chunk by chunk, over chunks that cross several frames."""
    from friture_b200.delay import ArrayDelayEstimator, DelayEstimator
    P, n = 3, 61440
    arr = ArrayDelayEstimator(2 * P, [(2 * p, 2 * p + 1) for p in range(P)], delayrange_s=delayrange_s)
    ref = DelayEstimator(P, delayrange_s=delayrange_s)
    frames = 0
    g = torch.Generator().manual_seed(7)
    for c in range(6):
        x0 = torch.randn(P, n, generator=g)
        x1 = torch.roll(x0, 64 * (c + 1), dims=1) + 0.1 * torch.randn(P, n, generator=g)
        x = torch.stack([x0, x1], dim=1).reshape(2 * P, n)     # rows 2p, 2p+1: the pair's channels
        r = arr.handle_new_data(x.cuda())
        assert ref.handle_new_data(x0.cuda(), x1.cuda()) == r
        frames += r
        for name in ("delay_ms", "distance_m", "correlation", "Xcorr_extremum"):
            a, b = getattr(arr, name), getattr(ref, name)
            assert a.dtype == b.dtype and np.array_equal(a, b), (c, name)
    assert frames >= 3
