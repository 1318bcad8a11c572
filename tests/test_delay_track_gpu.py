"""GPU: every frame a delay-estimator call covers in one pass (frt_gcc_phat_frames,
frt_gcc_phat_pairs_frames, GccPhat / PairGccPhat.estimate_frames, the estimators' ``track``).

* The same bits as one frt_gcc_phat / frt_gcc_phat_pairs call per frame, in idx, val and the final
  smoothing state, on both routes, with all three have_prev modes on frame 0, silent frames and a pair
  silent from the start; std against numpy.std of the per-frame route's smoothed rows.
* The same track rows however the stream is cut into calls, and however the frames fall into groups.
* DelayEstimator and ArrayDelayEstimator against the widget's loop restated with the oracle, frame by
  frame.
* Refused calls, and the stream order of the new calls (the method of test_stream_order_gpu.py).
"""
import ctypes
import time

import numpy as np
import pytest
import torch

from friture_b200 import _lib, filter_data
from friture_b200.correlation import GccPhat, PairGccPhat
from friture_b200.delay import ArrayDelayEstimator, DelayEstimator

pytestmark = pytest.mark.gpu

SMEM_LENGTHS = [2400, 24000]
LONG_LENGTHS = [16800, 55199]


def n_sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def pair_counts():
    return [1, 3, 2 * n_sms() + 5]


def vp(t, offset=0):
    """Pointer to element `offset` of a float32 / int32 tensor."""
    return ctypes.c_void_p(t.data_ptr() + 4 * offset)


def planted(P, T, hop, seed):
    """[P, T] rows d0, d1 on the GPU: noise, d1 = d0 delayed by an integer that changes every three
    hops, plus a little noise.  Pair 1 (if any) has d1 constant over [hop, hop + L) of frame 1 only
    (set by the caller); the last pair's d0 is constant for its first frames (set by the caller)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    base = torch.randn((P, T + 400), generator=g, device="cuda")
    t = torch.arange(T, device="cuda")
    shift = 7 + 13 * ((t // (3 * hop)) % 5)                    # 7, 20, 33, 46, 59 samples
    d0 = base[:, 200:200 + T].contiguous()
    d1 = base[:, 200 - shift + t] + 0.05 * torch.randn((P, T), generator=g, device="cuda")
    return d0, d1.contiguous()


def make_silences(d0, d1, L, hop, F):
    P = d0.shape[0]
    if P >= 2 and F >= 2:
        d1[1, hop:hop + L] = 0.25                              # pair 1: frame 1 silent on one channel
    if P >= 3 and F >= 4:
        d1[2, 3 * hop:3 * hop + L] = -1.0                      # pair 2: frame 3 silent
    d0[P - 1, :min(d0.shape[1], 2 * hop + L)] = 0.5            # the last pair: frames 0..2 silent


def initial_state(P, Lr, mode, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    sm = torch.randn((P, Lr), generator=g, device="cuda") * 1e-3
    if mode == 2:
        sm[::2, 0] = float("nan")                              # every other pair: "no previous" yet
    return sm


def per_frame(h, d0, d1, stride, hop, F, P, sm, mode, sel):
    """F frt_gcc_phat calls, frame 0 with have_prev = mode, later ones 2.  Returns idx, val [F, P],
    the final state and, per frame, the smoothed rows of the pairs `sel` in float64."""
    idx = torch.empty((F, P), dtype=torch.int32, device="cuda")
    val = torch.empty((F, P), dtype=torch.float32, device="cuda")
    rows = []
    for f in range(F):
        h.call("frt_gcc_phat", vp(d0, f * hop), vp(d1, f * hop), stride, P, None, vp(sm), mode if f == 0 else 2,
               vp(idx, f * P), vp(val, f * P), _lib.current_stream_ptr())
        rows.append(sm[sel].double().cpu().numpy())
    return idx, val, sm, rows


def frames_call(h, d0, d1, stride, hop, F, P, sm, mode):
    idx = torch.empty((F, P), dtype=torch.int32, device="cuda")
    val = torch.empty((F, P), dtype=torch.float32, device="cuda")
    std = torch.empty((F, P), dtype=torch.float64, device="cuda")
    h.call("frt_gcc_phat_frames", vp(d0), vp(d1), stride, hop, F, P, vp(sm), mode, vp(idx), vp(val), vp(std),
           _lib.current_stream_ptr())
    return idx, val, std


def check_std(std, idx, val, rows, sel):
    std = std.cpu().numpy()
    silent = ((idx == 0) & (val == 0)).cpu().numpy()
    for f, r in enumerate(rows):
        for k, p in enumerate(sel):
            if silent[f, p]:
                assert std[f, p] == 0.0
            else:
                want = np.std(r[k])
                assert abs(std[f, p] - want) <= 1e-12 * want, (f, p, std[f, p], want)


@pytest.mark.parametrize("L", SMEM_LENGTHS + LONG_LENGTHS)
def test_frames_match_per_frame(L):
    from friture_b200._lib import default_handle
    h = default_handle()
    Lr = L - (L & 1)
    h.call("frt_gcc_plan", L)
    for P in pair_counts():
        hop = L // 2 if P <= 3 else max(1, L // 16)
        for F, mode in ((1, 0), (1, 1), (7, 2), (7, 0), (64, 1), (64, 2), (64, 0)):
            T = (F - 1) * hop + L + 5
            d0, d1 = planted(P, T, hop, seed=L + 7 * P + F)
            make_silences(d0, d1, L, hop, F)
            sel = list(range(P)) if P <= 3 else [0, 1, 2, P - 1]
            sm0 = initial_state(P, Lr, mode, seed=F)
            ri, rv, rs, rows = per_frame(h, d0, d1, T, hop, F, P, sm0.clone(), mode, sel)
            sm = sm0.clone()
            gi, gv, gs = frames_call(h, d0, d1, T, hop, F, P, sm, mode)
            where = "L=%d P=%d F=%d have_prev=%d" % (L, P, F, mode)
            assert torch.equal(gi, ri), where
            assert torch.equal(gv.view(torch.int32), rv.view(torch.int32)), where
            assert torch.equal(sm.view(torch.int32), rs.view(torch.int32)), where
            check_std(gs, gi, gv, rows, sel)
            # the planted delays are found where both inputs are live
            if P <= 3 and F == 64:
                delay = gi[:, 0].cpu().numpy()
                assert np.isin(delay[8:], [7, 20, 33, 46, 59]).mean() > 0.9, where


@pytest.mark.parametrize("L", SMEM_LENGTHS + LONG_LENGTHS)
def test_pairs_frames(L):
    """All pairs of M = 5 channels (an odd last channel) against per-frame PairGccPhat.estimate; the
    table (0,1), (2,3) against GccPhat.estimate_frames on the even and odd rows."""
    M, F = 5, 9
    hop = L // 2
    T = (F - 1) * hop + L + 3
    g = torch.Generator(device="cuda").manual_seed(L)
    x = torch.randn((M, T), generator=g, device="cuda")
    x[3, hop:hop + L] = 1.0                                    # channel 3 silent in frame 1
    x[4, :L] = 0.0                                             # channel 4 silent in frame 0
    pairs = [(i, j) for i in range(M) for j in range(M) if i < j]
    ref = PairGccPhat(L, M, pairs)
    got = PairGccPhat(L, M, pairs)
    want_i, want_v = [], []
    for f in range(F):
        i, v, _ = ref.estimate(x[:, f * hop:f * hop + L])
        want_i.append(i)
        want_v.append(v)
    gi, gv, gs = got.estimate_frames(x, hop, F)
    assert torch.equal(gi, torch.stack(want_i))
    assert torch.equal(gv.view(torch.int32), torch.stack(want_v).view(torch.int32))
    assert torch.equal(got._smoothed.view(torch.int32), ref._smoothed.view(torch.int32))
    # a second call continues the smoothing
    x2 = torch.randn((M, T), generator=g, device="cuda")
    for f in range(3):
        ref.estimate(x2[:, f * hop:f * hop + L])
    got.estimate_frames(x2, hop, 3)
    assert torch.equal(got._smoothed.view(torch.int32), ref._smoothed.view(torch.int32))

    table = PairGccPhat(L, M, [(0, 1), (2, 3)])
    single = GccPhat(L)
    ti, tv, ts = table.estimate_frames(x, hop, F)
    si, sv, ss = single.estimate_frames(x[0:4:2], x[1:4:2], hop, F)
    assert torch.equal(ti, si) and torch.equal(tv.view(torch.int32), sv.view(torch.int32))
    assert torch.equal(ts.view(torch.int64), ss.view(torch.int64))
    assert torch.equal(table._smoothed.view(torch.int32), single._smoothed.view(torch.int32))


def test_frame_groups():
    """Enough pairs x frames to split the call into several frame groups: the same bits as two calls
    cut elsewhere."""
    from friture_b200._lib import default_handle
    h = default_handle()
    L, P, hop, F = 24000, 2 * n_sms() + 5, 240, 120           # ~26 MB of workspace a frame: 2 groups
    h.call("frt_gcc_plan", L)
    T = (F - 1) * hop + L
    d0, d1 = planted(P, T, hop, seed=5)
    make_silences(d0, d1, L, hop, F)
    sm0 = initial_state(P, L, 0, seed=1)
    sm_a = sm0.clone()
    ia, va, sa = frames_call(h, d0, d1, T, hop, F, P, sm_a, 0)
    sm_b = sm0.clone()
    cut = 37
    ib0, vb0, sb0 = frames_call(h, d0, d1, T, hop, cut, P, sm_b, 0)
    ib1, vb1, sb1 = frames_call(h, d0[:, cut * hop:], d1[:, cut * hop:], T, hop, F - cut, P, sm_b, 2)
    assert torch.equal(ia, torch.cat([ib0, ib1]))
    assert torch.equal(va.view(torch.int32), torch.cat([vb0, vb1]).view(torch.int32))
    assert torch.equal(sa.view(torch.int64), torch.cat([sb0, sb1]).view(torch.int64))
    assert torch.equal(sm_a.view(torch.int32), sm_b.view(torch.int32))


def stereo(n, seed, fs=48000, shifts=((0.0, 0.037), (4.0, -0.012))):
    """Two 48 kHz channels, the second lagging the first by shifts[k][1] s from shifts[k][0] s on."""
    rng = np.random.default_rng(seed)
    base = rng.standard_normal(n + 2 * fs) * 0.1
    t = np.arange(n)
    lag = np.zeros(n, dtype=np.int64)
    for t0, s in shifts:
        lag[t >= int(t0 * fs)] = int(round(s * fs))
    x0 = base[fs:fs + n]
    x1 = base[fs - lag + t] + 0.01 * rng.standard_normal(n)
    return x0.astype(np.float32), x1.astype(np.float32)


def feed(est, chunks, *xs):
    rows = []
    for p in range(0, xs[0].shape[1], chunks):
        if len(xs) == 1:
            r = est.handle_new_data(xs[0][:, p:p + chunks])
        else:
            r = est.handle_new_data(xs[0][:, p:p + chunks], xs[1][:, p:p + chunks])
        assert est.track.end_index.shape[0] == r
        rows.append(est.track)
    return [np.concatenate([getattr(t, k) for t in rows]) for k in rows[0]._fields]


def test_cut_invariance():
    n = 48000 * 6
    x0, x1 = stereo(n, seed=3)
    P = 2
    a = torch.from_numpy(np.tile(x0, (P, 1))).cuda()
    b = torch.from_numpy(np.tile(x1, (P, 1))).cuda()
    want = feed(DelayEstimator(P), n, a, b)
    assert want[0].shape[0] >= 5
    for chunk in (256, 1024, 12288):
        got = feed(DelayEstimator(P), chunk, a, b)
        for w, g_ in zip(want, got):
            assert np.array_equal(w, g_), chunk
    x = torch.stack([a[0], b[0], a[0] * 0.5])
    want = feed(ArrayDelayEstimator(3, [(0, 1), (2, 1)]), n, x)
    for chunk in (256, 1024, 12288):
        got = feed(ArrayDelayEstimator(3, [(0, 1), (2, 1)]), chunk, x)
        for w, g_ in zip(want, got):
            assert np.array_equal(w, g_), chunk


def widget_track(x0, x1, delayrange_s, chunk):
    """The widget's loop (delay_estimator.py:87-176) restated with the oracle for one pair: per frame
    (end index, delay ms, distance m, correlation before int(), Xcorr extremum)."""
    from oracle import friture_oracle as fo
    bdec, adec, _ = filter_data.decimator()
    z0 = [np.zeros(12), np.zeros(12)]
    z1 = [np.zeros(12), np.zeros(12)]
    L = int(2 * delayrange_s * 12000)
    hop = int(0.5 * L)
    hist0, hist1 = np.zeros(L), np.zeros(L)
    old_index, offset, old_xc, out = 0, 0, None, []
    for p in range(0, len(x0), chunk):
        d0, z0 = fo.decimate_multiple(2, bdec, adec, x0[p:p + chunk], z0)
        d1, z1 = fo.decimate_multiple(2, bdec, adec, x1[p:p + chunk], z1)
        hist0, hist1 = np.concatenate([hist0, d0]), np.concatenate([hist1, d1])
        offset += len(d0)
        for _ in range(int((offset - old_index) / hop)):
            old_index += hop
            a, b = hist0[old_index:old_index + L], hist1[old_index:old_index + L]
            if np.std(a) == 0 or np.std(b) == 0:
                out.append((old_index, 0.0, 0.0, 0.0, 0.0))
                continue
            xc = fo.generalized_cross_correlation(a, b)
            i, v, old_xc = fo.delay_peak(xc, old_xc)
            std = np.std(old_xc)
            norm = abs(v) / (3 * std) if std > 0 else 0.0
            d = 1e3 * i / 12000.0
            time_ = 2 * delayrange_s
            d = d - 1e3 * time_ if d > 1e3 * time_ / 2 else d
            x = (norm > 1.) * (norm - 1.)
            x = (0.12 * x) ** 3
            out.append((old_index, d, d * 1e-3 * 340., (x / (1. + x)) * 100, v))
    return np.array(out)


def compare_widget(rows, ref, p):
    end, delay, dist, corr, ext = rows
    assert end.shape[0] == ref.shape[0] > 5
    # the framer's old_index is the widget's, whose frames end at old_index + L: both count hops
    assert np.array_equal(end, ref[:, 0].astype(np.int64))
    assert np.allclose(delay[:, p], ref[:, 1], atol=1e-9)
    assert np.allclose(dist[:, p], ref[:, 2], atol=1e-9)
    assert np.allclose(ext[:, p], ref[:, 4], atol=1e-4)
    near = np.abs(ref[:, 3] - np.round(ref[:, 3])) < 1e-9
    assert np.array_equal(corr[~near, p], ref[~near, 3].astype(int))


def test_estimators_against_widget():
    chunk, rng_s = 512, 0.5
    n = chunk * (48000 * 9 // chunk)
    x0, x1 = stereo(n, seed=11)
    ref = widget_track(x0, x1, rng_s, chunk)
    planted_ms = np.where(ref[:, 0] / 12000.0 < 4.0, 37.0, -12.0)
    # frames whose window and smoothing history lie after the change recover the new delay, and the
    # frames before it the old one
    settled = (ref[:, 0] / 12000.0 < 4.0) | (ref[:, 0] / 12000.0 > 4.0 + 5 * rng_s)
    assert np.all(np.abs(ref[settled, 1] - planted_ms[settled]) < 0.2)
    P = 2
    est = DelayEstimator(P, delayrange_s=rng_s)
    rows = feed(est, chunk, torch.from_numpy(np.tile(x0, (P, 1))).cuda(),
                torch.from_numpy(np.tile(x1, (P, 1))).cuda())
    for p in range(P):
        compare_widget(rows, ref, p)
    assert np.all(np.abs(rows[1][settled, 0] - planted_ms[settled]) < 0.2)
    arr = ArrayDelayEstimator(3, [(0, 1), (1, 0), (2, 1)], delayrange_s=rng_s)
    x = torch.from_numpy(np.stack([x0, x1, x0])).cuda()
    rows_a = feed(arr, chunk, x)
    compare_widget(rows_a, ref, 0)
    compare_widget(rows_a, ref, 2)
    ref_rev = widget_track(x1, x0, rng_s, chunk)
    compare_widget(rows_a, ref_rev, 1)
    assert np.array_equal(est.delay_ms, rows[1][-1]) and np.array_equal(arr.correlation, rows_a[3][-1])


def test_refusals_keep_the_handle_and_state():
    from friture_b200._lib import FrtError, FrtValueError, Handle
    L, P, F, hop = 2400, 3, 5, 1200
    T = (F - 1) * hop + L
    d0, d1 = planted(P, T, hop, seed=2)
    h = Handle(0)
    sm = torch.zeros((P, L), device="cuda")
    out_i = torch.empty((F, P), dtype=torch.int32, device="cuda")
    out_v = torch.empty((F, P), dtype=torch.float32, device="cuda")
    out_s = torch.empty((F, P), dtype=torch.float64, device="cuda")
    st = _lib.current_stream_ptr()
    args = lambda **k: [k.get("d0", vp(d0)), vp(d1), k.get("stride", T), k.get("fs", hop), k.get("F", F), P,  # noqa: E731
                        k.get("sm", vp(sm)), k.get("hp", 0), vp(out_i), vp(out_v), k.get("std", vp(out_s)), st]
    with pytest.raises(FrtError) as e:
        h.call("frt_gcc_phat_frames", *args())                 # no plan yet
    assert e.value.code == _lib.FRT_ESTATE
    h.call("frt_gcc_plan", L)
    for bad in (dict(F=-1), dict(fs=0), dict(sm=None), dict(std=None), dict(hp=3), dict(stride=L - 1),
                dict(d0=None)):
        with pytest.raises(FrtValueError):
            h.call("frt_gcc_phat_frames", *args(**bad))
    h.call("frt_gcc_phat_frames", *args(F=0, sm=None, std=None))   # nothing to do
    h.call("frt_gcc_phat_frames", *args(F=1, fs=0))                  # one frame needs no frame stride
    sm.zero_()
    h.call("frt_gcc_phat_frames", *args())
    want = GccPhat(L).estimate_frames(d0, d1, hop, F)
    assert torch.equal(out_i, want[0]) and torch.equal(out_v, want[1]) and torch.equal(out_s, want[2])
    # the pairs variant: no table, then a table, a bad call, and a good one continuing the state
    with pytest.raises(FrtError) as e:
        h.call("frt_gcc_phat_pairs_frames", vp(d0), T, hop, F, vp(sm), 2, vp(out_i), vp(out_v), vp(out_s), st)
    assert e.value.code == _lib.FRT_ESTATE
    est = PairGccPhat(L, P, [(0, 1), (1, 2), (2, 0)])
    ref = PairGccPhat(L, P, [(0, 1), (1, 2), (2, 0)])
    est.estimate_frames(d0, hop, 2)
    ref.estimate_frames(d0, hop, 2)
    with pytest.raises(ValueError):
        est.estimate_frames(d0, hop, F + 1)                    # rows too short
    with pytest.raises(FrtValueError):
        est.handle.call("frt_gcc_phat_pairs_frames", vp(d0), T, 0, 3, vp(est._smoothed), 2, vp(out_i), vp(out_v),
                        vp(out_s), st)
    a = est.estimate_frames(d0[:, hop:], hop, 3)
    b = ref.estimate_frames(d0[:, hop:], hop, 3)
    assert all(torch.equal(u, v) for u, v in zip(a, b))
    assert torch.equal(est._smoothed, ref._smoothed)


HOLD_CYCLES = 250_000_000
WAITED_S = 0.05


@pytest.mark.parametrize("way", ["current", "explicit"])
@pytest.mark.parametrize("L", [24000, 16800])
def test_stream_order(L, way):
    """The calls queued behind a busy side stream, on inputs that are NaN until a copy on that stream
    lands, give the bits of the same calls run alone."""
    s = torch.cuda.Stream()
    P, F, hop = 3, 6, L // 2
    T = (F - 1) * hop + L
    d0, d1 = planted(P, T, hop, seed=L)
    x = torch.cat([d0, d1[:1]])

    def run(a, b, xx, kw):
        # no torch work of the test's own here: it would run on the current stream, not the call's
        g = GccPhat(L)
        pg = PairGccPhat(L, 4, [(0, 1), (3, 0), (2, 1)])
        out = [g.estimate_frames(a, b, hop, F, **kw), pg.estimate_frames(xx, hop, F, **kw)]
        out.append(g.estimate_frames(a[:, hop:], b[:, hop:], hop, 2, **kw))
        return [t for o in out for t in o] + [g._smoothed, pg._smoothed]

    want = run(d0, d1, x, {})
    torch.cuda.synchronize()
    bufs = [torch.full_like(t, float("nan")) for t in (d0, d1, x)]
    torch.cuda.synchronize()
    ctx = torch.cuda.stream(s) if way == "current" else None
    kw = {} if way == "current" else {"stream": s.cuda_stream}
    if ctx is not None:
        ctx.__enter__()
    try:
        with torch.cuda.stream(s):
            torch.cuda._sleep(HOLD_CYCLES)
            for dst, src in zip(bufs, (d0, d1, x)):
                dst.copy_(src)
        t0 = time.perf_counter()
        got = run(*bufs, kw)
        pending = not s.query()
        waited = time.perf_counter() - t0 >= WAITED_S
    finally:
        if ctx is not None:
            ctx.__exit__(None, None, None)
    torch.cuda.synchronize()
    for g_, w in zip(got, want):
        assert torch.equal(g_.view(torch.int32) if g_.dtype == torch.float32 else g_,
                           w.view(torch.int32) if w.dtype == torch.float32 else w)
    assert pending or waited, "the calls neither left work queued nor waited: the hold ran out early"
