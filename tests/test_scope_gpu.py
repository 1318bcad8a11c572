"""GPU: ScopeAnalyzer against oracle/scope.py (itself checked against the unmodified reference widget
and RingBuffer by test_scope_oracle.py) and against tests/golden/scope.npz.

- Every tick's window start is the oracle's exactly; the curves each scope holds after a call are the
  oracle's float64 curve rounded to float32, bit for bit, for one- and two-channel scopes.
- S in {1, 2, 3, 1024} with rows at an odd pitch; buffers of 512, 1, 17 and 4096.
- One tick per call, the whole stream in one call and random cuts give the same bits.
- set_timerange in mid-stream in both directions across 500 ms, with the ring growths that read zeros
  only and zeros and moved samples.
- Edge signals: silence, all negative, a sample exactly at the level, crossings at the first pair and
  only at the last pair, NaN, +Inf and -Inf samples, a scope that never triggers.
- Each call in order on its caller's stream.
"""
import os

import numpy as np
import pytest
import torch

from friture_b200.scope import NOT_DRAWN, ScopeAnalyzer, scope_points, scope_width
from oracle.scope import (GOLDEN_BUFFER, GOLDEN_SCHEDULE, GOLDEN_TICKS, ScopeOracle, golden_stream,
                          place_edge)

pytestmark = pytest.mark.gpu

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "scope.npz")


def signal(S, nch, T, seed):
    """float32 [S, nch, T]: per scope a different mix of tones, noise, DC offsets and silence."""
    rng = np.random.default_rng(seed)
    t = np.arange(T) / 48000.
    f = rng.uniform(20, 3000, (S, nch, 1))
    amp = 10 ** rng.uniform(-3, 0, (S, nch, 1))
    x = amp * np.sin(2 * np.pi * f * t + rng.uniform(0, 6, (S, nch, 1)))
    x += rng.uniform(0, 0.3, (S, nch, 1)) * rng.standard_normal((S, nch, T))
    x += rng.uniform(-0.3, 0.3, (S, nch, 1)) * (rng.random((S, nch, 1)) < 0.3)
    x[rng.random(S) < 0.1] = 0.0
    return np.clip(x, -1, 1).astype(np.float32)


def padded(x):
    """x on the GPU with rows at an odd pitch: [S, n] or [S, 2, n] views of a larger buffer."""
    S, nch, T = x.shape
    buf = torch.full((S, nch, T + 37), float("nan"), device="cuda")
    buf[:, :, :T] = torch.from_numpy(x).cuda()
    v = buf[:, :, :T]
    return v[:, 0] if nch == 1 else v


def cuts_for(R, events, seed=None, per_call=None):
    """Call lengths in ticks covering R ticks with a boundary at every event tick: per_call ticks
    each, or random lengths (seed)."""
    rng = np.random.default_rng(seed)
    stops = sorted(set([k for k in events if 0 < k < R] + [R]))
    out, pos = [], 0
    for stop in stops:
        while pos < stop:
            n = per_call if per_call else int(rng.integers(1, 60))
            n = min(n, stop - pos)
            out.append(n)
            pos += n
    return out


def run_gpu(a, x, buffer, cuts, events=(), after=None):
    """Run x (GPU [S, n] or [S, 2, n]) through `a` in calls of cuts[i] ticks, with set_timerange(v)
    before tick k for (k, v) in events.  Returns the window starts [S, R] and the curves
    (scaled_y, scaled_y2, timerange) on the host after each call (after None) or after the calls that
    end at the ticks in `after`."""
    ev = dict(events)
    starts, curves, tick = [], {}, 0
    for n in cuts:
        if tick in ev:
            a.set_timerange(ev[tick])
        tr = a.handle_new_data(x[..., tick * buffer:(tick + n) * buffer], buffer=buffer)
        assert tr.end_index.tolist() == [(tick + r + 1) * buffer for r in range(n)]
        starts.append(tr.window_start.cpu().numpy())
        tick += n
        if after is None or tick - 1 in after:
            c = a.curve()
            curves[tick - 1] = tuple(None if v is None else v.cpu().numpy() for v in c)
    return np.concatenate(starts, axis=1), curves


def run_oracle(S, nch, x, buffer, R, events=(), at=()):
    """The oracle over R ticks: starts [S, R] and, for each tick in `at`, its held curves."""
    ev = dict(events)
    o = ScopeOracle(S, two_channels=nch == 2, timerange=ev.get(0, 50))
    starts, held = np.zeros((S, R), np.int64), {}
    for k in range(R):
        if k in ev:
            o.set_timerange(ev[k])
        starts[:, k] = o.handle_new_data(x[:, :nch, k * buffer:(k + 1) * buffer])
        if k in at:
            held[k] = list(o.y)
    return starts, held


def check_curves(got, want, nch):
    """got: (scaled_y, scaled_y2, timerange) of the analyzer; want: the oracle's per-scope held curves."""
    y, y2, tr = got
    for s, w in enumerate(want):
        if w is None:
            assert np.isnan(tr[s]), "scope %d never drew" % s
            continue
        t, wy, wy2, wtr = w
        assert tr[s] == wtr
        n = scope_points(wtr)
        assert len(wy) == n
        np.testing.assert_array_equal(y[s, :n], wy.astype(np.float32), err_msg="scope %d" % s)
        if nch == 2:
            np.testing.assert_array_equal(y2[s, :n], wy2.astype(np.float32), err_msg="scope %d ch 1" % s)


def compare(S, nch, x, buffer, cuts, events=(), every_call=True):
    a = ScopeAnalyzer(S, two_channels=nch == 2, timerange=dict(events).get(0, 50))
    R = sum(cuts)
    ends = set(np.cumsum(cuts) - 1)
    starts, curves = run_gpu(a, padded(x), buffer, cuts, events, after=None if every_call else {R - 1})
    want, held = run_oracle(S, nch, x, buffer, R, events, at=ends if every_call else {R - 1})
    np.testing.assert_array_equal(starts, want)
    for k, c in curves.items():
        check_curves(c, held[k], nch)
    return starts, curves


@pytest.mark.parametrize("nch", [1, 2])
@pytest.mark.parametrize("S", [1, 2, 3, 1024])
def test_matches_oracle(S, nch):
    x = signal(S, nch, 96 * 512, seed=S + 10 * nch)
    events = [(0, 50), (40, 10), (70, 123.4)]
    compare(S, nch, x, 512, cuts_for(96, dict(events), per_call=24), events, every_call=S < 1024)


@pytest.mark.parametrize("buffer,events,R", [
    (512, [(0, 50), (60, 700), (90, 20)], 120),
    (1, [(0, 0.3), (700, 2), (1500, 0.1)], 2200),
    (17, [(0, 5), (200, 60), (400, 520), (1800, 3)], 1900),
    (4096, [(0, 50), (10, 10000), (140, 400), (160, 0.1)], 170),
])
def test_buffers(buffer, events, R):
    S, nch = 3, 2
    x = signal(S, nch, R * buffer, seed=buffer)
    compare(S, nch, x, buffer, cuts_for(R, dict(events), seed=buffer), events)


def test_chunkings_identical():
    """One tick per call, the whole stream per timerange in one call, and random cuts: the same bits."""
    S, nch, R = 3, 2, 220
    events = {0: 50, 50: 125, 90: 600, 130: 300, 170: 10000, 200: 40}
    x = padded(signal(S, nch, R * 512, seed=4))
    runs = []
    for cuts in (cuts_for(R, events, per_call=1), cuts_for(R, events, per_call=R), cuts_for(R, events, seed=5)):
        a = ScopeAnalyzer(S, two_channels=True)
        runs.append(run_gpu(a, x, 512, cuts, events.items(), after={R - 1, 129, 169}))
    for starts, curves in runs[1:]:
        np.testing.assert_array_equal(starts, runs[0][0])
        for k in (R - 1, 129, 169):
            for g, w in zip(curves[k], runs[0][1][k]):
                np.testing.assert_array_equal(g, w)


def test_timerange_changes_grow_the_ring():
    """set_timerange across 500 ms both ways; the first 125 ms tick grows the wrapped 10000-sample ring
    so that its window reads zeros and samples moved by 8000 positions, the 600 ms tick grows it again
    with zeros and moved samples, 500 ms and 10 s grow it with zeros only."""
    S, nch, R = 3, 2, 500
    events = [(0, 50), (41, 125), (60, 0.1), (80, 123.4), (110, 600), (150, 300), (190, 500.1), (230, 500),
              (300, 50), (330, 10000), (480, 1000), (490, 2)]
    x = signal(S, nch, R * 512, seed=12)
    a_starts, _ = compare(S, nch, x, 512, cuts_for(R, dict(events), seed=13), events)
    assert (a_starts[:, 110] == 111 * 512 - scope_width(600)).all()


def test_reset():
    S, nch = 2, 1
    x = signal(S, nch, 60 * 512, seed=3)
    a = ScopeAnalyzer(S)
    run_gpu(a, padded(x), 512, [30])
    a.reset()
    starts, curves = run_gpu(a, padded(x), 512, [60])
    want, held = run_oracle(S, nch, x, 512, 60, at={59})
    np.testing.assert_array_equal(starts, want)
    check_curves(curves[59], held[59], nch)


# ---------------------------------------------------------------- edge signals
EDGES = ["silence", "negative", "at_level", "first", "last", "nan", "posinf", "neginf", "noise"]


def test_edge_signals():
    S, R, tick = len(EDGES), 40, 25
    w = scope_width(50)
    x = np.zeros((S, 1, R * 512), np.float32)
    rng = np.random.default_rng(1)
    for s, kind in enumerate(EDGES):
        row = x[s, 0]
        if kind == "negative":
            row[:] = -0.1 - np.abs(rng.standard_normal(row.shape))
        elif kind in ("at_level", "first", "last"):
            row[:] = -0.5
            place_edge(row, tick, w, kind)
        elif kind != "silence":
            row[:] = 0.5 * np.sin(2 * np.pi * 300 * np.arange(row.size) / 48000.)
            v = {"nan": np.nan, "posinf": np.inf, "neginf": -np.inf, "noise": None}[kind]
            if v is not None:
                row[(tick + 1) * 512 - w] = v
    starts, curves = compare(S, 1, x, 512, [7, 1, 17, 15])
    first = (tick + 1) * 512 - 2 * w
    for s, kind in enumerate(EDGES):
        if kind in ("silence", "negative"):
            assert (starts[s] == NOT_DRAWN).all() and np.isnan(curves[R - 1][2][s])
    assert starts[EDGES.index("first"), tick] == first
    assert starts[EDGES.index("last"), tick] == first + w - 2
    assert starts[EDGES.index("at_level"), tick] == first + w // 5 - 1
    assert starts[EDGES.index("nan"), tick] == NOT_DRAWN           # NaN in the window: no trigger
    assert starts[EDGES.index("posinf"), tick] != NOT_DRAWN


def test_golden():
    """The golden stream: window starts equal the reference's, and the kept curves are the reference's
    rounded to float32, with calls cut at the schedule and at the kept curves' ticks.  The curves held
    after ticks 42 and 110, right after the two ring growths whose windows read zeros and moved samples
    (at ticks 41 and 110), are checked against the oracle, whose curve at every tick
    test_scope_oracle.py ties to the reference's float64 bits."""
    g = np.load(GOLDEN)
    x = golden_stream()
    ticks = [int(k) for k in g["curve_ticks"]]
    grown = [42, 110]
    events = dict(GOLDEN_SCHEDULE)
    stops = dict(events)
    for k in ticks + grown:
        stops.setdefault(k + 1, None)
    cuts = cuts_for(GOLDEN_TICKS, stops, seed=2)
    for scopes, nch in (([0, 1, 2], 1), ([3, 4], 2)):
        a = ScopeAnalyzer(len(scopes), two_channels=nch == 2)
        starts, curves = run_gpu(a, padded(x[scopes, :nch]), GOLDEN_BUFFER, cuts, events.items(),
                                 after=set(ticks + grown))
        np.testing.assert_array_equal(starts, g["start"][scopes])
        _, held = run_oracle(len(scopes), nch, x[scopes, :nch], GOLDEN_BUFFER, max(grown) + 1, events.items(),
                             at=set(grown))
        for k in grown:
            check_curves(curves[k], held[k], nch)
        for k in ticks:
            y, y2, tr = curves[k]
            for j, s in enumerate(scopes):
                key = "y_%d_%d" % (k, s)
                if key not in g.files:
                    assert np.isnan(tr[j])
                    continue
                want = g[key]
                n = want.shape[1]
                assert n == scope_points(tr[j])
                np.testing.assert_array_equal(y[j, :n], want[0])
                if nch == 2:
                    np.testing.assert_array_equal(y2[j, :n], want[1])


# ---------------------------------------------------------------- stream order
HOLD_CYCLES = 250_000_000


@pytest.mark.parametrize("way", ["current", "explicit"])
def test_stream_order(way):
    """Each call on the caller's stream, queued behind a spin kernel with NaN-poisoned inputs that are
    filled on that stream, gives the same bits as the same calls run alone.  The handle is made
    before the hold, so every call of the window must return with the held work still queued."""
    S = 3
    x = torch.from_numpy(signal(S, 2, 40 * 512, seed=21)).cuda()
    s = torch.cuda.Stream()

    def calls(a, src, kw, pending=None):
        out = []
        for k in range(4):
            if k == 2:
                a.set_timerange(700)
            if pending is not None:
                pending.append(not s.query())
            out.append(a.handle_new_data(src[..., k * 5120:(k + 1) * 5120], **kw).window_start)
            if pending is not None:
                pending.append(not s.query())
            out.extend(v for v in a.curve(**kw) if v is not None)
        return out

    ref = calls(ScopeAnalyzer(S, two_channels=True), x, {})
    torch.cuda.synchronize()
    a = ScopeAnalyzer(S, two_channels=True)
    a.handle_new_data(torch.zeros(S, 2, 512, device="cuda"))        # the handle, made beforehand
    a.reset()
    buf = torch.full_like(x, float("nan"))
    torch.cuda.synchronize()
    pending = []
    if way == "current":
        with torch.cuda.stream(s):
            torch.cuda._sleep(HOLD_CYCLES)
            buf.copy_(x)
            got = calls(a, buf, {}, pending)
    else:
        with torch.cuda.stream(s):
            torch.cuda._sleep(HOLD_CYCLES)
            buf.copy_(x)
        got = calls(a, buf, {"stream": s.cuda_stream}, pending)
    torch.cuda.synchronize()
    assert all(pending), "a call waited for the held work: %s" % pending
    assert len(got) == len(ref)
    for g, w in zip(got, ref):
        np.testing.assert_array_equal(g.cpu().numpy(), w.cpu().numpy())
