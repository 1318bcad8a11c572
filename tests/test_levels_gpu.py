"""GPU: LevelsAnalyzer and LongLevelsAnalyzer against oracle/levels.py on the same float32 input.

- Meter: the peak state old_max, the ballistic hold counters and decay factors are the same bits;
  level_rms, level_max, peak_iec and the carried ballistic peak within 1e-12 relative (the weighted
  sum of x^2 is not NumPy's dot product order, and log10 is not NumPy's).  The ballistic recurrence
  itself is checked bit for bit: replayed in NumPy on the GPU's own level_rms and level_max, it gives
  the GPU's peak_iec, carried peak, hold counters and decay factors exactly.
- Long-term levels: the linear level is the same bits, its dB within 1e-12 relative; the curve is
  the oracle's to float32 rounding (the history is stored as float32 dB).
- C in {1, 2, 3, 1024}, rows padded to an odd stride; every chunking gives the same bits; reset and
  every setter mid-stream; silence until both meter states underflow and the long-term level reaches
  its 1e-150 floor; NaN samples, which propagate as in NumPy; each call in order on its caller's
  stream.
"""
import numpy as np
import pytest
import torch

from friture_b200.levels import LevelsAnalyzer, LongLevelsAnalyzer
from oracle.levels import LevelsOracle, LongLevelsOracle, db_to_iec

pytestmark = pytest.mark.gpu

CHANNELS = [1, 2, 3, 1024]


def signal(C, T, seed):
    """float32 [C, T]: per channel a different mix of noise, a tone, DC, impulses and silence."""
    rng = np.random.default_rng(seed)
    t = np.arange(T) / 48000.
    amp = 10 ** rng.uniform(-4, 0, (C, 1))
    x = amp * rng.standard_normal((C, T)) * (0.6 + 0.4 * np.sin(2 * np.pi * t / rng.uniform(0.05, 2, (C, 1))))
    tone = rng.random(C) < 0.3
    x[tone] = np.sin(2 * np.pi * rng.uniform(50, 5000, (tone.sum(), 1)) * t)
    dc = rng.random(C) < 0.1
    x[dc, : T // 3] = rng.uniform(-1, 1, (dc.sum(), 1))
    quiet = rng.random(C) < 0.3
    x[quiet, T // 2:] *= 1e-4
    for c in np.flatnonzero(rng.random(C) < 0.2):
        x[c, rng.integers(0, T, 3)] = rng.uniform(-1, 1, 3)
    return np.clip(x, -1, 1).astype(np.float32)


def padded(x):
    """x on the GPU with rows at an odd pitch (not 16-byte aligned)."""
    C, T = x.shape
    buf = torch.full((C, T + 37), float("nan"), device="cuda")
    buf[:, :T] = torch.from_numpy(x).cuda()
    return buf[:, :T]


def rel(got, want):
    got, want = np.asarray(got), np.asarray(want)
    same = (np.isinf(want) & (got == want)) | (np.isnan(want) & np.isnan(got))
    with np.errstate(invalid="ignore"):
        d = np.where(same, 0.0, np.abs(got - want) / np.maximum(np.abs(want), 1e-300))
    return float(np.max(d)) if d.size else 0.0


# ---------------------------------------------------------------- meter
def run_meter(a, x, buffer, per_call):
    outs = []
    R = x.shape[1] // buffer
    for r0 in range(0, R, per_call):
        t = a.handle_new_data(x[:, r0 * buffer:min(R, r0 + per_call) * buffer], buffer=buffer)
        outs.append([v.cpu().numpy() for v in t])
    return [np.concatenate([o[i] for o in outs], axis=1) for i in range(3)]


def run_meter_oracle(o, x, buffer):
    xs = x.astype(np.float64)
    res = [o.handle_new_data(xs[:, r * buffer:(r + 1) * buffer]) for r in range(x.shape[1] // buffer)]
    return [np.stack([r[i] for r in res], axis=1) for i in range(3)]


def replay_ballistic(level_rms, level_max):
    """BallisticPeak from its initial state on dB_to_IEC(max(level_max, level_rms)) of the given
    levels [C, R]: the IEC peak after each buffer and the final state."""
    o = LevelsOracle(level_rms.shape[0])
    peaks = np.empty_like(level_rms)
    for r in range(level_rms.shape[1]):
        lr, lm = level_rms[:, r], level_max[:, r]
        o.step_peak(db_to_iec(np.where(lr > lm, lr, lm)))
        peaks[:, r] = o.peak
    return peaks, o.state()


def check_meter(got, want, gs, ws):
    """got / want: (level_rms, level_max, peak_iec) [C, R] of a run from the initial state; gs / ws
    the states after it."""
    assert rel(got[0], want[0]) < 1e-12, "level_rms"
    assert rel(got[1], want[1]) < 1e-12, "level_max"
    assert rel(got[2], want[2]) < 1e-12, "peak_iec"
    np.testing.assert_array_equal(gs["old_max"], ws["old_max"])
    np.testing.assert_array_equal(gs["hold"], ws["hold"])
    np.testing.assert_array_equal(gs["decay"], ws["decay"])
    assert rel(gs["old_rms"], ws["old_rms"]) < 1e-12
    assert rel(gs["peak_iec"], ws["peak_iec"]) < 1e-12
    # the recurrence is the widget's bit for bit on the levels the GPU computed
    peaks, rs = replay_ballistic(got[0], got[1])
    np.testing.assert_array_equal(got[2], peaks)
    np.testing.assert_array_equal(gs["peak_iec"], got[2][:, -1])
    for k in ("peak_iec", "hold", "decay"):
        np.testing.assert_array_equal(gs[k], rs[k], err_msg=k)


@pytest.mark.parametrize("C", CHANNELS)
def test_meter_matches_oracle(C):
    x = signal(C, 96 * 512, seed=C)
    a, o = LevelsAnalyzer(C), LevelsOracle(C)
    got = run_meter(a, padded(x), 512, 40)
    want = run_meter_oracle(o, x, 512)
    check_meter(got, want, a.state(), o.state())


@pytest.mark.parametrize("rt", [0.025, 0.125, 1.0])
@pytest.mark.parametrize("buffer", [1, 100, 512, 4096])
def test_meter_settings(rt, buffer):
    C = 3
    x = signal(C, 48 * 4096, seed=int(rt * 1000) + buffer)
    a, o = LevelsAnalyzer(C, response_time=rt), LevelsOracle(C, response_time=rt)
    T = (x.shape[1] // buffer) * buffer
    if T // buffer > 6000:
        T = 6000 * buffer
    x = x[:, :T]
    got = run_meter(a, padded(x), buffer, 1000)
    want = run_meter_oracle(o, x, buffer)
    check_meter(got, want, a.state(), o.state())


@pytest.mark.parametrize("C", [2, 1024])
def test_meter_chunkings_identical(C):
    x = padded(signal(C, 70 * 512, seed=5))
    runs = [run_meter(LevelsAnalyzer(C), x, 512, k) for k in (1, 3, 32, 33, 70)]
    for r in runs[1:]:
        for g, w in zip(r, runs[0]):
            np.testing.assert_array_equal(g, w)


def test_meter_buffer_change_and_reset():
    C = 3
    x = signal(C, 40 * 512, seed=11)
    a, o = LevelsAnalyzer(C), LevelsOracle(C)
    xd = padded(x)
    got, want = [], []
    for lo, hi, buffer in [(0, 5120, 512), (5120, 8320, 100), (8320, 10240, 1920)]:
        got.append([v.cpu().numpy() for v in a.handle_new_data(xd[:, lo:hi], buffer=buffer)])
        want.append(run_meter_oracle(o, x[:, lo:hi], buffer))
    check_meter([np.concatenate([g[i] for g in got], 1) for i in range(3)],
                [np.concatenate([w[i] for w in want], 1) for i in range(3)], a.state(), o.state())
    a.reset()
    o = LevelsOracle(C)
    got = run_meter(a, xd[:, 10240:], 512, 7)
    want = run_meter_oracle(o, x[:, 10240:], 512)
    check_meter(got, want, a.state(), o.state())


def test_meter_underflow():
    """Silence until both meter states underflow.  At rt = 0.025 s and 4096-sample buffers old_rms falls
    by (1 - alpha)^4096 = 0.028 per buffer and reaches 0: level_rms is -inf.  old_max falls by
    1 - alpha2 = 0.59 per buffer, which rounds the smallest subnormal, 5e-324, back to itself: it stays
    there (level_max -6467 dB), as it does in the widget's arithmetic.  The IEC peak falls to 0."""
    C = 2
    buffer = 4096
    x = np.zeros((C, 1700 * buffer), np.float32)
    x[:, :4 * buffer] = signal(C, 4 * buffer, seed=3)
    a, o = LevelsAnalyzer(C, response_time=0.025), LevelsOracle(C, response_time=0.025)
    got = run_meter(a, padded(x), buffer, 600)
    want = run_meter_oracle(o, x, buffer)
    s = a.state()
    tiny = np.nextafter(0.0, 1.0)
    assert (s["old_rms"] == 0).all() and (s["old_max"] == tiny).all()
    assert np.isneginf(got[0][:, -1]).all() and (got[2][:, -1] == 0).all()
    check_meter(got, want, s, o.state())


# ---------------------------------------------------------------- long-term levels
def run_long(a, x, chunks, events=()):
    """Push x in chunks (sizes), applying events {chunk number: (setter, value)} before that chunk.
    Returns (end_index, level, db) of every block and the curve after every call that made one."""
    ev = dict(events)
    ends, lv, db, curves = [], [], [], []
    pos = 0
    for i, n in enumerate(chunks):
        if i in ev:
            name, value = ev[i]
            getattr(a, name)(*(() if value is None else (value,)))
        tr = a.handle_new_data(x[:, pos:pos + n])
        pos += n
        if isinstance(a, LongLevelsAnalyzer):
            e, l_, d = tr.end_index, tr.level.cpu().numpy(), tr.level_rms.cpu().numpy()
            if len(e):
                t, y = a.curve()
                curves.append((t, y.cpu().numpy()))
        else:
            e, l_, d = tr
            if len(e):
                curves.append(a.curve)
        ends.append(e)
        lv.append(l_)
        db.append(d)
    return np.concatenate(ends), np.concatenate(lv, axis=1), np.concatenate(db, axis=1), curves


def check_long(got, want, curves=True):
    np.testing.assert_array_equal(got[0], want[0])
    np.testing.assert_array_equal(got[1], want[1])
    assert rel(got[2], want[2]) < 1e-12
    if curves:
        assert len(got[3]) == len(want[3])
        for (tg, yg), (tw, yw) in zip(got[3], want[3]):
            np.testing.assert_array_equal(tg, tw)
            np.testing.assert_allclose(yg, yw, rtol=0, atol=2e-6)


def chunk_sizes(T, seed, hi=30000):
    rng = np.random.default_rng(seed)
    out = []
    while sum(out) < T:
        out.append(int(min(rng.integers(1, hi), T - sum(out))))
    return out


@pytest.mark.parametrize("C", CHANNELS)
def test_long_levels_match_oracle(C):
    T = 200_000
    x = signal(C, T, seed=100 + C)
    chunks = chunk_sizes(T, C)
    got = run_long(LongLevelsAnalyzer(C, response_time=1, duration=5), padded(x), chunks)
    want = run_long(LongLevelsOracle(C, response_time=1, duration=5), x, chunks)
    check_long(got, want)


@pytest.mark.parametrize("rt", list(range(1, 21)))
def test_long_levels_every_response_time(rt):
    C = 3
    needed = 2 ** int(np.floor(np.log2(rt * 480)))
    T = 24 * needed + 1000
    x = signal(C, T, seed=rt)
    chunks = chunk_sizes(T, rt, hi=3 * needed)
    got = run_long(LongLevelsAnalyzer(C, response_time=rt, duration=5), padded(x), chunks)
    want = run_long(LongLevelsOracle(C, response_time=rt, duration=5), x, chunks)
    check_long(got, want)


@pytest.mark.parametrize("C", [2, 1024])
def test_long_levels_chunkings_identical(C):
    T = 120 * 512
    x = padded(signal(C, T, seed=9))
    runs = [run_long(LongLevelsAnalyzer(C, response_time=1, duration=5), x, chunks)
            for chunks in ([512] * 120, [T], chunk_sizes(T, 4, hi=2000), [1, 255, 256, 257] + [T - 769])]
    for r in runs[1:]:
        for i in range(3):
            np.testing.assert_array_equal(r[i], runs[0][i])
        np.testing.assert_array_equal(r[3][-1][1], runs[0][3][-1][1])


def test_long_levels_setters_and_reset():
    """Response time, range and duration changed mid-stream; a duration increase grows the level
    ring after it has wrapped (10000 slots at first), the widget's ring growth moving what it keeps."""
    C = 3
    T = 3_300_000                   # 11 000 blocks before the duration increase: the ring has wrapped
    x = signal(C, T, seed=77)
    chunks = chunk_sizes(T, 8, hi=60000)
    events = {2: ("setresptime", 3), 8: ("setmin", -95), 12: ("setmax", -5), 15: ("setresptime", 1),
              20: ("setduration", 7), 24: ("setresptime", 20), 27: ("setresptime", 1),
              len(chunks) - 5: ("setduration", 60), len(chunks) - 2: ("setduration", 3600)}
    a = LongLevelsAnalyzer(C, response_time=1, duration=5)
    got = run_long(a, padded(x), chunks, events)
    want = run_long(LongLevelsOracle(C, response_time=1, duration=5), x, chunks, events)
    assert len(got[0]) > 10000 and a._ring_len == int(1.5 * 3600 * 187.5)
    check_long(got, want)
    a.reset()
    o = LongLevelsOracle(C, response_time=1, duration=3600, level_min=-95, level_max=-5)
    chunks = chunk_sizes(50_000, 9, hi=5000)
    check_long(run_long(a, padded(x[:, :50_000]), chunks), run_long(o, x[:, :50_000], chunks))


def test_long_levels_floor():
    C = 2
    x = np.zeros((C, 40 * 256), np.float32)
    got = run_long(LongLevelsAnalyzer(C, response_time=1, duration=5), padded(x), [x.shape[1]])
    want = run_long(LongLevelsOracle(C, response_time=1, duration=5), x, [x.shape[1]])
    assert (got[1] == 0).all() and (got[2] == want[2]).all()
    assert np.allclose(got[2], -1500.0, rtol=1e-15)
    check_long(got, want)


def test_nan_samples_act_as_in_the_widget():
    """A NaN sample: the widget's max|x| is NaN, so old_max takes its decay step, and old_rms and
    level_rms stay NaN.  A NaN or infinite sample in the long-term widget: its transposed-form filters
    take y*0 into their state, so from that block on the levels are NaN (max(level, 1e-150) keeps NaN)
    until setresptime or a reset rebuilds them."""
    C = 3
    x = signal(C, 60 * 512, seed=31)
    x[1, 10 * 512 + 7] = np.nan
    x[2, 20 * 512] = np.nan
    a, o = LevelsAnalyzer(C), LevelsOracle(C)
    got = run_meter(a, padded(x), 512, 16)
    want = run_meter_oracle(o, x, 512)
    assert np.isnan(got[0][1, 10:]).all() and not np.isnan(got[1]).any() and not np.isnan(got[2]).any()
    check_meter(got, want, a.state(), o.state())

    x = signal(C, 300 * 256, seed=32)
    x[0, 50 * 256 + 3] = np.nan                  # read by the block that ends at 51 * 256
    x[2, 70 * 256 + 200] = np.inf
    chunks = chunk_sizes(x.shape[1], 3, hi=5000)
    b = LongLevelsAnalyzer(C, response_time=1, duration=5)
    got = run_long(b, padded(x), chunks)
    want = run_long(LongLevelsOracle(C, response_time=1, duration=5), x, chunks)
    lv = got[1]
    assert np.isfinite(lv[0, :51]).all() and np.isnan(lv[0, 52:]).all()
    assert np.isfinite(lv[1]).all()
    assert np.isfinite(lv[2, :71]).all() and np.isnan(lv[2, 72:]).all()
    check_long(got, want)
    b.setresptime(1)                             # the same depth: the filters restart, old_index is kept
    tail = signal(C, 40 * 256, seed=33)
    tr = b.handle_new_data(padded(tail))
    assert np.isfinite(tr.level.cpu().numpy()).all()


# ---------------------------------------------------------------- stream order
HOLD_CYCLES = 250_000_000


@pytest.mark.parametrize("way", ["current", "explicit"])
def test_stream_order(way):
    """Each call on the caller's stream, queued behind a spin kernel with NaN-poisoned inputs that are
    filled on that stream, gives the same bits as the same calls run alone.  Plans and first
    allocations are made before the hold, so every call of the window must return with the held
    work still queued."""
    C = 3
    x = signal(C, 40 * 512, seed=21)
    xt = torch.from_numpy(x).cuda()
    s = torch.cuda.Stream()

    def make():
        return LevelsAnalyzer(C), LongLevelsAnalyzer(C, response_time=1, duration=5)

    def calls(a, b, src, kw, pending=None):
        out = []                    # every output is a new tensor: nothing to copy on another stream
        for k in range(4):
            chunk = src[:, k * 5120:(k + 1) * 5120]
            if pending is not None:
                pending.append(not s.query())
            out.append(list(a.handle_new_data(chunk, **kw)))
            if pending is not None:
                pending.append(not s.query())
            tr = b.handle_new_data(chunk, **kw)
            out.append([tr.level, tr.level_rms])
        if pending is not None:
            pending.append(not s.query())
        out.append([b.curve(**kw)[1]])
        if pending is not None:
            pending.append(not s.query())
        return out

    ref = calls(*make(), xt, {})
    torch.cuda.synchronize()
    a, b = make()
    # the plans (which wait for the device) and the blocks the window reuses, made on s beforehand
    with torch.cuda.stream(s):
        a.handle_new_data(torch.zeros(C, 5120, device="cuda"))
        b.handle_new_data(torch.zeros(C, 5120, device="cuda"))
        b.curve()
    a.reset()
    b.reset()
    assert b._plan_ndec == b.Ndec
    buf = torch.full_like(xt, float("nan"))
    torch.cuda.synchronize()
    pending = []
    if way == "current":
        with torch.cuda.stream(s):
            torch.cuda._sleep(HOLD_CYCLES)
            buf.copy_(xt)
            got = calls(a, b, buf, {}, pending)
    else:
        with torch.cuda.stream(s):
            torch.cuda._sleep(HOLD_CYCLES)
            buf.copy_(xt)
        got = calls(a, b, buf, {"stream": s.cuda_stream}, pending)
    torch.cuda.synchronize()
    assert all(pending), "a call waited for the held work: %s" % pending
    for g, w in zip(got, ref):
        for gv, wv in zip(g, w):
            assert torch.equal(gv, wv)
