"""The levels widget's meter (Levels_Widget.handle_new_data, friture/levels.py:84-131, BallisticPeak,
friture/ballistic_peak.py:43-66, dB_to_IEC, friture/iec.py) and the long-term levels widget
(LongLevelWidget.handle_new_data and its setters, friture/longlevels.py:150-230) for C channels.

TEST INFRASTRUCTURE ONLY (see ``oracle/__init__.py``).

- ``LevelsOracle`` and ``LongLevelsOracle``: plain float64 NumPy restatements, element-wise across
  channels, which need nothing but NumPy.  Every product and sum is the widget's, in the widget's
  order; only the meter's dot product is NumPy's matrix product instead of one np.dot per channel.
- ``reference_widgets()``: the UNMODIFIED ``friture.levels``, ``friture.longlevels``,
  ``friture.ballistic_peak`` and ``friture.iec`` under the minimal PyQt6 stub of
  ``oracle/plot_curves.py``, as the source of ``tests/golden/levels.npz``.
"""
from __future__ import annotations

import numpy as np

SAMPLING_RATE = 48000
PEAK_DECAY_RATE = 1.0 - 3E-6 / 500.
PEAK_FALLOFF = 32


def db_to_iec(db):
    """dB_to_IEC (iec.py:20-33) element-wise."""
    db = np.asarray(db, dtype=np.float64)
    return np.select([db < -70.0, db < -60.0, db < -50.0, db < -40.0, db < -30.0, db < -20.0],
                     [0.0 * db, (db + 70.0) * 0.0025, (db + 60.0) * 0.005 + 0.025,
                      (db + 50.0) * 0.0075 + 0.075, (db + 40.0) * 0.015 + 0.15, (db + 30.0) * 0.02 + 0.3],
                     (db + 20.0) * 0.025 + 0.5)


class LevelsOracle:
    def __init__(self, n_channels, response_time=0.3):
        C = int(n_channels)
        w = 0.65
        n = response_time * SAMPLING_RATE
        N = 5 * n
        self.alpha = 1. - (1. - w) ** (1. / (n + 1))
        self.kernel = (1. - self.alpha) ** (np.arange(0, N)[::-1])
        n2 = 0.025 / (25 / 1000.)
        self.alpha2 = 1. - (1. - w) ** (1. / (n2 + 1))
        self.old_rms = np.full(C, 1e-30)
        self.old_max = np.full(C, 1e-30)
        self.peak = np.zeros(C)
        self.hold = np.zeros(C, dtype=np.int64)
        self.decay = np.full(C, PEAK_DECAY_RATE)

    def state(self):
        return dict(old_rms=self.old_rms.copy(), old_max=self.old_max.copy(), peak_iec=self.peak.copy(),
                    decay=self.decay.copy(), hold=self.hold.copy())

    def handle_new_data(self, floatdata):
        """One buffer, floatdata [C, N] (float64 of float32 samples).  Returns (level_rms, level_max,
        peak_iec) [C]."""
        y = np.asarray(floatdata, dtype=np.float64)
        N = y.shape[1]
        Nk = self.kernel.shape[0]
        assert 1 <= N <= Nk
        value_max = np.abs(y).max(axis=1)
        lim = self.old_max * (1. - self.alpha2)
        self.old_max = np.where(value_max > lim, value_max, lim)
        conv = (y ** 2) @ self.kernel[Nk - N:Nk]
        self.old_rms = self.alpha * conv + self.old_rms * (1.0 - self.alpha) ** N
        with np.errstate(divide="ignore"):
            level_rms = 10. * np.log10(self.old_rms + 0. * 1e-80)
            level_max = 20. * np.log10(self.old_max + 0. * 1e-80)
        self.step_peak(db_to_iec(np.where(level_rms > level_max, level_rms, level_max)))
        return level_rms, level_max, self.peak.copy()

    def step_peak(self, p):
        """BallisticPeak.peak_iec's setter, element-wise."""
        rise = p > self.peak
        hold = ~rise & (self.hold + 1 <= PEAK_FALLOFF)
        fall = ~rise & ~hold
        fallen = self.decay * self.peak
        catch = fall & (fallen < p)
        decay_on = fall & ~catch
        self.peak = np.where(rise | catch, p, np.where(decay_on, fallen, self.peak))
        self.hold = np.where(rise | catch, 0, np.where(hold, self.hold + 1, self.hold))
        self.decay = np.where(rise | catch, PEAK_DECAY_RATE, np.where(decay_on, self.decay * self.decay, self.decay))


def gauss(n=11, sigma=1):
    r = range(-int(n / 2), int(n / 2) + 1)
    return [1 / (sigma * np.sqrt(2 * np.pi)) * np.exp(-float(x) ** 2 / (2 * sigma ** 2)) for x in r]


def fir_nested(b, state, x, latched):
    """lfilter_float64_1D(b, [1, 0, ...], x, zi) (lfilter.py:132-139) for rows of x [C, L], with
    state [C, len(b)-1] the last inputs before x (zeros for a zero zi): y[n] = (...(b[-1] x[n-T+1]
    + b[-2] x[n-T+2]) + ...) + b[0] x[n].  In the transposed form the state takes y[n] * a[k] = y[n] * 0,
    which is NaN once y[n] is NaN or infinite: from the output after a row's first non-finite input on,
    its outputs are NaN for good (latched [C], until the filter is rebuilt).  Returns (y, new state,
    new latched)."""
    T = len(b)
    xin = np.concatenate([state, x], axis=1)
    L = x.shape[1]
    y = b[T - 1] * xin[:, 0:L]
    for t in range(T - 2, -1, -1):
        y = y + b[t] * xin[:, T - 1 - t:T - 1 - t + L]
    bad = ~np.isfinite(x)
    first = np.where(bad.any(axis=1), bad.argmax(axis=1), L)
    nan_from = np.where(latched, 0, first + 1)
    y = np.where(np.arange(L)[None, :] >= nan_from[:, None], np.nan, y)
    return y, xin[:, xin.shape[1] - (T - 1):], latched | (first < L)


class LevelRing:
    """The widget's level RingBuffer (ringbuffer.py) for C rows: slot offset % length, and
    grow_if_needed's move of slot s to (s + shift) % new."""

    def __init__(self, n_channels, length=10000):
        self.buf = np.zeros((n_channels, length))
        self.offset = 0

    def push(self, v):
        self.buf[:, self.offset % self.buf.shape[1]] = v
        self.offset += 1

    def grow_if_needed(self, length):
        old = self.buf.shape[1]
        if length <= old:
            return
        new = int(1.5 * length)
        shift = (self.offset % new - self.offset % old) % new
        nb = np.zeros((self.buf.shape[0], new))
        nb[:, (np.arange(old) + shift) % new] = self.buf
        self.buf = nb

    def data(self, length):
        self.grow_if_needed(length)
        return self.buf[:, (self.offset - length + np.arange(length)) % self.buf.shape[1]]


class LongLevelsOracle:
    def __init__(self, n_channels, response_time=20, duration=600, level_min=-70, level_max=-20):
        self.C = int(n_channels)
        self.level_min, self.level_max = level_min, level_max
        self.length_seconds = duration
        self.stream = np.zeros((self.C, 0))
        self.old_index = 0
        self.ring = LevelRing(self.C)
        self.setresptime(response_time)
        self.curve = None

    def setresptime(self, value):
        self.response_time = value
        self.Ndec = int(max(0, np.floor((np.log2(self.response_time * SAMPLING_RATE / 100.)))))
        self.b = np.array(gauss(10 * 4 + 1, 2. * 4))
        self.bdec = np.array(gauss(11, 2.))
        self.zf = np.zeros((self.C, 40))
        self.zis = [np.zeros((self.C, 10)) for _ in range(self.Ndec)]
        self.latched = [np.zeros(self.C, dtype=bool) for _ in range(self.Ndec + 1)]   # the last: the 41-tap FIR
        self.subsampled_sampling_rate = SAMPLING_RATE / 2 ** (self.Ndec)
        self.setduration(self.length_seconds)

    def setduration(self, value):
        self.length_seconds = value
        self.length_samples = int(self.length_seconds * self.subsampled_sampling_rate)

    def setmin(self, value):
        self.level_min = value

    def setmax(self, value):
        self.level_max = value

    def block(self, end, length):
        start = end - length
        out = np.zeros((self.C, length))
        lo = max(start, 0)
        out[:, lo - start:] = self.stream[:, lo:end]
        return out

    def handle_new_data(self, floatdata):
        """floatdata [C, n].  Returns (end_index [r], level [C, r], level_rms [C, r])."""
        self.stream = np.concatenate([self.stream, np.asarray(floatdata, dtype=np.float64)], axis=1)
        needed = int(2 ** self.Ndec)
        realizable = int(np.floor((self.stream.shape[1] - self.old_index) / needed))
        ends, levels, dbs = [], [], []
        for _ in range(realizable):
            y = self.block(self.old_index, needed) ** 2
            for s in range(self.Ndec):
                y, self.zis[s], self.latched[s] = fir_nested(self.bdec, self.zis[s], y, self.latched[s])
                y = y[:, ::2]
            level, self.zf, self.latched[-1] = fir_nested(self.b, self.zf, y, self.latched[-1])
            level = level[:, 0]
            db = 10. * np.log10(np.where(1e-150 > level, 1e-150, level))
            self.ring.push(db)
            ends.append(self.old_index)
            levels.append(level)
            dbs.append(db)
            self.old_index += needed
        if realizable > 0:
            time = np.arange(self.length_samples) / self.subsampled_sampling_rate
            levels_ring = self.ring.data(self.length_samples)
            scaled_t = time / self.length_seconds
            scaled_y = np.clip(1. - (levels_ring - self.level_min) / (self.level_max - self.level_min), 0., 1.)
            self.curve = (scaled_t, scaled_y)
        shape = (self.C, 0)
        return (np.array(ends, dtype=np.int64),
                np.stack(levels, axis=1) if levels else np.zeros(shape),
                np.stack(dbs, axis=1) if dbs else np.zeros(shape))


# ---------------------------------------------------------------- the unmodified reference widgets
def reference_widgets():
    """(levels, longlevels, ballistic_peak, iec, ringbuffer) modules of the reference, unmodified."""
    from . import ref_import
    from .plot_curves import _install_pyqt6_stub
    ns = ref_import.load()
    _install_pyqt6_stub()
    import friture.ballistic_peak as ballistic_peak
    import friture.iec as iec
    import friture.levels as levels
    import friture.longlevels as longlevels
    return levels, longlevels, ballistic_peak, iec, ns.ringbuffer


# ---------------------------------------------------------------- tests/golden/levels.npz's stream
GOLDEN_SAMPLES = 3_000_000
GOLDEN_METER_BUFFERS = 1024


def golden_stream(seed=20261018):
    """The two-channel float32 stream of tests/golden/levels.npz [2, GOLDEN_SAMPLES]: silence,
    full-scale tones, DC, quiet noise with isolated impulses, a quiet tail in which the ballistic
    peak reaches its decay phase, then noise under a slow envelope with a silent stretch."""
    rng = np.random.default_rng(seed)
    t = np.arange(GOLDEN_SAMPLES) / SAMPLING_RATE
    x = np.zeros((2, GOLDEN_SAMPLES))
    x[0, 24000:72000] = np.sin(2 * np.pi * 1000 * t[24000:72000])
    x[1, 24000:72000] = 0.9 * np.sin(2 * np.pi * 440 * t[24000:72000])
    x[0, 72000:96000] = 0.5
    x[1, 72000:96000] = -0.25
    x[:, 96000:144000] = 1e-3 * rng.standard_normal((2, 48000))
    x[0, 96000:144000:7000] = 0.8
    x[1, 99500:144000:7000] = -0.8
    x[:, 144000:300000] = 1e-5 * rng.standard_normal((2, 156000))
    env = 0.05 * (1.2 + np.sin(2 * np.pi * t[300000:] / 7.0))
    x[:, 300000:] = env * rng.standard_normal((2, GOLDEN_SAMPLES - 300000))
    x[:, 900000:996000] = 0.0
    return x.astype(np.float32)


def golden_schedule(seed=7):
    """The long-term widget's chunks and setters: a list of (n_samples, setter or None, value).
    Uneven chunks; response time changes mid-stream, and once the 10000-slot level ring has wrapped,
    a duration increase that grows it."""
    rng = np.random.default_rng(seed)
    events = {400_000: ("setresptime", 3), 600_000: ("setresptime", 1), 700_000: ("setmin", -90),
              800_000: ("setmax", -10), 2_940_000: ("setduration", 60)}
    out, pos = [("setresptime", 1), ("setduration", 5)], 0
    keys = sorted(events)
    while pos < GOLDEN_SAMPLES:
        n = int(rng.integers(1, 40000))
        nxt = next((k for k in keys if k > pos), None)
        if nxt is not None and pos + n >= nxt:
            n = nxt - pos
        n = min(n, GOLDEN_SAMPLES - pos)
        out.append(n)
        pos += n
        if pos in events:
            out.append(events[pos])
    return out
