"""The scope widget (Scope_Widget.handle_new_data and set_timerange, friture/scope.py:78-148) for S
scopes, each reading its own audio ring buffer (friture/ringbuffer.py).

TEST INFRASTRUCTURE ONLY (see ``oracle/__init__.py``).

- ``ScopeOracle``: a plain float64 NumPy restatement, scope by scope, which needs nothing but NumPy.
  Each tick pushes one buffer into the ring and reads the widget's window from it; the ring is the
  single-copy ring of ``oracle.levels.LevelRing`` (slot p % length, grow_if_needed's move of slot s
  to (s + shift) % new), pushed a buffer at a time.
- ``reference_scope()``: the UNMODIFIED ``friture.scope`` and ``friture.ringbuffer`` under the minimal
  PyQt6 stub of ``oracle/plot_curves.py``, as the source of ``tests/golden/scope.npz``.
"""
from __future__ import annotations

import numpy as np

from .levels import LevelRing

SAMPLING_RATE = 48000
NOT_DRAWN = np.iinfo(np.int64).min


class AudioRing(LevelRing):
    """The widget's audio RingBuffer for C rows: push writes a block of samples."""

    def push_block(self, x):
        n = x.shape[1]
        self.grow_if_needed(n)
        self.buf[:, (self.offset + np.arange(n)) % self.buf.shape[1]] = x
        self.offset += n


def width_of(timerange):
    time = timerange * 1e-3
    return int(time * SAMPLING_RATE)


class ScopeOracle:
    def __init__(self, n_scopes, two_channels=False, timerange=50):
        self.S, self.nch = int(n_scopes), 2 if two_channels else 1
        self.ring = AudioRing(self.S * self.nch)
        self.timerange = timerange
        self.y = [None] * self.S           # per scope: (scaled_y, scaled_y2 or None, timerange) float64
        self.drawn_at = [None] * self.S

    def set_timerange(self, timerange):
        self.timerange = timerange

    def handle_new_data(self, x):
        """One buffer x [S, nch, b] (float32 samples).  Returns the window starts [S] int64: the stream
        index each scope's drawn window starts at, or NOT_DRAWN."""
        S, nch = self.S, self.nch
        self.ring.push_block(np.asarray(x, dtype=np.float64).reshape(S * nch, -1))
        width = width_of(self.timerange)
        trigger = not self.timerange > 500.0
        need = 2 * width if trigger else width
        d = self.ring.data(need).reshape(S, nch, need)
        first = self.ring.offset - need
        starts = np.full(S, NOT_DRAWN, dtype=np.int64)
        for s in range(S):
            if not trigger:
                i, y = 0, d[s]
            else:
                t = d[s, 0, width // 2: width // 2 + width]
                level = t.max() * 2. / 3.
                hits = np.flatnonzero((t[:-1] < level) & (t[1:] >= level))
                if len(hits) == 0:
                    continue
                i = int(hits[0])
                y = d[s, :, i:i + 2 * (width // 2)]
            starts[s] = first + i
            time = (np.arange(y.shape[1]) - width // 2) / float(SAMPLING_RATE)
            scaled_t = (time * 1e3 + self.timerange / 2.) / self.timerange
            sy = 1. - (y + 1) / 2.
            self.y[s] = (scaled_t, sy[0], sy[1] if nch == 2 else None, self.timerange)
        return starts


# ---------------------------------------------------------------- the unmodified reference widget
def reference_scope():
    """(friture.scope, friture.ringbuffer) of the reference, unmodified."""
    from . import ref_import
    from .plot_curves import _install_pyqt6_stub
    ns = ref_import.load()
    _install_pyqt6_stub()
    import friture.scope as scope
    return scope, ns.ringbuffer


# ---------------------------------------------------------------- tests/golden/scope.npz's stream
# (tick, value): set_timerange(value) before that tick.  See golden_growths for the ring's growths.
GOLDEN_SCHEDULE = ((0, 50), (41, 125), (60, 0.1), (70, 0.3), (80, 123.4), (110, 600), (150, 300),
                   (190, 500.1), (230, 500), (300, 50), (330, 10000), (450, 1000), (460, 2))
GOLDEN_TICKS = 490
GOLDEN_BUFFER = 512


def golden_growths(schedule=GOLDEN_SCHEDULE, buffer=GOLDEN_BUFFER, ticks=GOLDEN_TICKS):
    """The ring growths of the schedule: (tick, offset after its push, old length, new length, the
    length asked for, the number of zeros and of moved samples the tick's window reads)."""
    sched, L, out = dict(schedule), 10000, []
    tr = None
    for k in range(ticks):
        tr = sched.get(k, tr)
        w = width_of(tr)
        need = 2 * w if not tr > 500.0 else w
        if need > L:
            off = (k + 1) * buffer
            new = int(1.5 * need)
            o = off % L
            zeros = min(need, new - L + o) - o if need > o else 0
            moved = max(0, need - (new - L + o))
            out.append((k, off, L, new, need, zeros, moved))
            L = new
    return out


def golden_stream(seed=20261019):
    """float32 [5, 2, GOLDEN_TICKS * 512]: five scopes' two channels (the one-channel scopes use
    channel 0).  Scope 0: tones, noise and a chirp; 1: silence, then all negative, then a sample exactly
    at the level, crossings at the first and last pair; 2: noise with NaN, +Inf and -Inf samples;
    3 and 4: two-channel tones and noise."""
    rng = np.random.default_rng(seed)
    T = GOLDEN_TICKS * GOLDEN_BUFFER
    t = np.arange(T) / SAMPLING_RATE
    x = np.zeros((5, 2, T))
    x[0, 0] = 0.6 * np.sin(2 * np.pi * (200 + 3000 * t / t[-1]) * t) + 0.05 * rng.standard_normal(T)
    x[0, 0, T // 2:] = 0.3 * np.sin(2 * np.pi * 37 * t[T // 2:])
    x[1, 0, 100 * 512:200 * 512] = -np.abs(rng.standard_normal(100 * 512)) - 0.1
    x[1, 0, 200 * 512:] = 0.2 * np.sin(2 * np.pi * 440 * t[200 * 512:])
    x[1, 0, 260 * 512:261 * 512] = 0.0
    x[2, 0] = 0.3 * rng.standard_normal(T)
    for k, v in ((3000, np.nan), (30000, np.inf), (61000, -np.inf), (90001, np.nan), (150000, np.inf),
                 (180000, -np.inf), (240000, np.nan)):
        x[2, 0, k] = v
    x[3, 0] = 0.8 * np.sin(2 * np.pi * 1000 * t) * (0.5 + 0.5 * np.sin(2 * np.pi * 0.5 * t))
    x[3, 1] = 0.1 * rng.standard_normal(T)
    x[4, 0] = np.sign(np.sin(2 * np.pi * 90 * t)) * 0.5 + 0.01 * rng.standard_normal(T)
    x[4, 1] = -x[3, 0]
    for tick, kind in EDGE_TICKS:
        place_edge(x[1, 0], tick, width_of(50), kind)
    return x.astype(np.float32)


EDGE_TICKS = ((305, "first"), (315, "last"), (325, "at_level"))


def place_edge(row, tick, width, kind, buffer=GOLDEN_BUFFER):
    """Write into row [T] the search window of the trigger-mode tick `tick` (its samples end at
    (tick + 1) * buffer): "first", a crossing at the first pair only; "last", at the last pair only;
    "at_level", a sample exactly at level = 0.75 * 2 / 3 = 0.5 after one below it."""
    a = (tick + 1) * buffer - 2 * width + width // 2
    s = row[a:a + width]
    if kind == "first":
        s[:] = 0.5
        s[0] = 0.0
    elif kind == "last":
        s[:] = 0.5
        s[-2] = 0.0
    else:
        s[:] = 0.0
        s[width // 3] = 0.75
        s[width // 5] = 0.5
