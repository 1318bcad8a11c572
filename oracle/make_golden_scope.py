#!/usr/bin/env python
"""Generate tests/golden/scope.npz by running the UNMODIFIED reference ``Scope_Widget.handle_new_data``
and ``RingBuffer`` (imported in place under the minimal PyQt6 stub of oracle/plot_curves.py) on the
stream of ``oracle.scope.golden_stream``.  TEST INFRASTRUCTURE ONLY; run where the reference tree
exists:

    python oracle/make_golden_scope.py

Scopes 0-2 are one-channel widgets (channel 0 of the stream), scopes 3-4 two-channel widgets.  Each
has its own RingBuffer, into which every 512-sample buffer is pushed before handle_new_data runs, as
friture/analyzer.py does; set_timerange is called before the ticks of ``GOLDEN_SCHEDULE``.  The method
runs on a light holder object with the attributes it reads, not on a built widget.  The trigger
position is what the widget's own ``where`` call returned (a wrapper passes it through unchanged).
Keys, K = GOLDEN_TICKS:
  start [5, K] int64: the stream index the drawn window starts at, or NOT_DRAWN;
  npts [5, K] int64: the curve's point count after the tick;
  digest [5, K, 20] uint8: sha1 of the float64 scaled_t, scaled_y (and scaled_y2) the widget holds;
  curve_ticks [N]: the ticks after which whole curves are kept (short ranges, to keep the file small;
  the digests cover every tick); for each scope s that holds a curve then, y_<tick>_<s> [n_ch, L]
  float32(scaled_y, scaled_y2).
"""
import hashlib
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.scope import (GOLDEN_BUFFER, GOLDEN_SCHEDULE, GOLDEN_TICKS, NOT_DRAWN, golden_stream,  # noqa: E402
                          reference_scope)

OUT = os.path.join(ROOT, "tests", "golden", "scope.npz")
CURVE_TICKS = (41, 80, 305, 315, 325)


class _Curve:
    def __init__(self):
        self.x = self.y = None

    def setData(self, x, y):
        self.x, self.y = np.array(x), np.array(y)


class _ScopeData:
    def __init__(self):
        self.plot_items = [None]
        self.horizontal_axis = self

    def setRange(self, lo, hi):
        pass

    def add_plot_item(self, item):
        self.plot_items.append(item)

    def remove_plot_item(self, item):
        self.plot_items.remove(item)


class _Holder:
    """What Scope_Widget.handle_new_data reads and writes of the widget."""

    def __init__(self, ring):
        self.audiobuffer = ring
        self._scope_data = _ScopeData()
        self._curve, self._curve_2 = _Curve(), _Curve()


def digest(*arrays):
    h = hashlib.sha1()
    for a in arrays:
        if a is not None:
            h.update(np.ascontiguousarray(a, dtype=np.float64).tobytes())
    return np.frombuffer(h.digest(), dtype=np.uint8)


def run():
    scope, ringbuffer = reference_scope()
    x = golden_stream()
    orig_where = scope.where
    found = []

    def recorded(cond):
        r = orig_where(cond)
        found.append(r[0])
        return r

    scope.where = recorded
    K = GOLDEN_TICKS
    res = dict(start=np.full((5, K), NOT_DRAWN, dtype=np.int64), npts=np.zeros((5, K), np.int64),
               digest=np.zeros((5, K, 20), np.uint8), curve_ticks=np.array(CURVE_TICKS, dtype=np.int64))
    sched = dict(GOLDEN_SCHEDULE)
    for s in range(5):
        nch = 1 if s < 3 else 2
        ring = ringbuffer.RingBuffer()
        w = _Holder(ring)
        for k in range(K):
            if k in sched:
                scope.Scope_Widget.set_timerange(w, sched[k])
            buf = x[s, :nch, k * GOLDEN_BUFFER:(k + 1) * GOLDEN_BUFFER].astype(np.float64)
            ring.push(buf, 0.)
            before = w._curve.y
            found.clear()
            scope.Scope_Widget.handle_new_data(w, buf)
            width = int(w.timerange * 1e-3 * 48000)
            if w._curve.y is not before:
                if w.timerange > 500.0:
                    res["start"][s, k] = ring.offset - width
                else:
                    res["start"][s, k] = ring.offset - 2 * width + int(found[-1][0])
            y2 = w._curve_2.y if nch == 2 else None
            res["npts"][s, k] = 0 if w._curve.y is None else len(w._curve.y)
            res["digest"][s, k] = digest(w._curve.x, w._curve.y, y2)
            if k in CURVE_TICKS and w._curve.y is not None:
                res["y_%d_%d" % (k, s)] = np.stack([w._curve.y] + ([y2] if nch == 2 else [])).astype(np.float32)
    scope.where = orig_where
    return res


if __name__ == "__main__":
    out = run()
    np.savez_compressed(OUT, **out)
    print("wrote %s: %s" % (OUT, {k: v.shape for k, v in out.items()}))
