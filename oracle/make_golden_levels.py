#!/usr/bin/env python
"""Generate tests/golden/levels.npz by running the UNMODIFIED reference classes ``Levels_Widget``,
``LongLevelWidget``, ``BallisticPeak`` and ``dB_to_IEC`` (imported in place under the minimal PyQt6 stub
of oracle/plot_curves.py) on the stream of ``oracle.levels.golden_stream``.  TEST INFRASTRUCTURE ONLY;
run where the reference tree exists:

    python oracle/make_golden_levels.py

The meter takes the first GOLDEN_METER_BUFFERS 512-sample buffers of both channels (one widget, its
two channels).  The long-term widget runs each channel on its own widget (it reads channel 0 only),
fed through a stub AudioBuffer holding the reference RingBuffer, with the chunks and setters of
``golden_schedule``.  Keys:
  m_rms, m_max, m_iec [2, B]: level_rms, level_max, peak_iec after each buffer;
  m_old_rms, m_old_max, m_decay [2, B] float64 and m_hold [2, B] int: the state after each buffer;
  l_end [K] int64, l_level, l_db [2, K]: every block's end index, linear level and dB;
  l_curve_call [S]: the chunk numbers after which a curve was taken (the 101st, the first after the
  duration increase that grows the wrapped level ring, the last), l_curve_<s> [2, L_s] scaled_y and
  l_t_<s> [L_s] scaled_t.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.levels import GOLDEN_METER_BUFFERS, golden_schedule, golden_stream, reference_widgets  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "levels.npz")


class _Holder:
    pass


class AudioBuffer:
    """What LongLevelWidget.handle_new_data reads of friture.audiobuffer.AudioBuffer."""

    def __init__(self, RingBuffer):
        self.ringbuffer = RingBuffer()
        self.lastDataTime = 0.

    def push(self, floatdata):
        self.ringbuffer.push(floatdata, 0.)

    def data_indexed(self, start, length):
        return self.ringbuffer.data_indexed(start, length)


def meter(levels, ballistic_peak, x):
    vm = _Holder()
    for n in ("level_data", "level_data_2", "level_data_slow", "level_data_slow_2"):
        setattr(vm, n, _Holder())
    vm.level_data_ballistic = ballistic_peak.BallisticPeak()
    vm.level_data_ballistic_2 = ballistic_peak.BallisticPeak()
    w = levels.Levels_Widget(None, vm)
    keys = ("rms", "max", "iec", "old_rms", "old_max", "decay", "hold")
    out = {k: np.zeros((2, GOLDEN_METER_BUFFERS)) for k in keys}
    for b in range(GOLDEN_METER_BUFFERS):
        w.handle_new_data(x[:, b * 512:(b + 1) * 512].astype(np.float64))
        for c, (ld, bp, rms, mx) in enumerate([(vm.level_data, vm.level_data_ballistic, w.old_rms, w.old_max),
                                               (vm.level_data_2, vm.level_data_ballistic_2, w.old_rms_2,
                                                w.old_max_2)]):
            vals = (ld.level_rms, ld.level_max, bp.peak_iec, rms, mx, bp._peak_decay_factor, bp._peak_hold_counter)
            for k, v in zip(keys, vals):
                out[k][c, b] = v
    res = {"m_" + k: v for k, v in out.items()}
    res["m_hold"] = res["m_hold"].astype(np.int64)
    return res


def long_levels(longlevels, RingBuffer, x):
    """Each channel on its own widget.  Every block's linear level is what the widget's own
    lfilter_float64_1D call on the 41-tap filter returned (recorded by a wrapper that passes the
    call through unchanged); its dB is what the widget pushed to its level ring."""
    sched = golden_schedule()
    n_calls = sum(1 for e in sched if not isinstance(e, tuple))
    first_after_grow = sum(1 for e in sched[:sched.index(("setduration", 60))] if not isinstance(e, tuple))
    curve_calls = (100, first_after_grow, n_calls - 1)
    orig = longlevels.lfilter_float64_1D
    res = {"l_curve_call": np.array(curve_calls, dtype=np.int64)}
    level, db, ends = [[], []], [[], []], []
    for c in range(2):
        def recorded(b, a, x_, zi, _c=c):
            y, z = orig(b, a, x_, zi)
            if len(b) == 41:
                level[_c].append(float(y[0]))
            return y, z
        longlevels.lfilter_float64_1D = recorded
        w = longlevels.LongLevelWidget(None)
        ab = AudioBuffer(RingBuffer)
        w.set_buffer(ab)
        pos, call = 0, 0
        for ev in sched:
            if isinstance(ev, tuple):
                getattr(w, ev[0])(ev[1])
                continue
            ab.push(x[c:c + 1, pos:pos + ev].astype(np.float64))
            pos += ev
            before, needed = w.old_index, int(2 ** w.Ndec)
            w.handle_new_data(None)
            k = (w.old_index - before) // needed
            if k:
                db[c].extend(w.ringbuffer.data(k)[0].tolist())
                if c == 0:
                    ends.extend(range(before, w.old_index, needed))
            if call in curve_calls:
                res["l_curve_%d" % call] = res.get("l_curve_%d" % call, []) + [np.array(w._curve._y_array)]
                res["l_t_%d" % call] = np.array(w._curve._x_array)
            call += 1
    longlevels.lfilter_float64_1D = orig
    res["l_end"] = np.array(ends, dtype=np.int64)
    res["l_level"] = np.array(level)
    res["l_db"] = np.array(db)
    for call in curve_calls:
        res["l_curve_%d" % call] = np.stack(res["l_curve_%d" % call])
    return res


if __name__ == "__main__":
    levels, longlevels, ballistic_peak, iec, ringbuffer = reference_widgets()
    x = golden_stream()
    out = meter(levels, ballistic_peak, x)
    out.update(long_levels(longlevels, ringbuffer.RingBuffer, x))
    np.savez_compressed(OUT, **out)
    print("wrote %s: %s" % (OUT, {k: v.shape for k, v in out.items()}))
