"""The spectrum and octave widgets' plotted curves and peak hold (SpectrumPlotWidget.setdata and
compute_peaks, friture/spectrumPlotWidget.py:122-200; HistPlot.setdata and compute_peaks,
friture/histplot.py:77-130).

TEST INFRASTRUCTURE ONLY (see ``oracle/__init__.py``).

- ``PlotCurvesOracle``: a plain float64 NumPy restatement of one channel's per-call step, which needs
  nothing but NumPy and so runs where the reference tree does not exist.
- ``reference_widgets()``: the UNMODIFIED ``friture.spectrumPlotWidget`` and ``friture.histplot``
  imported from the reference tree under a minimal ``PyQt6`` stub (below), as the checker of the
  restatement and the source of ``tests/golden/plot_curves.npz``.
"""
from __future__ import annotations

import sys
import types

import numpy as np

PEAK_DECAY_RATE = 1.0 - 3e-6
D0 = 20.0 * np.log10(PEAK_DECAY_RATE) * 5000       # compute_peaks' decay step


class PlotCurvesOracle:
    """One channel of either widget: ``setspecrange`` then ``setdata(y)`` per dB vector (float64
    arithmetic, NumPy element-wise, like the reference).  ``setdata`` returns the float64
    (scaled_y, z, scaled_peak, z_peak) the widget hands its two curves; with ``peaks`` False the
    peak state is left alone and the last two are None."""

    def __init__(self, spec_min=0., spec_max=1.):
        self.peak = np.zeros(3)                     # length 3: the first call resets
        self.peak_int = np.zeros(3)
        self.peak_decay = np.ones(3) * PEAK_DECAY_RATE
        self.setspecrange(spec_min, spec_max)

    def setspecrange(self, spec_min, spec_max):
        if spec_min > spec_max:
            spec_min, spec_max = spec_max, spec_min
        self.m, self.mx = spec_min, spec_max

    def to_screen(self, v):
        if self.mx == self.m:
            return 0 + 0. * v
        return (v - self.m) * 1 / (self.mx - self.m) + 0

    def step_peaks(self, y):
        if self.peak.shape != y.shape:
            self.peak = np.full(y.shape, -500.0)
            self.peak_int = np.zeros(y.shape)
            self.peak_decay = np.full(y.shape, D0)
        rise = self.peak < y
        fall = ~rise & (self.peak_int < 0.2)
        hold = ~rise & (self.peak_int >= 0.2)
        old_decay = self.peak_decay
        self.peak = np.where(rise, y, np.where(fall, self.peak + old_decay, self.peak))
        self.peak_decay = np.where(rise, D0, np.where(fall, old_decay + D0, old_decay))
        self.peak_int = np.where(rise, 1.0, np.where(hold, self.peak_int * 0.975, self.peak_int))

    def setdata(self, y, peaks=True):
        """y: [K], or [C, K] for C independent channels (with the same range) at once."""
        y = np.asarray(y, dtype=np.float64)
        M = np.max(y, axis=-1, keepdims=True)
        z = (y - self.m) / (np.abs(M - self.m) + 1e-3)
        scaled_y = 1.0 - self.to_screen(y)
        if not peaks:
            return scaled_y, z, None, None
        self.step_peaks(y)
        return scaled_y, z, 1.0 - self.to_screen(self.peak), self.peak_int.copy()


def fixture_ticks(g, case):
    """The calls of one case of tests/golden/plot_curves.npz (see oracle/make_golden_plot.py), as
    dicts: y float32 [K], spec_min, spec_max, paused, peaks, data_baseline, fmax, fpitch, and the
    curves the reference widget held after the call: sy, z, speak, zpeak float64 [K], baseline."""
    K = g[case + "_K"]
    offs = np.concatenate([[0], np.cumsum(K)])
    ctrl = g[case + "_ctrl"]
    for t in range(len(K)):
        sl = slice(offs[t], offs[t + 1])
        d = dict(t=t, y=g[case + "_y"][sl], spec_min=ctrl[t, 0], spec_max=ctrl[t, 1],
                 paused=bool(ctrl[t, 2]), peaks=bool(ctrl[t, 3]), data_baseline=bool(ctrl[t, 4]),
                 fmax=g[case + "_fmax"][t], fpitch=g[case + "_fpitch"][t],
                 baseline=g[case + "_baseline"][t])
        for n in ("sy", "z", "speak", "zpeak"):
            d[n] = g[case + "_" + n][sl]
        yield d


# ---------------------------------------------------------------- the unmodified reference widgets
def _install_pyqt6_stub():
    """Just what the two widgets' modules touch: QObject (with setParent), pyqtProperty, pyqtSlot,
    pyqtSignal and QQmlListProperty.  Qt widgets, settings and QML types are dummies."""
    if "PyQt6" in sys.modules:
        return

    class _Signal:
        def __init__(self, *a, **k):
            pass

        def __get__(self, obj, owner):
            return self

        def emit(self, *a):
            pass

        def connect(self, *a):
            pass

    class QObject:
        def __init__(self, *a, **k):
            pass

        def setParent(self, parent):
            self._parent = parent

        def parent(self):
            return getattr(self, "_parent", None)

    def pyqtProperty(*a, **k):
        class _Prop(property):
            def setter(self, f):
                return _Prop(self.fget, f)
        return lambda f: _Prop(f)

    def pyqtSlot(*a, **k):
        return lambda f: f

    class _Dummy:
        def __init__(self, *a, **k):
            pass

        def __getattr__(self, name):
            return _Dummy()

        def __call__(self, *a, **k):
            return _Dummy()

    class _Mod(types.ModuleType):
        def __getattr__(self, name):
            if name.startswith("__"):
                raise AttributeError(name)
            return type(name, (_Dummy,), {})

    mods = {n: _Mod(n) for n in ("PyQt6", "PyQt6.QtCore", "PyQt6.QtQml", "PyQt6.QtWidgets",
                                  "PyQt6.QtGui", "PyQt6.QtQuick")}
    qc = mods["PyQt6.QtCore"]
    qc.QObject, qc.pyqtProperty, qc.pyqtSlot, qc.pyqtSignal = QObject, pyqtProperty, pyqtSlot, _Signal
    mods["PyQt6.QtQml"].QQmlListProperty = type("QQmlListProperty", (_Dummy,), {})
    for n, m in mods.items():
        sys.modules[n] = m
        if n != "PyQt6":
            setattr(mods["PyQt6"], n.split(".")[1], m)


def reference_widgets():
    """(friture.spectrumPlotWidget, friture.histplot, friture.plotting.frequency_scales), unmodified."""
    from . import ref_import
    ref_import.load()
    _install_pyqt6_stub()
    import friture.spectrumPlotWidget as spw
    import friture.histplot as hp
    import friture.plotting.frequency_scales as fscales
    return spw, hp, fscales


def curve_arrays(curve):
    """Copies of (x_left, x_right, y, z) a FilledCurve was last given, and its baseline.  Copies:
    the peak curve's z is the widget's own peak_int, which the next compute_peaks scales in place."""
    arrays = (curve._x_left_array, curve._x_right_array, curve._y_array, curve._z_array)
    return tuple(None if a is None else np.array(a, copy=True) for a in arrays) + (curve._baseline,)
