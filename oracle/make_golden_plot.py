#!/usr/bin/env python
"""Generate tests/golden/plot_curves.npz by running the UNMODIFIED reference widgets
``friture.spectrumPlotWidget.SpectrumPlotWidget`` and ``friture.histplot.HistPlot`` (imported in place
under a minimal PyQt6 stub, oracle/plot_curves.py).  TEST INFRASTRUCTURE ONLY; run where the
reference tree exists:

    python oracle/make_golden_plot.py

Writes that one file and leaves the other fixtures untouched.

Each case is one channel driven through a schedule of setdata calls with float32-representable dB
vectors: bursts that rise, holds longer than the 64 hold ticks followed by long, accelerating falls,
per-bin bursts that re-rise during a fall, repeated vectors (exact ties y == peak), silence at
-300 dB, and per-tick settings: the spec range (swapped, changed midway, empty), pause, peaks off and
back on with the dual-channel baseline, and a change of the bin count.  Keys per case ``<c>_``:
  K [T] bins per tick, y float32 [sum K] the dB vectors back to back, ctrl float64 [T, 5]
  (spec_min, spec_max as given to setspecrange, paused, peaks enabled, data baseline), fmax /
  fpitch [T]; after each call the curves the widget holds: sy, z, speak, zpeak float64 [sum K],
  baseline [T]; the final state peak / peak_int / decay and x edges xl / xr; for the spectrum the
  tracker fields fmax_x, fpitch_x [T], fmax_text, fpitch_text; for the octave widget f_nominal.
  ``settings`` holds (scale name, minfreq, maxfreq) of the spectrum cases, or the bands per octave.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle.plot_curves import curve_arrays, reference_widgets  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "plot_curves.npz")
FS = 48000

# spectrum cases: (name, scale, minfreq, maxfreq, K, ticks, events)
SPECTRUM = [
    ("mel", "Mel", 20, 20000, 129, 230, True),
    ("lin", "Linear", 0, 24000, 33, 90, False),
    ("log", "Logarithmic", 20, 20000, 33, 90, False),
    ("log0", "Logarithmic", 0, 24000, 17, 40, False),        # the clipped branch of toScreen
    ("erb", "ERB", 20, 20000, 65, 90, False),
    ("oct", "Octave", 40, 16000, 65, 90, False),
]
OCTAVE = [("hist3", 3, 220, True), ("hist24", 24, 90, False)]


def db_sequence(rng, K, T):
    """float32 dB vectors [T, K]: bursts at ticks 0-5 and 150, ties (ticks 6-7 repeat the peak of
    ticks 0-5), a floor near -90 dB with per-bin bursts, silence at ticks 60-125 (the hold of the
    first burst ends near tick 70, then the peak falls until a burst or tick 126 lifts it)."""
    base = rng.uniform(-70, -30, K)
    y = -90 + 4 * rng.standard_normal((T, K))
    y[:6] = base + 3 * rng.standard_normal((6, K))
    y[6:8] = y[:6].max(axis=0)
    if T > 150:
        y[150] = base + 10
    burst = rng.random((T, K)) < 0.015
    y[burst] = rng.uniform(-60, -20, burst.sum())
    y[60:126] = -300.
    return y.astype(np.float32)


def schedule(T, events, peak_toggle):
    """ctrl rows (spec_min, spec_max, paused, peaks, data_baseline) and, per tick, whether the bin
    count has changed (from tick 200 on)."""
    ctrl = np.zeros((T, 5))
    ctrl[:, 0], ctrl[:, 1], ctrl[:, 3] = -100, -20, 1
    changed = np.zeros(T, dtype=bool)
    if events:
        ctrl[30:36, 2] = 1                    # paused
        if peak_toggle:                       # the spectrum widget's dual-channel mode:
            ctrl[40:52, 3] = 0                # peaks off ...
            ctrl[40:52, 4] = 1                # ... with the data baseline
        ctrl[120:, 0], ctrl[120:, 1] = -20, -120      # swapped, wider: state kept, curves rescaled
        ctrl[140:143, 0] = ctrl[140:143, 1] = -50     # empty range
        changed[200:] = True                  # bin count change: state reset
    return ctrl, changed


def run_case(w, rng, sizes, T, events, setdata):
    """Drive widget w through T calls; sizes = (K, K after the change).  setdata(w, y, fmax, fpitch,
    peaks, data_baseline) makes one call.  Returns the case's fixture arrays."""
    ctrl, changed = schedule(T, events, hasattr(w, "set_peaks_enabled"))
    ys = [db_sequence(rng, K, T) for K in sizes]
    out = {n: [] for n in ("K", "y", "sy", "z", "speak", "zpeak", "baseline", "fmax", "fpitch",
                           "fmax_x", "fpitch_x", "fmax_text", "fpitch_text")}
    for t in range(T):
        sm, sM, paused, peaks, data_base = ctrl[t]
        w.setspecrange(sm, sM)
        w.pause() if paused else w.restart()
        y = ys[int(changed[t])][t].astype(np.float64)
        K = len(y)
        fmax = float(np.linspace(0, FS // 2, K)[np.argmax(y)])
        fpitch = [1e-20, 65.4, 440.0, 1234.5, 20000.0][t % 5]
        setdata(w, y, fmax, fpitch, bool(peaks), bool(data_base))
        sig = curve_arrays(w._curve_signal)
        pk = curve_arrays(w._curve_peak)
        out["K"].append(K)
        out["y"].append(y.astype(np.float32))
        out["fmax"].append(fmax)
        out["fpitch"].append(fpitch)
        for n, a in (("sy", sig[2]), ("z", sig[3]), ("speak", pk[2]), ("zpeak", pk[3])):
            # the peak curve of a spectrum widget with peaks off keeps older arrays: not compared
            a = np.zeros(K) if a is None or np.size(a) != K else np.asarray(a, dtype=np.float64)
            out[n].append(a)
        out["baseline"].append(float(sig[4]))
        d = getattr(w, "_spectrum_data", None)      # the spectrum widget's trackers
        if d is not None:
            out["fmax_x"].append(float(d._fmax_logical_value))
            out["fpitch_x"].append(float(d._fpitch_value))
            out["fmax_text"].append(d._fmax_value)
            out["fpitch_text"].append(d._fpitch_display)
    res = {"ctrl": ctrl, "K": np.array(out["K"]), "y": np.concatenate(out["y"]),
           "fmax": np.array(out["fmax"]), "fpitch": np.array(out["fpitch"]),
           "baseline": np.array(out["baseline"]), "peak": w.peak, "peak_int": w.peak_int,
           "decay": w.peak_decay, "xl": np.asarray(sig[0], np.float64), "xr": np.asarray(sig[1], np.float64)}
    for n in ("sy", "z", "speak", "zpeak"):
        res[n] = np.concatenate(out[n])
    if out["fmax_x"]:
        res.update(fmax_x=np.array(out["fmax_x"]), fpitch_x=np.array(out["fpitch_x"]),
                   fmax_text=np.array(out["fmax_text"]), fpitch_text=np.array(out["fpitch_text"]))
    return res


def generate():
    """The fixture's arrays, from the unmodified reference."""
    spw, hp, fscales = reference_widgets()
    from oracle import ref_import
    ref = ref_import.load()
    scales = {s.NAME: s for s in fscales.ALL}
    gold = {}

    def spectrum_setdata(w, y, fmax, fpitch, peaks, data_base):
        if peaks != w.peaks_enabled:
            w.set_peaks_enabled(peaks)
        w.set_baseline_dataUnits(0.) if data_base else w.set_baseline_displayUnits(0.)
        w.setdata(np.linspace(0, FS // 2, len(y)), y, fmax, fpitch)   # x: the analyzer's freq

    for i, (name, scale, fmin, fmax, K, T, events) in enumerate(SPECTRUM):
        w = spw.SpectrumPlotWidget(None)
        w.set_peaks_enabled(True)             # as Spectrum_Widget's single-channel mode does
        w.setfreqscale(scales[scale])
        w.setfreqrange(fmin, fmax)
        # the bin count change is a change of FFT size: N -> 2N
        r = run_case(w, np.random.default_rng(100 + i), (K, 2 * K - 1), T, events, spectrum_setdata)
        r["settings"] = np.array([scale, str(fmin), str(fmax)])
        gold.update({"%s_%s" % (name, k): v for k, v in r.items()})

    for i, (name, bpo, T, events) in enumerate(OCTAVE):
        # the bin count change is a change of bands per octave: bpo -> 1
        filters = {len(f.flow): f for f in (ref.octavefilters.Octave_Filters(b) for b in (1, bpo))}

        def hist_setdata(w, y, fmax, fpitch, peaks, data_base):
            f = filters[len(y)]
            w.setdata(f.flow, f.fhigh, f.f_nominal, y)

        r = run_case(hp.HistPlot(None), np.random.default_rng(200 + i), (bpo * 9, 9), T, events,
                     hist_setdata)
        r["settings"] = np.array([str(bpo)])
        r["f_nominal"] = np.array(filters[bpo * 9].f_nominal)
        gold.update({"%s_%s" % (name, k): v for k, v in r.items()})
    return gold


def main():
    gold = generate()
    np.savez_compressed(OUT, **gold)
    print("wrote %s (%d keys, %.0f kB)" % (OUT, len(gold), os.path.getsize(OUT) / 1024))


if __name__ == "__main__":
    main()
