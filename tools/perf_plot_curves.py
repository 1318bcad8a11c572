#!/usr/bin/env python
"""The spectrum and octave widgets' plotted curves and peak hold for many channels
(frt_plot_curves): the spectrum widget's tick (one dB vector per channel) and the octave widget's
call (one dB vector per channel and block).  Prints the card and its power limit and, per shape:
- the kernel's device time from torch.profiler, averaged over many launches in a run of its own;
- the time per call from CUDA events over a window of at least 0.2 s of back-to-back calls;
- the algorithmic bytes (each dB value read once, the float64 state read and written, the four
  float32 curves written) and their rate against the 3.35 TB/s HBM3 bandwidth of the H100 SXM data
  sheet, on the profiler's kernel time;
- the whole SpectrumPlot.push / HistPlot.push (host clock around the call and a device
  synchronise), and, for the spectrum, the tracker text of all channels formatted on access;
- for comparison, the host route: the D2H copy of the dB stack, then a float64 NumPy setdata +
  compute_peaks per channel and step (oracle.plot_curves.PlotCurvesOracle, timed on a few channels
  and scaled to C).

    python tools/perf_plot_curves.py [--channels 1024] [--rounds 5]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_PEAK = 3.35e12     # H100 SXM data sheet, bytes/s


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                            capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:      # the figure is then reported as unknown, not guessed
        pl = "unknown (%s)" % e
    return name, pl


def time_cuda(fn, reps):
    import torch
    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(reps):
        fn()
    t1.record()
    torch.cuda.synchronize()
    return t0.elapsed_time(t1) / 1e3 / reps


def kernel_bytes(C, S, K):
    """dB read once, the float64 state read and written, four float32 curves written."""
    return 4 * C * S * K + 2 * 3 * 8 * C * K + 4 * 4 * C * K


def profiled_kernel_s(fn, launches):
    """Mean device time of plot_curves_kernel over `launches` calls, from torch.profiler, and the
    number of launches the profiler recorded."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(launches):
            fn()
        torch.cuda.synchronize()
    d = [e.time_range.elapsed_us() for e in prof.events() if "plot_curves_kernel" in e.name]
    if not d:
        raise RuntimeError("profiler saw none of %d plot_curves_kernel launches" % launches)
    return float(np.mean(d)) * 1e-6, len(d)


def host_clock_s(fn, reps):
    """Seconds per call of fn, host clock, ending in a device synchronise."""
    import torch
    torch.cuda.synchronize()
    t = time.perf_counter()
    for _ in range(reps):
        fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t) / reps


def host_route(db, steps, probe=8):
    """Seconds for the D2H copy of db [C, S, K] and for the per-channel NumPy steps, scaled to C."""
    import torch
    from oracle.plot_curves import PlotCurvesOracle
    torch.cuda.synchronize()
    t = time.perf_counter()
    host = db.cpu().numpy()
    d2h = time.perf_counter() - t
    C = db.shape[0]
    orcs = [PlotCurvesOracle(-100, -20) for _ in range(probe)]
    for o, c in zip(orcs, range(probe)):      # warm-up (first call resets the state)
        o.setdata(host[c, 0].astype(np.float64))
    t = time.perf_counter()
    for o, c in zip(orcs, range(probe)):
        for s in range(steps):
            o.setdata(host[c, s].astype(np.float64))
    per_channel = (time.perf_counter() - t) / probe
    return d2h, per_channel * C


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--channels", type=int, default=1024)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--window", type=float, default=0.2, help="seconds per CUDA-event window")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("perf_plot_curves: no CUDA device")
    from ctypes import c_double
    from friture_b200 import _lib
    from friture_b200.octavespectrum import OctaveSpectrumAnalyzer
    from friture_b200.plotcurves import PEAK_DECAY, HistPlot, SpectrumPlot, _PlotState
    h, ptr, sp = _lib.default_handle(), _lib._ptr, _lib.current_stream_ptr()
    name, pl = card()
    print("card: %s   power.limit, clocks.max.sm: %s" % (name, pl), flush=True)
    C = args.channels
    # spectrum widget default N = 8192 (4097 bins), one dB vector per tick; octave widget at bpo 3
    # and 24 over 9 octaves, 64 blocks of 512 samples per call
    shapes = {"spectrum_N8192": (1, 4097, None), "octave_bpo3_64blocks": (64, 27, 3),
              "octave_bpo24_64blocks": (64, 216, 24)}
    g = torch.Generator(device="cuda").manual_seed(C)
    fmax = np.linspace(20., 20000., C)
    results = {}
    for key, (S, K, bpo) in shapes.items():
        db = (torch.randn((C, S, K), generator=g, device="cuda") * 10 - 70).float()
        st = _PlotState(C, -100, -20, None)
        st._run(db, True)                       # allocates and resets the state
        out = [torch.empty((C, K), device="cuda") for _ in range(4)]
        args_ = [ptr(db), S * K, K, C, S, K, c_double(-100.), c_double(-20.), c_double(PEAK_DECAY), 1, 0,
                 ptr(st.peak), ptr(st.peak_int), ptr(st.peak_decay)] + [ptr(t) for t in out]
        fn = lambda: h.call("frt_plot_curves", *args_, sp)      # noqa: E731
        for _ in range(5):
            fn()
        torch.cuda.synchronize()
        once = time_cuda(fn, 20)
        reps = max(50, int(args.window / once))
        times = [time_cuda(fn, reps) for _ in range(args.rounds)]
        per_call = float(np.median(times))
        kern, seen = profiled_kernel_s(fn, 200)
        b = kernel_bytes(C, S, K)
        if bpo is None:
            plot = SpectrumPlot(C)
            push = lambda: plot.push(db[:, 0], fmax, fmax)      # noqa: E731
        else:
            plot = HistPlot(C, OctaveSpectrumAnalyzer(C, bandsperoctave=bpo))
            push = lambda: plot.push(db)                        # noqa: E731
        push()
        push_s = host_clock_s(push, 50)
        r = {"channels": C, "steps": S, "bins": K, "kernel_ms": kern * 1e3, "kernel_launches_profiled": seen,
             "events_ms_per_call": per_call * 1e3, "events_reps_per_window": reps, "bytes": b,
             "hbm_frac": b / kern / HBM_PEAK, "spread_ms": [round(v * 1e3, 4) for v in times],
             "push_ms": push_s * 1e3}
        if bpo is None:
            c = push()
            t = time.perf_counter()
            c.fmax_text, c.fpitch_text
            r["tracker_text_all_channels_ms"] = (time.perf_counter() - t) * 1e3
        d2h, host = host_route(db, S)
        r.update(host_d2h_ms=d2h * 1e3, host_numpy_steps_ms=host * 1e3)
        results[key] = r
        print(key, json.dumps(r), flush=True)
    print(json.dumps({"card": name, "power_limit_and_max_sm_clock": pl, "shapes": results}))


if __name__ == "__main__":
    main()
