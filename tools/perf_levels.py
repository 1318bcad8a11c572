#!/usr/bin/env python
"""The levels widget's meter and the long-term levels widget for many channels
(frt_levels_process, frt_longlevels_process).  Prints the card and its power limit and, per shape:
- the time per call from CUDA events over a window of at least 0.2 s of back-to-back calls, after
  warm-up, for the library call alone and for the analyzer's handle_new_data (which for the
  long-term widget also copies the chunk into its stream buffer);
- the bytes the kernel must move (each sample read once, the per-buffer or per-block outputs
  written), computed from the shape, and their rate against the 3.35 TB/s HBM3 bandwidth of the H100
  SXM data sheet;
- for comparison, the host route: the float64 NumPy restatement of the widgets
  (oracle/levels.py, element-wise across channels) timed on 8 channels and scaled to C.

    python tools/perf_levels.py [--channels 1024] [--buffers 480]
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
WINDOW_S = 0.2


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit,clocks.max.sm", "--format=csv,noheader"],
                            capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:      # the figure is then reported as unknown, not guessed
        pl = "unknown (%s)" % e
    return name, pl


def per_call_s(fn):
    """Seconds per call over a window of at least WINDOW_S of back-to-back calls, after warm-up."""
    import torch
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    reps = 1
    while True:
        t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        t0.record()
        for _ in range(reps):
            fn()
        t1.record()
        torch.cuda.synchronize()
        s = t0.elapsed_time(t1) / 1e3
        if s >= WINDOW_S:
            return s / reps
        reps *= 2


def host_s(fn, C_host, C):
    t0 = time.perf_counter()
    fn()
    return (time.perf_counter() - t0) * C / C_host


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--channels", type=int, default=1024)
    ap.add_argument("--buffers", type=int, default=480)
    args = ap.parse_args()
    import torch
    from friture_b200 import _lib
    from friture_b200.levels import LevelsAnalyzer, LongLevelsAnalyzer
    from oracle.levels import LevelsOracle, LongLevelsOracle

    C, R, N = args.channels, args.buffers, 512
    T = R * N
    name, pl = card()
    print("card: %s, power limit / max SM clock: %s" % (name, pl))
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn((C, T), generator=g, device="cuda") * 0.1
    xh = x[:8].cpu().numpy()
    results = []

    # meter: R buffers of 512 samples per channel and call
    a = LevelsAnalyzer(C)
    a.handle_new_data(x, buffer=N)
    outs = [torch.empty((C, R), dtype=torch.float64, device="cuda") for _ in range(3)]
    sp = _lib.current_stream_ptr()
    lib_s = per_call_s(lambda: a.handle.call("frt_levels_process", _lib._ptr(x), T, R,
                                             *(_lib._ptr(o) for o in outs), sp))
    call_s = per_call_s(lambda: a.handle_new_data(x, buffer=N))
    o = LevelsOracle(8)
    host = host_s(lambda: [o.handle_new_data(xh[:, r * N:(r + 1) * N]) for r in range(R)], 8, C)
    nbytes = 4 * C * T + 3 * 8 * C * R
    results.append(dict(widget="levels", C=C, buffers=R, buffer=N, bytes=nbytes, lib_call_s=lib_s,
                        handle_new_data_s=call_s, hbm_share=nbytes / lib_s / HBM_PEAK,
                        realtime_factor=T / 48000 / lib_s, host_route_s=host))

    # long-term levels at rt = 1 s (256-sample blocks) and 20 s (8192-sample blocks)
    for rt in (1, 20):
        b = LongLevelsAnalyzer(C, response_time=rt, duration=600)
        nblk = T // b.needed
        b.handle_new_data(x)
        b._plan()
        lv = torch.empty((C, nblk), dtype=torch.float64, device="cuda")
        db = torch.empty_like(lv)
        lib_s = per_call_s(lambda: b.handle.call("frt_longlevels_process", _lib._ptr(x), T, nblk, _lib._ptr(lv),
                                                 _lib._ptr(db), _lib._ptr(b._ring), b._ring_len, 0, sp))
        call_s = per_call_s(lambda: b.handle_new_data(x))
        curve_s = per_call_s(lambda: b.curve())
        ol = LongLevelsOracle(8, response_time=rt, duration=600)
        host = host_s(lambda: ol.handle_new_data(xh), 8, C)
        nbytes = 4 * C * T + 2 * 8 * C * nblk + 4 * C * nblk
        results.append(dict(widget="longlevels", rt=rt, C=C, blocks=nblk, block=b.needed, bytes=nbytes,
                            lib_call_s=lib_s, handle_new_data_s=call_s, curve_s=curve_s,
                            curve_length=b.length_samples, hbm_share=nbytes / lib_s / HBM_PEAK,
                            realtime_factor=T / 48000 / lib_s, host_route_s=host))
    for r in results:
        print(json.dumps(r))


if __name__ == "__main__":
    main()
