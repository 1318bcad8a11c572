#!/usr/bin/env python
"""The scope widget for many scopes (frt_scope_process, ScopeAnalyzer.handle_new_data).  Prints the
card and its power limit and, per shape and time range:
- the time per call from CUDA events over a window of at least 0.2 s of back-to-back calls, after
  warm-up, for the library call alone (on a staged buffer) and for the analyzer's handle_new_data,
  which also stages each scope's window history and the chunk and pushes the chunk into its ring;
- the bytes each must move, computed from the shape: the library reads the trigger channel's search
  windows once (w + (R-1)*buffer samples per scope; the crossing search reads on from each window's
  start to its first crossing, which depends on the signal and is not counted), reads and writes the
  drawn curve and writes the window starts; the analyzer adds the staging copy (the ring's window and
  the chunk read, the staged rows written) and the push (the chunk read, the ring written).  Their
  rate is given against the 3.35 TB/s HBM3 bandwidth of the H100 SXM data sheet;
- for comparison, the host route: the float64 NumPy restatement of the widget (oracle/scope.py, a
  loop over scopes and ticks) timed on 8 scopes and scaled to S.

    python tools/perf_scope.py [--buffers 96]
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from perf_levels import HBM_PEAK, card, host_s, per_call_s  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--buffers", type=int, default=96)
    args = ap.parse_args()
    import torch
    from friture_b200 import _lib
    from friture_b200.scope import ScopeAnalyzer, is_trigger, scope_points, scope_width
    from oracle.scope import ScopeOracle

    R, N = args.buffers, 512
    T = R * N
    name, pl = card()
    print("card: %s, power limit / max SM clock: %s" % (name, pl))
    results = []
    for S, nch in ((1024, 1), (512, 2)):
        g = torch.Generator(device="cuda").manual_seed(S)
        t = torch.arange(T, device="cuda", dtype=torch.float64) / 48000.
        f = 100 + 2000 * torch.rand((S, nch, 1), generator=g, device="cuda", dtype=torch.float64)
        x = (0.5 * torch.sin(2 * np.pi * f * t) + 0.05 * torch.randn((S, nch, T), generator=g, device="cuda",
                                                                      dtype=torch.float64)).float()
        x = x[:, 0] if nch == 1 else x
        xh = x[:8].cpu().numpy().reshape(8, nch, T)
        for tr in (50, 500, 10000):
            a = ScopeAnalyzer(S, two_channels=nch == 2, timerange=tr)
            for _ in range(3):
                a.handle_new_data(x)
            w, trig, pts = scope_width(tr), is_trigger(tr), scope_points(tr)
            need = 2 * w if trig else w
            rows = S * nch
            staged = torch.cat(a._read(need) + [x.reshape(rows, T)], dim=1)
            start = torch.empty((S, R), dtype=torch.int64, device="cuda")
            sp = _lib.current_stream_ptr()
            lib_s = per_call_s(lambda: a.handle.call(
                "frt_scope_process", _lib._ptr(staged), staged.shape[1], S, nch, need, R, N, w, int(trig), 0,
                _lib._ptr(start), _lib._ptr(a._curve), a._curve.shape[1], float(tr), _lib._ptr(a._drawn), sp))
            call_s = per_call_s(lambda: a.handle_new_data(x))
            lib_bytes = (4 * S * (w + (R - 1) * N) * trig + 2 * 4 * rows * pts + 8 * S * R)
            call_bytes = lib_bytes + 4 * rows * (2 * (need + T)) + 4 * rows * 2 * T
            o = ScopeOracle(8, two_channels=nch == 2, timerange=tr)
            host = host_s(lambda: [o.handle_new_data(xh[:, :, r * N:(r + 1) * N]) for r in range(R)], 8, S)
            results.append(dict(S=S, channels=nch, timerange_ms=tr, buffers=R, buffer=N, width=w, points=pts,
                                lib_bytes=lib_bytes, lib_call_s=lib_s, lib_hbm_share=lib_bytes / lib_s / HBM_PEAK,
                                call_bytes=call_bytes, handle_new_data_s=call_s,
                                call_hbm_share=call_bytes / call_s / HBM_PEAK,
                                realtime_factor=T / 48000 / call_s, host_route_s=host))
            print(json.dumps(results[-1]), flush=True)
            del a, staged


if __name__ == "__main__":
    main()
