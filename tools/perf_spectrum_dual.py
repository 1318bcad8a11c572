#!/usr/bin/env python
"""The spectrum widget's dual-channel tick for many pairs: the STFT over the 2P rows, the dual
reduce over the P pairs (frt_spectrum_reduce_dual) and, for comparison, the single-channel reduce
over the same 2P channels' power (frt_spectrum_reduce), timed alternately with CUDA events after
warm-up.  Prints the card and its power limit, each kernel's time, and the reduces' algorithmic
bytes over time against the 3.35 TB/s HBM3 bandwidth of the H100 SXM data sheet.

    python tools/perf_spectrum_dual.py [--pairs 512] [--fft-size 8192] [--frames 16] [--rounds 5]
"""
import argparse
import json
import os
import subprocess
import sys
from ctypes import c_float

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


def reduce_bytes(channels, frames, nbins, db_rows):
    """Power read once, states read and written, dB written, two indices per output row."""
    return 4 * (channels * frames * nbins + 2 * channels * nbins + db_rows * nbins) + 8 * db_rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--pairs", type=int, default=512)
    ap.add_argument("--fft-size", type=int, default=8192)       # the widget's default
    ap.add_argument("--frames", type=int, default=16)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        sys.exit("perf_spectrum_dual: no CUDA device")
    from friture_b200 import _lib
    from friture_b200.spectrum import SpectrumAnalyzer
    name, pl = card()
    print("card: %s   power.limit, clocks.max.sm: %s" % (name, pl), flush=True)

    P, N, F = args.pairs, args.fft_size, args.frames
    an = SpectrumAnalyzer(P, fft_size=N, response_time=0.125, dual_channels=True)
    h, hop, nb = an.proc.handle, an.hop, N // 2 + 1
    T = N + (F - 1) * hop
    g = torch.Generator(device="cuda").manual_seed(P)
    x = torch.randn((P, 2, T), generator=g, device="cuda") * 0.1
    rows = x.view(2 * P, T)
    power = torch.empty((2 * P, F, nb), dtype=torch.float32, device="cuda")
    alpha = c_float(an.alpha)
    st = _lib.current_stream_ptr()
    ptr = _lib._ptr
    d1, d2 = (torch.zeros((P, nb), device="cuda") for _ in range(2))
    dbd = torch.empty((P, nb), device="cuda")
    i1, i2 = (torch.empty(P, dtype=torch.int32, device="cuda") for _ in range(2))
    ds = torch.zeros((2 * P, nb), device="cuda")
    dbs = torch.empty((2 * P, nb), device="cuda")
    j1, j2 = (torch.empty(2 * P, dtype=torch.int32, device="cuda") for _ in range(2))

    def stft():
        an.proc.stft(rows, hop=hop, log=False, out=power)

    def dual():
        h.call("frt_spectrum_reduce_dual", ptr(power), ptr(power.data_ptr() + 4 * F * nb), 2 * F * nb, nb,
               P, F, nb, alpha, ptr(d1), ptr(d2), ptr(dbd), ptr(i1), ptr(i2), st)

    def single():
        h.call("frt_spectrum_reduce", ptr(power), F * nb, nb, 2 * P, F, nb, alpha, ptr(ds), None,
               ptr(dbs), ptr(j1), ptr(j2), st)

    stft()
    dual()
    single()
    torch.cuda.synchronize()
    same = bool(torch.equal(ds[0::2], d1) and torch.equal(ds[1::2], d2))
    for fn in (stft, dual, single):          # warm-up
        for _ in range(5):
            fn()
    torch.cuda.synchronize()
    times = {"stft": [], "reduce_dual": [], "reduce_single": []}
    for _ in range(args.rounds):
        for key, fn in (("stft", stft), ("reduce_dual", dual), ("reduce_single", single)):
            times[key].append(time_cuda(fn, args.reps))
    med = {k: float(np.median(v)) for k, v in times.items()}
    b_dual = reduce_bytes(2 * P, F, nb, P)
    b_single = reduce_bytes(2 * P, F, nb, 2 * P)
    print(json.dumps({
        "card": name, "power_limit_and_max_sm_clock": pl, "pairs": P, "fft_size": N, "frames": F,
        "stft_ms": med["stft"] * 1e3, "reduce_dual_ms": med["reduce_dual"] * 1e3,
        "reduce_single_2P_ms": med["reduce_single"] * 1e3,
        "reduce_dual_bytes": b_dual, "reduce_single_bytes": b_single,
        "reduce_dual_hbm_frac": b_dual / med["reduce_dual"] / HBM_PEAK,
        "reduce_single_hbm_frac": b_single / med["reduce_single"] / HBM_PEAK,
        "states_bit_identical_dual_vs_single": same,
        "spread_ms": {k: [round(v * 1e3, 4) for v in vs] for k, vs in times.items()},
    }))


if __name__ == "__main__":
    main()
