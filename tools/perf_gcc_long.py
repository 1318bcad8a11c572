#!/usr/bin/env python
"""Rates of GCC-PHAT's Bluestein route (friture_b200/csrc/gcc_long.cu) with CUDA events after
warm-up, at L = 16800, 26400, 55199, 240000, 2.4e6 and 24e6, lengths GccPhat runs on that route.
Prints one JSON line per case plus the card's name and power limit read in the same run.

Two byte counts per case, each over 3.35 TB/s (H100 SXM HBM3): the algorithmic bytes (the 2L
floats of input, plus L' floats of smoothed buffer read and written) and the traffic the passes
of the kernels actually move (workspace, tables, inputs, outputs; see traffic())."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from friture_b200.correlation import GccPhat  # noqa: E402

HBM = 3.35e12


def fft_points(L):
    return 1 << int(2 * L - 2).bit_length()


def traffic(L):
    """Bytes one pair's call moves through memory: per transform a column pass (write the M-point
    workspace), a row pass (read it, read B^, write it) and a column pass back (read it); plus the
    inputs, window, chirps, the cross-spectrum G and the outputs with smoothing."""
    M, Lp = fft_points(L), L - (L & 1)
    H = Lp // 2 + 1
    ws = 2 * (8 * M + 3 * 8 * M + 8 * M)
    tables = 4 * L + 8 * L + 8 * L + 8 * Lp + 8 * Lp        # window, chirp (two passes), chirp'
    io = 8 * L + 8 * L + 8 * L                              # means pass, first load, Z store
    g = 3 * 8 * H + 8 * H                                   # split reads Z twice, writes G; PHAT load
    out = 3 * 4 * Lp                                        # smoothed read and write, Xcorr write
    return ws + tables + io + g + out


def algorithmic(L):
    Lp = L - (L & 1)
    return 2 * L * 4 + 2 * Lp * 4


def time_calls(est, d0, d1, iters):
    est.estimate(d0, d1, smooth=True)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(iters):
        est.estimate(d0, d1, smooth=True)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / iters


def inputs(P, L, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    d0 = torch.randn(P, L, device="cuda", generator=g)
    d1 = torch.roll(d0, L // 7, 1) + 0.1 * torch.randn(P, L, device="cuda", generator=g)
    return d0, d1


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default=None, help="also write the JSON lines to this file")
    args = ap.parse_args()
    card = torch.cuda.get_device_name(0)
    try:
        power = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except OSError:
        power = "unknown"
    lines = [{"card": card, "power_limit": power}]
    for L in (16800, 26400, 55199, 240000, 2400000, 24000000):
        # enough pairs for about 2^28 workspace points (at least 8 column CTAs per SM), at most 4096
        P = max(2, min(4096, (1 << 28) // fft_points(L)))
        d0, d1 = inputs(P, L)
        ms = time_calls(GccPhat(L), d0, d1, args.iters)
        lines.append({"path": "long", "L": L, "pairs": P, "ms_per_call": round(ms, 4),
                      "pairs_per_s": P / ms * 1e3,
                      "algorithmic_share_of_hbm": P * algorithmic(L) / (ms * 1e-3) / HBM,
                      "pass_traffic_share_of_hbm": P * traffic(L) / (ms * 1e-3) / HBM})
        del d0, d1
        torch.cuda.empty_cache()
    for ln in lines:
        print(json.dumps(ln))
    if args.out:
        with open(args.out, "w") as f:
            f.write("\n".join(json.dumps(ln) for ln in lines) + "\n")


if __name__ == "__main__":
    main()
