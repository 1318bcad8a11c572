"""Delay estimation over many frames: one GccPhat.estimate call per frame followed by what the delay
estimators published per frame before estimate_frames existed (torch.std of the smoothed buffer
and three device-to-host reads), against one estimate_frames call and its three reads.

    python tools/perf_delay_track.py [--rounds 3]

Frames overlap by half (the widget's hop L/2).  Times are CUDA events around the whole route, after
one warm-up run of each, median of the rounds; the card's name and power limit are printed with them.
"""
import argparse
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from friture_b200.correlation import GccPhat  # noqa: E402

SHAPES = [(1, 1200, 24000), (1, 120, 240000), (64, 64, 24000), (4096, 4, 24000)]


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return out or torch.cuda.get_device_name(0) + ", power limit unknown"


def per_frame(g, d0, d1, hop, F, L):
    out = []
    for f in range(F):
        idx, val, _ = g.estimate(d0[:, f * hop:f * hop + L], d1[:, f * hop:f * hop + L])
        std = torch.std(g._smoothed.double(), dim=1, unbiased=False)
        out.append((idx.cpu(), val.cpu(), std.cpu()))
    return out


def frames(g, d0, d1, hop, F, L):
    idx, val, std = g.estimate_frames(d0, d1, hop, F)
    return idx.cpu(), val.cpu(), std.cpu()


def timed(fn, rounds):
    fn()
    ms = []
    for _ in range(rounds):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
    return float(np.median(ms))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    print("card: %s" % card())
    print("| pairs | frames | L | per-frame route ms | estimate_frames ms | ratio |")
    print("|---|---|---|---|---|---|")
    for P, F, L in SHAPES:
        hop = L // 2
        T = (F - 1) * hop + L
        g = torch.Generator(device="cuda").manual_seed(P + F)
        d0 = torch.randn((P, T), generator=g, device="cuda")
        d1 = torch.roll(d0, 37, dims=1) + 0.1 * torch.randn((P, T), generator=g, device="cuda")
        est_a, est_b = GccPhat(L), GccPhat(L)
        t_a = timed(lambda: per_frame(est_a, d0, d1, hop, F, L), args.rounds)
        t_b = timed(lambda: frames(est_b, d0, d1, hop, F, L), args.rounds)
        print("| %d | %d | %d | %.2f | %.2f | %.1fx |" % (P, F, L, t_a, t_b, t_a / t_b), flush=True)
        del d0, d1, est_a, est_b
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
