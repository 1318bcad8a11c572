#!/usr/bin/env python
"""GCC-PHAT between channels of one frame: the pair path (PairGccPhat: each channel transformed
once) against the per-pair path (the pairs' rows copied with index_select, then GccPhat on the two
row sets), alternated in one run, timed with CUDA events after warm-up.  Cases: all pairs of
M = 16 and M = 64 channels at L = 24 000 (shared-memory route) and 240 000 (Bluestein route), and
the M - 1 pairs against channel 0 at M = 256, L = 24 000.  Prints one JSON line per case, the
median of the rounds for each path, and the card's name and power limit read in the same run."""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

from friture_b200.correlation import GccPhat, PairGccPhat  # noqa: E402

CASES = [("all", 16, 24000), ("all", 64, 24000), ("all", 16, 240000), ("all", 64, 240000),
         ("vs0", 256, 24000)]


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, IndexError, subprocess.SubprocessError):
        return torch.cuda.get_device_name(0) + ", power limit unknown"


def table(kind, M):
    if kind == "all":
        return [(i, j) for i in range(M) for j in range(i + 1, M)]
    return [(0, j) for j in range(1, M)]


def timed(fn, reps):
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(reps):
        fn()
    stop.record()
    stop.synchronize()
    return start.elapsed_time(stop) / reps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--min-ms", type=float, default=200.0, help="time per path and round")
    args = ap.parse_args()
    print(json.dumps({"card": card()}), flush=True)
    for kind, M, L in CASES:
        pairs = table(kind, M)
        P = len(pairs)
        x = torch.randn(M, L, device="cuda")
        i0 = torch.tensor([p[0] for p in pairs], device="cuda")
        i1 = torch.tensor([p[1] for p in pairs], device="cuda")
        pair_est = PairGccPhat(L, M, pairs)
        rows_est = GccPhat(L)

        def pair_path():
            pair_est.estimate(x, smooth=False)

        def rows_path():
            rows_est.estimate(x.index_select(0, i0), x.index_select(0, i1), smooth=False)

        a = pair_est.estimate(x, smooth=False)[0]      # warm-up, and the same peaks both ways
        b = rows_est.estimate(x.index_select(0, i0), x.index_select(0, i1), smooth=False)[0]
        rows_path()
        ms = max(timed(pair_path, 1), timed(rows_path, 1))
        reps = max(1, int(args.min_ms / max(ms, 1e-3)))
        t_pair, t_rows = [], []
        for _ in range(args.rounds):
            t_pair.append(timed(pair_path, reps))
            t_rows.append(timed(rows_path, reps))
        med = lambda t: sorted(t)[len(t) // 2]
        print(json.dumps({"case": "%s pairs of M=%d" % (kind, M), "L": L, "pairs": P, "reps": reps,
                          "pair_path_ms": round(med(t_pair), 3), "per_pair_path_ms": round(med(t_rows), 3),
                          "speedup": round(med(t_rows) / med(t_pair), 2),
                          "pair_path_ms_all": [round(t, 3) for t in t_pair],
                          "per_pair_path_ms_all": [round(t, 3) for t in t_rows],
                          "same_peaks": bool(torch.equal(a, b))}), flush=True)
        del x, pair_est, rows_est
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
