"""Spectrogram widget: the fused path (frt_stft_screen_rows + frt_display_rows) against the two-call
path (frt_stft_process LOGPOWER + frt_display_columns) on the same frames, alternated in one process,
timed with CUDA events over windows of at least --window seconds after a warm-up.  Prints the bytes of
each path's per-frame intermediate (computed from the shapes), the card and its power limit, both
paths' times and whether their pixels are identical.

    python tools/perf_spectrogram.py [--channels 1024] [--sizes 4096 16384] [--height 512]
"""
import argparse
import os
import subprocess
import sys

import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
from friture_b200 import _lib  # noqa: E402
from friture_b200.audioproc import audioproc  # noqa: E402
from friture_b200.display import SpectrogramDisplay  # noqa: E402
from friture_b200.spectrogram import SpectrogramAnalyzer  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name()


def timed(fn, window):
    """Mean time of one fn() over repeats filling at least `window` seconds (CUDA events)."""
    fn()
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    fn()
    e.record()
    e.synchronize()
    reps = max(1, int(window * 1e3 / max(s.elapsed_time(e), 1e-3)))
    s.record()
    for _ in range(reps):
        fn()
    e.record()
    e.synchronize()
    return s.elapsed_time(e) / reps * 1e-3


def run(C, N, H, W, seconds, window, rounds):
    hop = N // 4
    F = int(seconds * 48000) // hop
    T = N + (F - 1) * hop
    g = torch.Generator(device="cuda").manual_seed(N)
    x = 0.1 * torch.randn(C, T, device="cuda", generator=g)
    nb = N // 2 + 1
    kw = dict(fft_size=N, height=H, width=W, timerange_s=seconds)
    two, fused = SpectrogramDisplay(C, **kw), SpectrogramDisplay(C, **kw)
    proc = audioproc()
    proc.set_fftsize(N)
    db = torch.empty((C, F, nb), device="cuda")
    rows = torch.empty((C, F, H), device="cuda")
    an = SpectrogramAnalyzer(C, **kw)      # the fused path's screen-row call, as the analyzer makes it
    T_f = fused.tables(x.device)

    def path_two():
        proc.stft(x, hop, log=True, out=db)
        return two.push(db)

    def path_fused():
        h = an.handle
        h.call("frt_stft_plan", N)
        h.call("frt_stft_screen_rows", _lib._ptr(x), T, C, F, hop, _lib._ptr(T_f["w"]),
               _lib.c_float(fused.spec_min), _lib.c_float(fused.spec_max), _lib._ptr(T_f["i0"]),
               _lib._ptr(T_f["t"]), H, _lib._ptr(rows), F * H, H, _lib.current_stream_ptr())
        return fused.push_rows(rows)

    same = torch.equal(path_two(), path_fused()) and torch.equal(two._old, fused._old)
    t_two, t_fused = [], []
    for _ in range(rounds):
        t_two.append(timed(path_two, window))
        t_fused.append(timed(path_fused, window))
    print("C=%d N=%d hop=%d H=%d W=%d %.0f s: %d frames per channel" % (C, N, hop, H, W, seconds, F))
    print("  intermediate per frame: two-call %d B (the LOGPOWER column), fused %d B (the screen rows)"
          % (4 * nb, 4 * H))
    print("  two-call %.3f ms (min of %d), fused %.3f ms (min of %d), ratio %.2f; pixels identical: %s" % (
        1e3 * min(t_two), rounds, 1e3 * min(t_fused), rounds, min(t_two) / min(t_fused), same))
    return same


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--channels", type=int, default=1024)
    ap.add_argument("--sizes", type=int, nargs="+", default=[4096, 16384])
    ap.add_argument("--height", type=int, default=512)
    ap.add_argument("--width", type=int, default=1024)
    ap.add_argument("--seconds", type=float, default=10.)
    ap.add_argument("--window", type=float, default=0.2)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("perf_spectrogram: needs a CUDA device")
    print("card:", card())
    ok = True
    for N in a.sizes:
        ok &= run(a.channels, N, a.height, a.width, a.seconds, a.window, a.rounds)
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
