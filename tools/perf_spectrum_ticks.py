"""The spectrum widget over many ticks: one SpectrumAnalyzer.process call per tick (an STFT launch, a
reduction launch and two device-to-host reads each) against one process_ticks call and its two reads.

    python tools/perf_spectrum_ticks.py [--rounds 5] [--lib OTHER/libfrt_b200.so]

Each tick has the widget's default frames (one 512-sample buffer: one frame at N >= 2048).  Times are
CUDA events around the whole route, after one warm-up run of each, median of the rounds; the card's
name and power limit are printed with them.

It also times one tick's reduction alone, at the shapes above with their default frames and at the
multi-GPU bench's tick (1024 channels, N = 2048, hop 1024, one tick of 128 frames), two ways: with
frt_spectrum_reduce, which process uses, and as a one-tick frt_spectrum_reduce_ticks call.  Both run
in this tree's library and, given --lib, in another build of it (e.g. the parent commit's), in ABBA
order, after a check that every way gives the same bits (rows, indices, state) on the same power.
"""
import argparse
import ctypes
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from friture_b200 import _lib  # noqa: E402
from friture_b200.spectrum import SpectrumAnalyzer  # noqa: E402

# (channels or pairs, FFT size, ticks, dual)
CASES = [(1, 8192, 2000, False), (1024, 2048, 64, False), (256, 8192, 64, True)]
# (channels, FFT size, frames) of the one-tick reductions: the cases' ticks and the multi-GPU bench's
REDUCE_SHAPES = [(C, N, max(1, 512 // (N // 4))) for C, N, _, _ in CASES] + [(1024, 2048, 128)]


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return out or torch.cuda.get_device_name(0) + ", power limit unknown"


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


def per_tick(an, x, g, R):
    span = g * an.hop + an.fft_size - an.hop
    for r in range(R):
        an.process(x[..., r * g * an.hop:r * g * an.hop + span])


def one_tick_reduce(lib_path, ticks, C, nb, g):
    """One tick of g frames ([C, g, nb] seeded power, seeded state) through the library at lib_path,
    with frt_spectrum_reduce or (ticks) a one-tick frt_spectrum_reduce_ticks call: (run, outputs,
    close) with run() making 20 calls and outputs the rows, indices and state after one."""
    lib = ctypes.CDLL(lib_path)
    name = "frt_spectrum_reduce_ticks" if ticks else "frt_spectrum_reduce"
    fn = getattr(lib, name)
    fn.restype, fn.argtypes = _lib.SIGNATURES[name]
    lib.frt_create.argtypes = [ctypes.c_int, ctypes.POINTER(ctypes.c_void_p)]
    lib.frt_destroy.argtypes = [ctypes.c_void_p]
    h = ctypes.c_void_p()
    assert lib.frt_create(torch.cuda.current_device(), ctypes.byref(h)) == 0
    gen = torch.Generator(device="cuda").manual_seed(C + nb + g)
    power = torch.rand((C, g, nb), generator=gen, device="cuda")
    disp = torch.rand((C, nb), generator=gen, device="cuda")
    db = torch.empty((C, nb), device="cuda")
    idx = torch.empty((2, C), dtype=torch.int32, device="cuda")
    shape = [g, 1] if ticks else [g]
    st = _lib.current_stream_ptr()

    def once():
        rc = fn(h, _lib._ptr(power), g * nb, nb, C, *shape, nb, ctypes.c_float(0.1), _lib._ptr(disp), None,
                _lib._ptr(db), _lib._ptr(idx[0]), _lib._ptr(idx[1]), st)
        assert rc == 0

    once()
    torch.cuda.synchronize()
    outputs = [db.clone().view(torch.int32), idx.clone(), disp.clone().view(torch.int32)]

    def run():
        for _ in range(20):
            once()

    def close():
        torch.cuda.synchronize()
        lib.frt_destroy(h)
    return run, outputs, close


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--lib", help="another build of libfrt_b200.so to time the one-tick reductions with")
    args = ap.parse_args()
    print("card: %s" % card())
    print("| channels | N | mode | ticks | per-tick route ms | process_ticks ms | ratio |")
    print("|---|---|---|---|---|---|---|")
    for C, N, R, dual in CASES:
        an_a = SpectrumAnalyzer(C, fft_size=N, dual_channels=dual)
        an_b = SpectrumAnalyzer(C, fft_size=N, dual_channels=dual)
        g = an_a.default_frames_per_tick()
        T = R * g * an_a.hop + N - an_a.hop
        gen = torch.Generator(device="cuda").manual_seed(C + N)
        x = torch.randn((C, 2, T) if dual else (C, T), generator=gen, device="cuda")
        t_a = timed(lambda: per_tick(an_a, x, g, R), args.rounds)
        t_b = timed(lambda: an_b.process_ticks(x, frames_per_tick=g), args.rounds)
        print("| %d | %d | %s | %d | %.2f | %.2f | %.1fx |" % (C, N, "dual" if dual else "single", R, t_a, t_b,
                                                               t_a / t_b), flush=True)
        del x, an_a, an_b
        torch.cuda.empty_cache()
    libs = [("this tree", _lib.lib_path())] + ([("--lib", args.lib)] if args.lib else [])
    ways = [(lib, ticks) for lib in libs for ticks in (False, True)]
    print()
    print("one tick's reduction, us per call, median of the rounds in ABBA order; the same bits every way:")
    print("| channels | N | frames | " + " | ".join("%s, %s" % (n, "one-tick _ticks" if t else "reduce")
                                                   for (n, _), t in ways) + " |")
    print("|---|---|---|" + "---|" * len(ways))
    for C, N, g in REDUCE_SHAPES:
        runs = [one_tick_reduce(p, t, C, N // 2 + 1, g) for (_, p), t in ways]
        for _, outputs, _ in runs[1:]:
            assert all(torch.equal(a, b) for a, b in zip(runs[0][1], outputs)), (C, N, g)
        ms = [[] for _ in runs]
        for k in range(args.rounds):
            for i in (range(len(runs)) if k % 2 == 0 else reversed(range(len(runs)))):
                ms[i].append(timed(runs[i][0], 1) / 20)
        for _, _, close in runs:
            close()
        print("| %d | %d | %d | %s |" % (C, N, g, " | ".join("%.1f" % (1e3 * np.median(m)) for m in ms)), flush=True)


if __name__ == "__main__":
    main()
