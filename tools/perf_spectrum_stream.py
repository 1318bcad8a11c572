"""The spectrum widget fed from the stream: SpectrumAnalyzer.handle_new_data(chunk, buffer=512) (each
frame's power column smoothed on chip, frt_spectrum_frames) against process_ticks on the same frames
(an STFT launch writing every power column, then the chain and stats kernels of
frt_spectrum_reduce_ticks), with and without the dB rows.

    python tools/perf_spectrum_stream.py [--channels 1024] [--rounds 20]

One call is one second of 512-sample buffers (93 buffers, 47616 samples per channel) at 48 kHz; the
same chunk is pushed on every call.  process_ticks gets the frames the first call cuts (zeros before
the stream, as the widget's framing gives), one tick per buffer: one frame per tick at N >= 2048,
512 / hop frames per tick below.  The two routes are timed alternately in the same run with CUDA
events around each whole call (host work and the index reads included), median of the rounds, after
a warm-up of each.  The byte model is from
shapes: HBM bytes a route must move per call beyond reading its input once, over the call's time,
against the H100 SXM data sheet's 3.35 TB/s.  The card's name and power limit are read in the same run.
"""
import argparse
import os
import subprocess
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from friture_b200.spectrum import SpectrumAnalyzer  # noqa: E402

HBM_BPS = 3.35e12
BUFFERS = 93   # one second of 512-sample buffers at 48 kHz


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        out = ""
    return out or torch.cuda.get_device_name(0) + ", power limit unknown"


def event_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def case(C, N, want_db, rounds):
    n = 512 * BUFFERS
    g = torch.Generator(device="cuda").manual_seed(N)
    x = torch.randn(C, n, device="cuda", generator=g) * 0.1
    stream = SpectrumAnalyzer(C, fft_size=N)
    ticks = SpectrumAnalyzer(C, fft_size=N)
    hop, nb = stream.hop, N // 2 + 1
    per_tick = max(512 // hop, 1)   # frames a 512-sample buffer cuts: 1 for N >= 2048, 512 / hop below
    # the frames process_ticks gets: those the first call cuts, per_tick per tick.  Frame f ends at
    # old_index = f hop, with zeros before the stream starts.
    first = stream.handle_new_data(x, buffer=512, want_db=want_db)
    F = int(first.n_frames.sum())
    assert np.all(first.n_frames == per_tick)
    frames = torch.cat([torch.zeros(C, N, device="cuda"), x], dim=1)[:, :(F - 1) * hop + N].contiguous()
    check = SpectrumAnalyzer(C, fft_size=N).process_ticks(frames, frames_per_tick=per_tick, want_db=True)
    assert np.array_equal(check.fmax_hz, first.fmax_hz)     # the same frames, the same peaks

    def run_stream():
        return stream.handle_new_data(x, buffer=512, want_db=want_db)

    def run_ticks():
        return ticks.process_ticks(frames, frames_per_tick=per_tick, want_db=want_db)

    run_stream()
    run_ticks()
    t_s, t_t = [], []
    for _ in range(rounds):   # alternating
        t_s.append(event_ms(run_stream))
        t_t.append(event_ms(run_ticks))
    F_s = int(run_stream().n_frames.sum())   # frames per call in steady state
    ms_s, ms_t = float(np.median(t_s)), float(np.median(t_t))
    row = 4 * nb
    # beyond the input: fused = the dB rows (+ both ends of the state once per call); ticks = the power
    # column written and read, the state row written and read, the dB rows written
    b_s = C * (F_s * (row if want_db else 0) + 2 * row)
    b_t = C * F * (4 * row + (row if want_db else 0)) + C * 2 * row
    b_in = 4 * C * n
    return dict(C=C, N=N, db=want_db, frames_per_call=F_s, stream_ms=ms_s, ticks_ms=ms_t,
                speedup=ms_t / ms_s, model_bytes_per_channel_frame_stream=b_s / (C * F_s),
                model_bytes_per_channel_frame_ticks=b_t / (C * F),
                stream_share_of_hbm=(b_s + b_in) / (ms_s * 1e-3) / HBM_BPS,
                ticks_share_of_hbm=(b_t + 4 * C * ((F - 1) * hop + N)) / (ms_t * 1e-3) / HBM_BPS)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--channels", type=int, default=1024)
    ap.add_argument("--rounds", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("needs a GPU")
    print("card: %s" % card())
    print("%5s %6s %3s %7s %10s %10s %7s %12s %12s %8s %8s" % (
        "C", "N", "dB", "frames", "stream ms", "ticks ms", "ratio", "B/ch-frame s", "B/ch-frame t",
        "HBM% s", "HBM% t"))
    for N in (8192, 2048, 1024, 256, 128, 64):
        for want_db in (True, False):
            r = case(args.channels, N, want_db, args.rounds)
            print("%5d %6d %3s %7d %10.3f %10.3f %7.2f %12.0f %12.0f %8.1f %8.1f" % (
                r["C"], r["N"], "yes" if r["db"] else "no", r["frames_per_call"], r["stream_ms"], r["ticks_ms"],
                r["speedup"], r["model_bytes_per_channel_frame_stream"], r["model_bytes_per_channel_frame_ticks"],
                100 * r["stream_share_of_hbm"], 100 * r["ticks_share_of_hbm"]))


if __name__ == "__main__":
    main()
