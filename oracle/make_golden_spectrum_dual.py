#!/usr/bin/env python
"""Generate tests/golden/spectrum_dual.npz by running the UNMODIFIED reference (imported in place
via oracle/ref_import.py).  TEST INFRASTRUCTURE ONLY; run where the reference tree exists:

    python oracle/make_golden_spectrum_dual.py

Writes that one file and leaves the other fixtures untouched.

The spectrum widget's two-channel tick (friture/spectrum.py:141-182): the reference's own
`audioproc.analyzelive` and `exp_smoothed_value_2d` (friture/signal/exp_smoothing.py:59-107), with
the widget's framing, alpha and kernel (spectrum.py:137-155,196-222), its dual / single branches
and its A weighting restated (the widget itself imports PyQt6).  One seeded float32 stereo stream:
channel 1 is channel 0 through a short FIR and a delay, plus independent noise.  Per (N, T) case a
schedule of (frames, dual) ticks that switches dual -> single -> dual; per tick the shown dB,
peak and pitch indices and both smoothed states dispbuffers1 / dispbuffers2.
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_import  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "spectrum_dual.npz")
FS = 48000
FIR = np.array([0.5, -0.25, 0.125, 0.0625])      # channel 1 = FIR(channel 0) delayed by DELAY
DELAY = 37
SCHEDULES = {                                     # (frames, dual) per tick
    1024: [(1, True), (7, True), (3, False), (12, False), (5, True), (9, True)],
    8192: [(1, True), (3, False), (2, True)],
}
RESPONSE_TIMES = (0.125, 1.0)


def stereo_stream(n):
    rng = np.random.default_rng(2718)
    t = np.arange(n) / float(FS)
    x0 = 0.05 * rng.standard_normal(n) + sum(0.3 / k * np.sin(2 * np.pi * 440.0 * k * t) for k in (1, 2, 3))
    x1 = np.zeros(n)
    x1[DELAY:] = np.convolve(x0, FIR)[:n - DELAY]
    x1 += 0.01 * rng.standard_normal(n)
    return np.stack([x0, x1]).astype(np.float32)


def main():
    ref = ref_import.load()
    from friture.signal.exp_smoothing import exp_smoothed_value_2d
    n = max(N + (sum(f for f, _ in s) - 1) * N // 4 for N, s in SCHEDULES.items())
    x = stereo_stream(n)
    d = {"x": x, "fir": FIR, "delay": np.int64(DELAY)}
    for N, schedule in SCHEDULES.items():
        proc = ref.audioproc.audioproc()
        proc.set_fftsize(N)
        freq = proc.get_freq_scale()
        w = proc.get_freq_weighting()[0]                                  # A
        hop = N * (1. - 3. / 4.)                                          # spectrum.py:137
        for T in RESPONSE_TIMES:
            alpha = 1. - (1. - 0.65) ** (1. / (T * FS / hop + 1))         # spectrum.py:213-218
            kernel = (1. - alpha) ** np.arange(2 * 4096 - 1, -1, -1)
            disp1, disp2 = np.zeros(len(freq)), np.zeros(len(freq))
            pos = 0
            out = {k: [] for k in ("db", "imax", "ipitch", "sp1", "sp2")}
            for frames, dual in schedule:
                sp1n = np.zeros((len(freq), frames))
                sp2n = np.zeros((len(freq), frames))
                for i in range(frames):
                    floatdata = x[:, pos:pos + N].astype(np.float64)
                    sp1n[:, i] = proc.analyzelive(floatdata[0, :])
                    if dual:
                        sp2n[:, i] = proc.analyzelive(floatdata[1, :])
                    pos += int(hop)
                disp1 = exp_smoothed_value_2d(kernel, alpha, sp1n, disp1)
                disp2 = exp_smoothed_value_2d(kernel, alpha, sp2n, disp2)
                if dual:
                    db = 10. * np.log10(disp2 + 1e-30) - 10. * np.log10(disp1 + 1e-30)
                else:
                    db = 10. * np.log10(disp1 + 1e-30) + w
                hps = disp1[:len(freq) // 3] * disp1[::2][:len(freq) // 3] * disp1[::3][:len(freq) // 3]
                for k, v in (("db", db), ("imax", np.argmax(db)), ("ipitch", np.argmax(hps)),
                             ("sp1", disp1), ("sp2", disp2)):
                    out[k].append(v)
            key = "N%d_t%d" % (N, round(T * 1000))
            d["alpha_" + key] = np.float64(alpha)
            d["frames_" + key] = np.array([f for f, _ in schedule])
            d["dual_" + key] = np.array([m for _, m in schedule])
            for k, v in out.items():
                d["%s_%s" % (k, key)] = np.array(v)
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    np.savez_compressed(OUT, **d)
    print(OUT, os.path.getsize(OUT))


if __name__ == "__main__":
    main()
