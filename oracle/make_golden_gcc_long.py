#!/usr/bin/env python
"""Generate tests/golden/gcc_long.npz by running the UNMODIFIED reference (imported in place via
oracle/ref_import.py).  TEST INFRASTRUCTURE ONLY; run in the build container:

    python oracle/make_golden_gcc_long.py

Two frames per length at 16800 (0.7 s), 55199 (2.3 s: odd, Xcorr has L-1 samples) and 240000
(10 s): generalized_cross_correlation (friture/signal/correlation.py:24-43), then the widget's
smoothing and peak pick (friture/delay_estimator.py:129-142).

The inputs are not stored: golden_frames() builds them with exact integer arithmetic (a counter
hash, no library random generator), so the tests rebuild the same float32 samples anywhere.  The
float64 outputs are incompressible, so the fixture keeps them at golden_indices(): every 61st
index and the 513 around the peak.  Stored per length: those indices, the first frame's Xcorr and
the smoothed Xcorr after the second frame there, the output length and both peaks."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_import  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "gcc_long.npz")
LENGTHS = (16800, 55199, 240000)
STRIDE = 61          # prime: the sampled indices meet every residue of small periods
PEAK_HALF = 256


def _hash(n, seed):
    """splitmix64 of seed + n (uint64 arrays wrap modulo 2^64: exact on every platform)."""
    z = (n.astype(np.uint64) + np.uint64(seed)) * np.uint64(0x9E3779B97F4A7C15)
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def _noise(L, seed):
    """Near-Gaussian integers: the sum of four 12-bit uniforms, centred (-8190 .. 8190)."""
    z = _hash(np.arange(L), seed)
    s = sum(((z >> np.uint64(16 * i)) & np.uint64(0xFFF)).astype(np.int64) for i in range(4))
    return s - 8190


def golden_frames(L):
    """Two float32 frames (d0, d1) of length L: d1 = d0 delayed by int(0.3 L) plus an eighth of
    independent noise, in 16-bit steps of 2^-12 (exact in float32); the second frame is the first
    one turned by L // 3 samples."""
    q0 = _noise(L, 2 * L)
    q1 = np.roll(q0, int(0.3 * L)) + (_noise(L, 2 * L + 1) >> 3)
    a0 = (q0.astype(np.float32) / np.float32(4096)).astype(np.float32)
    a1 = (q1.astype(np.float32) / np.float32(4096)).astype(np.float32)
    return (a0, a1), (np.roll(a0, L // 3), np.roll(a1, L // 3))


def golden_indices(n_out, peak):
    """Every STRIDE-th output index and the PEAK_HALF on either side of the peak, sorted."""
    near = np.arange(peak - PEAK_HALF, peak + PEAK_HALF + 1) % n_out
    return np.unique(np.concatenate([np.arange(0, n_out, STRIDE), near]))


def main():
    ref = ref_import.load()
    d = {}
    for L in LENGTHS:
        (a0, a1), (b0, b1) = golden_frames(L)
        # the reference subtracts the means in place: hand it float64 copies
        xa = ref.correlation.generalized_cross_correlation(a0.astype(np.float64), a1.astype(np.float64))
        xb = ref.correlation.generalized_cross_correlation(b0.astype(np.float64), b1.astype(np.float64))
        sm = 0.3 * xb + 0.7 * xa                                       # delay_estimator.py:134-139
        peaks = np.array([int(np.argmax(np.abs(xa))), int(np.argmax(np.abs(sm)))])
        idx = golden_indices(len(xa), int(peaks[1]))
        d["n_out_%d" % L] = len(xa)
        d["index_%d" % L] = idx.astype(np.int32)
        d["xcorr_%d" % L] = xa[idx]
        d["smoothed_%d" % L] = sm[idx]
        d["argmax_%d" % L] = peaks
    np.savez_compressed(OUT, **d)


if __name__ == "__main__":
    main()
