"""CPU checks of the STFT kernels' decompositions (friture_b200/csrc/stft.cu) through the executable
model in stft_layout_model.py: lane/register layouts, split-step partners, the on-the-fly Hann
window and the conflict-free 8-byte scatter, against numpy.fft."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import stft_layout_model as m  # noqa: E402


def reference(x):
    n = x.shape[-1]
    return np.abs(np.fft.rfft(x * m.hann(n))) ** 2 / n ** 2      # friture/audioproc.py:42-50


@pytest.mark.parametrize("Q", [1, 2, 4, 8, 16, 32])
def test_small_kernel_layout(Q):
    G, N = 32 // Q, 64 * Q
    x = np.random.default_rng(Q).standard_normal((G, N))
    got = m.small_frames(x, Q)
    ref = reference(x)
    assert got.shape == ref.shape
    assert np.max(np.abs(got - ref)) < 1e-12 * np.max(ref)


@pytest.mark.parametrize("Q", [2, 4, 8, 16, 32])
def test_small_kernel_partner_identity(Q):
    """bin of (lane, register m) + bin of (partner lane, register 31 - m) = M for k1 > 0."""
    M = 32 * Q
    for lane in range(32):
        g, k1 = divmod(lane, Q)
        if k1 == 0:
            continue
        src = g * Q + (Q - k1) % Q
        for mm in range(16):
            assert (k1 + Q * mm) + ((src % Q) + Q * (31 - mm)) == M


@pytest.mark.parametrize("R", [2, 4])
def test_large_kernel_layout(R):
    N = 2048 * R
    x = np.random.default_rng(R).standard_normal(N)
    got = m.large_frame(x, R)
    ref = reference(x)
    assert np.max(np.abs(got - ref)) < 1e-10 * np.max(ref)


@pytest.mark.parametrize("R", [2, 4])
def test_on_the_fly_window_is_the_symmetric_hann(R):
    assert np.max(np.abs(m.hann_on_the_fly(R) - m.hann(2048 * R))) < 1e-12


@pytest.mark.parametrize("R", [2, 4])
def test_scatter_is_bank_conflict_free_per_half_warp(R):
    """8-byte shared accesses are served per half-warp: the 16 elements a half-warp scatters must
    fall on 16 different 8-byte bank pairs of the 128-byte bank line."""
    tile_bytes = m.TILE * 8
    for base in range(0, 1024 * R, 16):
        pairs = set()
        for e in range(base, base + 16):
            w, pos = m.scatter_position(e, R)
            pairs.add(((w * tile_bytes + pos * 8) % 128) // 8)
        assert len(pairs) == 16
    # and every element lands inside its tile, below the region the transposes use afterwards
    for e in range(1024 * R):
        w, pos = m.scatter_position(e, R)
        assert 0 <= pos < m.TILE
