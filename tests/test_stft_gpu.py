"""GPU parity: fused STFT kernels (through the C ABI) vs the CPU oracle on the same inputs."""
import numpy as np
import os
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

pytestmark = pytest.mark.gpu

from parity import TOL, assert_logpower_parity, assert_power_parity  # noqa: E402


def make_input(kind, C, T, seed):
    rng = np.random.default_rng(seed)
    if kind == "randn":
        return (rng.standard_normal((C, T)) * 0.1).astype(np.float32)
    if kind == "uniform":
        return rng.uniform(-1, 1, (C, T)).astype(np.float32)
    if kind == "sine":
        t = np.arange(T) / 48000.0
        return (0.5 * np.sin(2 * np.pi * 1000.0 * t)[None, :]
                + 1e-3 * rng.standard_normal((C, T))).astype(np.float32)
    if kind == "zeros":
        return np.zeros((C, T), dtype=np.float32)
    raise ValueError(kind)


def run_gpu(x, n_fft, hop, log):
    import torch
    from friture_b200 import audioproc
    proc = audioproc()
    proc.set_fftsize(n_fft)
    return proc.stft(torch.from_numpy(x).cuda(), hop=hop, log=log).cpu().numpy().astype(np.float64)


@pytest.mark.parametrize("n_fft", [32, 64, 128, 256, 512, 1024, 2048, 4096, 8192, 16384])
def test_power_all_sizes(n_fft):
    from oracle import friture_oracle as fo
    x = make_input("randn", 3, n_fft + 5 * (n_fft // 4), seed=n_fft)
    got = run_gpu(x, n_fft, n_fft // 4, log=False)       # 75 % overlap (spectrum.py:66)
    ref = fo.stft_power_batch(x, n_fft, n_fft // 4)
    assert got.shape == ref.shape
    assert_power_parity(got, ref)
    got = run_gpu(x, n_fft, n_fft // 4, log=True)
    # few bins per frame at the small sizes: allow more of them below the floor
    assert_logpower_parity(got, fo.log_spectrogram(ref), min_frac=0.95 if n_fft < 1024 else 0.9999)


@pytest.mark.parametrize("kind", ["randn", "uniform"])
@pytest.mark.parametrize("hop", [1024, 512, 2048, 1000, 333])
def test_logpower_2048(kind, hop):
    from oracle import friture_oracle as fo
    x = make_input(kind, 5, 2048 + 9 * hop, seed=7)
    got = run_gpu(x, 2048, hop, log=True)
    ref = fo.log_spectrogram(fo.stft_power_batch(x, 2048, hop))
    assert got.shape == ref.shape == (5, 10, 1025)
    assert_logpower_parity(got, ref)


def test_config2_shape_sample():
    """BASELINE config #2 geometry (256 ch, N=2048, hop 1024) on a 64-hop stream."""
    from oracle import friture_oracle as fo
    x = make_input("randn", 256, 1024 * 65, seed=1234)
    got = run_gpu(x, 2048, 1024, log=True)
    ref = fo.log_spectrogram(fo.stft_power_batch(x, 2048, 1024))
    assert got.shape == (256, 64, 1025)
    e = assert_logpower_parity(got, ref)
    print("config #2 sample parity:", e)


def test_tonal_above_floor():
    """Pure tone: bins far below the tone are float32 rounding noise relative to the frame's
    rms (SURVEY 7), so the log-power criterion applies down to 50 dB below the mean power and
    the noise-floor allowance of tests/parity.py below that."""
    from oracle import friture_oracle as fo
    x = make_input("sine", 2, 2048 * 4, seed=3)
    got = run_gpu(x, 2048, 1024, log=True)
    ref = fo.log_spectrogram(fo.stft_power_batch(x, 2048, 1024))
    e = assert_logpower_parity(got, ref, min_frac=0.0, strict=False, floor_db=40.0)
    peak = ref >= ref.max() - 30.0
    assert np.max(np.abs(got[peak] - ref[peak])) / max(np.max(np.abs(ref)), 1.0) < TOL, e


def test_zeros_is_minus_300_db():
    got = run_gpu(make_input("zeros", 2, 4096, 0), 2048, 1024, log=True)
    assert np.all(np.abs(got + 300.0) < 1e-3)


def test_empty_and_short_inputs():
    import torch
    from friture_b200 import audioproc
    proc = audioproc()
    proc.set_fftsize(2048)
    assert tuple(proc.stft(torch.zeros(3, 100).cuda(), hop=1024).shape) == (3, 0, 1025)
    assert tuple(proc.stft(torch.zeros(0, 4096).cuda(), hop=1024).shape) == (0, 3, 1025)


def test_analyzelive_dropin_plumbing():
    """BASELINE config #1: 1 ch, 1024-pt, one frame, host NumPy in/out through the shim."""
    from friture_b200 import audioproc
    from oracle import friture_oracle as fo
    rng = np.random.default_rng(11)
    x = rng.standard_normal(1024) * 0.1
    proc = audioproc()
    proc.set_fftsize(1024)
    sp = proc.analyzelive(x)
    assert sp.dtype == np.float64 and sp.shape == (513,)
    ref = fo.analyzelive(x.astype(np.float32))
    assert_logpower_parity(10 * np.log10(sp + 1e-30), fo.log_spectrogram(ref))
    assert_power_parity(sp, ref)
    with pytest.raises(ValueError):
        proc.analyzelive(x[:100])


def test_host_path_matches_device_path():
    import torch
    from friture_b200 import audioproc
    x = make_input("randn", 7, 2048 + 40 * 1024, seed=5)
    proc = audioproc()
    proc.set_fftsize(2048)
    a = proc.stft(torch.from_numpy(x).cuda(), hop=1024).cpu().numpy()
    b = proc.stft_host(x, hop=1024)
    assert np.array_equal(a, b)
    xp = torch.from_numpy(x).pin_memory()
    c = proc.stft_host(xp, hop=1024)
    assert np.array_equal(a, c.numpy())


def test_unaligned_input_uses_scalar_loads():
    import torch
    from friture_b200 import audioproc
    from oracle import friture_oracle as fo
    x = make_input("randn", 2, 2048 * 3 + 1, seed=9)
    proc = audioproc()
    proc.set_fftsize(2048)
    xd = torch.from_numpy(x).cuda()[:, 1:]          # odd offset -> 4-byte aligned only
    got = proc.stft(xd, hop=1024).cpu().numpy().astype(np.float64)
    ref = fo.log_spectrogram(fo.stft_power_batch(x[:, 1:], 2048, 1024))
    assert_logpower_parity(got, ref)


def test_plan_cache_alternating_sizes():
    """Two processors of different FFT sizes sharing one handle (as the spectrum and spectrogram
    widgets would) can be called alternately; the handle keeps one plan per size."""
    import torch
    from friture_b200 import audioproc
    from oracle import friture_oracle as fo
    x = make_input("randn", 2, 8192 + 3 * 2048, seed=21)
    xd = torch.from_numpy(x).cuda()
    pa, pb = audioproc(), audioproc()
    pa.set_fftsize(8192)
    pb.set_fftsize(4096)
    assert pa.handle is pb.handle
    for _ in range(3):
        a = pa.stft(xd, hop=2048).cpu().numpy().astype(np.float64)
        b = pb.stft(xd, hop=1024).cpu().numpy().astype(np.float64)
    assert_logpower_parity(a, fo.log_spectrogram(fo.stft_power_batch(x, 8192, 2048)))
    assert_logpower_parity(b, fo.log_spectrogram(fo.stft_power_batch(x, 4096, 1024)))


@pytest.mark.parametrize("n_fft,hop,C,F", [(64, 32, 5, 71), (128, 64, 3, 45), (256, 100, 7, 37), (512, 256, 9, 33),
                                           (1024, 512, 7, 37), (1024, 333, 2, 19), (4096, 2048, 7, 37),
                                           (8192, 4096, 5, 23), (8192, 1024, 3, 150), (4096, 1001, 2, 11)])
def test_ragged_frame_counts_all_kernels(n_fft, hop, C, F):
    """Frame counts that do not divide into the kernels' frame groups / warps, odd hops (scalar or
    unaligned-load paths), many channels: every size class against the oracle."""
    from oracle import friture_oracle as fo
    x = make_input("randn", C, n_fft + (F - 1) * hop, seed=n_fft + hop)
    got = run_gpu(x, n_fft, hop, log=False)
    ref = fo.stft_power_batch(x, n_fft, hop)
    assert got.shape == ref.shape == (C, F, n_fft // 2 + 1)
    assert_power_parity(got, ref)
    got = run_gpu(x, n_fft, hop, log=True)
    assert_logpower_parity(got, fo.log_spectrogram(ref), min_frac=0.95 if n_fft < 1024 else 0.9999)


def test_large_sizes_unaligned_input_falls_back():
    import torch
    from friture_b200 import audioproc
    from oracle import friture_oracle as fo
    x = make_input("randn", 2, 4096 * 3 + 1, seed=19)
    proc = audioproc()
    proc.set_fftsize(4096)
    xd = torch.from_numpy(x).cuda()[:, 1:]          # 4-byte aligned only
    got = proc.stft(xd, hop=2048).cpu().numpy().astype(np.float64)
    assert_logpower_parity(got, fo.log_spectrogram(fo.stft_power_batch(x[:, 1:], 4096, 2048)))
