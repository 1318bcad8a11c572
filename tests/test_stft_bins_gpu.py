"""Every STFT kernel instance (friture_b200/csrc/stft.cu) bin by bin, in both output modes, at every
frame alignment, at the frame edges and in every layout the C ABI accepts.

Power mode is held to ``parity.assert_power_parity`` (a per-bin amplitude bound relative to the
frame rms and the bin's own level, exact zero for a silent frame).  Log mode is held to
``parity.assert_logpower_parity`` and to its power twin on the same buffer:
    |L - 10 log10(P + 1e-30)| <= LOG_TWIN_DB + LOG_TWIN_ULPS ulp(L)
L is kLog10Scale * lg2.approx(fmaf(|X|^2, scale, 1e-30)) and P = |X|^2 * scale.  The ulps cover the
rounding of lg2's float32 result (up to 1 ulp of L once scaled by 10/log2(10)), of kLog10Scale and
of the final product: a correctly rounded log2 in their place already reaches 1.46 ulp(L) (numpy
emulation over 1e-36 .. 1e2), and lg2.approx is not correctly rounded.  LOG_TWIN_DB covers
lg2.approx's absolute error (2^-22 in log2, 7.2e-7 dB) and the two float32 roundings of the power
(the fmaf in log mode, the product in power mode: 2.6e-7 dB each).  Measured on an H100 80GB HBM3 at
a 400 W power limit the difference reaches 1.92 x (2e-6 dB + 1 ulp(L)).

Which instance runs a case comes from ``test_stft_dispatch_gpu.kernel_for`` (that file checks it
under the profiler); ``test_grid_reaches_every_instance`` fails on the CPU when an instance has no
case here.  The CPU tests (no mark) check that the power bound accepts a float32 transform and
rejects plausible bugs, among them the window stft_large_kernel computed on the fly up to this
change (0.5 - 0.5 cos(theta n) cancels at both ends of the frame)."""
import json
import os
import sys
from ctypes import c_void_p

import numpy as np
import pytest

from oracle import friture_oracle as fo

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from parity import (AMP_TOL, REL_AMP_TOL, assert_logpower_parity, assert_power_parity,  # noqa: E402
                    power_errors)
from test_stft_dispatch_gpu import INSTANCES, LOGPOWER, POWER, kernel_for  # noqa: E402

SIZES = [2 ** k for k in range(5, 15)]          # 32 .. 16384, every size frt_stft_plan accepts
MODES = (POWER, LOGPOWER)
ALIGN_OFFSET = {16: 0, 8: 2, 4: 1}              # frame alignment in bytes -> offset in floats mod 4
SOURCES = ("offset", "stride", "hop")           # frame_alignment's three inputs
LOG_TWIN_DB = 4e-6
LOG_TWIN_ULPS = 3
SENTINEL = 0x7FC5A5A5                           # a quiet-NaN bit pattern no kernel computes

CASES = [(n, mode, align) for n in SIZES for mode in MODES for align in ALIGN_OFFSET]


def cos_bins(n):
    """Bin-centred cosines: DC, bin 1, M/2, M-1 and Nyquist (M = N/2); for the R-warp kernels also
    bin 512 (the k0 = 512 group) and 1024 q +- 1 (next to each combine boundary)."""
    m = n // 2
    ks = {0, 1, m // 2, m - 1, m}
    if n >= 4096:
        ks |= {512} | {1024 * q + d for q in range(1, n // 2048) for d in (-1, 1)}
    return sorted(ks)


def test_grid_reaches_every_instance():
    assert {kernel_for(n, mode, align) for n, mode, align in CASES} == INSTANCES


# --------------------------------------------------------------------------- CPU: the power bound
def f32_power(frames, n, window=None):
    """|rfft|^2 / N^2 of float32-windowed frames by numpy's float32 transform."""
    w = (fo.hann_window(n) if window is None else window).astype(np.float32)
    X = np.fft.rfft((frames * w).astype(np.float32), axis=-1)
    assert X.dtype == np.complex64
    p = (X.real * X.real + X.imag * X.imag).astype(np.float32) * np.float32(1.0 / n ** 2)
    return p.astype(np.float64)


def bound_inputs(n, rng):
    t = np.arange(n)
    F = max(4, 2 ** 16 // n)
    return {
        "noise": (rng.standard_normal((F, n)) * 0.1).astype(np.float32),
        "tone": (0.5 * np.sin(2 * np.pi * (n / 8 + 0.3) * t / n)[None]
                 + 1e-4 * rng.standard_normal((F, n))).astype(np.float32),
        "cosines": np.stack([np.cos(2 * np.pi * k * t / n) for k in cos_bins(n)]).astype(np.float32),
        "nyquist": ((-1.0) ** t)[None].astype(np.float32),
        "impulses": np.eye(n, dtype=np.float32)[1:-1:max(1, n // 64)],
    }


def ref_power(frames):
    return np.stack([fo.analyzelive(r) for r in frames])


@pytest.mark.parametrize("n", SIZES)
def test_power_bound_accepts_float32_transform(n):
    for kind, x in bound_inputs(n, np.random.default_rng(n)).items():
        e = power_errors(f32_power(x, n), ref_power(x))
        assert e["worst_ratio"] < 0.2, (kind, e)


def swapped_partner_power(x, n):
    """The split step pairing X[k] with X[M - k]'s partner: the spectrum mirrored about M/2."""
    p = f32_power(x, n)
    m = n // 2
    p[..., 1:m] = p[..., m - 1:0:-1]
    return p


@pytest.mark.parametrize("n", [64, 2048, 4096, 16384])
def test_power_bound_rejects_bugs(n):
    """Each structural bug exceeds the bound 50x or more on the inputs of the GPU tests (a
    one-sample shift, for one, shows on noise and impulses but hardly on a long steady tone); a
    uniform 1e-5 relative power error exceeds it on noise and on a tone alone."""
    rng = np.random.default_rng(n + 1)
    t = np.arange(n)
    periodic = 0.5 * (1 - np.cos(2 * np.pi * t / n))
    worst = {}
    for kind, x in bound_inputs(n, rng).items():
        ref = ref_power(x)
        bugs = {"periodic Hann": f32_power(x, n, periodic),
                "one-sample shift": f32_power(np.roll(x, 1, axis=-1), n)}
        if kind == "nyquist":
            p = f32_power(x, n)
            p[..., -1] *= 4
            bugs["Nyquist bin x4"] = p
        if kind in ("noise", "tone"):
            bugs["swapped split partner"] = swapped_partner_power(x, n)
            p = f32_power(x, n) * (1 + 1e-5)
            assert power_errors(p, ref)["worst_ratio"] > 1.5, (kind, "1e-5 relative power error")
        for bug, p in bugs.items():
            worst[bug] = max(worst.get(bug, 0.0), power_errors(p, ref)["worst_ratio"])
    assert len(worst) == 4 and min(worst.values()) > 50, worst


def fma32(a, b, c):
    """float32 fmaf: the product of two float32 values is exact in float64."""
    return (np.float64(a) * np.float64(b) + np.float64(c)).astype(np.float32)


def large_kernel_window(R, table_blocks=()):
    """stft_large_kernel's float32 window for N = 2048 R: w[n] = 0.5 - 0.5 cos(theta n) from the
    constant-bank (0.5 cos A, 0.5 sin A) of register block n1 and the lane's (cos B, sin B),
    n = 64 R n1 + 2 R t + 2 w + e.  Blocks in table_blocks take float32(Hann) instead."""
    N = 2048 * R
    theta = 2 * np.pi / (N - 1)
    exact = fo.hann_window(N)
    out = np.zeros(N, dtype=np.float32)
    b = theta * np.arange(64 * R)                  # 2 R t + 2 w + e runs over 0 .. 64 R - 1
    cb, sb = np.cos(b).astype(np.float32), np.sin(b).astype(np.float32)
    for n1 in range(32):
        idx = 64 * R * n1 + np.arange(64 * R)
        if n1 in table_blocks:
            out[idx] = exact[idx].astype(np.float32)
            continue
        a = theta * 64 * R * n1
        ca, sa = np.float32(0.5 * np.cos(a)), np.float32(0.5 * np.sin(a))
        out[idx] = fma32(sa, sb, fma32(-ca, cb, np.float32(0.5)))
    return out


@pytest.mark.parametrize("R", [2, 4])
def test_power_bound_rejects_on_the_fly_window_at_frame_edges(R):
    """An impulse at the last sample must give exactly zero power, and one at n = 1 the power of
    w[1]; the on-the-fly window misses both.  Reading float32(Hann) in register blocks 0 and 31
    (what the kernel does now) passes the bound at every sample position."""
    n = 2048 * R
    exact = fo.hann_window(n)
    for pos in (1, 2, 8, n - 9, n - 2, n - 1):
        x = np.zeros((1, n), dtype=np.float32)
        x[0, pos] = 0.75
        ref = ref_power(x)
        p = f32_power(x, n, large_kernel_window(R).astype(np.float64))
        assert power_errors(p, ref)["worst_ratio"] > (100 if pos in (1, n - 1) else 1.5), pos
        p = f32_power(x, n, large_kernel_window(R, (0, 31)).astype(np.float64))
        assert power_errors(p, ref)["worst_ratio"] < 0.2, pos
    # closed form over all positions: an impulse's spectrum is flat, (a w[n])^2 / N^2
    fixed = large_kernel_window(R, (0, 31)).astype(np.float64)
    inner = slice(1, n - 1)
    rel = np.abs(fixed[inner] - exact[inner]) / exact[inner]
    assert fixed[0] == 0 and fixed[-1] == 0
    assert rel.max() < 0.5 * (AMP_TOL + REL_AMP_TOL), rel.max()


# --------------------------------------------------------------------------- GPU helpers
WORST = {}          # (kernel, check) -> worst ratio to its bound over the module


@pytest.fixture(scope="module", autouse=True)
def report_worst():
    yield
    if WORST:
        print("\nworst ratio to the bound per instance:")
        print(json.dumps({"%s | %s" % k: round(v, 4) for k, v in sorted(WORST.items())}, indent=1))


def note(kernel, check, ratio):
    WORST[(kernel, check)] = max(WORST.get((kernel, check), 0.0), float(ratio))


def handle():
    from friture_b200._lib import default_handle
    return default_handle()


def stream():
    import torch
    return c_void_p(torch.cuda.current_stream().cuda_stream)


def process(h, n, x_ptr, x_stride, C, F, hop, out, osc, osf, mode):
    h.call("frt_stft_plan", int(n))
    h.call("frt_stft_process", c_void_p(int(x_ptr)), int(x_stride), int(C), int(F), int(hop),
           c_void_p(out.data_ptr()), int(osc), int(osf), int(mode), stream())


def run_dense(h, n, xd, x_off, x_stride, C, F, hop, mode):
    """[C, F, N/2+1] float32 output of one frt_stft_process call on device buffer xd, frame 0 of
    channel 0 at element x_off."""
    import torch
    nb = n // 2 + 1
    out = torch.empty((C, F, nb), dtype=torch.float32, device="cuda")
    assert xd.data_ptr() % 16 == 0
    process(h, n, xd.data_ptr() + 4 * x_off, x_stride, C, F, hop, out, F * nb, nb, mode)
    return out


def check_log(kernel, got_db, got_p, ref_p, log_parity=True, **parity_kw):
    """Log output against its power twin and (log_parity) against the float64 reference."""
    got_db = np.asarray(got_db, dtype=np.float32)
    twin = 10 * np.log10(np.asarray(got_p, dtype=np.float64) + 1e-30)
    allowed = LOG_TWIN_DB + LOG_TWIN_ULPS * np.spacing(np.abs(got_db)).astype(np.float64)
    ratio = float(np.max(np.abs(got_db.astype(np.float64) - twin) / allowed))
    note(kernel, "log vs power twin", ratio)
    assert ratio <= 1.0, ratio
    if log_parity:
        e = assert_logpower_parity(got_db, fo.log_spectrogram(ref_p), **parity_kw)
        note(kernel, "log parity", e["worst_ratio_all"])


def check_power(kernel, got, ref):
    e = assert_power_parity(got, ref)
    note(kernel, "power bound", e["worst_ratio"])


def run_both_modes(h, n, align, xd, x_off, x_stride, C, F, hop, ref, log_parity=True, **parity_kw):
    """Power and log on the same buffer, both held to their bounds; returns the power output."""
    got = {}
    for mode in MODES:
        got[mode] = run_dense(h, n, xd, x_off, x_stride, C, F, hop, mode).cpu().numpy()
    check_power(kernel_for(n, POWER, align), got[POWER], ref)
    check_log(kernel_for(n, LOGPOWER, align), got[LOGPOWER], got[POWER], ref, log_parity, **parity_kw)
    return got[POWER]


def min_frac(n):
    """Share of noise bins that must lie within FLOOR_DB of their frame's mean power: a few
    thousand bins hold one deeper null now and then, whatever computed them.  Those nulls are also
    why the log checks of noise here are not strict; the power bound holds every bin."""
    return 0.95 if n < 1024 else 0.99


def frames_per_case(n):
    """A frame count that is not a multiple of stft_small_kernel's frame group (G = 32/Q frames
    per warp) where G > 1."""
    return 32 // (n // 64) + 3 if 64 <= n <= 1024 else 5


def sweep_layout(n, source, align):
    """(offset of frame 0 mod 4, row stride, hop, channels, frames) with the alignment class set by
    one of frame_alignment's three inputs; the hop case steps frames further than N apart."""
    cls = ALIGN_OFFSET[align]
    C, F = 3, frames_per_case(n)
    hop = n // 4
    if source == "hop":
        hop = n + 4 + cls
        cls = 0
    row = n + (F - 1) * hop
    stride = (row + 7) // 4 * 4 + 8          # row padding, a multiple of 4
    if source == "offset":
        return cls, stride, hop, C, F
    if source == "stride":
        return 0, stride + cls, hop, C, F
    return 0, stride, hop, C, F


# --------------------------------------------------------------------------- GPU: the sweep
@pytest.mark.gpu
@pytest.mark.parametrize("source", SOURCES)
@pytest.mark.parametrize("n", SIZES)
def test_sweep_poisoned_input_padded_output(n, source):
    """Every alignment class set through each of frame_alignment's inputs.  Every input sample no
    frame covers (before frame 0, between frames, row padding) is NaN.  The output goes to a padded
    layout (out_stride_f = nbins + 3, out_stride_c = F out_stride_f + 7) prefilled with SENTINEL:
    every bin must be written and every pad must keep its bits."""
    import torch
    h = handle()
    nb = n // 2 + 1
    rng = np.random.default_rng(n * 7 + SOURCES.index(source))
    for align in ALIGN_OFFSET:
        off, stride, hop, C, F = sweep_layout(n, source, align)
        row = n + (F - 1) * hop
        lead = 4 + off                                  # NaN samples before frame 0
        buf = np.full(lead + (C - 1) * stride + row + 5, np.nan, dtype=np.float32)
        for c in range(C):
            data = (rng.standard_normal(row) * 0.1).astype(np.float32)
            for f in range(F):
                s = lead + c * stride + f * hop
                buf[s:s + n] = data[f * hop:f * hop + n]
        rows = np.stack([buf[lead + c * stride:lead + c * stride + row] for c in range(C)])
        ref = fo.stft_power_batch(rows, n, hop)
        xd = torch.from_numpy(buf).cuda()
        osf, osc = nb + 3, F * (nb + 3) + 7
        written = np.zeros(C * osc + 11, dtype=bool)
        for c in range(C):
            for f in range(F):
                written[c * osc + f * osf:c * osc + f * osf + nb] = True
        got = {}
        for mode in MODES:
            out = torch.full((C * osc + 11,), SENTINEL, dtype=torch.int32, device="cuda")
            process(h, n, xd.data_ptr() + 4 * lead, stride, C, F, hop, out.view(torch.float32),
                    osc, osf, mode)
            bits = out.cpu().numpy()
            assert np.all(bits[~written] == SENTINEL), (align, mode, "a pad was written")
            vals = bits[written].view(np.float32).reshape(C, F, nb)
            assert np.all(np.isfinite(vals)), (align, mode, "NaN: a bin was not written or an "
                                               "uncovered sample was read")
            got[mode] = vals
        check_power(kernel_for(n, POWER, align), got[POWER], ref)
        check_log(kernel_for(n, LOGPOWER, align), got[LOGPOWER], got[POWER], ref, min_frac=min_frac(n),
                  strict=False)


# --------------------------------------------------------------------------- GPU: frame edges
def device_frames(x, off):
    """float32 rows x[C, L] placed at float offset `off` (mod 4 class) of a 16-byte aligned device
    buffer with a row stride that is a multiple of 4: returns (buffer, offset, stride)."""
    import torch
    C, L = x.shape
    stride = (L + 3) // 4 * 4 + 4
    buf = np.zeros(off + C * stride, dtype=np.float32)
    for c in range(C):
        buf[off + c * stride:off + c * stride + L] = x[c]
    return torch.from_numpy(buf).cuda(), off, stride


@pytest.mark.gpu
@pytest.mark.parametrize("n,mode,align", CASES)
def test_impulse_at_every_frame_index(n, mode, align):
    """An impulse swept through the frame: channel r (r < 4) holds it at sample N - 1 + r and the
    hop is 4, so frame f of channel r sees it at index N - 1 + r - 4 f, and between them the frames
    put it at every index 0 .. N-1 (the others are silent).  The reference is flat,
    (a w64[i])^2 / N^2 in every bin, and exactly 0 at i = 0 and N - 1 and for silent frames.  The
    per-frame extremes over the bins are checked: the bound is monotone in the error of a flat
    reference."""
    import torch
    h = handle()
    a, hop, C = 0.75, 4, 4
    F = n // hop + 1
    x = np.zeros((C, n + (F - 1) * hop), dtype=np.float32)
    for r in range(C):
        x[r, n - 1 + r] = a
    xd, off, stride = device_frames(x, ALIGN_OFFSET[align])
    out = run_dense(h, n, xd, off, stride, C, F, hop, mode)
    lo, hi = torch.aminmax(out.double(), dim=-1)
    ext = torch.stack([lo, hi], dim=-1).cpu().numpy()         # [C, F, 2]
    assert np.all(np.isfinite(ext))
    w64 = fo.hann_window(n)
    idx = n - 1 + np.arange(C)[:, None] - hop * np.arange(F)[None, :]
    inside = (idx >= 0) & (idx < n)
    assert inside.sum() == n
    ref = np.where(inside, (a * w64[np.clip(idx, 0, n - 1)]) ** 2 / n ** 2, 0.0)
    ref = np.repeat(ref[..., None], 2, axis=-1)
    kernel = kernel_for(n, mode, align)
    if mode == POWER:
        e = power_errors(ext, ref)
        note(kernel, "impulse", e["worst_ratio"])
        bad = idx[e["worst_index"][:2]]
        lit = power_errors(ext[inside], ref[inside])       # frames with a non-zero window weight
        assert e["worst_ratio"] <= 1.0, ("worst at frame index %d" % bad, e,
                                         "worst where w64 > 0: %.3g at index %d"
                                         % (lit["worst_ratio"], idx[inside][lit["worst_index"][0]]))
    else:
        e = assert_logpower_parity(ext, fo.log_spectrogram(ref))
        note(kernel, "impulse (log parity)", e["worst_ratio_all"])


@pytest.mark.gpu
@pytest.mark.parametrize("n,align", [(n, a) for n in SIZES for a in ALIGN_OFFSET])
def test_onsets_and_bin_centred_cosines(n, align):
    """Frames silent except their first or last k samples (k = 1, 2, 8, 64), and bin-centred
    cosines at the bins where the kernels' split step and radix-R combine change partners."""
    rng = np.random.default_rng(n + align)
    h = handle()
    t = np.arange(n)
    rows = []
    for k in (1, 2, 8, 64):
        k = min(k, n - 1)
        for first in (True, False):
            r = np.zeros(n, dtype=np.float32)
            sl = slice(0, k) if first else slice(n - k, n)
            r[sl] = rng.standard_normal(k).astype(np.float32) * 0.5
            rows.append(r)
    onsets = np.stack(rows)
    cosines = np.stack([np.cos(2 * np.pi * k * t / n) for k in cos_bins(n)]).astype(np.float32)
    xd, off, stride = device_frames(onsets, ALIGN_OFFSET[align])
    # log mode: the tonal setting of assert_logpower_parity; its power twin carries the precision
    run_both_modes(h, n, align, xd, off, stride, len(onsets), 1, n, ref_power(onsets)[:, None, :],
                   min_frac=0.0, strict=False, floor_db=40.0)
    # a bin-centred cosine puts bins 200+ dB below its peak, where float32 rounding noise (within
    # the power bound) is tens of dB above the reference and outside the dB criterion's noise
    # allowance even for numpy's float32 rfft: log mode is held to its power twin alone
    xd, off, stride = device_frames(cosines, ALIGN_OFFSET[align])
    run_both_modes(h, n, align, xd, off, stride, len(cosines), 1, n, ref_power(cosines)[:, None, :],
                   log_parity=False)


# --------------------------------------------------------------------------- GPU: exact properties
def noise_rows(C, L, seed, scale=0.1):
    return (np.random.default_rng(seed).standard_normal((C, L)) * scale).astype(np.float32)


@pytest.mark.gpu
@pytest.mark.parametrize("n,align", [(n, a) for n in SIZES for a in ALIGN_OFFSET])
def test_power_of_two_scaling_is_exact(n, align):
    """x 2^j -> P 4^j bit for bit, j = -20 .. 20: every step of the transform scales exactly."""
    h = handle()
    F, hop = 3, n // 4
    x0 = noise_rows(1, n + (F - 1) * hop, seed=n, scale=1.0)
    js = np.arange(-20, 21)
    x = (x0 * np.exp2(js)[:, None]).astype(np.float32)
    xd, off, stride = device_frames(x, ALIGN_OFFSET[align])
    got = run_dense(h, n, xd, off, stride, len(js), F, hop, POWER).cpu().numpy()
    base = got[20]
    assert np.all(base > 0)
    for i, j in enumerate(js):
        assert np.array_equal(got[i], base * np.float32(4.0 ** j)), j
    check_power(kernel_for(n, POWER, align), got[20:21], fo.stft_power_batch(x0, n, hop))


def rounds_channels(n, mode, align, F, sm):
    """A channel count C such that C x F items make the instance's per-warp, per-group or
    grid-stride loop run at least three rounds, and that no warp, group or CTA count divides."""
    k = kernel_for(n, mode, align)
    if k.startswith("stft_small_kernel"):
        G = 32 // (n // 64)
        units = [16 * sm * G, 16 * sm, 2 * sm, sm]          # 16 warps per SM, G frames per warp
    elif k.startswith("stft_large_kernel"):
        units = [sm * (16 // (n // 2048)), sm]              # 16/R frame groups per CTA, one CTA per SM
    elif k.startswith("stft_multi_kernel"):
        R = n // 2048
        units = [sm * (2 if R == 8 else 4 if R == 4 else 8)]
    else:                                                   # one CTA per frame
        units = [sm]
    C = -(-(3 * units[0] + 1) // F)
    while any(C * F % u == 0 for u in units):
        C += 1
    return C


@pytest.mark.gpu
@pytest.mark.parametrize("n,mode,align", CASES)
def test_expanded_rows_are_bit_identical(n, mode, align):
    """One row repeated with stride 0 (what torch's expand gives) over enough channels that every
    loop over items runs at least three rounds: every channel must equal channel 0 bit for bit."""
    import torch
    h = handle()
    F, hop = 5, n // 4
    C = rounds_channels(n, mode, align, F, h.sm_count)
    x = noise_rows(1, n + (F - 1) * hop, seed=n + 3)
    xd, off, _ = device_frames(x, ALIGN_OFFSET[align])
    out = run_dense(h, n, xd, off, 0, C, F, hop, mode)
    assert torch.equal(out, out[:1].expand_as(out))
    ref = fo.stft_power_batch(x, n, hop)
    row = out[0:1].cpu().numpy()
    if mode == POWER:
        check_power(kernel_for(n, mode, align), row, ref)
    else:
        assert_logpower_parity(row, fo.log_spectrogram(ref), min_frac=min_frac(n), strict=False)


@pytest.mark.gpu
@pytest.mark.parametrize("n,mode,align", CASES)
def test_channel_stride_equal_to_hop(n, mode, align):
    """x_stride = hop: channel c's frame f is channel 0's frame f + c, bit for bit."""
    h = handle()
    C, F = 4, 9
    hop = n // 4 + {16: 0, 8: 2, 4: 1}[align]
    x = noise_rows(1, n + (F + C - 2) * hop, seed=n + 5)
    xd, _, _ = device_frames(x, 0)
    out = run_dense(h, n, xd, 0, hop, C, F, hop, mode).cpu().numpy()
    for c in range(1, C):
        assert np.array_equal(out[c, :F - c], out[0, c:]), c


@pytest.mark.gpu
@pytest.mark.parametrize("n", SIZES)
def test_alignment_classes_same_arithmetic(n):
    """The three alignment classes load the same data differently; where they run one FFT (every
    size but 4096 and 8192) the outputs are the same bits.  At 4096 / 8192 the 16- and 8-byte
    classes run stft_large_kernel and must match each other; the 4-byte class runs
    stft_multi_kernel and is held to the bound."""
    h = handle()
    F, hop = 7, n // 4
    x = noise_rows(2, n + (F - 1) * hop, seed=n + 9)
    ref = fo.stft_power_batch(x, n, hop)
    for mode in MODES:
        got = {}
        for align, off in ALIGN_OFFSET.items():
            xd, o, stride = device_frames(x, off)
            got[align] = run_dense(h, n, xd, o, stride, 2, F, hop, mode).cpu().numpy()
        assert np.array_equal(got[16], got[8])
        if n in (4096, 8192):
            if mode == POWER:
                check_power(kernel_for(n, mode, 4), got[4], ref)
        else:
            assert np.array_equal(got[16], got[4])


# --------------------------------------------------------------------------- GPU: host path
def host_alignment(n, hop, frames):
    """The alignment class of the device staging buffer stft_host fills (cudaMalloc'd, rows of
    (nf - 1) hop + N samples for a chunk of nf frames, chunked as frt_stft_process_host does) and
    the number of frame chunks."""
    nb = n // 2 + 1
    budget = 32 << 20
    fchunk = min(frames, max(1, budget // (4 * nb)))
    aligns = []
    for f0 in range(0, frames, fchunk):
        nf = min(fchunk, frames - f0)
        ns = (nf - 1) * hop + n
        aligns.append(16 if ns % 4 == 0 and hop % 4 == 0 else 8 if ns % 2 == 0 and hop % 2 == 0 else 4)
    return min(aligns), len(aligns)


@pytest.mark.gpu
@pytest.mark.parametrize("n,hop,C,F,layout", [
    (16384, 2048, 1, 1100, "numpy"),          # two frame chunks (1023 + 77 frames of 32 MiB)
    (2048, 1024, 200, 100, "numpy"),          # channel groups of 81, 81 and 38
    (4096, 1001, 3, 50, "pinned strided"),    # odd hop, rows T + 16 floats apart, frame 0 at float 3
])
def test_host_path(n, hop, C, F, layout):
    """stft_host meets the bound; where it runs the same kernel as the device path on the same
    data, the outputs are the same bits.  Each case runs once."""
    import torch
    from friture_b200 import audioproc
    T = n + (F - 1) * hop
    x = noise_rows(C, T, seed=n + C)
    p = audioproc()
    p.set_fftsize(n)
    if layout == "pinned strided":
        big = torch.zeros((C, T + 16), dtype=torch.float32).pin_memory()
        big[:, 3:3 + T] = torch.from_numpy(x)
        xh = big[:, 3:3 + T]
        assert xh.is_pinned() and xh.stride(0) == T + 16
        got = p.stft_host(xh, hop=hop, log=False).numpy()
        dev = p.stft(big.cuda()[:, 3:3 + T], hop=hop, log=False).cpu().numpy()
        dev_align = 4
    else:
        got = p.stft_host(x, hop=hop, log=False)
        dev = p.stft(torch.from_numpy(x).cuda(), hop=hop, log=False).cpu().numpy()
        dev_align = 16 if T % 4 == 0 and hop % 4 == 0 else 8 if T % 2 == 0 and hop % 2 == 0 else 4
    assert got.shape == (C, F, n // 2 + 1)
    align, chunks = host_alignment(n, hop, F)
    if n == 16384:
        assert chunks == 2
    for c0 in range(0, C, 40):                  # the reference in slices of channels
        check_power(kernel_for(n, POWER, align), got[c0:c0 + 40],
                    fo.stft_power_batch(x[c0:c0 + 40], n, hop))
    if kernel_for(n, POWER, align) == kernel_for(n, POWER, dev_align):
        assert np.array_equal(got, dev)


# --------------------------------------------------------------------------- GPU: plans
@pytest.mark.gpu
def test_plans_shuffled_on_one_handle_and_windows():
    """All ten sizes planned on one handle in a shuffled order give the same bits as a fresh
    handle per size, and frt_stft_window is float32 of the float64 symmetric Hann."""
    import torch
    from friture_b200._lib import Handle
    x = noise_rows(2, 16384 + 3 * 4096, seed=17)
    xd, off, stride = device_frames(x, 0)

    def run_and_window(hd, n):
        outs = [run_dense(hd, n, xd, off, stride, 2, 3, n // 4, mode).cpu().numpy() for mode in MODES]
        win = np.empty(n, dtype=np.float32)
        hd.call("frt_stft_window", c_void_p(win.ctypes.data))
        assert np.array_equal(win, fo.hann_window(n).astype(np.float32)), n
        return outs

    fresh = {}
    for n in SIZES:
        hd = Handle(torch.cuda.current_device())
        try:
            fresh[n] = run_and_window(hd, n)
        finally:
            hd.close()
    shared = Handle(torch.cuda.current_device())
    try:
        # each size twice: the second time from the handle's plan cache
        for n in list(np.random.default_rng(2).permutation(SIZES)) * 2:
            for a, b in zip(run_and_window(shared, int(n)), fresh[int(n)]):
                assert np.array_equal(a, b), n
    finally:
        shared.close()


# --------------------------------------------------------------------------- GPU: 64-bit offsets
@pytest.mark.gpu
@pytest.mark.parametrize("n,which", [(4096, "out_stride_c"), (2048, "x_stride")])
def test_offsets_above_2_to_31_floats(n, which):
    """Two channels whose second row (input or output) lies more than 2^31 floats past the first."""
    import torch
    free, _ = torch.cuda.mem_get_info()
    if free < 20e9:
        print("skipped: %.1f GB free on the device, the case needs 20 GB" % (free / 1e9))
        pytest.skip("needs 20 GB of free device memory, %.1f GB free" % (free / 1e9))
    h = handle()
    F, hop, nb = 4, n // 4, n // 2 + 1
    T = n + (F - 1) * hop
    big = (1 << 31) + 4096
    x = noise_rows(2, T, seed=n + 1)
    ref = fo.stft_power_batch(x, n, hop)
    if which == "out_stride_c":
        xd = torch.from_numpy(x).cuda()
        out = torch.empty(big + F * nb, dtype=torch.float32, device="cuda")
        process(h, n, xd.data_ptr(), T, 2, F, hop, out, big, nb, POWER)
        got = torch.stack([out[:F * nb], out[big:big + F * nb]]).view(2, F, nb).cpu().numpy()
    else:
        xd = torch.empty(big + T, dtype=torch.float32, device="cuda")
        xd[:T] = torch.from_numpy(x[0]).cuda()
        xd[big:] = torch.from_numpy(x[1]).cuda()
        out = torch.empty((2, F, nb), dtype=torch.float32, device="cuda")
        process(h, n, xd.data_ptr(), big, 2, F, hop, out, F * nb, nb, POWER)
        got = out.cpu().numpy()
    torch.cuda.synchronize()
    del xd, out
    torch.cuda.empty_cache()
    check_power(kernel_for(n, POWER, 16), got, ref)
