"""GCC-PHAT and the delay estimator at every frame length the delay widget can plan.

The widget's delay range goes from 0.1 s to 1000 s in 0.1 s steps (friture/delay_estimator.py:
222-226) and frames are L = int(2 * range * 12000) samples long (:114-115).  The kernel plans
L = 2^a 3^b 5^c up to its shared-memory limit as radix 16/4/2 passes, then 25, 15, 5 and 3; these
tests run every accepted widget length and one length of every pass class against the float64
oracle (oracle/friture_oracle.py).

Accuracy is judged against a bound that scales with the case: the same formula restated in float32
with scipy.fft, on the same float32 input, shows what float32 error this input allows, and the
kernel may be at most K times further from the float64 oracle than that.  A CPU test plants
plausible bugs in the float64 formula and checks that each one exceeds the bound."""
import numpy as np
import pytest
import scipy.fft

from oracle import friture_oracle as fo

K = 20                # kernel error may be K times the float32 restatement's error, plus 1e-7
ABS_FLOOR = 1e-7

# every accepted widget range below the shared-memory limit: 0.1 .. 1.0 s except 0.7 s (factor 7)
WIDGET_LENGTHS = [2400, 4800, 7200, 9600, 12000, 14400, 19200, 21600, 24000]
# one length per class of pass sequence the planner produces
CLASS_LENGTHS = [
    4, 6,            # shorter than one sweep of the 384-thread CTA
    18, 162,         # radix-2 first pass (mean removal and window fused into it), then radix 3
    30, 50, 90, 150,  # radix 2, then 15 or 25, then a radix-3 pass last
    4374, 13122,     # 2 * 3^7, 2 * 3^8: long radix-3 chains
    6250,            # 2 * 5^5: radix-25 passes, then radix 5
    27648,           # 16*16*4*3*3*3: the longest accepted frame (37 of 38 register slots)
]
ALL_LENGTHS = WIDGET_LENGTHS + CLASS_LENGTHS
PAIR_KINDS = ["shift 0", "shift 1", "shift L/2-1", "shift L/2", "shift L-1", "random shift",
              "inverted", "DC offset"]

# decimator error relative to the channel's peak; the worst channel measured 1.03e-6 (65 channels,
# two stages) on an H100 80GB HBM3 at a 400 W power limit
DEC_REL_TOL = 3e-6


# --------------------------------------------------------------------------- references
def as64(a):
    """The oracle's input: float32-rounded, widened to float64."""
    return np.asarray(a, dtype=np.float32).astype(np.float64)


def gcc_f64(d0, d1):
    return fo.generalized_cross_correlation(as64(d0), as64(d1))


def gcc_f32(d0, d1):
    """generalized_cross_correlation (friture/signal/correlation.py:24-43) in single precision."""
    d0 = np.asarray(d0, dtype=np.float32)
    d1 = np.asarray(d1, dtype=np.float32)
    L = d0.shape[0]
    w = np.hanning(L).astype(np.float32)
    D0 = scipy.fft.rfft((d0 - d0.mean(dtype=np.float32)) * w)
    D1 = scipy.fft.rfft((d1 - d1.mean(dtype=np.float32)) * w)
    G = D0.conjugate() * D1
    absG = np.abs(G)
    W = np.float32(1.0) / (np.float32(1e-10) * absG.max() + absG)
    x = scipy.fft.irfft(W * G, n=L)
    assert x.dtype == np.float32
    return x


def smooth_f64(x, old):
    """delay_estimator.py:134-139 (old None: no previous frame)."""
    return x if old is None else 0.3 * x + 0.7 * old


def smooth_f32(x, old):
    return x if old is None else np.float32(0.3) * x + np.float32(0.7) * old


def gcc_f64_variant(d0, d1, periodic_hann=False, remove_mean=True, conj_split=True):
    """The kernel's route in float64: one complex FFT of a + jb, split into the two spectra through
    the Hermitian symmetry.  The keyword arguments plant bugs."""
    d0 = as64(d0)
    d1 = as64(d1)
    L = d0.shape[0]
    if remove_mean:
        d0 = d0 - d0.mean()
        d1 = d1 - d1.mean()
    n = np.arange(L)
    w = 0.5 - 0.5 * np.cos(2 * np.pi * n / (L if periodic_hann else L - 1))
    Z = np.fft.fft(d0 * w + 1j * (d1 * w))
    k = np.arange(L // 2 + 1)
    Zm = Z[(-k) % L]
    if conj_split:
        Zm = Zm.conjugate()
    D0 = (Z[k] + Zm) / 2
    D1 = (Z[k] - Zm) / 2j
    G = D0.conjugate() * D1
    absG = np.abs(G)
    return np.fft.irfft(G / (1e-10 * absG.max() + absG), L)


# --------------------------------------------------------------------------- the error bound
def error_bound(ref, f32):
    """K * (float32 restatement's error) + 1e-7."""
    return K * float(np.max(np.abs(np.asarray(f32, np.float64) - ref))) + ABS_FLOOR


def bound_check(got, ref, f32):
    """(error, bound, ratio): max|got - ref|, the bound, and the error over the float32 error."""
    got = np.asarray(got, dtype=np.float64)
    err = float(np.max(np.abs(got - ref)))
    e32 = float(np.max(np.abs(np.asarray(f32, np.float64) - ref)))
    return err, K * e32 + ABS_FLOOR, err / max(e32, 1e-30)


def assert_within(got, ref, f32, label):
    err, bound, ratio = bound_check(got, ref, f32)
    print("%s: err %.3g  bound %.3g  ratio %.2f" % (label, err, bound, ratio))
    assert err <= bound, "%s: max|got-ref| %.3g > bound %.3g (ratio %.1f > K = %d)" % (
        label, err, bound, ratio, K)
    return ratio


# --------------------------------------------------------------------------- inputs
def length_cases(L, seed=0):
    """Eight pairs of frame length L: d1 is d0 circularly shifted (shifts 0, 1, L/2-1, L/2, L-1
    and three random ones), one pair with inverted polarity, one with a DC offset of 3.0 on noise of
    sigma 0.1; independent noise at a tenth of the signal's level on d1.  Returns float32 d0, d1
    [8, L] and the shifts."""
    rng = np.random.default_rng([L, seed])
    r = [int(v) for v in rng.integers(0, L, 3)]
    shifts = [0, 1, L // 2 - 1, L // 2, L - 1, r[0], r[1], r[2]]
    d0 = rng.standard_normal((8, L))
    d0[7] = 3.0 + 0.1 * rng.standard_normal(L)
    d1 = np.stack([np.roll(d0[p], shifts[p]) for p in range(8)])
    d1[6] *= -1.0
    noise = 0.1 * rng.standard_normal((8, L))
    noise[7] *= 0.1
    d1 = d1 + noise
    return d0.astype(np.float32), d1.astype(np.float32), shifts


def shift_recoverable(L, s):
    """Whether the planted shift must show as the peak.  A circular shift near L/2 moves the signal
    under the other half of the Hann window; short frames then have too few bins to lift that
    weak overlap above the noise, so below 1000 samples only lags within L/4 count (below 8
    none)."""
    return L >= 1000 or (L >= 8 and min(s, L - s) <= L // 4)


def peak_margin(x):
    """Gap between the largest and the second largest |x|: the arg-max is only well defined when
    this exceeds what the compared results may differ by."""
    a = np.sort(np.abs(x))
    return float(a[-1] - a[-2])


# --------------------------------------------------------------------------- CPU: bound has teeth
@pytest.mark.parametrize("L", ALL_LENGTHS)
def test_cases_are_well_posed(L):
    """The oracle finds every recoverable planted shift, and each arg-max stands clear of the
    runner-up by more than twice the bound, so an exact index comparison with the kernel is
    meaningful."""
    d0, d1, shifts = length_cases(L)
    for p in range(8):
        ref = gcc_f64(d0[p], d1[p])
        i, _, _ = fo.delay_peak(ref)
        if shift_recoverable(L, shifts[p]):
            assert i == shifts[p], (PAIR_KINDS[p], i, shifts[p])
        assert peak_margin(ref) > 2 * error_bound(ref, gcc_f32(d0[p], d1[p])), PAIR_KINDS[p]


@pytest.mark.parametrize("L", ALL_LENGTHS)
def test_bound_catches_planted_bugs(L):
    """Plausible kernel bugs, restated in float64, each exceed the bound on these inputs: a
    periodic Hann window (L instead of L-1), means not removed (pair with a DC offset), swapped
    smoothing weights (0.7 X + 0.3 old), and the Hermitian split with Z[L-k] un-conjugated.
    The window bug barely moves pairs whose lag is near 0 (their peak sits where the two windows
    agree); the pairs with lags near L/2 show it at every length."""
    d0, d1, _ = length_cases(L)
    e0, e1, _ = length_cases(L, seed=1)        # the next frame, for the smoothing
    excess = {"periodic Hann": [], "unconjugated split": [], "swapped smoothing": []}
    for p in range(8):
        ref = gcc_f64(d0[p], d1[p])
        f32 = gcc_f32(d0[p], d1[p])
        err, bound, _ = bound_check(gcc_f64_variant(d0[p], d1[p]), ref, f32)
        assert err < 1e-12 and err <= bound, "the un-planted split route must match the oracle"
        err, bound, _ = bound_check(gcc_f64_variant(d0[p], d1[p], periodic_hann=True), ref, f32)
        excess["periodic Hann"].append(err / bound)
        err, bound, _ = bound_check(gcc_f64_variant(d0[p], d1[p], conj_split=False), ref, f32)
        excess["unconjugated split"].append(err / bound)
        if PAIR_KINDS[p] == "DC offset":
            err, bound, _ = bound_check(gcc_f64_variant(d0[p], d1[p], remove_mean=False), ref, f32)
            assert err > bound, ("means kept", err, bound)
        nxt, nxt32 = gcc_f64(e0[p], e1[p]), gcc_f32(e0[p], e1[p])
        sm = smooth_f64(nxt, ref)
        sm32 = smooth_f32(nxt32, f32)
        err, bound, _ = bound_check(0.7 * nxt + 0.3 * ref, sm, sm32)
        excess["swapped smoothing"].append(err / bound)
    assert max(excess["periodic Hann"]) > 10, excess["periodic Hann"]
    assert min(excess["unconjugated split"]) > 1, excess["unconjugated split"]
    assert min(excess["swapped smoothing"]) > 1, excess["swapped smoothing"]


# --------------------------------------------------------------------------- GPU: every length
def cuda(a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float32)).cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("L", ALL_LENGTHS)
def test_length_vs_oracle(L):
    from friture_b200.correlation import GccPhat
    d0, d1, shifts = length_cases(L)
    idx, val, xc = GccPhat(L).estimate(cuda(d0), cuda(d1), smooth=False, want_xcorr=True)
    idx, val, xc = idx.cpu().numpy(), val.cpu().numpy(), xc.cpu().numpy()
    worst = 0.0
    for p in range(8):
        ref = gcc_f64(d0[p], d1[p])
        f32 = gcc_f32(d0[p], d1[p])
        worst = max(worst, assert_within(xc[p], ref, f32, "L=%d %s" % (L, PAIR_KINDS[p])))
        i, v, _ = fo.delay_peak(ref)
        assert int(idx[p]) == i, (PAIR_KINDS[p], int(idx[p]), i)
        if shift_recoverable(L, shifts[p]):
            assert i == shifts[p]
        assert abs(float(val[p]) - v) <= error_bound(ref, f32), PAIR_KINDS[p]
    if shift_recoverable(L, shifts[6]):
        assert float(val[6]) < 0      # inverted polarity shows in the sign of the extremum
    print("L=%d worst ratio %.2f" % (L, worst))


# --------------------------------------------------------------------------- GPU: CTA pair loop
@pytest.mark.gpu
@pytest.mark.parametrize("L", [7200, 2400])
def test_pairs_beyond_sm_count_smoothing_and_silence(L):
    """2*S+5 pairs, so every CTA runs two or three pairs and reuses its shared memory; rows L+3
    floats apart (4-byte aligned only).  Four calls with silent pairs at 0, S, S+1 and P-1, checked
    after each call against a per-pair restatement of delay_estimator.py:129-142: raw Xcorr,
    smoothed buffer, index and value, and the kernel's "no previous frame" marker (NaN in slot
    0)."""
    import torch
    from friture_b200 import _lib
    S = torch.cuda.get_device_properties(0).multi_processor_count
    P = 2 * S + 5
    stride = L + 3
    FILL = 7.0                       # initial smoothed buffer: untouched slots must keep it
    # silent pairs per call: "zero" = both channels 0, "const" = both 0.25,
    # "const0" / "const1" = only that channel at 0.25
    calls = [
        (0, {0: "zero", S: "const", S + 1: "const0", P - 1: "const1"}),
        # S and P-1 get their first real frame
        (2, {0: "const", S + 1: "zero"}),
        # 0 and S+1 get their first real frame; 1, S+2 and P-2 go silent after real frames
        (2, {1: "zero", S + 2: "const", P - 2: "const1"}),
        # every pair has had a real frame, so every non-silent pair blends
        (1, {2: "const0", S: "zero"}),
    ]
    rng = np.random.default_rng(L + 1)
    h = _lib.Handle(0)
    h.call("frt_gcc_plan", L)
    d0s = torch.full((P, stride), float("nan"), device="cuda")   # the padding must never be read
    d1s = torch.full((P, stride), float("nan"), device="cuda")
    xc = torch.empty((P, L), device="cuda")
    sm = torch.full((P, L), FILL, device="cuda")
    idx = torch.empty(P, dtype=torch.int32, device="cuda")
    val = torch.empty(P, dtype=torch.float32, device="cuda")
    old64 = [None] * P
    old32 = [None] * P
    for c, (have_prev, silent) in enumerate(calls):
        shifts = rng.integers(0, L, P)
        a = rng.standard_normal((P, L))
        b = np.stack([np.roll(a[p], shifts[p]) for p in range(P)])
        b += 0.1 * rng.standard_normal((P, L))
        for p, kind in silent.items():
            if kind in ("zero", "const"):
                a[p] = b[p] = 0.0 if kind == "zero" else 0.25
            elif kind == "const0":
                a[p] = 0.25
            else:
                b[p] = 0.25
        a = a.astype(np.float32)
        b = b.astype(np.float32)
        d0s[:, :L] = cuda(a)
        d1s[:, :L] = cuda(b)
        sm_before = sm.clone()
        h.call("frt_gcc_phat", _lib._ptr(d0s), _lib._ptr(d1s), stride, P, _lib._ptr(xc),
               _lib._ptr(sm), have_prev, _lib._ptr(idx), _lib._ptr(val), _lib.current_stream_ptr())
        torch.cuda.synchronize()
        g_xc, g_sm = xc.cpu().numpy(), sm.cpu().numpy()
        g_idx, g_val = idx.cpu().numpy(), val.cpu().numpy()
        for p in range(P):
            label = "L=%d call %d pair %d" % (L, c + 1, p)
            if p in silent:
                assert g_idx[p] == 0 and g_val[p] == 0.0, label
                assert not np.any(g_xc[p]), label
                if old64[p] is None:
                    assert np.isnan(g_sm[p, 0]), label
                    assert np.all(g_sm[p, 1:] == FILL), label
                else:
                    assert torch.equal(sm[p], sm_before[p]), label     # state left alone
                continue
            x64 = gcc_f64(a[p], b[p])
            x32 = gcc_f32(a[p], b[p])
            s64 = smooth_f64(x64, old64[p])
            s32 = smooth_f32(x32, old32[p])
            old64[p], old32[p] = s64, s32
            assert_within(g_xc[p], x64, x32, label + " xcorr")
            assert_within(g_sm[p], s64, s32, label + " smoothed")
            i, v, _ = fo.delay_peak(s64)
            assert g_idx[p] == i, label
            assert abs(float(g_val[p]) - v) <= error_bound(s64, s32), label
    assert all(o is not None for o in old64)


# --------------------------------------------------------------------------- GPU: end to end
class DelayPipelineModel:
    """CPU restatement of Delay_Estimator_Widget.handle_new_data (friture/delay_estimator.py:87-176)
    for several pairs: float64 decimation with carried states, 50 %-overlap frames ending at the
    advanced old_index, float64 GCC-PHAT and smoothing, and the published delay, extremum and
    confidence.  Alongside, the float32 restatement of the same frames for the error bound."""

    def __init__(self, n_pairs, delayrange_s):
        from friture_b200 import filter_data
        self.bdec, self.adec, _ = filter_data.decimator()
        self.fs = 12000.0
        self.time = 2 * delayrange_s
        self.L = int(self.time * self.fs)
        self.hop = int(0.5 * self.L)
        self.P = n_pairs
        self.z0 = [[np.zeros(12), np.zeros(12)] for _ in range(n_pairs)]
        self.z1 = [[np.zeros(12), np.zeros(12)] for _ in range(n_pairs)]
        self.hist0 = np.zeros((n_pairs, self.L))      # the ring buffer starts as zeros
        self.hist1 = np.zeros((n_pairs, self.L))
        self.offset = 0
        self.old_index = 0
        self.old64 = [None] * n_pairs
        self.old32 = [None] * n_pairs

    def push(self, x0, x1):
        """Chunks [P, n] at 48 kHz; returns the number of frames and, per pair, the last frame's
        (delay_ms, extremum, bound on the extremum, confidence before int())."""
        d0, d1 = [], []
        for p in range(self.P):
            y0, self.z0[p] = fo.decimate_multiple(2, self.bdec, self.adec, x0[p], self.z0[p])
            y1, self.z1[p] = fo.decimate_multiple(2, self.bdec, self.adec, x1[p], self.z1[p])
            d0.append(y0)
            d1.append(y1)
        self.hist0 = np.concatenate([self.hist0, np.stack(d0)], axis=1)
        self.hist1 = np.concatenate([self.hist1, np.stack(d1)], axis=1)
        self.offset += len(d0[0])
        n = int((self.offset - self.old_index) / self.hop)
        out = None
        for _ in range(n):
            self.old_index += self.hop
            f0 = self.hist0[:, self.old_index:self.old_index + self.L]
            f1 = self.hist1[:, self.old_index:self.old_index + self.L]
            out = [self._frame(p, f0[p], f1[p]) for p in range(self.P)]
        return n, out

    def _frame(self, p, f0, f1):
        s64 = smooth_f64(gcc_f64(f0, f1), self.old64[p])
        s32 = smooth_f32(gcc_f32(f0, f1), self.old32[p])
        self.old64[p], self.old32[p] = s64, s32
        i = int(np.argmax(np.abs(s64)))
        v = float(s64[i])
        norm = abs(v) / (3 * np.std(s64))
        delay = 1e3 * float(i) / self.fs
        if delay > 1e3 * self.time / 2.:
            delay -= 1e3 * self.time
        x = (norm > 1.) * (norm - 1.)
        x = (0.12 * x) ** 3
        return delay, v, error_bound(s64, s32), (x / (1. + x)) * 100


@pytest.mark.gpu
@pytest.mark.parametrize("delayrange_s, L", [(0.1, 2400), (0.3, 7200), (0.9, 21600)])
def test_delay_estimator_at_new_ranges(delayrange_s, L):
    """Three pairs: x1 lagging x0, x1 leading x0 (the wrap of delay_estimator.py:150-151), and a
    lag near the edge of the range; 512-sample chunks, then 1024-sample chunks."""
    import torch
    from friture_b200.delay import DelayEstimator
    fs = 48000
    # in whole 12 kHz samples, so that each peak falls on one index
    lags = [4 * round(f * delayrange_s * fs / 4) for f in (0.37, -0.23, 0.85)]
    model = DelayPipelineModel(3, delayrange_s)
    est = DelayEstimator(3, delayrange_s=delayrange_s)
    assert est.length == model.L == L
    hop48 = 4 * model.hop
    n512 = -(-5 * hop48 // 512)
    n1024 = -(-5 * hop48 // 1024)
    n = 512 * n512 + 1024 * n1024
    rng = np.random.default_rng(L)
    M = max(abs(d) for d in lags)
    base = 0.1 * rng.standard_normal(n + 2 * M)
    x0 = np.tile(base[M:M + n], (3, 1))
    x1 = np.stack([base[M - d:M - d + n] for d in lags]) + 0.01 * rng.standard_normal((3, n))
    x0, x1 = x0.astype(np.float32), x1.astype(np.float32)
    cuts = [512] * n512 + [1024] * n1024
    pos, frames, worst = 0, 0, 0.0
    for m in cuts:
        a, b = x0[:, pos:pos + m], x1[:, pos:pos + m]
        pos += m
        r = est.handle_new_data(cuda(a), cuda(b))
        r_ref, out = model.push(a.astype(np.float64), b.astype(np.float64))
        assert r == r_ref
        if r == 0:
            continue
        frames += r
        for p, (delay, v, bound, conf) in enumerate(out):
            label = "range %.1f frame %d pair %d" % (delayrange_s, frames, p)
            assert est.delay_ms[p] == delay, label
            dv = abs(float(est.Xcorr_extremum[p]) - v)
            assert dv <= bound, label
            worst = max(worst, dv * K / max(bound - ABS_FLOOR, 1e-30))
            if abs(conf - round(conf)) < 1e-6:
                assert abs(int(est.correlation[p]) - int(conf)) <= 1, label
            else:
                assert int(est.correlation[p]) == int(conf), label
    print("range %.1f: %d frames, worst extremum ratio %.2f" % (delayrange_s, frames, worst))
    assert frames >= 9
    truth = [1e3 * d / fs for d in lags]
    assert np.allclose(est.delay_ms, truth, atol=1e3 / 12000.0 + 1e-9)
    assert torch.isfinite(est.gcc._smoothed).all()


# --------------------------------------------------------------------------- GPU: decimator
@pytest.mark.gpu
@pytest.mark.parametrize("n_stages", [1, 2])
@pytest.mark.parametrize("C", [1, 3, 65])
def test_decimator_channels_and_chunks(C, n_stages):
    """decimate_multiple with carried state (friture/signal/decimate.py:45-71) for C channels (65:
    an odd number of the kernel's two-warp CTAs), one stream cut into 256, 768, 4096, 0 and 512
    samples.  Each channel is compared relative to its own peak: channels differ in level by four
    orders of magnitude, so a channel mix-up or a shared state shows."""
    import torch
    from friture_b200 import filter_data
    from friture_b200.delay import Decimator
    bdec, adec, _ = filter_data.decimator()
    rng = np.random.default_rng(C * 10 + n_stages)
    cuts = [256, 768, 4096, 0, 512]
    T = sum(cuts)
    t = np.arange(T) / 48000.0
    level = 10.0 ** (np.arange(C) % 5 - 2)
    freq = 100.0 + 9000.0 * rng.random(C)
    x = 0.1 * rng.standard_normal((C, T)) + np.sin(2 * np.pi * freq[:, None] * t)
    x = (level[:, None] * x).astype(np.float32)
    dec = Decimator(C, n_stages)
    outs, pos = [], 0
    for m in cuts:
        o = dec.process(cuda(x[:, pos:pos + m]) if m else torch.empty((C, 0), device="cuda"))
        assert tuple(o.shape) == (C, m >> n_stages)
        outs.append(o)
        pos += m
    got = torch.cat(outs, dim=1).cpu().numpy().astype(np.float64)
    rel = []
    for c in range(C):
        want, _ = fo.decimate_multiple(n_stages, bdec, adec, as64(x[c]), [np.zeros(12)] * n_stages)
        rel.append(float(np.max(np.abs(got[c] - want)) / np.max(np.abs(want))))
    print("decimator C=%d n_stages=%d worst channel rel err %.3g" % (C, n_stages, max(rel)))
    assert max(rel) < DEC_REL_TOL, rel


# --------------------------------------------------------------------------- GPU: routes, rejected lengths
SMEM_LAUNCHES = 1          # gcc_phat_kernel
BLUESTEIN_LAUNCHES = 10    # the gl_* kernels of one workspace group


def assert_route(est, launches):
    """est's length runs on the route frt_gcc_plan picks for it: frt_gcc_fits says so, and one call
    on one pair launches `launches` kernels."""
    import torch
    from friture_b200 import _lib
    assert _lib.load_library().frt_gcc_fits(est.length) == (launches == SMEM_LAUNCHES)
    x = torch.randn((1, est.length), device="cuda")
    n = est.handle.launch_count
    est.estimate(x, x, smooth=False)
    assert est.handle.launch_count - n == launches


@pytest.mark.gpu
def test_rejected_lengths_leave_both_routes_usable():
    """0.7 s and 1.1 s (factors 7 and 11), 28160 (fits the shared memory, factor 11), an odd length
    (Xcorr has L-1 samples) and 7168 (factor 7) run on the Bluestein route within the bound.  2, 3
    and 24 000 001 raise ValueError; after each, a shared-memory and a Bluestein estimator on the
    same handle give the same bits as their first call, each on its own route."""
    import torch
    import gcc_long_model as gm
    from friture_b200._lib import FrtValueError, Handle
    from friture_b200.correlation import GccPhat
    h = Handle(0)
    for L in (16800, 26400, 28160, 2401, 7168):
        d0, d1, _ = length_cases(L)
        est = GccPhat(L, handle=h)
        idx, val, xc = est.estimate(cuda(d0), cuda(d1), smooth=False, want_xcorr=True)
        assert xc.shape == (8, L - (L & 1))
        idx, val, xc = idx.cpu().numpy(), val.cpu().numpy(), xc.cpu().numpy()
        for p in range(8):
            ref, f32 = gcc_f64(d0[p], d1[p]), gm.gcc_f32_any(d0[p], d1[p])
            assert_within(xc[p], ref, f32, "L=%d %s" % (L, PAIR_KINDS[p]))
            i, v, _ = fo.delay_peak(ref)
            assert int(idx[p]) == i, (L, PAIR_KINDS[p], int(idx[p]), i)
            assert abs(float(val[p]) - v) <= error_bound(ref, f32), (L, PAIR_KINDS[p])
        assert_route(est, BLUESTEIN_LAUNCHES)
    good = []
    for L, launches in ((2400, SMEM_LAUNCHES), (55199, BLUESTEIN_LAUNCHES)):
        d0, d1, _ = length_cases(L)
        est, a, b = GccPhat(L, handle=h), cuda(d0), cuda(d1)
        good.append((est, a, b, launches, est.estimate(a, b, smooth=False, want_xcorr=True)))
    for bad in (3, 2, 24000001):
        z = torch.zeros((1, bad), device="cuda")
        with pytest.raises(FrtValueError):
            GccPhat(bad, handle=h).estimate(z, z + 1.0)
        for est, a, b, launches, first in good:
            n = h.launch_count
            again = est.estimate(a, b, smooth=False, want_xcorr=True)
            assert h.launch_count - n == launches, (bad, est.length)
            assert all(torch.equal(x, y) for x, y in zip(again, first)), (bad, est.length)
