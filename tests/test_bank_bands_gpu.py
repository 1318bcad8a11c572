"""Every filterbank kernel instance, band by band, on the inputs where a multirate float32 IIR bank
goes wrong (tests/bank_signals.py: tones at band centres, on a band edge and around a decimator's
cut-off, a log sweep, a DC offset, a Nyquist-rate sequence, impulses at block ends and at odd / even
decimated samples, silence, a burst decaying into silence, clipped full-scale noise, noise at 1e-6 and
1e-12, white noise), one signal per channel row.

Every (plan, signal, check) is its own test: the per-band bound of tests/parity.py on the energies,
the north-star vector criterion (TOL) on the energies, the same two on the dB energies with
A-weighting, and the per-sample bound on the ragged band outputs.  The kernel runs once per plan.

Where the float32 model (tests/bank_f32_model.py) itself fails a check, float32 arithmetic cannot meet
it: MODEL_LIMITED lists exactly those (plan, signal, check) with the model's number, and they are
expected failures that may pass.  Where a kernel fails a check the model passes, the kernel is worse
than float32 has to be: KNOWN_EXCESS lists those with the kernel's number, as strict expected
failures.  Every other (plan, signal, check) is asserted.  The CPU tests check the calibration, that
MODEL_LIMITED is exactly the model's failures, and that the bound rejects realistic mistakes the
vector criterion lets through."""
import functools
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import bank_signals as bs  # noqa: E402
from bank_f32_model import BankF32Model  # noqa: E402
from parity import BAND_REL_TOL, TOL, band_db_errors, band_errors, y_errors  # noqa: E402
from test_bank_dispatch_gpu import CASES, INSTANCES  # noqa: E402

ZERO_LIMITED = ("dc_offset", "nyquist")   # reach the bands only through the zeros at z = +-1
NAMES = bs.signal_names()
CHECKS = ("energy-band", "energy-vector", "dB-band", "dB-vector", "y")

# GPU plans: (bpo, octaves, channels, block, want_y, response time, label).  The dispatch cases launch
# every compiled instance; then the narrowest (highest-Q) bands, the 10-octave bank, and the response
# times at which the burst decays through the float32 subnormal range (0.025 s) or barely at all (5 s).
PLANS = ([(b, n, c, k, y, 1.0, name) for b, n, c, k, y, name in CASES]
         + [(12, 9, 2, 512, False, 1.0, "bpo12"), (24, 9, 2, 256, True, 1.0, "bpo24-y"),
            (24, 9, 1536, 1024, False, 1.0, "bpo24"), (3, 10, 3072, 1024, False, 1.0, "oct10"),
            (1, 10, 2, 512, True, 1.0, "bpo1-oct10-y")]
         + [(3, 9, c, k, y, T, "T%g-C%d-b%d" % (T, c, k)) for T in (0.025, 5.0)
            for c, k, y in ((3072, 512, False), (3073, 256, False), (2, 256, True), (1536, 768, False))])
# CPU calibration plans: (bpo, octaves, block, response time)
MODEL_PLANS = [(3, 9, 512, 1.0), (3, 9, 256, 0.025), (3, 9, 1024, 5.0), (1, 9, 512, 1.0),
               (6, 9, 768, 1.0), (12, 9, 512, 1.0), (24, 9, 512, 1.0), (3, 10, 1024, 1.0),
               (3, 3, 512, 1.0)]

# (bpo, octaves, block, response time, signal, check) -> the float32 model's own number, where it fails
# the check.  Four kinds: the DC offset and the Nyquist sequence (the section zeros at z = +-1); the
# dB vector of tones at 0.025 s (stopband bands near 1e-20 of the tone, where a float32 error of
# 1e-11 of the tone is tens of dB); the start-up transient of a low tone, a sweep and a DC offset in
# the lowest 1/12 and 1/24-octave bands; the decay of impulses and of the burst at 0.025 s.
MODEL_LIMITED = {
    (1, 9, 256, 1.0, 'nyquist', 'energy-vector'): 0.000148,
    (1, 9, 512, 1.0, 'nyquist', 'energy-vector'): 0.000148,
    (1, 10, 512, 1.0, 'nyquist', 'energy-vector'): 0.000148,
    (3, 3, 512, 1.0, 'nyquist', 'energy-vector'): 0.000127,
    (3, 9, 256, 0.025, 'tone_top', 'dB-vector'): 0.016,
    (3, 9, 256, 0.025, 'tone_mid', 'dB-vector'): 0.125,
    (3, 9, 256, 0.025, 'tone_edge', 'dB-vector'): 0.0899,
    (3, 9, 256, 0.025, 'tone_dec_transition', 'dB-vector'): 0.00111,
    (3, 9, 256, 0.025, 'tone_dec_alias', 'dB-vector'): 0.0696,
    (3, 9, 256, 0.025, 'dc_offset', 'energy-vector'): 0.000187,
    (3, 9, 256, 0.025, 'nyquist', 'energy-band'): 2.37,
    (3, 9, 256, 0.025, 'nyquist', 'energy-vector'): 0.000475,
    (3, 9, 256, 0.025, 'nyquist', 'dB-band'): 2.29,
    (3, 9, 256, 0.025, 'impulse_odd', 'energy-vector'): 1e-05,
    (3, 9, 256, 0.025, 'burst_then_silence', 'energy-vector'): 2.3e-05,
    (3, 9, 256, 1.0, 'nyquist', 'energy-vector'): 0.000127,
    (3, 9, 256, 5.0, 'nyquist', 'energy-vector'): 6.47e-05,
    (3, 9, 512, 0.025, 'tone_top', 'dB-vector'): 0.0251,
    (3, 9, 512, 0.025, 'tone_mid', 'dB-vector'): 0.191,
    (3, 9, 512, 0.025, 'tone_edge', 'dB-vector'): 0.147,
    (3, 9, 512, 0.025, 'tone_dec_transition', 'dB-vector'): 0.00187,
    (3, 9, 512, 0.025, 'tone_dec_alias', 'dB-vector'): 0.114,
    (3, 9, 512, 0.025, 'dc_offset', 'energy-vector'): 0.000187,
    (3, 9, 512, 0.025, 'nyquist', 'energy-band'): 2.37,
    (3, 9, 512, 0.025, 'nyquist', 'energy-vector'): 0.000475,
    (3, 9, 512, 0.025, 'nyquist', 'dB-band'): 2.29,
    (3, 9, 512, 0.025, 'nyquist', 'dB-vector'): 1.19e-05,
    (3, 9, 512, 0.025, 'impulse_odd', 'energy-vector'): 1e-05,
    (3, 9, 512, 0.025, 'burst_then_silence', 'energy-vector'): 2.3e-05,
    (3, 9, 512, 1.0, 'nyquist', 'energy-vector'): 0.000127,
    (3, 9, 512, 5.0, 'nyquist', 'energy-vector'): 6.47e-05,
    (3, 9, 768, 0.025, 'tone_top', 'dB-vector'): 0.0249,
    (3, 9, 768, 0.025, 'tone_mid', 'dB-vector'): 0.191,
    (3, 9, 768, 0.025, 'tone_edge', 'dB-vector'): 0.148,
    (3, 9, 768, 0.025, 'tone_dec_transition', 'dB-vector'): 0.00188,
    (3, 9, 768, 0.025, 'tone_dec_alias', 'dB-vector'): 0.114,
    (3, 9, 768, 0.025, 'dc_offset', 'energy-vector'): 0.000183,
    (3, 9, 768, 0.025, 'nyquist', 'energy-band'): 2.37,
    (3, 9, 768, 0.025, 'nyquist', 'energy-vector'): 0.000475,
    (3, 9, 768, 0.025, 'nyquist', 'dB-band'): 2.29,
    (3, 9, 768, 0.025, 'nyquist', 'dB-vector'): 1.32e-05,
    (3, 9, 768, 0.025, 'burst_then_silence', 'energy-vector'): 2.28e-05,
    (3, 9, 768, 1.0, 'nyquist', 'energy-vector'): 0.000127,
    (3, 9, 768, 5.0, 'nyquist', 'energy-vector'): 6.47e-05,
    (3, 9, 1024, 1.0, 'nyquist', 'energy-vector'): 0.000127,
    (3, 9, 1536, 1.0, 'nyquist', 'energy-vector'): 0.000127,
    (3, 10, 1024, 1.0, 'nyquist', 'energy-vector'): 0.000127,
    (6, 9, 512, 1.0, 'nyquist', 'energy-vector'): 2.62e-05,
    (6, 9, 1024, 1.0, 'nyquist', 'energy-vector'): 2.62e-05,
    (12, 9, 512, 1.0, 'tone_bottom', 'energy-vector'): 2.04e-05,
    (12, 9, 512, 1.0, 'log_sweep', 'energy-vector'): 1.54e-05,
    (12, 9, 512, 1.0, 'dc_offset', 'energy-vector'): 1.31e-05,
    (12, 9, 512, 1.0, 'nyquist', 'energy-vector'): 8.71e-05,
    (24, 9, 256, 1.0, 'tone_bottom', 'energy-vector'): 2.53e-05,
    (24, 9, 256, 1.0, 'dc_offset', 'energy-vector'): 2.21e-05,
    (24, 9, 256, 1.0, 'nyquist', 'energy-vector'): 5.52e-05,
    (24, 9, 1024, 1.0, 'tone_bottom', 'energy-vector'): 2.38e-05,
    (24, 9, 1024, 1.0, 'dc_offset', 'energy-vector'): 2.13e-05,
    (24, 9, 1024, 1.0, 'nyquist', 'energy-vector'): 5.52e-05,
}
# (plan label, signal, check) -> the kernel's number on an H100, where a kernel fails a check the
# float32 model passes (the model's number alongside).  The pipelined kernel on the Nyquist sequence:
# its bands see the sequence only through the zeros at z = -1, where the numerator cancels to 1e-4 of
# its terms, and its operation order loses ~3x more there than the sequential model.  Impulses, the
# 1/24-octave sweep and the 0.025 s sweep: 1.0 to 1.7x the model, within a few float32 roundings of
# the limit.  Strict: a fix makes these pass and must remove the entry.
KNOWN_EXCESS = {
    ('bank_pipe_kernel<6, 1, 1>', 'nyquist', 'energy-band'): 2.27,   # model 0.738
    ('bank_pipe_kernel<6, 1, 1>', 'nyquist', 'dB-band'): 2.2,   # model 0.715
    ('bank_pipe_kernel<6, 1, 1>', 'nyquist', 'dB-vector'): 1.19e-05,   # model 3.87e-06
    ('bank_pipe_kernel<6, 1, 3>', 'nyquist', 'energy-band'): 1.01,   # model 0.637
    ('bank_pipe_kernel<5, 1, 1>', 'nyquist', 'energy-band'): 2.26,   # model 0.738
    ('bank_pipe_kernel<5, 1, 1>', 'nyquist', 'dB-band'): 2.19,   # model 0.715
    ('bank_pipe_kernel<5, 2, 1>', 'nyquist', 'energy-band'): 2.26,   # model 0.738
    ('bank_pipe_kernel<5, 2, 1>', 'nyquist', 'dB-band'): 2.19,   # model 0.715
    ('bank_pipe_kernel<5, 2, 1>', 'nyquist', 'dB-vector'): 1.18e-05,   # model 3.87e-06
    ('bpo24-y', 'log_sweep', 'energy-vector'): 1.12e-05,   # model 9.82e-06
    ('bpo1-oct10-y', 'nyquist', 'energy-band'): 1.63,   # model 0.738
    ('bpo1-oct10-y', 'nyquist', 'dB-band'): 1.58,   # model 0.715
    ('T0.025-C3072-b512', 'impulse_even', 'energy-vector'): 1.31e-05,   # model 7.68e-06
    ('T0.025-C3073-b256', 'impulse_even', 'energy-vector'): 1.31e-05,   # model 7.49e-06
    ('T0.025-C2-b256', 'log_sweep', 'energy-band'): 1.02,   # model 0.212
    ('T0.025-C2-b256', 'impulse_block_last', 'energy-vector'): 1.03e-05,   # model 9.62e-06
    ('T0.025-C2-b256', 'impulse_even', 'energy-vector'): 1.1e-05,   # model 7.49e-06
    ('T0.025-C1536-b768', 'impulse_block_last', 'energy-vector'): 1.01e-05,   # model 9.48e-06
    ('T0.025-C1536-b768', 'impulse_even', 'energy-vector'): 1.07e-05,   # model 6.95e-06
}


def model_plan(p):
    return (p[0], p[1], p[3], p[5])


def plan_id(p):
    return "%s-bpo%d-oct%d-C%d-b%d%s-T%g" % (p[6], p[0], p[1], p[2], p[3], "-y" if p[4] else "", p[5])


@functools.lru_cache(maxsize=None)
def model_run(bpo, n_oct, block, response_time):
    """float32 model energies [S, blocks, bands] and y of the signal set (float64 copies)."""
    from friture_b200.octavefilters import smoothing_alphas
    bank, x, _, _ = bs.signal_set(bpo, n_oct, block, response_time)
    E, Y = BankF32Model(bank, n_oct, smoothing_alphas(response_time, n_oct)).run(x, block, want_y=True)
    return E.astype(np.float64), [v.astype(np.float64) for v in Y]


def a_weights(bpo, n_oct):
    from friture_b200.octavefilters import Octave_Filters
    return np.asarray(Octave_Filters(bpo, n_octaves=n_oct).A, dtype=np.float32).astype(np.float64)


def measure(check, s, E, Y, got, ys, db, A, scale=1.0):
    """(value, passes) of one check on signal row s: a fraction of the bound or a vector error."""
    if check in ("energy-band", "energy-vector"):
        e = band_errors(got[s], E[s], scale)
    elif check in ("dB-band", "dB-vector"):
        e = band_db_errors(db[s], E[s], A, scale=scale)
    if check == "y":
        v = y_errors([q[s] for q in ys], [q[s] for q in Y])["worst_ratio"] / scale
        return v, v <= 1.0
    if check.endswith("vector"):
        return e["vector_rel"], e["vector_rel"] < TOL
    return e["worst_ratio"], e["worst_ratio"] <= 1.0


@functools.lru_cache(maxsize=None)
def model_measure(mp, signal, check, scale=1.0):
    bpo, n_oct, block, T = mp
    _, _, E, Y = bs.signal_set(bpo, n_oct, block, T)
    Em, Ym = model_run(*mp)
    A = a_weights(bpo, n_oct)
    return measure(check, NAMES.index(signal), E, Y, Em, Ym, 10 * np.log10(Em + 1e-30) + A, A, scale)


def cases():
    out = []
    for p in PLANS:
        for name in NAMES:
            for check in CHECKS:
                if check == "y" and not p[4]:
                    continue
                mark = ()
                lim = MODEL_LIMITED.get(model_plan(p) + (name, check))
                exc = KNOWN_EXCESS.get((p[6], name, check))
                if lim is not None:
                    mark = pytest.mark.xfail(strict=False, reason="float32 limit: the model gives %.3g" % lim)
                elif exc is not None:
                    mark = pytest.mark.xfail(strict=True, reason="kernel excess over the float32 model: %.3g"
                                             % exc)
                out.append(pytest.param(p, name, check, marks=mark,
                                        id="%s-%s-%s" % (plan_id(p), name, check)))
    return out


# --------------------------------------------------------------------------- CPU: the bound itself
def test_cases_cover_every_instance():
    assert {c[-1] for c in CASES} == INSTANCES
    assert {p[6] for p in PLANS} >= INSTANCES


@pytest.mark.parametrize("bpo,n_oct,block,response_time", MODEL_PLANS)
def test_float32_model_uses_a_quarter_of_the_bound(bpo, n_oct, block, response_time):
    """The float32 model passes a quarter of the per-band bound (energies, dB image, y) on every
    signal except the two that reach the bands through the zeros at z = +-1; silence from reset
    stays exactly 0."""
    mp = (bpo, n_oct, block, response_time)
    Em, _ = model_run(*mp)
    assert np.all(Em[NAMES.index("zeros")] == 0.0)
    over = {}
    for name in NAMES:
        if name in ZERO_LIMITED:
            continue
        # each value is the fraction used of the bound scaled by 1/4 (for dB: of the dB image of a
        # quarter of the energy bound; the image is compressive, so it is not a quarter in dB)
        used = {c: model_measure(mp, name, c, 0.25) for c in ("energy-band", "dB-band", "y")}
        if not all(ok for _, ok in used.values()):
            over[name] = {c: round(v, 3) for c, (v, _) in used.items()}
    assert not over, over


@pytest.mark.parametrize("mp", sorted({model_plan(p) for p in PLANS}))
def test_model_limited_lists_exactly_the_model_failures(mp):
    """MODEL_LIMITED holds exactly the (signal, check) on which the float32 model fails, with its
    number to 10 %: nothing the model passes is exempt."""
    fails = {}
    for name in NAMES:
        for check in CHECKS:
            v, ok = model_measure(mp, name, check)
            if not ok:
                fails[mp + (name, check)] = v
    listed = {k: v for k, v in MODEL_LIMITED.items() if k[:4] == mp}
    assert set(fails) == set(listed), (sorted(set(fails) - set(listed)), sorted(set(listed) - set(fails)))
    for k, v in fails.items():
        assert abs(listed[k] - v) <= 0.1 * v, (k, v, listed[k])


def _mutations(bpo, n_oct, block, response_time):
    """The oracle energies and four mistakes a kernel could make, as energies [S, blocks, bands]."""
    from friture_b200.octavefilters import smoothing_alphas
    bank, _, E, Y = bs.signal_set(bpo, n_oct, block, response_time)
    alphas = smoothing_alphas(response_time, n_oct)
    j = n_oct - 1                                 # the lowest-rate stage: bands 0 .. bpo-1
    L = block >> j
    low = range(bpo)
    # the oracle's smoothing as a float64 recursion (checked against the oracle: a sanity check of the
    # mutations, which reuse it)
    for k in low:
        assert np.allclose(bs.smooth64(Y[k], alphas[j], L), E[:, :, k], rtol=1e-9, atol=0)
    muts = {}
    # 1. one quiet band off by 1e-3: the band ~40 dB under the loudest one, per signal
    m = E.copy()
    for s in range(len(E)):
        rel = E[s].min(axis=0) / np.maximum(E[s].max(axis=(0, 1)), 1e-300)
        k = int(np.argmin(np.abs(np.log10(np.maximum(rel, 1e-300)) + 4)))
        m[s, :, k] *= 1 + 1e-3
    muts["quiet band x(1+1e-3)"] = m
    # 2. the smoothing decay of the lowest octave off by 1e-4
    m = E.copy()
    for k in low:
        m[:, :, k] = bs.smooth64(Y[k], alphas[j] * (1 + 1e-4), L)
    muts["decay of one octave x(1+1e-4)"] = m
    # 3. the lowest stage's block-end energies one sample late
    m = E.copy()
    for k in low:
        m[:, :, k] = bs.smooth64(Y[k], alphas[j], L, shift=1)
    muts["block end one sample late"] = m
    # 4. the chain gain of band 0 rounded to 8 significant bits (every octave's band 0)
    g = float(np.prod(np.asarray(bank._sos_band, dtype=np.float64).reshape(bpo, 2, 6)[0, :, 0]))
    mant, ex = np.frexp(g)
    gr = np.ldexp(np.round(mant * 256) / 256, ex)
    m = E.copy()
    m[:, :, 0::bpo] *= (gr / g) ** 2
    muts["chain gain rounded to 8 bits"] = m
    return E, muts


@pytest.mark.parametrize("bpo,n_oct,block,response_time", [(3, 9, 256, 0.025)])
def test_bound_rejects_what_the_vector_criterion_misses(bpo, n_oct, block, response_time):
    E, muts = _mutations(bpo, n_oct, block, response_time)
    for i, (what, m) in enumerate(muts.items()):
        caught = [n for s, n in enumerate(NAMES) if band_errors(m[s], E[s])["worst_ratio"] > 1.0]
        missed_by_vector = [n for s, n in enumerate(NAMES)
                            if n in caught and band_errors(m[s], E[s])["vector_rel"] < TOL]
        assert caught, what
        if i < 3:
            assert missed_by_vector, what
    # the bound is not so loose that a relative error just above BAND_REL_TOL on a loud band passes
    s = NAMES.index("white_noise")
    assert band_errors(E[s] * (1 + 1.5 * BAND_REL_TOL), E[s])["worst_ratio"] > 1.0


def test_bound_exact_zero_nan_and_negative():
    ref = np.array([[0.0, 1e-3, 1.0]])
    assert band_errors(ref, ref)["worst_ratio"] == 0.0
    assert band_errors(np.array([[1e-45, 1e-3, 1.0]]), ref)["worst_ratio"] == np.inf
    assert band_errors(np.array([[0.0, np.nan, 1.0]]), ref)["worst_ratio"] == np.inf
    assert band_errors(np.array([[-0.0, -1e-3, 1.0]]), ref)["worst_ratio"] == np.inf
    # below FLT_MIN on an absolute scale: a float32 subnormal rounding of a tiny reference passes
    tiny = np.array([[1e-40, 1e-3, 1.0]])
    assert band_errors(np.array([[0.0, 1e-3, 1.0]]), tiny)["worst_ratio"] <= 1.0
    assert band_db_errors(10 * np.log10(ref + 1e-30), ref)["worst_ratio"] <= 1.0


@pytest.mark.parametrize("bpo,n_oct,block,response_time", [
    (3, 9, 256, 0.025), (3, 9, 512, 0.025), (1, 9, 512, 0.025), (24, 9, 512, 0.025)])
def test_bound_rejects_what_the_vector_criterion_misses(bpo, n_oct, block, response_time):
    E, muts = _mutations(bpo, n_oct, block, response_time)
    for i, (what, m) in enumerate(muts.items()):
        caught = [n for s, n in enumerate(NAMES) if band_errors(m[s], E[s])["worst_ratio"] > 1.0]
        missed_by_vector = [n for s, n in enumerate(NAMES)
                            if n in caught and band_errors(m[s], E[s])["vector_rel"] < TOL]
        assert caught, what
        if i < 3:
            assert missed_by_vector, what
    # the bound is not so loose that a relative error just above BAND_REL_TOL on a loud band passes
    s = NAMES.index("white_noise")
    assert band_errors(E[s] * (1 + 1.5 * BAND_REL_TOL), E[s])["worst_ratio"] > 1.0


def test_bound_exact_zero_nan_and_negative():
    ref = np.array([[0.0, 1e-3, 1.0]])
    assert band_errors(ref, ref)["worst_ratio"] == 0.0
    assert band_errors(np.array([[1e-45, 1e-3, 1.0]]), ref)["worst_ratio"] == np.inf
    assert band_errors(np.array([[0.0, np.nan, 1.0]]), ref)["worst_ratio"] == np.inf
    assert band_errors(np.array([[-0.0, -1e-3, 1.0]]), ref)["worst_ratio"] == np.inf
    # below FLT_MIN on an absolute scale: a float32 subnormal rounding of a tiny reference passes
    tiny = np.array([[1e-40, 1e-3, 1.0]])
    assert band_errors(np.array([[0.0, 1e-3, 1.0]]), tiny)["worst_ratio"] <= 1.0
    assert band_db_errors(10 * np.log10(ref + 1e-30), ref)["worst_ratio"] <= 1.0


# --------------------------------------------------------------------------- GPU: every kernel instance
def on_device(x, C):
    """the S signal rows repeated to C >= S channels on the GPU"""
    import torch
    k = len(x)
    return torch.from_numpy(np.ascontiguousarray(x)).cuda().repeat((C + k - 1) // k, 1)[:C].contiguous()


def distinct(out, k):
    """out[:k] (numpy) after checking that every channel equals its distinct row bit for bit."""
    import torch
    idx = torch.arange(out.shape[0], device=out.device) % k
    assert torch.equal(out, out[idx]), "repeated rows differ"
    return out[:k].cpu().numpy().astype(np.float64)


@functools.lru_cache(maxsize=None)
def run_kernel(bpo, n_oct, channels, block, want_y, response_time):
    """Energies (and y) of the signal set through Octave_Filters.filter_batch on max(channels, S)
    channels (the kernel choice depends on the channel count only through the 1536 and 3072
    thresholds, so this runs the kernel test_bank_dispatch_gpu.py pins for `channels`), then the dB
    energies with A-weighting from a fresh bank through the same kernel (same want_y)."""
    from friture_b200.octavefilters import Octave_Filters
    _, x, _, _ = bs.signal_set(bpo, n_oct, block, response_time)
    S = len(x)
    xd = on_device(x, max(channels, S))
    bank = Octave_Filters(bpo, n_octaves=n_oct, response_time=response_time)
    y, e = bank.filter_batch(xd, block=block, want_y=want_y)
    got = distinct(e, S)
    ys = [distinct(v, S) for v in y] if want_y else None
    del y
    bank = Octave_Filters(bpo, n_octaves=n_oct, response_time=response_time)
    bank.set_weighting("A")
    db = distinct(bank.filter_batch(xd, block=block, want_y=want_y, db=True)[1], S)
    return got, ys, db, np.asarray(bank.A, dtype=np.float32).astype(np.float64)


@pytest.mark.gpu
@pytest.mark.parametrize("plan,signal,check", cases())
def test_band_by_band(plan, signal, check):
    bpo, n_oct, channels, block, want_y, T, _ = plan
    _, _, E, Y = bs.signal_set(bpo, n_oct, block, T)
    got, ys, db, A = run_kernel(bpo, n_oct, channels, block, want_y, T)
    s = NAMES.index(signal)
    v, ok = measure(check, s, E, Y, got, ys, db, A)
    m, _ = model_measure(model_plan(plan), signal, check)
    print("BANDS %s %s %s kernel %.3g model %.3g" % (plan_id(plan), signal, check, v, m))
    assert ok, (v, "model", m)


@functools.lru_cache(maxsize=None)
def run_analyzer(path):
    import torch
    from friture_b200.analyzer import ChannelAnalyzer
    _, x, _, _ = bs.signal_set(3, 10, 1024, 1.0)
    an = ChannelAnalyzer(len(x))
    if path == "device":
        return an.process(torch.from_numpy(x).cuda())[1].cpu().numpy().astype(np.float64)
    return an.process_host(torch.from_numpy(x).pin_memory())[1].numpy().astype(np.float64)


ANALYZER = [pytest.param(path, name, check, id="%s-%s-%s" % (path, name, check),
                         marks=(pytest.mark.xfail(strict=False, reason="float32 limit: the model gives %.3g"
                                                  % MODEL_LIMITED[(3, 10, 1024, 1.0, name, check)])
                                if (3, 10, 1024, 1.0, name, check) in MODEL_LIMITED else
                                pytest.mark.xfail(strict=True, reason="kernel excess over the float32 model")
                                if ("analyzer", name, check) in KNOWN_EXCESS else ()))
            for path in ("device", "host") for name in NAMES for check in ("dB-band", "dB-vector")]


@pytest.mark.gpu
@pytest.mark.parametrize("path,signal,check", ANALYZER)
def test_channel_analyzer_band_by_band(path, signal, check):
    """ChannelAnalyzer reaches the bank through frt_bank_process_strided (dB without weighting,
    10 octaves, hop 1024), on the device path and on the host path."""
    _, _, E, Y = bs.signal_set(3, 10, 1024, 1.0)
    zero = np.zeros(E.shape[-1])
    v, ok = measure(check, NAMES.index(signal), E, Y, None, None, run_analyzer(path), zero)
    m, _ = model_measure((3, 10, 1024, 1.0), signal, check)
    print("BANDS analyzer-%s %s %s kernel %.3g model %.3g" % (path, signal, check, v, m))
    assert ok, (v, "model", m)
