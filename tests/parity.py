"""Parity metrics shared by the GPU tests, the CPU tests and bench.py's parity gate.

north_star: outputs match the reference "within 1e-5 relative float32 on the log-power and
band-energy vectors".  The relative error of a vector is max|got-ref| / max(max|ref|, 1)
(SURVEY.md 8d).

The criterion is asserted STRICTLY (`rel_all`, every bin) on broadband inputs of up to
STRICT_MAX_BINS bins -- the sizes at which north_star's number is defined and measured (bench.py's
parity gate, smoke()).  float32 arithmetic has an amplitude noise floor: a 2048-point float32 FFT
carries an absolute error of about 2e-7 x (rms spectral amplitude of the frame) in every bin,
whatever the bin's own level.  On the dB scale that stays below 1e-5 x max|ref| (about 1e-3 dB)
only for bins above ~ -55 dB of the frame's mean power; for broadband input a bin falls below -50 dB
with probability ~1e-5, so a sample of 1e7 bins is certain to contain dozens of such deep nulls
where NO float32 transform can meet the dB criterion.  Large samples and tonal inputs are therefore
judged bin by bin: the criterion as is for bins no more than FLOOR_DB below the frame's mean power
(>= 99.99 % of the bins of a broadband input, reported), and for every bin, nulls included,
TOL*max|ref| + 20*log10(1 + AMP_TOL*rms/|X_ref|), i.e. the same tolerance widened by the dB image
of an amplitude error of AMP_TOL x (frame rms) -- ~80 float32 epsilons, about 20x the rms rounding
noise of an 11-stage float32 FFT.
"""
import numpy as np

TOL = 1e-5        # relative error of the log-power / band-energy vector
FLOOR_DB = 50.0   # below ~this far under the frame mean power float32 cannot resolve 1e-3 dB
AMP_TOL = 5e-6    # amplitude noise allowance for deep nulls, relative to the frame rms
STRICT_MAX_BINS = 65536    # strict every-bin criterion up to this sample size (expected number of
                           # float32-unresolvable nulls, ~3e-6 per bin, stays below 0.2)


def rel_err(got, ref):
    got = np.asarray(got, dtype=np.float64)
    ref = np.asarray(ref, dtype=np.float64)
    if got.size == 0:
        return 0.0
    return float(np.max(np.abs(got - ref)) / max(np.max(np.abs(ref)), 1.0))


def logpower_errors(got_db, ref_db, eps=1e-30, floor_db=None):
    """got_db, ref_db: [..., bins] log-power (10*log10(P+eps)).  Returns a dict with
    rel_above_floor (vector-relative error over bins >= mean-FLOOR_DB), amp_err (worst
    amplitude error over ALL bins, relative to the frame rms), rel_all, frac_above_floor."""
    got_db = np.asarray(got_db, dtype=np.float64)
    ref_db = np.asarray(ref_db, dtype=np.float64)
    p_ref = np.maximum(10.0 ** (ref_db / 10.0) - eps, 0.0)
    mean_p = np.mean(p_ref, axis=-1, keepdims=True)
    floor_db = 10.0 * np.log10(mean_p + eps) - (FLOOR_DB if floor_db is None else floor_db)
    mask = ref_db >= floor_db
    denom = max(float(np.max(np.abs(ref_db))), 1.0) if ref_db.size else 1.0
    diff = np.abs(got_db - ref_db)
    rms = np.sqrt(mean_p)
    amp_ref = np.sqrt(p_ref)
    noise_db = 20.0 * np.log10(1.0 + AMP_TOL * rms / np.maximum(amp_ref, 1e-300))
    noise_db = np.where(rms > 0, noise_db, 0.0)
    allowed = TOL * denom + noise_db
    return {
        "rel_above_floor": float(np.max(diff[mask]) / denom) if mask.any() else 0.0,
        "rel_all": float(np.max(diff) / denom) if diff.size else 0.0,
        "worst_ratio_all": float(np.max(diff / allowed)) if diff.size else 0.0,
        "frac_above_floor": float(np.mean(mask)) if mask.size else 1.0,
    }


def logpower_ok(e, min_frac=0.9999, strict=False):
    ok = (e["rel_above_floor"] < TOL and e["worst_ratio_all"] < 1.0
          and e["frac_above_floor"] >= min_frac)
    if strict:
        ok = ok and e["rel_all"] < TOL
    return ok


def assert_logpower_parity(got_db, ref_db, min_frac=0.9999, strict=None, floor_db=None):
    """Broadband inputs: strict every-bin criterion up to STRICT_MAX_BINS bins (strict=None picks
    that), and (almost) every bin above the floor.  Tonal inputs, whose mean power is dominated by
    a few bins, pass min_frac=0, strict=False and floor_db=40 (the frame mean is the tone there: the
    float32 noise floor sits only ~45 dB below it)."""
    e = logpower_errors(got_db, ref_db, floor_db=floor_db)
    if strict is None:
        strict = np.asarray(ref_db).size <= STRICT_MAX_BINS and min_frac > 0
    assert logpower_ok(e, min_frac, strict), e
    return e


# Power mode (|X|^2 / N^2, no log) is judged bin by bin on the amplitude scale:
#     |sqrt(P[k]) - sqrt(Pr[k])| <= AMP_TOL * rms + REL_AMP_TOL * sqrt(Pr[k])
# with rms = sqrt(mean_k Pr[k]) of the frame.  AMP_TOL is the float32 transform's amplitude noise
# allowance above; REL_AMP_TOL covers the rounding of a strong bin's own value (float32 window,
# |X|^2 and the 1/N^2 scale).  The bound is scale-free, so it means the same at every FFT size and
# level, and a frame whose reference is exactly zero must come out exactly zero.  numpy's float32
# rfft of float32-windowed frames uses at most 8 % of it on noise, tones, bin-centred cosines, a
# Nyquist sequence and impulses at N = 32 .. 16384 (tests/test_stft_bins_gpu.py checks that, and
# what the bound rejects).
REL_AMP_TOL = 1e-6


def power_errors(got, ref):
    """got, ref: [..., bins] power.  Returns worst_ratio (largest error over the bound above, inf
    for a NaN, a negative value, or anything but 0 where the reference frame is exactly 0) and the
    index of that bin."""
    got = np.asarray(got, dtype=np.float64)
    ref = np.asarray(ref, dtype=np.float64)
    assert got.shape == ref.shape, (got.shape, ref.shape)
    if got.size == 0:
        return {"worst_ratio": 0.0, "worst_index": None}
    amp_ref = np.sqrt(ref)
    rms = np.sqrt(np.mean(ref, axis=-1, keepdims=True))
    allowed = AMP_TOL * rms + REL_AMP_TOL * amp_ref
    with np.errstate(invalid="ignore", divide="ignore"):
        err = np.abs(np.sqrt(got) - amp_ref)
        ratio = np.where(allowed > 0, err / allowed, np.where(err == 0, 0.0, np.inf))
    ratio = np.where(np.isnan(ratio), np.inf, ratio)
    i = int(np.argmax(ratio))
    return {"worst_ratio": float(ratio.flat[i]), "worst_index": np.unravel_index(i, ratio.shape)}


def assert_power_parity(got, ref):
    e = power_errors(got, ref)
    assert e["worst_ratio"] <= 1.0, e
    return e
