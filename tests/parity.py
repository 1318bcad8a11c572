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


# Filterbank band energies are judged band by band, per channel and per block, on top of the vector
# criterion above (which divides by the loudest band, so a band 50 dB down is effectively unchecked):
#     |e[k] - e_ref[k]| <= BAND_REL_TOL * e_ref[k] + BAND_FLOOR * max_k' e_ref[k']  (+ FLT_MIN)
# The FLT_MIN term judges energies in the float32 subnormal range on an absolute scale; where
# e_ref[k] is exactly 0 (silence from reset) e[k] must be exactly 0.  NaN and negative values fail.
# Calibration: tests/bank_f32_model.py runs the kernels' arithmetic (normalised float32 sections,
# chain gains applied once per chain, decimation, the chunked float32 smoothing) against the float64
# oracle on the signal set of tests/bank_signals.py (tones at band centres, on a band edge and in a
# decimator's transition band, a log sweep, impulses at block ends and at odd / even decimated
# samples, silence, a burst decaying into silence, clipped full-scale noise, noise at 1e-6 and 1e-12,
# white noise) at bpo 1 .. 24, 9 and 10 octaves, blocks 256 .. 1024 and response times 0.025 .. 5 s.
# It needs a relative term of 5e-5 (the lowest bands of the 1/12 and 1/24-octave banks during the
# start-up transient of a low tone) and a floor of 1e-11 of the loudest band (stopband bands of the
# tones, whose float32-rounded coefficients move the response's deep nulls); the constants are four
# times that, so the model uses at most a quarter of the bound (tests/test_bank_bands_gpu.py checks
# this, and that the bound rejects a quiet band off by 1e-3, a smoothing decay off by 1e-4, a block
# end one sample late and a chain gain rounded to fewer bits).
# Two inputs are outside that calibration: a DC offset and a Nyquist-rate sequence reach the bands
# only through the zeros at z = +-1, where the normalised numerator x + c*x1 + x2 (c ~ -+2) cancels
# to 1e-4 of its terms; float32 loses ~4 digits there (the model is off by up to 1.9e-4 and 4.8e-4
# of the loudest band).  Tests hold kernels on such inputs to a multiple of the model's own error.
BAND_REL_TOL = 2e-4
BAND_FLOOR = 4e-11
FLT_MIN = float(np.finfo(np.float32).tiny)
# ragged band outputs y, per sample: relative to the band's own peak plus a floor relative to the
# loudest band's peak (same model and signals; the model uses at most a quarter of it)
Y_REL_TOL = 4e-4
Y_FLOOR = 1e-5


def band_bound(ref, scale=1.0):
    """Allowed |e - e_ref| for band energies ref [..., bands] (see above); `scale` shrinks the
    relative and floor terms (scale=0.25: the quarter of the bound the float32 model may use)."""
    ref = np.asarray(ref, dtype=np.float64)
    top = np.max(ref, axis=-1, keepdims=True)
    return scale * (BAND_REL_TOL * ref + BAND_FLOOR * top) + np.where(ref > 0, FLT_MIN, 0.0)


def _worst(ratio):
    ratio = np.where(np.isnan(ratio), np.inf, ratio)
    if ratio.size == 0:
        return {"worst_ratio": 0.0, "worst_index": None}
    i = int(np.argmax(ratio))
    return {"worst_ratio": float(ratio.flat[i]), "worst_index": np.unravel_index(i, ratio.shape)}


def band_errors(got, ref, scale=1.0):
    """got, ref: [..., bands] smoothed band energies.  Returns worst_ratio (largest error over the
    bound, inf for a NaN, a negative value or a nonzero value where ref is exactly 0), its index, and
    vector_rel (the north-star vector criterion, max over vectors of max|got-ref| / max(ref))."""
    got = np.asarray(got, dtype=np.float64)
    ref = np.asarray(ref, dtype=np.float64)
    assert got.shape == ref.shape, (got.shape, ref.shape)
    allowed = np.where(ref > 0, band_bound(ref, scale), 0.0)
    err = np.abs(got - ref)
    with np.errstate(invalid="ignore", divide="ignore"):
        ratio = np.where(allowed > 0, err / allowed, np.where(err == 0, 0.0, np.inf))
    ratio = np.where(got < 0, np.inf, ratio)
    e = _worst(ratio)
    top = np.max(ref, axis=-1, keepdims=True)
    with np.errstate(invalid="ignore", divide="ignore"):
        vec = np.where(top > 0, err / top, np.where(err == 0, 0.0, np.inf))
    e["vector_rel"] = float(np.max(np.where(np.isnan(vec), np.inf, vec))) if vec.size else 0.0
    return e


def band_db_errors(got_db, ref, weight=0.0, scale=1.0):
    """got_db: [..., bands] 10*log10(e + 1e-30) + weight from a kernel; ref: the reference band
    ENERGIES.  The bound is the dB image of band_bound, 10*log10(1 + bound / (e_ref + 1e-30)) (both
    sides saturate at 10*log10(1e-30) + weight), plus 4 float32 ulps of the dB value itself."""
    got_db = np.asarray(got_db, dtype=np.float64)
    ref = np.asarray(ref, dtype=np.float64)
    ref_db = 10.0 * np.log10(ref + 1e-30) + weight
    allowed = (10.0 * np.log10(1.0 + band_bound(ref, scale) / (ref + 1e-30))
               + 4.0 * np.abs(ref_db) * float(np.finfo(np.float32).eps))
    e = _worst(np.abs(got_db - ref_db) / allowed)
    e["vector_rel"] = rel_err(got_db, ref_db)
    return e


def y_errors(got, ref):
    """got, ref: lists (one per band) of [..., samples] ragged band outputs of the same channels.
    Bound per sample: Y_REL_TOL * (band's peak) + Y_FLOOR * (loudest band's peak), per channel;
    exactly 0 where every band of the channel is exactly 0."""
    peaks = np.stack([np.max(np.abs(np.asarray(r, dtype=np.float64)), axis=-1) for r in ref], axis=-1)
    top = np.max(peaks, axis=-1)
    worst = {"worst_ratio": 0.0, "worst_index": None}
    for k, (g, r) in enumerate(zip(got, ref)):
        g = np.asarray(g, dtype=np.float64)
        r = np.asarray(r, dtype=np.float64)
        allowed = (Y_REL_TOL * peaks[..., k] + Y_FLOOR * top)[..., None]
        err = np.abs(g - r)
        with np.errstate(invalid="ignore", divide="ignore"):
            ratio = np.where(allowed > 0, err / allowed, np.where(err == 0, 0.0, np.inf))
        e = _worst(ratio)
        if e["worst_ratio"] > worst["worst_ratio"]:
            worst = {"worst_ratio": e["worst_ratio"], "worst_index": (k,) + tuple(e["worst_index"])}
    return worst
