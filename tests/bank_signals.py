"""Signals on which a multirate float32 IIR filterbank goes wrong, and a cached float64 oracle for
them (tests/test_bank_bands_gpu.py).

Each signal is one channel row, so one kernel launch checks all of them.  The set depends on the
bank (its band centres and edges) and on the block length (impulses at block ends)."""
import functools

import numpy as np

FS = 48000
N_SAMPLES = 49152          # 1.02 s: a whole number of every block length the tests use (<= 4096, 768, 1536)
BURST = 4096               # noise burst, then silence


def signal_names():
    return ["tone_top", "tone_mid", "tone_bottom", "tone_edge", "tone_dec_transition",
            "tone_dec_alias", "log_sweep", "dc_offset", "nyquist", "impulse_block_last",
            "impulse_block_first", "impulse_odd", "impulse_even", "zeros", "burst_then_silence",
            "clipped_full_scale", "noise_1e-6", "noise_1e-12", "white_noise"]


def _tone(f, n, amp=0.5):
    t = np.arange(n, dtype=np.float64)
    return amp * np.sin(2 * np.pi * f / FS * t + 0.3)


def make_signals(fi, fhigh, block, n=N_SAMPLES, seed=1234):
    """[len(signal_names()), n] float32 rows.  fi, fhigh: the bank's band centres and upper edges."""
    rng = np.random.default_rng(seed)
    nb = len(fi)
    mid_block = (n // block) // 2 * block         # start of a block in the middle of the signal
    rows = {}
    rows["tone_top"] = _tone(fi[-1], n)
    rows["tone_mid"] = _tone(fi[nb // 2], n)
    rows["tone_bottom"] = _tone(fi[0], n)
    rows["tone_edge"] = _tone(fhigh[nb // 2], n)                    # shared edge of two bands
    # stage 1 (rate fs/2) decimator: just below its output Nyquist fs/8, and just above it
    rows["tone_dec_transition"] = _tone(0.95 * FS / 8, n)
    rows["tone_dec_alias"] = _tone(1.05 * FS / 8, n)
    t = np.arange(n, dtype=np.float64) / FS
    dur = n / FS
    k = np.log(20000.0 / 20.0)
    rows["log_sweep"] = 0.5 * np.sin(2 * np.pi * 20.0 * dur / k * (np.exp(t / dur * k) - 1.0))
    rows["dc_offset"] = 0.5 + 0.5e-3 * rng.standard_normal(n)     # noise 60 dB below the offset
    rows["nyquist"] = 0.5 * (1.0 - 2.0 * (np.arange(n) & 1))
    for name, at in (("impulse_block_last", mid_block - 1), ("impulse_block_first", mid_block),
                     ("impulse_odd", mid_block + 8 * 37),        # odd sample of stage 3 (rate fs/8)
                     ("impulse_even", mid_block + 8 * 38)):      # even sample of stage 3
        v = np.zeros(n)
        v[at] = 1.0
        rows[name] = v
    rows["zeros"] = np.zeros(n)
    v = np.zeros(n)
    v[:BURST] = 0.3 * rng.standard_normal(BURST)
    rows["burst_then_silence"] = v
    rows["clipped_full_scale"] = np.clip(rng.standard_normal(n), -1.0, 1.0)   # ~32 % exactly +-1
    rows["noise_1e-6"] = 1e-6 * rng.standard_normal(n)
    rows["noise_1e-12"] = 1e-12 * rng.standard_normal(n)
    rows["white_noise"] = 0.1 * rng.standard_normal(n)
    return np.stack([rows[s] for s in signal_names()]).astype(np.float32)


@functools.lru_cache(maxsize=None)
def _cached(bpo, n_octaves, block, response_time, n):
    from friture_b200.octavefilters import Octave_Filters
    bank = Octave_Filters(bpo, n_octaves=n_octaves, response_time=response_time)
    x = make_signals(bank.fi, bank.fhigh, block, n)
    E, Y = oracle_run_whole(bank, x, block, n_octaves, response_time)
    for a in (x, E, *Y):
        a.setflags(write=False)
    return bank, x, E, Y


def signal_set(bpo, n_octaves, block, response_time=1.0, n=N_SAMPLES):
    """(bank, x [S, n] float32, oracle energies [S, n/block, nbands] float64, oracle y: list of
    nbands arrays [S, n >> j]) for the bank plan, cached per plan, block and response time."""
    return _cached(bpo, n_octaves, block, response_time, n)


def oracle_run_whole(bank, x, block, n_octaves, response_time):
    """OctaveSpectrumOracle on every row: the IIR bank over the whole row in one call (the same
    float64 recursion as block by block: lfilter carries its state exactly and every block is even
    at every stage), then the widget's exp_smoothed_value block by block as push() does."""
    from oracle import friture_oracle as fo
    S, T = x.shape
    nb = T // block
    E = np.zeros((S, nb, bank.nbands))
    Y = [np.zeros((S, T >> (n_octaves - 1 - k // bank.bandsperoctave))) for k in range(bank.nbands)]
    for s in range(S):
        orc = fo.OctaveSpectrumOracle(bank.bdec, bank.adec, bank.boct, bank.aoct,
                                      response_time=response_time, noctave=n_octaves)
        y, dec = orc.filter(x[s].astype(np.float64))
        prev = [0.0] * bank.nbands
        for k in range(bank.nbands):
            Y[k][s] = y[k]
            L = block // dec[k]
            y2 = y[k] ** 2
            for b in range(nb):
                prev[k] = fo.exp_smoothed_value(orc.kernels[k], orc.alphas[k], y2[b * L:(b + 1) * L], prev[k])
                E[s, b, k] = prev[k]
    return E, Y


def smooth64(y, alpha, L, shift=0):
    """float64 smoothing of y^2 [S, n] (rate of the band) sampled at block ends every L samples,
    shifted by `shift` samples (the oracle's values for shift 0, up to rounding)."""
    from scipy.signal import lfilter
    e = lfilter([alpha], [1.0, -(1.0 - alpha)], y ** 2, axis=-1)
    idx = np.arange(1, y.shape[-1] // L + 1) * L - 1 + shift
    return e[:, np.minimum(idx, y.shape[-1] - 1)]
