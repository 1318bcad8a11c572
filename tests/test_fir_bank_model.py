"""CPU: the float64 model of fir_bank_kernel<R> (tests/fir_bank_model.py) against the oracle's live bank,
its cut invariance, the mistakes its criterion rejects, and the share of samples it pins bit for bit on
the signal set of tests/test_fir_bank_bands_gpu.py."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import fir_bank_model as fm  # noqa: E402
from parity import TOL, rel_err  # noqa: E402

# The GPU test asserts at least these shares of bit-equal y samples and linear levels per plan.  The
# model's own shares on the signal set are printed by test_exact_share_on_the_signal_set: 7 to 8 % of
# the library banks' y samples are tainted.  The lowest shares were 0.940 (y) and 0.911 (levels) here
# (bpo 6 with 10 octaves); they were 0.941 and 0.897 over the GPU test's plans.  The floors sit below.
EXACT_Y_FLOOR = 0.9
EXACT_LEVEL_FLOOR = 0.85


def lib_model(bpo, n_oct, rows, **kw):
    from friture_b200 import filter_data
    from friture_b200.octavefilters import smoothing_alphas
    m = fm.FirBankModel(*filter_data.fir_taps(bpo), n_oct, rows, **kw)
    m.set_smoothing(smoothing_alphas(1.0, n_oct))
    return m


@pytest.mark.parametrize("bpo", [1, 3, 6, 12, 24])
def test_model_matches_the_oracle_within_its_roundings(bpo):
    """Tracking the float32 rounding of every stage sample, the model's intervals hold the float64
    bank of oracle.fir_bank_direct sample by sample and LiveOctaveSpectrumOracle's smoothed energies
    band by band (blocks of 2048: the oracle's direct form)."""
    from friture_b200 import filter_data
    from oracle import friture_oracle as fo
    from oracle.live_octave import LiveOctaveSpectrumOracle
    block, n_oct = 2048, 9
    rng = np.random.default_rng(bpo)
    x = np.stack([0.1 * rng.standard_normal(2 * block), fm.make_signals(bpo, n_oct, block, 2 * block)[1],
                  1e-6 * rng.standard_normal(2 * block)]).astype(np.float32)
    m = lib_model(bpo, n_oct, len(x), track=True)
    res = m.run(x, block, levels=True)
    boct, bdec = filter_data.fir_taps(bpo)
    ys, sp = [], []
    for r in range(len(x)):
        hist = [np.zeros(boct.shape[1] - 1) for _ in range(n_oct)]
        orc = LiveOctaveSpectrumOracle(boct, bdec, noctave=n_oct)
        parts = []
        for b in range(2):
            xb = x[r, b * block:(b + 1) * block].astype(np.float64)
            y, hist = fo.fir_bank_direct(boct, bdec, xb, hist, n_oct)
            parts.append(y)
            sp.append(orc.push(xb)[0])
        ys.append([np.concatenate([p[k] for p in parts]) for k in range(bpo * n_oct)])
    got = [np.stack([ys[r][k] for r in range(len(x))]).astype(np.float32) for k in range(bpo * n_oct)]
    worst, where = fm.y_violations(got, res)
    assert worst == 0.0, (worst, where)
    sp = np.array(sp).reshape(len(x), 2, -1)
    worst, where = fm.level_violations(sp.astype(np.float32), None, res)
    assert worst == 0.0, (worst, where)
    # the intervals are float32 wide, not wider: the oracle is a float64 bank, the model a float32 one
    assert max(np.max(np.abs(res["y"][k][0].astype(np.float64) - ys[0][k])) / np.max(np.abs(ys[0][k]))
               for k in range(bpo * n_oct)) < 1e-6


def test_cut_invariance():
    """Any cut of a stream into calls of whole blocks gives the same model bits, y and levels."""
    block, n_oct, bpo = 256, 9, 3
    x = fm.make_signals(bpo, n_oct, block, 6 * block)
    whole = lib_model(bpo, n_oct, len(x)).run(x, block, levels=True)
    m = lib_model(bpo, n_oct, len(x))
    parts = [m.run(x[:, a * block:b * block], block, levels=True) for a, b in ((0, 1), (1, 4), (4, 6))]
    for k in range(bpo * n_oct):
        for key in ("y", "ylo", "yhi"):
            got = np.concatenate([p[key][k] for p in parts], axis=1)
            assert np.array_equal(got.view(np.int32), whole[key][k].view(np.int32)), (key, k)
    for key in ("sp", "bsp", "lin", "db"):
        got = np.concatenate([p[key] for p in parts], axis=1)
        assert np.array_equal(got, whole[key]), key


def old_criteria(mut, ref, s):
    """The checks the live bank had before the model, on signal row s: every band's y within 1e-5 of
    its peak, every linear band-energy vector within 1e-5 of its peak, every dB vector within TOL."""
    y_ok = all(np.max(np.abs(mut["y"][k][s].astype(np.float64) - ref["y"][k][s]))
               <= 1e-5 * np.max(np.abs(ref["y"][k][s].astype(np.float64))) for k in range(len(ref["y"])))
    e = np.max(np.abs(mut["sp"][s] - ref["sp"][s]) / np.max(np.abs(ref["sp"][s]), axis=-1, keepdims=True))
    return y_ok and e < TOL and rel_err(mut["db"][s].astype(np.float64), ref["db"][s].astype(np.float64)) < TOL


def test_mutants_are_rejected():
    """Each realistic mistake, applied to the model itself, puts some y sample or level outside the
    criterion.  Float32 taps and float32 accumulation pass the checks the bank had before (1e-5 of a
    band's peak, on noise); every mistake here fails the new criterion."""
    block, n_oct, bpo = 512, 9, 3
    x = fm.make_signals(bpo, n_oct, block, 8 * block)
    ref = lib_model(bpo, n_oct, len(x)).run(x, block, levels=True)
    noise = fm.SIGNALS.index("white_full_scale")
    caught, passed_old = {}, []
    for mutant in fm.MUTANTS:
        mut = lib_model(bpo, n_oct, len(x), mutant=mutant).run(x, block, levels=True)
        wy, _ = fm.y_violations(mut["y"], ref)
        wl, _ = fm.level_violations(mut["lin"], mut["db"], ref)
        caught[mutant] = (wy, wl)
        if old_criteria(mut, ref, noise):
            passed_old.append(mutant)
        print("MUTANT %-22s y %-10.3g levels %-10.3g old checks %s"
              % (mutant, wy, wl, "pass" if mutant in passed_old else "fail"))
    assert all(max(v) > 1.0 for v in caught.values()), caught
    assert passed_old == ["taps_float32", "float32_accumulation"], passed_old


def test_unmutated_model_passes_its_own_criterion():
    block, n_oct, bpo = 512, 9, 3
    x = fm.make_signals(bpo, n_oct, block, 4 * block)
    ref = lib_model(bpo, n_oct, len(x)).run(x, block, levels=True)
    assert fm.y_violations(ref["y"], ref) == (0.0, None)
    assert fm.level_violations(ref["lin"], ref["db"], ref) == (0.0, None)


@pytest.mark.parametrize("bpo,n_oct,block", [(1, 9, 512), (3, 9, 256), (6, 10, 1024), (12, 9, 512),
                                             (24, 9, 256), ("syn7-L509", 9, 256), ("syn2-L3", 9, 256)])
def test_exact_share_on_the_signal_set(bpo, n_oct, block):
    """The shares of tainted and of bit-pinned y samples and of bit-pinned linear levels on the GPU
    test's signal set; the GPU floors are set from these."""
    if isinstance(bpo, str):
        b, L = bpo[3:].split("-L")
        m = fm.FirBankModel(*fm.synthetic_taps(int(b), int(L), seed=int(L)), n_oct, len(fm.SIGNALS))
        from friture_b200.octavefilters import smoothing_alphas
        m.set_smoothing(smoothing_alphas(1.0, n_oct))
        nb = int(b)
    else:
        m, nb = lib_model(bpo, n_oct, len(fm.SIGNALS)), bpo
    x = fm.make_signals(nb, n_oct, block, 8 * block)
    res = m.run(x, block, levels=True)
    ey, tf = fm.exact_fraction(res), fm.taint_fraction(res)
    el = float(np.mean(res["linlo"] == res["linhi"]))
    print("TAINT bpo %s oct %d block %d: tainted %.2e, exact y %.6f, exact levels %.4f" % (bpo, n_oct, block, tf, ey, el))
    assert ey >= EXACT_Y_FLOOR and el >= EXACT_LEVEL_FLOOR
