"""CPU: the float32 model of the long GCC-PHAT path (tests/gcc_long_model.py) stays within the bound
of test_gcc_lengths_gpu against the float64 oracle, and plausible kernel bugs planted in it exceed
that bound; the path chooser picks the shared-memory kernel for exactly the widget lengths that
kernel takes; the golden fixture of the long lengths matches the oracle."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import gcc_long_model as gm  # noqa: E402
from test_gcc_lengths_gpu import PAIR_KINDS, bound_check, length_cases  # noqa: E402

from oracle import friture_oracle as fo  # noqa: E402

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
BUGS = {"chirp n^2 mod L": dict(mod_2n=False), "M one power of two short": dict(m_short=True),
        "odd L inverted at length L": dict(odd_inverse_at_L=True),
        "conjugated twiddle": dict(conj_twiddle=True)}


@pytest.mark.parametrize("L", [16800, 26400, 55199, 240000])
def test_model_within_bound_and_bugs_exceed_it(L):
    d0, d1, _ = length_cases(L)
    excess = {k: [] for k in BUGS}
    for p in range(8):
        ref = gm.gcc_f64(d0[p], d1[p])
        f32 = gm.gcc_f32_any(d0[p], d1[p])
        assert ref.shape == (gm.out_length(L),)
        err, bound, ratio = bound_check(gm.gcc_long(d0[p], d1[p]), ref, f32)
        assert err <= bound, (PAIR_KINDS[p], err, bound, ratio)
        for name, kw in BUGS.items():
            if name.startswith("odd") and L % 2 == 0:
                continue
            err, bound, _ = bound_check(gm.gcc_long(d0[p], d1[p], **kw), ref, f32)
            excess[name].append(err / bound)
    for name, e in excess.items():
        if e:
            assert min(e) > 1, (name, e)


def widget_lengths():
    """L = int(2 * range * 12000) for the widget's ranges 0.1 .. 1000 s in 0.1 s steps
    (friture/delay_estimator.py:114-117,222-226)."""
    return [int(2 * (r / 10) * 12000.0) for r in range(1, 10001)]


def test_path_choice_over_every_widget_range():
    """frt_gcc_fits (pure host code) takes exactly the ranges 0.1 .. 1.0 s except 0.7 s; the other
    9 991 settings go to the long path, whose limits they all satisfy."""
    from friture_b200 import _lib
    lib = _lib.load_library()
    lengths = widget_lengths()
    fits = [r + 1 for r, L in enumerate(lengths) if lib.frt_gcc_fits(L)]
    assert fits == [1, 2, 3, 4, 5, 6, 8, 9, 10]
    rest = [L for L in lengths if not lib.frt_gcc_fits(L)]
    assert len(rest) == 9991 and min(rest) >= 4 and max(rest) == 24000000
    assert sum(L % 2 for L in lengths) == 746
    assert lengths[22] == 55199 and lengths[6982] == 16759199
    assert not any(lib.frt_gcc_fits(L) for L in (2, 3, 2401, 16800, 28160, 28800, 30000))


def test_golden_matches_oracle():
    """The fixture's inputs are rebuilt by exact integer arithmetic; the oracle matches the
    reference's outputs stored at the fixture's indices to 1e-12."""
    from oracle.make_golden_gcc_long import golden_frames, golden_indices
    g = np.load(os.path.join(GOLD, "gcc_long.npz"))
    for L in (16800, 55199, 240000):
        (a0, a1), (b0, b1) = golden_frames(L)
        xa = fo.generalized_cross_correlation(a0, a1)
        assert xa.shape == (gm.out_length(L),) and int(g["n_out_%d" % L]) == gm.out_length(L)
        xb = fo.generalized_cross_correlation(b0, b1)
        ia, _, sa = fo.delay_peak(xa)
        ib, _, sm = fo.delay_peak(xb, sa)
        idx = g["index_%d" % L]
        assert np.array_equal(idx, golden_indices(len(xa), ib))
        assert np.allclose(xa[idx], g["xcorr_%d" % L], rtol=0, atol=1e-12)
        assert np.allclose(sm[idx], g["smoothed_%d" % L], rtol=0, atol=1e-12)
        assert [ia, ib] == list(g["argmax_%d" % L]) == [int(0.3 * L)] * 2
