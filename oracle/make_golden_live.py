#!/usr/bin/env python
"""Generate tests/golden/octave_widget_live.npz by running the UNMODIFIED reference (imported in
place via oracle/ref_import.py).  TEST INFRASTRUCTURE ONLY; run where the reference tree exists:

    python oracle/make_golden_live.py

Writes that one file and leaves the other fixtures (oracle/make_golden.py) untouched.

The octave widget's levels on its LIVE bank (friture/octavespectrum.py:91-121,140-156): the
reference's own `Octave_Filters.filter` and `exp_smoothed_value`, with the widget's alphas and
kernels (octavespectrum.py:77-81,140-156) restated.  One seeded float32 stream; series
sp_bpo{bpo}_block{block}_t{ms} [n_blocks, nbands] of smoothed energies, plus one A-weighted dB
series (10*log10(sp + 1e-30) + A, octavespectrum.py:111-121).
"""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from oracle import ref_import  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "octave_widget_live.npz")


def main():
    ref = ref_import.load()
    from friture.filter import NOCTAVE
    from friture.signal.exp_smoothing import exp_smoothed_value
    rng = np.random.default_rng(4242)
    x = (rng.standard_normal(16 * 1024) * 0.1).astype(np.float32)
    d = {"x": x}
    for bpo, block, rt in ((3, 512, 0.125), (3, 512, 1.0), (24, 512, 0.125), (24, 512, 1.0),
                           (3, 1024, 1.0)):
        of = ref.octavefilters.Octave_Filters(bpo)
        decs = of.get_decs()
        alphas = [1. - (1. - 0.65) ** (1. / (rt * 48000 / dec + 1)) for dec in decs]
        kernels = [(1. - a) ** np.arange(int(2 * 4096 / dec) - 1, -1, -1) for a, dec in zip(alphas, decs)]
        disp = [0] * (NOCTAVE * bpo)
        sp = []
        for b in range(16):
            y, _ = of.filter(x[b * block:(b + 1) * block].astype(np.float64))
            disp = [exp_smoothed_value(k, a, yy ** 2, old) for yy, k, a, old in zip(y, kernels, alphas, disp)]
            sp.append(np.array(disp))
        key = "bpo%d_block%d_t%d" % (bpo, block, round(rt * 1000))
        d["sp_" + key] = np.array(sp)
        if (bpo, block, rt) == (3, 512, 1.0):
            d["db_A_" + key] = 10 * np.log10(np.array(sp) + 1e-30) + of.A
    os.makedirs(os.path.dirname(OUT), exist_ok=True)
    np.savez_compressed(OUT, **d)
    print(OUT, os.path.getsize(OUT))


if __name__ == "__main__":
    main()
