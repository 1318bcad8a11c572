"""CPU: the oracle of the octave widget's levels on its live bank (LiveOctaveSpectrumOracle) against
the reference's own outputs (tests/golden/octave_widget_live.npz), and OctaveSpectrumAnalyzer's
argument checks, which all run before any GPU handle exists."""
import os

import numpy as np
import pytest

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "octave_widget_live.npz")
SERIES = [(3, 512, 125), (3, 512, 1000), (24, 512, 125), (24, 512, 1000), (3, 1024, 1000)]


def load():
    with np.load(GOLD) as d:
        return {k: d[k] for k in d.files}


@pytest.mark.parametrize("bpo,block,ms", SERIES)
def test_live_oracle_matches_reference(bpo, block, ms):
    from friture_b200 import filter_data
    from oracle import friture_oracle as fo
    from oracle.live_octave import LiveOctaveSpectrumOracle
    g = load()
    orc = LiveOctaveSpectrumOracle(*filter_data.fir_taps(bpo), response_time=ms / 1000.)
    key = "bpo%d_block%d_t%d" % (bpo, block, ms)
    ref = g["sp_" + key]
    got = np.array([orc.push(g["x"][b * block:(b + 1) * block])[0] for b in range(ref.shape[0])])
    np.testing.assert_allclose(got, ref, rtol=1e-12, atol=0)
    if "db_A_" + key in g:
        A = fo.weighting_tables(fo.octave_frequencies(9 * bpo, bpo)[0], eps=0.0)[0]
        np.testing.assert_allclose(10 * np.log10(got + 1e-30) + A, g["db_A_" + key], rtol=1e-12)


def test_live_oracle_response_time_keeps_state():
    """set_response_time changes the smoothing from the next block on, nothing before it."""
    from friture_b200 import filter_data
    from oracle.live_octave import LiveOctaveSpectrumOracle
    x = load()["x"]
    a = LiveOctaveSpectrumOracle(*filter_data.fir_taps(3), response_time=1.0)
    b = LiveOctaveSpectrumOracle(*filter_data.fir_taps(3), response_time=1.0)
    for i in range(4):
        assert np.array_equal(a.push(x[i * 512:(i + 1) * 512])[0], b.push(x[i * 512:(i + 1) * 512])[0])
    b.set_response_time(0.125)
    sa, sb = a.push(x[2048:2560])[0], b.push(x[2048:2560])[0]
    assert not np.array_equal(sa, sb)
    with pytest.raises(ValueError):
        a.push(x[:2048])          # a stream keeps to one side of the 1024-sample line


@pytest.mark.parametrize("bpo", [3, 24])
def test_direct_form_matches_fft_form(bpo):
    """The form used above 1024 samples computes the same levels as the reference's FFT form."""
    from friture_b200 import filter_data
    from oracle import friture_oracle as fo
    from oracle.live_octave import LiveOctaveSpectrumOracle
    x = (np.random.default_rng(5).standard_normal(8 * 512) * 0.1).astype(np.float32)
    taps = filter_data.fir_taps(bpo)
    f = LiveOctaveSpectrumOracle(*taps)
    d = LiveOctaveSpectrumOracle(*taps)
    d.form = "direct"
    for b in range(8):
        xb = x[b * 512:(b + 1) * 512].astype(np.float64)
        ef = f.push(xb)[0]
        y, d.hist = fo.fir_bank_direct(d.boct_fir, d.bdec_fir, xb, d.hist)
        d.dispbuffers = [fo.exp_smoothed_value(k, a, yy ** 2, old)
                         for yy, k, a, old in zip(y, d.kernels, d.alphas, d.dispbuffers)]
        np.testing.assert_allclose(np.array(d.dispbuffers), ef, rtol=1e-9)


def test_analyzer_argument_checks_without_gpu():
    import torch
    from friture_b200.octavespectrum import OctaveSpectrumAnalyzer
    an = OctaveSpectrumAnalyzer(2)
    assert an.nbands == 27 and an.bandsperoctave == 3 and len(an.f_nominal) == 27
    assert an.alphas.shape == (9,) and an.filters._handle is None
    x = torch.zeros((2, 1024), dtype=torch.float32)
    bad = [
        (torch.zeros((2, 1024), dtype=torch.float64), 512),      # dtype
        (torch.zeros((3, 1024), dtype=torch.float32), 512),      # channel count
        (torch.zeros((2, 2, 512), dtype=torch.float32), 512),    # shape
        (x, 384),                                                # not a multiple of 256
        (x, 0),
        (torch.zeros((2, 8192), dtype=torch.float32), 8192),     # longer than 4096
        (torch.zeros((2, 1000), dtype=torch.float32), 256),      # T % block
        (torch.zeros((2, 0), dtype=torch.float32), 256),         # empty
        (torch.zeros((1024, 2), dtype=torch.float32).t(), 512),  # not contiguous along time
        (x, 512),                                                # a CPU tensor
        (np.zeros((2, 1024), dtype=np.float32), 512),            # not a tensor
    ]
    for xx, block in bad:
        with pytest.raises(ValueError):
            an.process(xx, block=block)
    with pytest.raises(ValueError):
        an.setweighting(4)
    an.setweighting("A")
    assert np.array_equal(an._w, np.float32(an.filters.A))
    an.setbandsperoctave(24)
    assert an.nbands == 216 and an._w.shape == (216,)
    an.setresponsetime(0.125)
    assert an.alphas[0] > OctaveSpectrumAnalyzer(2).alphas[0]
    assert an.filters._handle is None      # nothing above needed a GPU
