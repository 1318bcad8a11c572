"""GPU: OctaveSpectrumAnalyzer, the octave widget's levels on the live FIR bank
(friture/octavespectrum.py:91-163 around friture/filter.py:136-247), against the CPU oracle
(LiveOctaveSpectrumOracle) and the reference's own outputs (tests/golden/octave_widget_live.npz);
cut invariance, the setters' state semantics and exact silence."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from parity import TOL, rel_err  # noqa: E402

pytestmark = pytest.mark.gpu
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "octave_widget_live.npz")


def energy_rel_err(got, ref):
    """relative error of each band-energy vector (per channel, per block)"""
    return float(np.max(np.abs(got - ref) / np.max(np.abs(ref), axis=-1, keepdims=True)))


def make_x(C, T, seed):
    return (np.random.default_rng(seed).standard_normal((C, T)) * 0.1).astype(np.float32)


def oracle_levels(x, bpo, block, response_time=1.0, n_octaves=9):
    from friture_b200 import filter_data
    from oracle.live_octave import LiveOctaveSpectrumOracle
    taps = filter_data.fir_taps(bpo)
    E = []
    for c in range(x.shape[0]):
        orc = LiveOctaveSpectrumOracle(*taps, response_time=response_time, noctave=n_octaves)
        E.append([orc.push(x[c, b * block:(b + 1) * block])[0] for b in range(x.shape[1] // block)])
    return np.array(E)


def run(x, bpo=3, block=512, response_time=1.0, n_octaves=9, weighting=0, db=False):
    import torch
    from friture_b200.octavespectrum import OctaveSpectrumAnalyzer
    an = OctaveSpectrumAnalyzer(x.shape[0], bandsperoctave=bpo, response_time=response_time,
                                weighting=weighting, n_octaves=n_octaves)
    xd = x if isinstance(x, torch.Tensor) else torch.from_numpy(x).cuda()
    return an.process(xd, block=block, db=db).cpu().numpy().astype(np.float64)


def check(x, bpo=3, block=512, response_time=1.0, n_octaves=9):
    E = oracle_levels(x, bpo, block, response_time, n_octaves)
    got = run(x, bpo, block, response_time, n_octaves)
    assert got.shape == E.shape
    assert energy_rel_err(got, E) < TOL
    db = run(x, bpo, block, response_time, n_octaves, db=True)
    assert rel_err(db, 10 * np.log10(E + 1e-30)) < TOL


@pytest.mark.parametrize("bpo", [1, 3, 6, 12, 24])
def test_bands_per_octave(bpo):
    check(make_x(3, 8 * 512, seed=bpo), bpo=bpo)


@pytest.mark.parametrize("block", [256, 1024, 2048, 4096])
def test_block_sizes(block):
    n_blocks = {256: 16, 1024: 8, 2048: 4, 4096: 4}[block]
    check(make_x(2, n_blocks * block, seed=block), block=block)


def test_thirty_bands_ten_octaves():
    check(make_x(2, 8 * 512, seed=30), n_octaves=10)


@pytest.mark.parametrize("response_time", [0.025, 0.125, 0.3, 1.0, 5.0])
def test_response_times(response_time):
    check(make_x(2, 8 * 512, seed=int(response_time * 1000)), response_time=response_time)


@pytest.mark.parametrize("C", [1, 5, 64])
def test_channel_counts(C):
    check(make_x(C, 6 * 512, seed=C))


def test_strided_input():
    import torch
    x = make_x(4, 8 * 512 + 300, seed=8)
    view = torch.from_numpy(x).cuda()[:, 100:100 + 8 * 512]      # row stride 4396
    assert view.stride(0) == 8 * 512 + 300
    E = oracle_levels(np.ascontiguousarray(x[:, 100:100 + 8 * 512]), 3, 512)
    assert energy_rel_err(run(view), E) < TOL


@pytest.mark.parametrize("bpo,block,ms", [(3, 512, 125), (3, 512, 1000), (24, 512, 125),
                                          (24, 512, 1000), (3, 1024, 1000)])
def test_reference_golden(bpo, block, ms):
    with np.load(GOLD) as g:
        x, ref = g["x"], g["sp_bpo%d_block%d_t%d" % (bpo, block, ms)]
        dbA = g["db_A_bpo%d_block%d_t%d" % (bpo, block, ms)] if (bpo, block, ms) == (3, 512, 1000) else None
    xs = x[None, :ref.shape[0] * block]
    got = run(xs, bpo, block, ms / 1000.)[0]
    assert energy_rel_err(got, ref) < TOL
    if dbA is not None:
        db = run(xs, bpo, block, ms / 1000., weighting="A", db=True)[0]
        assert np.max(np.abs(db - dbA)) / np.max(np.abs(dbA)) < 10 * TOL


def test_cut_invariance_bit_exact():
    import torch
    from friture_b200.octavespectrum import OctaveSpectrumAnalyzer
    xd = torch.from_numpy(make_x(5, 8 * 512, seed=81)).cuda()
    for db in (False, True):
        one = OctaveSpectrumAnalyzer(5, weighting="C").process(xd, block=512, db=db)
        an = OctaveSpectrumAnalyzer(5, weighting="C")
        parts = [an.process(xd[:, a * 512:b * 512], block=512, db=db) for a, b in ((0, 1), (1, 4), (4, 8))]
        assert torch.equal(one, torch.cat(parts, dim=1))


def test_setters_keep_or_restart_state():
    import torch
    from friture_b200 import filter_data
    from friture_b200.octavespectrum import OctaveSpectrumAnalyzer
    from oracle.live_octave import LiveOctaveSpectrumOracle
    x = make_x(2, 8 * 512, seed=5)
    xd = torch.from_numpy(x).cuda()
    # mid-stream setresponsetime: the levels and the filter state carry on, like the widget's
    an = OctaveSpectrumAnalyzer(2, response_time=1.0)
    a = an.process(xd[:, :2048]).cpu().numpy()
    an.setresponsetime(0.125)
    b = an.process(xd[:, 2048:], db=False).cpu().numpy().astype(np.float64)
    E = []
    for c in range(2):
        orc = LiveOctaveSpectrumOracle(*filter_data.fir_taps(3), response_time=1.0)
        ref = [orc.push(x[c, i * 512:(i + 1) * 512]) for i in range(4)]
        assert rel_err(a[c], np.array([r[1] for r in ref])) < TOL
        orc.set_response_time(0.125)
        E.append([orc.push(x[c, i * 512:(i + 1) * 512])[0] for i in range(4, 8)])
    assert energy_rel_err(b, np.array(E)) < TOL
    # setweighting keeps the state: only the dB offset changes
    an.setweighting("A")
    fresh = OctaveSpectrumAnalyzer(2, response_time=1.0)
    fresh.process(xd[:, :2048])
    fresh.setresponsetime(0.125)
    fresh.process(xd[:, 2048:])
    fresh.setweighting("A")
    assert torch.equal(an.process(xd[:, :1024]), fresh.process(xd[:, :1024]))
    # setbandsperoctave and reset restart from zero: equal to a new analyzer, bit for bit
    ref12 = OctaveSpectrumAnalyzer(2, bandsperoctave=12, response_time=0.125, weighting="A").process(xd)
    an.setbandsperoctave(12)
    assert torch.equal(an.process(xd), ref12)
    an.reset()
    assert torch.equal(an.process(xd), ref12)


def test_silence_is_exactly_minus_300_db():
    import torch
    from friture_b200.octavespectrum import OctaveSpectrumAnalyzer
    z = torch.zeros((3, 4 * 512), dtype=torch.float32, device="cuda")
    assert bool((OctaveSpectrumAnalyzer(3).process(z) == -300.0).all())
    an = OctaveSpectrumAnalyzer(3, bandsperoctave=6, weighting="B")
    want = (np.float64(-300.0) + an._w.astype(np.float64)).astype(np.float32)
    got = an.process(z).cpu().numpy()
    assert np.array_equal(got, np.broadcast_to(want, got.shape))
    assert bool((an.process(z, db=False) == 0.0).all())


def test_levels_before_smoothing_is_a_state_error():
    import torch
    from friture_b200 import _lib
    from friture_b200.octavefilters import Octave_Filters
    bank = Octave_Filters(3, mode="fft")
    bank._ensure_fir_plan(1)
    x = torch.zeros((1, 512), dtype=torch.float32, device="cuda")
    out = torch.empty((1, 1, 27), dtype=torch.float32, device="cuda")
    sp = _lib.current_stream_ptr(x.device)
    with pytest.raises(_lib.FrtError) as ei:
        bank.handle.call("frt_firbank_levels", _lib._ptr(x), 512, 512, 1, _lib._ptr(out), 1, sp)
    assert ei.value.code == _lib.FRT_ESTATE
    alphas = np.full(9, 0.01)
    bank.handle.call("frt_firbank_set_smoothing", _lib._ptr(alphas), None)
    for args in ((384, 1), (8192, 1), (512, 2)):      # block rule, block limit, x_stride < block*n_blocks
        with pytest.raises(ValueError):
            bank.handle.call("frt_firbank_levels", _lib._ptr(x), 512, args[0], args[1], _lib._ptr(out), 1, sp)
    bank.handle.call("frt_firbank_levels", _lib._ptr(x), 512, 512, 1, _lib._ptr(out), 1, sp)
    assert bool((out == -300.0).all())
