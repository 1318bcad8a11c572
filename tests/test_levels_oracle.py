"""CPU: oracle/levels.py, the NumPy restatement of the levels and long-term levels widgets, reproduces
tests/golden/levels.npz, which the unmodified reference widgets wrote (oracle/make_golden_levels.py).
The meter's peak state, hold counters and decay factors and the long-term linear levels are the same
bits; the meter's RMS (NumPy's dot product order) and IEC peak to 1e-13 relative, dB to 1e-11."""
import os

import numpy as np
import pytest

from oracle.levels import (GOLDEN_METER_BUFFERS, LevelsOracle, LongLevelsOracle, golden_schedule,
                           golden_stream)

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "levels.npz")


@pytest.fixture(scope="module")
def g():
    return np.load(GOLDEN)


@pytest.fixture(scope="module")
def x():
    return golden_stream()


def test_meter(g, x):
    o = LevelsOracle(2)
    keys = ("rms", "max", "iec", "old_rms", "old_max", "decay", "hold")
    got = {k: np.zeros((2, GOLDEN_METER_BUFFERS)) for k in keys}
    for b in range(GOLDEN_METER_BUFFERS):
        rms, mx, iec = o.handle_new_data(x[:, b * 512:(b + 1) * 512])
        s = o.state()
        for k, v in zip(keys, (rms, mx, iec, s["old_rms"], s["old_max"], s["decay"], s["hold"])):
            got[k][:, b] = v
    for k in ("old_max", "decay", "hold"):
        np.testing.assert_array_equal(got[k], g["m_" + k], err_msg=k)
    # the IEC peak follows level_rms where RMS is the larger level, so it carries the dot product's rounding
    np.testing.assert_allclose(got["iec"], g["m_iec"], rtol=1e-13, atol=0)
    np.testing.assert_allclose(got["old_rms"], g["m_old_rms"], rtol=1e-13, atol=0)
    np.testing.assert_allclose(got["rms"], g["m_rms"], rtol=1e-11, atol=0)
    np.testing.assert_allclose(got["max"], g["m_max"], rtol=1e-11, atol=0)
    # the stream reaches every phase of the ballistic peak: rise, hold and decay
    assert (np.diff(g["m_iec"], axis=1) < 0).any() and (g["m_hold"] == 32).any()


def test_long_levels(g, x):
    o = LongLevelsOracle(2)
    ends, levels, dbs, curves = [], [], [], {}
    pos = call = 0
    calls = set(g["l_curve_call"].tolist())
    for ev in golden_schedule():
        if isinstance(ev, tuple):
            getattr(o, ev[0])(ev[1])
            continue
        e, lv, db = o.handle_new_data(x[:, pos:pos + ev])
        pos += ev
        ends.append(e)
        levels.append(lv)
        dbs.append(db)
        if call in calls:
            curves[call] = o.curve
        call += 1
    np.testing.assert_array_equal(np.concatenate(ends), g["l_end"])
    np.testing.assert_array_equal(np.concatenate(levels, axis=1), g["l_level"])
    np.testing.assert_allclose(np.concatenate(dbs, axis=1), g["l_db"], rtol=1e-12, atol=0)
    assert g["l_end"][0] == 0 and len(g["l_end"]) > 10000     # the zero block, and a wrapped ring
    for call in calls:
        t, y = curves[call]
        np.testing.assert_array_equal(t, g["l_t_%d" % call])
        np.testing.assert_allclose(y, g["l_curve_%d" % call], rtol=0, atol=1e-12)
