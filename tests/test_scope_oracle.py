"""CPU: oracle/scope.py, the NumPy restatement of the scope widget with its ring buffer, reproduces
tests/golden/scope.npz, which the unmodified reference widget and RingBuffer wrote
(oracle/make_golden_scope.py): every tick's window start, point count and the sha1 of the float64
scaled_t and scaled_y the widget holds, and the kept curves to the float32 bit; the oracle's scaled_t
is the analyzer's host scope_time.  Where the reference
tree exists, the oracle's ring is also checked against the reference RingBuffer directly."""
import hashlib
import os

import numpy as np
import pytest

from friture_b200.scope import scope_time
from oracle import ref_import
from oracle.scope import (GOLDEN_BUFFER, GOLDEN_SCHEDULE, GOLDEN_TICKS, NOT_DRAWN, AudioRing, ScopeOracle,
                          golden_growths, golden_stream)

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "scope.npz")


def digest(*arrays):
    h = hashlib.sha1()
    for a in arrays:
        if a is not None:
            h.update(np.ascontiguousarray(a, dtype=np.float64).tobytes())
    return np.frombuffer(h.digest(), dtype=np.uint8)


@pytest.fixture(scope="module")
def g():
    return np.load(GOLDEN)


@pytest.fixture(scope="module")
def oracle_run():
    """The oracle on the golden stream: starts [5, K], npts [5, K], digests [5, K, 20] and the curves
    it holds after each of the golden's curve ticks."""
    x = golden_stream()
    sched = dict(GOLDEN_SCHEDULE)
    K = GOLDEN_TICKS
    starts = np.full((5, K), NOT_DRAWN, dtype=np.int64)
    npts = np.zeros((5, K), np.int64)
    dig = np.zeros((5, K, 20), np.uint8)
    kept = {}
    ticks = set(np.load(GOLDEN)["curve_ticks"].tolist())
    for scopes, nch in (((0, 1, 2), 1), ((3, 4), 2)):
        o = ScopeOracle(len(scopes), two_channels=nch == 2)
        for k in range(K):
            if k in sched:
                o.set_timerange(sched[k])
            st = o.handle_new_data(x[list(scopes), :nch, k * GOLDEN_BUFFER:(k + 1) * GOLDEN_BUFFER])
            for j, s in enumerate(scopes):
                starts[s, k] = st[j]
                if o.y[j] is None:
                    dig[s, k] = digest()
                    continue
                t, y, y2, tr = o.y[j]
                np.testing.assert_array_equal(t, scope_time(tr))
                npts[s, k] = len(y)
                dig[s, k] = digest(t, y, y2)
                if k in ticks:
                    kept[(k, s)] = (t, np.stack([y] + ([y2] if nch == 2 else [])))
    return starts, npts, dig, kept


def test_schedule_grows_the_ring_both_ways():
    """The golden schedule grows the ring once where the window reads moved samples as well as zeros
    past the kept samples, and once where it reads only zeros; it crosses 500 ms both ways."""
    grow = golden_growths()
    assert any(z > 0 and m > 0 for *_, z, m in grow)
    assert any(z > 0 and m == 0 for *_, z, m in grow)
    ranges = [v for _, v in GOLDEN_SCHEDULE]
    assert any(a <= 500 < b for a, b in zip(ranges, ranges[1:]))
    assert any(a > 500 >= b for a, b in zip(ranges, ranges[1:]))


def test_window_starts(g, oracle_run):
    np.testing.assert_array_equal(oracle_run[0], g["start"])
    # scopes that found no trigger on some ticks, and scopes that drew on others
    assert (g["start"] == NOT_DRAWN).any() and (g["start"] != NOT_DRAWN).any()


def test_curves_bit_for_bit(g, oracle_run):
    _, npts, dig, kept = oracle_run
    np.testing.assert_array_equal(npts, g["npts"])
    np.testing.assert_array_equal(dig, g["digest"])
    for (k, s), (t, y) in kept.items():
        np.testing.assert_array_equal(y.astype(np.float32), g["y_%d_%d" % (k, s)])
    assert set(kept) == {tuple(int(v) for v in n[2:].split("_")) for n in g.files if n.startswith("y_")}


@pytest.mark.skipif(not ref_import.available(), reason="reference tree not present")
def test_ring_against_reference_ringbuffer():
    """AudioRing reads what the reference RingBuffer reads, through growths with and without moved
    samples; the example of the widget's growth: at offset 20992, data(12000) is 8000 zeros and 3008
    moved samples, and stream position 8992 holds sample 16992."""
    from oracle.scope import reference_scope
    _, ringbuffer = reference_scope()
    ref = ringbuffer.RingBuffer()
    ours = AudioRing(1)
    x = np.arange(1, 200_001, dtype=np.float64)[None, :]
    pos = 0
    for n, ask in ((20992, 12000), (9000, 9000), (30000, 40000), (512, 61000), (70000, 5000)):
        for p in range(pos, pos + n, 512):                # the widget's buffers, one push each
            ref.push(x[:, p:min(p + 512, pos + n)], 0.)
            ours.push_block(x[:, p:min(p + 512, pos + n)])
        pos += n
        want = np.array(ref.data(ask))
        got = ours.data(ask)
        np.testing.assert_array_equal(got, want)
        if pos == 20992:
            zeros = (got[0] == 0).sum()
            moved = got[0] - (pos - ask + np.arange(ask) + 1)
            assert zeros == 8000 and (moved[:3008] == 8000).all()
            assert got[0, 8992 - (pos - ask)] == 16992 + 1       # x holds position p at value p + 1
