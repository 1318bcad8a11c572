"""CPU: the scope analyzer's host arithmetic (window width, trigger level and scaled_t, as
friture/scope.py:79-127 computes them), its ring model (push, read and growth, run on CPU tensors)
against the NumPy ring of oracle/scope.py and the reference RingBuffer, and its refusals, which come
with ValueError before any device work (no handle is created) and leave the state unchanged."""
import numpy as np
import pytest
import torch

from friture_b200.scope import (ScopeAnalyzer, is_trigger, scope_points, scope_time, scope_width,
                                trigger_level)
from oracle import ref_import
from oracle.scope import AudioRing, golden_growths

# timerange (ms) -> (width, trigger mode, points)
CASES = {0.1: (4, True, 4), 0.3: (14, True, 14), 123.4: (5923, True, 5922), 500: (24000, True, 24000),
         500.1: (24004, False, 24004), 10000: (480000, False, 480000)}


@pytest.mark.parametrize("tr", sorted(CASES))
def test_width_and_points(tr):
    w, trig, n = CASES[tr]
    assert scope_width(tr) == w == int(tr * 1e-3 * 48000)
    assert is_trigger(tr) == trig and scope_points(tr) == n


@pytest.mark.parametrize("tr", sorted(CASES))
def test_scaled_t(tr):
    w = scope_width(tr)
    n = scope_points(tr)
    want = ((np.arange(n) - w // 2) / 48000. * 1e3 + tr / 2.) / tr
    np.testing.assert_array_equal(scope_time(tr), want)
    # the search window d[w//2 : -w//2] of the 2w samples holds exactly w samples, odd widths too
    if is_trigger(tr):
        assert len(np.arange(2 * w)[w // 2: -w // 2]) == w


def test_trigger_level():
    assert trigger_level(np.float32([0.1, 0.75, -1])) == 0.5
    assert trigger_level(np.float32([0.3, 0.2])) == np.float64(np.float32(0.3)) * 2. / 3.
    assert np.isnan(trigger_level(np.float32([0.3, np.nan, 0.2])))
    assert trigger_level(np.float32([-np.inf, -np.inf])) == -np.inf
    assert trigger_level(np.float32([0.1, np.inf])) == np.inf


def ring_run(a, o, pushes, ref=None):
    """Push the same samples into the analyzer's ring model (CPU tensors) as one chunk, and into
    AudioRing and optionally the reference RingBuffer 512 samples at a time, as the widget's buffers
    arrive; after each chunk read `ask` samples from all of them."""
    x = np.arange(1, 1 + sum(n for n, _ in pushes), dtype=np.float64)[None, :].repeat(2, 0)
    x[1] *= -1
    pos = 0
    for n, ask in pushes:
        a._push(torch.from_numpy(x[:, pos:pos + n].astype(np.float32)))
        for p in range(pos, pos + n, 512):
            piece = x[:, p:min(p + 512, pos + n)]
            o.push_block(piece)
            if ref is not None:
                ref.push(piece, 0.)
        pos += n
        a._ring, a._ring_len = grow_ring_of(a, ask)
        got = torch.cat(a._read(ask), dim=1).numpy()
        want = o.data(ask)
        np.testing.assert_array_equal(got, want)
        if ref is not None:
            np.testing.assert_array_equal(got, ref.data(ask))
        assert a._ring_len == o.buf.shape[1]


def grow_ring_of(a, length):
    from friture_b200.levels import grow_ring
    return grow_ring(a._ring, a._offset, length)


def fresh(n_rows=2):
    a = ScopeAnalyzer(1, two_channels=n_rows == 2)
    a._ring = torch.zeros(n_rows, a._ring_len)
    return a


def test_ring_model_golden_growths():
    """The golden schedule's growths (each tick one 512-sample push): with zeros and moved samples,
    and with zeros only."""
    a, o = fresh(), AudioRing(2)
    pushes, last = [], 0
    for k, off, old, new, need, zeros, moved in golden_growths():
        pushes += [(512, 100)] * (k - last) + [(512, need)]
        last = k + 1
    ring_run(a, o, pushes)
    assert a._ring_len == golden_growths()[-1][3]


def test_ring_model_moved_samples():
    """At offset 20992, data(12000) grows the 10000-sample ring to 18000: 8000 zeros and 3008 samples
    moved by 8000 positions; stream position 8992 holds sample 16992."""
    a, o = fresh(), AudioRing(2)
    ring_run(a, o, [(512, 512)] * 41)
    a._push(torch.from_numpy(np.zeros((2, 0), np.float32)))
    a._ring, a._ring_len = grow_ring_of(a, 12000)
    got = torch.cat(a._read(12000), dim=1).numpy()[0]
    pos = np.arange(20992 - 12000, 20992)
    assert (got == 0).sum() == 8000
    assert got[0] == 16992 + 1 and (got[:3008] == pos[:3008] + 8000 + 1).all()
    assert (got[-992:] == pos[-992:] + 1).all()


@pytest.mark.skipif(not ref_import.available(), reason="reference tree not present")
def test_ring_model_against_reference():
    from oracle.scope import reference_scope
    _, ringbuffer = reference_scope()
    pushes = [(20992, 12000), (512, 12000), (9000, 9000), (30000, 40000), (512, 61000), (4096, 100),
              (70000, 5000), (1, 91000), (17, 3)]
    ring_run(fresh(), AudioRing(2), pushes, ref=ringbuffer.RingBuffer())


# ---------------------------------------------------------------- refusals
@pytest.mark.parametrize("n", [0, -2])
def test_scope_count_refused(n):
    with pytest.raises(ValueError):
        ScopeAnalyzer(n)


@pytest.mark.parametrize("tr", [0.0, 0.05, 10000.5, -1, float("nan")])
def test_timerange_refused(tr):
    with pytest.raises(ValueError):
        ScopeAnalyzer(1, timerange=tr)
    a = ScopeAnalyzer(1, timerange=123.4)
    with pytest.raises(ValueError):
        a.set_timerange(tr)
    assert a.timerange == 123.4


@pytest.mark.parametrize("two,make", [
    (False, lambda: torch.zeros(3, 1024)), (False, lambda: torch.zeros(1024)),
    (False, lambda: torch.zeros(2, 2, 512)), (False, lambda: np.zeros((2, 1024), np.float32)),
    (True, lambda: torch.zeros(2, 1024)), (True, lambda: torch.zeros(2, 3, 512)),
    (True, lambda: torch.zeros(3, 2, 512)), (False, lambda: torch.zeros(2, 1024)),
    (True, lambda: torch.zeros(2, 2, 1024)), (False, lambda: torch.zeros(1024, 2).t()),
])
def test_bad_chunks_refused(two, make):
    a = ScopeAnalyzer(2, two_channels=two)
    with pytest.raises(ValueError):
        a.handle_new_data(make())          # CPU tensors: refused as not CUDA, after the layout checks
    assert a._handle is None and a._ring is None and a._offset == 0


@pytest.mark.parametrize("n,buffer", [(500, 512), (1000, 512), (1024, 1000), (512, 0), (20002, 10001)])
def test_bad_buffers_refused(n, buffer):
    a = ScopeAnalyzer(1)
    with pytest.raises(ValueError):
        a.handle_new_data(torch.zeros(1, n), buffer=buffer)
    assert a._handle is None and a._ring is None and a._offset == 0


def test_curve_before_any_tick():
    c = ScopeAnalyzer(3).curve()
    assert c.scaled_y is None and c.scaled_y2 is None and c.timerange is None
