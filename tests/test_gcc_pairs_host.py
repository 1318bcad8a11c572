"""CPU: PairGccPhat's argument checks, and the pair table it keeps in sync on a shared handle (the
library holds one table per handle, so an estimator sets its own again when another has replaced
it)."""
import numpy as np
import pytest

from friture_b200.correlation import PairGccPhat


class RecordingHandle:
    """Stands in for a Handle: records the calls instead of making them."""

    def __init__(self):
        self.calls = []

    def call(self, name, *args):
        self.calls.append((name, args))


@pytest.mark.parametrize("pairs", [
    [(0, 4)],                     # past the last channel
    [(0, 1), (-1, 2)],            # negative
    [(0, 1, 2)],                  # not pairs
    [0, 1],                       # flat
    [(0.0, 1.0)],                 # not integers
])
def test_bad_pairs_are_refused(pairs):
    with pytest.raises(ValueError):
        PairGccPhat(2400, 4, pairs)


def test_bad_channel_count_is_refused():
    with pytest.raises(ValueError):
        PairGccPhat(2400, 0, [])


def test_table_layout():
    est = PairGccPhat(2400, 3, [(2, 0), (1, 1), (0, 2), (0, 2)], handle=RecordingHandle())
    assert est.n_pairs == 4 and est.pairs.dtype == np.int32 and est.pairs.flags.c_contiguous
    assert est.pairs.tolist() == [[2, 0], [1, 1], [0, 2], [0, 2]]
    assert PairGccPhat(2400, 3, [], handle=RecordingHandle()).pairs.shape == (0, 2)


def test_cpu_tensor_is_refused_without_a_handle():
    import torch
    est = PairGccPhat(2400, 2, [(0, 1)])
    with pytest.raises(ValueError):
        est.estimate(torch.zeros(2, 2400))
    assert est._handle is None


def test_table_is_set_again_after_another_estimator_set_its_own():
    h = RecordingHandle()
    a = PairGccPhat(2400, 4, [(0, 1), (2, 3)], handle=h)
    b = PairGccPhat(2400, 4, [(3, 0)], handle=h)
    tables = lambda: [(args[0], args[2]) for name, args in h.calls if name == "frt_gcc_set_pairs"]
    a._sync_table()
    a._sync_table()
    assert tables() == [(4, 2)]            # set once while it stays on the handle
    b._sync_table()
    assert tables() == [(4, 2), (4, 1)]
    a._sync_table()
    a._sync_table()
    assert tables() == [(4, 2), (4, 1), (4, 2)]
    other = RecordingHandle()              # a table on another handle does not count
    c = PairGccPhat(2400, 4, [(1, 2)], handle=other)
    c._sync_table()
    b._sync_table()
    assert tables() == [(4, 2), (4, 1), (4, 2), (4, 1)] and len(other.calls) == 1
