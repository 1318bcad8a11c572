"""CPU: the host classes reach the C ABI through friture_b200/_lib.py alone.  Which handle an object
uses, which stream a call runs on, what a device input must be and which row stride the library is
told are decided there once; the row helpers are checked here on host arrays and on CPU tensors
that stand in for device tensors."""
import os

import numpy as np
import pytest
import torch

from friture_b200 import _lib

PKG = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "friture_b200")

ONLY_IN_LIB = [
    "current_stream_ptr(",
    "c_void_p(int(stream))",
    "torch.cuda.ExternalStream(",   # call_stream makes the caller's stream current
    "torch.cuda.current_device()",
    "default_handle()",
    "check_device(",
    "if C > 1 else",            # the row stride of a [C, T] array
]


@pytest.mark.parametrize("text", ONLY_IN_LIB)
def test_only_in_lib(text):
    names = sorted(f for f in os.listdir(PKG) if f.endswith(".py"))
    assert "_lib.py" in names and len(names) >= 10
    src = {f: open(os.path.join(PKG, f)).read() for f in names}
    assert text in src["_lib.py"]
    elsewhere = [f for f, s in src.items() if f != "_lib.py" and text in s]
    assert not elsewhere, "%r belongs in _lib.py only, found in %s" % (text, elsewhere)


def test_host_rows():
    T = 1000
    cases = [
        (np.zeros((3, T), np.float32), 3, T),
        (np.zeros((3, 2 * T), np.float32)[:, :T], 3, 2 * T),     # padded rows
        (np.empty((T, 1), np.float32).T, 1, T),                   # strides (4, 4)
        (np.zeros(T, np.float32), 1, T),
        (torch.zeros((3, T)), 3, T),
        (torch.zeros((3, 2 * T))[:, :T], 3, 2 * T),
        (torch.empty((T, 1)).t(), 1, T),                          # strides (1, 1)
        (torch.zeros(T), 1, T),
    ]
    for x, C, stride in cases:
        rows, s = _lib.host_rows(x)
        assert tuple(rows.shape) == (C, T) and s == stride and type(s) is int


def test_host_rows_rejections():
    """The library reads host input as float32 rows at the returned stride: anything else is refused."""
    T = 1000
    bad = [
        np.zeros((3, T), np.float64),                      # read as float32 it would be other samples
        torch.zeros((3, T), dtype=torch.float64),
        np.zeros((T, 3), np.float32).T,                    # not contiguous along time
        torch.zeros((T, 3)).t(),
        np.zeros((2, 3, T), np.float32),                   # not [C, T]
        np.zeros((3, T), np.float32)[::-1],                # rows overlap / run backwards
        [[0.0] * T],                                       # not an array
    ]
    for x in bad:
        with pytest.raises(ValueError):
            _lib.host_rows(x)


def test_check_host_out():
    shape = (2, 3, 5)
    _lib.check_host_out(np.zeros(shape, np.float32), shape, "out")
    _lib.check_host_out(torch.zeros(shape), shape, "out")
    for out in (np.zeros(shape, np.float64), torch.zeros(shape, dtype=torch.float64), np.zeros((2, 4, 5), np.float32),
                np.zeros((2, 3, 6), np.float32)[..., :5], torch.zeros((2, 5, 3)).transpose(1, 2), [[0.0]]):
        with pytest.raises(ValueError):
            _lib.check_host_out(out, shape, "out")


def test_bank_block_rule():
    """ChannelAnalyzer refuses the hops the filterbank kernels refuse (bank.cu, frt_bank_check_block)."""
    from friture_b200.analyzer import bank_block_ok
    assert [b for b in range(0, 4097, 128) if bank_block_ok(b, 10)] == [512, 1024, 1536, 2048, 2560, 3072, 3584, 4096]
    assert [b for b in range(0, 2049, 128) if bank_block_ok(b, 9)] == list(range(256, 2049, 256))
    assert bank_block_ok(256, 1) and not bank_block_ok(384, 1) and not bank_block_ok(-256, 3)


class StandInHandle:
    """The handle's device check, bound to cuda:0 without a GPU."""
    device = 0
    check_device = _lib.Handle.check_device


class Owner:
    handle = StandInHandle()


def on_cuda(t, index=0):
    """A CPU tensor that reports itself on cuda:index."""
    cls = type("OnCuda%d" % index, (torch.Tensor,), {"is_cuda": True, "device": torch.device("cuda", index)})
    return t.as_subclass(cls)


def test_filter_batch_refuses_a_block_the_bank_refuses_before_any_call():
    """768 samples pass the old weaker check at 10 octaves; the bank's own rule refuses them, with the
    same message ChannelAnalyzer gives, before any plan or launch."""
    from friture_b200.octavefilters import Octave_Filters

    class NoCalls(StandInHandle):
        def call(self, *args):
            raise AssertionError("library called for a refused block: %s" % (args,))

    for mode in ("iir", "fft"):
        bank = Octave_Filters(3, n_octaves=10, handle=NoCalls(), mode=mode)
        for block in (768, 384, 256):
            with pytest.raises(ValueError, match="no %d-sample blocks at 10 octaves" % block):
                bank.filter_batch(on_cuda(torch.zeros((2, 4 * block))), block, energies=mode == "iir",
                                  want_y=mode == "fft")


def test_device_rows_accepts_and_gives_the_row_stride():
    T = 1000
    for x, C, stride in [(torch.zeros((3, T)), 3, T), (torch.zeros((3, 2 * T))[:, :T], 3, 2 * T),
                         (torch.empty((T, 1)).t(), 1, T), (torch.zeros(T), 1, T),
                         (torch.zeros((0, T)), 0, T)]:
        rows, s = _lib.device_rows(Owner(), on_cuda(x), "x")
        assert tuple(rows.shape) == (C, T) and s == stride and type(s) is int


def test_device_rows_rejections():
    T = 1000
    bad = [
        (on_cuda(torch.zeros((2, T), dtype=torch.float64)), ValueError),      # dtype
        (torch.zeros((2, T)), ValueError),                                      # not CUDA
        (np.zeros((2, T), np.float32), ValueError),                             # not a tensor
        (on_cuda(torch.zeros((2, 2, T))), ValueError),                          # not [C, T]
        (on_cuda(torch.zeros((T, 2)).t()), ValueError),                         # not contiguous along time
        (on_cuda(torch.zeros((2, T)), 1), _lib.FrtValueError),                  # another GPU
    ]
    for x, err in bad:
        with pytest.raises(err):
            _lib.device_rows(Owner(), x, "x")
    for x, err in bad[:2] + bad[-1:]:
        with pytest.raises(err):
            _lib.check_tensor(Owner(), x, "x")


def test_rejected_input_creates_no_handle():
    class NoGpu:
        @property
        def handle(self):
            raise AssertionError("handle looked up for an input rejected on its own")

    for x in (torch.zeros((2, 8)), on_cuda(torch.zeros((2, 8), dtype=torch.float64))):
        with pytest.raises(ValueError):
            _lib.device_rows(NoGpu(), x, "x")


def test_device_index_without_gpu():
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    for device in (None, 0, torch.device("cuda", 0)):
        with pytest.raises(_lib.FrtError) as ei:
            _lib.device_index(device)
        assert ei.value.code == _lib.FRT_ECUDA
