"""ctypes binding of ``libfrt_b200.so`` (the C ABI declared in ``include/frt.h``)."""
from __future__ import annotations

import contextlib
import ctypes
import os
import threading
from ctypes import (POINTER, c_char_p, c_double, c_float, c_int, c_int64, c_size_t, c_void_p)

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_NAME = "libfrt_b200.so"

FRT_OK = 0
FRT_EINVAL = -1
FRT_ECUDA = -2
FRT_ENOMEM = -3
FRT_ESTATE = -4

STFT_POWER = 0
STFT_LOGPOWER = 1


class FrtError(RuntimeError):
    """Raised for every non-zero return code of the C ABI (bad argument -> ValueError subclass)."""

    def __init__(self, code, message):
        super().__init__("frt error %d: %s" % (code, message))
        self.code = code


class FrtValueError(FrtError, ValueError):
    pass


def lib_path() -> str:
    # FRT_B200_LIB: tuning knob to A/B another build of the same library
    return os.environ.get("FRT_B200_LIB") or os.path.join(_HERE, _LIB_NAME)


# every exported symbol with (restype, argtypes); tests check that the built library exports
# exactly the functions declared in include/frt.h
_f32p = POINTER(c_float)
SIGNATURES = {
    "frt_version": (c_int, []),
    "frt_create": (c_int, [c_int, POINTER(c_void_p)]),
    "frt_destroy": (c_int, [c_void_p]),
    "frt_last_error": (c_char_p, [c_void_p]),
    "frt_device_sm_count": (c_int, [c_void_p]),
    "frt_launch_count": (c_int64, [c_void_p]),
    "frt_host_alloc": (c_int, [c_void_p, c_size_t, POINTER(c_void_p)]),
    "frt_host_free": (c_int, [c_void_p, c_void_p]),
    "frt_peer_alloc": (c_int, [c_void_p, c_size_t, POINTER(c_void_p)]),
    "frt_peer_free": (c_int, [c_void_p, c_void_p]),
    "frt_peer_export": (c_int, [c_void_p, c_void_p, c_void_p]),
    "frt_peer_import": (c_int, [c_void_p, c_void_p, POINTER(c_void_p)]),
    "frt_peer_close": (c_int, [c_void_p, c_void_p]),
    "frt_peer_copy": (c_int, [c_void_p, c_void_p, c_void_p, c_size_t, c_void_p]),
    "frt_peer_push": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_size_t, c_int, c_void_p]),
    "frt_stft_plan": (c_int, [c_void_p, c_int]),
    "frt_stft_window": (c_int, [c_void_p, c_void_p]),
    "frt_stft_process": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int64, c_int, c_void_p,
                                 c_int64, c_int64, c_int, c_void_p]),
    "frt_stft_process_host": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int64, c_int,
                                      c_void_p, c_int]),
    "frt_bank_plan": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "frt_bank_reset": (c_int, [c_void_p]),
    "frt_bank_set_weighting": (c_int, [c_void_p, c_void_p]),
    "frt_bank_schedule": (c_int, [c_int, c_int, c_int64, c_void_p, c_void_p]),
    "frt_bank_process": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int, c_void_p, c_void_p,
                                 c_int64, c_int, c_void_p]),
    "frt_bank_process_strided": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int, c_void_p, c_int64,
                                         c_int, c_void_p]),
    "frt_combined_process_host": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int64, c_int, c_void_p,
                                          c_void_p, c_int, c_int]),
    "frt_bank_state_size": (c_int, [c_void_p, POINTER(c_int64), POINTER(c_int64)]),
    "frt_bank_get_state": (c_int, [c_void_p, c_void_p, c_void_p]),
    "frt_bank_set_state": (c_int, [c_void_p, c_void_p, c_void_p]),
    "frt_firbank_plan": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "frt_firbank_reset": (c_int, [c_void_p]),
    "frt_firbank_process": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_void_p, c_int64, c_void_p]),
    "frt_firbank_set_smoothing": (c_int, [c_void_p, c_void_p, c_void_p]),
    "frt_firbank_levels": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int, c_void_p, c_int, c_void_p]),
    "frt_gcc_plan": (c_int, [c_void_p, c_int]),
    "frt_gcc_phat": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_void_p, c_void_p, c_int,
                             c_void_p, c_void_p, c_void_p]),
    "frt_gcc_fits": (c_int, [c_int]),
    "frt_gcc_set_pairs": (c_int, [c_void_p, c_int, c_void_p, c_int]),
    "frt_gcc_phat_pairs": (c_int, [c_void_p, c_void_p, c_int64, c_void_p, c_void_p, c_int, c_void_p,
                                   c_void_p, c_void_p]),
    "frt_gcc_phat_frames": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int, c_int, c_void_p,
                                    c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "frt_gcc_phat_pairs_frames": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_int, c_void_p, c_int,
                                          c_void_p, c_void_p, c_void_p, c_void_p]),
    "frt_spectrum_reduce": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_int, c_int, c_int,
                                    c_float, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                    c_void_p]),
    "frt_spectrum_reduce_dual": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int, c_int,
                                         c_int, c_float, c_void_p, c_void_p, c_void_p, c_void_p,
                                         c_void_p, c_void_p]),
    "frt_spectrum_reduce_ticks": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_int, c_int, c_int,
                                          c_int, c_float, c_void_p, c_void_p, c_void_p, c_void_p,
                                          c_void_p, c_void_p]),
    "frt_spectrum_reduce_dual_ticks": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int,
                                               c_int, c_int, c_int, c_float, c_void_p, c_void_p,
                                               c_void_p, c_void_p, c_void_p, c_void_p]),
    "frt_spectrum_frames": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int64, c_int, c_void_p, c_int,
                                    c_float, c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_void_p,
                                    c_void_p, c_void_p]),
    "frt_spectrum_frames_dual": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int64, c_int,
                                         c_void_p, c_int, c_float, c_void_p, c_void_p, c_void_p, c_int64,
                                         c_int64, c_void_p, c_void_p, c_void_p]),
    "frt_plot_curves": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_int, c_int, c_int, c_double,
                                c_double, c_double, c_int, c_int, c_void_p, c_void_p, c_void_p,
                                c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "frt_decimate_plan": (c_int, [c_void_p, c_int, c_int, c_void_p]),
    "frt_decimate_process": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_void_p, c_int64, c_void_p]),
    "frt_display_columns": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_int, c_int, c_int,
                                    c_void_p, c_float, c_float, c_void_p, c_void_p, c_int, c_void_p,
                                    c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "frt_stft_screen_rows": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int64, c_int, c_void_p, c_float,
                                     c_float, c_void_p, c_void_p, c_int, c_void_p, c_int64, c_int64, c_void_p]),
    "frt_display_rows": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_int, c_int, c_int, c_void_p, c_void_p,
                                 c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "frt_levels_plan": (c_int, [c_void_p, c_int, c_int, c_void_p, c_double, c_double, c_double]),
    "frt_levels_reset": (c_int, [c_void_p]),
    "frt_levels_state": (c_int, [c_void_p, c_void_p, c_void_p]),
    "frt_levels_process": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_void_p, c_void_p, c_void_p,
                                   c_void_p]),
    "frt_longlevels_plan": (c_int, [c_void_p, c_int, c_int, c_void_p, c_void_p]),
    "frt_longlevels_reset": (c_int, [c_void_p]),
    "frt_longlevels_process": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_void_p, c_void_p, c_void_p,
                                       c_int64, c_int64, c_void_p]),
    "frt_longlevels_history": (c_int, [c_void_p, c_void_p, c_int64, c_int64, c_int, c_int, c_double,
                                       c_double, c_void_p, c_void_p]),
    "frt_scope_process": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int, c_int64, c_int, c_int, c_int,
                                  c_int, c_int64, c_void_p, c_void_p, c_int64, c_double, c_void_p, c_void_p]),
}

_lib = None
_lib_lock = threading.Lock()


def load_library():
    """Load ``libfrt_b200.so`` (built in-tree by ``__graft_entry__.build()`` /
    ``make -C friture_b200/csrc``).  Raises if it is missing -- there is no fallback path."""
    global _lib
    with _lib_lock:
        if _lib is not None:
            return _lib
        path = lib_path()
        if not os.path.isfile(path):
            raise FrtError(FRT_ESTATE, "%s not built; run `python -c 'import __graft_entry__ as g; "
                           "g.build()'` or `make -C friture_b200/csrc` (no CPU fallback exists)"
                           % path)
        lib = ctypes.CDLL(path, mode=ctypes.RTLD_GLOBAL)
        for name, (restype, argtypes) in SIGNATURES.items():
            fn = getattr(lib, name)
            fn.restype = restype
            fn.argtypes = argtypes
        _lib = lib
        return lib


def _ptr(obj):
    """Raw pointer of a torch tensor / numpy array / int / None."""
    if obj is None:
        return None
    if isinstance(obj, int):
        return c_void_p(obj)
    if hasattr(obj, "data_ptr"):
        return c_void_p(obj.data_ptr())
    if hasattr(obj, "ctypes"):
        return c_void_p(obj.ctypes.data)
    raise TypeError("cannot take a pointer of %r" % type(obj))


class Handle:
    """Owns one ``frt_handle`` (one GPU).  Not re-entrant: one handle <-> one stream at a time,
    like the reference's widgets, which call the hot path from a single thread
    (friture/analyzer.py:193-195)."""

    def __init__(self, device: int = 0):
        self._lib = load_library()
        self._h = c_void_p()
        rc = self._lib.frt_create(int(device), ctypes.byref(self._h))
        if rc != FRT_OK:
            msg = self._lib.frt_last_error(None)
            raise FrtError(rc, msg.decode() if msg else "frt_create failed")
        self.device = int(device)

    def check(self, rc):
        if rc == FRT_OK:
            return
        msg = self._lib.frt_last_error(self._h)
        msg = msg.decode() if msg else "?"
        if rc == FRT_EINVAL:
            raise FrtValueError(rc, msg)
        raise FrtError(rc, msg)

    def check_device(self, tensor):
        """A tensor on another GPU than the handle's would surface as an illegal-address error
        deep inside a kernel; say it plainly instead."""
        idx = getattr(getattr(tensor, "device", None), "index", None)
        if idx is not None and idx != self.device:
            raise FrtValueError(FRT_EINVAL, "tensor lives on cuda:%d, this handle is bound to cuda:%d"
                                % (idx, self.device))

    def call(self, name, *args):
        self.check(getattr(self._lib, name)(self._h, *args))

    @property
    def launch_count(self) -> int:
        return int(self._lib.frt_launch_count(self._h))

    @property
    def sm_count(self) -> int:
        return int(self._lib.frt_device_sm_count(self._h))

    def close(self):
        if getattr(self, "_h", None) is not None and self._h:
            self._lib.frt_destroy(self._h)
            self._h = c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def device_index(device=None) -> int:
    """Index of the CUDA device named by None (the current one), an int or a torch.device."""
    import torch
    if not torch.cuda.is_available():
        raise FrtError(FRT_ECUDA, "no CUDA device available; friture_b200 has no CPU fallback")
    if isinstance(device, torch.device):
        device = device.index
    return torch.cuda.current_device() if device is None else int(device)


_default_handles = {}


def default_handle(device=None) -> Handle:
    """Process-wide handle per device (the drop-in classes share it, as the reference's widgets
    share one process)."""
    device = device_index(device)
    h = _default_handles.get(device)
    if h is None:
        h = Handle(device)
        _default_handles[device] = h
    return h


def lazy_handle(make):
    """A ``handle`` property that sets ``self._handle = make(self)`` on first use, so that an object
    can be built and configured without a GPU."""
    def get(self):
        if self._handle is None:
            self._handle = make(self)
        return self._handle
    return property(get)


# the ``handle`` of the classes that share the process-wide handle of the current device
shared_handle = lazy_handle(lambda self: default_handle())


def current_stream_ptr(device=None):
    import torch
    return c_void_p(torch.cuda.current_stream(device).cuda_stream)


@contextlib.contextmanager
def call_stream(device, stream=None):
    """The stream a call runs on: the caller's ``stream`` (a CUDA stream handle as an int), else the
    current torch stream of ``device``.  It is the current stream for the body, so that the
    wrapper's own torch work -- allocations, fills, uploads, copies and host reads -- is ordered
    with the library's kernels on it, and the temporaries it frees go back to that stream's pool.
    Yields the handle to pass to the library."""
    if stream is None:
        yield current_stream_ptr(device)
        return
    import torch
    with torch.cuda.stream(torch.cuda.ExternalStream(int(stream), device=device)):
        yield c_void_p(int(stream))


def _row_stride(shape, stride0):
    # a length-1 axis may carry any stride: the library is told T for a one-row array
    C, T = shape
    return int(stride0) if C > 1 else int(T)


def check_tensor(owner, x, name):
    """Raise ValueError unless ``x`` is a CUDA float32 tensor on the GPU of ``owner.handle``.  The
    handle is looked up last, so that a host array or CPU tensor is rejected without a GPU and
    without creating a handle."""
    import torch
    if not isinstance(x, torch.Tensor) or x.dtype != torch.float32 or not x.is_cuda:
        raise ValueError("%s must be a CUDA float32 tensor" % name)
    owner.handle.check_device(x)


def device_rows(owner, x, name):
    """``x`` as [C, T] (a 1-D tensor is one row) and the row stride to pass for it, once it is
    checked to be a CUDA float32 tensor on the GPU of ``owner.handle``, contiguous along time."""
    check_tensor(owner, x, name)
    if x.dim() == 1:
        x = x[None, :]
    if x.dim() != 2 or (x.shape[1] > 0 and x.stride(1) != 1):
        raise ValueError("%s must be [C, T], contiguous along time" % name)
    return x, _row_stride(x.shape, x.stride(0))


def _host_float32(x):
    """True for a float32 NumPy array or CPU torch tensor."""
    import numpy as np
    if isinstance(x, np.ndarray):
        return x.dtype == np.float32
    import torch
    return isinstance(x, torch.Tensor) and x.dtype == torch.float32 and x.device.type == "cpu"

def _elem_strides(x):
    return tuple(x.stride()) if hasattr(x, "data_ptr") else tuple(s // 4 for s in x.strides)


def host_rows(x, name="x"):
    """Host twin of ``device_rows``: ``x`` as [C, T] and its row stride in floats, once it is checked
    to be a float32 NumPy array or CPU tensor [C, T] or [T], contiguous along time.  The library
    reads it at that stride as float32, so any other layout would be read as different samples."""
    if not _host_float32(x):
        raise ValueError("%s must be a float32 NumPy array or CPU tensor" % name)
    if x.ndim == 1:
        x = x[None, :]
    if x.ndim != 2:
        raise ValueError("%s must be [C, T], contiguous along time" % name)
    if not hasattr(x, "data_ptr") and any(s % 4 for s in x.strides):
        raise ValueError("%s must be [C, T], contiguous along time" % name)
    s0, s1 = _elem_strides(x)
    if (x.shape[1] > 1 and s1 != 1) or (x.shape[0] > 1 and s0 < x.shape[1]):
        raise ValueError("%s must be [C, T], contiguous along time" % name)
    return x, _row_stride(x.shape, s0)


def check_host_out(out, shape, name):
    """Raise ValueError unless ``out`` is a C-contiguous float32 NumPy array or CPU tensor of exactly
    ``shape``: the library writes it densely at the pitch that shape implies."""
    if (not _host_float32(out) or tuple(out.shape) != tuple(shape)
            or not (out.is_contiguous() if hasattr(out, "data_ptr") else out.flags.c_contiguous)):
        raise ValueError("%s must be a contiguous float32 NumPy array or CPU tensor of shape %s"
                         % (name, tuple(shape)))
