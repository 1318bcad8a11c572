"""friture_b200 -- H100-native (sm_90a) implementation of Friture's per-chunk spectral hot path.

Host side: Python mirrors of the reference's call surface (``audioproc``, ``Octave_Filters``,
``generalized_cross_correlation`` ...) over a ctypes C ABI (``include/frt.h``) into hand-written
CUDA kernels.  There is no CPU fallback: importing the classes works anywhere (so that host
logic can be unit-tested), but creating a handle without ``libfrt_b200.so`` or without a CUDA
device raises.
"""
from ._lib import FrtError, Handle, lib_path, load_library  # noqa: F401
from .audioproc import audioproc, AudioProc, SAMPLING_RATE, FRAMES_PER_BUFFER  # noqa: F401
from .octavefilters import Octave_Filters, OctaveFilters  # noqa: F401
from .correlation import generalized_cross_correlation, GccPhat, PairGccPhat  # noqa: F401
from .analyzer import ChannelAnalyzer  # noqa: F401

__all__ = ["FrtError", "Handle", "lib_path", "load_library", "audioproc", "AudioProc",
           "Octave_Filters", "OctaveFilters", "generalized_cross_correlation", "GccPhat", "PairGccPhat",
           "ChannelAnalyzer", "SAMPLING_RATE", "FRAMES_PER_BUFFER"]
