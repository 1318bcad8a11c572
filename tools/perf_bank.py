"""Throughput of the filterbank kernels on the GPU box (tuning aid, not the bench):
python tools/perf_bank.py [channels ...]   (FRT_B200_LIB selects another build of the library)
Prints, per shape, the kernel the library picks and its channel-blocks per second."""
import os
import re
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

from friture_b200.octavefilters import Octave_Filters  # noqa: E402


def run(C, block, nblk, noct=9, reps=5):
    x = (torch.randn((C, block * nblk), dtype=torch.float32, device="cuda") * 0.1)
    bank = Octave_Filters(3, n_octaves=noct)
    bank.energies_batch(x, block=block, db=True)
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        bank.energies_batch(x, block=block, db=True)
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / reps
    return C * nblk / (ms * 1e-3), ms


def kernel_name(C, block, noct):
    """The filterbank kernel one call at this shape launches (in a profiled run of its own)."""
    x = torch.zeros((C, block), dtype=torch.float32, device="cuda")
    bank = Octave_Filters(3, n_octaves=noct)
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        bank.energies_batch(x, block=block, db=True)
        torch.cuda.synchronize()
    names = [re.search(r"bank\w*<[^>]*>", e.name) for e in prof.events()]
    return ", ".join(m.group(0) for m in names if m)


if __name__ == "__main__":
    chans = [int(v) for v in sys.argv[1:]] or [1024, 2048, 8192]
    print("library:", os.environ.get("FRT_B200_LIB", "default"))
    for C in chans:
        for block, noct in ((256, 9), (512, 9), (1024, 10)):
            nblk = 131072 // block
            r, ms = run(C, block, nblk, noct)
            print("C=%d block=%d noct=%d nblk=%d: %s %.3g (%.2f ms)"
                  % (C, block, noct, nblk, kernel_name(C, block, noct), r, ms), flush=True)
