"""Throughput of the filterbank kernels on the GPU box (tuning aid, not the bench):
python tools/perf_bank.py [channels ...]   (FRT_B200_LIB selects another build of the library)"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from friture_b200.octavefilters import Octave_Filters  # noqa: E402


def run(C, block, nblk, noct, reps=5):
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


if __name__ == "__main__":
    chans = [int(v) for v in sys.argv[1:]] or [1024, 2048, 8192]
    print("library:", os.environ.get("FRT_B200_LIB", "default"))
    for C in chans:
        for block, noct in ((512, 9), (1024, 10)):
            nblk = 256 if block == 512 else 128
            row = []
            for kern, pack, logch in (("pipe", 1, 5), ("pipe", 2, 5), ("pipe", 1, 6), ("pipe", 2, 6)):
                os.environ["FRT_BANK_KERNEL"] = kern
                os.environ["FRT_BANK_PACK"] = str(pack)
                os.environ["FRT_BANK_LOGCH"] = str(logch)
                r, ms = run(C, block, nblk, noct)
                row.append("p%d/c%d %.3g (%.2f ms)" % (pack, 1 << logch, r, ms))
            print("C=%d block=%d noct=%d nblk=%d: %s" % (C, block, noct, nblk, " | ".join(row)), flush=True)
