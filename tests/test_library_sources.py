"""CPU: the CUDA sources keep one copy of the launch path and of the device primitives the kernel
files share.  Every kernel launch goes through frt_launch (friture_b200/csrc/frt_internal.cuh), which
sets the dynamic shared-memory limit, checks the launch and counts it; the fast log2 and the cp.async
wrappers are defined there once.  So are frt_sync_copy and frt_sync_zero, the only synchronous copies
and fills: they drain the device before and after, so that no kernel queued on any stream sees a plan,
setter or reset that came after it, and no kernel launched next misses one that came before.  Every
device allocation goes through frt_malloc, which clears a failure from the runtime's last error so
that the next launch's check does not report it, and FRT_CUDA reports running out of memory as
FRT_ENOMEM."""
import os

import pytest

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "friture_b200", "csrc")
HOME = "frt_internal.cuh"

ONLY_IN_HOME = [
    "<<<",                      # kernel launches
    "cudaFuncSetAttribute",     # the dynamic shared-memory limit
    "launches++",               # frt_launch_count
    "lg2.approx",               # lg2_fast
    "cp.async.ca",              # cp_async4 / cp_async8
    "cp.async.cg",              # cp_async16
    "commit_group",             # cp_async_commit
    "wait_group",               # cp_async_wait<N>
    "cudaMemcpy(",              # frt_sync_copy
    "cudaMemset(",              # frt_sync_zero
    "cudaMalloc(",              # frt_malloc
    "cudaGetLastError",         # frt_launch's check, and frt_alloc_status clearing a failed allocation
    "cudaErrorMemoryAllocation",   # FRT_CUDA reports it as FRT_ENOMEM
]


def sources():
    names = sorted(f for f in os.listdir(CSRC) if f.endswith((".cu", ".cuh", ".inc")))
    assert HOME in names and len(names) >= 9
    return {f: open(os.path.join(CSRC, f)).read() for f in names}


@pytest.mark.parametrize("text", ONLY_IN_HOME)
def test_only_in_internal_header(text):
    src = sources()
    assert text in src[HOME]
    elsewhere = [f for f, s in src.items() if f != HOME and text in s]
    assert not elsewhere, "%r belongs in %s only, found in %s" % (text, HOME, elsewhere)
