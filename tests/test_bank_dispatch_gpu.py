"""Which filterbank kernel each input shape runs (friture_b200/csrc/bank.cu, bank_process_impl).

The choice is a function of the plan (bands per octave, octaves, channels), the block length and
whether the ragged band outputs are requested.  Every case runs one call under the CUDA profiler and
checks the name of the kernel that ran; between them the cases launch every compiled instance."""
import re

import pytest

# (bands per octave, octaves, channels, block, want_y) -> kernel (demangled name, template arguments)
CASES = [
    # pipelined kernel: bpo 1 or 3, power-of-two block, energies only
    *[(bpo, 9, 3072, 512, False, "bank_pipe_kernel<6, 1, %d>" % bpo) for bpo in (1, 3)],
    *[(bpo, 9, 3072, 256, False, "bank_pipe_kernel<5, 1, %d>" % bpo) for bpo in (1, 3)],
    *[(bpo, 9, 3073, 512, False, "bank_pipe_kernel<5, 2, %d>" % bpo) for bpo in (1, 3)],
    # chunk-scan kernel: tile 1024/512/256 by divisibility; three warps per channel below 1536
    # channels when the bank has more octaves than scan-mode stages and the tile is at most 512
    (6, 9, 2, 512, False, "bank_kernel3<16, false>"),
    (3, 9, 2, 768, False, "bank_kernel3<8, false>"),
    (3, 9, 2, 256, True, "bank_kernel3<8, true>"),
    (3, 9, 2, 512, True, "bank_kernel3<16, true>"),
    (3, 9, 2, 1024, True, "bank_kernel<32, true>"),
    (3, 3, 2, 512, True, "bank_kernel<16, true>"),
    (3, 9, 1537, 256, True, "bank_kernel<8, true>"),
    (6, 9, 2, 1024, False, "bank_kernel<32, false>"),
    (3, 9, 1536, 1536, False, "bank_kernel<16, false>"),
    (3, 9, 1536, 768, False, "bank_kernel<8, false>"),
]

INSTANCES = ({"bank_pipe_kernel<%d, %d, %d>" % v for v in ((6, 1, 1), (6, 1, 3), (5, 1, 1), (5, 1, 3),
                                                            (5, 2, 1), (5, 2, 3))}
             | {"bank_kernel<%d, %s>" % (L, y) for L in (8, 16, 32) for y in ("false", "true")}
             | {"bank_kernel3<%d, %s>" % (L, y) for L in (8, 16) for y in ("false", "true")})


def test_cases_cover_every_instance():
    assert {c[-1] for c in CASES} == INSTANCES


@pytest.mark.gpu
@pytest.mark.parametrize("bpo,noct,channels,block,want_y,kernel", CASES)
def test_kernel_choice(bpo, noct, channels, block, want_y, kernel):
    import torch
    from torch.profiler import ProfilerActivity, profile
    from friture_b200.octavefilters import Octave_Filters
    g = torch.Generator(device="cuda").manual_seed(block + channels)
    x = torch.randn(channels, 2 * block, generator=g, device="cuda") * 0.1
    bank = Octave_Filters(bpo, n_octaves=noct)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        bank.filter_batch(x, block=block, want_y=want_y)
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if re.search(r"\bbank(_pipe)?_kernel", e.name)]
    assert len(names) == 1, names
    pattern = r"\b" + re.escape(kernel).replace(r"\ ", " ?") + r"\("
    assert re.search(pattern, names[0]), (names[0], kernel)
