"""Which STFT kernel each FFT size and input alignment runs (friture_b200/csrc/stft.cu, frt_stft_process and
frt_stft_screen_rows).

The choice is a function of the planned size, the output mode and how far every frame's start is aligned
(16 bytes, 8 bytes only, or 4 bytes).  Every case runs one audioproc.stft call (power, log power) or one
frt_stft_screen_rows call (screen rows, as SpectrogramAnalyzer makes them) under the CUDA profiler and checks
the name of the kernel that ran; between them the cases launch every compiled instance."""
import json
import os
import re
import subprocess
import sys

import pytest

POWER, LOGPOWER, SCREEN = 0, 1, 2
MODES = (POWER, LOGPOWER, SCREEN)
ALIGNS = {16: 0, 8: 2, 4: 1}     # frame alignment in bytes -> offset of the first sample in floats


def kernel_for(n, mode, align):
    """(N, mode, alignment) -> kernel (demangled name, template arguments)."""
    if n == 32:
        return "stft_generic_kernel<%d>" % mode
    if n <= 2048:
        return "stft_small_kernel<%d, %d, %s>" % (n // 64, mode, "true" if n == 2048 and align == 16 else "false")
    if n <= 8192 and align >= 8:
        return "stft_large_kernel<%d, %d>" % (n // 2048, mode)
    return "stft_multi_kernel<%d, %d>" % (n // 2048, mode)


CASES = [(n, mode, align, kernel_for(n, mode, align))
         for n in (32, 64, 128, 256, 512, 1024, 2048, 4096, 8192, 16384)
         for mode in MODES for align in ALIGNS]


def instances(modes):
    """Every compiled instance of the output modes ``modes``."""
    return ({"stft_small_kernel<%d, %d, false>" % (q, m) for q in (1, 2, 4, 8, 16, 32) for m in modes}
            | {"stft_small_kernel<32, %d, true>" % m for m in modes}
            | {"stft_large_kernel<%d, %d>" % (r, m) for r in (2, 4) for m in modes}
            | {"stft_multi_kernel<%d, %d>" % (r, m) for r in (2, 4, 8) for m in modes}
            | {"stft_generic_kernel<%d>" % m for m in modes})


INSTANCES = instances((POWER, LOGPOWER))      # test_stft_bins_gpu checks each of these bin by bin
SCREEN_INSTANCES = instances((SCREEN,))


def test_cases_cover_every_instance():
    assert {c[-1] for c in CASES} == INSTANCES | SCREEN_INSTANCES


def launch_all():
    """Runs every case under the CUDA profiler and prints {case: names of the STFT kernels that ran}."""
    from ctypes import c_float

    import torch
    from torch.profiler import ProfilerActivity, profile
    from friture_b200 import _lib, audioproc
    launched = {}
    for n, mode, align, _ in CASES:
        hop, frames = n // 2, 5
        t = n + (frames - 1) * hop
        off = ALIGNS[align]
        g = torch.Generator(device="cuda").manual_seed(n + align)
        # two channels, row stride a multiple of 4 floats: the offset alone sets the frames' alignment
        buf = torch.randn(2, t + 4, generator=g, device="cuda") * 0.1
        x = buf[:, off:off + t]
        assert x.data_ptr() % 16 == 4 * off
        p = audioproc()
        p.set_fftsize(n)
        if mode == SCREEN:      # eight screen rows, between bins 0 and 8
            H = 8
            i0 = torch.arange(H, dtype=torch.int32, device="cuda")
            t = torch.full((H,), 0.25, device="cuda")
            rows = torch.empty((2, frames, H), device="cuda")

            def run():
                p.handle.call("frt_stft_plan", n)
                p.handle.call("frt_stft_screen_rows", _lib._ptr(x), int(x.stride(0)), 2, frames, hop, None,
                              c_float(-140.), c_float(0.), _lib._ptr(i0), _lib._ptr(t), H, _lib._ptr(rows),
                              frames * H, H, _lib.current_stream_ptr())
        else:
            def run():
                p.stft(x, hop=hop, log=mode == LOGPOWER)
        run()                   # plans the size outside the profiled window
        torch.cuda.synchronize()
        for _ in range(3):      # the profiler has been seen to record the launch call but not the kernel
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                run()
                torch.cuda.synchronize()
            names = [e.name for e in prof.events() if re.search(r"\bstft\w*_kernel", e.name)]
            if names:
                break
        launched["%d-%d-%d" % (n, mode, align)] = names
    print(json.dumps(launched))


@pytest.fixture(scope="module")
def launched():
    # a fresh process: late in a long test session the profiler has been seen to record the launch
    # call but not the kernel
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    run = subprocess.run([sys.executable, os.path.abspath(__file__)], cwd=root, capture_output=True, text=True)
    assert run.returncode == 0, run.stderr[-4000:]
    return json.loads(run.stdout.strip().splitlines()[-1])


@pytest.mark.gpu
@pytest.mark.parametrize("n,mode,align,kernel", CASES)
def test_kernel_choice(launched, n, mode, align, kernel):
    names = launched["%d-%d-%d" % (n, mode, align)]
    assert len(names) == 1, names
    pattern = r"\b" + re.escape(kernel).replace(r"\ ", " ?") + r"\("
    assert re.search(pattern, names[0]), (names[0], kernel)


if __name__ == "__main__":
    sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
    launch_all()
