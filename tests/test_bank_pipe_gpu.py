"""GPU parity of the lane-pipelined filterbank kernel (friture_b200/csrc/bank_pipe.cu), every
variant (32- / 64-sample steps, one / two channels per lane), through the C ABI vs the CPU oracle
(the reference's IIR bank friture/filter.py:86-118 + friture/octavespectrum.py:101-121)."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from parity import TOL, rel_err  # noqa: E402
from test_bank_gpu import energy_rel_err, make_x, oracle_run  # noqa: E402

pytestmark = pytest.mark.gpu

# (channels per lane, log2 step)
VARIANTS = [(1, 5), (2, 5), (1, 6), (2, 6)]


@pytest.fixture
def variant(request):
    pack, logch = request.param
    old = {k: os.environ.get(k) for k in ("FRT_BANK_KERNEL", "FRT_BANK_PACK", "FRT_BANK_LOGCH")}
    os.environ["FRT_BANK_KERNEL"] = "pipe"
    os.environ["FRT_BANK_PACK"] = str(pack)
    os.environ["FRT_BANK_LOGCH"] = str(logch)
    yield pack, logch
    for k, v in old.items():
        if v is None:
            os.environ.pop(k, None)
        else:
            os.environ[k] = v


@pytest.mark.parametrize("variant", VARIANTS, indirect=True)
# 4096 at 32-sample steps: 128 steps per block, more than the event mask holds (phase B every step)
@pytest.mark.parametrize("block,noct", [(256, 9), (512, 9), (1024, 10), (512, 10), (2048, 9), (4096, 9)])
def test_pipe_energies_vs_oracle(variant, block, noct):
    import torch
    from friture_b200.octavefilters import Octave_Filters
    x = make_x(5, 8192, seed=block + noct)          # odd channel count: the last warp holds one channel
    bank = Octave_Filters(3, n_octaves=noct)
    e = bank.energies_batch(torch.from_numpy(x).cuda(), block=block)
    E, _ = oracle_run(bank, x, block, n_octaves=noct)
    assert tuple(e.shape) == (5, 8192 // block, 3 * noct)
    assert energy_rel_err(e.cpu().numpy().astype(np.float64), E) < TOL


@pytest.mark.parametrize("variant", VARIANTS, indirect=True)
def test_pipe_long_stream_and_response_times(variant):
    """65536 samples per channel: the smoothing decays are applied in complement form, so long
    time constants stay inside the tolerance (a float32-rounded (1-alpha) would drift to 1e-4)."""
    import torch
    from friture_b200.octavefilters import Octave_Filters
    x = make_x(2, 65536, seed=3)
    for T in (0.025, 1.0, 5.0):
        bank = Octave_Filters(3, response_time=T)
        e = bank.energies_batch(torch.from_numpy(x).cuda(), block=1024)
        E, _ = oracle_run(bank, x, 1024, response_time=T)
        assert energy_rel_err(e.cpu().numpy().astype(np.float64), E) < TOL, T


@pytest.mark.parametrize("variant", VARIANTS, indirect=True)
def test_pipe_streaming_calls_bit_exact_and_resume(variant):
    import torch
    from friture_b200.octavefilters import Octave_Filters
    x = make_x(3, 8192, seed=5)
    xd = torch.from_numpy(x).cuda()
    once = Octave_Filters(3).energies_batch(xd, block=512).cpu().numpy()
    bank = Octave_Filters(3)
    parts = [bank.energies_batch(xd[:, i:i + 512].contiguous(), block=512).cpu().numpy()
             for i in range(0, 8192, 512)]
    assert np.array_equal(np.concatenate(parts, axis=1), once)
    b = Octave_Filters(3)
    b.energies_batch(xd[:, :4096].contiguous(), block=512)
    z, e = b.get_state()
    c = Octave_Filters(3)
    c.energies_batch(xd[:, :1024].contiguous(), block=512)
    c.set_state(z, e)
    tail = c.energies_batch(xd[:, 4096:].contiguous(), block=512).cpu().numpy()
    assert np.array_equal(tail, once[:, 8:])


@pytest.mark.parametrize("variant", VARIANTS, indirect=True)
def test_pipe_octave_bands_few_octaves_db_weighting(variant):
    import torch
    from friture_b200.octavefilters import Octave_Filters
    x = make_x(4, 4096, seed=11)
    xd = torch.from_numpy(x).cuda()
    bank = Octave_Filters(1)                                       # bpo = 1: 8 sections per stage
    e = bank.energies_batch(xd, block=512)
    E, _ = oracle_run(bank, x, 512)
    assert energy_rel_err(e.cpu().numpy().astype(np.float64), E) < TOL
    for noct in (1, 3, 6, 7):
        bank = Octave_Filters(3, n_octaves=noct)
        e = bank.energies_batch(xd, block=256)
        E, _ = oracle_run(bank, x, 256, n_octaves=noct)
        assert energy_rel_err(e.cpu().numpy().astype(np.float64), E) < TOL, noct
    bank = Octave_Filters(3)
    bank.set_weighting("A")                                        # octavespectrum.py:108-121
    db = bank.energies_batch(xd, block=512, db=True)
    E, _ = oracle_run(bank, x, 512)
    ref = 10 * np.log10(E + 1e-30) + bank.A
    assert rel_err(db.cpu().numpy(), ref) < TOL
    bank.set_weighting(None)
    db = Octave_Filters(3).energies_batch(xd, block=512, db=True)
    assert rel_err(db.cpu().numpy(), 10 * np.log10(E + 1e-30)) < TOL


@pytest.mark.parametrize("variant", VARIANTS, indirect=True)
def test_pipe_and_scan_kernels_share_state(variant):
    """The fused-energy kernel and the chunk-scan kernel (ragged y outputs) can alternate on one
    stream: both carry the state of the same normalised sections."""
    import torch
    from friture_b200.octavefilters import Octave_Filters
    x = make_x(2, 6144, seed=21)
    xd = torch.from_numpy(x).cuda()
    bank = Octave_Filters(3)
    e1 = bank.energies_batch(xd[:, :2048].contiguous(), block=512)                   # pipe
    y, e2 = bank.filter_batch(xd[:, 2048:4096].contiguous(), block=512, want_y=True)  # scan
    e3 = bank.energies_batch(xd[:, 4096:].contiguous(), block=512)                   # pipe
    E, Y = oracle_run(bank, x, 512)
    got = torch.cat([e1, e2, e3], dim=1).cpu().numpy().astype(np.float64)
    assert energy_rel_err(got, E) < TOL
    for k in (0, 13, 26):
        ref = Y[0][k][(2048 >> (8 - k // 3)):(4096 >> (8 - k // 3))]
        gotk = y[k][0].cpu().numpy().astype(np.float64)
        assert np.max(np.abs(gotk - ref)) / np.max(np.abs(ref)) < 5e-5


@pytest.mark.parametrize("variant", VARIANTS, indirect=True)
def test_pipe_unaligned_rows_and_many_channels(variant):
    import torch
    from friture_b200.octavefilters import Octave_Filters
    big = torch.from_numpy(make_x(301, 1025, seed=13)).cuda()
    a = Octave_Filters(3).energies_batch(big[:, 1:], block=512)                # 4-byte aligned rows
    b = Octave_Filters(3).energies_batch(big[:, 1:].contiguous(), block=512)
    assert torch.equal(a, b)
    x = big[:7, 1:].cpu().numpy()
    bank = Octave_Filters(3)
    E, _ = oracle_run(bank, x, 512)
    assert energy_rel_err(b[:7].cpu().numpy().astype(np.float64), E) < TOL
