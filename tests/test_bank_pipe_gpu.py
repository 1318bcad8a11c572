"""GPU parity of the lane-pipelined filterbank kernel (friture_b200/csrc/bank_pipe.cu), through the C ABI
vs the CPU oracle (the reference's IIR bank friture/filter.py:86-118 + friture/octavespectrum.py:101-121).

Each test runs at (channels, block) pairs that the library maps to each pipelined variant
(test_bank_dispatch_gpu.py pins the mapping): up to 3072 channels, 32-sample steps for 256-sample
blocks and 64-sample steps for longer ones; above 3072 channels, 32-sample steps with two channels per
lane.  A many-channel input is a few seeded rows repeated on the device, so the oracle runs once per
distinct row and the repeats must come out bit-equal."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from parity import TOL, rel_err  # noqa: E402
from test_bank_gpu import energy_rel_err, make_x, oracle_run  # noqa: E402

pytestmark = pytest.mark.gpu

MANY = 3073       # two channels per lane; odd, so the last warp holds one channel
DISTINCT = 3      # seeded rows behind a many-channel input


def rows(C, T, seed):
    """[C, T] input on the GPU and the distinct rows it is made of (numpy): C seeded rows, or for more
    than 512 channels DISTINCT seeded rows repeated (channel c is row c % DISTINCT)."""
    import torch
    base = make_x(C if C <= 512 else DISTINCT, T, seed)
    k = len(base)
    xd = torch.from_numpy(base).cuda().repeat((C + k - 1) // k, 1)[:C].contiguous()
    return xd, base


def distinct(out, k):
    """out[:k] (numpy) after checking that every channel equals its distinct row bit for bit."""
    import torch
    C = out.shape[0]
    idx = torch.arange(C, device=out.device) % k
    assert torch.equal(out, out[idx]), "repeated rows differ"
    return out[:k].cpu().numpy()


@pytest.mark.parametrize("channels,block,noct", [
    (5, 256, 9), (3072, 256, 9),                                                     # 32-sample steps
    *[(C, b, n) for C in (5, 3072) for b, n in ((512, 9), (1024, 10), (512, 10), (2048, 9), (4096, 9))],
    # two channels per lane; 4096: 128 steps per block, more than the event mask holds (phase B every step)
    *[(C, b, n) for C in (MANY, 4096)
      for b, n in ((256, 9), (512, 9), (1024, 10), (512, 10), (2048, 9), (4096, 9))],
])
def test_pipe_energies_vs_oracle(channels, block, noct):
    from friture_b200.octavefilters import Octave_Filters
    xd, x = rows(channels, 8192, seed=block + noct)
    bank = Octave_Filters(3, n_octaves=noct)
    e = bank.energies_batch(xd, block=block)
    E, _ = oracle_run(bank, x, block, n_octaves=noct)
    assert tuple(e.shape) == (channels, 8192 // block, 3 * noct)
    assert energy_rel_err(distinct(e, len(x)).astype(np.float64), E) < TOL


@pytest.mark.parametrize("channels,block", [(2, 256), (2, 1024), (MANY, 256), (MANY, 1024)])
def test_pipe_long_stream_and_response_times(channels, block):
    """65536 samples per channel: the smoothing decays are applied in complement form, so long
    time constants stay inside the tolerance (a float32-rounded (1-alpha) would drift to 1e-4)."""
    from friture_b200.octavefilters import Octave_Filters
    xd, x = rows(channels, 65536, seed=3)
    for T in (0.025, 1.0, 5.0):
        bank = Octave_Filters(3, response_time=T)
        e = bank.energies_batch(xd, block=block)
        E, _ = oracle_run(bank, x, block, response_time=T)
        assert energy_rel_err(distinct(e, len(x)).astype(np.float64), E) < TOL, T


@pytest.mark.parametrize("channels,block", [(3, 256), (3, 512), (MANY, 256), (MANY, 512)])
def test_pipe_streaming_calls_bit_exact_and_resume(channels, block):
    from friture_b200.octavefilters import Octave_Filters
    xd, _ = rows(channels, 8192, seed=5)
    once = Octave_Filters(3).energies_batch(xd, block=block).cpu().numpy()
    bank = Octave_Filters(3)
    parts = [bank.energies_batch(xd[:, i:i + 512].contiguous(), block=block).cpu().numpy()
             for i in range(0, 8192, 512)]
    assert np.array_equal(np.concatenate(parts, axis=1), once)
    b = Octave_Filters(3)
    b.energies_batch(xd[:, :4096].contiguous(), block=block)
    z, e = b.get_state()
    c = Octave_Filters(3)
    c.energies_batch(xd[:, :1024].contiguous(), block=block)
    c.set_state(z, e)
    tail = c.energies_batch(xd[:, 4096:].contiguous(), block=block).cpu().numpy()
    assert np.array_equal(tail, once[:, 4096 // block:])


@pytest.mark.parametrize("channels,block", [(4, 256), (4, 512), (MANY, 256), (MANY, 512)])
def test_pipe_octave_bands_few_octaves_db_weighting(channels, block):
    from friture_b200.octavefilters import Octave_Filters
    xd, x = rows(channels, 4096, seed=11)
    k = len(x)
    bank = Octave_Filters(1)                                       # bpo = 1: 8 sections per stage
    e = bank.energies_batch(xd, block=block)
    E, _ = oracle_run(bank, x, block)
    assert energy_rel_err(distinct(e, k).astype(np.float64), E) < TOL
    for noct in (1, 3, 6, 7):
        bank = Octave_Filters(3, n_octaves=noct)
        e = bank.energies_batch(xd, block=block)
        E, _ = oracle_run(bank, x, block, n_octaves=noct)
        assert energy_rel_err(distinct(e, k).astype(np.float64), E) < TOL, noct
    bank = Octave_Filters(3)
    bank.set_weighting("A")                                        # octavespectrum.py:108-121
    db = bank.energies_batch(xd, block=block, db=True)
    E, _ = oracle_run(bank, x, block)
    ref = 10 * np.log10(E + 1e-30) + bank.A
    assert rel_err(distinct(db, k), ref) < TOL
    bank.set_weighting(None)
    db = Octave_Filters(3).energies_batch(xd, block=block, db=True)
    assert rel_err(distinct(db, k), 10 * np.log10(E + 1e-30)) < TOL


@pytest.mark.parametrize("channels,block", [(2, 256), (2, 512), (MANY, 256), (MANY, 512)])
def test_pipe_and_scan_kernels_share_state(channels, block):
    """The fused-energy kernel and the chunk-scan kernel (ragged y outputs) can alternate on one
    stream: both carry the state of the same normalised sections."""
    import torch
    from friture_b200.octavefilters import Octave_Filters
    xd, x = rows(channels, 6144, seed=21)
    k = len(x)
    bank = Octave_Filters(3)
    e1 = bank.energies_batch(xd[:, :2048].contiguous(), block=block)                   # pipe
    y, e2 = bank.filter_batch(xd[:, 2048:4096].contiguous(), block=block, want_y=True)  # scan
    e3 = bank.energies_batch(xd[:, 4096:].contiguous(), block=block)                   # pipe
    E, Y = oracle_run(bank, x, block)
    got = distinct(torch.cat([e1, e2, e3], dim=1), k).astype(np.float64)
    assert energy_rel_err(got, E) < TOL
    for b in (0, 13, 26):
        yb = distinct(y[b], k)
        for c in range(k):
            ref = Y[c][b][(2048 >> (8 - b // 3)):(4096 >> (8 - b // 3))]
            assert np.max(np.abs(yb[c].astype(np.float64) - ref)) / np.max(np.abs(ref)) < 5e-5, (c, b)


@pytest.mark.parametrize("channels,block", [(301, 256), (301, 512), (MANY, 256), (MANY, 512)])
def test_pipe_unaligned_rows_and_many_channels(channels, block):
    import torch
    from friture_b200.octavefilters import Octave_Filters
    big, x = rows(channels, 1025, seed=13)
    a = Octave_Filters(3).energies_batch(big[:, 1:], block=block)                # 4-byte aligned rows
    b = Octave_Filters(3).energies_batch(big[:, 1:].contiguous(), block=block)
    assert torch.equal(a, b)
    got = distinct(b, len(x))[:7]
    bank = Octave_Filters(3)
    E, _ = oracle_run(bank, x[:7, 1:], block)
    assert energy_rel_err(got.astype(np.float64), E) < TOL
