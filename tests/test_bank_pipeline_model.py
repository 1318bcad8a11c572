"""CPU checks of the lane-pipelined filterbank schedule (friture_b200/csrc/bank_pipe.cu):
the executable model in bank_pipeline_model.py against the oracle, and the library's own schedule
arithmetic (frt_bank_schedule, pure host code) against the model's."""
import ctypes
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from bank_pipeline_model import PipeModel, flush_delta, n_steps_for, stage_start_steps  # noqa: E402

EN_RING = 8   # staged band-energy blocks per channel slot (bank_pipe.cu)
PIPE_MIN_BLOCK = {5: 256, 6: 512}   # logch -> shortest block bank_route runs in such steps (bank_internal.cuh)


def _oracle_energies(bpo, n_oct, block, x, response_time=1.0):
    from friture_b200 import filter_data
    from oracle import friture_oracle as fo
    bdec, adec, _ = filter_data.decimator()
    boct, aoct, _ = filter_data.bands(bpo)
    orc = fo.OctaveSpectrumOracle(bdec, adec, list(boct), list(aoct), noctave=n_oct,
                                  response_time=response_time)
    return np.array([orc.push(x[b * block:(b + 1) * block])[0] for b in range(len(x) // block)])


def _model(bpo, n_oct, logch, response_time=1.0):
    from friture_b200 import filter_data
    from friture_b200.octavefilters import smoothing_alphas
    _, _, sos_dec = filter_data.decimator()
    _, _, sos = filter_data.bands(bpo)
    return PipeModel(sos, sos_dec, smoothing_alphas(response_time, n_oct), n_oct, logch=logch)


@pytest.mark.parametrize("bpo,n_oct,block,T,logch", [
    (3, 9, 512, 2048, 5), (3, 10, 512, 4096, 5), (3, 9, 256, 2048, 5), (3, 10, 1024, 4096, 6),
    (1, 9, 512, 2048, 5), (3, 3, 512, 1024, 5), (3, 1, 256, 1024, 5), (3, 7, 256, 1024, 6),
    (3, 9, 512, 2048, 6),
])
def test_schedule_model_matches_oracle(bpo, n_oct, block, T, logch):
    x = np.random.default_rng(bpo + n_oct + block).standard_normal(T) * 0.1
    E = _oracle_energies(bpo, n_oct, block, x)
    got = _model(bpo, n_oct, logch).process(x, block)
    assert np.max(np.abs(got - E) / np.max(np.abs(E), axis=-1, keepdims=True)) < 1e-10


def test_schedule_model_streaming_and_state():
    """Block-by-block launches (pipeline drained and refilled every time) == one launch."""
    x = np.random.default_rng(4).standard_normal(4096) * 0.1
    E = _oracle_energies(3, 9, 512, x)
    m = _model(3, 9, 5)
    got = np.concatenate([m.process(x[i:i + 512], 512) for i in range(0, 4096, 512)])
    assert np.max(np.abs(got - E) / np.max(np.abs(E), axis=-1, keepdims=True)) < 1e-10


def ring_slots(n_oct, logch, block):
    """Energy-ring slots a block needs: a block's vector leaves flush_delta steps after its last chunk,
    and the blocks staged meanwhile plus the one being written must fit (frt_pipe_prepare)."""
    fdelta = flush_delta(n_oct, logch, stage_start_steps(n_oct, logch))
    nb = block >> logch
    return (fdelta + nb - 1) // nb + 2


def test_energy_ring_holds_every_supported_block():
    """The ring holds the shortest block bank_route gives each step size at every octave count, so
    frt_pipe_prepare never turns the pipelined kernel off for a bank the library plans; longer
    power-of-two blocks need no more slots, which is why it checks the shortest only."""
    for n_oct in range(1, 11):
        for logch, shortest in PIPE_MIN_BLOCK.items():
            need = ring_slots(n_oct, logch, shortest)
            assert need <= EN_RING, (n_oct, logch, shortest, need)
            for block in (shortest << b for b in range(1, 9)):
                assert ring_slots(n_oct, logch, block) <= need, (n_oct, logch, block)
    assert max(ring_slots(n_oct, 6, 512) for n_oct in range(1, 11)) == 6
    # 256-sample blocks in 64-sample steps, which bank_route does not take, would fill the ring at 9
    # octaves and overflow it at 10 (where the block rule refuses 256-sample blocks anyway)
    assert [ring_slots(n_oct, 6, 256) for n_oct in (8, 9, 10)] == [8, 8, 9]
    assert all(ring_slots(n_oct, 6, 256) <= EN_RING for n_oct in range(1, 10))


def test_library_schedule_matches_model():
    from friture_b200 import _lib
    lib = _lib.load_library()
    for n_oct in (1, 3, 6, 7, 9, 10):
        for logch in (5, 6):
            for T in (512, 1024, 4096, 1024 * 256):
                ss = (ctypes.c_int * 10)()
                ns = ctypes.c_int()
                assert lib.frt_bank_schedule(n_oct, logch, T, ss, ctypes.byref(ns)) == 0
                Tm = stage_start_steps(n_oct, logch)
                assert list(ss) == Tm[:10]
                assert ns.value == n_steps_for(n_oct, logch, T, Tm)
    assert lib.frt_bank_schedule(0, 5, 512, (ctypes.c_int * 10)(), None) != 0
    assert lib.frt_bank_schedule(9, 4, 512, (ctypes.c_int * 10)(), None) != 0
