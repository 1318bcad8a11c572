"""Handle lifecycle through the C ABI: destroying a handle returns every byte of device memory it
allocated, and a plan call that is rejected leaves the handle's previous plan of that kind working.

The first test plans every kind of plan a handle holds, runs every entry point that uses one
(including the two host-buffer entry points, which keep their own streams and staging buffers),
re-plans at other sizes and closes the handle, three times over; free device memory must come back
to the same value after each cycle."""
import numpy as np
import pytest

C = 8                 # channels
T = 8192              # samples per channel
HOP = 1024            # STFT hop and filterbank block
N_OCT = 9
STFT_SIZES = (4096, 2048)   # the second is current when the process calls run
GCC_LENGTHS = (2400, 16800)  # planned (shared-memory route), then re-planned and run (Bluestein route)
GCC_PAIRS = 4
DEC_STAGES = 2


def _tables(bpo):
    """(sos_band, sos_dec, alphas, fir_band, fir_dec, weight_db) for a bpo bank of N_OCT octaves."""
    from friture_b200 import filter_data
    from friture_b200.octavefilters import smoothing_alphas
    sos_band = np.ascontiguousarray(filter_data.bands(bpo)[2], dtype=np.float64)
    sos_dec = np.ascontiguousarray(filter_data.decimator()[2], dtype=np.float64)
    fir_band, fir_dec = filter_data.fir_taps(bpo)
    weight = np.linspace(-30.0, 3.0, N_OCT * bpo).astype(np.float32)
    return (sos_band, sos_dec, smoothing_alphas(1.0, N_OCT),
            np.ascontiguousarray(fir_band, dtype=np.float64),
            np.ascontiguousarray(fir_dec, dtype=np.float64), weight)


def _bank_plan(h, bpo, tables):
    from friture_b200._lib import _ptr
    sos_band, sos_dec, alphas, _, _, weight = tables
    h.call("frt_bank_plan", C, bpo, N_OCT, _ptr(sos_band), _ptr(sos_dec), _ptr(alphas))
    h.call("frt_bank_set_weighting", _ptr(weight))


def _fir_plan(h, bpo, tables):
    from friture_b200._lib import _ptr
    _, _, alphas, fir_band, fir_dec, weight = tables
    h.call("frt_firbank_plan", C, bpo, N_OCT, fir_band.shape[1], _ptr(fir_band), _ptr(fir_dec))
    h.call("frt_firbank_set_smoothing", _ptr(alphas), _ptr(weight))


@pytest.fixture(scope="module")
def bufs():
    """Every input and output the cycles use, allocated once so that torch allocates nothing
    while handles come and go."""
    import torch
    from friture_b200.octavefilters import ragged_layout
    g = torch.Generator().manual_seed(7)
    x = torch.randn((C, T), generator=g, dtype=torch.float32)
    nbins = STFT_SIZES[-1] // 2 + 1
    frames = (T - STFT_SIZES[-1]) // HOP + 1
    offsets, lengths = ragged_layout(HOP, 3, N_OCT)
    L = max(GCC_LENGTHS)
    b = {
        "x": x.cuda(),
        "x_host": x.pin_memory(),
        "spec": torch.empty((C, frames, nbins), device="cuda"),
        "spec_host": torch.empty((C, frames, nbins)).pin_memory(),
        "comb_spec_host": torch.empty((C, frames, nbins)).pin_memory(),
        "bands_host": torch.empty((C, T // HOP, N_OCT * 3)).pin_memory(),
        "energies": torch.empty((C, T // HOP, N_OCT * 3), device="cuda"),
        "levels": torch.empty((C, T // HOP, N_OCT * 3), device="cuda"),
        "y": torch.empty((C, int(offsets[-1] + lengths[-1])), device="cuda"),
        "dec": torch.empty((C, T >> DEC_STAGES), device="cuda"),
        "d0": torch.randn((GCC_PAIRS, L), generator=g).cuda(),
        "d1": torch.randn((GCC_PAIRS, L), generator=g).cuda(),
        "xcorr": torch.empty((GCC_PAIRS, L), device="cuda"),
        "idx": torch.empty((GCC_PAIRS,), dtype=torch.int32, device="cuda"),
        "val": torch.empty((GCC_PAIRS,), device="cuda"),
    }
    torch.cuda.synchronize()
    return b


def _cycle(b, tables3, tables6):
    import torch
    from friture_b200._lib import Handle, _ptr, current_stream_ptr
    h = Handle(0)
    st = current_stream_ptr(b["x"].device)
    # plan every kind
    for n in STFT_SIZES:
        h.call("frt_stft_plan", n)
    _bank_plan(h, 3, tables3)
    _fir_plan(h, 3, tables3)
    h.call("frt_gcc_plan", GCC_LENGTHS[0])
    h.call("frt_decimate_plan", C, DEC_STAGES, _ptr(tables3[1]))
    # every entry point that runs a plan, once
    N = STFT_SIZES[-1]
    nbins, frames = N // 2 + 1, (T - N) // HOP + 1
    h.call("frt_stft_process", _ptr(b["x"]), T, C, frames, HOP, _ptr(b["spec"]), frames * nbins, nbins,
           1, st)
    h.call("frt_bank_process", _ptr(b["x"]), T, HOP, T // HOP, _ptr(b["energies"]), None, 0, 1, st)
    h.call("frt_firbank_process", _ptr(b["x"]), T, HOP, _ptr(b["y"]), b["y"].shape[1], st)
    h.call("frt_firbank_levels", _ptr(b["x"]), T, HOP, T // HOP, _ptr(b["levels"]), 1, st)
    gcc_phat = lambda: h.call("frt_gcc_phat", _ptr(b["d0"]), _ptr(b["d1"]), b["d0"].shape[1], GCC_PAIRS,
                              _ptr(b["xcorr"]), None, 0, _ptr(b["idx"]), _ptr(b["val"]), st)
    gcc_phat()
    h.call("frt_decimate_process", _ptr(b["x"]), T, T, _ptr(b["dec"]), T >> DEC_STAGES, st)
    torch.cuda.synchronize()
    h.call("frt_stft_process_host", _ptr(b["x_host"]), T, C, T, HOP, _ptr(b["spec_host"]), 1)
    h.call("frt_combined_process_host", _ptr(b["x_host"]), T, C, T, HOP, _ptr(b["comb_spec_host"]),
           _ptr(b["bands_host"]), N_OCT * 3, 1)
    # re-plan at other sizes: the replaced plans are freed on the way; the second GCC length adds
    # the Bluestein plan and its workspace next to the shared-memory plan
    _bank_plan(h, 6, tables6)
    _fir_plan(h, 6, tables6)
    h.call("frt_gcc_plan", GCC_LENGTHS[1])
    gcc_phat()
    h.close()
    torch.cuda.synchronize()


@pytest.mark.gpu
def test_teardown_returns_device_memory(bufs):
    """One warm-up cycle loads the kernel modules; free device memory after each of three more
    cycles equals its value after the warm-up."""
    import torch
    tables3, tables6 = _tables(3), _tables(6)
    _cycle(bufs, tables3, tables6)
    free0 = torch.cuda.mem_get_info()[0]
    after = []
    for _ in range(3):
        _cycle(bufs, tables3, tables6)
        after.append(torch.cuda.mem_get_info()[0])
    assert after == [free0] * 3, (free0, after)


def _rejecting_copy(sos):
    """The SOS table with b2 != b0 in its first row: zeros off the unit circle, which the plan
    calls reject."""
    bad = sos.copy()
    bad.reshape(-1, 6)[0, 2] = 1.5 * bad.reshape(-1, 6)[0, 0]
    return bad


@pytest.mark.gpu
def test_rejected_plan_keeps_previous_plan(bufs):
    """A bank plan and a decimator plan run a chunk on two handles.  One handle then gets a plan
    call with a rejected SOS table, which raises FrtValueError; the next chunk must still run on
    both handles from the same state and give bit-identical outputs."""
    import torch
    from friture_b200._lib import FrtValueError, Handle, _ptr, current_stream_ptr
    tables = _tables(3)
    sos_band, sos_dec, alphas = tables[:3]
    x = bufs["x"]
    st = current_stream_ptr(x.device)
    ref, h = Handle(0), Handle(0)
    try:
        outs = {}
        for name, hd in (("ref", ref), ("h", h)):
            _bank_plan(hd, 3, tables)
            hd.call("frt_decimate_plan", C, DEC_STAGES, _ptr(sos_dec))
            e = torch.empty((2, C, T // HOP, N_OCT * 3), device="cuda")
            d = torch.empty((2, C, T >> DEC_STAGES), device="cuda")
            for k in range(2):
                if k == 1 and hd is h:
                    with pytest.raises(FrtValueError):
                        hd.call("frt_bank_plan", C, 3, N_OCT, _ptr(_rejecting_copy(sos_band)), _ptr(sos_dec),
                                _ptr(alphas))
                    with pytest.raises(FrtValueError):
                        hd.call("frt_decimate_plan", C, DEC_STAGES, _ptr(_rejecting_copy(sos_dec)))
                hd.call("frt_bank_process", _ptr(x), T, HOP, T // HOP, _ptr(e[k]), None, 0, 1, st)
                hd.call("frt_decimate_process", _ptr(x), T, T, _ptr(d[k]), T >> DEC_STAGES, st)
            torch.cuda.synchronize()
            outs[name] = (e, d)
        for k in range(2):
            assert torch.equal(outs["h"][0][k], outs["ref"][0][k]), "bank energies, chunk %d" % k
            assert torch.equal(outs["h"][1][k], outs["ref"][1][k]), "decimator output, chunk %d" % k
        assert torch.isfinite(outs["h"][0]).all()
    finally:
        ref.close()
        h.close()
