"""An allocation the device cannot hold is refused with FRT_ENOMEM and leaves the handle usable.

Each case makes one entry point ask for at least twice the device's memory through its arguments
alone, so the driver refuses the request without taking memory from anything else on the device.
None of these arguments sizes a host buffer.  After the refusal, no kernel has been launched, and the
plans from before the call (STFT, IIR and FIR filterbanks, decimator, GCC-PHAT) still run and give the
same bits as the same calls on a fresh handle: the CUDA runtime may keep a refused allocation as its
last error, and the check after the next kernel launch must not report it."""
import numpy as np
import pytest

C = 4                  # channels of the calls that must still run
T = 2048               # samples per channel
N_FFT = 256
HOP = 1024             # STFT hop and filterbank block
BPO, N_OCT = 3, 9
GCC_L = 2400           # a shared-memory route length
INT_MAX = 2**31 - 1


def _tables():
    from friture_b200 import filter_data
    from friture_b200.octavefilters import smoothing_alphas
    fir_band, fir_dec = filter_data.fir_taps(BPO)
    return {
        "sos_band": np.ascontiguousarray(filter_data.bands(BPO)[2], dtype=np.float64),
        "sos_dec": np.ascontiguousarray(filter_data.decimator()[2], dtype=np.float64),
        "alphas": smoothing_alphas(1.0, N_OCT),
        "fir_band": np.ascontiguousarray(fir_band, dtype=np.float64),
        "fir_dec": np.ascontiguousarray(fir_dec, dtype=np.float64),
    }


@pytest.fixture(scope="module")
def env():
    import torch
    from friture_b200.octavefilters import ragged_layout
    g = torch.Generator().manual_seed(11)
    offsets, lengths = ragged_layout(HOP, BPO, N_OCT)
    nbins = 513
    frames = (T - N_FFT) // HOP + 1
    b = {
        "x": torch.randn((C, T), generator=g).cuda(),
        "d0": torch.randn((2, GCC_L), generator=g).cuda(),
        "d1": torch.randn((2, GCC_L), generator=g).cuda(),
        "power": torch.rand((1, 1, nbins), generator=g).cuda(),
        "unused": torch.zeros((4096,), device="cuda"),   # outputs of the refused calls: never reached
    }
    torch.cuda.synchronize()
    return {"b": b, "t": _tables(), "mem": torch.cuda.get_device_properties(0).total_memory,
            "frames": frames, "y_len": int(offsets[-1] + lengths[-1]), "nbins": nbins}


def _plan(h, t):
    """The plans both handles hold before the refused call."""
    from friture_b200._lib import _ptr
    h.call("frt_stft_plan", N_FFT)
    h.call("frt_bank_plan", C, BPO, N_OCT, _ptr(t["sos_band"]), _ptr(t["sos_dec"]), _ptr(t["alphas"]))
    h.call("frt_firbank_plan", C, BPO, N_OCT, t["fir_band"].shape[1], _ptr(t["fir_band"]), _ptr(t["fir_dec"]))
    h.call("frt_decimate_plan", C, 2, _ptr(t["sos_dec"]))
    h.call("frt_gcc_plan", GCC_L)


def _run(h, env):
    """Every planned entry point once, on the current stream; returns the outputs."""
    import torch
    from friture_b200._lib import STFT_LOGPOWER, _ptr, current_stream_ptr
    b, x = env["b"], env["b"]["x"]
    st = current_stream_ptr(x.device)
    nbins, F = N_FFT // 2 + 1, env["frames"]
    out = {
        "spec": torch.empty((C, F, nbins), device="cuda"),
        "energies": torch.empty((C, T // HOP, N_OCT * BPO), device="cuda"),
        "y": torch.empty((C, env["y_len"]), device="cuda"),
        "dec": torch.empty((C, T >> 2), device="cuda"),
        "xcorr": torch.empty((2, GCC_L), device="cuda"),
        "idx": torch.empty((2,), dtype=torch.int32, device="cuda"),
        "val": torch.empty((2,), device="cuda"),
    }
    h.call("frt_stft_process", _ptr(x), T, C, F, HOP, _ptr(out["spec"]), F * nbins, nbins, STFT_LOGPOWER, st)
    h.call("frt_bank_process", _ptr(x), T, HOP, T // HOP, _ptr(out["energies"]), None, 0, 1, st)
    h.call("frt_firbank_process", _ptr(x), T, HOP, _ptr(out["y"]), env["y_len"], st)
    h.call("frt_decimate_process", _ptr(x), T, T, _ptr(out["dec"]), T >> 2, st)
    h.call("frt_gcc_phat", _ptr(b["d0"]), _ptr(b["d1"]), GCC_L, 2, _ptr(out["xcorr"]), None, 0, _ptr(out["idx"]),
           _ptr(out["val"]), st)
    torch.cuda.synchronize()
    return out


def _refuse(h, case, env):
    """The case's call, which must be refused."""
    import ctypes
    from friture_b200._lib import _ptr, current_stream_ptr
    b, t, st = env["b"], env["t"], current_stream_ptr(env["b"]["x"].device)
    x, p, u = b["x"], b["power"], _ptr(b["unused"])
    if case == "bank_plan":
        h.call("frt_bank_plan", INT_MAX, BPO, N_OCT, _ptr(t["sos_band"]), _ptr(t["sos_dec"]), _ptr(t["alphas"]))
    elif case == "firbank_plan":
        h.call("frt_firbank_plan", INT_MAX, BPO, N_OCT, t["fir_band"].shape[1], _ptr(t["fir_band"]),
               _ptr(t["fir_dec"]))
    elif case == "decimate_plan":
        h.call("frt_decimate_plan", INT_MAX, 2, _ptr(t["sos_dec"]))
    elif case == "gcc_phat_pairs":
        h.call("frt_gcc_set_pairs", 2**30, _ptr(np.array([0, 1], dtype=np.int32)), 1)
        h.call("frt_gcc_phat_pairs", _ptr(x), GCC_L, None, None, 0, u, u, st)
    elif case == "gcc_phat_frames":
        h.call("frt_gcc_phat_frames", _ptr(b["d0"]), _ptr(b["d1"]), GCC_L, GCC_L, 1, 2**30, u, 0, u, u, u, st)
    elif case == "spectrum_reduce_ticks":
        h.call("frt_spectrum_reduce_ticks", _ptr(p), env["nbins"], env["nbins"], 2**30, 1, 1, env["nbins"],
               0.5, u, None, None, u, u, st)
    elif case == "peer_alloc":
        ptr = ctypes.c_void_p()
        h.call("frt_peer_alloc", ctypes.c_size_t(2**50), ctypes.byref(ptr))


# at least the bytes of the allocation each case cannot make, from the code that sizes it
REQUEST = {
    "bank_plan": 4 * N_OCT * (2 * BPO + 6) * 2 * INT_MAX,      # the filter state
    "firbank_plan": 4 * INT_MAX * N_OCT * (512 - 1),           # the filter history at 512 taps
    "decimate_plan": 4 * 2 * 6 * 2 * INT_MAX,                  # the filter state of 2 stages
    "gcc_phat_pairs": 8 * 2**30 * (GCC_L // 2 + 1),            # the spectra of 2^30 channels
    "gcc_phat_frames": 2**30 * 4 * GCC_L,                      # one frame's raw rows of 2^30 pairs
    "spectrum_reduce_ticks": 4 * 2**30 * 513,                  # one tick's state rows of 2^30 channels
    "peer_alloc": 2**50,
}


@pytest.mark.gpu
@pytest.mark.parametrize("case", sorted(REQUEST))
def test_refused_allocation_leaves_handle_usable(env, case):
    from friture_b200._lib import FRT_ENOMEM, FrtError, Handle
    assert env["t"]["fir_band"].shape[1] == 512
    assert REQUEST[case] >= 2 * env["mem"], "the request must be far beyond the device's memory"
    ref, h = Handle(0), Handle(0)
    try:
        for hd in (ref, h):
            _plan(hd, env["t"])
        launches = h.launch_count
        with pytest.raises(FrtError) as ei:
            _refuse(h, case, env)
        assert ei.value.code == FRT_ENOMEM, str(ei.value)
        assert h.launch_count == launches
        got, want = _run(h, env), _run(ref, env)
        for name in want:
            assert np.array_equal(got[name].cpu().numpy(), want[name].cpu().numpy()), name
    finally:
        ref.close()
        h.close()
