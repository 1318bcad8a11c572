"""GPU: every route of the combined per-hop analysis (friture_b200.analyzer.ChannelAnalyzer) at every
geometry it takes, against each other on the whole output and against the oracle on distinct rows.

The routes: `process`, `process(overlap=True)`, `process_host` on pinned buffers (csrc/combined.cu:
H2D copies, both kernels and D2H copies pipelined over 1, 4, 8 or 16 time segments) and the same
stream fed to `process` in two calls.  The columns are the bits of `audioproc.stft` on the same
samples.  The band levels are the same bits on every route: the launches are cut at block boundaries
and the filterbank kernel is chosen from the plan and the block length alone, so any blocking of a
stream gives the same result (include/frt.h).  Then the calls the layer must refuse, before it queues
anything."""
import functools
import os
import sys
import zlib

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from parity import TOL, assert_logpower_parity, band_db_errors  # noqa: E402

pytestmark = pytest.mark.gpu

OCTAVE_CHOICES = (10, 9, 3)


def block_ok(hop, n_oct):
    """The filterbank's block rule, restated: a multiple of 256 samples whose tile (the longest of 1024,
    512 and 256 that divides it) is still even at the last of the n_oct - 1 halvings."""
    tile = 1024 if hop % 1024 == 0 else (512 if hop % 512 == 0 else 256)
    return hop > 0 and hop % 256 == 0 and (tile >> (n_oct - 1)) >= 1


# ---------------------------------------------------------------------------------------------- oracle
def oracle_bands(bank, x, hop, n_oct, response_time):
    """Band ENERGIES [C, B, nbands] (float64) of OctaveSpectrumOracle pushed one hop-sized block at a
    time per row, as the octave widget runs it (friture/octavespectrum.py:91-121)."""
    from oracle import friture_oracle as fo
    C, T = x.shape
    out = np.zeros((C, T // hop, bank.nbands))
    for c in range(C):
        orc = fo.OctaveSpectrumOracle(bank.bdec, bank.adec, bank.boct, bank.aoct,
                                      response_time=response_time, noctave=n_oct)
        for b in range(T // hop):
            out[c, b] = orc.push(x[c, b * hop:(b + 1) * hop].astype(np.float64))[0]
    return out


def weight_of(bank, weighting):
    """The dB offsets the library adds: the bank's table rounded to float32."""
    if weighting is None:
        return 0.0
    return np.asarray(getattr(bank, weighting), dtype=np.float32).astype(np.float64)


def check_oracle(an, x, spec, bands, rows, response_time, weighting):
    """spec / bands (numpy, all rows of x) against the float64 oracle on the given distinct rows."""
    from oracle import friture_oracle as fo
    xs = x[rows]
    if spec.shape[1]:
        ref = fo.log_spectrogram(fo.stft_power_batch(xs, an.fft_size, an.hop))
        assert_logpower_parity(spec[rows], ref)
    E = oracle_bands(an.bank, xs, an.hop, an.bank._n_octaves, response_time)
    e = band_db_errors(bands[rows], E, weight_of(an.bank, weighting))
    assert e["worst_ratio"] <= 1.0, e
    assert e["vector_rel"] < TOL, e
    return e


# ---------------------------------------------------------------------------------------------- inputs
def signal(C, T, seed):
    return (np.random.default_rng(seed).standard_normal((C, T)) * 0.1).astype(np.float32)


def device_rows(x, pad):
    """x as the first T columns of a device buffer whose row pitch is T + pad."""
    import torch
    C, T = x.shape
    buf = torch.full((C, T + pad), float("nan"), device="cuda")
    buf[:, :T] = torch.from_numpy(x).cuda()
    return buf[:, :T]


def host_rows(x, pad):
    """Same in pinned host memory."""
    import torch
    C, T = x.shape
    buf = torch.full((C, T + pad), float("nan")).pin_memory()
    buf[:, :T] = torch.from_numpy(x)
    return buf[:, :T]


def analyzer(C, N, hop, bpo=3, n_oct=10, response_time=1.0, weighting=None):
    from friture_b200.analyzer import ChannelAnalyzer
    return ChannelAnalyzer(C, fft_size=N, hop=hop, bandsperoctave=bpo, n_octaves=n_oct,
                           response_time=response_time, weighting=weighting)


def stft_bits(x_dev, N, hop):
    from friture_b200.audioproc import audioproc
    p = audioproc()
    p.set_fftsize(N)
    return p.stft(x_dev, hop=hop, log=True)


def run_routes(geom, x, pad, split=None):
    """(spec, bands) of every route on x [C, T] (numpy): dict route -> (spec or None, bands) as CPU
    tensors, after checking the columns against audioproc.stft bit for bit.

    The device routes give the bits of audioproc.stft on the same tensor.  The host route stages the
    samples as contiguous rows, so it gives the bits of audioproc.stft on a contiguous copy: at 4096
    and 8192 points the STFT picks its kernel from the frames' alignment (stft_large_kernel for 8-byte
    aligned frames, stft_multi_kernel otherwise), and the two round differently in the last bit."""
    import torch
    C, T = x.shape
    N, hop = geom["N"], geom["hop"]
    xd = device_rows(x, pad)
    xh = host_rows(x, pad)
    out = {}
    out["device"] = analyzer(C, **geom).process(xd)
    out["overlap"] = analyzer(C, **geom).process(xd, overlap=True)
    out["host"] = analyzer(C, **geom).process_host(xh)
    B = T // hop
    split = B // 2 if split is None else split
    an = analyzer(C, **geom)
    sa, ba = an.process(xd[:, :split * hop])
    sb, bb = an.process(xd[:, split * hop:])
    torch.cuda.synchronize()
    ref = stft_bits(xd, N, hop).cpu()
    for route in ("device", "overlap"):
        assert torch.equal(out[route][0].cpu(), ref), route
    assert torch.equal(out["host"][0], stft_bits(xd.contiguous(), N, hop).cpu()), "host"
    if N not in (4096, 8192) or pad % 2 == 0 or C == 1:
        assert torch.equal(out["host"][0], ref), "host"
    assert torch.equal(sa.cpu(), stft_bits(xd[:, :split * hop], N, hop).cpu())
    assert torch.equal(sb.cpu(), stft_bits(xd[:, split * hop:], N, hop).cpu())
    out["two calls"] = (None, torch.cat([ba, bb], 1))
    out = {k: (None if s is None else s.cpu(), b.cpu()) for k, (s, b) in out.items()}
    for route, (_, b) in out.items():
        assert torch.equal(b, out["device"][1]), "%s bands differ from the device route's" % route
    return out


# ---------------------------------------------------------------------------------------------- 1. geometry grid
GEOMETRIES = [(2048, 1024), (32, 256), (256, 256), (1024, 2048), (4096, 1024), (8192, 512), (16384, 256),
              (2048, 768), (4096, 1536)]
BPOS = (1, 3, 6, 12, 24)
WEIGHTINGS = (None, "A", "C")
CHANNELS = (1, 3, 7)
PADS = (0, 1, 2, 5, 6)           # row pitch T + pad: T is a multiple of 256, so pitch = pad (mod 4)


def grid():
    """Two cases per (N, hop); across them every bpo, octave count the hop allows, response time,
    weighting, channel count and row pitch (mod 4) appears."""
    cases = []
    for i, (N, hop) in enumerate(GEOMETRIES):
        octs = [o for o in OCTAVE_CHOICES if block_ok(hop, o)]
        for j in range(2):
            k = 2 * i + j
            cases.append(dict(N=N, hop=hop, bpo=BPOS[k % 5], n_oct=octs[k % len(octs)],
                              response_time=(0.025, 5.0)[j], weighting=WEIGHTINGS[k % 3],
                              C=CHANNELS[(i + j) % 3], pad=PADS[k % 5]))
    return cases


def grid_id(c):
    return "N%d-hop%d-bpo%d-oct%d-T%g-%s-C%d-pad%d" % (c["N"], c["hop"], c["bpo"], c["n_oct"], c["response_time"],
                                                       c["weighting"] or "flat", c["C"], c["pad"])


def test_grid_covers_the_issue_axes():
    cases = grid()
    assert {c["bpo"] for c in cases} == set(BPOS)
    assert {c["n_oct"] for c in cases} == set(OCTAVE_CHOICES)
    assert {c["weighting"] for c in cases} == set(WEIGHTINGS)
    assert {c["C"] for c in cases} == set(CHANNELS)
    assert {(c["N"], c["hop"]) for c in cases} == set(GEOMETRIES)
    assert {c["pad"] % 4 for c in cases if c["C"] > 1} >= {1, 2}


@pytest.mark.parametrize("case", grid(), ids=grid_id)
def test_routes_agree_and_match_oracle(case):
    case = dict(case)
    C, pad = case.pop("C"), case.pop("pad")
    N, hop = case["N"], case["hop"]
    hops = -(-N // hop) + 5                  # at least 6 columns (for N <= hop) past the first one
    x = signal(C, hops * hop, seed=zlib.crc32(grid_id(dict(case, C=C, pad=pad)).encode()))
    out = run_routes(case, x, pad)
    spec, bands = out["device"]
    assert tuple(spec.shape) == (C, (hops * hop - N) // hop + 1, N // 2 + 1)
    assert tuple(bands.shape) == (C, hops, case["bpo"] * case["n_oct"])
    an = analyzer(1, **case)
    check_oracle(an, x, spec.numpy(), bands.numpy(), list(range(C)), case["response_time"], case["weighting"])


# ---------------------------------------------------------------------------------------------- 2. host segmentation
@pytest.mark.parametrize("n_blocks", [1, 3, 7, 8, 63, 64, 127, 128, 129, 143, 256])
def test_host_segments_match_device_and_carry_state(n_blocks):
    """nseg 1, 4, 8 and 16, ragged last segments and empty trailing ones (129 blocks: 16 segments of
    9 with the last one empty); a second call continues bit-equal on both routes."""
    import torch
    geom = dict(N=2048, hop=1024)
    C, pad = 3, 1
    x = signal(C, 2 * n_blocks * 1024, seed=n_blocks)
    halves = (x[:, :n_blocks * 1024], x[:, n_blocks * 1024:])
    dev, host = analyzer(C, **geom), analyzer(C, **geom)
    got = []
    for part in halves:
        sd, bd = dev.process(device_rows(part, pad))
        sh, bh = host.process_host(host_rows(part, pad))
        assert torch.equal(sh, sd.cpu()) and torch.equal(bh, bd.cpu())
        assert torch.equal(sh, stft_bits(device_rows(part, 0), 2048, 1024).cpu())
        got.append(bh)
    if n_blocks in (1, 129):
        # the second call's bands carry the first call's state: both against one oracle run
        check_oracle(analyzer(1, **geom), x, np.zeros((C, 0, 1025), np.float32), torch.cat(got, 1).numpy(),
                     [0, 2], 1.0, None)


@pytest.mark.parametrize("N,hop,n_blocks,n_oct", [(16384, 256, 3, 9), (16384, 256, 129, 9), (4096, 1024, 2, 10)])
def test_host_columns_straddle_segments(N, hop, n_blocks, n_oct):
    """T < N (bands, no columns), and 16384-point columns spanning many of the 16 segments."""
    geom = dict(N=N, hop=hop, n_oct=n_oct)
    C = 3
    x = signal(C, n_blocks * hop, seed=N + n_blocks)
    out = run_routes(geom, x, pad=2)
    assert out["host"][0].shape[1] == max(0, (n_blocks * hop - N) // hop + 1)
    check_oracle(analyzer(1, **geom), x, out["device"][0].numpy(), out["device"][1].numpy(), [0, 2], 1.0, None)


# ---------------------------------------------------------------------------------------------- 3. the bench's shape
def test_bench_shape_every_channel_and_hop():
    """C = 1024, N = 2048, hop 1024, 10 octaves, 129 hops: device, overlapped and host routes equal on
    every channel and hop, and the oracle on channels 0, 1, 511 and 1023 over all 129 hops."""
    import torch
    C, hops = 1024, 129
    x = signal(C, hops * 1024, seed=7)
    geom = dict(N=2048, hop=1024)
    xd = torch.from_numpy(x).cuda()
    sd, bd = analyzer(C, **geom).process(xd)
    so, bo = analyzer(C, **geom).process(xd, overlap=True)
    xh = torch.from_numpy(x).pin_memory()
    sh, bh = analyzer(C, **geom).process_host(xh)
    torch.cuda.synchronize()
    assert torch.equal(so, sd) and torch.equal(bo, bd)
    sd, bd = sd.cpu(), bd.cpu()
    assert torch.equal(sh, sd) and torch.equal(bh, bd)
    rows = [0, 1, 511, 1023]
    e = check_oracle(analyzer(1, **geom), x, sd.numpy(), bd.numpy(), rows, 1.0, None)
    assert e["vector_rel"] < 1e-5


@functools.lru_cache(maxsize=None)
def three_rows():
    x = signal(3, 129 * 1024, seed=11)
    an = analyzer(1, 2048, 1024)
    return x, oracle_bands(an.bank, x, 1024, 10, 1.0)


def distinct(out, k):
    """out[:k] (numpy) after checking that channel c equals channel c % k bit for bit."""
    import torch
    idx = torch.arange(out.shape[0], device=out.device) % k
    assert torch.equal(out, out[idx]), "repeated rows differ"
    return out[:k].cpu().numpy()


@pytest.mark.parametrize("C", [1536, 1537, 3072, 3073])
def test_dispatch_threshold_channel_counts(C):
    """Channel counts at the filterbank's kernel switches (three-warp below 1536, two channels per lane
    above 3072): three seeded rows repeated, every repeat bit-equal, on the device and host routes."""
    import torch
    base, E = three_rows()
    geom = dict(N=2048, hop=1024)
    xd = torch.from_numpy(base).cuda().repeat((C + 2) // 3, 1)[:C].contiguous()
    sd, bd = analyzer(C, **geom).process(xd)
    sh, bh = analyzer(C, **geom).process_host(xd.cpu().pin_memory())
    torch.cuda.synchronize()
    assert torch.equal(sh, sd.cpu()) and torch.equal(bh, bd.cpu())
    d = distinct(bd, 3)
    distinct(sd, 3)
    e = band_db_errors(d, E)
    assert e["worst_ratio"] <= 1.0 and e["vector_rel"] < TOL, e
    del xd, sd, bd, sh, bh


# ---------------------------------------------------------------------------------------------- 4. refusals
def nan_like(shape, pinned=False, device=None):
    import torch
    t = torch.full(shape, float("nan"), device=device)
    return t.pin_memory() if pinned else t


def untouched(*ts):
    import torch
    torch.cuda.synchronize()
    return all(bool(torch.isnan(t).all()) for t in ts)


C0, HOPS = 3, 9
T0 = HOPS * 1024
F0 = (T0 - 2048) // 1024 + 1


def host_case(name):
    """(x_host, spec_host, bands_host) for process_host: one of them wrong as `name` says."""
    import torch
    x = torch.from_numpy(signal(C0, T0, 21)).pin_memory()
    spec = nan_like((C0, F0, 1025), pinned=True)
    bands = nan_like((C0, HOPS, 30), pinned=True)
    if name == "x-float64-numpy":
        x = x.numpy().astype(np.float64)
    elif name == "x-float64-tensor":
        x = x.double()
    elif name == "x-cuda":
        x = x.cuda()
    elif name == "x-not-contiguous-along-time":
        x = torch.from_numpy(np.ascontiguousarray(x.numpy().T)).t()
    elif name == "x-one-dimensional":
        x = x[0]
    elif name == "spec-one-frame-more":
        spec = nan_like((C0, F0 + 1, 1025), pinned=True)
    elif name == "spec-one-frame-less":
        spec = nan_like((C0, F0 - 1, 1025), pinned=True)
    elif name == "spec-float64":
        spec = spec.double()
    elif name == "spec-cuda":
        spec = spec.cuda()
    elif name == "bands-one-channel-less":
        bands = nan_like((C0 - 1, HOPS, 30), pinned=True)
    elif name == "bands-32-wide-view":
        bands = nan_like((C0, HOPS, 32), pinned=True)[..., :30]
    elif name == "bands-cuda":
        bands = bands.cuda()
    return x, spec, bands


HOST_CASES = ["x-float64-numpy", "x-float64-tensor", "x-cuda", "x-not-contiguous-along-time", "x-one-dimensional",
              "spec-one-frame-more", "spec-one-frame-less", "spec-float64", "spec-cuda", "bands-one-channel-less",
              "bands-32-wide-view", "bands-cuda"]


def fresh_bits(x):
    """(spec, bands) of a fresh analyzer on x (CPU float32 [C0, T0]), both routes."""
    import torch
    d = analyzer(C0, 2048, 1024).process(x.cuda())
    h = analyzer(C0, 2048, 1024).process_host(x.pin_memory())
    torch.cuda.synchronize()
    return d, h


def check_next_call_is_fresh(an):
    import torch
    x = torch.from_numpy(signal(C0, T0, 22))
    (sd, bd), (sh, bh) = fresh_bits(x)
    s2, b2 = an.process(x.cuda())
    assert torch.equal(s2, sd) and torch.equal(b2, bd)
    an.bank.reset()
    s3, b3 = an.process_host(x.pin_memory())
    assert torch.equal(s3, sh) and torch.equal(b3, bh)


@pytest.mark.parametrize("name", HOST_CASES)
def test_process_host_refuses_wrong_buffers(name):
    from friture_b200._lib import FrtError
    an = analyzer(C0, 2048, 1024)
    x, spec, bands = host_case(name)
    n0 = an.handle.launch_count
    with pytest.raises(ValueError) as info:
        an.process_host(x, spec, bands)
    assert not isinstance(info.value, FrtError) or info.value.code == -1
    assert an.handle.launch_count == n0
    assert untouched(spec, bands)
    check_next_call_is_fresh(an)


def device_case(name):
    """(x, spec, bands) for process: one of them wrong as `name` says."""
    import torch
    x = torch.from_numpy(signal(C0, T0, 23)).cuda()
    spec = nan_like((C0, F0, 1025), device="cuda")
    bands = nan_like((C0, HOPS, 30), device="cuda")
    if name == "bands-32-wide-view":
        bands = nan_like((C0, HOPS, 32), device="cuda")[..., :30]
    elif name == "bands-one-channel-less":
        bands = nan_like((C0 - 1, HOPS, 30), device="cuda")
    elif name == "bands-one-hop-less":
        bands = nan_like((C0, HOPS - 1, 30), device="cuda")
    elif name == "bands-one-band-more":
        bands = nan_like((C0, HOPS, 31), device="cuda")
    elif name == "bands-cpu":
        bands = nan_like((C0, HOPS, 30))
    elif name == "bands-float64":
        bands = bands.double()
    elif name == "bands-transposed-hops":
        bands = nan_like((HOPS, C0, 30), device="cuda").transpose(0, 1)
    elif name == "spec-cpu":
        spec = nan_like((C0, F0, 1025))
    elif name == "spec-one-frame-more":
        spec = nan_like((C0, F0 + 1, 1025), device="cuda")
    return x, spec, bands


DEVICE_CASES = ["bands-32-wide-view", "bands-one-channel-less", "bands-one-hop-less", "bands-one-band-more",
                "bands-cpu", "bands-float64", "bands-transposed-hops", "spec-cpu", "spec-one-frame-more"]


@pytest.mark.parametrize("overlap", [False, True])
@pytest.mark.parametrize("name", DEVICE_CASES)
def test_process_refuses_wrong_outputs(name, overlap):
    an = analyzer(C0, 2048, 1024)
    x, spec, bands = device_case(name)
    n0 = an.handle.launch_count
    with pytest.raises(ValueError):
        an.process(x, spec, bands, overlap=overlap)
    assert an.handle.launch_count == n0
    assert untouched(spec, bands)
    check_next_call_is_fresh(an)


def test_process_sharded_refuses_wrong_bands_before_any_work():
    an = analyzer(C0, 2048, 1024)
    x, _, bands = device_case("bands-one-channel-less")
    n0 = an.handle.launch_count
    with pytest.raises(ValueError):
        an.process_sharded(x[:, :8 * 1024 + 1024], bands=bands[:, :9], n_chunks=1, transport="nccl")
    assert an.handle.launch_count == n0
    assert untouched(bands)


@pytest.mark.parametrize("hop", [768, 384, 256, 2304])
def test_analyzer_refuses_a_hop_the_bank_cannot_block(hop):
    """At 10 octaves a block's tile (the longest of 1024, 512 and 256 that divides it) must hold 512
    samples: 768, 256 and 2304 only divide by 256, which 9 octaves take; 384 is no multiple of 256."""
    with pytest.raises(ValueError):
        analyzer(C0, 2048, hop)
    if hop % 256 == 0:
        analyzer(C0, 2048, hop, n_oct=9)
    for ok in (512, 1536, 2560):
        analyzer(C0, 2048, ok)


def c_call(an, x, spec, bands, C=C0, T=T0, hop=1024, nbands=30, x_stride=None):
    from friture_b200 import _lib
    an.handle.call("frt_combined_process_host", _lib._ptr(x), int(T if x_stride is None else x_stride), int(C),
                   int(T), int(hop), _lib._ptr(spec), _lib._ptr(bands), int(nbands), 1)


C_CASES = {
    "nbands-larger-than-plan": dict(nbands=32),
    "nbands-smaller-than-plan": dict(nbands=29),
    "fewer-channels-than-plan": dict(C=C0 - 1),
    "more-channels-than-plan": dict(C=C0 + 1),
    "hop-768-at-10-octaves": dict(hop=768, T=12 * 768),
    "hop-384": dict(hop=384, T=24 * 384),
}


@pytest.mark.parametrize("name", list(C_CASES))
def test_c_entry_refuses_before_queueing(name):
    """frt_combined_process_host against its plans: FRT_EINVAL before any copy, kernel or output write.
    The buffers are large enough for every argument set (a call that was not refused stays in bounds)."""
    from friture_b200 import _lib
    an = analyzer(C0, 2048, 1024)
    an.proc._ensure_plan()
    an.bank._ensure_plan(C0)
    kw = C_CASES[name]
    C, T, nb = kw.get("C", C0), kw.get("T", T0), kw.get("nbands", 30)
    x = nan_like((C0 + 1, 24 * 1024), pinned=True)
    x[:] = torch_from(signal(C0 + 1, 24 * 1024, 24))
    spec = nan_like((C0 + 1, 24, 1025), pinned=True)
    bands = nan_like((C0 + 1, 24, 32), pinned=True)
    n0 = an.handle.launch_count
    with pytest.raises(_lib.FrtValueError) as info:
        c_call(an, x, spec, bands, C=C, T=T, hop=kw.get("hop", 1024), nbands=nb, x_stride=24 * 1024)
    assert info.value.code == _lib.FRT_EINVAL
    assert an.handle.launch_count == n0
    assert untouched(spec, bands)
    check_next_call_is_fresh(an)


def torch_from(a):
    import torch
    return torch.from_numpy(a)


def test_stft_refuses_out_on_another_device():
    import torch
    from friture_b200.audioproc import audioproc
    p = audioproc()
    p.set_fftsize(2048)
    x = torch.from_numpy(signal(2, 4 * 1024, 25)).cuda()
    out = nan_like((2, 3, 1025))
    n0 = p.handle.launch_count
    with pytest.raises(ValueError):
        p.stft(x, hop=1024, out=out)
    assert p.handle.launch_count == n0 and untouched(out)


@pytest.mark.parametrize("name", ["x-float64-tensor", "x-cuda", "x-not-contiguous-along-time", "out-float64",
                                  "out-one-frame-more", "out-cuda", "out-not-contiguous"])
def test_stft_host_refuses_wrong_buffers(name):
    import torch
    from friture_b200.audioproc import audioproc
    p = audioproc()
    p.set_fftsize(2048)
    x = torch.from_numpy(signal(2, 4 * 1024, 26)).pin_memory()
    out = nan_like((2, 3, 1025), pinned=True)
    if name == "x-float64-tensor":
        x = x.double()
    elif name == "x-cuda":
        x = x.cuda()
    elif name == "x-not-contiguous-along-time":
        x = torch.from_numpy(np.ascontiguousarray(x.numpy().T)).t()
    elif name == "out-float64":
        out = out.double()
    elif name == "out-one-frame-more":
        out = nan_like((2, 4, 1025), pinned=True)
    elif name == "out-cuda":
        out = out.cuda()
    elif name == "out-not-contiguous":
        out = nan_like((2, 1025, 3), pinned=True).transpose(1, 2)
    n0 = p.handle.launch_count
    with pytest.raises(ValueError):
        p.stft_host(x, hop=1024, out=out)
    assert p.handle.launch_count == n0 and untouched(out)
    good = p.stft_host(torch.from_numpy(signal(2, 4 * 1024, 26)), hop=1024)
    assert torch.equal(good, p.stft(torch.from_numpy(signal(2, 4 * 1024, 26)).cuda(), hop=1024).cpu())
