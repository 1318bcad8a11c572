"""GPU: ``SpectrumAnalyzer.handle_new_data`` -- the spectrum widget fed from stream chunks, each frame's
power column smoothed on chip (``frt_spectrum_frames`` / ``_dual``).

The yardstick is ``process`` on the frames the widget's framing cuts, one tick at a time: the rows,
both indices and both carried states must be the same bits, at every FFT size (so every STFT kernel
family), single and dual, every weighting, frame offsets of every alignment class, and chunkings from
one sample to the whole stream; the entry points called directly on frames of every alignment class
(16-, 8- and 4-byte: every kernel family, with and without TMA and vector loads).  Then the widget oracle over a stream with every setter in mid-stream,
the edge cases, the refusals, the plot, and stream order on the caller's stream."""
import dataclasses
from ctypes import c_float

import numpy as np
import pytest
import torch

from friture_b200 import _lib
from friture_b200.plotcurves import SpectrumPlot
from friture_b200.spectrum import SpectrumAnalyzer, SpectrumTicks
from friture_b200.stream import StreamFramer
from oracle import friture_oracle as fo
from oracle.spectrum_dual import DualSpectrumWidgetOracle

pytestmark = pytest.mark.gpu

FFT_SIZES = [2 ** k for k in range(5, 15)]


def stream(C, pairs, n, seed):
    g = torch.Generator().manual_seed(seed)
    t = torch.arange(n, dtype=torch.float64)
    f = 440. + 1000. * torch.rand(C, 1, generator=g, dtype=torch.float64)
    x = 0.3 * torch.sin(2 * np.pi * f * t / 48000.) + 0.05 * torch.randn(C, n, generator=g, dtype=torch.float64)
    if pairs:
        y = 0.5 * torch.roll(x, 17, dims=1) + 0.02 * torch.randn(C, n, generator=g, dtype=torch.float64)
        x = torch.stack([x, y], dim=1)
    return x.float().cuda()


class ProcessTwin:
    """The same widget through ``process``: its own framer over the same chunks, one call per tick."""

    def __init__(self, C, pairs, **kw):
        self.a = SpectrumAnalyzer(C, **kw)
        self.pairs = pairs
        self.rows = 2 * C if pairs else C
        self.fr = None

    def tick(self, x):
        a = self.a
        if self.fr is None:
            self.fr = StreamFramer(self.rows, a.fft_size, a.hop, x.device, history=16384)
        self.fr.push(x.reshape(self.rows, x.shape[-1]))
        view, F = self.fr.take()
        if F == 0:
            return None
        T = (F - 1) * a.hop + a.fft_size
        v = view[:, :T]
        if self.pairs:
            v = v.reshape(a.n_channels, 2, T)
        db, fmax, fpitch = a.process(v)
        return db.clone(), fmax, fpitch, F

    def setfftsize(self, n):
        self.a.setfftsize(n)
        if self.fr is not None:
            self.fr.set_geometry(n, self.a.hop)


def same_state(a, b):
    for s, t in ((a._disp, b._disp), (a._disp2, b._disp2)):
        assert (s is None) == (t is None)
        if s is not None:
            assert torch.equal(s, t)


def feed_and_compare(a, twin, x, chunks, buffer=None):
    """Push x in the given chunk sizes into a (handle_new_data) and the twin (one process per tick)."""
    pos = 0
    rows = 0
    for n in chunks:
        c = x[..., pos:pos + n]
        pos += n
        out = a.handle_new_data(c, buffer=buffer)
        b = n if buffer is None else buffer
        want = [twin.tick(c[..., i * b:(i + 1) * b]) for i in range(n // b)] if n else [twin.tick(c)]
        ticks = [i for i, w in enumerate(want) if w is not None]
        assert list(out.tick) == ticks
        for r, i in enumerate(ticks):
            db, fmax, fpitch, F = want[i]
            assert out.n_frames[r] == F
            assert torch.equal(out.db[:, r], db), "tick %d dB" % i
            assert np.array_equal(out.fmax_hz[r], fmax) and np.array_equal(out.fpitch_hz[r], fpitch)
        rows += len(ticks)
        same_state(a, twin.a)
    assert pos == x.shape[-1]
    return rows


def chunkings(N, L):
    hop = N // 4
    out = {"whole": [L], "512": [512] * (L // 512) + [L % 512], "4097": [4097] * (L // 4097) + [L % 4097]}
    if N <= 256:
        out["1"] = [1] * L
    else:   # one-sample chunks over the first frames only; the rest in 777s
        k = min(L, N + 2 * hop)
        out["1"] = [1] * k + [777] * ((L - k) // 777) + [(L - k) % 777]
    return out


@pytest.mark.parametrize("dual", [False, True])
@pytest.mark.parametrize("N", FFT_SIZES)
def test_bits_equal_process_per_tick(N, dual):
    """Every chunking of the same stream, one tick per call, with C in {1, 3, 64} and every weighting.
    The framer's view here is 16-byte aligned below N = 16384; test_entry_points_at_every_alignment
    covers the other alignment classes."""
    L = 2 * N + 9 * (N // 4) + 131
    for k, (name, ch) in enumerate(sorted(chunkings(N, L).items())):
        C = (1, 3, 64, 3)[k % 4]
        w = k % 4
        x = stream(C, dual, L, seed=N + k)
        kw = dict(fft_size=N, weighting=w, response_time=0.05 + 0.3 * k, dual_channels=dual)
        a = SpectrumAnalyzer(C, **kw)
        twin = ProcessTwin(C, dual, **kw)
        assert feed_and_compare(a, twin, x, ch) > 0, name


@pytest.mark.parametrize("N", [32, 256, 2048, 4096, 8192, 16384])
def test_single_mode_on_pairs_decays_the_second_state(N):
    """[C, 2, n] in single mode reads the reference rows; after a dual stretch the second state decays
    by (1 - alpha)^frames per tick, as process does it."""
    C, L = 3, 3 * N + 1001
    x = stream(C, True, L, seed=7)
    a = SpectrumAnalyzer(C, fft_size=N, dual_channels=True, weighting=2)
    twin = ProcessTwin(C, True, fft_size=N, dual_channels=True, weighting=2)
    half = L // 2
    feed_and_compare(a, twin, x[..., :half], [half // 3, half - half // 3])
    a.setdualchannels(False)
    twin.a.setdualchannels(False)
    first = min(1000, (L - half) // 2)
    feed_and_compare(a, twin, x[..., half:], [first, L - half - first])


@pytest.mark.parametrize("dual", [False, True])
@pytest.mark.parametrize("N", [64, 2048, 8192, 16384])
@pytest.mark.parametrize("b", [1, 480, 512])
def test_buffers_in_one_call_are_the_same_bits_as_separate_calls(N, dual, b):
    C = 5
    L = b * ((3 * N) // b + 3)
    x = stream(C, dual, L, seed=b)
    a1 = SpectrumAnalyzer(C, fft_size=N, dual_channels=dual, weighting=1)
    a2 = SpectrumAnalyzer(C, fft_size=N, dual_channels=dual, weighting=1)
    out = a1.handle_new_data(x, buffer=b)
    per = [a2.handle_new_data(x[..., i * b:(i + 1) * b]) for i in range(L // b)]
    ticks = [i for i, p in enumerate(per) if len(p.tick)]
    assert list(out.tick) == ticks
    for r, i in enumerate(ticks):
        assert torch.equal(out.db[:, r], per[i].db[:, 0])
        assert np.array_equal(out.fmax_hz[r], per[i].fmax_hz[0])
        assert np.array_equal(out.fpitch_hz[r], per[i].fpitch_hz[0])
        assert out.n_frames[r] == per[i].n_frames[0]
    same_state(a1, a2)
    assert a1.old_index == a2.old_index


def test_against_the_widget_oracle_with_every_setter_in_mid_stream():
    """The reference's handle_new_data logic (old_index, realizable, zeros before the stream) over a
    chunked stream, in float64, with the FFT size, response time, weighting, dual mode and frequency
    range changed in mid-stream; the tolerances of the analyzer's end-to-end checks."""
    C, L = 2, 48000
    x = stream(C, True, L, seed=3).cpu().double().numpy()
    a = SpectrumAnalyzer(C, fft_size=1024, dual_channels=True)
    old_index = 0
    offset = 0
    N = 1024

    def oracles(N, rt, w, dual):
        return [DualSpectrumWidgetOracle(N, response_time=rt, weight=w, dual_channels=dual) for _ in range(C)]

    rt, wsel, dual = 0.025, 0, True
    orc = oracles(N, rt, None, dual)
    plan = {6000: ("fft", 4096), 12000: ("rt", 0.5), 20000: ("w", 1), 26000: ("dual", False),
            31000: ("fft", 512), 36000: ("minmax", (100., 5000.)), 41000: ("dual", True)}
    pos, step = 0, 1000
    history = np.zeros((C, 2, 16384))
    while pos < L:
        if pos in plan:
            what, v = plan[pos]
            keep = [(o.disp, o.disp2) for o in orc]
            if what == "fft":
                N = v
                a.setfftsize(N)
                orc = oracles(N, rt, None, dual)                 # the widget restarts both states
            elif what == "rt":
                rt = v
                a.setresponsetime(v)
                orc = oracles(N, rt, None, dual)
                for o, (d1, d2) in zip(orc, keep):
                    o.disp, o.disp2 = d1, d2
            elif what == "w":
                wsel = v
                a.setweighting(v)
            elif what == "dual":
                dual = v
                a.setdualchannels(v)
                for o in orc:
                    o.setdualchannels(v)
            elif what == "minmax":
                a.setMinMaxFreq(*v)
                for o in orc:
                    o.disp = np.zeros_like(o.disp)
                    o.disp2 = np.zeros_like(o.disp2)
        chunk = x[..., pos:pos + step]
        pos += step
        history = np.concatenate([history, chunk], axis=-1)
        offset += step
        out = a.handle_new_data(torch.from_numpy(chunk).float().cuda())
        hop = N // 4
        realizable = (offset - old_index) // hop
        if realizable == 0:
            assert len(out.tick) == 0
            continue
        start = old_index - N                                # the first frame ends at old_index
        base = offset - history.shape[-1]                    # stream index of history[..., 0]
        seg = history[..., start - base:start - base + (realizable - 1) * hop + N]
        old_index += realizable * hop
        A, B, Cw = a.proc.get_freq_weighting()
        w = [0. * A, A, B, Cw][wsel]
        assert list(out.tick) == [0]
        for c in range(C):
            orc[c].w = w
            res = orc[c].tick(seg[c] if dual else seg[c, :1])
            db_ref, fmax, fpitch, i, pitch = res
            got = out.db[c, 0].cpu().double().numpy()
            assert np.max(np.abs(got - db_ref)) < 0.05, "tick at %d ch %d" % (pos, c)
            assert abs(a._disp[c].cpu().double().numpy() - orc[c].disp).max() <= \
                1e-4 * max(orc[c].disp.max(), 1e-30)
            peak = int(round(out.fmax_hz[0, c] / (48000 / N)))
            assert out.fmax_hz[0, c] == fmax or db_ref.max() - db_ref[peak] < 0.05
            hps = fo.harmonic_product_spectrum(orc[c].disp)
            ip = int(round(out.fpitch_hz[0, c] / (48000 / N)))
            assert out.fpitch_hz[0, c] == fpitch or hps[ip] >= hps.max() * (1 - 1e-3), "pitch at %d" % pos
        history = history[..., -16384 - 4096:]


# ---- the entry points on frames of every alignment class ---------------------------------------------
# (sample offset of row 0, row pitch mod 4) -> how far every frame is aligned: 16, 8 or 4 bytes.  In dual
# mode x2 = x + pitch and the pair stride is 2 pitch, as handle_new_data passes them.
ALIGNMENTS = {16: (0, 0), 8: (2, 2), 4: (1, 1)}
TICKS = [1, 2, 1, 3, 5, 1]     # frames per tick: ends 1, 3, 4, 7, 12, 13


def direct_case(N, C, dual, align, want_db, seed):
    """frt_spectrum_frames(_dual) once over all the ticks against frt_stft_process(POWER) + frt_spectrum_reduce
    (_dual) one tick at a time on the same frames: the same bits in every row, index and state."""
    h = _lib.default_handle()
    h.call("frt_stft_plan", N)
    hop, nb, nf, R = N // 4, N // 2 + 1, sum(TICKS), len(TICKS)
    off, pmod = ALIGNMENTS[align]
    T = (nf - 1) * hop + N
    pitch = (T + 3) // 4 * 4 + pmod
    rows = 2 * C if dual else C
    g = torch.Generator(device="cuda").manual_seed(seed)
    base = torch.randn(rows * pitch + 4, device="cuda", generator=g) * 0.2
    x = base.data_ptr() + 4 * off
    w = torch.from_numpy(np.ascontiguousarray(SpectrumAnalyzer(1, fft_size=N, handle=h, weighting=1).w,
                                              dtype=np.float32)).cuda()
    alpha = c_float(0.3)
    d0 = [torch.rand(C, nb, device="cuda", generator=g) * 1e-3 for _ in range(2)]
    ends = torch.tensor(np.cumsum(TICKS), dtype=torch.int32, device="cuda")
    sp = _lib.current_stream_ptr()

    disp = [d.clone() for d in d0]
    db = torch.full((C, R, nb), float("nan"), device="cuda") if want_db else None
    imax = torch.full((R, C), -1, dtype=torch.int32, device="cuda")
    ipitch = torch.full((R, C), -1, dtype=torch.int32, device="cuda")
    if dual:
        h.call("frt_spectrum_frames_dual", _lib._ptr(x), _lib._ptr(x + 4 * pitch), 2 * pitch, C, nf, hop,
               _lib._ptr(ends), R, alpha, _lib._ptr(disp[0]), _lib._ptr(disp[1]), _lib._ptr(db), R * nb, nb,
               _lib._ptr(imax), _lib._ptr(ipitch), sp)
    else:
        h.call("frt_spectrum_frames", _lib._ptr(x), pitch, C, nf, hop, _lib._ptr(ends), R, alpha,
               _lib._ptr(disp[0]), _lib._ptr(w), _lib._ptr(db), R * nb, nb, _lib._ptr(imax), _lib._ptr(ipitch), sp)

    ref = [d.clone() for d in d0]
    f0 = 0
    for r, k in enumerate(TICKS):
        power = torch.empty((rows, k, nb), device="cuda")
        h.call("frt_stft_process", _lib._ptr(x + 4 * f0 * hop), pitch, rows, k, hop, _lib._ptr(power), k * nb, nb,
               _lib.STFT_POWER, sp)
        rdb = torch.empty((C, nb), device="cuda")
        ri = torch.empty(C, dtype=torch.int32, device="cuda")
        rp = torch.empty(C, dtype=torch.int32, device="cuda")
        if dual:   # pair c: reference row 2c, measurement row 2c + 1
            p = power.data_ptr()
            h.call("frt_spectrum_reduce_dual", _lib._ptr(p), _lib._ptr(p + 4 * k * nb), 2 * k * nb, nb, C, k, nb,
                   alpha, _lib._ptr(ref[0]), _lib._ptr(ref[1]), _lib._ptr(rdb), _lib._ptr(ri), _lib._ptr(rp), sp)
        else:
            h.call("frt_spectrum_reduce", _lib._ptr(power), k * nb, nb, C, k, nb, alpha, _lib._ptr(ref[0]),
                   _lib._ptr(w), _lib._ptr(rdb), _lib._ptr(ri), _lib._ptr(rp), sp)
        where = "N %d C %d dual %s align %d tick %d" % (N, C, dual, align, r)
        if want_db:
            assert torch.equal(db[:, r], rdb), where
        assert torch.equal(imax[r], ri) and torch.equal(ipitch[r], rp), where
        f0 += k
    assert torch.equal(disp[0], ref[0])
    assert torch.equal(disp[1], ref[1] if dual else d0[1])


@pytest.mark.parametrize("align", [16, 8, 4])
@pytest.mark.parametrize("dual", [False, True])
@pytest.mark.parametrize("N", FFT_SIZES)
def test_entry_points_at_every_alignment(N, dual, align):
    """16-byte frames take the TMA path at N = 2048 and the large kernel at 4096 / 8192; 8-byte frames the
    plain small kernel at 2048; 4-byte frames the scalar loads of the small kernel and the multi kernel at
    4096 / 8192.  Ticks of 1 to 5 frames; without the dB rows once per size."""
    direct_case(N, 3, dual, align, want_db=align != 8, seed=N + align)


@pytest.mark.parametrize("dual", [False, True])
@pytest.mark.parametrize("N", [64, 2048, 4096, 8192, 16384])
def test_entry_points_with_more_channels_than_slots(N, dual):
    """1100 channels (pairs): more than the warps, frame groups or CTAs of one launch, so slots walk
    several channels in turn."""
    for k, align in enumerate((16, 4)):
        direct_case(N, 1100, dual, align, want_db=True, seed=N + k)


def test_silence_ties_and_no_frame_calls():
    N, C = 2048, 4
    a = SpectrumAnalyzer(C, fft_size=N)
    out = a.handle_new_data(torch.zeros(C, 100, device="cuda"))
    assert len(out.tick) == 0 and out.db.shape == (C, 0, N // 2 + 1) and a._disp is None
    out = a.handle_new_data(torch.zeros(C, 5000, device="cuda"), buffer=500)
    assert len(out.tick) == 9 and out.n_frames.sum() * 512 == a.old_index       # buffer 8 cuts no frame
    assert list(out.tick) == [0, 1, 2, 3, 4, 5, 6, 7, 9] and torch.all(out.db == out.db[0, 0, 0])
    # silence: every bin ties, the first bin wins
    assert np.all(out.fmax_hz == 0.) and np.all(out.fpitch_hz == 1e-20)
    assert torch.all(a._disp == 0)


@pytest.mark.parametrize("dual", [False, True])
def test_refusals_leave_the_analyzer_usable(dual):
    C, N = 3, 256
    a = SpectrumAnalyzer(C, fft_size=N, dual_channels=dual)
    twin = ProcessTwin(C, dual, fft_size=N, dual_channels=dual)
    x = stream(C, dual, 4000, seed=11)
    feed_and_compare(a, twin, x[..., :1000], [1000])
    long = torch.zeros(x.shape[:-1] + (64 * 8193,), device="cuda")                 # one tick of 8193 frames
    for bad, kw in ((x[..., :100], dict(buffer=7)), (long, {}),
                    (x[:, 0] if dual else torch.stack([x, x], 1), {}), (x[:2], {}), (x.cpu(), {})):
        with pytest.raises(ValueError):
            a.handle_new_data(bad, **kw)
    feed_and_compare(a, twin, x[..., 1000:], [1500, 1500])


def test_plot_takes_the_ticks():
    C, N = 2, 1024
    a = SpectrumAnalyzer(C, fft_size=N)
    ticks = a.handle_new_data(stream(C, False, 8 * 512, seed=5), buffer=512)
    assert isinstance(ticks, SpectrumTicks) and len(ticks.tick) == 8
    p = SpectrumPlot(C)
    got = p.push_ticks(ticks)
    q = SpectrumPlot(C)
    for r in range(len(ticks.tick)):
        want = q.push(ticks.db[:, r], ticks.fmax_hz[r], ticks.fpitch_hz[r])

    def eq(g, w):
        if dataclasses.is_dataclass(g):
            return all(eq(getattr(g, f.name), getattr(w, f.name)) for f in dataclasses.fields(g))
        if isinstance(g, (tuple, list)):
            return len(g) == len(w) and all(eq(u, v) for u, v in zip(g, w))
        if torch.is_tensor(g):
            return torch.equal(g, w)
        return np.array_equal(np.asarray(g), np.asarray(w))
    assert eq(got, want)


@pytest.mark.parametrize("way", ["current", "explicit"])
def test_stream_order_on_the_callers_stream(way):
    """The stream under test is held by a bounded spin kernel (``torch.cuda._sleep``) and the samples are
    copied into a NaN-filled input behind it.  C1: the call runs after the work queued before it on the
    caller's stream (it reads the samples, not NaN).  C2: work queued after it on that stream sees its
    results.  C3: it queues nothing on another stream (the default stream, with the side stream
    ``explicit``ly passed, is idle while the hold runs)."""
    C, N = 64, 4096
    x = stream(C, True, 6 * 4096, seed=2)
    ref = SpectrumAnalyzer(C, fft_size=N, dual_channels=True)
    want = ref.handle_new_data(x.clone(), buffer=4096)
    torch.cuda.synchronize()
    a = SpectrumAnalyzer(C, fft_size=N, dual_channels=True)
    a.handle_new_data(torch.zeros(C, 2, 0, device="cuda"))       # the plan and the handle, outside the hold
    y = torch.full_like(x, float("nan"))
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        torch.cuda._sleep(250_000_000)
        y.copy_(x)
    if way == "current":
        with torch.cuda.stream(side):
            got = a.handle_new_data(y, buffer=4096)
            db = got.db.clone()
    else:
        got = a.handle_new_data(y, buffer=4096, stream=side.cuda_stream)
        with torch.cuda.stream(side):
            db = got.db.clone()
        assert torch.cuda.current_stream().query()                # C3: nothing of the call on the default stream
    side.synchronize()
    assert list(got.tick) == list(want.tick)
    assert torch.equal(db, want.db)
    assert np.array_equal(got.fmax_hz, want.fmax_hz) and np.array_equal(got.fpitch_hz, want.fpitch_hz)
    assert torch.equal(a._disp, ref._disp) and torch.equal(a._disp2, ref._disp2)
