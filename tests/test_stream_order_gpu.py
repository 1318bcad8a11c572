"""GPU: every call runs in order on its caller's stream, and setters, resets and the host-buffer call
wait for work still queued (INTEGRATION.md, "Streams").

Each case holds the stream under test with a bounded spin kernel (``torch.cuda._sleep``), queues the
calls behind it and compares what they return with the same calls on a fresh object, run on the
default stream with a device synchronise after each.  The kernels are deterministic, so device
outputs must be bit-equal and host outputs exactly equal.

- The input buffers are filled with NaN and synchronised; the real samples are copied in on the
  stream under test, behind the hold.  Work that runs on any other stream reads NaN.
- Plans, tables and allocator blocks are built by a warm-up call before the window (where a case says
  otherwise, the state is created inside it), so only host microseconds fall inside the window.
- Every host action between two calls (a setter, a reset, a host-buffer call) is issued while the
  queued work is still pending, and so is every case's last call: it either returns while that work
  is pending or it waited for it.  A run where the hold ran out early fails instead of passing.
- A side stream is a ``torch.cuda.Stream()``: non-blocking, so the legacy default stream does not wait
  for it.  The ``side`` fixture checks that by behaviour before any case relies on it.

Each case with a ``stream`` parameter runs twice: with the side stream made current ("current"), and
with ``stream=`` passed while the default stream is current ("explicit").
"""
import contextlib
import time

import numpy as np
import pytest
import torch

from friture_b200 import ChannelAnalyzer
from friture_b200.audioproc import audioproc
from friture_b200.correlation import GccPhat
from friture_b200.delay import Decimator, DelayEstimator
from friture_b200.display import SpectrogramDisplay
from friture_b200.octavefilters import Octave_Filters
from friture_b200.octavespectrum import OctaveSpectrumAnalyzer
from friture_b200.plotcurves import HistPlot, SpectrumPlot
from friture_b200.spectrum import SpectrumAnalyzer

pytestmark = pytest.mark.gpu

# ~125 ms at the H100's top SM clock (1.98 GHz), longer at lower clocks; about 70 holds in this file
HOLD_CYCLES = 250_000_000
WAITED_S = 0.05       # a call that took this long waited for the hold (it takes milliseconds otherwise)
WAYS = ["current", "explicit"]


@pytest.fixture(scope="module")
def side():
    s = torch.cuda.Stream()
    a = torch.ones(1 << 20, device="cuda")
    b = torch.empty_like(a)
    torch.cuda.synchronize()
    hold(s)
    b.copy_(a)
    torch.cuda.default_stream().synchronize()
    still_held = not s.query()
    s.synchronize()
    assert still_held, "the default stream waited for a side stream: these tests would prove nothing"
    return s


def hold(s):
    with torch.cuda.stream(s):
        torch.cuda._sleep(HOLD_CYCLES)


@contextlib.contextmanager
def on(way, s):
    """The keyword arguments that run a call on ``s``: current, or passed as ``stream=``."""
    if way == "current":
        with torch.cuda.stream(s):
            yield {}
    else:
        yield {"stream": s.cuda_stream}


def tensors(x):
    return list(x) if isinstance(x, tuple) else [x]


def poisoned(x):
    """NaN-filled buffers with the layout (shape and strides) of the real inputs ``x``."""
    return tuple(torch.empty_strided(t.shape, t.stride(), dtype=t.dtype, device=t.device).fill_(float("nan"))
                 for t in tensors(x))


def as_input(x, bufs):
    return bufs if isinstance(x, tuple) else bufs[0]


def same(got, want, where="out"):
    if isinstance(want, torch.Tensor):
        assert isinstance(got, torch.Tensor), where
        assert got.shape == want.shape and got.dtype == want.dtype, where
        ok = torch.equal(got, want)
        assert ok, "%s differs from the synchronised run in %d of %d values" % (
            where, int((got != want).sum()), want.numel())
    elif isinstance(want, np.ndarray):
        ok = np.array_equal(np.asarray(got), want)
        assert ok, "%s differs from the synchronised run: %s, not %s" % (where, got, want)
    elif isinstance(want, (list, tuple)):
        assert len(got) == len(want), where
        for i, (g, w) in enumerate(zip(got, want)):
            same(g, w, "%s[%d]" % (where, i))
    elif isinstance(want, dict):
        assert got.keys() == want.keys(), where
        for k in want:
            same(got[k], want[k], "%s.%s" % (where, k))
    elif hasattr(want, "__dataclass_fields__"):
        same(vars(got), vars(want), where)
    else:
        assert got == want, where


def check(make, steps, way, s, warm=None, after=None, window=contextlib.nullcontext):
    """Run ``steps`` on ``make()`` behind a hold of ``s`` and compare with a synchronised run.

    steps: (fn, x) pairs.  ``fn(obj, x, kw)`` is a call on real inputs x (a tensor or a tuple of
    tensors), with kw the stream keyword arguments; ``fn(obj, None, kw)`` (x is None) is a host
    action, which must be issued while the queued work is pending.  ``warm(obj, kw)`` runs before the
    window on both objects.  ``after(obj, outputs)`` runs right after the last step, inside the
    window (for sentinel allocations), and ``window()`` is a context around the window's calls.
    Returns the held run's outputs and what ``after`` returned."""
    ref = make()
    if warm is not None:
        warm(ref, {})
    torch.cuda.synchronize()
    want = []
    for fn, x in steps:
        want.append(fn(ref, x, {}))
        torch.cuda.synchronize()
    del ref

    obj = make()
    if warm is not None:
        with on(way, s) as kw:
            warm(obj, kw)
    bufs = [None if x is None else poisoned(x) for _, x in steps]

    def fill():
        with torch.cuda.stream(s):
            for (_, x), b in zip(steps, bufs):
                if x is not None:
                    for dst, src in zip(b, tensors(x)):
                        dst.copy_(src)

    fill()     # once before the window: the first launch of a kernel may wait for the device
    for b in bufs:
        for t in b or ():
            t.fill_(float("nan"))
    torch.cuda.synchronize()
    got = []
    pending_before_host = []
    with on(way, s) as kw, window():
        hold(s)
        fill()
        t0 = time.perf_counter()
        for (fn, x), b in zip(steps, bufs):
            if x is None:
                pending_before_host.append(not s.query())
                got.append(fn(obj, None, kw))
            else:
                got.append(fn(obj, as_input(x, b), kw))
        extra = after(obj, got) if after is not None else None
        pending_after = not s.query()
        waited = time.perf_counter() - t0 >= WAITED_S
    torch.cuda.synchronize()
    same(got, want)
    assert all(pending_before_host), "a host action ran after the held work had finished"
    assert pending_after or waited, "the calls neither left work queued nor waited: the hold ran out early"
    return got, extra


def rng(seed):
    return torch.Generator().manual_seed(seed)


def signal(shape, seed, fs=48000.0):
    """Noise plus a tone per row, float32 on the GPU."""
    g = rng(seed)
    x = 0.1 * torch.randn(*shape, generator=g, dtype=torch.float64)
    n = torch.arange(shape[-1], dtype=torch.float64)
    f = 300.0 + 1700.0 * torch.rand(*shape[:-1], 1, generator=g, dtype=torch.float64)
    x += 0.5 * torch.sin(2 * np.pi * f * n / fs)
    return x.float().cuda()


# ---------------------------------------------------------------------------------------------
# C1: every call on its stream

STFT_CASES = [(1024, 0), (4096, 0), (16384, 0), (4096, 3)]   # (N, row padding: 3 -> unaligned rows)


@pytest.mark.parametrize("way", WAYS)
@pytest.mark.parametrize("log", [False, True])
@pytest.mark.parametrize("n_fft,pad", STFT_CASES)
def test_stft(side, n_fft, pad, log, way):
    hop = n_fft // 4
    C, T = 3, n_fft + 5 * hop
    x = signal((C, T + pad), 1)[:, :T]

    def make():
        p = audioproc()
        p.set_fftsize(n_fft)
        return p

    def stft(p, x, kw):
        return p.stft(x, hop=hop, log=log, **kw)

    # the warm-up has the same row layout: a kernel's first launch may load its module, which waits
    check(make, [(stft, x)], way, side, warm=lambda p, kw: stft(p, signal((C, T + pad), 2)[:, :T], kw))


@pytest.mark.parametrize("way", WAYS)
@pytest.mark.parametrize("kernel", ["pipelined", "scan_y"])
def test_filter_batch_iir(side, kernel, way):
    if kernel == "pipelined":
        C, block, kwargs = 3072, 512, dict(energies=True, want_y=False)
    else:
        C, block, kwargs = 2, 256, dict(energies=True, want_y=True)
    T = 2 * block

    def fb(f, x, kw):
        return f.filter_batch(x, block, **kwargs, **kw)

    check(lambda: Octave_Filters(3), [(fb, signal((C, T), 3)), (fb, signal((C, T), 4))], way, side,
          warm=lambda f, kw: fb(f, signal((C, T), 5), kw))


@pytest.mark.parametrize("way", WAYS)
def test_filter_batch_fft_mode(side, way):
    C, block = 3, 512

    def fb(f, x, kw):
        return f.filter_batch(x, block, energies=False, want_y=True, **kw)

    check(lambda: Octave_Filters(3, mode="fft"), [(fb, signal((C, 4 * block), 6))], way, side,
          warm=lambda f, kw: fb(f, signal((C, block), 7), kw))


def octave_levels(a, x, kw, db):
    return a.process(x, block=512, db=db, **kw)


@pytest.mark.parametrize("way", WAYS)
@pytest.mark.parametrize("db", [True, False])
@pytest.mark.parametrize("bpo", [3, 24])
def test_octave_spectrum(side, bpo, db, way):
    C = 4

    def run(a, x, kw):
        return octave_levels(a, x, kw, db)

    check(lambda: OctaveSpectrumAnalyzer(C, bandsperoctave=bpo, response_time=0.125, weighting="A"),
          [(run, signal((C, 2048), 8)), (run, signal((C, 1024), 9))], way, side,
          warm=lambda a, kw: run(a, signal((C, 512), 10), kw))


@pytest.mark.parametrize("way", WAYS)
@pytest.mark.parametrize("L,contiguous", [(2400, True), (16800, True), (2400, False)])
def test_gcc_phat(side, L, contiguous, way):
    P = 3

    def pair(seed):
        d = signal((2, P, L), seed)
        d1 = torch.roll(d[0], 17, dims=1) + 0.3 * d[1]
        if contiguous:
            return d[0].contiguous(), d1.contiguous()
        return d[0].t().contiguous().t(), d1.t().contiguous().t()   # [P, L] with strides (1, P)

    def est(g, x, kw):
        return g.estimate(x[0], x[1], smooth=True, want_xcorr=True, **kw)

    check(lambda: GccPhat(L), [(est, pair(11)), (est, pair(12)), (est, pair(13))], way, side,
          warm=lambda g, kw: est(g, pair(14), kw))


def noncontiguous(C, T, seed):
    return signal((T, C), seed).t()      # [C, T] with strides (1, C)


@pytest.mark.parametrize("way", WAYS)
def test_decimator(side, way):
    C, T = 3, 2048

    def dec(d, x, kw):
        return d.process(x, **kw)

    check(lambda: Decimator(C, 2), [(dec, noncontiguous(C, T, 15)), (dec, noncontiguous(C, T, 16))], way, side,
          warm=lambda d, kw: dec(d, noncontiguous(C, T, 17), kw))


def test_delay_estimator(side):
    P, n = 2, 18432      # 0.5 s range: 6000-sample hops at 12 kHz; four chunks give three frames

    def push(e, x, kw):
        r = e.handle_new_data(x[0], x[1])
        return r, e.delay_ms.copy(), e.Xcorr_extremum.copy(), e.correlation.copy()

    def chunk(seed):
        a = signal((P, n), seed)
        return a, torch.roll(a, 40, dims=1) + 0.05 * signal((P, n), seed + 100)

    got, _ = check(lambda: DelayEstimator(P, delayrange_s=0.5), [(push, chunk(20 + i)) for i in range(4)],
                   "current", side, warm=lambda e, kw: push(e, chunk(19), kw))
    assert sum(r[0] for r in got) == 3


def spectrum_input(C, dual, T, seed):
    return signal((C, 2, T), seed) if dual else signal((C, T), seed)


@pytest.mark.parametrize("way", WAYS)
@pytest.mark.parametrize("dual", [False, True])
def test_spectrum_first_call(side, dual, way):
    """The first call creates the smoothing state and the weighting table inside the window."""
    C, N = 3, 4096
    T = N + 3 * (N // 4)

    def make():
        return SpectrumAnalyzer(C, fft_size=N, weighting=1, dual_channels=dual)

    def warm(a, kw):      # the transform's plan only, not the analyzer's state
        a.proc.stft(signal((C, N), 30), hop=N // 4, log=False, **kw)

    def run(a, x, kw):
        return a.process(x, **kw)

    check(make, [(run, spectrum_input(C, dual, T, 31)), (run, spectrum_input(C, dual, T, 32))], way, side,
          warm=warm)


def display_db(C, F, nb, seed):
    return (-140.0 * torch.rand(C, F, nb, generator=rng(seed))).cuda()


@pytest.mark.parametrize("way", WAYS)
@pytest.mark.parametrize("first", [True, False])
def test_display_push(side, first, way):
    """``first``: the screen tables and the carried column are created inside the window."""
    C, N, F = 2, 4096, 8

    def make():
        return SpectrogramDisplay(C, fft_size=N, weighting=1, height=300, width=1024)

    def push(d, x, kw):
        return d.push(x, **kw)

    got, _ = check(make, [(push, display_db(C, F, N // 2 + 1, 40))], way, side,
                   warm=None if first else (lambda d, kw: push(d, display_db(C, F, N // 2 + 1, 41), kw)))
    assert got[0].shape[2] > 0


def test_spectrum_plot(side):
    C, K = 3, 1025

    def push(p, x, kw):
        return p.push(x, np.full(C, 1000.0), np.full(C, 440.0))

    check(lambda: SpectrumPlot(C), [(push, -60 + 20 * signal((C, K), 50)), (push, -60 + 20 * signal((C, K), 51))],
          "current", side, warm=lambda p, kw: push(p, -60 + 20 * signal((C, K), 52), kw))


def test_hist_plot(side):
    C = 3
    an = OctaveSpectrumAnalyzer(C, bandsperoctave=3)

    def push(p, x, kw):
        return p.push(x)

    def levels(seed):
        return -50 + 20 * signal((C, 4, an.nbands), seed)

    check(lambda: HistPlot(C, an), [(push, levels(53)), (push, levels(54))], "current", side,
          warm=lambda p, kw: push(p, levels(55), kw))


@pytest.mark.parametrize("overlap", [False, True])
def test_channel_analyzer(side, overlap):
    C, hop = 4, 1024

    def run(a, x, kw):
        return a.process(x, overlap=overlap)

    check(lambda: ChannelAnalyzer(C, fft_size=2048, hop=hop, n_octaves=10, weighting="A"),
          [(run, signal((C, 8 * hop), 60)), (run, signal((C, 4 * hop), 61))], "current", side,
          warm=lambda a, kw: run(a, signal((C, 2 * hop), 62), kw))


# ---------------------------------------------------------------------------------------------
# C2: a setter, reset or re-plan changes no call already queued

OCTAVE_ACTIONS = {
    "setresponsetime": lambda a: a.setresponsetime(0.025),
    "setweighting": lambda a: a.setweighting("C"),
    "reset": lambda a: a.reset(),
    "setbandsperoctave": lambda a: a.setbandsperoctave(6),
}


@pytest.mark.parametrize("action", sorted(OCTAVE_ACTIONS))
def test_octave_spectrum_setter_waits(side, action):
    C = 4

    def run(a, x, kw):
        return octave_levels(a, x, kw, True)

    def act(a, x, kw):
        OCTAVE_ACTIONS[action](a)

    check(lambda: OctaveSpectrumAnalyzer(C, bandsperoctave=3, response_time=1.0, weighting="A"),
          [(run, signal((C, 2048), 70)), (act, None), (run, signal((C, 2048), 71))], "current", side,
          warm=lambda a, kw: run(a, signal((C, 1024), 72), kw))


IIR_ACTIONS = {
    "reset": lambda f: f.reset(),
    "set_weighting": lambda f: f.set_weighting("C"),
    "set_response_time": lambda f: f.set_response_time(0.125),
    "set_state": lambda f: f.set_state(*f.get_state()),
}


@pytest.mark.parametrize("action", sorted(IIR_ACTIONS))
def test_filter_batch_iir_setter_waits(side, action):
    C, block = 8, 512

    def run(f, x, kw):
        return f.filter_batch(x, block, db=True)

    def act(f, x, kw):
        IIR_ACTIONS[action](f)

    def make():
        f = Octave_Filters(3)
        f.set_weighting("A")
        return f

    check(make, [(run, signal((C, 2 * block), 73)), (act, None), (run, signal((C, 2 * block), 74))],
          "current", side, warm=lambda f, kw: run(f, signal((C, block), 75), kw))


# ---------------------------------------------------------------------------------------------
# C3: the host-buffer call sees every earlier call on the handle

@pytest.mark.parametrize("stream", ["default", "side"])
def test_channel_analyzer_host_call_waits(side, stream):
    s = torch.cuda.default_stream() if stream == "default" else side
    C, hop = 4, 1024
    x2 = signal((C, 6 * hop), 81).cpu().pin_memory()

    def run(a, x, kw):
        return a.process(x)

    def host(a, x, kw):
        return a.process_host(x2)

    check(lambda: ChannelAnalyzer(C, fft_size=2048, hop=hop, n_octaves=10),
          [(run, signal((C, 8 * hop), 80)), (host, None)], "current", s,
          warm=lambda a, kw: (run(a, signal((C, 2 * hop), 82), kw), a.process_host(signal((C, 6 * hop), 83).cpu())))


# ---------------------------------------------------------------------------------------------
# allocator reuse: a call given stream= allocates and frees its temporaries on that stream

POOLS = []   # kept for the module's lifetime: tensors from them outlive the window


def fresh_pool():
    """The window's allocations come from a new pool, whose only free blocks are those the window's
    calls free: a sentinel of a temporary's size gets the temporary's block if the call freed it to
    the default stream."""
    POOLS.append(torch.cuda.MemPool())
    return torch.cuda.use_mem_pool(POOLS[-1])


def sentinels(*specs):
    """Default-stream tensors of the temporaries' sizes, in the order the call allocates them, filled
    right away: had the call freed a temporary to the default stream while its kernel was still
    queued, the sentinel would take its block and the kernel would read it.  specs: (size, dtype,
    value); the values are ones the kernels can read safely (an index stays in range)."""
    return [(torch.full((n,), v, dtype=dt, device="cuda"), v) for n, dt, v in specs]


def untouched(ts):
    for t, v in ts:
        assert bool((t == v).all()), "a call on another stream wrote into a block of the default pool"


def test_gcc_phat_temporaries_stay_on_the_stream(side):
    P, L = 3, 2400

    def est(g, x, kw):
        return g.estimate(x[0], x[1], smooth=True, want_xcorr=True, **kw)

    x = (signal((L, P), 90).t(), signal((L, P), 91).t())
    _, sent = check(lambda: GccPhat(L), [(est, x)], "explicit", side,
                    warm=lambda g, kw: est(g, (signal((L, P), 92).t(), signal((L, P), 93).t()), kw),
                    after=lambda g, out: sentinels((P * L, torch.float32, -1e4), (P * L, torch.float32, -1e4)),
                    window=fresh_pool)
    untouched(sent)


def test_decimator_temporaries_stay_on_the_stream(side):
    C, T = 3, 2048

    def dec(d, x, kw):
        return d.process(x, **kw)

    _, sent = check(lambda: Decimator(C, 2), [(dec, noncontiguous(C, T, 94))], "explicit", side,
                    warm=lambda d, kw: dec(d, noncontiguous(C, T, 95), kw),
                    after=lambda d, out: sentinels((C * T, torch.float32, -1e4)), window=fresh_pool)
    untouched(sent)


def test_display_temporaries_stay_on_the_stream(side):
    C, N, F = 2, 4096, 8

    def make():
        return SpectrogramDisplay(C, fft_size=N, weighting=1, height=300, width=1024)

    def push(d, x, kw):
        return d.push(x, **kw)

    # the push's column index and weight uploads are [n_out] int32 and float32
    warm_db, db = display_db(C, F, N // 2 + 1, 96), display_db(C, F, N // 2 + 1, 97)
    probe = make()
    probe.push(warm_db)
    n_out = probe.push(db).shape[2]
    del probe
    assert n_out > 0
    _, sent = check(make, [(push, db)], "explicit", side, warm=lambda d, kw: push(d, warm_db, kw),
                    after=lambda d, out: sentinels((n_out, torch.int32, F - 1), (n_out, torch.float32, 0.5)),
                    window=fresh_pool)
    untouched(sent)


def test_spectrum_host_values_come_from_the_stream(side):
    """fmax and fpitch are read from [C] int32 device indices.  Blocks of that size, filled with a
    wrong bin index, are put back in the default stream's pool first: a read on the wrong stream
    would return that bin."""
    C, N, wrong = 3, 4096, 1
    T = N + 3 * (N // 4)

    def make():
        return SpectrumAnalyzer(C, fft_size=N, weighting=1)

    def run(a, x, kw):
        return a.process(x, **kw)

    def warm(a, kw):
        a.proc.stft(signal((C, N), 98), hop=N // 4, log=False, **kw)
        torch.cuda.synchronize()
        blocks = [torch.full((C,), wrong, dtype=torch.int32, device="cuda") for _ in range(512)]
        torch.cuda.synchronize()
        del blocks

    got, _ = check(make, [(run, signal((C, T), 99))], "explicit", side, warm=warm)
    freq = make().freq
    assert not np.any(got[0][1] == freq[wrong]) and not np.any(got[0][2] == freq[wrong])
