"""GPU: the spectrogram widget from stream chunks to pixels (SpectrogramAnalyzer,
frt_stft_screen_rows, frt_display_rows).

- Same bits as the two-call path (frt_stft_process LOGPOWER + frt_display_columns) at every FFT size,
  scale, weighting, a range of heights and every frame alignment the kernels dispatch on.
- Against SpectrogramWidgetOracle on chunked streams, with every setter between chunks.
- Argument errors, and C1-C3 of INTEGRATION.md ("Streams") for the new entries and the setters.
"""
from ctypes import c_float

import numpy as np
import pytest
import torch

from friture_b200 import _lib
from friture_b200.audioproc import audioproc
from friture_b200.display import SCALES, Erb, Linear, Logarithmic, Octave, SpectrogramDisplay
from friture_b200.spectrogram import SpectrogramAnalyzer
from spectrogram_oracle import SpectrogramWidgetOracle
from test_stream_order_gpu import check, side  # noqa: F401  (side is a fixture)

pytestmark = pytest.mark.gpu

SIZES = [32 << k for k in range(10)]
PIX_TOL = 1e-5       # as tests/test_widget_reductions_gpu.py: pixel = lut[int(v' * 255)], |v' - v| <= PIX_TOL


def signal(C, T, seed):
    g = torch.Generator().manual_seed(seed)
    n = torch.arange(T, dtype=torch.float64)
    f = 200.0 + 15000.0 * torch.rand(C, 1, generator=g, dtype=torch.float64)
    x = 0.5 * torch.sin(2 * np.pi * f * n / 48000) + 0.01 * torch.randn(C, T, generator=g, dtype=torch.float64)
    return x.float().cuda()


def screen_rows(d, view, F, hop):
    """frt_stft_screen_rows on frames of ``view`` with the tables of display ``d``."""
    C = view.shape[0]
    T = d.tables(view.device)
    rows = torch.empty((C, F, d.height), dtype=torch.float32, device=view.device)
    h = d.handle
    h.call("frt_stft_plan", int(d.fft_size))
    h.call("frt_stft_screen_rows", _lib._ptr(view), int(view.stride(0)), C, F, hop, _lib._ptr(T["w"]),
           c_float(d.spec_min), c_float(d.spec_max), _lib._ptr(T["i0"]), _lib._ptr(T["t"]), d.height,
           _lib._ptr(rows), F * d.height, d.height, _lib.current_stream_ptr())
    return rows


# ---------------------------------------------------------------------------------------------
# 5. same bits as today's two calls


@pytest.mark.parametrize("offset", [0, 1, 2])     # 16-byte, 4-byte and 8-byte aligned frames
@pytest.mark.parametrize("N", SIZES)
def test_same_bits_as_two_calls(N, offset):
    C, hop = 3, N // 4
    F = 6
    x = signal(C, offset + N + (F - 1) * hop + 8, N)
    view = x[:, offset:]
    proc = audioproc()
    proc.set_fftsize(N)
    db = proc.stft(view, hop, log=True)
    F = db.shape[1]
    for k, (scale, wgt, H) in enumerate([(s, w, h) for s in SCALES.values() for w in range(4) for h in (1, 7, 512)]):
        if (k + N) % 3 and H == 512 and N > 4096:
            continue        # the large sizes cycle through the 512-row cases
        kw = dict(fft_size=N, freqscale=scale, minfreq=20., maxfreq=24000., weighting=wgt, height=H, width=700,
                  timerange_s=1.)
        a, b = SpectrogramDisplay(C, **kw), SpectrogramDisplay(C, **kw)
        want = a.push(db)
        rows = screen_rows(b, view, F, hop)
        got = b.push_rows(rows)
        lab = (N, offset, scale.NAME, wgt, H)
        assert torch.equal(got, want), lab
        assert torch.equal(rows[:, F - 1], a._old), lab       # the last row is the carried column
        assert torch.equal(b._old, a._old), lab


@pytest.mark.parametrize("N", SIZES)
def test_analyzer_same_bits_as_two_calls(N):
    """handle_new_data over a chunked stream equals SpectrogramDisplay.push(audioproc.stft(view)) on
    the framer's views, call by call."""
    C, hop = 2, N // 4
    x = signal(C, 6 * N + 3, 7)
    an = SpectrogramAnalyzer(C, fft_size=N, weighting=1, height=64, width=900, timerange_s=1.)
    ref = SpectrogramDisplay(C, fft_size=N, weighting=1, height=64, width=900, timerange_s=1.)
    proc = audioproc()
    proc.set_fftsize(N)
    from friture_b200.stream import StreamFramer
    fr = StreamFramer(C, N, hop, x.device, history=16384)
    pos = 0
    for n in [1, hop - 1, 512, 3 * N, x.shape[1]]:
        chunk = x[:, pos:pos + n]
        pos += chunk.shape[1]
        out = an.handle_new_data(chunk, want_rows=True)
        fr.push(chunk)
        view, F = fr.take()
        assert out.n_frames == F
        if F == 0:
            assert out.pixels.shape == (C, 64, 0) and out.rows is None
            continue
        want = ref.push(proc.stft(view[:, :N + (F - 1) * hop], hop, log=True))
        assert torch.equal(out.pixels, want), (N, n)
        assert torch.equal(out.rows[:, F - 1], ref._old), (N, n)


# ---------------------------------------------------------------------------------------------
# 6. against the reference


def pixel_ok(got, v, lut):
    """Pixels that are lut[int(v' * 255)] for some v' within PIX_TOL of clip(v, 0, 1)."""
    vc = np.clip(v, 0.0, 1.0)
    lo = (np.clip(vc - PIX_TOL, 0.0, 1.0) * 255).astype(np.intp)
    hi = (np.clip(vc + PIX_TOL, 0.0, 1.0) * 255).astype(np.intp)
    return (got == lut[lo]) | (got == lut[hi])


SETTERS = [
    ("setfftsize", 16384), ("setfftsize", 1024), ("setminfreq", 100.), ("setmaxfreq", 12000.),
    ("setfreqscale", Linear), ("setfreqscale", Erb), ("setfreqscale", Logarithmic), ("setfreqscale", Octave),
    ("setmin", -120.), ("setmax", -20.), ("setweighting", 1), ("setweighting", 3), ("timerangechanged", 3.),
    ("set_screen", (100, 700)), ("set_screen", (100, 1500)), ("setfftsize", 64),
]


@pytest.mark.parametrize("C", [1, 3, 256])
def test_against_oracle_chunked_with_setters(C):
    from friture_b200.display import load_lut
    lut = load_lut()
    N0 = 4096
    T = 9 * 16384
    x = signal(C, T, 11 + C)
    x_np = x.cpu().numpy().astype(np.float64)
    kw = dict(fft_size=N0, height=100, width=1024, timerange_s=2.)
    an = SpectrogramAnalyzer(C, **kw)
    check_c = list(range(C)) if C <= 3 else [0, 77, 255]
    orcs = [SpectrogramWidgetOracle(**kw) for _ in check_c]
    pos, step = 0, 0
    sizes = [1, N0 // 4 - 1, 512, 5000]
    while pos < T:
        n = sizes[step % len(sizes)] if step < 2 * len(sizes) + len(SETTERS) else T - pos
        chunk = x[:, pos:pos + n]
        out = an.handle_new_data(chunk, want_rows=True)
        outs = [o.push(x_np[c, pos:pos + n]) for c, o in zip(check_c, orcs)]
        lab = ("step", step, n)
        got = out.pixels.cpu().numpy().view(np.uint32)
        for i, c in enumerate(check_c):
            pix, rows, F, vals = outs[i]
            assert out.n_frames == F, lab
            assert got[c].shape == pix.shape, lab
            if F == 0:
                assert out.rows is None
                continue
            ok = pixel_ok(got[c], vals, lut)
            assert ok.mean() >= 0.999, (lab, c, ok.mean())
            r = out.rows[c].cpu().numpy().T.astype(np.float64)
            span = orcs[i].spec_max - orcs[i].spec_min
            # float32 log-power accuracy on a tonal input: rows within 40 dB of the column's peak (the
            # float32 noise floor sits ~45 dB below a frame's mean, tests/parity.py)
            tonal = rows >= rows.max(axis=0, keepdims=True) - 40.0 / span
            err = np.abs(r - rows)[tonal] * span            # in dB
            assert err.max() <= 0.05, (lab, c, err.max())
        pos += chunk.shape[1]
        if len(sizes) <= step < len(sizes) + len(SETTERS):
            name, arg = SETTERS[step - len(sizes)]
            args = arg if isinstance(arg, tuple) else (arg,)
            getattr(an, name)(*args)
            for o in orcs:
                getattr(o, name)(*args)
        step += 1


# ---------------------------------------------------------------------------------------------
# 7. argument errors


def test_argument_errors_leave_the_handle_usable():
    C, N = 2, 1024
    d = SpectrogramDisplay(C, fft_size=N, height=16)
    x = signal(C, 4 * N, 3)
    T = d.tables(x.device)
    h = d.handle
    h.call("frt_stft_plan", N)
    rows = torch.empty((C, 4, 16), device="cuda")
    sp = _lib.current_stream_ptr()
    P = _lib._ptr

    def sr(**o):
        a = dict(x=P(x), xs=x.stride(0), C=C, F=4, hop=N // 4, w=None, lo=-140., hi=0., i0=P(T["i0"]),
                 t=P(T["t"]), H=16, rows=P(rows), sc=64, sf=16)
        a.update(o)
        h.call("frt_stft_screen_rows", a["x"], a["xs"], a["C"], a["F"], a["hop"], a["w"], c_float(a["lo"]),
               c_float(a["hi"]), a["i0"], a["t"], a["H"], a["rows"], a["sc"], a["sf"], sp)

    for bad in [dict(C=-1), dict(F=-1), dict(hop=0), dict(H=0), dict(lo=0.), dict(x=None), dict(i0=None),
                dict(t=None), dict(rows=None), dict(sf=15)]:
        with pytest.raises(_lib.FrtValueError):
            sr(**bad)
    sr(F=0, x=None, rows=None)                    # no frames: a no-op, buffers unread
    sr()
    want = rows.clone()
    old = torch.zeros((C, 16), device="cuda")
    lut = T["lut"]
    cols = torch.zeros(3, dtype=torch.int32, device="cuda")
    av = torch.zeros(3, device="cuda")
    pix = torch.empty((C, 16, 3), dtype=torch.int32, device="cuda")

    def dr(**o):
        a = dict(rows=P(rows), C=C, F=4, H=16, cols=P(cols), a=P(av), n=3, old=P(old), lut=P(lut), pix=P(pix))
        a.update(o)
        h.call("frt_display_rows", a["rows"], 64, 16, a["C"], a["F"], a["H"], a["cols"], a["a"], a["n"], a["old"],
               a["lut"], a["pix"], sp)

    for bad in [dict(C=-1), dict(F=-1), dict(H=0), dict(n=-1), dict(rows=None), dict(old=None), dict(lut=None),
                dict(cols=None), dict(pix=None)]:
        with pytest.raises(_lib.FrtValueError):
            dr(**bad)
    dr()
    torch.cuda.synchronize()
    assert torch.equal(old, rows[:, 3])
    sr()
    torch.cuda.synchronize()
    assert torch.equal(rows, want)
    h2 = _lib.Handle(torch.cuda.current_device())   # no plan yet
    with pytest.raises(_lib.FrtError):
        h2.call("frt_stft_screen_rows", P(x), x.stride(0), C, 4, N // 4, None, c_float(-140.), c_float(0.),
                P(T["i0"]), P(T["t"]), 16, P(rows), 64, 16, sp)
    h2.close()


# ---------------------------------------------------------------------------------------------
# 8. C1-C3: calls on the caller's stream, setters for later calls only


@pytest.mark.parametrize("way", ["current", "explicit"])
@pytest.mark.parametrize("N", [256, 2048, 8192, 16384])
def test_analyzer_stream_order(side, N, way):  # noqa: F811
    C = 3

    def make():
        return SpectrogramAnalyzer(C, fft_size=N, weighting=2, height=50, width=1024, timerange_s=2.)

    def run(a, x, kw):
        out = a.handle_new_data(x, want_rows=True, **kw)
        return (out.pixels, out.rows)

    def setter(name, *args):
        def act(a, x, kw):
            getattr(a, name)(*args)
        return act

    x = [signal(C, n, 30 + i) for i, n in enumerate([2 * N, N, N // 2, 3 * N])]
    steps = [(run, x[0]), (setter("setfftsize", 1024 if N != 1024 else 512), None), (run, x[1]),
             (setter("setweighting", 1), None), (setter("setmin", -100.), None), (run, x[2]),
             (setter("set_screen", 60, 800), None), (setter("setfreqscale", Linear), None), (run, x[3])]
    def warm(a, kw):      # the analyzer's tensors, and the plan of the size it switches to
        a.handle_new_data(signal(C, 2 * N, 29), **kw)
        a.handle.call("frt_stft_plan", 1024 if N != 1024 else 512)

    check(make, steps, way, side, warm=warm)


@pytest.mark.parametrize("way", ["current", "explicit"])
def test_push_rows_stream_order(side, way):  # noqa: F811
    C, N, F = 2, 4096, 8

    def make():
        return SpectrogramDisplay(C, fft_size=N, weighting=1, height=300, width=1024)

    def push(d, x, kw):
        p = d.push_rows(x, **kw)
        with _lib.call_stream(x.device, kw.get("stream")):    # the carried column, read on the same stream
            return p, d._old.clone()

    g = torch.Generator().manual_seed(40)
    rows = [torch.rand(C, F, 300, generator=g).cuda() for _ in range(2)]
    check(make, [(push, rows[0]), (push, rows[1])], way, side)
