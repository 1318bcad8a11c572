"""GPU: fir_bank_kernel<R>, the live FIR bank behind frt_firbank_process and frt_firbank_levels, sample by
sample and band by band against the float64 model of its arithmetic (tests/fir_bank_model.py), at the
bank shapes its two kernels serve: the library's taps and seeded synthetic taps through the C ABI, every
filter-group remainder, tap counts that exercise the L & 3 tail and histories longer than a block,
blocks down to one sample at the last stage, one, three and 2*SMs+1 channels, strided input and padded
output rows.

Criterion: every y sample equals the model bit for bit, or, where the model's rounding is ambiguous or
its window holds a tainted input, lies in the model's float32 interval; every linear level lies within
the model's bound B_sp, every dB level within one float32 ulp plus the dB image of B_sp.  A floor on the
bit-pinned share keeps the criterion from going vacuous.  Also: the two entry points on one plan, the
setters, reset and re-plan, and the refusal of banks and blocks that do not fit in shared memory."""
import functools
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import fir_bank_model as fm  # noqa: E402
from test_fir_bank_model import EXACT_LEVEL_FLOOR, EXACT_Y_FLOOR  # noqa: E402

pytestmark = pytest.mark.gpu
MANY = "2SM+1"

# (taps, bpo, octaves, taps per filter, block, channels); "lib" is the library's 512-tap table
S = len(fm.SIGNALS)
PLANS = [("lib", 1, 9, 512, 256, S), ("lib", 3, 9, 512, 1024, MANY), ("lib", 6, 9, 512, 768, S),
         ("lib", 12, 9, 512, 256, S), ("lib", 24, 9, 512, 4096, S), ("lib", 3, 10, 512, 512, 3),
         ("lib", 24, 10, 512, 1024, 1), ("lib", 12, 10, 512, 512, MANY), ("lib", 3, 1, 512, 1, 3),
         ("lib", 12, 4, 512, 8, S), ("lib", 24, 4, 512, 256, 1),
         ("syn", 2, 9, 2, 256, 3), ("syn", 4, 9, 3, 256, S), ("syn", 7, 9, 5, 512, S),
         ("syn", 8, 9, 127, 256, S), ("syn", 10, 6, 509, 32, S), ("syn", 11, 9, 513, 768, S),
         ("syn", 13, 5, 1024, 16, S), ("syn", 23, 9, 127, 1024, MANY), ("syn", 4, 10, 1024, 512, 1),
         ("syn", 7, 3, 5, 4096, 3)]
# with fewer channels than signals, these come first
FIRST = ("white_full_scale", "impulse_then_silence", "tone_mid")


def plan_id(p):
    return "%s-bpo%d-oct%d-L%d-b%d-C%s" % p


def n_samples(block):
    """whole blocks, at least two and about 2048 samples (1024 for blocks under 64)"""
    return block * max(2, -(-(2048 if block >= 64 else 1024) // block))


def taps_of(p):
    kind, bpo, _, L, _, _ = p
    if kind == "lib":
        from friture_b200 import filter_data
        return filter_data.fir_taps(bpo)
    return fm.synthetic_taps(bpo, L, seed=1000 * bpo + L)


def weights(p):
    """a dB offset per band on every other plan"""
    if PLANS.index(p) % 2:
        return None
    return np.random.default_rng(PLANS.index(p)).uniform(-60.0, 20.0, p[1] * p[2]).astype(np.float32)


def ptr(v):
    from friture_b200 import _lib
    return _lib._ptr(v)


def stream():
    from friture_b200 import _lib
    return _lib.current_stream_ptr()


def ragged(block, bpo, n_oct):
    from friture_b200.octavefilters import ragged_layout
    off, lens = ragged_layout(block, bpo, n_oct)
    return [int(o) for o in off], [int(n) for n in lens], int(off[-1] + lens[-1])


def model_of(p, rows, w=None):
    from friture_b200.octavefilters import smoothing_alphas
    fb, fd = taps_of(p)
    m = fm.FirBankModel(fb, fd, p[2], rows)
    m.set_smoothing(smoothing_alphas(1.0, p[2]), w)
    return m


@functools.lru_cache(maxsize=None)
def run_plan(p):
    """Run the plan once on the GPU: every block through frt_firbank_process (x at an odd element
    offset in padded rows, y in NaN-filled padded rows with a spare row), then the whole stream through
    frt_firbank_levels with db = 0 and db = 1 after resets.  Returns the signals of the distinct rows,
    the kernel's results for them, and the model's."""
    import torch
    from friture_b200 import _lib
    kind, bpo, n_oct, L, block, C = p
    h = _lib.Handle(0)
    C = 2 * h.sm_count + 1 if C == MANY else C
    T = n_samples(block)
    nb = T // block
    sig = fm.make_signals(bpo, n_oct, block, T)
    order = [fm.SIGNALS.index(s) for s in FIRST] + [i for i in range(len(sig)) if fm.SIGNALS[i] not in FIRST]
    rows = [order[c % len(order)] for c in range(C)]
    xs = np.full((C, T + 3), np.nan, np.float32)
    xs[:, 1:T + 1] = sig[rows]
    xd = torch.from_numpy(xs).cuda()
    x0 = xd.data_ptr() + 4
    fb, fd = (np.ascontiguousarray(v, np.float64) for v in taps_of(p))
    h.call("frt_firbank_plan", C, bpo, n_oct, L, ptr(fb), ptr(fd))
    off, lens, need = ragged(block, bpo, n_oct)
    ys = need + 5
    yd = torch.full((nb, C + 1, ys), float("nan"), dtype=torch.float32, device="cuda")
    sp = stream()
    for b in range(nb):
        h.call("frt_firbank_process", x0 + 4 * b * block, T + 3, block, yd[b].data_ptr(), ys, sp)
    from friture_b200.octavefilters import smoothing_alphas
    alphas = smoothing_alphas(1.0, n_oct)
    w = weights(p)
    out = []
    for db in (0, 1):
        h.call("frt_firbank_reset")
        h.call("frt_firbank_set_smoothing", ptr(alphas), ptr(w))
        lv = torch.empty((C, nb, bpo * n_oct), dtype=torch.float32, device="cuda")
        h.call("frt_firbank_levels", x0, T + 3, block, nb, lv.data_ptr(), db, sp)
        out.append(lv.cpu().numpy())
    y = yd.cpu().numpy()
    h.close()
    # padding and the spare row keep their NaN sentinels
    assert np.isnan(y[:, :C, need:]).all() and np.isnan(y[:, C]).all(), "y written outside its rows"
    yk = [np.concatenate([y[b, :C, off[k]:off[k] + lens[k]] for b in range(nb)], axis=1) for k in range(len(off))]
    distinct = sorted(set(rows))
    first = [rows.index(s) for s in distinct]
    for c in range(C):      # every channel equals the first channel with its signal, bit for bit
        f = first[distinct.index(rows[c])]
        assert all(np.array_equal(v[c].view(np.int32), v[f].view(np.int32)) for v in yk), ("y", c)
        assert np.array_equal(out[0][c], out[0][f]) and np.array_equal(out[1][c], out[1][f]), ("levels", c)
    res = model_of(p, len(distinct), w).run(sig[distinct], block, levels=True)
    got = {"y": [v[first] for v in yk], "lin": out[0][first], "db": out[1][first]}
    return [fm.SIGNALS[s] for s in distinct], first, got, res


def where_text(p, names, first, idx, kind):
    block, bpo, n_oct = p[4], p[1], p[2]
    if kind == "y":
        k, r, n = idx
        j = n_oct - 1 - k // bpo
        return "signal %s, channel %d, block %d, band %d, sample %d" % (names[r], first[r], n // (block >> j), k,
                                                                       n % (block >> j))
    what, r, b, k = idx
    return "%s level: signal %s, channel %d, block %d, band %d" % (what, names[r], first[r], b, k)


@pytest.mark.parametrize("p", PLANS, ids=plan_id)
def test_band_outputs(p):
    names, first, got, res = run_plan(p)
    worst, where = fm.y_violations(got["y"], res)
    ey = fm.exact_fraction(res)
    print("FIRBANK %s y: exact share %.6f, tainted %.2e, worst %.3g" % (plan_id(p), ey, fm.taint_fraction(res), worst))
    assert worst == 0.0, "%s: %s, %.3g of the interval" % (plan_id(p), where_text(p, names, first, where, "y"), worst)
    assert ey >= EXACT_Y_FLOOR, ey


@pytest.mark.parametrize("p", PLANS, ids=plan_id)
def test_levels(p):
    names, first, got, res = run_plan(p)
    worst, where = fm.level_violations(got["lin"], got["db"], res)
    el = float(np.mean(res["linlo"] == res["linhi"]))
    print("FIRBANK %s levels: exact share %.4f, worst %.3g" % (plan_id(p), el, worst))
    assert worst == 0.0, "%s: %s, %.3g of the bound" % (plan_id(p), where_text(p, names, first, where, "l"), worst)
    assert el >= EXACT_LEVEL_FLOOR, el


def test_flush_horizon_is_exactly_silent():
    """After one impulse, every band is exactly 0.0 from the flush horizon on, where it is in the run."""
    checked = 0
    for p in PLANS:
        bpo, n_oct, L, block = p[1], p[2], p[3], p[4]
        H = fm.flush_horizon(L, n_oct)
        if H >= n_samples(block):
            continue
        names, _, got, res = run_plan(p)
        if "impulse_then_silence" not in names:
            continue
        r = names.index("impulse_then_silence")
        for k, v in enumerate(got["y"]):
            j = n_oct - 1 - k // bpo
            tail = -(-H >> j)
            assert (res["y"][k][r, tail:] == 0).all()
            assert (v[r, tail:] == 0).all(), (plan_id(p), k)
        checked += 1
    assert checked >= 4


def handle_with_plan(bpo, n_oct, C, alphas=None, w=None):
    from friture_b200 import _lib, filter_data
    h = _lib.Handle(0)
    fb, fd = (np.ascontiguousarray(v, np.float64) for v in filter_data.fir_taps(bpo))
    h.call("frt_firbank_plan", C, bpo, n_oct, fb.shape[1], ptr(fb), ptr(fd))
    if alphas is not None:
        h.call("frt_firbank_set_smoothing", ptr(alphas), ptr(w))
    return h


@pytest.mark.parametrize("bpo", [3, 12], ids=["R1", "R4"])
def test_entry_points_share_one_plan_and_the_setters_keep_state(bpo):
    """process and levels on one plan: y and the history agree whichever entry point ran the previous
    block, levels continue from process's history and sp does not move in process; set_smoothing
    mid-stream keeps both states; levels over n blocks equals one call per block bit for bit; reset and
    a re-plan restart from zero."""
    import torch
    from friture_b200 import filter_data
    from friture_b200.octavefilters import smoothing_alphas
    n_oct, block, C = 9, 256, 3
    nb = 8
    sig = fm.make_signals(bpo, n_oct, block, nb * block)[[0, 2, 11]]
    xd = torch.from_numpy(sig).cuda()
    a1, a2 = smoothing_alphas(1.0, n_oct), smoothing_alphas(0.125, n_oct)
    w = np.random.default_rng(7).uniform(-30, 5, bpo * n_oct).astype(np.float32)
    off, lens, need = ragged(block, bpo, n_oct)
    sp = stream()
    h = handle_with_plan(bpo, n_oct, C, a1)
    m = model_of(("lib", bpo, n_oct, 512, block, C), C)

    def proc(b):
        y = torch.empty((C, need), dtype=torch.float32, device="cuda")
        h.call("frt_firbank_process", xd[:, b * block:].data_ptr(), nb * block, block, y.data_ptr(), need, sp)
        res = m.run(sig[:, b * block:(b + 1) * block], block)
        yy = y.cpu().numpy()
        worst, where = fm.y_violations([yy[:, o:o + n] for o, n in zip(off, lens)], res)
        assert worst == 0.0, ("process", b, where, worst)
        return yy

    def levels(b, n, db):
        lv = torch.empty((C, n, bpo * n_oct), dtype=torch.float32, device="cuda")
        h.call("frt_firbank_levels", xd[:, b * block:].data_ptr(), nb * block, block, n, lv.data_ptr(), db, sp)
        res = m.run(sig[:, b * block:(b + n) * block], block, levels=True)
        got = lv.cpu().numpy()
        worst, where = fm.level_violations(None if db else got, got if db else None, res)
        assert worst == 0.0, ("levels", b, db, where, worst)
        return got

    y0 = proc(0)
    levels(1, 1, 0)
    y2 = proc(2)
    levels(3, 2, 1)
    h.call("frt_firbank_set_smoothing", ptr(a2), ptr(w))
    m.set_smoothing(a2, w)
    levels(5, 1, 1)
    y6 = proc(6)
    levels(7, 1, 0)
    # the same blocks through process alone: the same y bits
    h2 = handle_with_plan(bpo, n_oct, C)
    allp = []
    for b in range(nb):
        y = torch.empty((C, need), dtype=torch.float32, device="cuda")
        h2.call("frt_firbank_process", xd[:, b * block:].data_ptr(), nb * block, block, y.data_ptr(), need, sp)
        allp.append(y.cpu().numpy())
    for b, ref in ((0, y0), (2, y2), (6, y6)):
        assert np.array_equal(allp[b].view(np.int32), ref.view(np.int32)), b
    # one levels call over every block against one call per block, and reset / re-plan against new handles
    for db in (0, 1):
        one = torch.empty((C, nb, bpo * n_oct), dtype=torch.float32, device="cuda")
        h3 = handle_with_plan(bpo, n_oct, C, a1, w)
        h3.call("frt_firbank_levels", xd.data_ptr(), nb * block, block, nb, one.data_ptr(), db, sp)
        parts = []
        h5 = handle_with_plan(bpo, n_oct, C, a1, w)
        for b in range(nb):
            lv = torch.empty((C, 1, bpo * n_oct), dtype=torch.float32, device="cuda")
            h5.call("frt_firbank_levels", xd[:, b * block:].data_ptr(), nb * block, block, 1, lv.data_ptr(), db, sp)
            parts.append(lv)
        assert torch.equal(one, torch.cat(parts, dim=1)), db
        for restart in ("frt_firbank_reset", "replan"):
            if restart == "replan":
                fb, fd = (np.ascontiguousarray(v, np.float64) for v in filter_data.fir_taps(bpo))
                h.call("frt_firbank_plan", C, bpo, n_oct, 512, ptr(fb), ptr(fd))
            else:
                h.call(restart)
            h.call("frt_firbank_set_smoothing", ptr(a1), ptr(w))
            again = torch.empty_like(one)
            h.call("frt_firbank_levels", xd.data_ptr(), nb * block, block, nb, again.data_ptr(), db, sp)
            assert torch.equal(again, one), (restart, db)


@pytest.mark.parametrize("n_oct", [1, 4])
def test_octave_filters_few_octaves(n_oct):
    """Octave_Filters(mode="fft", n_octaves=1 / 4) and OctaveSpectrumAnalyzer(n_octaves=4) reach the
    same kernel through the library's plan."""
    import torch
    from friture_b200.octavefilters import Octave_Filters
    from friture_b200.octavespectrum import OctaveSpectrumAnalyzer
    bpo, block, T = 12, 256, 2048
    sig = fm.make_signals(bpo, n_oct, block, T)[[0, 1, 3, 16]]
    xd = torch.from_numpy(sig).cuda()
    y, _ = Octave_Filters(bpo, mode="fft", n_octaves=n_oct).filter_batch(xd, block=block, energies=False, want_y=True)
    m = model_of(("lib", bpo, n_oct, 512, block, 4), len(sig))
    res = m.run(sig, block, levels=True)
    worst, where = fm.y_violations([v.cpu().numpy() for v in y], res)
    assert worst == 0.0, (where, worst)
    lin = OctaveSpectrumAnalyzer(len(sig), bandsperoctave=bpo, n_octaves=n_oct).process(xd, block=block, db=False)
    worst, where = fm.level_violations(lin.cpu().numpy(), None, res)
    assert worst == 0.0, (where, worst)


# ------------------------------------------------------------------------------------------------ refusals
def smem_bytes(L, bpo, n_oct, block):
    """FirSmem(L, bpo, n_oct, block).total of bank_fir.cu"""
    r4 = lambda n: (n + 3) & ~3  # noqa: E731
    nf, nbands = bpo + 1, bpo * n_oct
    red = 8 * ((nf * L + 1) & ~1)
    sp = red + 8 * 8 * 4
    hist = sp + 8 * ((nbands + 1) & ~1)
    xa = hist + 4 * r4(n_oct * (L - 1))
    xb = xa + 4 * (r4(L) + r4(block) + 4)
    return xb + 4 * (r4(L) + r4(block // 2) + 4)


# (bpo, octaves, taps, largest block that fits or None, a block that does not fit)
OVERSIZE = [(24, 9, 1024, None, 256), (20, 10, 1024, 1024, 2048), (19, 9, 1011, 2048, 4096)]


def other_calls_succeed(h):
    """a valid call of the FIR bank and of the IIR bank on handle h"""
    import torch
    from friture_b200.octavefilters import Octave_Filters
    x = torch.from_numpy(fm.make_signals(3, 9, 512, 1024)[:2]).cuda()
    fb = Octave_Filters(3, mode="fft", handle=h)
    y, _ = fb.filter_batch(x, block=512, energies=False, want_y=True)
    e = Octave_Filters(3, handle=h).energies_batch(x, block=512)
    torch.cuda.synchronize()
    assert bool(torch.isfinite(e).all()) and bool(torch.isfinite(y[0]).all())


@pytest.mark.parametrize("bpo,n_oct,L,fits,too_big", OVERSIZE)
def test_banks_and_blocks_beyond_shared_memory_are_refused(bpo, n_oct, L, fits, too_big):
    """A bank that does not fit in one CTA's shared memory at its shortest block is refused at plan; a
    block that does not fit is refused before any launch, and the plan's state is unchanged; the next
    valid calls, on this handle and on another, of this kernel family and of another, succeed."""
    import torch
    from friture_b200 import _lib
    from friture_b200.octavefilters import smoothing_alphas
    assert smem_bytes(512, 24, 10, 4096) == 153728
    optin = torch.cuda.get_device_properties(0).shared_memory_per_block_optin
    assert smem_bytes(L, bpo, n_oct, too_big) > optin
    fb, fd = fm.synthetic_taps(bpo, L, seed=L)
    h, other = _lib.Handle(0), _lib.Handle(0)
    C, sp = 2, stream()
    n0 = h.launch_count
    if fits is None:
        assert smem_bytes(L, bpo, n_oct, 1 << (n_oct - 1)) > optin
        with pytest.raises(_lib.FrtValueError) as ei:
            h.call("frt_firbank_plan", C, bpo, n_oct, L, ptr(fb), ptr(fd))
        assert ("%d" % optin) in str(ei.value)
        assert h.launch_count == n0
        other_calls_succeed(h)
        other_calls_succeed(other)
        return
    assert smem_bytes(L, bpo, n_oct, fits) <= optin
    h.call("frt_firbank_plan", C, bpo, n_oct, L, ptr(fb), ptr(fd))
    alphas = smoothing_alphas(1.0, n_oct)
    h.call("frt_firbank_set_smoothing", ptr(alphas), None)
    T = 2 * fits
    sig = fm.make_signals(bpo, n_oct, fits, T)[[0, 2]]
    xd = torch.from_numpy(sig).cuda()
    off, lens, need = ragged(too_big, bpo, n_oct)
    ybig = torch.empty((C, need), dtype=torch.float32, device="cuda")
    lbig = torch.empty((C, 1, bpo * n_oct), dtype=torch.float32, device="cuda")
    xbig = torch.zeros((C, too_big), dtype=torch.float32, device="cuda")
    with pytest.raises(_lib.FrtValueError) as ei:
        h.call("frt_firbank_process", xbig.data_ptr(), too_big, too_big, ybig.data_ptr(), need, sp)
    assert ("%d" % smem_bytes(L, bpo, n_oct, too_big)) in str(ei.value) and ("%d" % optin) in str(ei.value)
    with pytest.raises(_lib.FrtValueError):
        h.call("frt_firbank_levels", xbig.data_ptr(), too_big, too_big, 1, lbig.data_ptr(), 0, sp)
    assert h.launch_count == n0
    # the state is untouched: the blocks that fit give the model's results from zero
    m = fm.FirBankModel(fb, fd, n_oct, C)
    m.set_smoothing(alphas)
    off, lens, need = ragged(fits, bpo, n_oct)
    y = torch.empty((C, need), dtype=torch.float32, device="cuda")
    h.call("frt_firbank_process", xd.data_ptr(), T, fits, y.data_ptr(), need, sp)
    res = m.run(sig[:, :fits], fits)
    yy = y.cpu().numpy()
    worst, where = fm.y_violations([yy[:, o:o + n] for o, n in zip(off, lens)], res)
    assert worst == 0.0, (where, worst)
    lv = torch.empty((C, 1, bpo * n_oct), dtype=torch.float32, device="cuda")
    h.call("frt_firbank_levels", xd[:, fits:].data_ptr(), T, fits, 1, lv.data_ptr(), 0, sp)
    res = m.run(sig[:, fits:], fits, levels=True)
    worst, where = fm.level_violations(lv.cpu().numpy(), None, res)
    assert worst == 0.0, (where, worst)
    other_calls_succeed(h)
    other_calls_succeed(other)
