"""The arithmetic of fir_bank_kernel<R> (friture_b200/csrc/bank_fir.cu) restated in float64 NumPy, with
the bounds within which the kernel's results must lie.

This is not a second oracle: it rounds exactly where the kernel rounds.  Stage signals and band
outputs y are float32; the taps and every accumulation are float64.  Per stage j and filter f (bands
0..bpo-1, then the decimator):
    acc_f[n] = sum_k t_f[k] x_j[n-k]   over the carried L-1 float32 inputs followed by the block
    y = float32(acc),  x_{j+1} = float32(acc_dec[0::2]),  the new history = the last L-1 inputs
and, for the levels, sp <- alpha_j sum_n (1-alpha_j)^(N-1-n) acc_n^2 + sp (1-alpha_j)^N on the
unrounded acc, with (1-alpha)^m from pow as frt_firbank_set_smoothing tabulates it.

The kernel sums in another order (one fma chain per output), so its acc differs from the model's by at
most D = 2 gamma_L S, S = conv(|t|, |x|).  Where float32(acc +- D) is one value, y must equal the
model's bit for bit; otherwise the rounding is ambiguous.  An ambiguous decimator rounding taints the
next stage's samples it produces; their possible deviation propagates through every window that holds
them (conv(|t|, dev)), across blocks through the history and down the stages.  Every y sample gets the
interval [float32(acc - D'), float32(acc + D')], D' = D + that propagated deviation, and every level a
bound B_sp that runs through the same smoothing as sp, driven by 2|acc| D' + D'^2 per sample.

Each output is computed by the same sequence of float64 operations (the taps in k order, one whole-
array multiply and add per tap), whatever the blocking, so any cut of a stream gives the same bits."""
import numpy as np

U = 2.0 ** -53
SAFE = 1.0 + 2.0 ** -20          # covers the rounding of the bounds' own float64 arithmetic
DECAY_STRIDE = 4097              # (1-alpha)^m, m = 0..4096, as the library tabulates it
MUTANTS = ("taps_float32", "float32_accumulation", "history_one_short", "odd_decimation_phase",
           "bands_swapped", "no_level_decay", "history_not_carried")


def gamma(n):
    return n * U / (1.0 - n * U)


def f32_interval(v, d):
    """(float32(v), lo, hi): the float32 roundings of v and of the ends of [v - d, v + d]."""
    y = v.astype(np.float32)
    pos = d > 0
    lo = np.where(pos, np.nextafter(v - d, -np.inf).astype(np.float32), y)
    hi = np.where(pos, np.nextafter(v + d, np.inf).astype(np.float32), y)
    return y, lo, hi


def fir_acc(ext, taps, M, step=1, phase=0, dtype=np.float64):
    """acc[r, f, m] = sum_{k=0..L-1} taps[f, k] ext[r, L-1 + phase + m*step - k], summed in k order."""
    R = ext.shape[0]
    F, L = taps.shape
    acc = np.zeros((R, F, M), dtype)
    tmp = np.empty_like(acc)
    for k in range(L):
        s = L - 1 + phase - k
        np.multiply(taps[None, :, k, None], ext[:, None, s:s + step * (M - 1) + 1:step], out=tmp)
        acc += tmp
    return acc


def conv_abs(ext, taps, M, step=1, phase=0):
    """sum_k |taps[f, k]| ext[r, L-1 + phase + m*step - k] for ext >= 0 (S and the taint term)."""
    R = ext.shape[0]
    F, L = taps.shape
    out = np.zeros((R, F, M))
    if not ext.any():
        return out
    at = np.abs(taps)
    for r in range(R):
        if not ext[r].any():
            continue
        for f in range(F):
            full = np.convolve(ext[r], at[f], "valid")          # index m <-> output at L-1+m of ext
            out[r, f] = full[phase::step][:M]
    return out


class FirBankModel:
    """One plan of frt_firbank_*: fir_band [bpo][L], fir_dec [L] float64, rows independent channels.

    track=True compares with a float64 pipeline (oracle.fir_bank_direct): the deviation carried into
    the next stage is the actual float32 rounding of every stage sample instead of the ambiguity of
    its rounding, so y and sp bound the distance to the unrounded float64 bank."""

    def __init__(self, fir_band, fir_dec, n_oct, rows, mutant=None, track=False):
        fir_band = np.asarray(fir_band, np.float64)
        self.bpo, self.L = fir_band.shape
        self.n_oct, self.rows = n_oct, rows
        self.nbands = self.bpo * n_oct
        self.taps = np.vstack([fir_band, np.asarray(fir_dec, np.float64)[None]])
        if mutant is not None and mutant not in MUTANTS:
            raise ValueError(mutant)
        self.mutant, self.track = mutant, track
        self.kern_taps = self.taps.astype(np.float32).astype(np.float64) if mutant == "taps_float32" else self.taps
        self.alphas = None
        self.weight_db = None
        self.reset()

    def reset(self):
        Lm1 = self.L - 1
        self.hist = [np.zeros((self.rows, Lm1)) for _ in range(self.n_oct)]     # float32 values
        self.hdev = [np.zeros((self.rows, Lm1)) for _ in range(self.n_oct)]     # their deviation bounds
        self.sp = np.zeros((self.rows, self.nbands))
        self.bsp = np.zeros((self.rows, self.nbands))

    def set_smoothing(self, alphas, weight_db=None):
        self.alphas = np.asarray(alphas, np.float64)
        m = np.arange(DECAY_STRIDE, dtype=np.float64)
        self.decay = [np.power(1.0 - a, m) for a in self.alphas]
        self.weight_db = None if weight_db is None else np.asarray(weight_db, np.float32).astype(np.float64)

    def band(self, j, f):
        return (self.n_oct - 1 - j) * self.bpo + f

    # ----------------------------------------------------------------------------------------------
    def run(self, x, block, levels=False):
        """x [rows, n_blocks*block] float32: one call over whole blocks.  Returns a dict:
        y, ylo, yhi   per band k, [rows, T >> j] float32: the model's y and its interval;
        taint         per band k, [rows, T >> j] bool: the window held a tainted input;
        with levels:  sp, bsp [rows, n_blocks, nbands] float64 (model and bound), lin, linlo, linhi
                      float32, db float32 and dbtol (the bound on |db_kernel - db|)."""
        x = np.asarray(x, np.float32)
        if self.mutant in ("history_one_short", "history_not_carried") and x.shape[1] > block:
            parts = [self.run(x[:, b:b + block], block, levels) for b in range(0, x.shape[1], block)]
            return {k: ([np.concatenate([p[k][i] for p in parts], axis=1) for i in range(self.nbands)]
                        if isinstance(parts[0][k], list) else np.concatenate([p[k] for p in parts], axis=1))
                    for k in parts[0]}
        if self.mutant == "history_not_carried":
            self.hist = [np.zeros_like(h) for h in self.hist]
        R, T = x.shape
        assert R == self.rows and T % block == 0 and block % (1 << (self.n_oct - 1)) == 0
        nb = T // block
        L, bpo = self.L, self.bpo
        acc_dtype = np.float32 if self.mutant == "float32_accumulation" else np.float64
        out = {k: [None] * self.nbands for k in ("y", "ylo", "yhi", "taint")}
        if levels:
            sums = np.zeros((R, nb, self.nbands))
            errs = np.zeros((R, nb, self.nbands))
        xj = x.astype(np.float64)
        dj = np.zeros_like(xj)
        for j in range(self.n_oct):
            M, N = T >> j, block >> j
            ext = np.concatenate([self.hist[j], xj], axis=1)
            dext = np.concatenate([self.hdev[j], dj], axis=1)
            self.hist[j] = ext[:, -(L - 1):].copy() if L > 1 else ext[:, :0]
            self.hdev[j] = dext[:, -(L - 1):].copy() if L > 1 else dext[:, :0]
            if self.mutant == "history_one_short":
                ext = ext.copy()
                ext[:, 0] = 0.0
            acc = fir_acc(ext, self.kern_taps[:bpo], M, dtype=acc_dtype).astype(np.float64)
            D = self._bound(ext, dext, self.taps[:bpo], M)
            if self.mutant == "bands_swapped" and bpo > 1:
                acc[:, [0, 1]] = acc[:, [1, 0]]
                D[:, [0, 1]] = D[:, [1, 0]]
            y, lo, hi = f32_interval(acc, D)
            tainted = conv_abs(dext, self.taps[:bpo], M) > 0
            for f in range(bpo):
                k = self.band(j, f)
                out["y"][k], out["ylo"][k], out["yhi"][k], out["taint"][k] = y[:, f], lo[:, f], hi[:, f], tainted[:, f]
            if levels:
                a = acc.reshape(R, bpo, nb, N)
                da = D.reshape(R, bpo, nb, N)
                w = self.decay[j][:N][::-1].copy()                   # (1-alpha)^(N-1-n)
                ks = [self.band(j, f) for f in range(bpo)]
                sums[:, :, ks] = np.sum(w * (a * a), axis=-1).transpose(0, 2, 1)
                errs[:, :, ks] = np.sum(w * (2.0 * np.abs(a) * da + da * da), axis=-1).transpose(0, 2, 1)
            if j + 1 == self.n_oct:
                break
            phase = 1 if self.mutant == "odd_decimation_phase" else 0
            dec = fir_acc(ext, self.kern_taps[bpo:], M // 2, step=2, phase=phase, dtype=acc_dtype)[:, 0]
            dec = dec.astype(np.float64)
            Dd = self._bound(ext, dext, self.taps[bpo:], M // 2, step=2, phase=phase)[:, 0]
            xn, lo, hi = f32_interval(dec, Dd)
            xj = xn.astype(np.float64)
            if self.track:
                dj = np.abs(xj - dec) + Dd
            else:
                dj = np.maximum(hi.astype(np.float64) - xj, xj - lo.astype(np.float64))
        if levels:
            out.update(self._smooth(sums, errs, block))
        return out

    def _bound(self, ext, dext, taps, M, step=1, phase=0):
        L = taps.shape[1]
        S = conv_abs(np.abs(ext), taps, M, step, phase)
        Tt = conv_abs(dext, taps, M, step, phase)
        return (2.0 * gamma(L) * S + (1.0 + gamma(L)) * Tt) * SAFE

    def _smooth(self, sums, errs, block):
        R, nb, _ = sums.shape
        sp = np.zeros((R, nb, self.nbands))
        bsp = np.zeros_like(sp)
        for j in range(self.n_oct):
            N = block >> j
            a, d = self.alphas[j], (1.0 if self.mutant == "no_level_decay" else self.decay[j][N])
            ks = [self.band(j, f) for f in range(self.bpo)]
            for b in range(nb):
                old = self.sp[:, ks]
                s = sums[:, b, ks]
                self.sp[:, ks] = a * s + old * d
                self.bsp[:, ks] = (d * self.bsp[:, ks] + a * errs[:, b, ks]
                                   + 2.0 * gamma(N + 4) * (a * s + d * old)) * SAFE
                sp[:, b, ks] = self.sp[:, ks]
                bsp[:, b, ks] = self.bsp[:, ks]
        lin, linlo, linhi = f32_interval(sp, bsp)
        w = 0.0 if self.weight_db is None else self.weight_db
        ref = sp + 1e-30
        db = (10.0 * np.log10(ref) + w).astype(np.float32)
        down = np.where(bsp < ref, -10.0 * np.log10(np.maximum(1.0 - bsp / ref, 1e-300)), np.inf)
        image = np.maximum(10.0 * np.log10(1.0 + bsp / ref), down)
        ulp = np.spacing(np.abs(db)).astype(np.float64)
        return {"sp": sp, "bsp": bsp, "lin": lin, "linlo": linlo, "linhi": linhi, "db": db,
                "dbtol": ulp + image * SAFE + 1e-12 * np.abs(db)}


# ------------------------------------------------------------------------------------------------ signals
SIGNALS = ("white_full_scale", "tone_top", "tone_mid", "tone_bottom", "tone_edge", "tone_dec_transition",
           "tone_dec_alias", "dc_offset", "nyquist", "impulse_block_first", "impulse_block_last",
           "impulses_odd", "impulses_even", "noise_1e-6", "noise_1e-30", "zeros", "impulse_then_silence")
FLUSH_AT = 3                      # the impulse of impulse_then_silence


def flush_horizon(L, n_oct):
    """first stage-0 sample from which every band of impulse_then_silence is exactly zero"""
    return FLUSH_AT + (L - 1) * ((1 << n_oct) - 1) + 1


def make_signals(bpo, n_oct, block, T, seed=99):
    """[len(SIGNALS), T] float32, one signal per row, at levels orders of magnitude apart: tones at a
    band centre of the top, middle and bottom octave (every other band in deep stopband), on a band
    edge and around the first decimator's cut-off and its alias; a DC offset, the Nyquist sequence;
    impulses on the first and the last sample of a block and on odd and even samples of every stage;
    white noise at full scale, 1e-6 and 1e-30 (float32 subnormals in the stopbands); silence; one
    impulse followed by silence."""
    from friture_b200.octavefilters import octave_frequencies
    from bank_signals import FS, _tone
    fi, _, fhigh = octave_frequencies(bpo * n_oct, bpo)
    rng = np.random.default_rng(seed)
    mid = (T // block) // 2 * block
    rows = {"white_full_scale": rng.uniform(-1.0, 1.0, T),
            "tone_top": _tone(fi[(n_oct - 1) * bpo + bpo // 2], T),
            "tone_mid": _tone(fi[(n_oct // 2) * bpo + bpo // 2], T, 0.25),
            "tone_bottom": _tone(fi[bpo // 2], T, 0.9),
            "tone_edge": _tone(fhigh[(bpo * n_oct) // 2], T),
            "tone_dec_transition": _tone(0.95 * FS / 4, T, 0.7),
            "tone_dec_alias": _tone(1.05 * FS / 4, T, 0.7),
            "dc_offset": 0.5 + 0.5e-3 * rng.standard_normal(T),
            "nyquist": 0.5 * (1.0 - 2.0 * (np.arange(T) & 1))}
    for name, at in (("impulse_block_first", [mid]), ("impulse_block_last", [mid - 1]),
                     ("impulses_odd", [mid + (1 << j) * (2 * j + 1) for j in range(n_oct)]),
                     ("impulses_even", [mid + (2 << j) * (j + 1) for j in range(n_oct)])):
        v = np.zeros(T)
        v[[a for a in at if a < T]] = 1.0
        rows[name] = v
    rows["noise_1e-6"] = 1e-6 * rng.standard_normal(T)
    rows["noise_1e-30"] = 1e-30 * rng.standard_normal(T)
    rows["zeros"] = np.zeros(T)
    v = np.zeros(T)
    v[FLUSH_AT] = 0.8
    rows["impulse_then_silence"] = v
    return np.stack([rows[s] for s in SIGNALS]).astype(np.float32)


def synthetic_taps(bpo, L, seed):
    """seeded float64 taps [bpo][L] and [L]: unit-energy random filters, so that every stage keeps
    the signal's scale"""
    rng = np.random.default_rng(seed)
    t = rng.standard_normal((bpo + 1, L)) / np.sqrt(L)
    return t[:bpo].copy(), t[bpo].copy()


# ------------------------------------------------------------------------------------------------ criterion
def y_violations(got, res):
    """(worst, where): got[k] [rows, n] float32 per band against the model's intervals.  worst is the
    largest |got - y| / (half-width + tiny) outside its interval (0 when all inside); where = (band, row,
    sample) of the worst, or None.  Exact samples must match the model bit for bit."""
    worst, where = 0.0, None
    for k, g in enumerate(got):
        g = np.asarray(g, np.float32)
        y, lo, hi = res["y"][k], res["ylo"][k], res["yhi"][k]
        exact = lo == hi
        bad = (exact & (g.view(np.int32) != y.view(np.int32))) | ~((g >= lo) & (g <= hi))
        if bad.any():
            width = np.maximum(hi.astype(np.float64) - lo.astype(np.float64), np.spacing(np.abs(y)).astype(np.float64))
            r = np.where(bad, np.abs(g.astype(np.float64) - y) / width, 0.0)
            r = np.where(np.isnan(r), np.inf, r)
            i = np.unravel_index(int(np.argmax(r)), r.shape)
            if max(r[i], 1.0) > worst or where is None:
                worst, where = max(float(r[i]), 1.0), (k,) + tuple(int(v) for v in i)
    return worst, where


def level_violations(lin, db, res):
    """(worst, where) of the linear levels [rows, blocks, bands] and the dB levels against the model's
    bounds; worst is the largest excess ratio (0 when all inside), where = (kind, row, block, band)."""
    worst, where = 0.0, None
    if lin is not None:
        lin = np.asarray(lin, np.float32)
        bad = ~((lin >= res["linlo"]) & (lin <= res["linhi"]))
        if bad.any():
            r = np.where(bad, np.abs(lin - res["sp"]) / (res["bsp"] + 1e-300), 0.0)
            r = np.where(np.isnan(r), np.inf, r)
            i = np.unravel_index(int(np.argmax(r)), r.shape)
            worst, where = max(float(r[i]), 1.0), ("lin",) + tuple(int(v) for v in i)
    if db is not None:
        err = np.abs(np.asarray(db, np.float64) - res["db"].astype(np.float64))
        r = np.where(np.isnan(err), np.inf, err / res["dbtol"])
        if (r > 1.0).any():
            i = np.unravel_index(int(np.argmax(r)), r.shape)
            if r[i] > worst:
                worst, where = float(r[i]), ("db",) + tuple(int(v) for v in i)
    return worst, where


def exact_fraction(res):
    """share of y samples whose interval is one float32 value (the kernel must match them bit for bit)"""
    n = sum(v.size for v in res["y"])
    return sum(int(np.count_nonzero(lo == hi)) for lo, hi in zip(res["ylo"], res["yhi"])) / n


def taint_fraction(res):
    n = sum(v.size for v in res["y"])
    return sum(int(np.count_nonzero(t)) for t in res["taint"]) / n
