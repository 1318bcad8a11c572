"""float32 CPU model of the filterbank kernels' arithmetic, used to calibrate the per-band bound of
tests/parity.py (BAND_REL_TOL, BAND_FLOOR, Y_REL_TOL, Y_FLOOR).

TEST INFRASTRUCTURE, not a reference: the reference is the float64 OctaveSpectrumOracle.  The model
runs what friture_b200/csrc/bank_internal.cuh describes, one float32 rounding per operation:
- every section normalised to b = (1, c, 1), a = (1, a1, a2), with c, a1, a2 rounded to float32 and
  run as a direct-form-II-transposed recursion (scipy's sosfilt in float32);
- the chain gain (product of the section gains, rounded to float32) applied once per chain: on the
  band output, and on the decimator output where the even samples are kept;
- the widget's smoothing e <- q*e + v^2 on the normalised band output v, emitted as
  alpha_j * g^2 * e at every block end, in the kernels' chunked form: each chunk of up to 32
  samples is summed sequentially from zero (s <- s - om*s + v^2, om = float32(alpha_j)), and the
  carried e advances once per chunk, e <- e - om_L*e + s, om_L = float32(1 - q^L).  (A per-sample
  float32 recursion over the whole stream rounds the carried e once per sample: over the 1/alpha
  samples a 1 s response time remembers, that alone costs ~2e-5 of the energy.)
It is what a careful sequential float32 implementation computes; the kernels' operation orders
(chunk scans with A^(2^q) state powers, lane-pipelined steps) are other float32 orders of the same
arithmetic, so their errors are of the same size, not the same bits."""
import numpy as np
from scipy.signal import sosfilt

F32 = np.float32


def normalised_sections(sos):
    """sos [n, 6] float64 -> (float32 sos [n, 6] of the normalised sections, float64 chain gain)."""
    sos = np.asarray(sos, dtype=np.float64).reshape(-1, 6)
    out = np.zeros_like(sos, dtype=F32)
    g = 1.0
    for s, row in enumerate(sos):
        g *= row[0]
        out[s] = (1.0, F32(row[1] / row[0]), 1.0, 1.0, F32(row[4]), F32(row[5]))
    return out, g


def smooth_f32(v, alpha, L, n_per_block):
    """v [R, B, n] float32 normalised band outputs, chunks of L samples (L divides n_per_block).
    Returns e at every block end [R, B, n / n_per_block] (float32, e/alpha form)."""
    om = F32(alpha)
    omL = F32(1.0 - (1.0 - alpha) ** L)
    R, B, n = v.shape
    v2 = (v * v).astype(F32).reshape(R, B, n // L, L)
    s = np.zeros((R, B, n // L), dtype=F32)
    for k in range(L):
        s = (s - om * s) + v2[..., k]
    e = np.zeros((R, B), dtype=F32)
    out = np.empty((R, B, n // n_per_block), dtype=F32)
    per = n_per_block // L
    for c in range(n // L):
        e = (e - omL * e) + s[..., c]
        if (c + 1) % per == 0:
            out[..., c // per] = e
    return out


class BankF32Model:
    """float32 model of one bank plan over R independent rows (like the kernels' channels)."""

    def __init__(self, bank, n_octaves, alphas):
        self.bpo = bank.bandsperoctave
        self.n_oct = n_octaves
        sos_band = np.asarray(bank._sos_band, dtype=np.float64).reshape(self.bpo, 2, 6)
        self.band = [normalised_sections(sos_band[i]) for i in range(self.bpo)]
        self.gband = [F32(g) for _, g in self.band]
        self.dec, gdec = normalised_sections(bank._sos_dec)
        self.gdec = F32(gdec)
        self.alphas = np.asarray(alphas, dtype=np.float64)

    def run(self, x, block, want_y=False):
        """x [R, T] float32 from reset.  Returns (energies [R, T/block, nbands] float32, y: list of
        nbands arrays [R, T >> j] (the band outputs, chain gain applied) or None)."""
        x = np.asarray(x, dtype=F32)
        R, T = x.shape
        nb = T // block
        bpo, n_oct = self.bpo, self.n_oct
        E = np.empty((R, nb, n_oct * bpo), dtype=F32)
        Y = [None] * (n_oct * bpo) if want_y else None
        xj = x
        for j in range(n_oct):
            n = T >> j
            per = block >> j
            L = min(32, per & -per)         # largest power of two dividing the block, at most 32
            v = np.stack([sosfilt(self.band[i][0], xj, axis=-1).astype(F32) for i in range(bpo)], axis=1)
            e = smooth_f32(v, self.alphas[j], L, per)
            a = F32(self.alphas[j])
            for i in range(bpo):
                k = (n_oct - 1 - j) * bpo + i
                g = self.gband[i]
                E[:, :, k] = ((a * g) * g) * e[:, i, :]
                if want_y:
                    Y[k] = v[:, i, :] * g
            if j + 1 < n_oct:
                w = sosfilt(self.dec, xj, axis=-1).astype(F32)
                xj = (w[:, 0:n:2] * self.gdec).astype(F32)
        return E, Y
