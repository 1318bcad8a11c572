"""Executable model of the lane-pipelined filterbank kernel (friture_b200/csrc/bank_pipe.cu).

TEST INFRASTRUCTURE: a NumPy restatement of the *schedule* the CUDA kernel runs -- which lane
touches which sample at which step, through which shared-memory ring -- with the arithmetic in
float64, so that any difference from the oracle is a scheduling bug, not rounding.  The CUDA
kernel mirrors this file phase by phase (phase A = the lanes' biquad loops, phase B = smoothing
accumulators, block-end reductions, input prefetch, mailbox copy); the tests run it against
oracle/friture_oracle.py on CPU.

Lanes of one channel (one half-warp; NR = bpo + 3 roles per group, two biquad sections chained per lane):
  roles [0, NR)      group 0: stage 0 (rate fs)
  roles [NR, 2*NR)   group 1: the same roles for ALL stages >= 1, time-multiplexed: in the CH sample
                     slots of one step, slots [CH-2*len_j, CH-len_j) belong to stage j
                     (len_j = CH >> j, j = 1..LOGCH) and slot CH-1 to the one "ruler" stage
                     JR + ctz(u+1) >= JR = LOGCH+1 that has a sample due
  role r < bpo: band r (both sections); role bpo+d: decimator sections 2d, 2d+1 (d = 0, 1, 2)
  skew d: a decimator lane works on the chunk the previous lane of the chain finished one step
  earlier; bands and the first decimator lane read the stage input directly.
"""
import numpy as np

MAX_OCT = 10
DEC_DEPTH = 3      # decimator chain = 3 lanes (2 sections each): a stage trails its parent by 3 steps


def stage_start_steps(n_oct, logch):
    """T[j]: step at which the chain heads of stage j work on their first sample/chunk.
    Mirrors pipe_schedule() in bank_pipe.cu."""
    T = [0] * MAX_OCT
    jr = logch + 1
    for j in range(1, MAX_OCT):
        t = T[j - 1] + DEC_DEPTH
        if j >= jr:
            P = 1 << (j - logch)
            a = P // 2 - 1
            while t % P != a:
                t += 1
        T[j] = t
    return T


def n_steps_for(n_oct, logch, t_total, T):
    ch = 1 << logch
    jr = logch + 1
    n_chunks = t_total // ch
    last = 0
    for j in range(n_oct):
        dmax = 0 if j == n_oct - 1 else DEC_DEPTH - 1
        if j < jr:
            last = max(last, n_chunks - 1 + T[j] + dmax)
        else:
            m_last = (t_total >> j) - 1
            last = max(last, T[j] + (m_last << (j - logch)) + dmax)
    # block b's band vector leaves the staging ring at step (b+1)*NB - 1 + flush_delta
    return max(last, n_chunks - 1 + flush_delta(n_oct, logch, T)) + 1


def flush_delta(n_oct, logch, T):
    """Steps after a block's last stage-0 chunk until every stage has staged its band energies."""
    delta = 0
    for j in range(1, n_oct):
        delta = max(delta, T[j] if j <= logch else T[j] - (1 << (j - logch)) + 1)
    return delta


def ctz(v):
    if v == 0:
        return 32
    n = 0
    while (v & 1) == 0:
        v >>= 1
        n += 1
    return n


class PipeModel:
    def __init__(self, sos_band, sos_dec, alphas, n_oct, logch=5, rx=8, pf=4):
        sos_band = np.asarray(sos_band, dtype=np.float64)
        sos_dec = np.asarray(sos_dec, dtype=np.float64)
        self.bpo = sos_band.shape[0]
        self.n_oct = n_oct
        self.logch = logch
        self.CH = 1 << logch
        self.JR = logch + 1
        self.NR = self.bpo + DEC_DEPTH
        self.NSEC = 2 * self.NR
        assert 2 * self.NR <= 16
        self.RX, self.PF = rx, pf
        self.alphas = np.ones(MAX_OCT)
        self.alphas[:n_oct] = np.asarray(alphas, dtype=np.float64)[:n_oct]
        self.q = 1.0 - self.alphas
        # normalised sections: numerator (1, c, 1); the chain gain is applied once
        secs = np.concatenate([sos_band.reshape(-1, 6), sos_dec], axis=0)
        assert np.allclose(secs[:, 2], secs[:, 0], rtol=1e-9)
        self.c = secs[:, 1] / secs[:, 0]
        self.a1 = secs[:, 4]
        self.a2 = secs[:, 5]
        self.g_band = np.array([sos_band[i, 0, 0] * sos_band[i, 1, 0] for i in range(self.bpo)])
        self.g_dec = float(np.prod(sos_dec[:, 0]))
        self.T = stage_start_steps(n_oct, logch)
        # canonical state (normalised sections): z[n_oct][NSEC][2], e[n_oct][bpo] (e/alpha form)
        self.z = np.zeros((n_oct, self.NSEC, 2))
        self.e = np.zeros((n_oct, self.bpo))

    def mux_stage_of_slot(self, p):
        """stage owning slot p of the multiplexed vector (p < CH-1)."""
        CH = self.CH
        j = 1
        while p >= CH - (CH >> j):
            j += 1
        return j

    def process(self, x, block):
        x = np.asarray(x, dtype=np.float64)
        CH, JR, NR, bpo, n_oct, logch = self.CH, self.JR, self.NR, self.bpo, self.n_oct, self.logch
        RX, PF, T = self.RX, self.PF, self.T
        t_total = x.shape[0]
        assert block & (block - 1) == 0 and block >= 256 and t_total % block == 0
        assert (block >> (n_oct - 1)) >= 1
        n_chunks = t_total // CH
        NB = block // CH
        n_blocks = t_total // block
        n_steps = n_steps_for(n_oct, logch, t_total, T)
        nbands = n_oct * bpo
        energies = np.full((n_blocks, nbands), np.nan)
        # roles: lane = G*NR + r
        NL = 2 * NR
        # shared memory
        X = np.full((RX, 2 * CH), np.nan)
        L = np.full((NL, 2, CH), np.nan)                   # chain links (decimator lanes), 2 buffers
        BO = np.full((2, bpo, CH), np.nan)                 # band outputs of this step, per group
        S = np.zeros((MAX_OCT, NR, 4))                     # z1A z2A z1B z2B
        ER = np.zeros((MAX_OCT, bpo))                      # smoothed energies of the ruler stages
        MB = np.full((MAX_OCT + 1, 2), np.nan)             # mailboxes, double-buffered by sample parity
        S[:n_oct] = self.z.reshape(n_oct, NR, 4)
        ER[:n_oct] = self.e
        acc0 = np.zeros((bpo, CH))
        accm = np.zeros((bpo, CH))
        acc0[:, CH - 1] = self.e[0]
        slot_stage = np.array([self.mux_stage_of_slot(p) for p in range(CH - 1)] + [0])
        len_of = lambda j: CH >> j
        for j in range(1, min(JR, n_oct)):
            accm[:, CH - len_of(j) - 1] = self.e[j]        # last slot of stage j's range
        w0 = self.q[0] ** (CH - 1 - np.arange(CH))
        Q0 = self.q[0] ** CH
        wm = np.zeros(CH)
        Qm = np.zeros(CH)
        for p in range(CH - 1):
            j = slot_stage[p]
            if j < n_oct:
                pos = p - (CH - 2 * len_of(j))
                wm[p] = self.q[j] ** (len_of(j) - 1 - pos)
                Qm[p] = self.q[j] ** len_of(j)
        for cpre in range(min(PF, n_chunks)):
            X[cpre % RX, :CH] = x[cpre * CH:(cpre + 1) * CH]

        def band_out(stage, b, val):
            return (n_oct - 1 - stage) * bpo + b, self.alphas[stage] * val

        def sec_coefs(r):
            i = 2 * r
            return (self.c[i], -self.a1[i], -self.a2[i], self.c[i + 1], -self.a1[i + 1], -self.a2[i + 1])

        for k in range(n_steps):
            # ---------------------------------------------------------------- phase A
            Lnew, Xw, MBw, BOw = {}, {}, {}, {}
            for lane in range(NL):
                g, r = divmod(lane, NR)
                isband = r < bpo                  # band r; decimator lane d = r - bpo of the chain
                d = 0 if isband else r - bpo
                isdec2 = (r == NR - 1)
                maxstage = n_oct - 1 if isband else n_oct - 2
                u = k - d
                if d == 0:
                    inp = X[k % RX, g * CH:(g + 1) * CH].copy()
                else:
                    inp = L[lane - 1, (k - 1) & 1].copy()
                out = np.full(CH, np.nan)
                cA, n1A, n2A, cB, n1B, n2B = sec_coefs(r)
                segs = []
                for gg in range(logch):
                    ln = CH >> (gg + 1)
                    st = CH - 2 * ln
                    stage = g * (gg + 1)
                    cidx = u - (T[stage] if g else 0)
                    valid = (0 <= cidx < n_chunks) and stage <= maxstage
                    segs.append((st, ln, stage, cidx, valid))
                if g == 0:
                    segs.append((CH - 1, 1, 0, u, (0 <= u < n_chunks) and 0 <= maxstage))
                else:
                    jr = JR + ctz(u + 1) if u >= 0 else 99
                    valid, m = False, -1
                    if jr <= maxstage and u >= T[jr]:
                        m = (u - T[jr]) >> (jr - logch)
                        valid = m < (t_total >> jr)
                    segs.append((CH - 1, 1, min(jr, MAX_OCT - 1), m, valid))
                    if d == 0:
                        inp[CH - 1] = MB[min(jr, MAX_OCT), m & 1] if valid else np.nan
                for (st, ln, stage, cidx, valid) in segs:
                    z1a, z2a, z1b, z2b = S[stage, r]
                    for i in range(st, st + ln):
                        xv = inp[i]
                        ya = xv + z1a
                        z1a = n1A * ya + (cA * xv + z2a)
                        z2a = n2A * ya + xv
                        yb = ya + z1b
                        z1b = n1B * yb + (cB * ya + z2b)
                        z2b = n2B * yb + ya
                        out[i] = yb
                    if valid:
                        S[stage, r] = (z1a, z2a, z1b, z2b)
                    if st == CH - 1 and g == 1 and isband:
                        yy = out[CH - 1] * self.g_band[r]
                        e = ER[stage, r] * self.q[stage] + yy * yy
                        if valid:
                            ER[stage, r] = e
                            if ((cidx + 1) & ((block >> stage) - 1)) == 0:
                                kb, val = band_out(stage, r, e)
                                energies[(cidx + 1) // (block >> stage) - 1, kb] = val
                if isband:
                    BOw[(g, r)] = out
                elif isdec2:
                    base = CH + g * (CH // 2)
                    for i in range(0, CH - 2, 2):
                        Xw[((k + 1) % RX, base + i // 2)] = out[i] * self.g_dec
                    if g == 0:
                        Xw[((k + 1) % RX, base + (CH - 2) // 2)] = out[CH - 2] * self.g_dec
                    else:
                        st, ln, stage, cidx, valid = segs[logch - 1]     # the 1-sample stage JR-1
                        if valid and (cidx % 2 == 0):
                            MBw[(JR, (cidx // 2) & 1)] = out[CH - 2] * self.g_dec
                        st, ln, stage, cidx, valid = segs[logch]
                        if valid and (cidx % 2 == 0):
                            MBw[(stage + 1, (cidx // 2) & 1)] = out[CH - 1] * self.g_dec
                else:
                    Lnew[lane] = out
            for lane, out in Lnew.items():
                L[lane, k & 1] = out
            for (g, r), out in BOw.items():
                BO[g, r] = out
            for (slot, pos), v in Xw.items():
                X[slot, pos] = v
            for (j, par), v in MBw.items():
                MB[j, par] = v
            # ---------------------------------------------------------------- phase B
            c0 = k
            valid0 = 0 <= c0 < n_chunks
            for b in range(bpo):
                y0 = BO[0, b] * self.g_band[b]
                ym = BO[1, b] * self.g_band[b]
                if valid0:
                    acc0[b] = acc0[b] * Q0 + y0 * y0
                    if ((c0 + 1) & (NB - 1)) == 0:
                        tot = float(np.dot(w0, acc0[b]))
                        kb, val = band_out(0, b, tot)
                        energies[(c0 + 1) // NB - 1, kb] = val
                        acc0[b] = 0.0
                        acc0[b, CH - 1] = tot
                for j in range(1, min(JR, n_oct)):
                    cm = k - T[j]
                    if not (0 <= cm < n_chunks):
                        continue
                    lo, hi = CH - 2 * len_of(j), CH - len_of(j)
                    accm[b, lo:hi] = accm[b, lo:hi] * Qm[lo:hi] + ym[lo:hi] ** 2
                    if ((cm + 1) & (NB - 1)) == 0:
                        tot = float(np.dot(wm[lo:hi], accm[b, lo:hi]))
                        kb, val = band_out(j, b, tot)
                        energies[(cm + 1) // NB - 1, kb] = val
                        accm[b, lo:hi] = 0.0
                        accm[b, hi - 1] = tot
            cn = k + PF
            if cn < n_chunks:
                X[cn % RX, :CH] = x[cn * CH:(cn + 1) * CH]
        # epilogue: canonical state
        self.z = S[:n_oct].reshape(n_oct, self.NSEC, 2).copy()
        self.e[0] = acc0[:, CH - 1]
        for j in range(1, min(JR, n_oct)):
            self.e[j] = accm[:, CH - len_of(j) - 1]
        for j in range(JR, n_oct):
            self.e[j] = ER[j]
        assert not np.isnan(energies).any(), "some band energies were never emitted"
        return energies
