"""NumPy float32 model of the long GCC-PHAT path (friture_b200/csrc/gcc_long.cu) in the kernel's
order, and the odd-aware float32 restatement of generalized_cross_correlation that bounds it.

The kernel computes both transforms of GCC-PHAT as Bluestein transforms: DFT_N(v)[k] =
c_k (v c (*) conj c)[k], c_n = exp(-j pi (n^2 mod 2N) / N), the circular convolution by a four-step
power-of-two FFT of M = 2^m >= 2L-1 points (M = M1 M2, columns n1 first, rows n2 second, B^ applied
in the transposed order, then the steps in reverse).  Chirps and B^ come from float64 and are
rounded to complex64 like the plan's tables; every transform step runs in complex64.

For odd L the reference's irfft(W*G) has L' = L-1 points: the second transform is L' long and its
last bin, (L-1)/2, is the Nyquist bin whose imaginary part irfft drops.  The keyword arguments of
``gcc_long`` plant bugs the tests must catch."""
import numpy as np
import scipy.fft

from oracle import friture_oracle as fo


def out_length(L):
    return L - (L & 1)


def fft_log2(L):
    """log2 of the kernel's M: the least power of two >= 2L-1."""
    return int(2 * L - 2).bit_length()


def split_logs(log_m):
    """(log2 M1, log2 M2) of the kernel's four-step split."""
    log1 = min(12, log_m // 2)
    return log1, log_m - log1


def gcc_f32_any(d0, d1):
    """generalized_cross_correlation (friture/signal/correlation.py:24-43) in single precision,
    with the reference's default irfft length (L-1 points for odd L)."""
    d0 = np.asarray(d0, dtype=np.float32)
    d1 = np.asarray(d1, dtype=np.float32)
    w = np.hanning(d0.shape[0]).astype(np.float32)
    D0 = scipy.fft.rfft((d0 - d0.mean(dtype=np.float32)) * w)
    D1 = scipy.fft.rfft((d1 - d1.mean(dtype=np.float32)) * w)
    G = D0.conjugate() * D1
    absG = np.abs(G)
    x = scipy.fft.irfft(G * (np.float32(1.0) / (np.float32(1e-10) * absG.max() + absG)))
    assert x.dtype == np.float32
    return x


def chirp(N, mod_2n=True):
    n = np.arange(N, dtype=np.int64)
    r = (n * n) % (2 * N if mod_2n else N)
    return np.exp(-1j * np.pi * r / N)


def bluestein(v, N, log_m, mod_2n=True, conj_twiddle=False):
    """DFT_N of complex64 v (N values) in the kernel's order; complex64 result."""
    M = 1 << log_m
    log1, log2 = split_logs(log_m)
    M1, M2 = 1 << log1, 1 << log2
    c64 = chirp(N, mod_2n)
    c = c64.astype(np.complex64)
    h = np.zeros(M, dtype=np.complex128)
    h[:N] = c64.conjugate()
    h[M - N + 1:] = c64[1:][::-1].conjugate()
    if 2 * N - 1 > M:      # too short an FFT: the wrapped filter overlaps itself
        h = np.zeros(M, dtype=np.complex128)
        np.add.at(h, np.arange(-(N - 1), N) % M, np.concatenate([c64[1:][::-1], c64]).conjugate())
    bhat = np.fft.fft(h).astype(np.complex64)
    a = np.zeros(M, dtype=np.complex64)
    a[:N] = v.astype(np.complex64) * c
    n1 = np.arange(M1)[:, None]
    n2 = np.arange(M2)[None, :]
    tw = np.exp((2j if conj_twiddle else -2j) * np.pi * (n1 * n2) / M).astype(np.complex64)   # W_M^(n2 k1)
    A = a.reshape(M1, M2)                                    # [n1, n2], n = M2 n1 + n2
    T = scipy.fft.fft(A, axis=0) * tw                        # columns: [k1, n2]
    X = scipy.fft.fft(T, axis=1)                             # rows: [k1, k2] = X[k1 + M1 k2]
    X = X * bhat.reshape(M2, M1).T                           # B^ in the same transposed order
    Y = scipy.fft.ifft(X, axis=1) * np.float32(M2)           # rows back: [k1, n2]
    Y = Y * np.exp(2j * np.pi * (n1 * n2) / M).astype(np.complex64)
    y = (scipy.fft.ifft(Y, axis=0) * np.float32(M1)).reshape(M)   # columns back: natural order
    assert y.dtype == np.complex64
    return c * y[:N] * np.float32(1.0 / M)


def gcc_long(d0, d1, mod_2n=True, m_short=False, odd_inverse_at_L=False, conj_twiddle=False):
    """The kernel's route in float32; returns Xcorr (L' values).  Planted bugs: the chirp index
    n^2 mod N (mod_2n=False), M one power of two short, the odd-L inverse taken at length L (and cut
    to L'), the four-step twiddle conjugated."""
    d0 = np.asarray(d0, dtype=np.float32)
    d1 = np.asarray(d1, dtype=np.float32)
    L = d0.shape[0]
    Lp = L if odd_inverse_at_L else out_length(L)
    log_m = fft_log2(L) - (1 if m_short else 0)
    w = np.hanning(L).astype(np.float32)
    u = ((d0 - d0.mean(dtype=np.float32)) * w + 1j * ((d1 - d1.mean(dtype=np.float32)) * w)).astype(np.complex64)
    kw = dict(mod_2n=mod_2n, conj_twiddle=conj_twiddle)
    Z = bluestein(u, L, log_m, **kw)
    half = Lp // 2
    k = np.arange(half + 1)
    if odd_inverse_at_L:
        k = np.arange((L - 1) // 2 + 1)
    zk, zm = Z[k], Z[(-k) % L].conjugate()
    D0 = (zk + zm) * np.float32(0.5)
    D1 = (zk - zm) * np.complex64(-0.5j)
    G = D0.conjugate() * D1
    absG = np.abs(G)
    Y = G * (np.float32(1.0) / (np.float32(1e-10) * absG.max() + absG))
    Y[0] = Y[0].real
    if Lp % 2 == 0:
        Y[Lp // 2] = Y[Lp // 2].real
    full = np.zeros(Lp, dtype=np.complex64)
    full[:len(Y)] = Y.conjugate()
    j = np.arange(len(Y), Lp)
    full[j] = Y[Lp - j]
    x = bluestein(full, Lp, log_m, **kw).real * np.float32(1.0 / Lp)
    return x[:out_length(L)].astype(np.float32)


def gcc_f64(d0, d1):
    """The float64 oracle on the float32 input (reference semantics, odd lengths included)."""
    return fo.generalized_cross_correlation(np.asarray(d0, np.float32).astype(np.float64),
                                            np.asarray(d1, np.float32).astype(np.float64))
