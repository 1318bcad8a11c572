"""Executable model of the STFT kernels' decompositions (friture_b200/csrc/stft.cu).

TEST INFRASTRUCTURE: float64 NumPy restatements of the index arithmetic the CUDA kernels run --
which lane holds which sample, where the split-step partner of a bin lives, where the 8-byte
cp.async scatter puts an element -- so that the decompositions are checked against numpy.fft on
the CPU, independently of the GPU parity tests.

  small_frames(x, Q)   stft_small_kernel<Q>: N = 64 Q, one warp per G = 32/Q frames; Q = 32 is the
                       N = 2048 path, one frame per warp
  large_frame(x, R)    stft_large_kernel<R>: N = 2048 R, R warps per frame
Both return |X|^2 / N^2 of the Hann-windowed frame(s), the reference's audioproc.analyzelive
(friture/audioproc.py:42-50).
"""
import numpy as np

TILE = 32 * 33           # float2 elements per warp tile (stft.cu)


def hann(n):
    """Symmetric Hann, friture/audioproc.py:76-81."""
    return 0.5 * (1.0 - np.cos(2.0 * np.pi * np.arange(n) / (n - 1)))


def brev(r, bits):
    return int(("{:0%db}" % bits).format(r)[::-1], 2) if bits else 0


def split_step(Z, N):
    """Real-FFT split: X[k], k = 0..M from the M-point FFT Z of z[n] = x[2n] + j x[2n+1]."""
    M = N // 2
    X = np.zeros(M + 1, dtype=np.complex128)
    for k in range(M // 2 + 1):
        z, zp = Z[k], Z[(M - k) % M]
        E = z + np.conj(zp)
        O = z - np.conj(zp)
        T = (-1j * np.exp(-2j * np.pi * k / N)) * O          # U[k] = -j W_N^k
        X[k] = (E + T) / 2
        X[M - k] = np.conj(E - T) / 2
    return X


def small_frames(x, Q):
    """x: [G][N] frames (G = 32 // Q).  Follows the kernel lane by lane."""
    G, M = 32 // Q, 32 * Q
    N = 2 * M
    assert x.shape == (G, N)
    w = hann(N)
    v = np.zeros((32, 32), dtype=np.complex128)              # v[lane][register]
    for t in range(32):
        for g in range(G):
            for n1 in range(Q):
                i = 32 * n1 + t
                v[t, g * Q + n1] = (x[g, 2 * i] * w[2 * i]) + 1j * (x[g, 2 * i + 1] * w[2 * i + 1])
    # G radix-Q DFTs over n1 in registers, natural order here (the kernel's order is bit-reversed)
    a = np.zeros_like(v)
    for t in range(32):
        for g in range(G):
            a[t, g * Q:(g + 1) * Q] = np.fft.fft(v[t, g * Q:(g + 1) * Q])
    # twiddle W_M^(k1 t) and the 32x32 transpose through the tile: lane g*Q + k1 gets the 32 values over t
    tile = np.zeros((32, 32), dtype=np.complex128)
    for t in range(32):
        for g in range(G):
            for k1 in range(Q):
                tile[g * Q + k1, t] = a[t, g * Q + k1] * np.exp(-2j * np.pi * k1 * t / M)
    out = np.zeros((G, M + 1))
    zreg = np.zeros((32, 32), dtype=np.complex128)           # zreg[lane][k2] = Z_g[k1 + Q k2]
    for lane in range(32):
        zreg[lane] = np.fft.fft(tile[lane])
    for lane in range(32):
        g, k1 = divmod(lane, Q)
        src_lane = g * Q + (Q - k1) % Q
        for m in range(16):
            z = zreg[lane, m]
            # partner bin M - (k1 + Q m): another lane's register 31 - m, or this lane's 32 - m when k1 = 0
            zp = zreg[src_lane, 31 - m]
            if k1 == 0:
                zp = zreg[lane, 0] if m == 0 else zreg[lane, 32 - m]
            k = k1 + Q * m
            E = z + np.conj(zp)
            O = z - np.conj(zp)
            T = (-1j * np.exp(-2j * np.pi * k / N)) * O
            out[g, k] = abs((E + T) / 2) ** 2 / N ** 2
            out[g, M - k] = abs((E - T) / 2) ** 2 / N ** 2
        if k1 == 0:
            out[g, M // 2] = abs(zreg[lane, 16]) ** 2 / N ** 2     # bin M/2: X = conj(Z)
    return out


def hann_on_the_fly(R):
    """The window as stft_large_kernel computes it: n = 64 R n1 + (2 R t + 2 w + e),
    cos(theta n) = cos A cos B - sin A sin B, except register blocks 0 and 31, which read the window
    table (the formula cancels there).  Returns w[n] for n < N."""
    N = 2048 * R
    theta = 2.0 * np.pi / (N - 1)
    out = np.zeros(N)
    for n1 in range(32):
        if n1 in (0, 31):
            blk = slice(64 * R * n1, 64 * R * (n1 + 1))
            out[blk] = hann(N)[blk]
            continue
        ca, sa = 0.5 * np.cos(theta * 64 * R * n1), 0.5 * np.sin(theta * 64 * R * n1)
        for w in range(R):
            for t in range(32):
                for e in range(2):
                    b = theta * (2 * R * t + 2 * w + e)
                    out[64 * R * n1 + 2 * R * t + 2 * w + e] = 0.5 - ca * np.cos(b) + sa * np.sin(b)
    return out


def scatter_position(e, R):
    """Where the 8-byte cp.async puts element e (a float2) of the frame: (tile index, float2 offset)."""
    w, i = e % R, e // R
    return w, w * (16 // R) + i


def large_frame(x, R):
    """x: [N], N = 2048 R.  R decimated 1024-point FFTs, radix-R combine, split step."""
    M, N = 1024 * R, 2048 * R
    assert x.shape == (N,)
    z = (x * hann_on_the_fly(R)).reshape(M, 2)
    z = z[:, 0] + 1j * z[:, 1]
    tiles = np.zeros((R, TILE), dtype=np.complex128)
    for e in range(M):
        w, pos = scatter_position(e, R)
        tiles[w, pos] = z[e]
    Zw = np.zeros((R, 1024), dtype=np.complex128)
    for w in range(R):
        Zw[w] = np.fft.fft(tiles[w, w * (16 // R): w * (16 // R) + 1024])
    Z = np.zeros(M, dtype=np.complex128)
    for k0 in range(1024):
        t = np.array([Zw[w, k0] * np.exp(-2j * np.pi * w * k0 / M) for w in range(R)])
        Z[k0 + 1024 * np.arange(R)] = np.fft.fft(t)           # sum_w W_R^(wq) t[w]
    half = M // 2
    post = -1j * np.exp(-2j * np.pi * np.arange(half + 1) / N)       # table of M/2 + 1 entries

    def post_lookup(kk):
        return post[kk] if kk <= half else -1j * post[kk - half]

    out = np.zeros(M + 1)

    def store(kk, zz, zp):
        E = zz + np.conj(zp)
        O = zz - np.conj(zp)
        T = post_lookup(kk) * O
        out[kk] = abs((E + T) / 2) ** 2 / N ** 2
        out[M - kk] = abs((E - T) / 2) ** 2 / N ** 2

    for k0 in range(1, 512):
        A = Z[k0 + 1024 * np.arange(R)]
        B = Z[(1024 - k0) + 1024 * np.arange(R)]
        for q in range(R):
            store(k0 + 1024 * q, A[q], B[R - 1 - q])
    A = Z[1024 * np.arange(R)]
    store(0, A[0], A[0])
    for q in range(1, R // 2 + 1):
        store(1024 * q, A[q], A[R - q])
    A = Z[512 + 1024 * np.arange(R)]
    for q in range(R // 2):
        store(512 + 1024 * q, A[q], A[R - 1 - q])
    return out
