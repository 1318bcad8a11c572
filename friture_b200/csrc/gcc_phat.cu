// GCC-PHAT delay estimation for sm_90a: one CTA per channel pair, everything for a pair stays in
// shared memory.  Stands behind generalized_cross_correlation (friture/signal/correlation.py:24-43)
// and the smoothing + peak pick of the delay estimator (friture/delay_estimator.py:129-142).
//
//   a = (d0 - mean(d0)) * hanning(L),  b = (d1 - mean(d1)) * hanning(L)        correlation.py:27-31
//   Z = FFT_L(a + j b)  ->  D0[k] = (Z[k] + conj Z[L-k]) / 2,  D1[k] = (Z[k] - conj Z[L-k]) / 2j
//   G = conj(D0) D1,  W = 1 / (1e-10 max|G| + |G|),  X = irfft(W G)            correlation.py:34-41
//   Xs = 0.3 X + 0.7 Xs_prev (when a previous frame exists), i = argmax |Xs|   delay_estimator.py:134-142
//
// The two real transforms share ONE complex FFT of length L (L = 24 000 = 2^6 * 3 * 5^3 for the
// default one-second range at 12 kHz, delay_estimator.py:53-54,114-117); the inverse real
// transform is a second complex FFT of the conjugated Hermitian spectrum.  The FFT is an in-place
// mixed-radix (4/2/3/5) decimation-in-frequency over the 8*L-byte shared-memory buffer; results
// are addressed through the mixed-radix digit reversal instead of being permuted.
#include <algorithm>
#include <cmath>

#include "frt_internal.cuh"
#include "fft_radix.cuh"

namespace {

// A thread keeps its slice of the cross-spectrum G (GCC_MAX_PER_THREAD float2) in registers between
// the two FFTs.  On sm_90 512 threads (128 registers each) spill 432 B of stores and 1 072 B of loads
// per thread, and 256 threads leave too few warps to hide the shared-memory latency of the FFT
// passes; 384 threads (168 registers, 60 B / 84 B of spills) were fastest on an H100 80GB HBM3 at L = 24 000:
// 1.28e6 pairs/s against 1.11e6 (512) and 1.05e6 (256).
constexpr int GCC_THREADS = 384;
constexpr int GCC_MAX_PASSES = 16;
constexpr int GCC_MAX_PER_THREAD = 38;   // (L/2+1) / GCC_THREADS rounded up must not exceed this;
                                         // 38 covers the longest frame the shared memory takes (28160)

struct GccRadices {
    int n_passes;
    int radix[GCC_MAX_PASSES];
    unsigned magic[GCC_MAX_PASSES];   // ceil(2^32 / n_next) of the pass: idx / n_next == umulhi(idx, magic)
};

template <> __device__ __forceinline__ void dft<3>(float2 (&v)[3]) {
    const float s = 0.86602540378443864676f;
    const float2 t = cadd(v[1], v[2]);
    const float2 m1 = make_float2(fmaf(-0.5f, t.x, v[0].x), fmaf(-0.5f, t.y, v[0].y));
    const float2 m2 = cscale(mul_mj(csub(v[1], v[2])), s);
    v[0] = cadd(v[0], t);
    v[1] = cadd(m1, m2);
    v[2] = csub(m1, m2);
}
template <> __device__ __forceinline__ void dft<5>(float2 (&v)[5]) {
    const float c1 = 0.30901699437494742410f, c2 = -0.80901699437494742410f;
    const float s1 = 0.95105651629515357212f, s2 = 0.58778525229247312917f;
    const float2 a1 = cadd(v[1], v[4]), a2 = cadd(v[2], v[3]);
    const float2 b1 = csub(v[1], v[4]), b2 = csub(v[2], v[3]);
    const float2 t1 = make_float2(v[0].x + c1 * a1.x + c2 * a2.x, v[0].y + c1 * a1.y + c2 * a2.y);
    const float2 t2 = make_float2(v[0].x + c2 * a1.x + c1 * a2.x, v[0].y + c2 * a1.y + c1 * a2.y);
    const float2 u1 = mul_mj(make_float2(s1 * b1.x + s2 * b2.x, s1 * b1.y + s2 * b2.y));
    const float2 u2 = mul_mj(make_float2(s2 * b1.x - s1 * b2.x, s2 * b1.y - s1 * b2.y));
    v[0] = cadd(v[0], cadd(a1, a2));
    v[1] = cadd(t1, u1);
    v[4] = csub(t1, u1);
    v[2] = cadd(t2, u2);
    v[3] = csub(t2, u2);
}

#include "unit_roots.inc"

// Composite in-register DFT of R = R1*R2 points: R2 DFTs of size R1 over the stride-R2 sub-
// sequences, twiddles W_R^(q2 k1) (compile-time constants), R1 DFTs of size R2;
// V[k1 + R1 k2] = sum_q v[q] W_R^(q k), q = q1 R2 + q2.
template <int R1, int R2>
__device__ __forceinline__ void dft_comp(float2 (&v)[R1 * R2]) {
    constexpr int R = R1 * R2;
#pragma unroll
    for (int q2 = 0; q2 < R2; q2++) {
        float2 t[R1];
#pragma unroll
        for (int q1 = 0; q1 < R1; q1++) t[q1] = v[q1 * R2 + q2];
        dft<R1>(t);
#pragma unroll
        for (int k1 = 0; k1 < R1; k1++) {
            const int m = q2 * k1;
            v[k1 * R2 + q2] = (m == 0) ? t[k1]
                                       : cmul(t[k1], make_float2(UnitRoots<R>::c(m), -UnitRoots<R>::s(m)));
        }
    }
    float2 o[R];
#pragma unroll
    for (int k1 = 0; k1 < R1; k1++) {
        float2 t[R2];
#pragma unroll
        for (int q2 = 0; q2 < R2; q2++) t[q2] = v[k1 * R2 + q2];
        dft<R2>(t);
#pragma unroll
        for (int k2 = 0; k2 < R2; k2++) o[k1 + R1 * k2] = t[k2];
    }
#pragma unroll
    for (int k = 0; k < R; k++) v[k] = o[k];
}
template <> __device__ __forceinline__ void dft<16>(float2 (&v)[16]) { dft_comp<4, 4>(v); }
template <> __device__ __forceinline__ void dft<25>(float2 (&v)[25]) { dft_comp<5, 5>(v); }
template <> __device__ __forceinline__ void dft<15>(float2 (&v)[15]) { dft_comp<3, 5>(v); }

// One in-place DIF pass of radix R on sub-transforms of length n (n_next = n / R).
// FIRST: the pass also applies (x - mean) * hanning on its loads (correlation.py:27-31), so the
// windowing costs no extra sweep over shared memory.
template <int R, bool FIRST>
__device__ __forceinline__ void dif_pass(float2 *z, int L, int n, unsigned magic,
                                         const float2 *__restrict__ tw,
                                         const float *__restrict__ window, float m0, float m1) {
    const int n_next = n / R;
    const int tw_step = L / n;
    const int total = L / R;
    for (int idx = threadIdx.x; idx < total; idx += blockDim.x) {
        const int blk = (n_next == 1) ? idx : (int)__umulhi((unsigned)idx, magic);
        const int j = idx - blk * n_next;
        float2 *p = z + blk * n + j;
        float2 v[R];
#pragma unroll
        for (int q = 0; q < R; q++) {
            v[q] = p[q * n_next];
            if (FIRST) {
                const float w = __ldg(window + blk * n + j + q * n_next);
                v[q] = make_float2((v[q].x - m0) * w, (v[q].y - m1) * w);
            }
        }
        dft<R>(v);
        p[0] = v[0];
        // W_n^(j q), q = 1..R-1: one table read, the rest by successive products
        const float2 w1 = __ldg(tw + (size_t)j * tw_step);
        float2 wq = w1;
        p[n_next] = cmul(v[1], w1);
#pragma unroll
        for (int q = 2; q < R; q++) {
            wq = cmul(wq, w1);
            p[q * n_next] = cmul(v[q], wq);
        }
    }
}

template <bool FIRST>
__device__ __forceinline__ void run_pass(int r, float2 *z, int L, int n, unsigned magic,
                                         const float2 *__restrict__ tw,
                                         const float *__restrict__ window, float m0, float m1) {
    if (r == 16) dif_pass<16, FIRST>(z, L, n, magic, tw, window, m0, m1);
    else if (r == 25) dif_pass<25, FIRST>(z, L, n, magic, tw, window, m0, m1);
    else if (r == 15) dif_pass<15, FIRST>(z, L, n, magic, tw, window, m0, m1);
    else if (r == 4) dif_pass<4, FIRST>(z, L, n, magic, tw, window, m0, m1);
    else if (r == 5) dif_pass<5, FIRST>(z, L, n, magic, tw, window, m0, m1);
    else if (r == 3) dif_pass<3, FIRST>(z, L, n, magic, tw, window, m0, m1);
    else dif_pass<2, FIRST>(z, L, n, magic, tw, window, m0, m1);
}

// In-place FFT; when `window` is given the first pass also removes the means and applies it.
__device__ __noinline__ void fft_inplace(float2 *z, int L, const GccRadices &rd,
                                         const float2 *__restrict__ tw,
                                         const float *__restrict__ window, float m0, float m1) {
    int n = L;
    for (int i = 0; i < rd.n_passes; i++) {
        const int r = rd.radix[i];
        if (i == 0 && window) run_pass<true>(r, z, L, n, rd.magic[i], tw, window, m0, m1);
        else run_pass<false>(r, z, L, n, rd.magic[i], tw, window, m0, m1);
        n /= r;
        __syncthreads();
    }
}

// storage position of frequency (or time) index k after the in-place DIF passes
static int digit_reverse(int k, int L, const GccRadices &rd) {
    int pos = 0, n = L;
    for (int i = 0; i < rd.n_passes; i++) {
        const int r = rd.radix[i];
        n /= r;
        const int kq = k / r;
        pos += (k - kq * r) * n;
        k = kq;
    }
    return pos;
}

// The arguments of the three shared-memory kernels: gcc_args fills the plan's tables and the call's
// outputs, the entry points add the inputs.  The spectra workspace and the pair table of
// frt_gcc_phat_pairs are separate kernel parameters: the kernels copy this struct to the stack, and a
// larger one changes gcc_phat_kernel's code.
struct GccArgs {
    const float *d0, *d1;      // pair p: rows d0 + p*stride, d1 + p*stride (gcc_spectra_kernel: pair p
    long long stride;          // packs channels 2p and 2p+1)
    int n, L;                  // n: pairs, or channels in gcc_spectra_kernel
    const float *window;       // [L] np.hanning(L)
    const float2 *tw;          // [L] W_L^i
    const int *perm;           // [L] storage position of index k after the in-place DIF passes
    float *xcorr;              // [n_pairs][L] or NULL: raw Xcorr of this frame
    float *smoothed;           // [n_pairs][L] or NULL: in (if have_prev) / out smoothed Xcorr
    int have_prev;
    int *idx;                  // [n_pairs] argmax |Xs|
    float *val;                // [n_pairs] Xs[argmax]
    GccRadices rd;
};

// The device steps of one pair, shared by gcc_phat_kernel (rows d0, d1 of independent pairs) and
// the two phases of frt_gcc_phat_pairs (gcc_spectra_kernel, gcc_pairs_kernel).

// Loads two rows into z as d0 + j d1 and returns their means and spans (max - min); a span that is
// not > 0 marks a constant row, which the reference skips (delay_estimator.py:129-131).
// D1_MAY_BE_NULL: a NULL d1 reads as a row of zeros (mean 0, span 0: a constant row).
template <bool D1_MAY_BE_NULL = false>
__device__ __forceinline__ void gcc_load(float2 *z, const float *d0, const float *d1, int L, float *s_red,
                                         float &m0, float &m1, float &span0, float &span1) {
    const int tid = threadIdx.x, nt = blockDim.x;
    float s0 = 0.f, s1 = 0.f, mn0 = INFINITY, mx0 = -INFINITY, mn1 = INFINITY, mx1 = -INFINITY;
    for (int n = tid; n < L; n += nt) {
        const float u = __ldg(d0 + n), v = (D1_MAY_BE_NULL && !d1) ? 0.f : __ldg(d1 + n);
        z[n] = make_float2(u, v);
        s0 += u;
        s1 += v;
        mn0 = fminf(mn0, u); mx0 = fmaxf(mx0, u);
        mn1 = fminf(mn1, v); mx1 = fmaxf(mx1, v);
    }
    m0 = block_sum(s0, s_red) / (float)L;
    m1 = block_sum(s1, s_red) / (float)L;
    span0 = block_max(mx0, s_red) + block_max(-mn0, s_red);
    span1 = block_max(mx1, s_red) + block_max(-mn1, s_red);
}

// Outputs of a pair with a constant input: (0, 0), a zero Xcorr, the smoothed row left alone.
__device__ __forceinline__ void gcc_silent(int pair, int L, float *xcorr, float *smoothed, int have_prev,
                                           int *idx, float *val) {
    const int tid = threadIdx.x, nt = blockDim.x;
    if (tid == 0) {
        idx[pair] = 0;
        val[pair] = 0.f;
    }
    if (xcorr)
        for (int n = tid; n < L; n += nt) xcorr[(size_t)pair * L + n] = 0.f;
    // the reference leaves old_Xcorr alone on a silent frame (delay_estimator.py:129-131,162-165);
    // on the very first call there is none yet: mark the pair "no previous" (NaN in slot 0)
    if (smoothed && have_prev == 0 && tid == 0) smoothed[(size_t)pair * L] = nanf("");
    __syncthreads();
}

// From this thread's slice g of G[k], k = tid + i * blockDim.x <= L/2, and its max |G|: the PHAT
// weighting and the inverse transform, x[n] = Re(FFT(conj Yfull))[n] / L at z[perm[n]].
__device__ __forceinline__ void gcc_inverse(float2 *z, const float2 (&g)[GCC_MAX_PER_THREAD], float gmax,
                                            int L, float *s_red, const GccRadices &rd,
                                            const float2 *__restrict__ tw) {
    const int tid = threadIdx.x, nt = blockDim.x, half = L / 2;
    const float m = block_max(gmax, s_red);   // also orders the reads of z before the writes below
    const float floor_ = 1e-10f * m;
#pragma unroll
    for (int i = 0; i < GCC_MAX_PER_THREAD; i++) {
        const int k = tid + i * nt;
        if (k <= half) {
            const float ag = sqrtf(g[i].x * g[i].x + g[i].y * g[i].y);
            const float w = 1.0f / (floor_ + ag);
            float2 y = make_float2(g[i].x * w, g[i].y * w);
            if (k == 0 || k == half) y.y = 0.f;          // irfft ignores these imaginary parts
            // second FFT runs on conj(Y): x = Re(FFT(conj Y)) / L
            z[k] = make_float2(y.x, -y.y);
            if (k != 0 && k != half) z[L - k] = y;        // Y[L-k] = conj(Y[k])
        }
    }
    __syncthreads();
    fft_inplace(z, L, rd, tw, nullptr, 0.f, 0.f);
}

// Smoothing (delay_estimator.py:134-139) and arg-max of |Xs| (first maximum wins) of the inverse
// transform in z; writes the pair's Xcorr, smoothed row, idx and val.
__device__ __forceinline__ void gcc_finish(const float2 *z, int L, const int *__restrict__ perm, int pair,
                                           float *xcorr, float *smoothed, int have_prev, int *idx,
                                           float *val, float *s_red, int *s_idx) {
    const int tid = threadIdx.x, nt = blockDim.x;
    const float inv = 1.0f / (float)L;
    float best = -1.f;
    int besti = 0x7fffffff;
    float *sm = smoothed ? smoothed + (size_t)pair * L : nullptr;
    float *xc = xcorr ? xcorr + (size_t)pair * L : nullptr;
    // have_prev: 1 = every pair has a previous smoothed frame; 2 = per pair, a NaN in slot 0
    // marks a pair that has had only silent frames so far (old_Xcorr is None there)
    bool prev = have_prev == 1;
    if (sm && have_prev == 2) prev = !isnan(sm[0]);
    __syncthreads();     // everyone has read the marker before slot 0 is rewritten
    for (int n = tid; n < L; n += nt) {
        float v = z[__ldg(perm + n)].x * inv;
        if (xc) xc[n] = v;
        if (sm) {
            if (prev) v = gcc_blend(v, sm[n]);
            sm[n] = v;
        }
        const float av = fabsf(v);
        if (av > best) {
            best = av;
            besti = n;
        }
    }
    // block arg-max
    for (int o = 16; o > 0; o >>= 1) {
        const float ob = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, besti, o);
        if (ob > best || (ob == best && oi < besti)) {
            best = ob;
            besti = oi;
        }
    }
    __syncthreads();
    if ((tid & 31) == 0) {
        s_red[tid >> 5] = best;
        s_idx[tid >> 5] = besti;
    }
    __syncthreads();
    if (tid < 32) {
        best = (tid < (nt >> 5)) ? s_red[tid] : -1.f;
        besti = (tid < (nt >> 5)) ? s_idx[tid] : 0x7fffffff;
        for (int o = 16; o > 0; o >>= 1) {
            const float ob = __shfl_xor_sync(0xffffffffu, best, o);
            const int oi = __shfl_xor_sync(0xffffffffu, besti, o);
            if (ob > best || (ob == best && oi < besti)) {
                best = ob;
                besti = oi;
            }
        }
        if (tid == 0) s_idx[32] = besti;
    }
    __syncthreads();
    if (tid == 0) {
        const int bi = s_idx[32];
        float v = z[__ldg(perm + bi)].x * inv;
        if (sm) v = sm[bi];
        idx[pair] = bi;
        val[pair] = v;
    }
    __syncthreads();
}

// G[k] = conj(D0[k]) D1[k] for this thread's k = tid + i * blockDim.x <= L/2, from the packed
// transform Z of d0 + j d1 in z, into the thread's slice g; returns the slice's max |G|.  The same
// floats as gcc_phat_kernel's loop, which is written out there.
__device__ __forceinline__ float gcc_packed_cross(const float2 *z, int L, const int *__restrict__ perm,
                                                  float2 (&g)[GCC_MAX_PER_THREAD]) {
    const int tid = threadIdx.x, nt = blockDim.x, half = L / 2;
    float gmax = 0.f;
#pragma unroll
    for (int i = 0; i < GCC_MAX_PER_THREAD; i++) {
        const int k = tid + i * nt;
        g[i] = make_float2(0.f, 0.f);
        if (k <= half) {
            float2 D0, D1;
            split_packed(z[__ldg(perm + k)], z[__ldg(perm + (k == 0 ? 0 : L - k))], D0, D1);
            g[i] = cross_spectrum(D0, D1);
            gmax = fmaxf(gmax, sqrtf(g[i].x * g[i].x + g[i].y * g[i].y));
        }
    }
    return gmax;
}

// The same slice from two stored spectra D_i, D_j (frt_gcc_phat_pairs' phase 2).
__device__ __forceinline__ float gcc_table_cross(const float2 *Di, const float2 *Dj, int L,
                                                 float2 (&g)[GCC_MAX_PER_THREAD]) {
    const int tid = threadIdx.x, nt = blockDim.x, half = L / 2;
    float gmax = 0.f;
#pragma unroll
    for (int i = 0; i < GCC_MAX_PER_THREAD; i++) {
        const int k = tid + i * nt;
        g[i] = make_float2(0.f, 0.f);
        if (k <= half) {
            g[i] = cross_spectrum(Di[k], Dj[k]);
            gmax = fmaxf(gmax, sqrtf(g[i].x * g[i].x + g[i].y * g[i].y));
        }
    }
    return gmax;
}

// Phase 1 of frt_gcc_phat_pairs for one packed channel pair, rows d0 and d1 (NULL: the missing
// partner of an odd last channel, read as zeros): the channels' constant flags in quiet[0], quiet[1]
// and, unless both are constant, their spectra D[k], k = 0..L/2, in spec[k] and spec[L/2+1 + k].
__device__ __forceinline__ void gcc_spectra_pack(float2 *z, float *s_red, const GccArgs &a, const float *d0,
                                                 const float *d1, float2 *spec, int *quiet) {
    const int L = a.L, H = L / 2 + 1;
    const int tid = threadIdx.x, nt = blockDim.x;
    const bool has1 = d1 != nullptr;
    float m0, m1, span0, span1;
    gcc_load<true>(z, d0, d1, L, s_red, m0, m1, span0, span1);
    const bool quiet0 = !(span0 > 0.f), quiet1 = !(span1 > 0.f);
    if (tid == 0) {
        quiet[0] = quiet0;
        if (has1) quiet[1] = quiet1;
    }
    if (quiet0 && quiet1) return;   // gcc_load's reductions ordered every read of z
    fft_inplace(z, L, a.rd, a.tw, a.window, m0, m1);
    for (int k = tid; k < H; k += nt) {
        float2 D0, D1;
        split_packed(z[__ldg(a.perm + k)], z[__ldg(a.perm + (k == 0 ? 0 : L - k))], D0, D1);
        spec[k] = D0;
        if (has1) spec[H + k] = D1;
    }
    __syncthreads();
}

__global__ void __launch_bounds__(GCC_THREADS, 1) gcc_phat_kernel(const GccArgs a) {
    extern __shared__ float2 z[];
    __shared__ float s_red[40];
    __shared__ int s_idx[33];
    const int L = a.L, half = L / 2;
    const int tid = threadIdx.x, nt = blockDim.x;
    for (int pair = blockIdx.x; pair < a.n; pair += gridDim.x) {
        float m0, m1, span0, span1;
        gcc_load(z, a.d0 + (size_t)pair * a.stride, a.d1 + (size_t)pair * a.stride, L, s_red, m0, m1, span0,
                 span1);
        if (!(span0 > 0.f) || !(span1 > 0.f)) {
            gcc_silent(pair, L, a.xcorr, a.smoothed, a.have_prev, a.idx, a.val);
            continue;
        }
        fft_inplace(z, L, a.rd, a.tw, a.window, m0, m1);   // mean removal + window fused in

        // G[k] = conj(D0[k]) D1[k], k = 0..L/2, kept in registers.  The loop of gcc_packed_cross, written
        // out here: calling it changes this kernel's register allocation (304 B of stack and 68 B / 96 B
        // of spills instead of 296 B and 60 B / 84 B), and this kernel's code is kept as it was.
        float2 g[GCC_MAX_PER_THREAD];
        float gmax = 0.f;
#pragma unroll
        for (int i = 0; i < GCC_MAX_PER_THREAD; i++) {
            const int k = tid + i * nt;
            g[i] = make_float2(0.f, 0.f);
            if (k <= half) {
                float2 D0, D1;
                split_packed(z[__ldg(a.perm + k)], z[__ldg(a.perm + (k == 0 ? 0 : L - k))], D0, D1);
                g[i] = cross_spectrum(D0, D1);
                gmax = fmaxf(gmax, sqrtf(g[i].x * g[i].x + g[i].y * g[i].y));
            }
        }
        gcc_inverse(z, g, gmax, L, s_red, a.rd, a.tw);
        gcc_finish(z, L, a.perm, pair, a.xcorr, a.smoothed, a.have_prev, a.idx, a.val, s_red, s_idx);
    }
}

// ---- frt_gcc_phat_pairs on the shared-memory route.  Phase 1: one CTA per two channels (2q, 2q+1;
// an odd last channel is packed with zeros) transforms them with one complex FFT, exactly as
// gcc_phat_kernel transforms a pair, and stores both spectra D_c[k], k = 0..L/2, and whether each
// channel is constant.  Phase 2: one CTA per table entry (i, j) forms G = conj(D_i) D_j and runs
// gcc_phat_kernel's PHAT weighting, inverse transform, smoothing and peak pick.
__global__ void __launch_bounds__(GCC_THREADS, 1) gcc_spectra_kernel(const GccArgs a, const GccSpectra w) {
    extern __shared__ float2 z[];
    __shared__ float s_red[40];
    const int L = a.L;
    for (int q = blockIdx.x; 2 * q < a.n; q += gridDim.x) {
        const int c0 = 2 * q;
        const bool has1 = c0 + 1 < a.n;
        gcc_spectra_pack(z, s_red, a, a.d0 + (size_t)q * a.stride, has1 ? a.d1 + (size_t)q * a.stride : nullptr,
                         w.spec + (size_t)c0 * (L / 2 + 1), w.quiet + c0);
    }
}

__global__ void __launch_bounds__(GCC_THREADS, 1) gcc_pairs_kernel(const GccArgs a, const GccSpectra w,
                                                                   const int2 *pairs) {
    extern __shared__ float2 z[];
    __shared__ float s_red[40];
    __shared__ int s_idx[33];
    const int L = a.L, H = L / 2 + 1;
    for (int pair = blockIdx.x; pair < a.n; pair += gridDim.x) {
        const int2 ij = __ldg(pairs + pair);
        if (__ldg(w.quiet + ij.x) || __ldg(w.quiet + ij.y)) {
            gcc_silent(pair, L, a.xcorr, a.smoothed, a.have_prev, a.idx, a.val);
            continue;
        }
        float2 g[GCC_MAX_PER_THREAD];
        const float gmax = gcc_table_cross(w.spec + (size_t)ij.x * H, w.spec + (size_t)ij.y * H, L, g);
        gcc_inverse(z, g, gmax, L, s_red, a.rd, a.tw);
        gcc_finish(z, L, a.perm, pair, a.xcorr, a.smoothed, a.have_prev, a.idx, a.val, s_red, s_idx);
    }
}

// ---- frt_gcc_phat_frames / frt_gcc_phat_pairs_frames.  Phase 1 (per route) writes the raw Xcorr of
// every (frame, pair) of a group of frames and whether the pair is silent in that frame; phase 2
// (gcc_track_*, both routes) runs the smoothing chain over the frames in order, then the arg-max and
// the moments of every smoothed row.

// Phase 1's frame geometry and outputs on the shared-memory route: item i = f * n + p of a launch is
// frame f of pair (or channel pack) p, whose rows start f * frame_stride after frame 0's.  A separate
// kernel parameter, not part of GccArgs (see there).
struct GccFrames {
    long long frame_stride;
    int n_frames;
    int n_channels;            // frt_gcc_phat_pairs_frames: the channels of a frame's spectra
    float *xraw;               // [n_frames][n_pairs][L] raw Xcorr
    int *silent;               // [n_frames][n_pairs]
};

// The raw Xcorr x[n] = Re(FFT(conj Yfull))[n] / L from z, as gcc_finish forms it.
__device__ __forceinline__ void gcc_store_raw(const float2 *z, int L, const int *__restrict__ perm, float *out) {
    const float inv = 1.0f / (float)L;
    for (int n = threadIdx.x; n < L; n += blockDim.x) out[n] = z[__ldg(perm + n)].x * inv;
    __syncthreads();   // the next item rewrites z
}

// Rows d0, d1 of independent pairs, as gcc_phat_kernel.
__global__ void __launch_bounds__(GCC_THREADS, 1) gcc_frames_kernel(const GccArgs a, const GccFrames fr) {
    extern __shared__ float2 z[];
    __shared__ float s_red[40];
    const int L = a.L, items = fr.n_frames * a.n;
    for (int it = blockIdx.x; it < items; it += gridDim.x) {
        const int f = it / a.n, pair = it - f * a.n;
        const size_t off = (size_t)pair * a.stride + (size_t)f * fr.frame_stride;
        float m0, m1, span0, span1;
        gcc_load(z, a.d0 + off, a.d1 + off, L, s_red, m0, m1, span0, span1);
        const bool quiet = !(span0 > 0.f) || !(span1 > 0.f);
        if (threadIdx.x == 0) fr.silent[it] = quiet;
        if (quiet) continue;   // gcc_load's reductions ordered every read of z
        fft_inplace(z, L, a.rd, a.tw, a.window, m0, m1);
        float2 g[GCC_MAX_PER_THREAD];
        const float gmax = gcc_packed_cross(z, L, a.perm, g);
        gcc_inverse(z, g, gmax, L, s_red, a.rd, a.tw);
        gcc_store_raw(z, L, a.perm, fr.xraw + (size_t)it * L);
    }
}

// The channel packs of every frame, as gcc_spectra_kernel; frame f's spectra and flags start at
// channel f * n_channels of the workspace.
__global__ void __launch_bounds__(GCC_THREADS, 1) gcc_frames_spectra_kernel(const GccArgs a, const GccSpectra w,
                                                                            const GccFrames fr) {
    extern __shared__ float2 z[];
    __shared__ float s_red[40];
    const int C = fr.n_channels, packs = (C + 1) / 2, H = a.L / 2 + 1, items = fr.n_frames * packs;
    for (int it = blockIdx.x; it < items; it += gridDim.x) {
        const int f = it / packs, q = it - f * packs, c0 = 2 * q;
        const size_t off = (size_t)q * a.stride + (size_t)f * fr.frame_stride;
        const size_t c = (size_t)f * C + c0;
        gcc_spectra_pack(z, s_red, a, a.d0 + off, c0 + 1 < C ? a.d1 + off : nullptr, w.spec + c * H, w.quiet + c);
    }
}

// The table's entries in every frame, as gcc_pairs_kernel.
__global__ void __launch_bounds__(GCC_THREADS, 1) gcc_frames_pairs_kernel(const GccArgs a, const GccSpectra w,
                                                                          const int2 *pairs, const GccFrames fr) {
    extern __shared__ float2 z[];
    __shared__ float s_red[40];
    const int L = a.L, H = L / 2 + 1, C = fr.n_channels, items = fr.n_frames * a.n;
    for (int it = blockIdx.x; it < items; it += gridDim.x) {
        const int f = it / a.n, pair = it - f * a.n;
        const int2 ij = __ldg(pairs + pair);
        const int *quiet = w.quiet + (size_t)f * C;
        const bool silent = quiet[ij.x] || quiet[ij.y];
        if (threadIdx.x == 0) fr.silent[it] = silent;
        if (silent) continue;
        const float2 *spec = w.spec + (size_t)f * C * H;
        float2 g[GCC_MAX_PER_THREAD];
        const float gmax = gcc_table_cross(spec + (size_t)ij.x * H, spec + (size_t)ij.y * H, L, g);
        gcc_inverse(z, g, gmax, L, s_red, a.rd, a.tw);
        gcc_store_raw(z, L, a.perm, fr.xraw + (size_t)it * L);
    }
}

// Phase 2 over a group of frames, rows of Lr samples (L on this route, L' on the Bluestein route).
constexpr int GCC_TRACK_THREADS = 256;
constexpr int GCC_TRACK_PER_THREAD = 8;
constexpr int GCC_TRACK_CHUNK = GCC_TRACK_THREADS * GCC_TRACK_PER_THREAD;   // lags per partial

struct GccTrack {
    float *xs;                     // [n_frames][n_pairs][Lr]: raw Xcorr in, smoothed Xcorr out
    const int *silent;             // [n_frames][n_pairs]
    const int *prev_in;            // [n_pairs]: the pair blends its first non-silent frame of the group
    int *prev_out;                 // [n_pairs]: the same for the next group
    float *smoothed;               // [n_pairs][Lr] the smoothing state
    unsigned long long *best;      // [n_frames][n_pairs][n_chunks]: |Xs| bits << 32 | (0xffffffff - index)
    double2 *moments;              // [n_frames][n_pairs][n_chunks]: mean and sum of squared deviations
    int *idx;                      // [n_frames][n_pairs] outputs of the group
    float *val;
    double *std;
    int Lr, n_pairs, n_frames, n_chunks;
    int have_prev;                 // the call's, for frame 0
};

// Before a call's first group: whether each pair blends its first non-silent frame (frt_gcc_phat's
// have_prev rule).  Read here, before any block rewrites the NaN marker in slot 0.
__global__ void __launch_bounds__(256) gcc_track_prev(const GccTrack t, int *prev) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p < t.n_pairs)
        prev[p] = t.have_prev == 1 || (t.have_prev == 2 && !isnan(t.smoothed[(size_t)p * t.Lr]));
}

// The smoothing chain: thread n of pair p walks the group's frames in order and blends each
// non-silent one into its state, as the per-frame calls would (a pair blends once it has had a
// non-silent frame); the smoothed rows replace the raw ones.  A silent frame leaves the state alone.
__global__ void __launch_bounds__(GCC_TRACK_THREADS) gcc_track_chain(const GccTrack t) {
    const int n = blockIdx.x * blockDim.x + threadIdx.x;
    if (n >= t.Lr) return;
    const size_t fstride = (size_t)t.n_pairs * t.Lr;
    for (int p = blockIdx.y; p < t.n_pairs; p += gridDim.y) {
        bool prev = t.prev_in[p];
        float *sm = t.smoothed + (size_t)p * t.Lr;
        float cur = prev ? sm[n] : 0.f;
        float *x = t.xs + (size_t)p * t.Lr + n;
        for (int f = 0; f < t.n_frames; f++) {
            if (t.silent[(size_t)f * t.n_pairs + p]) continue;
            float v = x[f * fstride];
            if (prev) v = gcc_blend(v, cur);
            x[f * fstride] = v;
            cur = v;
            prev = true;
        }
        if (prev) sm[n] = cur;
        else if (n == 0 && t.have_prev == 0) sm[0] = nanf("");   // no non-silent frame yet: "no previous"
        if (n == 0) t.prev_out[p] = prev;
    }
}

// Per (frame, pair, chunk of GCC_TRACK_CHUNK lags) of a non-silent row: the first maximum of |Xs| and
// the chunk's mean and sum of squared deviations, in double.
__global__ void __launch_bounds__(GCC_TRACK_THREADS) gcc_track_stats(const GccTrack t) {
    __shared__ double s_red[33];
    __shared__ unsigned long long s_best[GCC_TRACK_THREADS / 32];
    const int it = blockIdx.x, c = blockIdx.y;
    if (t.silent[it]) return;
    const float *row = t.xs + (size_t)it * t.Lr;
    const int n0 = c * GCC_TRACK_CHUNK, cnt = min(GCC_TRACK_CHUNK, t.Lr - n0);
    float v[GCC_TRACK_PER_THREAD];
    double s = 0.0;
    unsigned long long best = 0ull;
#pragma unroll
    for (int i = 0; i < GCC_TRACK_PER_THREAD; i++) {
        const int k = threadIdx.x + i * GCC_TRACK_THREADS;
        v[i] = 0.f;
        if (k < cnt) {
            v[i] = row[n0 + k];
            s += (double)v[i];
            const unsigned long long key =
                ((unsigned long long)__float_as_uint(fabsf(v[i])) << 32) | (0xffffffffu - (unsigned)(n0 + k));
            best = key > best ? key : best;
        }
    }
    const double mean = block_sum(s, s_red) / (double)cnt;
    double m2 = 0.0;
#pragma unroll
    for (int i = 0; i < GCC_TRACK_PER_THREAD; i++) {
        const double d = (double)v[i] - mean;
        if (threadIdx.x + i * GCC_TRACK_THREADS < cnt) m2 += d * d;
    }
    m2 = block_sum(m2, s_red);
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long ob = __shfl_xor_sync(0xffffffffu, best, o);
        best = ob > best ? ob : best;
    }
    if ((threadIdx.x & 31) == 0) s_best[threadIdx.x >> 5] = best;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < GCC_TRACK_THREADS / 32; w++) best = s_best[w] > best ? s_best[w] : best;
        const size_t o = (size_t)it * t.n_chunks + c;
        t.best[o] = best;
        t.moments[o] = make_double2(mean, m2);
    }
}

// Per (frame, pair): the chunks combined in index order (Chan et al.'s pairwise update of the
// moments), so the result depends on the length alone; silent rows give (0, 0, 0).
__global__ void __launch_bounds__(256) gcc_track_finish(const GccTrack t) {
    const int it = blockIdx.x * blockDim.x + threadIdx.x;
    if (it >= t.n_frames * t.n_pairs) return;
    if (t.silent[it]) {
        t.idx[it] = 0;
        t.val[it] = 0.f;
        t.std[it] = 0.0;
        return;
    }
    const unsigned long long *b = t.best + (size_t)it * t.n_chunks;
    const double2 *m = t.moments + (size_t)it * t.n_chunks;
    unsigned long long best = 0ull;
    double n = 0.0, mean = 0.0, m2 = 0.0;
    for (int c = 0; c < t.n_chunks; c++) {
        best = b[c] > best ? b[c] : best;
        const double nb = (double)min(GCC_TRACK_CHUNK, t.Lr - c * GCC_TRACK_CHUNK), nn = n + nb;
        const double2 mc = m[c];
        const double d = mc.x - mean;
        mean += d * (nb / nn);
        m2 += mc.y + d * d * (n * nb / nn);
        n = nn;
    }
    const int bi = (int)(0xffffffffu - (unsigned)(best & 0xffffffffull));
    t.idx[it] = bi;
    t.val[it] = t.xs[(size_t)it * t.Lr + bi];
    t.std[it] = sqrt(m2 / n);
}

}   // namespace

struct GccPlan {
    int L = 0;
    DeviceArray<float> window;
    DeviceArray<float2> tw;
    DeviceArray<int> perm;
    GccRadices rd;
};

void PlanDelete::operator()(GccPlan *p) const { delete p; }

// The lengths this kernel takes, and their pass sequence: NULL when `length` is accepted, else why not.
static const char *gcc_rule(int length, GccRadices &rd) {
    if (!(length >= 4 && (length % 2) == 0)) return "length must be even and >= 4";
    if (!((size_t)length * sizeof(float2) <= 220 * 1024))
        return "length too large for the shared-memory FFT (max 28160)";
    if (!((length / 2 + 1 + GCC_THREADS - 1) / GCC_THREADS <= GCC_MAX_PER_THREAD)) return "length too large";
    rd.n_passes = 0;
    int n = length;
    // large composite radices first (16 = 4x4, 25 = 5x5, 15 = 3x5 run in registers): every pass
    // is a full sweep over the 8*L-byte shared-memory buffer
    while (n % 16 == 0 && rd.n_passes < GCC_MAX_PASSES) { rd.radix[rd.n_passes++] = 16; n /= 16; }
    while (n % 4 == 0 && rd.n_passes < GCC_MAX_PASSES) { rd.radix[rd.n_passes++] = 4; n /= 4; }
    while (n % 2 == 0 && rd.n_passes < GCC_MAX_PASSES) { rd.radix[rd.n_passes++] = 2; n /= 2; }
    while (n % 25 == 0 && rd.n_passes < GCC_MAX_PASSES) { rd.radix[rd.n_passes++] = 25; n /= 25; }
    while (n % 15 == 0 && rd.n_passes < GCC_MAX_PASSES) { rd.radix[rd.n_passes++] = 15; n /= 15; }
    while (n % 5 == 0 && rd.n_passes < GCC_MAX_PASSES) { rd.radix[rd.n_passes++] = 5; n /= 5; }
    while (n % 3 == 0 && rd.n_passes < GCC_MAX_PASSES) { rd.radix[rd.n_passes++] = 3; n /= 3; }
    if (n != 1) return "length is not of the form 2^a 3^b 5^c";
    return nullptr;
}

extern "C" int frt_gcc_fits(int length) {
    GccRadices rd;
    return gcc_rule(length, rd) == nullptr;
}

std::vector<float> gcc_hanning(int length) {
    const double PI = 3.14159265358979323846;
    std::vector<float> win(length);
    for (int i = 0; i < length; i++)   // 0.5 - 0.5 cos(2 pi n / (L-1))   (correlation.py:31)
        win[i] = (float)(0.5 - 0.5 * cos(2.0 * PI * i / (double)(length - 1)));
    return win;
}

// The shared-memory route's plan for a length gcc_rule accepted, with its pass sequence rd.
static int gcc_smem_plan(frt_ctx *h, int length, GccRadices rd) {
    if (h->gcc && h->gcc->L == length) return FRT_OK;
    {
        int nn = length;
        for (int i = 0; i < rd.n_passes; i++) {
            const int n_next = nn / rd.radix[i];
            rd.magic[i] = n_next > 1 ? (unsigned)((0x100000000ULL + n_next - 1) / n_next) : 0u;
            nn = n_next;
        }
    }
    PlanPtr<GccPlan> pl(new (std::nothrow) GccPlan());
    if (!pl) return frt_fail(h, FRT_ENOMEM, "out of host memory");
    pl->L = length;
    pl->rd = rd;
    const double PI = 3.14159265358979323846;
    std::vector<float2> tw(length);
    for (int i = 0; i < length; i++) {
        const double ang = -2.0 * PI * (double)i / (double)length;
        tw[i] = make_float2((float)cos(ang), (float)sin(ang));
    }
    std::vector<int> perm(length);
    for (int i = 0; i < length; i++) perm[i] = digit_reverse(i, length, rd);
    FRT_CUDA(h, pl->window.upload(gcc_hanning(length)));
    FRT_CUDA(h, pl->perm.upload(perm));
    FRT_CUDA(h, pl->tw.upload(tw));
    h->gcc = std::move(pl);
    return FRT_OK;
}

extern "C" int frt_gcc_plan(frt_handle h, int length) {
    if (!h) return FRT_EINVAL;
    DeviceGuard g(h->device);
    GccRadices rd;
    const bool fits = gcc_rule(length, rd) == nullptr;
    const int rc = fits ? gcc_smem_plan(h, length, rd) : gcc_long_plan(h, length);
    if (rc == FRT_OK) {
        h->gcc_long_route = !fits;
        h->gcc_length = length;
    }
    return rc;
}

// The checks frt_gcc_phat and frt_gcc_phat_pairs share, after each one's own state checks: a plan,
// n_pairs, and unless there are no pairs (nothing to do) the buffers (`inputs`: the entry point's
// input pointers are all set), the row stride and have_prev.  L is the planned length.
static int gcc_call_checks(frt_ctx *h, const char *fn, int n_pairs, bool inputs, int64_t stride, int have_prev,
                           const float *smoothed_dev, const int *idx_dev, const float *val_dev, int &L) {
    L = h->gcc_length;
    if (L == 0) return frt_fail(h, FRT_ESTATE, "%s: call frt_gcc_plan first", fn);
    FRT_CHECK_ARG(h, n_pairs >= 0, "negative n_pairs");
    if (n_pairs == 0) return FRT_OK;
    FRT_CHECK_ARG(h, inputs && idx_dev && val_dev, "NULL buffer");
    FRT_CHECK_ARG(h, stride >= L, "stride smaller than the frame length");
    FRT_CHECK_ARG(h, have_prev >= 0 && have_prev <= 2, "have_prev must be 0, 1 or 2");
    FRT_CHECK_ARG(h, !have_prev || smoothed_dev, "have_prev needs the smoothed buffer");
    return FRT_OK;
}

// The shared-memory kernels' arguments from the plan and the call's outputs; the inputs are left to
// the caller.
static GccArgs gcc_args(const GccPlan *pl, float *xcorr_dev, float *smoothed_dev, int have_prev, int *idx_dev,
                        float *val_dev) {
    GccArgs a{};
    a.L = pl->L;
    a.window = pl->window.get();
    a.tw = pl->tw.get();
    a.perm = pl->perm.get();
    a.rd = pl->rd;
    a.xcorr = xcorr_dev;
    a.smoothed = smoothed_dev;
    a.have_prev = have_prev;
    a.idx = idx_dev;
    a.val = val_dev;
    return a;
}

extern "C" int frt_gcc_phat(frt_handle h, const float *d0_dev, const float *d1_dev, int64_t stride,
                            int n_pairs, float *xcorr_dev, float *smoothed_dev, int have_prev,
                            int *idx_dev, float *val_dev, void *stream) {
    if (!h) return FRT_EINVAL;
    int L;
    const int rc = gcc_call_checks(h, "frt_gcc_phat", n_pairs, d0_dev && d1_dev, stride, have_prev, smoothed_dev,
                                   idx_dev, val_dev, L);
    if (rc != FRT_OK || n_pairs == 0) return rc;
    DeviceGuard g(h->device);
    const cudaStream_t st = (cudaStream_t)stream;
    if (h->gcc_long_route)
        return gcc_long_phat(h, d0_dev, d1_dev, stride, n_pairs, xcorr_dev, smoothed_dev, have_prev, idx_dev,
                             val_dev, st);
    GccArgs a = gcc_args(h->gcc.get(), xcorr_dev, smoothed_dev, have_prev, idx_dev, val_dev);
    a.d0 = d0_dev;
    a.d1 = d1_dev;
    a.stride = stride;
    a.n = n_pairs;
    return frt_launch(h, gcc_phat_kernel, std::min(n_pairs, h->sm_count), GCC_THREADS, sizeof(float2) * L, st, a);
}

extern "C" int frt_gcc_set_pairs(frt_handle h, int n_channels, const int *pairs_host, int n_pairs) {
    if (!h) return FRT_EINVAL;
    FRT_CHECK_ARG(h, n_channels >= 1, "n_channels must be >= 1");
    FRT_CHECK_ARG(h, n_pairs >= 0, "negative n_pairs");
    FRT_CHECK_ARG(h, n_pairs == 0 || pairs_host, "NULL pair table");
    for (int p = 0; p < 2 * n_pairs; p++)
        if (pairs_host[p] < 0 || pairs_host[p] >= n_channels)
            return frt_fail(h, FRT_EINVAL, "pair %d: channel %d outside 0 .. %d", p / 2, pairs_host[p],
                            n_channels - 1);
    DeviceGuard g(h->device);
    DeviceArray<int2> table;
    if (n_pairs > 0) {
        std::vector<int2> t(n_pairs);
        for (int p = 0; p < n_pairs; p++) t[p] = make_int2(pairs_host[2 * p], pairs_host[2 * p + 1]);
        FRT_CUDA(h, table.upload(t));
    } else {
        FRT_CUDA(h, cudaDeviceSynchronize());   // no queued call still reads the table freed below
    }
    h->gcc_pairs = std::move(table);
    h->gcc_pairs_n = n_pairs;
    h->gcc_pairs_channels = n_channels;
    return FRT_OK;
}

// The spectrum workspace of frt_gcc_phat_pairs: [C][H] float2 spectra and [C] int flags.  Grow-only.
static int gcc_spectra_workspace(frt_ctx *h, int H, GccSpectra &w) {
    const size_t C = (size_t)h->gcc_pairs_channels;
    WsLayout l;
    const size_t o_spec = l.add(C * H * sizeof(float2)), o_quiet = l.add(C * sizeof(int));
    FRT_CUDA(h, h->gcc_spec_ws.grow(l.bytes));
    w.spec = (float2 *)(h->gcc_spec_ws.get() + o_spec);
    w.quiet = (int *)(h->gcc_spec_ws.get() + o_quiet);
    return FRT_OK;
}

extern "C" int frt_gcc_phat_pairs(frt_handle h, const float *x_dev, int64_t stride, float *xcorr_dev,
                                  float *smoothed_dev, int have_prev, int *idx_dev, float *val_dev,
                                  void *stream) {
    if (!h) return FRT_EINVAL;
    if (h->gcc_pairs_n < 0) return frt_fail(h, FRT_ESTATE, "frt_gcc_phat_pairs: call frt_gcc_set_pairs first");
    // the stride is checked right after the plan, so a short one is refused even with an empty table
    // (with no plan, gcc_call_checks refuses the call first)
    int L = h->gcc_length;
    if (L > 0) FRT_CHECK_ARG(h, stride >= L, "stride smaller than the frame length");
    const int n_pairs = h->gcc_pairs_n;
    int rc = gcc_call_checks(h, "frt_gcc_phat_pairs", n_pairs, x_dev != nullptr, stride, have_prev, smoothed_dev,
                             idx_dev, val_dev, L);
    if (rc != FRT_OK || n_pairs == 0) return rc;
    DeviceGuard g(h->device);
    const cudaStream_t st = (cudaStream_t)stream;
    GccSpectra w;
    rc = gcc_spectra_workspace(h, (L - (L & 1)) / 2 + 1, w);
    if (rc != FRT_OK) return rc;
    if (h->gcc_long_route)
        return gcc_long_phat_pairs(h, x_dev, stride, w, xcorr_dev, smoothed_dev, have_prev, idx_dev, val_dev, st);
    // phase 1: pair q packs channels 2q and 2q+1, rows x + 2q*stride and x + (2q+1)*stride
    GccArgs a = gcc_args(h->gcc.get(), xcorr_dev, smoothed_dev, have_prev, idx_dev, val_dev);
    a.d0 = x_dev;
    a.d1 = x_dev + stride;
    a.stride = 2 * stride;
    a.n = h->gcc_pairs_channels;
    rc = frt_launch(h, gcc_spectra_kernel, std::min((a.n + 1) / 2, h->sm_count), GCC_THREADS, sizeof(float2) * L,
                    st, a, w);
    a.n = n_pairs;
    if (rc == FRT_OK)
        rc = frt_launch(h, gcc_pairs_kernel, std::min(n_pairs, h->sm_count), GCC_THREADS, sizeof(float2) * L, st, a,
                        w, h->gcc_pairs.get());
    return rc;
}

// ---- frt_gcc_phat_frames / frt_gcc_phat_pairs_frames

// The frames entry points' own checks, after gcc_call_checks.  `work`: false when there is nothing to
// do (no pairs or no frames).
static int gcc_frames_checks(frt_ctx *h, int n_pairs, int n_frames, int64_t frame_stride, const float *smoothed_dev,
                             const double *std_dev, bool &work) {
    work = false;
    FRT_CHECK_ARG(h, n_frames >= 0, "negative n_frames");
    if (n_pairs == 0 || n_frames == 0) return FRT_OK;
    FRT_CHECK_ARG(h, n_frames == 1 || frame_stride >= 1, "frame_stride must be >= 1");
    FRT_CHECK_ARG(h, smoothed_dev && std_dev, "NULL buffer");
    work = true;
    return FRT_OK;
}

// Frames run in groups whose workspace (raw and smoothed rows, flags, partials and, for the pair table
// on the shared-memory route, the frames' spectra) fits this budget; at least one frame per group.
constexpr size_t GCC_TRACK_BUDGET = size_t(2) << 30;

// The workspace of a frames call, grow-only: groups of `group` frames of n_pairs rows of Lr samples,
// plus spec_channels spectra of H bins per frame.  t gets its buffers and the call's constants; prev is
// the two [n_pairs] halves the groups alternate between.
static int gcc_track_workspace(frt_ctx *h, int n_pairs, int n_frames, int Lr, int spec_channels, int H,
                               GccTrack &t, int *&prev, GccSpectra &w, int &group) {
    const size_t P = (size_t)n_pairs, C = (size_t)spec_channels;
    const int nc = (Lr + GCC_TRACK_CHUNK - 1) / GCC_TRACK_CHUNK;
    const size_t per_frame = P * ((size_t)Lr * sizeof(float) + sizeof(int) +
                                  (size_t)nc * (sizeof(unsigned long long) + sizeof(double2))) +
                             C * ((size_t)H * sizeof(float2) + sizeof(int));
    const size_t fixed = WsLayout::round(2 * P * sizeof(int)) + 7 * 256;
    const size_t g = frt_group_size(GCC_TRACK_BUDGET > fixed ? GCC_TRACK_BUDGET - fixed : 0, per_frame, n_frames);
    WsLayout l;
    const size_t o_xs = l.add(g * P * Lr * sizeof(float)), o_sil = l.add(g * P * sizeof(int)),
                 o_best = l.add(g * P * nc * sizeof(unsigned long long)), o_mom = l.add(g * P * nc * sizeof(double2)),
                 o_prev = l.add(2 * P * sizeof(int)), o_spec = l.add(g * C * H * sizeof(float2)),
                 o_quiet = l.add(g * C * sizeof(int));
    FRT_CUDA(h, h->gcc_track_ws.grow(l.bytes));
    unsigned char *ws = h->gcc_track_ws.get();
    t = GccTrack{};
    t.xs = (float *)(ws + o_xs);
    t.silent = (const int *)(ws + o_sil);
    t.best = (unsigned long long *)(ws + o_best);
    t.moments = (double2 *)(ws + o_mom);
    t.Lr = Lr;
    t.n_pairs = n_pairs;
    t.n_chunks = nc;
    prev = (int *)(ws + o_prev);
    if (C) {
        w.spec = (float2 *)(ws + o_spec);
        w.quiet = (int *)(ws + o_quiet);
    }
    group = (int)g;
    return FRT_OK;
}

// Both entry points after their checks: per group of frames, phase1(f0, nf, xraw, silent) writes the
// raw rows and flags of frames f0 .. f0+nf-1, then phase 2 smooths them in order and reduces them.
template <class Phase1>
static int gcc_frames_run(frt_ctx *h, int n_pairs, int n_frames, int Lr, int spec_channels, int H, float *smoothed_dev,
                          int have_prev, int *idx_dev, float *val_dev, double *std_dev, cudaStream_t st, GccSpectra &w,
                          Phase1 phase1) {
    GccTrack t;
    int *prev = nullptr, group = 0;
    int rc = gcc_track_workspace(h, n_pairs, n_frames, Lr, spec_channels, H, t, prev, w, group);
    if (rc != FRT_OK) return rc;
    t.smoothed = smoothed_dev;
    t.have_prev = have_prev;
    rc = frt_launch(h, gcc_track_prev, (n_pairs + 255) / 256, 256, 0, st, t, prev);
    const unsigned row_blocks = (unsigned)((Lr + GCC_TRACK_THREADS - 1) / GCC_TRACK_THREADS);
    for (int f0 = 0, g = 0; f0 < n_frames && rc == FRT_OK; f0 += group, g++) {
        const int nf = std::min(group, n_frames - f0);
        rc = phase1(f0, nf, t.xs, const_cast<int *>(t.silent));
        t.n_frames = nf;
        t.prev_in = prev + (size_t)(g & 1) * n_pairs;
        t.prev_out = prev + (size_t)((g + 1) & 1) * n_pairs;
        t.idx = idx_dev + (size_t)f0 * n_pairs;
        t.val = val_dev + (size_t)f0 * n_pairs;
        t.std = std_dev + (size_t)f0 * n_pairs;
        const int items = nf * n_pairs;
        if (rc == FRT_OK)
            rc = frt_launch(h, gcc_track_chain, dim3(row_blocks, std::min(n_pairs, 65535)), GCC_TRACK_THREADS, 0, st,
                            t);
        if (rc == FRT_OK)
            rc = frt_launch(h, gcc_track_stats, dim3(items, t.n_chunks), GCC_TRACK_THREADS, 0, st, t);
        if (rc == FRT_OK) rc = frt_launch(h, gcc_track_finish, (items + 255) / 256, 256, 0, st, t);
    }
    return rc;
}

extern "C" int frt_gcc_phat_frames(frt_handle h, const float *d0_dev, const float *d1_dev, int64_t stride,
                                   int64_t frame_stride, int n_frames, int n_pairs, float *smoothed_dev,
                                   int have_prev, int *idx_dev, float *val_dev, double *std_dev, void *stream) {
    if (!h) return FRT_EINVAL;
    int L;
    bool work;
    int rc = gcc_call_checks(h, "frt_gcc_phat_frames", n_pairs, d0_dev && d1_dev, stride, have_prev, smoothed_dev,
                             idx_dev, val_dev, L);
    if (rc == FRT_OK) rc = gcc_frames_checks(h, n_pairs, n_frames, frame_stride, smoothed_dev, std_dev, work);
    if (rc != FRT_OK || !work) return rc;
    DeviceGuard g(h->device);
    const cudaStream_t st = (cudaStream_t)stream;
    const int Lr = L - (L & 1);
    GccSpectra w{};
    if (h->gcc_long_route)
        return gcc_frames_run(h, n_pairs, n_frames, Lr, 0, 0, smoothed_dev, have_prev, idx_dev, val_dev, std_dev, st, w,
                              [&](int f0, int nf, float *xraw, int *silent) {
                                  int r = FRT_OK;
                                  for (int f = 0; f < nf && r == FRT_OK; f++) {
                                      const size_t off = (size_t)(f0 + f) * frame_stride, o = (size_t)f * n_pairs;
                                      // idx / val of the frame's rows are scratch until phase 2 fills them
                                      r = gcc_long_phat(h, d0_dev + off, d1_dev + off, stride, n_pairs, xraw + o * Lr,
                                                        nullptr, 0, idx_dev + (size_t)f0 * n_pairs + o,
                                                        val_dev + (size_t)f0 * n_pairs + o, st, silent + o);
                                  }
                                  return r;
                              });
    GccArgs a = gcc_args(h->gcc.get(), nullptr, nullptr, 0, nullptr, nullptr);
    a.stride = stride;
    a.n = n_pairs;
    return gcc_frames_run(h, n_pairs, n_frames, Lr, 0, 0, smoothed_dev, have_prev, idx_dev, val_dev, std_dev, st, w,
                          [&](int f0, int nf, float *xraw, int *silent) {
                              a.d0 = d0_dev + (size_t)f0 * frame_stride;
                              a.d1 = d1_dev + (size_t)f0 * frame_stride;
                              const GccFrames fr{frame_stride, nf, 0, xraw, silent};
                              return frt_launch(h, gcc_frames_kernel, std::min(nf * n_pairs, h->sm_count), GCC_THREADS,
                                                sizeof(float2) * L, st, a, fr);
                          });
}

extern "C" int frt_gcc_phat_pairs_frames(frt_handle h, const float *x_dev, int64_t stride, int64_t frame_stride,
                                         int n_frames, float *smoothed_dev, int have_prev, int *idx_dev, float *val_dev,
                                         double *std_dev, void *stream) {
    if (!h) return FRT_EINVAL;
    if (h->gcc_pairs_n < 0)
        return frt_fail(h, FRT_ESTATE, "frt_gcc_phat_pairs_frames: call frt_gcc_set_pairs first");
    int L = h->gcc_length;
    if (L > 0) FRT_CHECK_ARG(h, stride >= L, "stride smaller than the frame length");
    const int n_pairs = h->gcc_pairs_n, C = h->gcc_pairs_channels;
    bool work;
    int rc = gcc_call_checks(h, "frt_gcc_phat_pairs_frames", n_pairs, x_dev != nullptr, stride, have_prev,
                             smoothed_dev, idx_dev, val_dev, L);
    if (rc == FRT_OK) rc = gcc_frames_checks(h, n_pairs, n_frames, frame_stride, smoothed_dev, std_dev, work);
    if (rc != FRT_OK || !work) return rc;
    DeviceGuard g(h->device);
    const cudaStream_t st = (cudaStream_t)stream;
    const int Lr = L - (L & 1), H = Lr / 2 + 1;
    GccSpectra w{};
    if (h->gcc_long_route) {
        rc = gcc_spectra_workspace(h, H, w);   // one frame's spectra, reused frame by frame
        if (rc != FRT_OK) return rc;
        return gcc_frames_run(h, n_pairs, n_frames, Lr, 0, 0, smoothed_dev, have_prev, idx_dev, val_dev, std_dev, st, w,
                              [&](int f0, int nf, float *xraw, int *silent) {
                                  int r = FRT_OK;
                                  for (int f = 0; f < nf && r == FRT_OK; f++) {
                                      const size_t off = (size_t)(f0 + f) * frame_stride, o = (size_t)f * n_pairs;
                                      r = gcc_long_phat_pairs(h, x_dev + off, stride, w, xraw + o * Lr, nullptr, 0,
                                                              idx_dev + (size_t)f0 * n_pairs + o,
                                                              val_dev + (size_t)f0 * n_pairs + o, st, silent + o);
                                  }
                                  return r;
                              });
    }
    // phase 1 as frt_gcc_phat_pairs': pack q of a frame is channels 2q and 2q+1
    GccArgs a = gcc_args(h->gcc.get(), nullptr, nullptr, 0, nullptr, nullptr);
    a.stride = 2 * stride;
    return gcc_frames_run(h, n_pairs, n_frames, Lr, C, H, smoothed_dev, have_prev, idx_dev, val_dev, std_dev, st, w,
                          [&](int f0, int nf, float *xraw, int *silent) {
                              a.d0 = x_dev + (size_t)f0 * frame_stride;
                              a.d1 = a.d0 + stride;
                              const GccFrames fr{frame_stride, nf, C, xraw, silent};
                              a.n = C;
                              int r = frt_launch(h, gcc_frames_spectra_kernel, std::min(nf * ((C + 1) / 2), h->sm_count),
                                                 GCC_THREADS, sizeof(float2) * L, st, a, w, fr);
                              a.n = n_pairs;
                              if (r == FRT_OK)
                                  r = frt_launch(h, gcc_frames_pairs_kernel, std::min(nf * n_pairs, h->sm_count),
                                                 GCC_THREADS, sizeof(float2) * L, st, a, w, h->gcc_pairs.get(), fr);
                              return r;
                          });
}
