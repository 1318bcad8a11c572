// The Bluestein route of frt_gcc_plan / frt_gcc_phat (gcc_phat.cu), for the frames its
// shared-memory kernel cannot hold: any length L = 4 .. 24 000 000, odd or even -- the delay
// widget's ranges 0.1 s .. 1000 s give L = int(2 * range * 12000)
// (friture/delay_estimator.py:114-117,222-226).  Same numerics as gcc_phat_kernel
// (correlation.py:24-43, delay_estimator.py:129-142); for odd L numpy's irfft(W*G) has L' = L-1
// points, and everything after the forward transform is L' long.
//
//   u = (d0 - mean) hann + j (d1 - mean) hann      Z = DFT_L(u)          (one complex transform)
//   D0/D1 from Z[k], conj Z[L-k];  G = conj(D0) D1, k = 0..L'/2;  Y = G / (1e-10 max|G| + |G|)
//   x = Re DFT_L'(conj Yfull) / L'   (the conjugate trick of gcc_phat.cu; Yfull Hermitian)
//
// Both DFTs are Bluestein (chirp-z) transforms: DFT_N(v)[k] = c_k (v c (*) conj c)[k] with
// c_n = exp(-j pi n^2 / N), the circular convolution done by a power-of-two FFT of M = 2^m >= 2L-1
// points, m <= 26.  The chirps (n^2 mod 2N in int64, evaluated in double) and the filter spectrum
// B^ = FFT_M(conj c, wrapped) (a double-precision host FFT) are built once per plan and stored as
// float2.
//
// FFT_M is four-step, M = M1 * M2, n = M2 n1 + n2, k = k1 + M1 k2, and each transform costs three
// passes over the pair's M-point workspace, each one read and one write:
//   columns:  M1-point FFTs over n1 for C adjacent n2 (strided loads), times W_M^(n2 k1); the chirped,
//             windowed input (or the PHAT-weighted spectrum) is formed in the loads.  Output is in
//             transposed order, row k1 holding k2.
//   rows:     M2-point FFT over n2 (row k1 contiguous), times B^ (stored in this pass's order, so no
//             transpose pass exists), inverse M2-point FFT back to n2, times W_M^(-n2 k1).
//   columns:  inverse M1-point FFTs over k1, which brings natural order back; the output chirp and
//             1/M are applied in the store, and the last pass also smooths and picks the peak.
// The sub-FFTs run in shared memory: radix-4 decimation in frequency (a radix-2 pass when log2 N is
// odd) whose outputs land in bit-reversed order, and for the inverse in the row pass the exact
// transposed passes (decimation in time), which take bit-reversed input back to natural order.
//
// Per-pair reductions that cross CTAs: the means are partial sums over fixed chunks, summed in a
// fixed order by one CTA; max|G| and the arg-max are maxima, combined with atomicMax on their bit
// patterns (exact and order-free).  So a pair's results are the same bits run to run and whatever
// the number of pairs per call.
#include <algorithm>
#include <cmath>
#include <complex>
#include <new>
#include <vector>

#include "frt_internal.cuh"
#include "fft_radix.cuh"

namespace {

constexpr int GL_THREADS = 512;
constexpr int GL_LOG_TILE = 13;                // a column or row CTA transforms at least 2^13 points
constexpr int GL_MAX_LOG1 = 12;                // M1 <= 4096 columns' points, so M2 <= 16384 at m = 26
constexpr int GL_MAX_LOG_M = 26;
constexpr int GL_MAX_LENGTH = 24000000;        // the widget's 1000 s range at 12 kHz
constexpr int GL_STATS_CHUNK = 16384;          // samples per partial sum of the means
// Pairs run in groups whose workspace (8 M + 8 (L'/2 + 1) bytes per pair, plus a few bytes of
// partial sums) fits this budget; at least one pair per group.
constexpr size_t GL_WORKSPACE_BUDGET = size_t(2) << 30;
constexpr int GL_MAX_GROUP = 65535;            // gridDim.y

struct PairState {
    float m0, m1;
    int silent, prev;
    unsigned gmax;             // max|G| as float bits: non-negative floats order like their bits
    unsigned quiet;            // bit 0: d0 is constant, bit 1: d1 is constant
    unsigned long long best;   // bits of |Xs| << 32 | (0xffffffff - index): the max is the first maximum
};

struct GlArgs {
    const float *d0, *d1;      // the group's first pair
    long long stride;
    int L, Lp;                 // forward length, inverse length (L - 1 for odd L)
    int log1, log2;            // M1 = 2^log1 column points, M2 = 2^log2 row points
    int lgc, lgr;              // log2 of the columns per column CTA / rows per row CTA
    int tw_shift;              // W_M^e = tw_hi[e >> tw_shift] * tw_lo[e & (2^tw_shift - 1)]
    int n_chunks;
    const float *window;       // [L] numpy.hanning(L)
    const float2 *chirp;       // [L] or [L'] chirp of the transform this pass belongs to
    const float2 *bt;          // [M] its filter spectrum, row k1 = M1 bins in bit-reversed k2 order
    const float2 *tw_sub;      // [M2] W_M2^i
    const float2 *tw_lo, *tw_hi;
    float scale;               // 1/M (forward transform), 1/(M L') (inverse)
    float2 *buf;               // [group][M] workspace
    float2 *g;                 // [group][L'/2+1] cross-spectrum G
    float *part;               // [group][n_chunks][6] partial sums / maxima of the inputs
    PairState *st;             // [group]
    float *xcorr, *smoothed;   // the group's first pair, rows of L'
    int have_prev;
    int *idx;
    float *val;
    int *silent;               // NULL or the group's first pair: gl_finish's silent flags
    // frt_gcc_phat_pairs.  Phase 1 (a group of packed channel pairs d0 = channel ch0 + 2p, d1 = the next
    // one, read as zeros past the last channel): per_channel = 1, so that a pair is skipped only when
    // both channels are constant, and the spectra and flags of channels < n_ch land in spec / quiet.
    // Phase 2 (a group of table entries): pair p correlates channels pairs[p].
    int per_channel, ch0, n_ch;
    float2 *spec;              // [n_ch][L'/2+1]
    int *quiet;                // [n_ch]
    const int2 *pairs;
};

__device__ __forceinline__ float2 conj2(float2 a) { return make_float2(a.x, -a.y); }
__device__ __forceinline__ int brev(int k, int bits) { return (int)(__brev((unsigned)k) >> (32 - bits)); }
// Whether the pair blends with its smoothed row.  have_prev: 1 = every pair; 2 = the pairs without the
// "no previous" NaN in slot 0.  Read before the last pass rewrites slot 0.
__device__ __forceinline__ int gl_prev(const GlArgs &a, int pair) {
    return a.have_prev == 1 || (a.have_prev == 2 && !isnan(a.smoothed[(size_t)pair * a.Lp]));
}
// Whether the pair has a d1: in phase 1 of frt_gcc_phat_pairs an odd last channel has no partner.
__device__ __forceinline__ bool gl_has_d1(const GlArgs &a, int pair) {
    return !a.per_channel || a.ch0 + 2 * pair + 1 < a.n_ch;
}
// A pair's state before its transforms: means, constant flags (bit 0: d0, bit 1: d1), whether it is
// skipped -- in phase 1 of frt_gcc_phat_pairs only when both channels are constant -- and whether it
// blends with its smoothed row; max|G| and the peak still to come.
__device__ __forceinline__ void gl_init_state(const GlArgs &a, int pair, float m0, float m1, unsigned quiet) {
    const int silent = a.per_channel ? quiet == 3u : quiet != 0u;
    a.st[pair] = PairState{m0, m1, silent, gl_prev(a, pair), 0u, quiet, 0ull};
}
__device__ __forceinline__ float2 tw_m(const GlArgs &a, unsigned e) {
    return cmul(__ldg(a.tw_hi + (e >> a.tw_shift)), __ldg(a.tw_lo + (e & ((1u << a.tw_shift) - 1u))));
}

// cnt sequences of N = 2^logN points at s[c*sst + i], transformed in place: natural order in,
// bit-reversed order out.  INV: conjugated butterflies and twiddles, i.e. N times the inverse DFT.
// A radix-4 pass stores its outputs 0,1,2,3 at quarters 0,2,1,3, so that the mixed radix-4/2
// passes leave index k at bit-reversed position brev(k).  tws[i] = W_(2^tws_log)^i, N <= 2^tws_log.
template <bool INV>
__device__ void smem_dif(float2 *s, int logN, int cnt, int sst, const float2 *__restrict__ tws, int tws_log) {
    for (int lg = logN; lg > 0;) {
        const int r_lg = lg >= 2 ? 2 : 1;
        const int nn_lg = lg - r_lg, n_next = 1 << nn_lg;
        const int per_lg = logN - r_lg;             // butterflies per sequence: 2^per_lg
        const int total = cnt << per_lg;
        const int tsh = tws_log - lg;               // W_n^x = tws[x << tsh]
        for (int t = threadIdx.x; t < total; t += blockDim.x) {
            const int c = t >> per_lg, b = t & ((1 << per_lg) - 1);
            const int blk = b >> nn_lg, j = b & (n_next - 1);
            float2 *p = s + c * sst + (blk << lg) + j;
            if (r_lg == 2) {
                float2 v[4];
#pragma unroll
                for (int q = 0; q < 4; q++) v[q] = INV ? conj2(p[q * n_next]) : p[q * n_next];
                dft<4>(v);
                float2 w1 = __ldg(tws + (j << tsh)), w2 = __ldg(tws + ((2 * j) << tsh)),
                       w3 = __ldg(tws + ((3 * j) << tsh));
                if (INV) {
#pragma unroll
                    for (int q = 0; q < 4; q++) v[q] = conj2(v[q]);
                    w1 = conj2(w1); w2 = conj2(w2); w3 = conj2(w3);
                }
                p[0] = v[0];
                p[2 * n_next] = cmul(v[1], w1);
                p[n_next] = cmul(v[2], w2);
                p[3 * n_next] = cmul(v[3], w3);
            } else {   // n = 2: the last pass, no twiddle
                float2 v[2] = {p[0], p[1]};
                dft<2>(v);
                p[0] = v[0];
                p[1] = v[1];
            }
        }
        __syncthreads();
        lg = nn_lg;
    }
}

// The exact inverse of smem_dif<false> up to the factor N: each pass transposed, run in reverse
// order.  Bit-reversed order in, natural order out.
__device__ void smem_dit_inv(float2 *s, int logN, int cnt, int sst, const float2 *__restrict__ tws, int tws_log) {
    for (int lg = (logN & 1) ? 1 : 2; lg <= logN; lg += 2) {
        const int r_lg = lg == 1 ? 1 : 2;
        const int nn_lg = lg - r_lg, n_next = 1 << nn_lg;
        const int per_lg = logN - r_lg;
        const int total = cnt << per_lg;
        const int tsh = tws_log - lg;
        for (int t = threadIdx.x; t < total; t += blockDim.x) {
            const int c = t >> per_lg, b = t & ((1 << per_lg) - 1);
            const int blk = b >> nn_lg, j = b & (n_next - 1);
            float2 *p = s + c * sst + (blk << lg) + j;
            if (r_lg == 2) {
                const float2 w1 = __ldg(tws + (j << tsh)), w2 = __ldg(tws + ((2 * j) << tsh)),
                             w3 = __ldg(tws + ((3 * j) << tsh));
                // v[q] = conj(p[brev2(q)] * conj W^(jq)): the conjugated input of the inverse butterfly
                float2 v[4] = {conj2(p[0]), conj2(cmul(p[2 * n_next], conj2(w1))),
                               conj2(cmul(p[n_next], conj2(w2))), conj2(cmul(p[3 * n_next], conj2(w3)))};
                dft<4>(v);
#pragma unroll
                for (int q = 0; q < 4; q++) p[q * n_next] = conj2(v[q]);
            } else {
                float2 v[2] = {p[0], p[1]};
                dft<2>(v);
                p[0] = v[0];
                p[1] = v[1];
            }
        }
        __syncthreads();
    }
}

// ---- means and the silence test: partial sums over fixed chunks, then one CTA per pair
__global__ void __launch_bounds__(256) gl_stats(const GlArgs a) {
    __shared__ float s_red[33];
    const int pair = blockIdx.y;
    const float *d0 = a.d0 + (size_t)pair * a.stride, *d1 = a.d1 + (size_t)pair * a.stride;
    const bool has1 = gl_has_d1(a, pair);
    const int n0 = blockIdx.x * GL_STATS_CHUNK, n1 = min(a.L, n0 + GL_STATS_CHUNK);
    float s0 = 0.f, s1 = 0.f, mn0 = INFINITY, mx0 = -INFINITY, mn1 = INFINITY, mx1 = -INFINITY;
    for (int n = n0 + threadIdx.x; n < n1; n += blockDim.x) {
        const float u = __ldg(d0 + n), v = has1 ? __ldg(d1 + n) : 0.f;
        s0 += u;
        s1 += v;
        mn0 = fminf(mn0, u); mx0 = fmaxf(mx0, u);
        mn1 = fminf(mn1, v); mx1 = fmaxf(mx1, v);
    }
    const float r[6] = {block_sum(s0, s_red), block_sum(s1, s_red), block_max(mx0, s_red),
                        block_max(-mn0, s_red), block_max(mx1, s_red), block_max(-mn1, s_red)};
    if (threadIdx.x == 0) {
        float *o = a.part + ((size_t)pair * a.n_chunks + blockIdx.x) * 6;
        for (int i = 0; i < 6; i++) o[i] = r[i];
    }
}

__global__ void __launch_bounds__(256) gl_stats_finish(const GlArgs a) {
    __shared__ float s_red[33];
    const int pair = blockIdx.x;
    const float *p = a.part + (size_t)pair * a.n_chunks * 6;
    float v[6] = {0.f, 0.f, -INFINITY, -INFINITY, -INFINITY, -INFINITY};
    for (int c = threadIdx.x; c < a.n_chunks; c += blockDim.x) {
        v[0] += p[c * 6 + 0];
        v[1] += p[c * 6 + 1];
        for (int i = 2; i < 6; i++) v[i] = fmaxf(v[i], p[c * 6 + i]);
    }
    const float s0 = block_sum(v[0], s_red), s1 = block_sum(v[1], s_red);
    const float span0 = block_max(v[2], s_red) + block_max(v[3], s_red);
    const float span1 = block_max(v[4], s_red) + block_max(v[5], s_red);
    // constant inputs (std == 0) are skipped by the reference (delay_estimator.py:129-131)
    if (threadIdx.x == 0)
        gl_init_state(a, pair, s0 / (float)a.L, s1 / (float)a.L, (span0 > 0.f ? 0u : 1u) | (span1 > 0.f ? 0u : 2u));
}

// ---- column pass of a forward transform.  PHAT = false: the first transform's input
// (x - mean) * hann * chirp of the two channels as one complex sequence; true: the second
// transform's input conj(Yfull) * chirp', Y = G / (1e-10 max|G| + |G|) formed from the stored G.
template <bool PHAT>
__global__ void __launch_bounds__(GL_THREADS) gl_cols_fwd(const GlArgs a) {
    extern __shared__ float2 s[];
    const int pair = blockIdx.y;
    const PairState st = a.st[pair];
    if (st.silent) return;
    const int C = 1 << a.lgc, M1 = 1 << a.log1, sst = M1 + 1;   // +1: columns start in different banks
    const int col0 = blockIdx.x << a.lgc;
    const float *d0 = a.d0 + (size_t)pair * a.stride, *d1 = a.d1 + (size_t)pair * a.stride;
    const bool has1 = PHAT || gl_has_d1(a, pair);
    const float2 *g = a.g + (size_t)pair * (a.Lp / 2 + 1);
    const int half = a.Lp / 2;
    const float floor_ = 1e-10f * __uint_as_float(st.gmax);
    for (int e = threadIdx.x; e < (C << a.log1); e += blockDim.x) {
        const int c = e & (C - 1), i = e >> a.lgc;
        const int n = (i << a.log2) + col0 + c;
        float2 v = make_float2(0.f, 0.f);
        if (!PHAT && n < a.L) {
            const float w = __ldg(a.window + n);
            const float u1 = has1 ? __ldg(d1 + n) : 0.f;
            v = cmul(make_float2((__ldg(d0 + n) - st.m0) * w, (u1 - st.m1) * w), __ldg(a.chirp + n));
        } else if (PHAT && n < a.Lp) {
            const int k = n <= half ? n : a.Lp - n;
            const float2 gk = g[k];
            const float wt = 1.0f / (floor_ + hypotf(gk.x, gk.y));
            float2 y = make_float2(gk.x * wt, gk.y * wt);
            if (k == 0 || k == half) y.y = 0.f;           // irfft ignores these imaginary parts
            if (n <= half) y.y = -y.y;                    // conj(Yfull[n]); Yfull[n] = conj Y[L'-n] above L'/2
            v = cmul(y, __ldg(a.chirp + n));
        }
        s[c * sst + i] = v;
    }
    __syncthreads();
    smem_dif<false>(s, a.log1, C, sst, a.tw_sub, a.log2);
    float2 *buf = a.buf + ((size_t)pair << (a.log1 + a.log2));
    for (int e = threadIdx.x; e < (C << a.log1); e += blockDim.x) {
        const int c = e & (C - 1), k1 = e >> a.lgc;
        const int n2 = col0 + c;
        buf[(k1 << a.log2) + n2] = cmul(s[c * sst + brev(k1, a.log1)], tw_m(a, (unsigned)(k1 * n2)));
    }
}

// ---- row pass: forward M2-point FFT, times B^, inverse M2-point FFT, times W_M^(-n2 k1)
__global__ void __launch_bounds__(GL_THREADS) gl_rows(const GlArgs a) {
    extern __shared__ float2 s[];
    const int pair = blockIdx.y;
    if (a.st[pair].silent) return;
    const int M2 = 1 << a.log2, cnt = (1 << a.lgr) << a.log2;
    const int row0 = blockIdx.x << a.lgr;
    float2 *b = a.buf + ((size_t)pair << (a.log1 + a.log2)) + ((size_t)row0 << a.log2);
    const float2 *bt = a.bt + ((size_t)row0 << a.log2);
    for (int e = threadIdx.x; e < cnt; e += blockDim.x) s[e] = b[e];
    __syncthreads();
    smem_dif<false>(s, a.log2, 1 << a.lgr, M2, a.tw_sub, a.log2);
    for (int e = threadIdx.x; e < cnt; e += blockDim.x) s[e] = cmul(s[e], __ldg(bt + e));
    __syncthreads();
    smem_dit_inv(s, a.log2, 1 << a.lgr, M2, a.tw_sub, a.log2);
    for (int e = threadIdx.x; e < cnt; e += blockDim.x) {
        const int r = e >> a.log2, n2 = e & (M2 - 1);
        b[e] = cmul(s[e], conj2(tw_m(a, (unsigned)(n2 * (row0 + r)))));
    }
}

// ---- column pass of the inverse: natural order back.  FINAL = false: Z[n] = c_n y[n] / M for
// n < L, stored in place.  FINAL = true: x[n] = Re(c'_n y[n]) / (M L') for n < L', then the
// smoothing (delay_estimator.py:134-139) and the arg-max of |Xs| (first maximum wins).
template <bool FINAL>
__global__ void __launch_bounds__(GL_THREADS) gl_cols_inv(const GlArgs a) {
    extern __shared__ float2 s[];
    __shared__ unsigned long long s_best[GL_THREADS / 32];
    const int pair = blockIdx.y;
    const PairState st = a.st[pair];
    const int C = 1 << a.lgc, M1 = 1 << a.log1, sst = M1 + 1;
    const int col0 = blockIdx.x << a.lgc;
    float *xc = a.xcorr ? a.xcorr + (size_t)pair * a.Lp : nullptr;
    if (st.silent) {
        if (FINAL && xc)
            for (int e = threadIdx.x; e < (C << a.log1); e += blockDim.x) {
                const int n = ((e >> a.lgc) << a.log2) + col0 + (e & (C - 1));
                if (n < a.Lp) xc[n] = 0.f;
            }
        return;
    }
    float2 *buf = a.buf + ((size_t)pair << (a.log1 + a.log2));
    for (int e = threadIdx.x; e < (C << a.log1); e += blockDim.x) {
        const int c = e & (C - 1), k1 = e >> a.lgc;
        s[c * sst + k1] = buf[(k1 << a.log2) + col0 + c];
    }
    __syncthreads();
    smem_dif<true>(s, a.log1, C, sst, a.tw_sub, a.log2);
    if (!FINAL) {
        for (int e = threadIdx.x; e < (C << a.log1); e += blockDim.x) {
            const int c = e & (C - 1), n1 = e >> a.lgc;
            const int n = (n1 << a.log2) + col0 + c;
            if (n < a.L) buf[n] = cscale(cmul(s[c * sst + brev(n1, a.log1)], __ldg(a.chirp + n)), a.scale);
        }
        return;
    }
    float *sm = a.smoothed ? a.smoothed + (size_t)pair * a.Lp : nullptr;
    unsigned long long best = 0ull;
    for (int e = threadIdx.x; e < (C << a.log1); e += blockDim.x) {
        const int c = e & (C - 1), n1 = e >> a.lgc;
        const int n = (n1 << a.log2) + col0 + c;
        if (n >= a.Lp) continue;
        const float2 y = s[c * sst + brev(n1, a.log1)], ch = __ldg(a.chirp + n);
        float v = fmaf(y.x, ch.x, -y.y * ch.y) * a.scale;
        if (xc) xc[n] = v;
        if (sm) {
            if (st.prev) v = gcc_blend(v, sm[n]);
            sm[n] = v;
        }
        if (!xc && !sm) buf[n].x = v;                   // where gl_finish reads the peak's value
        const unsigned long long key =
            ((unsigned long long)__float_as_uint(fabsf(v)) << 32) | (0xffffffffu - (unsigned)n);
        best = key > best ? key : best;
    }
    for (int o = 16; o > 0; o >>= 1) {
        const unsigned long long ob = __shfl_xor_sync(0xffffffffu, best, o);
        best = ob > best ? ob : best;
    }
    if ((threadIdx.x & 31) == 0) s_best[threadIdx.x >> 5] = best;
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int w = 1; w < (int)(blockDim.x >> 5); w++) best = s_best[w] > best ? s_best[w] : best;
        atomicMax(&a.st[pair].best, best);
    }
}

// ---- Hermitian split of Z into the two spectra, G = conj(D0) D1 for k = 0..L'/2, and max|G|
__global__ void __launch_bounds__(GL_THREADS) gl_split(const GlArgs a) {
    __shared__ float s_red[33];
    const int pair = blockIdx.y;
    if (a.st[pair].silent) return;
    const float2 *z = a.buf + ((size_t)pair << (a.log1 + a.log2));
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    float ag = 0.f;
    if (k <= a.Lp / 2) {
        float2 D0, D1;
        split_packed(z[k], z[k == 0 ? 0 : a.L - k], D0, D1);
        const float2 G = cross_spectrum(D0, D1);
        a.g[(size_t)pair * (a.Lp / 2 + 1) + k] = G;
        ag = hypotf(G.x, G.y);
    }
    const float m = block_max(ag, s_red);
    if (threadIdx.x == 0) atomicMax(&a.st[pair].gmax, __float_as_uint(m));
}

// ---- frt_gcc_phat_pairs, phase 1: the Hermitian split of a packed channel pair's Z into the two
// channels' spectra, and the channels' constant flags
__global__ void __launch_bounds__(GL_THREADS) gl_split_spec(const GlArgs a) {
    const int pair = blockIdx.y, c0 = a.ch0 + 2 * pair, c1 = c0 + 1;
    const PairState st = a.st[pair];
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        a.quiet[c0] = st.quiet & 1u;
        if (c1 < a.n_ch) a.quiet[c1] = (st.quiet >> 1) & 1u;
    }
    if (st.silent) return;
    const float2 *z = a.buf + ((size_t)pair << (a.log1 + a.log2));
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    const size_t H = (size_t)(a.Lp / 2 + 1);
    if (k < (int)H) {
        float2 D0, D1;
        split_packed(z[k], z[k == 0 ? 0 : a.L - k], D0, D1);
        a.spec[(size_t)c0 * H + k] = D0;
        if (c1 < a.n_ch) a.spec[(size_t)c1 * H + k] = D1;
    }
}

// ---- phase 2, per table entry (i, j): the state gl_stats_finish gives a pair; silent when a channel
// is constant
__global__ void __launch_bounds__(256) gl_pair_state(const GlArgs a, int n_pairs) {
    const int pair = blockIdx.x * blockDim.x + threadIdx.x;
    if (pair >= n_pairs) return;
    const int2 ij = a.pairs[pair];
    gl_init_state(a, pair, 0.f, 0.f, (a.quiet[ij.x] ? 1u : 0u) | (a.quiet[ij.y] ? 2u : 0u));
}

// ---- phase 2: G = conj(D_i) D_j for k = 0..L'/2 from the stored spectra, and max|G| (as gl_split)
__global__ void __launch_bounds__(GL_THREADS) gl_cross(const GlArgs a) {
    __shared__ float s_red[33];
    const int pair = blockIdx.y;
    if (a.st[pair].silent) return;
    const int2 ij = a.pairs[pair];
    const size_t H = (size_t)(a.Lp / 2 + 1);
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    float ag = 0.f;
    if (k < (int)H) {
        const float2 G = cross_spectrum(a.spec[(size_t)ij.x * H + k], a.spec[(size_t)ij.y * H + k]);
        a.g[(size_t)pair * H + k] = G;
        ag = hypotf(G.x, G.y);
    }
    const float m = block_max(ag, s_red);
    if (threadIdx.x == 0) atomicMax(&a.st[pair].gmax, __float_as_uint(m));
}

// ---- per pair: index and value of the peak; silent pairs give (0, 0)
__global__ void __launch_bounds__(256) gl_finish(const GlArgs a, int n_pairs) {
    const int pair = blockIdx.x * blockDim.x + threadIdx.x;
    if (pair >= n_pairs) return;
    const PairState st = a.st[pair];
    float *sm = a.smoothed ? a.smoothed + (size_t)pair * a.Lp : nullptr;
    if (a.silent) a.silent[pair] = st.silent;
    if (st.silent) {
        a.idx[pair] = 0;
        a.val[pair] = 0.f;
        // the reference leaves old_Xcorr alone on a silent frame; on the first call there is none
        // yet: mark the pair "no previous" (NaN in slot 0)
        if (sm && a.have_prev == 0) sm[0] = nanf("");
        return;
    }
    const int bi = (int)(0xffffffffu - (unsigned)(st.best & 0xffffffffull));
    a.idx[pair] = bi;
    a.val[pair] = sm ? sm[bi] : a.xcorr ? a.xcorr[(size_t)pair * a.Lp + bi]
                                        : a.buf[((size_t)pair << (a.log1 + a.log2)) + bi].x;
}

// ---- host: plan tables
using cd = std::complex<double>;

// In-place forward FFT of a power-of-two length, double precision (plan time only).
void fft_double(std::vector<cd> &x) {
    const size_t n = x.size();
    for (size_t i = 1, j = 0; i < n; i++) {
        size_t bit = n >> 1;
        for (; j & bit; bit >>= 1) j ^= bit;
        j ^= bit;
        if (i < j) std::swap(x[i], x[j]);
    }
    std::vector<cd> w(n / 2);
    const double PI = 3.14159265358979323846;
    for (size_t k = 0; k < n / 2; k++) w[k] = std::polar(1.0, -2.0 * PI * (double)k / (double)n);
    for (size_t len = 2; len <= n; len <<= 1) {
        const size_t h = len / 2, step = n / len;
        for (size_t i = 0; i < n; i += len)
            for (size_t j = 0; j < h; j++) {
                const cd u = x[i + j], v = x[i + j + h] * w[j * step];
                x[i + j] = u + v;
                x[i + j + h] = u - v;
            }
    }
}

// Chirp c_n = exp(-j pi n^2 / N), n < N, and B^ = FFT_M(h), h[m] = conj c_|m| wrapped, stored as
// row k1 = bins k1 + M1 k2 in bit-reversed k2 order (the order the row pass holds them in).
void bluestein_tables(int N, int log1, int log2, std::vector<float2> &chirp, std::vector<float2> &bt) {
    const double PI = 3.14159265358979323846;
    const size_t M = size_t(1) << (log1 + log2), M1 = size_t(1) << log1, M2 = size_t(1) << log2;
    std::vector<cd> c(N), h(M, cd(0.0, 0.0));
    chirp.resize(N);
    for (int n = 0; n < N; n++) {
        const long long r = ((long long)n * n) % (2LL * N);   // exact: the chirp has period 2N in n^2
        c[n] = std::polar(1.0, -PI * (double)r / (double)N);
        chirp[n] = make_float2((float)c[n].real(), (float)c[n].imag());
    }
    h[0] = std::conj(c[0]);
    for (int m = 1; m < N; m++) h[m] = h[M - m] = std::conj(c[m]);
    fft_double(h);
    bt.resize(M);
    for (size_t k1 = 0; k1 < M1; k1++)
        for (size_t k2 = 0; k2 < M2; k2++) {
            size_t r = 0;
            for (int b = 0; b < log2; b++) r |= ((k2 >> b) & 1) << (log2 - 1 - b);
            const cd v = h[k1 + M1 * k2];
            bt[k1 * M2 + r] = make_float2((float)v.real(), (float)v.imag());
        }
}

}   // namespace

struct GccLongPlan {
    int L = 0, Lp = 0, log1 = 0, log2 = 0, lgc = 0, lgr = 0, tw_shift = 0;
    DeviceArray<float> window;
    DeviceArray<float2> chirp, bt;          // forward transform, length L
    DeviceArray<float2> chirp_p, bt_p;      // inverse transform, length L' = L - 1 (odd L only)
    DeviceArray<float2> tw_sub, tw_lo, tw_hi;
};

void PlanDelete::operator()(GccLongPlan *p) const { delete p; }

int gcc_long_plan(frt_ctx *h, int length) {
    FRT_CHECK_ARG(h, length >= 4 && length <= GL_MAX_LENGTH, "length must be 4 .. 24000000");
    if (h->gcc_long && h->gcc_long->L == length) return FRT_OK;
    PlanPtr<GccLongPlan> pl(new (std::nothrow) GccLongPlan());
    if (!pl) return frt_fail(h, FRT_ENOMEM, "out of host memory");
    int log_m = 0;
    while ((1LL << log_m) < 2LL * length - 1) log_m++;
    if (log_m > GL_MAX_LOG_M) return frt_fail(h, FRT_EINVAL, "length %d needs more than 2^26 points", length);
    pl->L = length;
    pl->Lp = length - (length & 1);
    pl->log1 = log_m / 2 < GL_MAX_LOG1 ? log_m / 2 : GL_MAX_LOG1;
    pl->log2 = log_m - pl->log1;
    // columns per column CTA (>= 4: 32-byte segments of the strided loads) and rows per row CTA
    pl->lgc = std::min(pl->log2, std::max(2, GL_LOG_TILE - pl->log1));
    pl->lgr = std::min(pl->log1, std::max(0, GL_LOG_TILE - pl->log2));
    pl->tw_shift = (log_m + 1) / 2;
    try {
        const double PI = 3.14159265358979323846;
        const double M = std::ldexp(1.0, log_m);
        FRT_CUDA(h, pl->window.upload(gcc_hanning(length)));
        std::vector<float2> t(size_t(1) << pl->log2);
        for (size_t i = 0; i < t.size(); i++) {
            const double ang = -2.0 * PI * (double)i / (double)t.size();
            t[i] = make_float2((float)cos(ang), (float)sin(ang));
        }
        FRT_CUDA(h, pl->tw_sub.upload(t));
        t.resize(size_t(1) << pl->tw_shift);
        for (size_t i = 0; i < t.size(); i++) {
            const double ang = -2.0 * PI * (double)i / M;
            t[i] = make_float2((float)cos(ang), (float)sin(ang));
        }
        FRT_CUDA(h, pl->tw_lo.upload(t));
        t.resize(size_t(1) << (log_m - pl->tw_shift));
        for (size_t i = 0; i < t.size(); i++) {
            const double ang = -2.0 * PI * (double)(i << pl->tw_shift) / M;
            t[i] = make_float2((float)cos(ang), (float)sin(ang));
        }
        FRT_CUDA(h, pl->tw_hi.upload(t));
        std::vector<float2> chirp, bt;
        bluestein_tables(length, pl->log1, pl->log2, chirp, bt);
        FRT_CUDA(h, pl->chirp.upload(chirp));
        FRT_CUDA(h, pl->bt.upload(bt));
        if (pl->Lp != length) {
            bluestein_tables(pl->Lp, pl->log1, pl->log2, chirp, bt);
            FRT_CUDA(h, pl->chirp_p.upload(chirp));
            FRT_CUDA(h, pl->bt_p.upload(bt));
        }
    } catch (const std::bad_alloc &) {
        return frt_fail(h, FRT_ENOMEM, "out of host memory");
    }
    h->gcc_long = std::move(pl);
    return FRT_OK;
}

// The arguments every pass of a call shares, and its workspace: groups of pairs whose buffers fit
// GL_WORKSPACE_BUDGET, at most n_pairs.  Returns the group size through `group`.
static int gl_setup(frt_ctx *h, const GccLongPlan *pl, int n_pairs, int64_t stride, int have_prev, GlArgs &a,
                    int &group) {
    const size_t M = size_t(1) << (pl->log1 + pl->log2), H = size_t(pl->Lp / 2 + 1);
    const int n_chunks = (pl->L + GL_STATS_CHUNK - 1) / GL_STATS_CHUNK;
    const size_t per_pair = WsLayout::round(M * sizeof(float2)) + WsLayout::round(H * sizeof(float2)) +
                            WsLayout::round(n_chunks * 6 * sizeof(float)) + WsLayout::round(sizeof(PairState));
    const size_t gr = frt_group_size(GL_WORKSPACE_BUDGET, per_pair, std::min(GL_MAX_GROUP, n_pairs));
    WsLayout l;
    const size_t o_buf = l.add(gr * M * sizeof(float2)), o_g = l.add(gr * H * sizeof(float2)),
                 o_part = l.add(gr * n_chunks * 6 * sizeof(float)), o_st = l.add(gr * sizeof(PairState));
    FRT_CUDA(h, h->gcc_long_ws.grow(l.bytes));
    unsigned char *ws = h->gcc_long_ws.get();
    group = (int)gr;

    a = GlArgs{};
    a.stride = stride;
    a.L = pl->L;
    a.Lp = pl->Lp;
    a.log1 = pl->log1;
    a.log2 = pl->log2;
    a.lgc = pl->lgc;
    a.lgr = pl->lgr;
    a.tw_shift = pl->tw_shift;
    a.n_chunks = n_chunks;
    a.window = pl->window.get();
    a.tw_sub = pl->tw_sub.get();
    a.tw_lo = pl->tw_lo.get();
    a.tw_hi = pl->tw_hi.get();
    a.buf = (float2 *)(ws + o_buf);
    a.g = (float2 *)(ws + o_g);
    a.part = (float *)(ws + o_part);
    a.st = (PairState *)(ws + o_st);
    a.have_prev = have_prev;
    return FRT_OK;
}

// The forward transform of np packed pairs d0 + j d1 (means, silence, the three passes), leaving Z in
// the pairs' buffers.
static int gl_forward(frt_ctx *h, const GccLongPlan *pl, GlArgs &a, int np, cudaStream_t st) {
    const int M1 = 1 << pl->log1, M2 = 1 << pl->log2;
    const size_t smem_cols = sizeof(float2) * (size_t)(M1 + 1) << pl->lgc;
    const size_t smem_rows = sizeof(float2) * (size_t)M2 << pl->lgr;
    const dim3 g_cols(M2 >> pl->lgc, np), g_rows(M1 >> pl->lgr, np);
    a.chirp = pl->chirp.get();
    a.bt = pl->bt.get();
    a.scale = (float)(1.0 / std::ldexp(1.0, pl->log1 + pl->log2));
    int rc = frt_launch(h, gl_stats, dim3(a.n_chunks, np), 256, 0, st, a);
    if (rc == FRT_OK) rc = frt_launch(h, gl_stats_finish, np, 256, 0, st, a);
    if (rc == FRT_OK) rc = frt_launch(h, gl_cols_fwd<false>, g_cols, GL_THREADS, smem_cols, st, a);
    if (rc == FRT_OK) rc = frt_launch(h, gl_rows, g_rows, GL_THREADS, smem_rows, st, a);
    if (rc == FRT_OK) rc = frt_launch(h, gl_cols_inv<false>, g_cols, GL_THREADS, smem_cols, st, a);
    return rc;
}

// From G and max|G| of np pairs: the inverse real transform of length L' through a forward transform of
// the conjugate, the smoothing and the peak pick.
static int gl_inverse(frt_ctx *h, const GccLongPlan *pl, GlArgs &a, int np, cudaStream_t st) {
    const int M1 = 1 << pl->log1, M2 = 1 << pl->log2;
    const size_t smem_cols = sizeof(float2) * (size_t)(M1 + 1) << pl->lgc;
    const size_t smem_rows = sizeof(float2) * (size_t)M2 << pl->lgr;
    const dim3 g_cols(M2 >> pl->lgc, np), g_rows(M1 >> pl->lgr, np);
    a.chirp = pl->Lp != pl->L ? pl->chirp_p.get() : pl->chirp.get();
    a.bt = pl->Lp != pl->L ? pl->bt_p.get() : pl->bt.get();
    a.scale = (float)(1.0 / std::ldexp(1.0, pl->log1 + pl->log2) / (double)pl->Lp);
    int rc = frt_launch(h, gl_cols_fwd<true>, g_cols, GL_THREADS, smem_cols, st, a);
    if (rc == FRT_OK) rc = frt_launch(h, gl_rows, g_rows, GL_THREADS, smem_rows, st, a);
    if (rc == FRT_OK) rc = frt_launch(h, gl_cols_inv<true>, g_cols, GL_THREADS, smem_cols, st, a);
    if (rc == FRT_OK) rc = frt_launch(h, gl_finish, (np + 255) / 256, 256, 0, st, a, np);
    return rc;
}

// The outputs of the group starting at pair p0.
static void gl_outputs(const GccLongPlan *pl, GlArgs &a, int p0, float *xcorr_dev, float *smoothed_dev,
                       int *idx_dev, float *val_dev, int *silent_dev) {
    a.xcorr = xcorr_dev ? xcorr_dev + (size_t)p0 * pl->Lp : nullptr;
    a.smoothed = smoothed_dev ? smoothed_dev + (size_t)p0 * pl->Lp : nullptr;
    a.idx = idx_dev + p0;
    a.val = val_dev + p0;
    a.silent = silent_dev ? silent_dev + p0 : nullptr;
}

int gcc_long_phat(frt_ctx *h, const float *d0_dev, const float *d1_dev, int64_t stride, int n_pairs,
                  float *xcorr_dev, float *smoothed_dev, int have_prev, int *idx_dev, float *val_dev,
                  cudaStream_t st, int *silent_dev) {
    const GccLongPlan *pl = h->gcc_long.get();
    GlArgs a;
    int group = 0;
    int rc = gl_setup(h, pl, n_pairs, stride, have_prev, a, group);
    const unsigned split_blocks = (unsigned)((pl->Lp / 2 + 1 + GL_THREADS - 1) / GL_THREADS);
    for (int p0 = 0; p0 < n_pairs && rc == FRT_OK; p0 += group) {
        const int np = n_pairs - p0 < group ? n_pairs - p0 : group;
        a.d0 = d0_dev + (size_t)p0 * stride;
        a.d1 = d1_dev + (size_t)p0 * stride;
        gl_outputs(pl, a, p0, xcorr_dev, smoothed_dev, idx_dev, val_dev, silent_dev);
        rc = gl_forward(h, pl, a, np, st);
        if (rc == FRT_OK) rc = frt_launch(h, gl_split, dim3(split_blocks, np), GL_THREADS, 0, st, a);
        if (rc == FRT_OK) rc = gl_inverse(h, pl, a, np, st);
    }
    return rc;
}

int gcc_long_phat_pairs(frt_ctx *h, const float *x_dev, int64_t stride, const GccSpectra &w, float *xcorr_dev,
                        float *smoothed_dev, int have_prev, int *idx_dev, float *val_dev, cudaStream_t st,
                        int *silent_dev) {
    const GccLongPlan *pl = h->gcc_long.get();
    const int C = h->gcc_pairs_channels, n_pairs = h->gcc_pairs_n;
    const int packs = (C + 1) / 2;
    const unsigned split_blocks = (unsigned)((pl->Lp / 2 + 1 + GL_THREADS - 1) / GL_THREADS);
    GlArgs a;
    int group = 0;
    int rc = gl_setup(h, pl, packs > n_pairs ? packs : n_pairs, 2 * stride, 0, a, group);
    a.spec = w.spec;
    a.quiet = w.quiet;
    a.n_ch = C;
    // phase 1: channels 2q and 2q+1 packed as d0 + j d1 (row stride 2 * stride); the partner of an odd
    // last channel reads as zeros
    a.per_channel = 1;
    for (int q0 = 0; q0 < packs && rc == FRT_OK; q0 += group) {
        const int np = packs - q0 < group ? packs - q0 : group;
        a.ch0 = 2 * q0;
        a.d0 = x_dev + (size_t)a.ch0 * stride;
        a.d1 = a.d0 + stride;
        rc = gl_forward(h, pl, a, np, st);
        if (rc == FRT_OK) rc = frt_launch(h, gl_split_spec, dim3(split_blocks, np), GL_THREADS, 0, st, a);
    }
    // phase 2: the table's entries in groups; d0 / d1 are not read
    a.per_channel = 0;
    a.have_prev = have_prev;
    a.d0 = a.d1 = x_dev;
    for (int p0 = 0; p0 < n_pairs && rc == FRT_OK; p0 += group) {
        const int np = n_pairs - p0 < group ? n_pairs - p0 : group;
        a.pairs = h->gcc_pairs.get() + p0;
        gl_outputs(pl, a, p0, xcorr_dev, smoothed_dev, idx_dev, val_dev, silent_dev);
        rc = frt_launch(h, gl_pair_state, (np + 255) / 256, 256, 0, st, a, np);
        if (rc == FRT_OK) rc = frt_launch(h, gl_cross, dim3(split_blocks, np), GL_THREADS, 0, st, a);
        if (rc == FRT_OK) rc = gl_inverse(h, pl, a, np, st);
    }
    return rc;
}
