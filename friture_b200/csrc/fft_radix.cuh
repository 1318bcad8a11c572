// Complex float2 helpers, the radix-2/4 butterflies and the block reductions shared by the two
// GCC-PHAT paths (gcc_phat.cu: whole frame in shared memory; gcc_long.cu: Bluestein over a
// four-step power-of-two FFT in global memory).
#pragma once

#include <cuda_runtime.h>

namespace {

__device__ __forceinline__ float2 cadd(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ float2 csub(float2 a, float2 b) { return make_float2(a.x - b.x, a.y - b.y); }
__device__ __forceinline__ float2 cmul(float2 a, float2 w) {
    return make_float2(fmaf(a.x, w.x, -a.y * w.y), fmaf(a.x, w.y, a.y * w.x));
}
__device__ __forceinline__ float2 mul_mj(float2 a) { return make_float2(a.y, -a.x); }   // * (-j)
__device__ __forceinline__ float2 cscale(float2 a, float s) { return make_float2(a.x * s, a.y * s); }

// The two real sequences packed as u + j v share one complex transform Z; zk = Z[k], zm = Z[L-k]
// (Z[0] for k = 0) give their spectra D0 = (Zk + conj Zm)/2 and D1 = (Zk - conj Zm)/(2j).
__device__ __forceinline__ void split_packed(float2 zk, float2 zm, float2 &D0, float2 &D1) {
    D0 = make_float2(0.5f * (zk.x + zm.x), 0.5f * (zk.y - zm.y));
    D1 = make_float2(0.5f * (zk.y + zm.y), -0.5f * (zk.x - zm.x));
}
// The cross-spectrum G = conj(D0) D1 of GCC (correlation.py:34).
__device__ __forceinline__ float2 cross_spectrum(float2 D0, float2 D1) {
    return make_float2(D0.x * D1.x + D0.y * D1.y, D0.x * D1.y - D0.y * D1.x);
}

// The widget's temporal smoothing Xs = 0.3 X + 0.7 Xs_prev (delay_estimator.py:134-139), rounded as
// fma(0.3, X, round(0.7 Xs_prev)).  Left to the compiler, the plain expression is contracted into an
// FFMA on either product depending on the surrounding code; written out, every kernel that blends
// (gcc_finish, gl_cols_inv, gcc_track_chain) gives the same bits for the same frame.
__device__ __forceinline__ float gcc_blend(float x, float prev) { return fmaf(0.3f, x, 0.7f * prev); }

// In-register forward DFT of R points, outputs in natural order.
template <int R> __device__ __forceinline__ void dft(float2 (&v)[R]);

template <> __device__ __forceinline__ void dft<2>(float2 (&v)[2]) {
    const float2 a = v[0], b = v[1];
    v[0] = cadd(a, b);
    v[1] = csub(a, b);
}
template <> __device__ __forceinline__ void dft<4>(float2 (&v)[4]) {
    const float2 s02 = cadd(v[0], v[2]), d02 = csub(v[0], v[2]);
    const float2 s13 = cadd(v[1], v[3]), d13 = mul_mj(csub(v[1], v[3]));
    v[0] = cadd(s02, s13);
    v[1] = cadd(d02, d13);
    v[2] = csub(s02, s13);
    v[3] = csub(d02, d13);
}

// Block-wide sum / max of one float (block_sum: or double) per thread (blockDim.x a multiple of 32);
// s_red holds 33 values.  Every thread gets the result.  The combination order is fixed, so a sum is
// the same bits every run.
template <class T>
__device__ __forceinline__ T block_sum(T v, T *s_red) {
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    __syncthreads();
    if (l == 0) s_red[w] = v;
    __syncthreads();
    T t = (threadIdx.x < (blockDim.x >> 5)) ? s_red[threadIdx.x] : T(0);
    if (w == 0) {
        for (int o = 16; o > 0; o >>= 1) t += __shfl_xor_sync(0xffffffffu, t, o);
        if (l == 0) s_red[32] = t;
    }
    __syncthreads();
    return s_red[32];
}

__device__ __forceinline__ float block_max(float v, float *s_red) {
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    __syncthreads();
    if (l == 0) s_red[w] = v;
    __syncthreads();
    float t = (threadIdx.x < (blockDim.x >> 5)) ? s_red[threadIdx.x] : -INFINITY;
    if (w == 0) {
        for (int o = 16; o > 0; o >>= 1) t = fmaxf(t, __shfl_xor_sync(0xffffffffu, t, o));
        if (l == 0) s_red[32] = t;
    }
    __syncthreads();
    return s_red[32];
}

}   // namespace
