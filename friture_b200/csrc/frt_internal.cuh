// Internal declarations shared by the translation units of libfrt_b200.so.
#pragma once

#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <map>
#include <string>
#include <vector>

#include "../../include/frt.h"

struct StftPlan {
    int n_fft = 0;
    float *win_dev = nullptr;      // [n_fft] symmetric Hann (audioproc.py:76-81)
    float2 *tw_dev = nullptr;      // N = 64..2048: [M/32][32] W_M^(k1*t); N >= 4096: [32][32] W_1024^(k1*t);
                                   // N = 32: [M] W_M^k
    float2 *post_dev = nullptr;    // U[k] = -j*W_N^k (real-FFT split twiddles), as many as the kernels read
    float4 *wlane_dev = nullptr;   // N = 4096/8192: per-(warp, lane) Hann phase factors
    float2 *comb_dev = nullptr;    // N >= 4096: [(R-1)][1024] W_M^(w k0)
    std::vector<float> win_host;
};
void frt_stft_free_plan(StftPlan &pl);   // frees the plan's device tables

struct HostPipe {                 // staging for the *_host entry points
    cudaStream_t s_in = nullptr, s_cmp = nullptr, s_out = nullptr;
    float *d_in[2] = {nullptr, nullptr};
    float *d_out[2] = {nullptr, nullptr};
    size_t in_bytes = 0, out_bytes = 0;
    cudaEvent_t ev_in[2] = {nullptr, nullptr}, ev_cmp[2] = {nullptr, nullptr},
                ev_out[2] = {nullptr, nullptr};
};

struct BankPlan;   // bank.cu
struct GccPlan;    // gcc_phat.cu

struct frt_ctx {
    int device = 0;
    int sm_count = 0;
    int64_t launches = 0;
    std::string err;
    StftPlan stft;                       // current plan (a copy of one cache entry)
    std::map<int, StftPlan> stft_cache;  // every size planned so far owns its device tables
    HostPipe pipe;
    BankPlan *bank = nullptr;
    GccPlan *gcc = nullptr;
    void *dec = nullptr;          // DecPlan (bank.cu)
    void *comb = nullptr;         // CombPipe (combined.cu)
    void *fir = nullptr;          // FirPlan (bank_fir.cu)
};

int frt_fail(frt_ctx *h, int code, const char *fmt, ...);

#define FRT_CUDA(h, call)                                                                  \
    do {                                                                                   \
        cudaError_t e__ = (call);                                                          \
        if (e__ != cudaSuccess)                                                            \
            return frt_fail((h), FRT_ECUDA, "%s failed: %s (%s:%d)", #call,                \
                            cudaGetErrorString(e__), __FILE__, __LINE__);                  \
    } while (0)

#define FRT_CHECK_ARG(h, cond, msg)                                                        \
    do {                                                                                   \
        if (!(cond)) return frt_fail((h), FRT_EINVAL, "%s (%s)", msg, #cond);              \
    } while (0)

// Each entry point runs on the handle's device.
struct DeviceGuard {
    int prev = -1;
    explicit DeviceGuard(int dev) {
        cudaGetDevice(&prev);
        if (prev != dev) cudaSetDevice(dev);
        else prev = -1;
    }
    ~DeviceGuard() {
        if (prev >= 0) cudaSetDevice(prev);
    }
};

// Component-wise float2 arithmetic (sm_90 has no packed FP32 instructions: one scalar FADD / FMUL /
// FFMA per component).  Plain operators on purpose: the compiler contracts a product that feeds a
// sum into one FFMA (e.g. the Hann window into the first butterfly), one rounding fewer, and the
// parity margins of the STFT kernels rest on that.
__device__ __forceinline__ float2 f2_add(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ float2 f2_mul(float2 a, float2 b) { return make_float2(a.x * b.x, a.y * b.y); }
__device__ __forceinline__ float2 f2_fma(float2 a, float2 b, float2 c) {
    return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y));
}

// bank.cu / gcc_phat.cu clean-up hooks
void frt_bank_release(frt_ctx *h);
void frt_gcc_release(frt_ctx *h);
void frt_dec_release(frt_ctx *h);
void frt_comb_release(frt_ctx *h);
void frt_fir_release(frt_ctx *h);
int frt_pipe_ensure(frt_ctx *h, size_t in_bytes, size_t out_bytes);
