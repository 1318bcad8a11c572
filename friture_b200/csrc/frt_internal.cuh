// Internal declarations shared by the translation units of libfrt_b200.so.
#pragma once

#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <map>
#include <memory>
#include <string>
#include <utility>
#include <vector>

#include "../../include/frt.h"

// ---- owning types.  Device memory, streams and events are released only by these destructors;
// they run inside the caller's DeviceGuard (frt_destroy holds one).
struct CudaFree {
    void operator()(void *p) const { cudaFree(p); }
};
struct StreamDestroy {
    void operator()(cudaStream_t s) const { cudaStreamDestroy(s); }
};
struct EventDestroy {
    void operator()(cudaEvent_t e) const { cudaEventDestroy(e); }
};

// Every host-side write to or read of device memory that is not ordered on a caller's stream (plans,
// setters, resets, state checkpoints) goes through these two.  A kernel of this handle may still be
// queued on any stream, blocking or not, and must run with what it saw when it was queued, so the
// device is drained first.  The device is drained again afterwards: a pageable host-to-device
// cudaMemcpy may return before the data has landed, and a kernel launched next on a non-blocking
// stream would not wait for it.
inline cudaError_t frt_sync_copy(void *dst, const void *src, size_t bytes, cudaMemcpyKind kind) {
    cudaError_t e = cudaDeviceSynchronize();
    if (e == cudaSuccess) e = cudaMemcpy(dst, src, bytes, kind);
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    return e;
}
inline cudaError_t frt_sync_zero(void *dst, size_t bytes) {
    cudaError_t e = cudaDeviceSynchronize();
    if (e == cudaSuccess) e = cudaMemset(dst, 0, bytes);
    if (e == cudaSuccess) e = cudaDeviceSynchronize();
    return e;
}

// Every allocation's status passes through here.  The runtime may also keep a failure as its last
// error, which would fail the next launch's check (frt_launch): clear it, and keep its size for FRT_CUDA.
inline thread_local size_t frt_refused_bytes = 0;
inline cudaError_t frt_alloc_status(cudaError_t e, size_t bytes) {
    if (e != cudaSuccess) {
        cudaGetLastError();
        frt_refused_bytes = bytes;
    }
    return e;
}
inline cudaError_t frt_malloc(void **p, size_t bytes) { return frt_alloc_status(cudaMalloc(p, bytes), bytes); }

// One cudaMalloc allocation of n elements of T, or none.  Move-only.
template <class T>
struct DeviceArray {
    std::unique_ptr<T[], CudaFree> p;
    size_t n = 0;

    T *get() const { return p.get(); }
    cudaError_t alloc(size_t count) {   // frees what it held first
        p.reset();
        n = 0;
        T *d = nullptr;
        cudaError_t e = frt_malloc((void **)&d, sizeof(T) * count);
        if (e != cudaSuccess) return e;
        p.reset(d);
        n = count;
        return cudaSuccess;
    }
    cudaError_t upload(const std::vector<T> &host) {
        cudaError_t e = alloc(host.size());
        if (e != cudaSuccess) return e;
        return frt_sync_copy(get(), host.data(), sizeof(T) * host.size(), cudaMemcpyHostToDevice);
    }
    // staging: reallocates only when a call needs more than it holds, so steady-state calls do not
    cudaError_t grow(size_t count) { return count <= n ? cudaSuccess : alloc(count); }
};

// The regions of a grow-only workspace, in order, each rounded up to 256 bytes: add returns a region's
// offset, and `bytes` is the size to grow the workspace to.
struct WsLayout {
    size_t bytes = 0;
    static size_t round(size_t region) { return (region + 255) & ~size_t(255); }
    size_t add(size_t region) { return std::exchange(bytes, bytes + round(region)); }
};

// How many items of per_item bytes a group of a call holds within `budget`: at least one, at most n.
inline size_t frt_group_size(size_t budget, size_t per_item, size_t n) {
    const size_t g = budget / per_item;
    return g < 1 ? 1 : g > n ? n : g;
}

struct Stream {   // non-blocking
    std::unique_ptr<CUstream_st, StreamDestroy> s;
    cudaStream_t get() const { return s.get(); }
    cudaError_t create() {
        cudaStream_t r = nullptr;
        cudaError_t e = cudaStreamCreateWithFlags(&r, cudaStreamNonBlocking);
        if (e == cudaSuccess) s.reset(r);
        return e;
    }
};

struct Event {    // timing disabled
    std::unique_ptr<CUevent_st, EventDestroy> ev;
    cudaEvent_t get() const { return ev.get(); }
    cudaError_t create() {
        cudaEvent_t r = nullptr;
        cudaError_t e = cudaEventCreateWithFlags(&r, cudaEventDisableTiming);
        if (e == cudaSuccess) ev.reset(r);
        return e;
    }
};

// Staging of a *_host entry point: streams for the H2D copies, the kernels and the D2H copies, NEV
// events of each kind between them, created on the first call; the device buffers grow as needed.
template <int NEV>
struct HostStaging {
    Stream s_in, s_cmp, s_out;
    Event ev_in[NEV], ev_cmp[NEV], ev_out[NEV];

    cudaError_t create() {
        if (ev_out[NEV - 1].get()) return cudaSuccess;   // created last: the set is complete
        cudaError_t e = s_in.create();
        if (e == cudaSuccess) e = s_cmp.create();
        if (e == cudaSuccess) e = s_out.create();
        for (int i = 0; i < NEV && e == cudaSuccess; i++) {
            e = ev_in[i].create();
            if (e == cudaSuccess) e = ev_cmp[i].create();
            if (e == cudaSuccess) e = ev_out[i].create();
        }
        return e;
    }
};

// frt_stft_process_host: chunks alternate between two input and two output buffers
struct StftStaging : HostStaging<2> {
    DeviceArray<float> d_in[2], d_out[2];
};

// frt_combined_process_host: one event of each kind per time segment
constexpr int COMB_MAX_SEG = 32;
struct CombStaging : HostStaging<COMB_MAX_SEG> {
    DeviceArray<float> d_x, d_spec, d_bands;
};

struct StftPlan {
    int n_fft = 0;
    DeviceArray<float> win_dev;     // [n_fft] symmetric Hann (audioproc.py:76-81)
    DeviceArray<float2> tw_dev;     // N = 64..2048: [M/32][32] W_M^(k1*t); N >= 4096: [32][32] W_1024^(k1*t);
                                    // N = 32: [M] W_M^k
    DeviceArray<float2> post_dev;   // U[k] = -j*W_N^k (real-FFT split twiddles), as many as the kernels read
    DeviceArray<float4> wlane_dev;  // N = 4096/8192: per-(warp, lane) Hann phase factors
    DeviceArray<float2> comb_dev;   // N >= 4096: [(R-1)][1024] W_M^(w k0)
    std::vector<float> win_host;
};

// The other plans are private to their .cu files; each defines its deleter next to the struct.
struct BankPlan;   // bank_internal.cuh
struct DecPlan;    // bank.cu
struct FirPlan;    // bank_fir.cu
struct GccPlan;    // gcc_phat.cu
struct GccLongPlan;   // gcc_long.cu
struct LevelsPlan;    // levels.cu
struct LongLevelsPlan;   // levels.cu
struct PlanDelete {
    void operator()(BankPlan *p) const;
    void operator()(DecPlan *p) const;
    void operator()(FirPlan *p) const;
    void operator()(GccPlan *p) const;
    void operator()(GccLongPlan *p) const;
    void operator()(LevelsPlan *p) const;
    void operator()(LongLevelsPlan *p) const;
};
template <class Plan>
using PlanPtr = std::unique_ptr<Plan, PlanDelete>;

// GCC-PHAT: frt_gcc_plan / frt_gcc_phat (gcc_phat.cu) run lengths the shared-memory kernel cannot
// hold on the Bluestein route of gcc_long.cu.  gcc_long_phat expects the arguments checked.
std::vector<float> gcc_hanning(int length);   // numpy.hanning(length), evaluated in double
int gcc_long_plan(frt_ctx *h, int length);
// silent_dev: NULL or [n_pairs], whether each pair had a constant input (the frames entry points'
// phase 1 on this route).
int gcc_long_phat(frt_ctx *h, const float *d0_dev, const float *d1_dev, int64_t stride, int n_pairs,
                  float *xcorr_dev, float *smoothed_dev, int have_prev, int *idx_dev, float *val_dev,
                  cudaStream_t st, int *silent_dev = nullptr);
// frt_gcc_phat_pairs: the spectra of the table's n_channels channels, D_c[k] for k = 0..L'/2, and
// whether each channel is constant.
struct GccSpectra {
    float2 *spec;
    int *quiet;
};
int gcc_long_phat_pairs(frt_ctx *h, const float *x_dev, int64_t stride, const GccSpectra &w, float *xcorr_dev,
                        float *smoothed_dev, int have_prev, int *idx_dev, float *val_dev, cudaStream_t st,
                        int *silent_dev = nullptr);

// A plan call builds into a local PlanPtr and moves it into its slot only on success, so a call
// that fails leaves the previous plan of that kind in place.
struct frt_ctx {
    int device = 0;
    int sm_count = 0;
    size_t smem_optin = 0;            // cudaDeviceProp::sharedMemPerBlockOptin of the device
    int64_t launches = 0;
    std::string err;
    std::map<int, StftPlan> stft_cache;  // every size planned so far
    const StftPlan *stft = nullptr;      // current plan: an entry of stft_cache (std::map keeps it in place)
    PlanPtr<BankPlan> bank;
    PlanPtr<DecPlan> dec;
    PlanPtr<FirPlan> fir;
    PlanPtr<GccPlan> gcc;             // frt_gcc_plan keeps one plan of each route, so that switching
    PlanPtr<GccLongPlan> gcc_long;    // lengths back and forth rebuilds neither
    bool gcc_long_route = false;      // the last accepted frt_gcc_plan length runs on gcc_long
    int gcc_length = 0;               // that length; 0 before the first accepted plan
    DeviceArray<unsigned char> gcc_long_ws;   // the Bluestein route's workspace, grow-only
    DeviceArray<int2> gcc_pairs;      // frt_gcc_set_pairs: the pair table (i, j) on the device
    int gcc_pairs_n = -1;             // its entries; -1 before the first accepted table
    int gcc_pairs_channels = 0;       // the channels of the input it indexes
    DeviceArray<unsigned char> gcc_spec_ws;   // frt_gcc_phat_pairs' per-channel spectra, grow-only
    DeviceArray<unsigned char> gcc_track_ws;  // frt_gcc_phat_frames / _pairs_frames' frame groups, grow-only
    PlanPtr<LevelsPlan> levels;       // the meter's buffer weights and per-channel state
    PlanPtr<LongLevelsPlan> longlevels;   // the long-term levels' filter taps and per-channel state
    DeviceArray<unsigned char> spec_ticks_ws;  // frt_spectrum_reduce_ticks / _dual_ticks' state rows, grow-only
    StftStaging stft_host;
    CombStaging comb_host;
};

int frt_fail(frt_ctx *h, int code, const char *fmt, ...);

// FRT_CUDA's failure: FRT_ENOMEM when memory ran out, else FRT_ECUDA; a refused allocation's size.
inline int frt_cuda_fail(frt_ctx *h, cudaError_t e, const char *call, const char *file, int line) {
    const int code = e == cudaErrorMemoryAllocation ? FRT_ENOMEM : FRT_ECUDA;
    if (const size_t bytes = std::exchange(frt_refused_bytes, 0))
        return frt_fail(h, code, "%s failed: %s, %zu bytes asked for (%s:%d)", call, cudaGetErrorString(e), bytes,
                        file, line);
    return frt_fail(h, code, "%s failed: %s (%s:%d)", call, cudaGetErrorString(e), file, line);
}

#define FRT_CUDA(h, call)                                                                  \
    do {                                                                                   \
        cudaError_t e__ = (call);                                                          \
        if (e__ != cudaSuccess) return frt_cuda_fail((h), e__, #call, __FILE__, __LINE__); \
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

// Without an opt-in a kernel may use 48 KiB of shared memory, static and dynamic together.  No kernel
// here declares more than 1 KiB of static shared memory (400 B at most), so launches up to 47 KiB of
// dynamic shared memory need no opt-in.
constexpr size_t FRT_SMEM_NO_OPT_IN = 47 * 1024;

// Every kernel launch of the library: kernel<<<grid, block, smem, st>>>(args...), reported through
// frt_fail and counted in frt_launch_count once it has been accepted.  A launch above
// FRT_SMEM_NO_OPT_IN first sets the kernel's dynamic shared-memory limit to exactly what it asks for.
// The limit is a per-device attribute of the kernel, shared by every handle: the values set are all
// above FRT_SMEM_NO_OPT_IN, so a launch that sets none never finds the limit below its need.
template <class... Params, class... Args>
int frt_launch(frt_ctx *h, void (*kernel)(Params...), dim3 grid, dim3 block, size_t smem, cudaStream_t st,
               Args &&...args) {
    if (smem > FRT_SMEM_NO_OPT_IN) {
        const cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) {
            cudaGetLastError();   // the runtime also keeps it as the last error: the next launch must not see it
            return frt_fail(h, FRT_ECUDA, "cudaFuncSetAttribute(%zu bytes of dynamic shared memory) failed: %s",
                            smem, cudaGetErrorString(e));
        }
    }
    kernel<<<grid, block, smem, st>>>(std::forward<Args>(args)...);
    const cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) return frt_fail(h, FRT_ECUDA, "kernel launch failed: %s", cudaGetErrorString(e));
    h->launches++;
    return FRT_OK;
}

// Component-wise float2 arithmetic (sm_90 has no packed FP32 instructions: one scalar FADD / FMUL /
// FFMA per component).  Plain operators on purpose: the compiler contracts a product that feeds a
// sum into one FFMA (e.g. the Hann window into the first butterfly), one rounding fewer, and the
// parity margins of the STFT kernels rest on that.
__device__ __forceinline__ float2 f2_add(float2 a, float2 b) { return make_float2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ float2 f2_mul(float2 a, float2 b) { return make_float2(a.x * b.x, a.y * b.y); }
__device__ __forceinline__ float2 f2_fma(float2 a, float2 b, float2 c) {
    return make_float2(fmaf(a.x, b.x, c.x), fmaf(a.y, b.y, c.y));
}

// MUFU.LG2.  Every caller's argument is >= 1e-30 (normal), so the denormal fix-up of __log2f is not
// needed.
__device__ __forceinline__ float lg2_fast(float v) {
    float r;
    asm("lg2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(v));
    return r;
}
constexpr float kLog10Scale = 3.01029995663981195f;   // 10 / log2(10): 10 log10(v) = kLog10Scale log2(v)

// One screen row of a log-power column: np.interp between bins i0 and i0+1 of
// (dB + w - spec_min) / (spec_max - spec_min) (friture/spectrogram.py:127-129,161-162;
// friture/signal/frequency_resampler.py:67-83), unclipped.  The column is read from global memory
// through the read-only path (display_kernel) or, SMEM, from the STFT kernels' shared-memory column
// (stft.cu).
template <bool SMEM = false>
__device__ __forceinline__ float screen_value(const float *__restrict__ col, const float *__restrict__ weight,
                                              int i0, float t, float spec_min, float inv_range) {
    auto ld = [](const float *p) {
        if constexpr (SMEM) return *p;
        else return __ldg(p);
    };
    float a = ld(col + i0), b = ld(col + i0 + 1);
    if (weight) {
        a += __ldg(weight + i0);
        b += __ldg(weight + i0 + 1);
    }
    a = (a - spec_min) * inv_range;
    b = (b - spec_min) * inv_range;
    return fmaf(t, b - a, a);
}

// ---- the spectrum widget's per-bin arithmetic, shared by the reduction kernels (reduce.cu) and the
// STFT kernels' smoothing output (stft.cu), so that both produce the same bits.
//
// One frame of exponential smoothing, s <- alpha x + (1-alpha) s (friture/signal/exp_smoothing.py:59-107),
// as s + alpha (x - s) in double.  In float32, (1-alpha) rounded biases the fixed point by about
// eps/alpha, and rounding every frame walks s off by about eps/sqrt(alpha): 1e-4 and 4e-6 of the peak at
// N = 32, T = 5 s (alpha = 3.5e-5).  The callers round s to float32 once per tick.
__device__ __forceinline__ double smooth_step(double s, float x, double a) { return fma(a, (double)x - s, s); }

// dB of one smoothed bin, 10 log10(sp + 1e-30) + weight (friture/spectrum.py:95-101,171).  The product
// and the sum are rounded separately, as the widget's NumPy does.
__device__ __forceinline__ float db_single(float sp, const float *__restrict__ weight, int k) {
    float v = __fmul_rn(kLog10Scale, lg2_fast(sp + 1e-30f));
    if (weight) v = __fadd_rn(v, __ldg(weight + k));
    return v;
}

// The transfer function 10 log10(sp2 + 1e-30) - 10 log10(sp1 + 1e-30) (spectrum.py:168-169), as the
// log of the ratio in double: two float32 dB values near -160 dB carry an ulp of 1.5e-5 dB each, and a
// silent reference against a loud measurement gives a ratio past the float32 range (1e10 / 1e-30).
__device__ __forceinline__ float db_dual(float sp1, float sp2) {
    return (float)(10.0 * log10(((double)sp2 + 1e-30) / ((double)sp1 + 1e-30)));
}

// Term k of the 3-harmonic product spectrum of the float32 smoothed power sp (spectrum.py:103-123), in
// double: a float32 product of three quiet bins (power 1e-16) underflows to 0 and the arg-max falls to
// index 0.  T is float (a stored row) or double (a row of float32 values held in double).
template <class T>
__device__ __forceinline__ double hps_term(const T *sp, int k) {
    return __dmul_rn(__dmul_rn((double)sp[k], (double)sp[2 * k]), (double)sp[3 * k]);
}

// The first arg-max: the larger value, the lower index on a tie.
__device__ __forceinline__ void argmax_merge(double &best, int &besti, double ob, int oi) {
    if (ob > best || (ob == best && oi < besti)) {
        best = ob;
        besti = oi;
    }
}

// cp.async: global -> shared copies that bypass the registers, waited for by commit group
__device__ __forceinline__ unsigned smem_u32(const void *p) {
    return (unsigned)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void cp_async4(void *smem, const void *gmem) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"(smem_u32(smem)), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async8(void *smem, const void *gmem) {
    asm volatile("cp.async.ca.shared.global [%0], [%1], 8;" ::"r"(smem_u32(smem)), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async16(void *smem, const void *gmem) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(smem_u32(smem)), "l"(gmem) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
template <int N> __device__ __forceinline__ void cp_async_wait() {   // all but the N newest groups landed
    asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}
