// Widget-level reductions behind the spectrum widget (SURVEY 8f-1): exponential smoothing across
// the frames of a tick, weighting, dB, arg-max and harmonic product spectrum, fused in one pass
// over the power columns.  Stands behind friture/spectrum.py:158-181 (exp_smoothed_value_2d,
// friture/signal/exp_smoothing.py:59-107; log_spectrogram spectrum.py:95-101;
// harmonic_product_spectrum spectrum.py:103-123), and in the widget's dual-channel mode the transfer
// function between a reference and a measurement channel (spectrum.py:141-182).
#include <algorithm>

#include "frt_internal.cuh"

namespace {

__device__ int block_argmax(double best, int besti, double *s_val, int *s_idx) {
    for (int o = 16; o > 0; o >>= 1) {
        const double ob = __shfl_xor_sync(0xffffffffu, best, o);
        const int oi = __shfl_xor_sync(0xffffffffu, besti, o);
        argmax_merge(best, besti, ob, oi);
    }
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    __syncthreads();
    if (l == 0) {
        s_val[w] = best;
        s_idx[w] = besti;
    }
    __syncthreads();
    if (w == 0) {
        const int nw = blockDim.x >> 5;
        best = l < nw ? s_val[l] : -INFINITY;
        besti = l < nw ? s_idx[l] : 0x7fffffff;
        for (int o = 16; o > 0; o >>= 1) {
            const double ob = __shfl_xor_sync(0xffffffffu, best, o);
            const int oi = __shfl_xor_sync(0xffffffffu, besti, o);
            argmax_merge(best, besti, ob, oi);
        }
        if (l == 0) s_idx[32] = besti;
    }
    __syncthreads();
    return s_idx[32];
}

// smooth_step across n_frames frames of one bin of NCH channels side by side (their loads in flight
// together).
template <int NCH>
__device__ __forceinline__ void smooth_frames(const float *const (&p)[NCH], long long stride_f,
                                              int n_frames, double a, double (&s)[NCH]) {
    for (int f = 0; f < n_frames; f++) {
#pragma unroll
        for (int i = 0; i < NCH; i++)
            s[i] = smooth_step(s[i], __ldg(p[i] + (size_t)f * stride_f), a);
    }
}

// One tick of smooth_frames; the carried states d are read and written back rounded to float32.
template <int NCH>
__device__ __forceinline__ void smooth_bin(const float *const (&p)[NCH], long long stride_f,
                                           int n_frames, double a, float *const (&d)[NCH],
                                           float (&out)[NCH]) {
    double s[NCH];
#pragma unroll
    for (int i = 0; i < NCH; i++) s[i] = *d[i];
    smooth_frames<NCH>(p, stride_f, n_frames, a, s);
#pragma unroll
    for (int i = 0; i < NCH; i++) {
        out[i] = (float)s[i];
        *d[i] = out[i];
    }
}

// The first arg-max of the harmonic product spectrum of sp[0 .. nbins), 3 harmonics (hps_term).
__device__ __forceinline__ int hps_argmax(const float *sp, int nbins, double *s_val, int *s_idx) {
    const int h = nbins / 3;
    double bestp = -INFINITY;
    int besti = 0x7fffffff;
    for (int k = threadIdx.x; k < h; k += blockDim.x) {
        const double r = hps_term(sp, k);
        if (r > bestp) {
            bestp = r;
            besti = k;
        }
    }
    return block_argmax(bestp, besti, s_val, s_idx);
}

// DUAL = false: one channel, dB = 10 log10(sp + 1e-30) + weight (spectrum.py:171).
// DUAL = true: one (reference, measurement) pair, both smoothed, dB = 10 log10(sp2 + 1e-30) -
// 10 log10(sp1 + 1e-30) without weighting (spectrum.py:168-169); the pitch comes from sp1 in both.
template <bool DUAL>
__global__ void __launch_bounds__(256)
spectrum_reduce_kernel(const float *__restrict__ power, const float *__restrict__ power2,
                       long long stride_c, long long stride_f, int n_frames, int nbins, float alpha,
                       float *__restrict__ disp, float *__restrict__ disp2,
                       const float *__restrict__ weight, float *__restrict__ db,
                       int *__restrict__ fmax_idx, int *__restrict__ pitch_idx) {
    extern __shared__ float s_sp[];   // [nbins] smoothed power of this channel (of sp1 when DUAL)
    __shared__ double s_val[32];
    __shared__ int s_idx[33];
    const int c = blockIdx.x;
    const float *p = power + (size_t)c * stride_c;
    float *d = disp + (size_t)c * nbins;
    const double a = alpha;
    float best = -INFINITY;
    int besti = 0x7fffffff;
    for (int k = threadIdx.x; k < nbins; k += blockDim.x) {
        float v;
        if constexpr (DUAL) {
            const float *const pk[2] = {p + k, power2 + (size_t)c * stride_c + k};
            float *const dk[2] = {d + k, disp2 + (size_t)c * nbins + k};
            float sp[2];
            smooth_bin<2>(pk, stride_f, n_frames, a, dk, sp);
            s_sp[k] = sp[0];
            v = db_dual(sp[0], sp[1]);
        } else {
            const float *const pk[1] = {p + k};
            float *const dk[1] = {d + k};
            float sp[1];
            smooth_bin<1>(pk, stride_f, n_frames, a, dk, sp);
            s_sp[k] = sp[0];
            v = db_single(sp[0], weight, k);
        }
        db[(size_t)c * nbins + k] = v;
        if (v > best) {     // on the stored float32 value, so that db[imax] == max(db)
            best = v;
            besti = k;
        }
    }
    const int imax = block_argmax(best, besti, s_val, s_idx);      // spectrum.py:175
    const int ipitch = hps_argmax(s_sp, nbins, s_val, s_idx);      // spectrum.py:180
    if (threadIdx.x == 0) {
        fmax_idx[c] = imax;
        pitch_idx[c] = ipitch;
    }
}

}   // namespace

extern "C" int frt_spectrum_reduce(frt_handle h, const float *power_dev, int64_t stride_c,
                                   int64_t stride_f, int n_channels, int n_frames, int nbins,
                                   float alpha, float *disp_dev, const float *weight_dev,
                                   float *db_dev, int *fmax_idx_dev, int *pitch_idx_dev,
                                   void *stream) {
    if (!h) return FRT_EINVAL;
    DeviceGuard g(h->device);
    FRT_CHECK_ARG(h, n_channels >= 0 && n_frames >= 0 && nbins >= 3, "bad shape");
    FRT_CHECK_ARG(h, n_frames <= 8192, "more frames than the reference's 8192-tap kernel");
    FRT_CHECK_ARG(h, alpha > 0.f && alpha <= 1.f, "alpha must be in (0, 1]");
    if (n_channels == 0) return FRT_OK;
    FRT_CHECK_ARG(h, (n_frames == 0 || power_dev) && disp_dev && db_dev && fmax_idx_dev &&
                         pitch_idx_dev, "NULL buffer");
    FRT_CHECK_ARG(h, sizeof(float) * (size_t)nbins <= 200 * 1024, "nbins too large");
    const size_t smem = sizeof(float) * (size_t)nbins;
    return frt_launch(h, spectrum_reduce_kernel<false>, n_channels, 256, smem, (cudaStream_t)stream,
                      power_dev, nullptr, stride_c, stride_f, n_frames, nbins, alpha, disp_dev, nullptr,
                      weight_dev, db_dev, fmax_idx_dev, pitch_idx_dev);
}

extern "C" int frt_spectrum_reduce_dual(frt_handle h, const float *power1_dev,
                                        const float *power2_dev, int64_t stride_c, int64_t stride_f,
                                        int n_pairs, int n_frames, int nbins, float alpha,
                                        float *disp1_dev, float *disp2_dev, float *db_dev,
                                        int *fmax_idx_dev, int *pitch_idx_dev, void *stream) {
    if (!h) return FRT_EINVAL;
    DeviceGuard g(h->device);
    FRT_CHECK_ARG(h, n_pairs >= 0 && n_frames >= 0 && nbins >= 3, "bad shape");
    FRT_CHECK_ARG(h, n_frames <= 8192, "more frames than the reference's 8192-tap kernel");
    FRT_CHECK_ARG(h, alpha > 0.f && alpha <= 1.f, "alpha must be in (0, 1]");
    if (n_pairs == 0) return FRT_OK;
    FRT_CHECK_ARG(h, (n_frames == 0 || (power1_dev && power2_dev)) && disp1_dev && disp2_dev &&
                         db_dev && fmax_idx_dev && pitch_idx_dev, "NULL buffer");
    FRT_CHECK_ARG(h, sizeof(float) * (size_t)nbins <= 200 * 1024, "nbins too large");
    const size_t smem = sizeof(float) * (size_t)nbins;
    return frt_launch(h, spectrum_reduce_kernel<true>, n_pairs, 256, smem, (cudaStream_t)stream,
                      power1_dev, power2_dev, stride_c, stride_f, n_frames, nbins, alpha, disp1_dev, disp2_dev,
                      nullptr, db_dev, fmax_idx_dev, pitch_idx_dev);
}

// ---------------------------------------------------------------------------------------------
// frt_spectrum_reduce_ticks / _dual_ticks: n_ticks consecutive ticks of frames_per_tick frames in one
// call, each tick's result kept.  The smoothing is elementwise per bin and only the arg-maxes cross
// bins, so the call runs in two kernels per group of ticks: a chain kernel walks every (channel, bin)
// through the group's frames in order, rounding its state to float32 at every tick end as
// smooth_bin does, and stores each tick's state row in the workspace; a stats kernel, one CTA per
// (tick, channel), forms that tick's dB and arg-maxes from the stored rows as spectrum_reduce_kernel
// does from its own.
namespace {

struct SpecTicks {
    const float *power[2];   // [C][frames][nbins] (strides in floats) at the group's first frame
    long long stride_c, stride_f;
    int n_channels, frames_per_tick, n_ticks, nbins;   // n_ticks: the group's
    double a;
    float *disp[2];          // [C][nbins] carried states
    float *state[2];         // [n_ticks][C][nbins] the workspace's state rows
    const float *weight;     // [nbins] or NULL (single mode)
    float *db;               // [C][R][nbins] at the group's first tick, or NULL
    int R;                   // ticks of the call: db's row count per channel
    int *fmax_idx, *pitch_idx;   // [ticks][C] at the group's first tick
};

template <int NCH>
__global__ void __launch_bounds__(256) spectrum_ticks_chain(SpecTicks t) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)t.n_channels * t.nbins) return;
    const size_t plane = (size_t)t.n_channels * t.nbins;
    const size_t o = (size_t)i;   // c * nbins + k
    const int c = (int)(i / t.nbins), k = (int)(i - (long long)c * t.nbins);
    const float *p[NCH];
    double s[NCH];
#pragma unroll
    for (int j = 0; j < NCH; j++) {
        p[j] = t.power[j] + (size_t)c * t.stride_c + k;
        s[j] = t.disp[j][o];
    }
    const size_t tick_stride = (size_t)t.frames_per_tick * t.stride_f;
    for (int r = 0; r < t.n_ticks; r++) {
        smooth_frames<NCH>(p, t.stride_f, t.frames_per_tick, t.a, s);
#pragma unroll
        for (int j = 0; j < NCH; j++) {
            const float v = (float)s[j];
            t.state[j][(size_t)r * plane + o] = v;
            s[j] = v;
            p[j] += tick_stride;
        }
    }
#pragma unroll
    for (int j = 0; j < NCH; j++) t.disp[j][o] = (float)s[j];
}

template <bool DUAL>
__global__ void __launch_bounds__(256) spectrum_ticks_stats(SpecTicks t) {
    __shared__ double s_val[32];
    __shared__ int s_idx[33];
    const int r = blockIdx.x / t.n_channels, c = blockIdx.x - r * t.n_channels;
    const size_t row = ((size_t)r * t.n_channels + c) * t.nbins;
    const float *sp = t.state[0] + row;
    float *db = t.db ? t.db + ((size_t)c * t.R + r) * t.nbins : nullptr;
    float best = -INFINITY;
    int besti = 0x7fffffff;
    for (int k = threadIdx.x; k < t.nbins; k += blockDim.x) {
        float v;
        if constexpr (DUAL) v = db_dual(__ldg(sp + k), __ldg(t.state[1] + row + k));
        else v = db_single(__ldg(sp + k), t.weight, k);
        if (db) db[k] = v;
        if (v > best) {     // on the float32 value, as spectrum_reduce_kernel
            best = v;
            besti = k;
        }
    }
    const int imax = block_argmax(best, besti, s_val, s_idx);
    const int ipitch = hps_argmax(sp, t.nbins, s_val, s_idx);
    if (threadIdx.x == 0) {
        t.fmax_idx[(size_t)r * t.n_channels + c] = imax;
        t.pitch_idx[(size_t)r * t.n_channels + c] = ipitch;
    }
}

}   // namespace

// Ticks run in groups whose state rows fit this budget; at least one tick per group.
constexpr size_t SPEC_TICKS_BUDGET = size_t(256) << 20;

// Both entry points: the checks they add to frt_spectrum_reduce's, the workspace and the groups.
// nch = 1 (single) or 2 (dual: power[1], disp[1] the measurement).  `work` is false when there is
// nothing to do.
static int spectrum_ticks_checks(frt_ctx *h, int n_channels, int frames_per_tick, int n_ticks, int nbins,
                                 float alpha, bool buffers, bool &work) {
    work = false;
    FRT_CHECK_ARG(h, n_channels >= 0 && n_ticks >= 0 && nbins >= 3, "bad shape");
    FRT_CHECK_ARG(h, frames_per_tick >= 1 && frames_per_tick <= 8192,
                  "frames_per_tick must be in 1..8192, the reference's 8192-tap kernel");
    FRT_CHECK_ARG(h, alpha > 0.f && alpha <= 1.f, "alpha must be in (0, 1]");
    if (n_channels == 0 || n_ticks == 0) return FRT_OK;
    FRT_CHECK_ARG(h, buffers, "NULL buffer");
    FRT_CHECK_ARG(h, sizeof(float) * (size_t)nbins <= 200 * 1024, "nbins too large");
    work = true;
    return FRT_OK;
}

template <int NCH>
static int spectrum_ticks_run(frt_ctx *h, SpecTicks t, int n_ticks, cudaStream_t st) {
    const size_t per_tick = NCH * (size_t)t.n_channels * t.nbins * sizeof(float);
    const size_t g = frt_group_size(SPEC_TICKS_BUDGET, per_tick, n_ticks);
    FRT_CUDA(h, h->spec_ticks_ws.grow(g * per_tick));
    float *ws = (float *)h->spec_ticks_ws.get();
    for (int j = 0; j < NCH; j++) t.state[j] = ws + (size_t)j * g * t.n_channels * t.nbins;
    const long long items = (long long)t.n_channels * t.nbins;
    const unsigned chain_blocks = (unsigned)((items + 255) / 256);
    const SpecTicks first = t;
    int rc = FRT_OK;
    for (int r0 = 0; r0 < n_ticks && rc == FRT_OK; r0 += (int)g) {
        t.n_ticks = std::min((int)g, n_ticks - r0);
        const size_t f0 = (size_t)r0 * t.frames_per_tick;
        for (int j = 0; j < NCH; j++) t.power[j] = first.power[j] + f0 * t.stride_f;
        t.db = first.db ? first.db + (size_t)r0 * t.nbins : nullptr;
        t.fmax_idx = first.fmax_idx + (size_t)r0 * t.n_channels;
        t.pitch_idx = first.pitch_idx + (size_t)r0 * t.n_channels;
        rc = frt_launch(h, spectrum_ticks_chain<NCH>, chain_blocks, 256, 0, st, t);
        if (rc == FRT_OK)
            rc = frt_launch(h, spectrum_ticks_stats<NCH == 2>, (unsigned)(t.n_ticks * t.n_channels), 256, 0, st, t);
    }
    return rc;
}

extern "C" int frt_spectrum_reduce_ticks(frt_handle h, const float *power_dev, int64_t stride_c,
                                         int64_t stride_f, int n_channels, int frames_per_tick,
                                         int n_ticks, int nbins, float alpha, float *disp_dev,
                                         const float *weight_dev, float *db_dev, int *fmax_idx_dev,
                                         int *pitch_idx_dev, void *stream) {
    if (!h) return FRT_EINVAL;
    DeviceGuard g(h->device);
    bool work;
    const int rc = spectrum_ticks_checks(h, n_channels, frames_per_tick, n_ticks, nbins, alpha,
                                         power_dev && disp_dev && fmax_idx_dev && pitch_idx_dev, work);
    if (rc != FRT_OK || !work) return rc;
    SpecTicks t{};
    t.power[0] = power_dev;
    t.stride_c = stride_c;
    t.stride_f = stride_f;
    t.n_channels = n_channels;
    t.frames_per_tick = frames_per_tick;
    t.nbins = nbins;
    t.a = alpha;
    t.disp[0] = disp_dev;
    t.weight = weight_dev;
    t.db = db_dev;
    t.R = n_ticks;
    t.fmax_idx = fmax_idx_dev;
    t.pitch_idx = pitch_idx_dev;
    return spectrum_ticks_run<1>(h, t, n_ticks, (cudaStream_t)stream);
}

extern "C" int frt_spectrum_reduce_dual_ticks(frt_handle h, const float *power1_dev,
                                              const float *power2_dev, int64_t stride_c,
                                              int64_t stride_f, int n_pairs, int frames_per_tick,
                                              int n_ticks, int nbins, float alpha, float *disp1_dev,
                                              float *disp2_dev, float *db_dev, int *fmax_idx_dev,
                                              int *pitch_idx_dev, void *stream) {
    if (!h) return FRT_EINVAL;
    DeviceGuard g(h->device);
    bool work;
    const int rc = spectrum_ticks_checks(h, n_pairs, frames_per_tick, n_ticks, nbins, alpha,
                                         power1_dev && power2_dev && disp1_dev && disp2_dev &&
                                             fmax_idx_dev && pitch_idx_dev,
                                         work);
    if (rc != FRT_OK || !work) return rc;
    SpecTicks t{};
    t.power[0] = power1_dev;
    t.power[1] = power2_dev;
    t.stride_c = stride_c;
    t.stride_f = stride_f;
    t.n_channels = n_pairs;
    t.frames_per_tick = frames_per_tick;
    t.nbins = nbins;
    t.a = alpha;
    t.disp[0] = disp1_dev;
    t.disp[1] = disp2_dev;
    t.db = db_dev;
    t.R = n_ticks;
    t.fmax_idx = fmax_idx_dev;
    t.pitch_idx = pitch_idx_dev;
    return spectrum_ticks_run<2>(h, t, n_ticks, (cudaStream_t)stream);
}

// ---------------------------------------------------------------------------------------------
// Plotted curves and peak hold of the spectrum and octave widgets (SpectrumPlotWidget.setdata and
// compute_peaks, friture/spectrumPlotWidget.py:122-200; HistPlot.setdata and compute_peaks,
// friture/histplot.py:77-130).  One CTA per channel; each bin's peak state is stepped through the
// call's dB vectors in registers, read once and written once.  All arithmetic in double with the
// rounding intrinsics, so that no contraction changes a bit against the reference's NumPy.
namespace {

// 1 - toScreen(v) on the linear vertical scale of range [m, mx] (plotting/coordinateTransform.py:
// 62-83 with length 1 and no borders: (v - m) * 1 / (mx - m) + 0); toScreen is 0 when mx == m.
__device__ __forceinline__ double screen_y(double v, double m, double mx) {
    if (mx == m) return 1.0;
    return __dsub_rn(1.0, __ddiv_rn(__dsub_rn(v, m), __dsub_rn(mx, m)));
}

__global__ void __launch_bounds__(256)
plot_curves_kernel(const float *__restrict__ y, long long stride_c, long long stride_s, int n_steps,
                   int nbins, double m, double mx, double d0, int peaks, int reset,
                   double *__restrict__ peak, double *__restrict__ peak_int,
                   double *__restrict__ decay, float *__restrict__ scaled_y, float *__restrict__ z,
                   float *__restrict__ scaled_peak, float *__restrict__ z_peak) {
    __shared__ float s_max[32];
    const int c = blockIdx.x;
    const float *yc = y + (size_t)c * stride_c;
    const float *ylast = yc + (size_t)(n_steps - 1) * stride_s;
    const size_t o = (size_t)c * nbins;
    float best = -INFINITY;
    for (int k = threadIdx.x; k < nbins; k += blockDim.x) {
        const double v = __ldg(ylast + k);
        best = fmaxf(best, (float)v);
        scaled_y[o + k] = (float)screen_y(v, m, mx);
        if (!peaks) continue;         // compute_peaks is not called: the state stays frozen
        double p = -500.0, pi = 0.0, dk = d0;     // the reset of compute_peaks
        if (!reset) {
            p = peak[o + k];
            pi = peak_int[o + k];
            dk = decay[o + k];
        }
        for (int s = 0; s < n_steps; s++) {
            const double ys = __ldg(yc + (size_t)s * stride_s + k);
            if (p < ys) {             // rise
                p = ys;
                pi = 1.0;
                dk = d0;
            } else if (pi < 0.2) {    // fall, faster every step
                p = __dadd_rn(p, dk);
                dk = __dadd_rn(dk, d0);
            } else {                  // hold
                pi = __dmul_rn(pi, 0.975);
            }
        }
        peak[o + k] = p;
        peak_int[o + k] = pi;
        decay[o + k] = dk;
        scaled_peak[o + k] = (float)screen_y(p, m, mx);
        z_peak[o + k] = (float)pi;
    }
    // M = max(y) of the last step; the max of float32 values is exact
    for (int off = 16; off > 0; off >>= 1) best = fmaxf(best, __shfl_xor_sync(0xffffffffu, best, off));
    const int w = threadIdx.x >> 5, l = threadIdx.x & 31;
    if (l == 0) s_max[w] = best;
    __syncthreads();
    if (w == 0) {
        best = l < (int)(blockDim.x >> 5) ? s_max[l] : -INFINITY;
        for (int off = 16; off > 0; off >>= 1)
            best = fmaxf(best, __shfl_xor_sync(0xffffffffu, best, off));
        if (l == 0) s_max[0] = best;
    }
    __syncthreads();
    // z = (y - m) / (|M - m| + 1e-3)
    const double den = __dadd_rn(fabs(__dsub_rn((double)s_max[0], m)), 1e-3);
    for (int k = threadIdx.x; k < nbins; k += blockDim.x)
        z[o + k] = (float)__ddiv_rn(__dsub_rn((double)__ldg(ylast + k), m), den);
}

}   // namespace

extern "C" int frt_plot_curves(frt_handle h, const float *y_dev, int64_t stride_c, int64_t stride_s,
                               int n_channels, int n_steps, int nbins, double spec_min,
                               double spec_max, double d0, int peaks, int reset, double *peak_dev,
                               double *peak_int_dev, double *decay_dev, float *scaled_y_dev,
                               float *z_dev, float *scaled_peak_dev, float *z_peak_dev,
                               void *stream) {
    if (!h) return FRT_EINVAL;
    DeviceGuard g(h->device);
    FRT_CHECK_ARG(h, n_channels >= 0 && n_steps >= 1 && nbins >= 1, "bad shape");
    // y is only read, so rows may overlap (a broadcast dB vector has stride 0)
    FRT_CHECK_ARG(h, stride_c >= 0 && stride_s >= 0, "negative stride");
    FRT_CHECK_ARG(h, spec_min <= spec_max, "spec_min > spec_max");
    if (n_channels == 0) return FRT_OK;
    FRT_CHECK_ARG(h, y_dev && scaled_y_dev && z_dev, "NULL buffer");
    FRT_CHECK_ARG(h, !peaks || (peak_dev && peak_int_dev && decay_dev && scaled_peak_dev && z_peak_dev),
                  "NULL peak buffer");
    return frt_launch(h, plot_curves_kernel, n_channels, 256, 0, (cudaStream_t)stream,
                      y_dev, stride_c, stride_s, n_steps, nbins, spec_min, spec_max, d0, peaks ? 1 : 0,
                      reset ? 1 : 0, peak_dev, peak_int_dev, decay_dev, scaled_y_dev, z_dev, scaled_peak_dev,
                      z_peak_dev);
}

// ---------------------------------------------------------------------------------------------
// Spectrogram display chain (SURVEY 8f-2): dB + weighting -> [0,1] scaling
// (friture/spectrogram.py:127-129,161-162) -> frequency-axis interpolation to the screen rows
// (np.interp on a Mel/Log/... grid, friture/signal/frequency_resampler.py:67-83) -> online linear
// resampling along time to the screen columns (friture/signal/online_linear_2D_resampler.py:61-97,
// friture/signal/linear_interp.py:11-62) -> clip + colour look-up lut[int(v*255)]
// (friture/signal/color_tranform.py:48-51, friture/signal/lookup_table.py:32-52), one kernel.
// The host works out which input column feeds which output column and with what weight (the
// resampler's scalar bookkeeping); the kernel is one thread per output pixel.
// ROWS = false: db holds log-power columns [C][n_frames][nbins] and each screen value is
// screen_value of two bins.  ROWS = true: db holds screen rows [C][n_frames][height] that
// frt_stft_screen_rows already interpolated (weight, spec_min, inv_range, row_i0 and row_t are not
// read), and the value of row r is read directly.  Both keep the same resampling expression.
namespace {

// the screen value of row r in the input column at col
template <bool ROWS>
__device__ __forceinline__ float display_value(const float *col, const float *__restrict__ weight, int r, int i0,
                                               float t, float spec_min, float inv_range) {
    if constexpr (ROWS) return __ldg(col + r);
    else return screen_value(col, weight, i0, t, spec_min, inv_range);
}

template <bool ROWS>
__global__ void display_kernel(const float *__restrict__ db, long long stride_c, long long stride_f,
                               int n_frames, const float *__restrict__ weight, float spec_min,
                               float inv_range, const int *__restrict__ row_i0,
                               const float *__restrict__ row_t, int height,
                               const int *__restrict__ out_col, const float *__restrict__ out_a,
                               int n_out, float *__restrict__ old_data,
                               const unsigned *__restrict__ lut, unsigned *__restrict__ pixels) {
    const int c = blockIdx.y;
    const long long gid = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    const long long total = (long long)height * (n_out > 0 ? n_out : 1);
    if (gid >= total) return;
    const int r = (int)(gid / (n_out > 0 ? n_out : 1));
    const int o = (int)(gid - (long long)r * (n_out > 0 ? n_out : 1));
    const float *base = db + (size_t)c * stride_c;
    const int i0 = ROWS ? 0 : __ldg(row_i0 + r);
    const float t = ROWS ? 0.f : __ldg(row_t + r);
    if (n_out > 0) {
        const int j = __ldg(out_col + o);       // input column this output column is drawn from
        const float a = __ldg(out_a + o);       // weight of the previous input column
        const float cur = display_value<ROWS>(base + (size_t)j * stride_f, weight, r, i0, t, spec_min, inv_range);
        const float old = (j > 0) ? display_value<ROWS>(base + (size_t)(j - 1) * stride_f, weight, r, i0, t,
                                                        spec_min, inv_range)
                                  : old_data[(size_t)c * height + r];
        float v = cur * (1.0f - a) + old * a;   // linear_interp.py:56-59
        v = fminf(fmaxf(v, 0.f), 1.f);          // color_tranform.py:50
        pixels[((size_t)c * height + r) * n_out + o] = __ldg(lut + (int)(v * 255.0f));
    }
    // carry the last column of this tick (online_linear_2D_resampler.py "shift"); one writer per row
    // and only after every reader of the old value is done -> done by a second launch (n_out == 0)
    if (n_out == 0 && n_frames > 0)
        old_data[(size_t)c * height + r] = display_value<ROWS>(base + (size_t)(n_frames - 1) * stride_f, weight, r,
                                                               i0, t, spec_min, inv_range);
}

// Both entry points: the pixels (n_out > 0), then the carried column in a second launch.
int display_run(frt_ctx *h, bool rows, const float *src, int64_t stride_c, int64_t stride_f, int n_channels,
                int n_frames, const float *weight, float spec_min, float inv_range, const int *row_i0,
                const float *row_t, int height, const int *out_col, const float *out_a, int n_out,
                float *old_data, const uint32_t *lut, uint32_t *pixels, cudaStream_t st) {
    auto launch = [&](auto kernel) {
        if (n_out > 0) {
            const long long total = (long long)height * n_out;
            dim3 grid((unsigned)((total + 255) / 256), (unsigned)n_channels);
            const int rc = frt_launch(h, kernel, grid, 256, 0, st, src, stride_c, stride_f, n_frames, weight,
                                      spec_min, inv_range, row_i0, row_t, height, out_col, out_a, n_out,
                                      old_data, reinterpret_cast<const unsigned *>(lut),
                                      reinterpret_cast<unsigned *>(pixels));
            if (rc) return rc;
        }
        dim3 grid2((unsigned)((height + 255) / 256), (unsigned)n_channels);
        return frt_launch(h, kernel, grid2, 256, 0, st, src, stride_c, stride_f, n_frames, weight, spec_min,
                          inv_range, row_i0, row_t, height, nullptr, nullptr, 0, old_data,
                          reinterpret_cast<const unsigned *>(lut), nullptr);
    };
    return rows ? launch(display_kernel<true>) : launch(display_kernel<false>);
}

}   // namespace

extern "C" int frt_display_columns(frt_handle h, const float *db_dev, int64_t stride_c,
                                   int64_t stride_f, int n_channels, int n_frames, int nbins,
                                   const float *weight_dev, float spec_min, float spec_max,
                                   const int *row_i0_dev, const float *row_t_dev, int height,
                                   const int *out_col_dev, const float *out_a_dev, int n_out,
                                   float *old_data_dev, const uint32_t *lut_dev,
                                   uint32_t *pixels_dev, void *stream) {
    if (!h) return FRT_EINVAL;
    DeviceGuard g(h->device);
    FRT_CHECK_ARG(h, n_channels >= 0 && n_frames >= 0 && height >= 1 && n_out >= 0 && nbins >= 2,
                  "bad shape");
    FRT_CHECK_ARG(h, spec_max != spec_min, "empty dB range");
    if (n_channels == 0 || n_frames == 0) return FRT_OK;
    FRT_CHECK_ARG(h, db_dev && row_i0_dev && row_t_dev && old_data_dev && lut_dev, "NULL buffer");
    FRT_CHECK_ARG(h, n_out == 0 || (out_col_dev && out_a_dev && pixels_dev), "NULL output buffer");
    const float inv_range = 1.0f / (spec_max - spec_min);
    return display_run(h, false, db_dev, stride_c, stride_f, n_channels, n_frames, weight_dev, spec_min, inv_range,
                       row_i0_dev, row_t_dev, height, out_col_dev, out_a_dev, n_out, old_data_dev, lut_dev,
                       pixels_dev, (cudaStream_t)stream);
}

extern "C" int frt_display_rows(frt_handle h, const float *rows_dev, int64_t stride_c, int64_t stride_f,
                                int n_channels, int n_frames, int height, const int *out_col_dev,
                                const float *out_a_dev, int n_out, float *old_data_dev,
                                const uint32_t *lut_dev, uint32_t *pixels_dev, void *stream) {
    if (!h) return FRT_EINVAL;
    DeviceGuard g(h->device);
    FRT_CHECK_ARG(h, n_channels >= 0 && n_frames >= 0 && height >= 1 && n_out >= 0, "bad shape");
    if (n_channels == 0 || n_frames == 0) return FRT_OK;
    FRT_CHECK_ARG(h, rows_dev && old_data_dev && lut_dev, "NULL buffer");
    FRT_CHECK_ARG(h, n_out == 0 || (out_col_dev && out_a_dev && pixels_dev), "NULL output buffer");
    return display_run(h, true, rows_dev, stride_c, stride_f, n_channels, n_frames, nullptr, 0.f, 0.f, nullptr,
                       nullptr, height, out_col_dev, out_a_dev, n_out, old_data_dev, lut_dev, pixels_dev,
                       (cudaStream_t)stream);
}
