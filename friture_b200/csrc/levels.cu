// The levels widget's meter (friture/levels.py:84-131, friture/ballistic_peak.py:43-66,
// friture/iec.py) and the long-term levels widget's history (friture/longlevels.py:150-230) for many
// channels, each call one launch over all of its buffers or blocks.
#include "frt_internal.cuh"

// ---------------------------------------------------------------------------------------------
// Meter.  Per channel and buffer: m = max|x| (exact in float32), conv = sum_j w[j] x[j]^2 in double
// (x^2 of a float32 sample is exact in double; the order of the sum is not NumPy's), then
//   old_max = m > old_max*keep ? m : old_max*keep                    (levels.py:105-111)
//   old_rms = alpha*conv + old_rms*decay                             (exp_smoothing.py:11-56)
//   level_rms = 10 log10(old_rms), level_max = 20 log10(old_max)     (levels.py:117-118)
//   the ballistic peak of dB_to_IEC(max(level_max, level_rms))       (ballistic_peak.py:43-66)
// in plain double multiplies and adds, as the widget's Python evaluates them.
struct LevelState {
    double rms, max, peak, decay;
    int hold;
};

struct LevelsPlan {
    int n_channels = 0, buffer = 0;
    double alpha = 0, decay = 0, keep = 0;
    DeviceArray<double> w;            // [buffer] the kernel's tail, kernel[Nk - buffer:]
    DeviceArray<LevelState> state;    // [C]
};
void PlanDelete::operator()(LevelsPlan *p) const { delete p; }

namespace {

constexpr double kPeakDecayRate = 1.0 - 3E-6 / 500.;   // ballistic_peak.py:22
constexpr int kPeakFalloff = 32;                        // ballistic_peak.py:24
constexpr int kGroup = 32;                              // buffers per group: one per lane of warp 0
constexpr int kReduceWarps = 8;

const LevelState kLevelReset = {1e-30, 1e-30, 0.0, kPeakDecayRate, 0};   // levels.py:62-64, ballistic_peak.py:33-35

struct LevelsArgs {
    const float *x;
    long long stride;
    int n_buffers, buffer;
    const double *w;
    double alpha, decay, keep;
    LevelState *state;
    double *rms_db, *max_db, *peak_iec;   // [C][n_buffers]
};

// iec.py:20-33, each product and sum rounded on its own
__device__ __forceinline__ double db_to_iec(double db) {
    if (db < -70.0) return 0.0;
    if (db < -60.0) return __dmul_rn(__dadd_rn(db, 70.0), 0.0025);
    if (db < -50.0) return __dadd_rn(__dmul_rn(__dadd_rn(db, 60.0), 0.005), 0.025);
    if (db < -40.0) return __dadd_rn(__dmul_rn(__dadd_rn(db, 50.0), 0.0075), 0.075);
    if (db < -30.0) return __dadd_rn(__dmul_rn(__dadd_rn(db, 40.0), 0.015), 0.15);
    if (db < -20.0) return __dadd_rn(__dmul_rn(__dadd_rn(db, 30.0), 0.02), 0.3);
    return __dadd_rn(__dmul_rn(__dadd_rn(db, 20.0), 0.025), 0.5);
}

// One CTA per channel: warps 1..8 reduce the buffers of group g into one half of the shared arrays
// while warp 0 steps the recurrences through group g-1 from the other half.  The recurrences are
// serial in tick order but cheap; the two logarithms per buffer are not serial, so lane 0 steps the
// peak and RMS states, the 32 lanes take the logarithms and the IEC mapping of one buffer each, and
// lane 0 steps the ballistic peak.
__global__ void __launch_bounds__(32 * (1 + kReduceWarps)) levels_ticks_kernel(LevelsArgs a) {
    __shared__ float s_max[2][kGroup];
    __shared__ double s_dot[2][kGroup];
    __shared__ double s_rms[kGroup], s_mx[kGroup], s_iec[kGroup];
    const int c = blockIdx.x, warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const float *x = a.x + (size_t)c * a.stride;
    const int n_groups = (a.n_buffers + kGroup - 1) / kGroup;
    LevelState st;
    if (warp == 0) st = a.state[c];
    double *rms_db = a.rms_db + (size_t)c * a.n_buffers, *max_db = a.max_db + (size_t)c * a.n_buffers;
    double *peak_iec = a.peak_iec + (size_t)c * a.n_buffers;
    for (int g = 0; g <= n_groups; g++) {
        if (warp > 0 && g < n_groups) {
            const int r0 = g * kGroup, nb = min(kGroup, a.n_buffers - r0);
            for (int b = warp - 1; b < nb; b += kReduceWarps) {
                const float *xb = x + (size_t)(r0 + b) * a.buffer;
                float m = 0.f;
                double d = 0.0;
#pragma unroll 8
                for (int j = lane; j < a.buffer; j += 32) {
                    const float v = __ldg(xb + j);
                    m = fmaxf(m, fabsf(v));
                    const double v2 = (double)v * (double)v;
                    d = fma(__ldg(a.w + j), v2, d);   // a NaN sample makes the sum NaN, as np.dot does
                }
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) {
                    m = fmaxf(m, __shfl_xor_sync(0xffffffffu, m, o));
                    d += __shfl_xor_sync(0xffffffffu, d, o);
                }
                // np.abs(y).max() is NaN when a sample is; fmaxf skips it.  The weights are positive and
                // the terms non-negative, so the sum is NaN exactly when a sample is.
                if (d != d) m = __int_as_float(0x7fffffff);
                if (lane == 0) {
                    s_max[g & 1][b] = m;
                    s_dot[g & 1][b] = d;
                }
            }
        }
        if (warp == 0 && g > 0) {
            const int r0 = (g - 1) * kGroup, nb = min(kGroup, a.n_buffers - r0), h = (g - 1) & 1;
            if (lane == 0) {
                for (int b = 0; b < nb; b++) {
                    const double m = s_max[h][b];
                    const double lim = __dmul_rn(st.max, a.keep);
                    st.max = m > lim ? m : lim;
                    st.rms = __dadd_rn(__dmul_rn(a.alpha, s_dot[h][b]), __dmul_rn(st.rms, a.decay));
                    s_rms[b] = st.rms;
                    s_mx[b] = st.max;
                }
            }
            __syncwarp();
            if (lane < nb) {
                const double lr = __dmul_rn(10.0, log10(s_rms[lane]));
                const double lm = __dmul_rn(20.0, log10(s_mx[lane]));
                rms_db[r0 + lane] = lr;
                max_db[r0 + lane] = lm;
                s_iec[lane] = db_to_iec(lr > lm ? lr : lm);   // Python's max(level_max, level_rms)
            }
            __syncwarp();
            if (lane == 0) {
                for (int b = 0; b < nb; b++) {
                    const double p = s_iec[b];
                    if (p > st.peak) {
                        st.peak = p;
                        st.hold = 0;
                        st.decay = kPeakDecayRate;
                    } else if (st.hold + 1 <= kPeakFalloff) {
                        st.hold++;
                    } else {
                        const double np_ = __dmul_rn(st.decay, st.peak);
                        if (np_ < p) {
                            st.peak = p;
                            st.hold = 0;
                            st.decay = kPeakDecayRate;
                        } else {
                            st.peak = np_;
                            st.decay = __dmul_rn(st.decay, st.decay);
                        }
                    }
                    peak_iec[r0 + b] = st.peak;
                }
            }
            __syncwarp();
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) a.state[c] = st;
}

}   // namespace

extern "C" int frt_levels_plan(frt_handle h, int n_channels, int buffer, const double *weights_host,
                               double alpha, double decay, double keep) {
    if (!h) return FRT_EINVAL;
    DeviceGuard g(h->device);
    FRT_CHECK_ARG(h, n_channels >= 1, "n_channels must be >= 1");
    FRT_CHECK_ARG(h, buffer >= 1, "buffer must be >= 1");
    FRT_CHECK_ARG(h, weights_host, "NULL weights");
    PlanPtr<LevelsPlan> p(new (std::nothrow) LevelsPlan());
    if (!p) return frt_fail(h, FRT_ENOMEM, "out of host memory");
    p->n_channels = n_channels;
    p->buffer = buffer;
    p->alpha = alpha;
    p->decay = decay;
    p->keep = keep;
    FRT_CUDA(h, p->w.upload(std::vector<double>(weights_host, weights_host + buffer)));
    if (h->levels && h->levels->n_channels == n_channels) {
        p->state = std::move(h->levels->state);   // a new buffer length keeps the meters' state
    } else {
        FRT_CUDA(h, p->state.upload(std::vector<LevelState>(n_channels, kLevelReset)));
    }
    h->levels = std::move(p);
    return FRT_OK;
}

extern "C" int frt_levels_reset(frt_handle h) {
    if (!h) return FRT_EINVAL;
    DeviceGuard g(h->device);
    if (!h->levels) return frt_fail(h, FRT_ESTATE, "frt_levels_reset before frt_levels_plan");
    const std::vector<LevelState> reset(h->levels->n_channels, kLevelReset);
    FRT_CUDA(h, frt_sync_copy(h->levels->state.get(), reset.data(), sizeof(LevelState) * reset.size(),
                              cudaMemcpyHostToDevice));
    return FRT_OK;
}

extern "C" int frt_levels_state(frt_handle h, double *state_host, int *hold_host) {
    if (!h) return FRT_EINVAL;
    DeviceGuard g(h->device);
    if (!h->levels) return frt_fail(h, FRT_ESTATE, "frt_levels_state before frt_levels_plan");
    FRT_CHECK_ARG(h, state_host && hold_host, "NULL buffer");
    const int C = h->levels->n_channels;
    std::vector<LevelState> s(C);
    FRT_CUDA(h, frt_sync_copy(s.data(), h->levels->state.get(), sizeof(LevelState) * C, cudaMemcpyDeviceToHost));
    for (int c = 0; c < C; c++) {
        state_host[c] = s[c].rms;
        state_host[C + c] = s[c].max;
        state_host[2 * C + c] = s[c].peak;
        state_host[3 * C + c] = s[c].decay;
        hold_host[c] = s[c].hold;
    }
    return FRT_OK;
}

extern "C" int frt_levels_process(frt_handle h, const float *x_dev, int64_t x_stride, int n_buffers,
                                  double *rms_db_dev, double *max_db_dev, double *peak_iec_dev, void *stream) {
    if (!h) return FRT_EINVAL;
    DeviceGuard g(h->device);
    if (!h->levels) return frt_fail(h, FRT_ESTATE, "frt_levels_process before frt_levels_plan");
    const LevelsPlan &p = *h->levels;
    FRT_CHECK_ARG(h, n_buffers >= 0, "n_buffers must be >= 0");
    if (n_buffers == 0) return FRT_OK;
    FRT_CHECK_ARG(h, x_dev && rms_db_dev && max_db_dev && peak_iec_dev, "NULL buffer");
    FRT_CHECK_ARG(h, p.n_channels == 1 || x_stride >= (int64_t)n_buffers * p.buffer,
                  "rows overlap: x_stride must be >= n_buffers * buffer");
    LevelsArgs a{x_dev, (long long)x_stride, n_buffers, p.buffer, p.w.get(), p.alpha, p.decay, p.keep,
                 p.state.get(), rms_db_dev, max_db_dev, peak_iec_dev};
    return frt_launch(h, levels_ticks_kernel, p.n_channels, 32 * (1 + kReduceWarps), 0, (cudaStream_t)stream, a);
}

// ---------------------------------------------------------------------------------------------
// Long-term levels.  Per block of 2^n_dec samples: x^2 through n_dec stages of the 11-tap gauss(11, 2)
// FIR keeping the even outputs (Subsampler.push, longlevels.py:71-89; decimate.py:27-42), then the
// 41-tap gauss(41, 8) FIR (longlevels.py:172), one value per block.  With a = [1, 0, ...],
// lfilter_float64_1D (lfilter.py:132-139) evaluates y[n] = (...((b10 x[n-10] + b9 x[n-9]) + ...) +
// b1 x[n-1]) + b0 x[n] in plain double multiplies and adds; fir_tap writes it in that order, so the
// linear level is the same bits.  A stage's state is its last 10 inputs (the final FIR's, its last 40):
// zeros after a reset, as the widget's zero zi.  The transposed form also adds y[n] * a[k] = y[n] * 0 to
// its state, which is NaN once y[n] is NaN or infinite: from the output after a stage's first
// non-finite input on, the widget's stage gives NaN for good.  Each stage carries that as a flag.
constexpr int LL_MAX_DEC = 13;            // rt = 20 s: floor(log2(20 * 48000 / 100))
constexpr int LL_FLAGS = LL_MAX_DEC * 10 + 40;       // the stages' NaN flags, the final FIR's at n_dec
constexpr int LL_STATE = LL_FLAGS + LL_MAX_DEC + 1;

struct LongLevelsPlan {
    int n_channels = 0, n_dec = 0;
    double bdec[11], bfir[41];
    DeviceArray<double> state;    // [C][LL_STATE]: stage s's last 10 inputs at 10 s, the final FIR's at
                                  // 10 n_dec, the NaN flags at LL_FLAGS
};
void PlanDelete::operator()(LongLevelsPlan *p) const { delete p; }

namespace {

constexpr int LL_THREADS = 256;
constexpr int LL_MIN_TILE = 4096;   // input samples per tile, at least one block

struct LongArgs {
    const float *x;
    long long stride;
    int n_blocks, n_dec;
    double bdec[11], bfir[41];
    double *state;
    double *level, *db;            // [C][n_blocks]
    float *ring;                   // [C][ring_len]
    long long ring_len, ring_pos;  // the slot of the call's first block is ring_pos % ring_len
};

// y = (...((b[T-1] in(-(T-1)) + b[T-2] in(-(T-2))) + ...) + b[0] in(0)), in[k] = src[k + T - 1]
template <int T, class Src>
__device__ __forceinline__ double fir_tap(const double *b, Src in) {
    double y = __dmul_rn(b[T - 1], in(0));
#pragma unroll
    for (int t = T - 2; t >= 0; t--) y = __dadd_rn(y, __dmul_rn(b[t], in(T - 1 - t)));
    return y;
}

// Shared memory of a CTA: the tile's samples (float), stage 0's history (10 doubles), stages
// 1..n_dec-1's inputs each behind their 10-value history, the final FIR's inputs behind its 40.
struct LongSmem {
    static size_t bytes(int n_dec) {
        const int tile = max(1 << n_dec, LL_MIN_TILE);
        size_t d = 10;
        for (int s = 1; s < n_dec; s++) d += 10 + (tile >> s);
        d += 40 + (tile >> n_dec);
        return sizeof(float) * tile + sizeof(double) * d;
    }
};

__global__ void __launch_bounds__(LL_THREADS) longlevels_kernel(const LongArgs a) {
    extern __shared__ __align__(16) unsigned char smem[];
    __shared__ int s_first[LL_MAX_DEC + 1];     // the tile's first non-finite input of each stage
    __shared__ int s_nan[LL_MAX_DEC + 1];       // the stage gives NaN for good
    const int c = blockIdx.x, tid = threadIdx.x, n_dec = a.n_dec;
    const int tile = max(1 << n_dec, LL_MIN_TILE), bpt = tile >> n_dec;   // blocks per tile
    // stage(s), s >= 1: stage s's history then its inputs; stage(n_dec): the final FIR's.  Stage s
    // starts after 10 + sum_{t<s} (10 + tile >> t) doubles.
    double *hist0 = (double *)smem;
    auto stage = [&](int s) { return hist0 + 10 * s + tile - (tile >> (s - 1)); };
    float *xs = (float *)(stage(n_dec) + 40 + bpt);
    double *st = a.state + (size_t)c * LL_STATE;
    // state -> shared memory
    for (int i = tid; i < 10 * n_dec + 40; i += LL_THREADS) {
        const int s = i / 10;
        if (s == 0) hist0[i] = st[i];
        else if (s < n_dec) stage(s)[i - 10 * s] = st[i];
        else stage(n_dec)[i - 10 * n_dec] = st[i];
    }
    if (tid <= n_dec) {
        s_first[tid] = INT_MAX;
        s_nan[tid] = st[LL_FLAGS + tid] != 0.0;
    }
    const double qnan = __longlong_as_double(0x7ff8000000000000ll);
    const float *x = a.x + (size_t)c * a.stride;
    for (int b0 = 0; b0 < a.n_blocks; b0 += bpt) {
        const int nb = min(bpt, a.n_blocks - b0), len0 = nb << n_dec;
        const float *xt = x + ((size_t)b0 << n_dec);
        for (int i = tid; i < len0; i += LL_THREADS) {
            const float v = __ldg(xt + i);
            xs[i] = v;
            if (!isfinite(v)) atomicMin(&s_first[0], i);
        }
        __syncthreads();
        // stage 0: even outputs of x^2
        {
            double *dst = n_dec > 1 ? stage(1) + 10 : stage(n_dec) + 40;
            for (int j = tid; j < (len0 >> 1); j += LL_THREADS) {
                const int base = 2 * j - 10;
                const double y = s_nan[0] || 2 * j > s_first[0] ? qnan : fir_tap<11>(a.bdec, [&](int k) {
                    const int i = base + k;
                    if (i < 0) return hist0[10 + i];
                    const double v = xs[i];
                    return v * v;
                });
                dst[j] = y;
                if (!isfinite(y)) atomicMin(&s_first[min(1, n_dec)], j);
            }
        }
        __syncthreads();
        for (int s = 1; s < n_dec; s++) {
            const double *src = stage(s);
            double *dst = s + 1 < n_dec ? stage(s + 1) + 10 : stage(n_dec) + 40;
            for (int j = tid; j < (len0 >> (s + 1)); j += LL_THREADS) {
                const double y = s_nan[s] || 2 * j > s_first[s] ? qnan
                                                                : fir_tap<11>(a.bdec, [&](int k) { return src[2 * j + k]; });
                dst[j] = y;
                if (!isfinite(y)) atomicMin(&s_first[s + 1], j);
            }
            __syncthreads();
        }
        if (tid < nb) {
            const double *src = stage(n_dec);
            const double lv = s_nan[n_dec] || tid > s_first[n_dec] ? qnan
                                                                   : fir_tap<41>(a.bfir, [&](int k) { return src[tid + k]; });
            const double db = __dmul_rn(10.0, log10(1e-150 > lv ? 1e-150 : lv));   // max(level, 1e-150), longlevels.py:174: NaN stays NaN
            const size_t o = (size_t)c * a.n_blocks + b0 + tid;
            a.level[o] = lv;
            a.db[o] = db;
            a.ring[(size_t)c * a.ring_len + (a.ring_pos + b0 + tid) % a.ring_len] = (float)db;
        }
        // every history moves to the last values of (history, inputs): read all, then write
        const int n_hist = 10 * n_dec + 40;
        double v[(10 * LL_MAX_DEC + 40 + LL_THREADS - 1) / LL_THREADS];
        int k = 0;
        for (int i = tid; i < n_hist; i += LL_THREADS, k++) {
            const int s = min(i / 10, n_dec);
            const int len = s == 0 ? len0 : len0 >> s;
            if (s == 0) {
                const double y = xs[len - 10 + i];
                v[k] = y * y;
            } else {
                const int off = s < n_dec ? i - 10 * s : i - 10 * n_dec;
                v[k] = stage(s)[len + off];
            }
        }
        __syncthreads();
        if (tid <= n_dec) {
            if (s_first[tid] != INT_MAX) s_nan[tid] = 1;
            s_first[tid] = INT_MAX;
        }
        k = 0;
        for (int i = tid; i < n_hist; i += LL_THREADS, k++) {
            const int s = min(i / 10, n_dec);
            if (s == 0) hist0[i] = v[k];
            else stage(s)[s < n_dec ? i - 10 * s : i - 10 * n_dec] = v[k];
        }
        __syncthreads();
    }
    for (int i = tid; i < 10 * n_dec + 40; i += LL_THREADS) {
        const int s = min(i / 10, n_dec);
        st[i] = s == 0 ? hist0[i] : stage(s)[s < n_dec ? i - 10 * s : i - 10 * n_dec];
    }
    if (tid <= n_dec) st[LL_FLAGS + tid] = s_nan[tid];
}

// longlevels.py:183-187: scaled_y = clip(1 - (levels - level_min) / (level_max - level_min), 0, 1) over the
// last `length` values of the ring, in double, rounded once to float32.
__global__ void __launch_bounds__(256) longlevels_curve_kernel(const float *ring, long long ring_len,
                                                               long long ring_pos, int length, double lo,
                                                               double hi, float *out) {
    const int c = blockIdx.y, j = blockIdx.x * blockDim.x + threadIdx.x;
    if (j >= length) return;
    long long slot = (ring_pos - length + j) % ring_len;
    if (slot < 0) slot += ring_len;
    const double l = ring[(size_t)c * ring_len + slot];
    double v = __dsub_rn(1.0, __ddiv_rn(__dsub_rn(l, lo), __dsub_rn(hi, lo)));
    v = v < 0.0 ? 0.0 : v > 1.0 ? 1.0 : v;   // np.clip: NaN stays NaN
    out[(size_t)c * length + j] = (float)v;
}

}   // namespace

extern "C" int frt_longlevels_plan(frt_handle h, int n_channels, int n_dec, const double *bdec_host,
                                   const double *bfir_host) {
    if (!h) return FRT_EINVAL;
    DeviceGuard g(h->device);
    FRT_CHECK_ARG(h, n_channels >= 1, "n_channels must be >= 1");
    FRT_CHECK_ARG(h, n_dec >= 1 && n_dec <= LL_MAX_DEC, "n_dec must be in 1..13");
    FRT_CHECK_ARG(h, bdec_host && bfir_host, "NULL coefficients");
    PlanPtr<LongLevelsPlan> p(new (std::nothrow) LongLevelsPlan());
    if (!p) return frt_fail(h, FRT_ENOMEM, "out of host memory");
    p->n_channels = n_channels;
    p->n_dec = n_dec;
    memcpy(p->bdec, bdec_host, sizeof(p->bdec));
    memcpy(p->bfir, bfir_host, sizeof(p->bfir));
    FRT_CUDA(h, p->state.alloc((size_t)n_channels * LL_STATE));
    FRT_CUDA(h, frt_sync_zero(p->state.get(), sizeof(double) * p->state.n));
    h->longlevels = std::move(p);
    return FRT_OK;
}

extern "C" int frt_longlevels_reset(frt_handle h) {
    if (!h) return FRT_EINVAL;
    DeviceGuard g(h->device);
    if (!h->longlevels) return frt_fail(h, FRT_ESTATE, "frt_longlevels_reset before frt_longlevels_plan");
    FRT_CUDA(h, frt_sync_zero(h->longlevels->state.get(), sizeof(double) * h->longlevels->state.n));
    return FRT_OK;
}

extern "C" int frt_longlevels_process(frt_handle h, const float *x_dev, int64_t x_stride, int n_blocks,
                                      double *level_dev, double *db_dev, float *ring_dev, int64_t ring_len,
                                      int64_t ring_pos, void *stream) {
    if (!h) return FRT_EINVAL;
    DeviceGuard g(h->device);
    if (!h->longlevels) return frt_fail(h, FRT_ESTATE, "frt_longlevels_process before frt_longlevels_plan");
    const LongLevelsPlan &p = *h->longlevels;
    FRT_CHECK_ARG(h, n_blocks >= 0 && ring_len >= 1 && ring_pos >= 0, "bad shape");
    if (n_blocks == 0) return FRT_OK;
    FRT_CHECK_ARG(h, x_dev && level_dev && db_dev && ring_dev, "NULL buffer");
    FRT_CHECK_ARG(h, p.n_channels == 1 || x_stride >= ((int64_t)n_blocks << p.n_dec),
                  "rows overlap: x_stride must be >= n_blocks * 2^n_dec");
    LongArgs a{};
    a.x = x_dev;
    a.stride = x_stride;
    a.n_blocks = n_blocks;
    a.n_dec = p.n_dec;
    memcpy(a.bdec, p.bdec, sizeof(a.bdec));
    memcpy(a.bfir, p.bfir, sizeof(a.bfir));
    a.state = p.state.get();
    a.level = level_dev;
    a.db = db_dev;
    a.ring = ring_dev;
    a.ring_len = ring_len;
    a.ring_pos = ring_pos;
    return frt_launch(h, longlevels_kernel, p.n_channels, LL_THREADS, LongSmem::bytes(p.n_dec),
                      (cudaStream_t)stream, a);
}

extern "C" int frt_longlevels_history(frt_handle h, const float *ring_dev, int64_t ring_len, int64_t ring_pos,
                                      int n_channels, int length, double level_min, double level_max,
                                      float *scaled_dev, void *stream) {
    if (!h) return FRT_EINVAL;
    DeviceGuard g(h->device);
    FRT_CHECK_ARG(h, n_channels >= 0 && length >= 0 && ring_len >= 1 && ring_pos >= 0, "bad shape");
    FRT_CHECK_ARG(h, length <= ring_len, "length must be <= ring_len");
    if (n_channels == 0 || length == 0) return FRT_OK;
    FRT_CHECK_ARG(h, ring_dev && scaled_dev, "NULL buffer");
    FRT_CHECK_ARG(h, n_channels <= 65535, "n_channels must be <= 65535");
    const dim3 grid((unsigned)((length + 255) / 256), (unsigned)n_channels);
    return frt_launch(h, longlevels_curve_kernel, grid, 256, 0, (cudaStream_t)stream, ring_dev, (long long)ring_len,
                      (long long)ring_pos, length, level_min, level_max, scaled_dev);
}
