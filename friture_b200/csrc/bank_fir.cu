// The reference's LIVE filterbank numerics for sm_90a: 512-tap minimum-phase FIR approximations of
// the fractional-octave and decimation filters, which Octave_Filters.filter() runs by FFT
// overlap-add (friture/octavefilters.py:49-58,123-158; friture/filter.py:136-247).  Overlap-add
// with a tail buffer IS an exact linear convolution, so the kernel computes the convolutions
// directly, carrying the last L-1 input samples of every stage instead of the L-1 pending output
// samples of every filter:
//     stage j:  y_i = (x_j * h_i)[0:N_j]  (i = bpo-1 .. 0),   x_{j+1} = (x_j * h_dec)[0:N_j:2]
// This is the parity mode for callers that want the live path's exact output (it differs from
// the IIR designs it approximates by ~5e-4 on band energy); the throughput path is the IIR bank
// of bank.cu / bank_pipe.cu.  One CTA per channel, the taps, the stage signal and every stage's
// input history in shared memory, double-precision accumulation (512-term sums with heavy
// cancellation in the stop bands).
//
// One kernel serves two entry points:
//   frt_firbank_process  one block, the ragged band outputs y (the literal `.filter()` contract);
//   frt_firbank_levels   n_blocks blocks in one launch, no y: per block and band the octave widget's
//                        smoothed level (friture/octavespectrum.py:101-121), accumulated in float64
//                        from the squared double accumulators.
// Each output is one double fma chain over k = 0..L-1, whatever the entry point or the blocking, so
// y is the same on both paths and any cut of a stream into launches gives the same bits.
#include <cmath>
#include <vector>

#include "frt_internal.cuh"

namespace {

constexpr int FIR_MAX_OCT = 10;
constexpr int FIR_THREADS = 256;
constexpr int FIR_WARPS = FIR_THREADS / 32;
constexpr int FIR_MAX_BLOCK = 4096;
constexpr int FIR_R = 4;    // consecutive outputs per thread (larger banks): each broadcast tap feeds FIR_R chains
constexpr int FIR_F = 4;    // filters per thread: each input sample feeds FIR_F chains
constexpr int FIR_DECAY_STRIDE = FIR_MAX_BLOCK + 1;   // decay table row: (1-alpha_j)^m, m = 0..4096

struct FirArgs {
    const float *x;
    long long x_stride;
    int block;               // samples per channel and block
    int n_blocks;
    int L;                   // taps
    int bpo, n_oct;
    const double *taps;      // [bpo + 1][L]: bands 0..bpo-1, then the decimator
    float *hist;             // [C][n_oct][L-1] last inputs of every stage
    float *y;                // NULL, or (n_blocks == 1) the ragged band outputs: channel c at
    long long y_stride;      //   y + c*y_stride, band k = (n_oct-1-j)*bpo + i holding block >> j samples
    // band levels (levels != NULL)
    const double *alpha;     // [n_oct]
    const double *decay;     // [n_oct][FIR_DECAY_STRIDE]
    const float *weight_db;  // [nbands] or NULL
    double *sp;              // [C][nbands] carried smoothed energies
    float *levels;           // [C][n_blocks][nbands]
    int db;
};

__host__ __device__ inline int round4(int n) { return (n + 3) & ~3; }

// Shared-memory layout, in bytes from the (16-byte aligned) dynamic base.  The stage buffers put
// x_j[0] at float index P = round4(L) so that the float4 input loads of the convolution are aligned;
// x_j[-(L-1)..-1] (the history) sits just below it.
struct FirSmem {
    int P;
    size_t taps, red, sp, hist, xa, xb, total;
    __host__ __device__ FirSmem(int L, int bpo, int n_oct, int block) {
        const int nf = bpo + 1, nbands = bpo * n_oct;
        P = round4(L);
        taps = 0;
        red = taps + sizeof(double) * (size_t)((nf * L + 1) & ~1);
        sp = red + sizeof(double) * FIR_WARPS * FIR_F;
        hist = sp + sizeof(double) * (size_t)((nbands + 1) & ~1);
        xa = hist + sizeof(float) * (size_t)round4(n_oct * (L - 1));
        xb = xa + sizeof(float) * (size_t)(P + round4(block) + FIR_R);
        total = xb + sizeof(float) * (size_t)(P + round4(block / 2) + FIR_R);
    }
};

// R consecutive outputs n0.. of FIR_F filters (nv of them valid) of one stage:
// acc[r][q] = sum_k t[q*L + k] * xs[n0 + r - k], one fma chain per output in k order.
// R = 4 reuses each broadcast tap for four outputs (n0 % 4 == 0, aligned float4 input loads);
// R = 1 keeps four times as many threads busy, for banks of at most two filter groups.
template <int R>
__device__ __forceinline__ void fir_tile(const double *__restrict__ t, int L, int nv,
                                         const float *__restrict__ xs, int n0,
                                         double (&acc)[R][FIR_F]) {
#pragma unroll
    for (int r = 0; r < R; r++)
#pragma unroll
        for (int q = 0; q < FIR_F; q++) acc[r][q] = 0.0;
    if constexpr (R == 1) {
        for (int k = 0; k < L; k++) {
            const double xv = (double)xs[n0 - k];
#pragma unroll
            for (int q = 0; q < FIR_F; q++)
                if (q < nv) acc[0][q] = fma(t[q * L + k], xv, acc[0][q]);
        }
        return;
    }
    // w[4 + d] = x[n0 - k0 + d], d = -4..3: the window of the current group of four taps
    double w[8];
    {
        const float4 v = *reinterpret_cast<const float4 *>(xs + n0);
        w[4] = v.x; w[5] = v.y; w[6] = v.z; w[7] = v.w;
    }
    const int L4 = L & ~3;
    for (int k0 = 0; k0 < L4; k0 += 4) {
        const float4 v = *reinterpret_cast<const float4 *>(xs + n0 - k0 - 4);
        w[0] = v.x; w[1] = v.y; w[2] = v.z; w[3] = v.w;
#pragma unroll
        for (int kk = 0; kk < 4; kk++) {
            const int k = k0 + kk;
            double tq[FIR_F];
#pragma unroll
            for (int q = 0; q < FIR_F; q++) tq[q] = (q < nv) ? t[q * L + k] : 0.0;
#pragma unroll
            for (int r = 0; r < R; r++) {
                const double xv = w[4 + r - kk];
#pragma unroll
                for (int q = 0; q < FIR_F; q++)
                    if (q < nv) acc[r][q] = fma(tq[q], xv, acc[r][q]);
            }
        }
#pragma unroll
        for (int d = 0; d < 4; d++) w[4 + d] = w[d];
    }
    for (int k = L4; k < L; k++) {
        double tq[FIR_F];
#pragma unroll
        for (int q = 0; q < FIR_F; q++) tq[q] = (q < nv) ? t[q * L + k] : 0.0;
#pragma unroll
        for (int r = 0; r < R; r++) {
            const double xv = (double)xs[n0 + r - k];
#pragma unroll
            for (int q = 0; q < FIR_F; q++)
                if (q < nv) acc[r][q] = fma(tq[q], xv, acc[r][q]);
        }
    }
}

template <int R>
__global__ void __launch_bounds__(FIR_THREADS, R == 1 ? 4 : 2) fir_bank_kernel(const FirArgs a) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int L = a.L, Lm1 = a.L - 1, nf = a.bpo + 1, nbands = a.bpo * a.n_oct;
    const FirSmem lay(L, a.bpo, a.n_oct, a.block);
    const int P = lay.P;
    double *s_taps = reinterpret_cast<double *>(smem_raw + lay.taps);   // [nf][L]
    double *s_red = reinterpret_cast<double *>(smem_raw + lay.red);     // [FIR_WARPS][FIR_F]
    double *s_sp = reinterpret_cast<double *>(smem_raw + lay.sp);       // [nbands]
    float *s_hist = reinterpret_cast<float *>(smem_raw + lay.hist);     // [n_oct][Lm1]
    float *s_xa = reinterpret_cast<float *>(smem_raw + lay.xa);         // stages 0, 2, 4, ...
    float *s_xb = reinterpret_cast<float *>(smem_raw + lay.xb);         // stages 1, 3, 5, ...
    const int c = blockIdx.x, tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const bool levels = a.levels != nullptr;

    for (int i = tid; i < nf * L; i += FIR_THREADS) s_taps[i] = a.taps[i];
    float *hist = a.hist + (size_t)c * a.n_oct * Lm1;
    for (int i = tid; i < a.n_oct * Lm1; i += FIR_THREADS) s_hist[i] = hist[i];
    if (levels)
        for (int i = tid; i < nbands; i += FIR_THREADS) s_sp[i] = a.sp[(size_t)c * nbands + i];
    // the padding the float4 loads may touch (never used by an output) starts out finite
    for (int i = tid; i < (int)((lay.total - lay.xa) / sizeof(float)); i += FIR_THREADS) s_xa[i] = 0.f;
    __syncthreads();

    // filters are processed FIR_F at a time: group g = filters g*FIR_F.., served by wpg warps
    const int n_groups = (nf + FIR_F - 1) / FIR_F;
    const int wpg = FIR_WARPS / n_groups >= 1 ? FIR_WARPS / n_groups : 1;
    const int g = warp / wpg;
    const int tig = tid - g * wpg * 32, tpg = wpg * 32;
    const int nv = min(FIR_F, nf - g * FIR_F);

    for (int b = 0; b < a.n_blocks; b++) {
        float *sx = s_xa, *sn = s_xb;
        int N = a.block;
        long long off = 0;     // ragged y: stages j' > j first (they are shorter)
        for (int jj = a.n_oct - 1; jj > 0; jj--) off += (long long)a.bpo * (a.block >> jj);
        for (int j = 0; j < a.n_oct; j++) {
            const bool last = (j + 1 == a.n_oct);
            float *xs = sx + P;                     // xs[m] = x_j[m], m = -(L-1) .. N-1
            for (int i = tid; i < Lm1; i += FIR_THREADS) xs[i - Lm1] = s_hist[(size_t)j * Lm1 + i];
            if (j == 0) {
                const float *xc = a.x + (size_t)c * a.x_stride + (size_t)b * a.block;
                for (int i = tid; i < N; i += FIR_THREADS) xs[i] = xc[i];
            }
            __syncthreads();
            if (g < n_groups) {
                const double *t = s_taps + (size_t)g * FIR_F * L;
                const double *dec = a.decay + (size_t)j * FIR_DECAY_STRIDE;
                double part[FIR_F] = {0.0, 0.0, 0.0, 0.0};
                const int n_chunks = (N + R - 1) / R;
                for (int ch = tig; ch < n_chunks; ch += tpg) {
                    const int n0 = ch * R;
                    double acc[R][FIR_F];
                    fir_tile<R>(t, L, nv, xs, n0, acc);
#pragma unroll
                    for (int r = 0; r < R; r++) {
                        const int n = n0 + r;
                        if (n >= N) break;
                        const double wn = levels ? __ldg(dec + (N - 1 - n)) : 0.0;
#pragma unroll
                        for (int q = 0; q < FIR_F; q++) {
                            const int f = g * FIR_F + q;
                            if (f < a.bpo) {
                                if (a.y) a.y[(size_t)c * a.y_stride + off + (long long)f * N + n] = (float)acc[r][q];
                                if (levels) part[q] = fma(wn, acc[r][q] * acc[r][q], part[q]);
                            } else if (f == a.bpo && !last && !(n & 1)) {
                                sn[P + (n >> 1)] = (float)acc[r][q];
                            }
                        }
                    }
                }
                if (levels) {
#pragma unroll
                    for (int q = 0; q < FIR_F; q++)
#pragma unroll
                        for (int o = 16; o > 0; o >>= 1) part[q] += __shfl_xor_sync(0xffffffffu, part[q], o);
                    if (lane == 0)
#pragma unroll
                        for (int q = 0; q < FIR_F; q++) s_red[warp * FIR_F + q] = part[q];
                }
            }
            __syncthreads();
            if (levels && tid < a.bpo) {
                // sp <- alpha * sum_n (1-alpha)^(N-1-n) y[n]^2 + sp * (1-alpha)^N
                // (exp_smoothed_value, friture/signal/exp_smoothing.py:40-56, with N <= its kernel)
                const int gg = tid / FIR_F, q = tid % FIR_F;
                double s = 0.0;
                for (int w = 0; w < wpg; w++) s += s_red[(gg * wpg + w) * FIR_F + q];
                const int k = (a.n_oct - 1 - j) * a.bpo + tid;
                s_sp[k] = a.alpha[j] * s + s_sp[k] * a.decay[(size_t)j * FIR_DECAY_STRIDE + N];
            }
            // this stage's new history = its last L-1 inputs
            for (int i = tid; i < Lm1; i += FIR_THREADS) s_hist[(size_t)j * Lm1 + i] = xs[N - Lm1 + i];
            __syncthreads();
            if (last) break;
            float *tmp = sx;
            sx = sn;
            sn = tmp;
            N >>= 1;
            off -= (long long)a.bpo * N;
        }
        if (levels) {
            float *lv = a.levels + ((size_t)c * a.n_blocks + b) * nbands;
            for (int k = tid; k < nbands; k += FIR_THREADS) {
                const double e = s_sp[k];
                lv[k] = a.db ? (float)(10.0 * log10(e + 1e-30) + (a.weight_db ? (double)a.weight_db[k] : 0.0))
                             : (float)e;
            }
        }
    }
    for (int i = tid; i < a.n_oct * Lm1; i += FIR_THREADS) hist[i] = s_hist[i];
    if (levels)
        for (int i = tid; i < nbands; i += FIR_THREADS) a.sp[(size_t)c * nbands + i] = s_sp[i];
}

}   // namespace

struct FirPlan {
    int n_channels = 0, bpo = 0, n_oct = 0, L = 0;
    DeviceArray<double> taps;
    DeviceArray<float> hist;
    DeviceArray<double> sp;          // [C][nbands]
    DeviceArray<double> alpha;       // [n_oct]
    DeviceArray<double> decay;       // [n_oct][FIR_DECAY_STRIDE]
    DeviceArray<float> weight_db;    // [nbands]
    bool smoothing = false;          // frt_firbank_set_smoothing has been called
    bool weighted = false;
};

void PlanDelete::operator()(FirPlan *p) const { delete p; }

extern "C" int frt_firbank_plan(frt_handle h, int n_channels, int bands_per_octave, int n_octaves,
                                int n_taps, const double *fir_band, const double *fir_dec) {
    if (!h) return FRT_EINVAL;
    DeviceGuard g(h->device);
    FRT_CHECK_ARG(h, n_channels >= 1, "n_channels must be >= 1");
    FRT_CHECK_ARG(h, bands_per_octave >= 1 && bands_per_octave <= 24, "bands_per_octave must be in [1, 24]");
    FRT_CHECK_ARG(h, n_octaves >= 1 && n_octaves <= FIR_MAX_OCT, "n_octaves must be in [1, 10]");
    FRT_CHECK_ARG(h, n_taps >= 2 && n_taps <= 1024, "n_taps must be in [2, 1024]");
    FRT_CHECK_ARG(h, fir_band && fir_dec, "NULL tap table");
    // the taps, the histories and two stage buffers live in one CTA's shared memory: a bank that does
    // not fit even at its shortest block, 2^(n_octaves-1), cannot run at all
    const size_t need = FirSmem(n_taps, bands_per_octave, n_octaves, 1 << (n_octaves - 1)).total;
    if (need > h->smem_optin)
        return frt_fail(h, FRT_EINVAL,
                        "frt_firbank_plan: the bank needs %zu bytes of shared memory at its shortest block, "
                        "the device allows %zu per block", need, h->smem_optin);
    PlanPtr<FirPlan> pl(new (std::nothrow) FirPlan());
    if (!pl) return frt_fail(h, FRT_ENOMEM, "out of host memory");
    pl->n_channels = n_channels;
    pl->bpo = bands_per_octave;
    pl->n_oct = n_octaves;
    pl->L = n_taps;
    const size_t nt = (size_t)(bands_per_octave + 1) * n_taps;
    const size_t nh = (size_t)n_channels * n_octaves * (n_taps - 1);
    const size_t nb = (size_t)bands_per_octave * n_octaves;
    FRT_CUDA(h, pl->taps.alloc(nt));
    FRT_CUDA(h, pl->hist.alloc(nh));
    FRT_CUDA(h, pl->sp.alloc(n_channels * nb));
    FRT_CUDA(h, pl->alpha.alloc(n_octaves));
    FRT_CUDA(h, pl->decay.alloc((size_t)n_octaves * FIR_DECAY_STRIDE));
    FRT_CUDA(h, pl->weight_db.alloc(nb));
    FRT_CUDA(h, frt_sync_copy(pl->taps.get(), fir_band, sizeof(double) * (size_t)bands_per_octave * n_taps,
                              cudaMemcpyHostToDevice));
    FRT_CUDA(h, frt_sync_copy(pl->taps.get() + (size_t)bands_per_octave * n_taps, fir_dec, sizeof(double) * n_taps,
                              cudaMemcpyHostToDevice));
    FRT_CUDA(h, frt_sync_zero(pl->hist.get(), sizeof(float) * nh));
    FRT_CUDA(h, frt_sync_zero(pl->sp.get(), sizeof(double) * n_channels * nb));
    h->fir = std::move(pl);
    return FRT_OK;
}

extern "C" int frt_firbank_reset(frt_handle h) {
    if (!h) return FRT_EINVAL;
    FirPlan *pl = h->fir.get();
    if (!pl) return frt_fail(h, FRT_ESTATE, "frt_firbank_reset: no plan");
    DeviceGuard g(h->device);
    FRT_CUDA(h, frt_sync_zero(pl->hist.get(), sizeof(float) * (size_t)pl->n_channels * pl->n_oct * (pl->L - 1)));
    FRT_CUDA(h, frt_sync_zero(pl->sp.get(), sizeof(double) * (size_t)pl->n_channels * pl->n_oct * pl->bpo));
    return FRT_OK;
}

extern "C" int frt_firbank_set_smoothing(frt_handle h, const double *alphas, const float *weight_db) {
    if (!h) return FRT_EINVAL;
    FirPlan *pl = h->fir.get();
    if (!pl) return frt_fail(h, FRT_ESTATE, "frt_firbank_set_smoothing: call frt_firbank_plan first");
    DeviceGuard g(h->device);
    FRT_CHECK_ARG(h, alphas, "NULL alphas");
    for (int j = 0; j < pl->n_oct; j++)
        FRT_CHECK_ARG(h, alphas[j] > 0.0 && alphas[j] <= 1.0, "alphas must be in (0, 1]");
    std::vector<double> decay((size_t)pl->n_oct * FIR_DECAY_STRIDE);
    for (int j = 0; j < pl->n_oct; j++)
        for (int m = 0; m < FIR_DECAY_STRIDE; m++)
            decay[(size_t)j * FIR_DECAY_STRIDE + m] = std::pow(1.0 - alphas[j], (double)m);
    FRT_CUDA(h, frt_sync_copy(pl->alpha.get(), alphas, sizeof(double) * pl->n_oct, cudaMemcpyHostToDevice));
    FRT_CUDA(h, frt_sync_copy(pl->decay.get(), decay.data(), sizeof(double) * decay.size(), cudaMemcpyHostToDevice));
    if (weight_db)
        FRT_CUDA(h, frt_sync_copy(pl->weight_db.get(), weight_db, sizeof(float) * (size_t)pl->n_oct * pl->bpo,
                                  cudaMemcpyHostToDevice));
    pl->weighted = weight_db != nullptr;
    pl->smoothing = true;
    return FRT_OK;
}

// Shared memory of one CTA at a block length; fir_bank_kernel declares no static shared memory.
static int fir_check_block(frt_handle h, const FirPlan *pl, int block, const char *fn) {
    const size_t need = FirSmem(pl->L, pl->bpo, pl->n_oct, block).total;
    if (need > h->smem_optin)
        return frt_fail(h, FRT_EINVAL, "%s: a block of %d samples needs %zu bytes of shared memory, the device "
                        "allows %zu per block", fn, block, need, h->smem_optin);
    return FRT_OK;
}

static int fir_launch(frt_handle h, FirPlan *pl, FirArgs &a, void *stream) {
    a.L = pl->L;
    a.bpo = pl->bpo;
    a.n_oct = pl->n_oct;
    a.taps = pl->taps.get();
    a.hist = pl->hist.get();
    const size_t smem = FirSmem(pl->L, pl->bpo, pl->n_oct, a.block).total;
    // a bank of one or two filter groups (bpo <= 7) leaves most threads idle at four outputs per
    // thread: on an H100 (400 W) at 1024 channels, 512-sample blocks, 3 and 6 bands per octave ran 40 % and
    // 20 % slower than one output per thread; 12 and 24 bands per octave ran 1.6x and 1.7x faster
    auto kernel = pl->bpo + 1 <= 2 * FIR_F ? fir_bank_kernel<1> : fir_bank_kernel<FIR_R>;
    return frt_launch(h, kernel, pl->n_channels, FIR_THREADS, smem, (cudaStream_t)stream, a);
}

extern "C" int frt_firbank_process(frt_handle h, const float *x_dev, int64_t x_stride, int n_samples,
                                   float *y_dev, int64_t y_stride, void *stream) {
    if (!h) return FRT_EINVAL;
    FirPlan *pl = h->fir.get();
    if (!pl) return frt_fail(h, FRT_ESTATE, "frt_firbank_process: call frt_firbank_plan first");
    DeviceGuard g(h->device);
    FRT_CHECK_ARG(h, n_samples >= 0, "negative length");
    if (n_samples == 0) return FRT_OK;
    FRT_CHECK_ARG(h, n_samples <= FIR_MAX_BLOCK, "n_samples must be <= 4096");
    FRT_CHECK_ARG(h, n_samples % (1 << (pl->n_oct - 1)) == 0,
                  "n_samples must be a multiple of 2^(n_octaves-1) (every stage keeps its even samples)");
    FRT_CHECK_ARG(h, x_dev && y_dev, "NULL buffer");
    FRT_CHECK_ARG(h, x_stride >= n_samples, "x_stride smaller than n_samples");
    long long need = 0;
    for (int j = 0; j < pl->n_oct; j++) need += (long long)pl->bpo * (n_samples >> j);
    FRT_CHECK_ARG(h, y_stride >= need, "y_stride smaller than the ragged output size");
    if (int rc = fir_check_block(h, pl, n_samples, "frt_firbank_process")) return rc;
    FirArgs a = {};
    a.x = x_dev;
    a.x_stride = x_stride;
    a.block = n_samples;
    a.n_blocks = 1;
    a.y = y_dev;
    a.y_stride = y_stride;
    return fir_launch(h, pl, a, stream);
}

extern "C" int frt_firbank_levels(frt_handle h, const float *x_dev, int64_t x_stride, int block, int n_blocks,
                                  float *levels_dev, int db, void *stream) {
    if (!h) return FRT_EINVAL;
    FirPlan *pl = h->fir.get();
    if (!pl) return frt_fail(h, FRT_ESTATE, "frt_firbank_levels: call frt_firbank_plan first");
    if (!pl->smoothing) return frt_fail(h, FRT_ESTATE, "frt_firbank_levels: call frt_firbank_set_smoothing first");
    DeviceGuard g(h->device);
    FRT_CHECK_ARG(h, block > 0, "block must be > 0");
    FRT_CHECK_ARG(h, n_blocks >= 0, "negative n_blocks");
    if (n_blocks == 0) return FRT_OK;
    FRT_CHECK_ARG(h, block <= FIR_MAX_BLOCK, "block must be <= 4096");
    FRT_CHECK_ARG(h, block % (1 << (pl->n_oct - 1)) == 0,
                  "block must be a multiple of 2^(n_octaves-1) (every stage keeps its even samples)");
    // exp_smoothed_value drops the carried value when a block is longer than its 8192/dec-tap
    // kernel (friture/signal/exp_smoothing.py:43-47); block <= 4096 keeps every stage clear of it
    for (int j = 0; j < pl->n_oct; j++)
        FRT_CHECK_ARG(h, (block >> j) <= (8192 >> j), "block longer than the smoothing kernel");
    FRT_CHECK_ARG(h, x_dev && levels_dev, "NULL buffer");
    FRT_CHECK_ARG(h, x_stride >= (int64_t)block * n_blocks, "x_stride smaller than block*n_blocks");
    if (int rc = fir_check_block(h, pl, block, "frt_firbank_levels")) return rc;
    FirArgs a = {};
    a.x = x_dev;
    a.x_stride = x_stride;
    a.block = block;
    a.n_blocks = n_blocks;
    a.alpha = pl->alpha.get();
    a.decay = pl->decay.get();
    a.weight_db = pl->weighted ? pl->weight_db.get() : nullptr;
    a.sp = pl->sp.get();
    a.levels = levels_dev;
    a.db = db;
    return fir_launch(h, pl, a, stream);
}
