// Multi-rate fractional-octave IIR filterbank + exponential RMS for sm_90a.
//
// Stands behind Octave_Filters.filter (friture/octavefilters.py:49-58) with the numerics of the
// reference's IIR bank octave_filter_bank_decimation (friture/filter.py:86-118: per stage j,
// bands bpo-1..0 filter x_j, then x_{j+1} = lowpass(x_j)[::2], friture/signal/decimate.py:39-41),
// and behind the widget's per-band smoothing exp_smoothed_value(y**2)
// (friture/octavespectrum.py:104, friture/signal/exp_smoothing.py:11-56).  The (b, a) filters of
// friture/generated_filters.py are run as float32 second-order sections (direct form II
// transposed, the recursion of friture/signal/lfilter.py:131-139 per section).
//
// ONE WARP PER CHANNEL.  An IIR recursion is serial in time, so the time axis of a tile of
// 32*L0 samples is split over the 32 lanes (lane l owns samples [l*L, (l+1)*L) of the stage's
// signal, in registers) and every biquad section is run as
//   pass 1  zero-state recursion over the lane's chunk -> local final state f_l
//   scan    s_l = A^L s_{l-1} + f_l over the lanes (5 shuffle steps with A^(L*2^k), 2x2)
//   pass 2  the recursion again from the true incoming state -> outputs, in place.
// The decimated output stays in the same lane (L halves each stage).  Once a stage has only
// 32 samples left per tile (one per lane) the remaining low-rate stages switch to
// "lane = filter chain": lanes 0..bpo-1 run the band chains and lane bpo the decimator chain
// serially over the <=32 samples, which are broadcast with shuffles.
// Filter and smoothing state lives in shared memory while the kernel runs (global in between).
#include <cmath>

#include "bank_internal.cuh"

namespace {

constexpr int MAX_BPO = BANK_MAX_BPO;
constexpr int MAX_OCT = BANK_MAX_OCT;
constexpr int NQ = BANK_NQ;

__device__ __forceinline__ float energy_out(float e, int db, const float *weight, int kband) {
    // friture/octavespectrum.py:119-121: 10*log10(sp + 1e-30) + w
    if (!db) return e;
    float v = kLog10Scale * lg2_fast(e + 1e-30f);
    if (weight) v += __ldg(weight + kband);
    return v;
}

// offset of band k in the ragged per-channel y layout (bands concatenated, k = 0 lowest)
__device__ __forceinline__ long long y_offset(int k, int bpo, int n_oct, long long t_total) {
    // bands of stage j (dec 2^j) are k = (n_oct-1-j)*bpo + i; lower k = higher j = shorter
    const int jk = n_oct - 1 - k / bpo;        // stage of band k
    const int i = k - (n_oct - 1 - jk) * bpo;
    // sum over stages j' > jk of bpo * (T >> j')  +  i * (T >> jk)
    long long off = 0;
    for (int j = n_oct - 1; j > jk; j--) off += (long long)bpo * (t_total >> j);
    return off + (long long)i * (t_total >> jk);
}

template <bool WANT_Y>
struct WarpCtxT {
    static constexpr bool kWantY = WANT_Y;   // compile the ragged-y stores in or out
    const BankParams *P;
    float *s_z;       // [n_oct][nsec][2]   this warp's filter state (shared memory)
    float *s_e;       // [n_oct][bpo]       this warp's smoothing state (e / alpha form)
    const float *s_coef;   // [nsec][8] CTA copy of the coefficients for lane-varying access
    float *energies;  // this channel, this block: [nbands] or NULL when not a block end
    float *y;         // this channel's ragged y base or NULL
    long long t_total;
    long long t_off;  // sample offset of this tile within the launch
    int lane;
    int db;
    const float *weight;   // dB offsets per band (db mode) or NULL
};

// context of channel c for the scan kernels; energies and t_off are set per tile
template <bool WANT_Y>
__device__ __forceinline__ void channel_ctx(WarpCtxT<WANT_Y> &w, const BankParams &P, const BankArgs &a,
                                            int c, int lane, float *s_z, float *s_e, const float *s_coef) {
    w.P = &P;
    w.s_z = s_z;
    w.s_e = s_e;
    w.s_coef = s_coef;
    w.lane = lane;
    w.db = a.db;
    w.weight = a.weight;
    w.t_total = a.t_total;
    w.y = a.y ? a.y + (size_t)c * a.y_stride : nullptr;
}

// this lane's L0 samples of a tile
template <int L0>
__device__ __forceinline__ void load_tile(const float *xp, bool vec_ok, float (&xc)[L0]) {
    if (vec_ok) {
#pragma unroll
        for (int k = 0; k < L0; k += 4) {
            const float4 v = __ldg(reinterpret_cast<const float4 *>(xp + k));
            xc[k] = v.x; xc[k + 1] = v.y; xc[k + 2] = v.z; xc[k + 3] = v.w;
        }
    } else {
#pragma unroll
        for (int k = 0; k < L0; k++) xc[k] = __ldg(xp + k);
    }
}

// where channel c writes its band energies after tile t, or NULL when t does not end a block
__device__ __forceinline__ float *block_energies(const BankArgs &a, int c, int t, int nbands) {
    const bool block_end = ((t + 1) % a.tiles_per_block) == 0;
    return (a.energies && block_end)
               ? a.energies + (size_t)c * a.e_stride + (size_t)(t / a.tiles_per_block) * nbands
               : nullptr;
}

// ---------------------------------------------------------------- scan-mode section
template <int L> struct Log2 { static constexpr int v = 1 + Log2<L / 2>::v; };
template <> struct Log2<1> { static constexpr int v = 0; };

template <int L, class W>
__device__ __forceinline__ void section_scan(const float (&in)[L], float (&out)[L],
                                             const W &w, int j, int sec) {
    const BankParams &P = *w.P;
    const float b0 = P.coef[sec][0], b1 = P.coef[sec][1], b2 = P.coef[sec][2];
    const float a1 = P.coef[sec][3], a2 = P.coef[sec][4];
    const float B1 = P.coef[sec][5], B2 = P.coef[sec][6];
    float *zp = w.s_z + (j * P.nsec + sec) * 2;
    const float c1 = zp[0], c2 = zp[1];
    // pass 1: state-only recursion from zero state
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int k = 0; k < L; k++) {
        const float x = in[k];
        const float n1 = fmaf(-a1, s1, fmaf(B1, x, s2));
        s2 = fmaf(-a2, s1, B2 * x);
        s1 = n1;
    }
    constexpr int q0 = Log2<L>::v;
    if (w.lane == 0) {   // fold the carried state into lane 0's segment
        const float *A = P.apow[sec][q0];
        s1 += fmaf(A[0], c1, A[1] * c2);
        s2 += fmaf(A[2], c1, A[3] * c2);
    }
#pragma unroll
    for (int k = 0; k < 5; k++) {
        const float *A = P.apow[sec][q0 + k];
        const float t1 = __shfl_up_sync(0xffffffffu, s1, 1 << k);
        const float t2 = __shfl_up_sync(0xffffffffu, s2, 1 << k);
        if (w.lane >= (1 << k)) {
            s1 = fmaf(A[0], t1, fmaf(A[1], t2, s1));
            s2 = fmaf(A[2], t1, fmaf(A[3], t2, s2));
        }
    }
    float i1 = __shfl_up_sync(0xffffffffu, s1, 1);
    float i2 = __shfl_up_sync(0xffffffffu, s2, 1);
    if (w.lane == 0) {
        i1 = c1;
        i2 = c2;
    }
    // pass 2: direct form II transposed (friture/signal/lfilter.py:131-139, order 2)
#pragma unroll
    for (int k = 0; k < L; k++) {
        const float x = in[k];
        const float y = fmaf(b0, x, i1);
        i1 = fmaf(-a1, y, fmaf(b1, x, i2));
        i2 = fmaf(-a2, y, b2 * x);
        out[k] = y;
    }
    __syncwarp();
    if (w.lane == 31) {   // state after the tile's last sample
        zp[0] = i1;
        zp[1] = i2;
    }
}

template <class W> __device__ __forceinline__ void serial_stages(float xin, int n, const W &w, int j);

// Band chains of one scan-mode stage (bands bpo-1 .. 0, friture/filter.py:105) with the smoothing
// of y^2: L samples per lane, 32 lanes active.
template <int L, class W>
__device__ __forceinline__ void bands_of_stage(const float (&xc)[L], const W &w, int j) {
    const BankParams &P = *w.P;
    const int bpo = P.bpo;
    float wk[L];
    for (int i = bpo - 1; i >= 0; i--) {
        section_scan<L>(xc, wk, w, j, 2 * i);
        section_scan<L>(wk, wk, w, j, 2 * i + 1);
        const int kband = (P.n_oct - 1 - j) * bpo + i;
        const float gb = P.gband[i];     // chain gain of the normalised sections
        if constexpr (W::kWantY) {
            float *yp = w.y + y_offset(kband, bpo, P.n_oct, w.t_total) + (w.t_off >> j) +
                        w.lane * L;
#pragma unroll
            for (int k = 0; k < L; k++) yp[k] = wk[k] * gb;
        }
        // exponential smoothing of y^2 (friture/signal/exp_smoothing.py:11-56), e/alpha form, in the
        // units of the normalised sections (the squared chain gain is applied to the output);
        // decays in complement form e - (1-q^n) e: the rounding of q must not bias long time constants
        const float om = P.omq[j][0];
        float e = 0.f;
#pragma unroll
        for (int k = 0; k < L; k++) e = fmaf(-om, e, e) + wk[k] * wk[k];
        float *ep = w.s_e + j * bpo + i;
        constexpr int q0 = Log2<L>::v;
        if (w.lane == 0) e += fmaf(-P.omq[j][q0], ep[0], ep[0]);
#pragma unroll
        for (int k = 0; k < 5; k++) {
            const float t = __shfl_up_sync(0xffffffffu, e, 1 << k);
            if (w.lane >= (1 << k)) e += fmaf(-P.omq[j][q0 + k], t, t);
        }
        __syncwarp();
        if (w.lane == 31) {
            ep[0] = e;
            if (w.energies) w.energies[kband] = energy_out(P.alpha[j] * gb * gb * e, w.db, w.weight, kband);
        }
    }
}

// Decimation low-pass of one scan-mode stage: 6 sections, full-rate output in wk
// (the caller keeps the even samples, friture/signal/decimate.py:39-41).
template <int L, class W>
__device__ __forceinline__ void dec_of_stage(const float (&xc)[L], float (&wk)[L], const W &w,
                                             int j) {
    const int bpo = w.P->bpo;
    section_scan<L>(xc, wk, w, j, 2 * bpo);
#pragma unroll 1
    for (int s = 1; s < 6; s++) section_scan<L>(wk, wk, w, j, 2 * bpo + s);
}

// One scan-mode stage, single-warp variant: bands, then the decimator, then the next stage.
template <int L, class W>
__device__ void scan_stage(const float (&xc)[L], const W &w, int j) {
    const BankParams &P = *w.P;
    bands_of_stage<L>(xc, w, j);
    if (j + 1 >= P.n_oct) return;   // the last decimator's output is discarded (filter.py:113)
    float wk[L];
    dec_of_stage<L>(xc, wk, w, j);
    if constexpr (L >= 4) {
        float xn[L / 2];
#pragma unroll
        for (int k = 0; k < L / 2; k++) xn[k] = wk[2 * k] * P.gdec;
        scan_stage<L / 2>(xn, w, j + 1);
    } else {
        // L == 2: one sample per lane is left -> switch to lane = chain
        serial_stages<W>(wk[0] * P.gdec, 32, w, j + 1);
    }
}

// ---- three-warp variant (one CTA of 96 threads per channel) --------------------------------
// warp 0 "D": decimator chain of the scan-mode stages (the critical path to the next stage),
// warp 1 "B": band chains of the scan-mode stages, one barrier behind D per stage,
// warp 2 "S": the low-rate serial stages of the PREVIOUS tile.
// D hands the decimated chunks to B through shared memory; named barrier 1 (64 threads) paces
// D and B stage by stage, __syncthreads() closes a tile.
__device__ __forceinline__ void bar_db() { asm volatile("bar.sync 1, 64;" ::: "memory"); }

template <int L, class W>
__device__ void stage_D(const float (&xc)[L], const W &w, int j, float *s_x, float *s_x32) {
    float wk[L];
    dec_of_stage<L>(xc, wk, w, j);
    if constexpr (L >= 4) {
        float xn[L / 2];
        float *dst = s_x + w.lane * (L / 2);     // stage j+1 chunk of this lane
#pragma unroll
        for (int k = 0; k < L / 2; k++) {
            xn[k] = wk[2 * k] * w.P->gdec;
            dst[k] = xn[k];
        }
        bar_db();
        stage_D<L / 2>(xn, w, j + 1, s_x + 32 * (L / 2), s_x32);
    } else {
        s_x32[w.lane] = wk[0] * w.P->gdec;       // 32 samples for the serial stages (warp S)
        bar_db();
    }
}

template <int L, class W>
__device__ void stage_B(const float (&xc)[L], const W &w, int j, const float *s_x) {
    bands_of_stage<L>(xc, w, j);
    bar_db();
    if constexpr (L >= 4) {
        float xn[L / 2];
        const float *src = s_x + w.lane * (L / 2);
#pragma unroll
        for (int k = 0; k < L / 2; k++) xn[k] = src[k];
        stage_B<L / 2>(xn, w, j + 1, s_x + 32 * (L / 2));
    }
}

// Serial-mode stages: the n samples of stage j sit one per lane (sample m in lane m).  Lane
// r < bpo runs band chain r (2 sections), lane bpo runs the decimator chain (6 sections); samples
// are broadcast one by one.  Continues through the remaining stages (n halves every stage).  One
// rolled copy of this code serves all low-rate stages: instruction-cache footprint matters here.
template <class W>
__device__ __forceinline__ void serial_stages(float xin, int n, const W &w, int j) {
    const BankParams &P = *w.P;
    const int bpo = P.bpo, lane = w.lane;
    const bool is_band = lane < bpo;
#pragma unroll 1
    for (; j < P.n_oct && n >= 1; j++, n >>= 1) {
        const bool last = (j + 1 >= P.n_oct);
        const bool is_dec = (lane == bpo) && !last;
        const int nchain = is_band ? 2 : (is_dec ? 6 : 0);
        const int sec0 = is_band ? 2 * lane : 2 * bpo;
        float z1[6], z2[6], cb0[6], cb1[6], cb2[6], ca1[6], ca2[6];
#pragma unroll
        for (int s = 0; s < 6; s++) {
            const bool on = s < nchain;
            const float *cf = w.s_coef + (sec0 + (on ? s : 0)) * 8;
            cb0[s] = cf[0]; cb1[s] = cf[1]; cb2[s] = cf[2]; ca1[s] = cf[3]; ca2[s] = cf[4];
            const float *zp = w.s_z + (j * P.nsec + sec0 + (on ? s : 0)) * 2;
            z1[s] = zp[0];
            z2[s] = zp[1];
        }
        const float om = P.omq[j][0];
        const float gout = is_band ? P.gband[is_band ? lane : 0] : P.gdec;   // chain gain
        // smoothing: this call's n samples are summed from zero and folded into the carried e once
        // (e <- q^n e + s, complement form), as the scan-mode stages do per chunk; a per-sample
        // recursion on the carried e rounds it once per sample over the 1/alpha samples it remembers
        float s = 0.f;
        const int kband = (P.n_oct - 1 - j) * bpo + (is_band ? lane : 0);
        float *yp = nullptr;
        if constexpr (W::kWantY) {
            if (is_band) yp = w.y + y_offset(kband, bpo, P.n_oct, w.t_total) + (w.t_off >> j);
        }
        float xnext = 0.f;
#pragma unroll 1
        for (int m = 0; m < n; m++) {
            float v = __shfl_sync(0xffffffffu, xin, m);
#pragma unroll
            for (int s = 0; s < 6; s++) {
                if (s < nchain) {
                    const float y = fmaf(cb0[s], v, z1[s]);
                    z1[s] = fmaf(-ca1[s], y, fmaf(cb1[s], v, z2[s]));
                    z2[s] = fmaf(-ca2[s], y, cb2[s] * v);
                    v = y;
                }
            }
            if (is_band) {
                s = fmaf(-om, s, s) + v * v;      // raw units; gain applied to the outputs
                if constexpr (W::kWantY) {
                    if (yp) yp[m] = v * gout;
                }
            } else {
                v *= gout;
            }
            if ((m & 1) == 0) {   // keep even samples (friture/signal/decimate.py:41)
                const float o = __shfl_sync(0xffffffffu, v, bpo);
                if (lane == (m >> 1)) xnext = o;
            }
        }
        __syncwarp();
#pragma unroll
        for (int s = 0; s < 6; s++) {
            if (s < nchain) {
                float *zp = w.s_z + (j * P.nsec + sec0 + s) * 2;
                zp[0] = z1[s];
                zp[1] = z2[s];
            }
        }
        if (is_band) {
            float e = w.s_e[j * bpo + lane];
            e = fmaf(-P.omq[j][__ffs(n) - 1], e, e) + s;   // n is a power of two, at most 32
            w.s_e[j * bpo + lane] = e;
            if (w.energies) w.energies[kband] = energy_out(P.alpha[j] * gout * gout * e, w.db, w.weight, kband);
        }
        __syncwarp();
        xin = xnext;
    }
}

template <int L0, bool WANT_Y>
__global__ void __launch_bounds__(64)
bank_kernel(const __grid_constant__ BankParams P, const BankArgs a) {
    extern __shared__ float smem[];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int warps = blockDim.x >> 5;
    const int nz = P.n_oct * P.nsec * 2, ne = P.n_oct * P.bpo;
    float *s_coef = smem;                        // [nsec][8]
    float *s_z = s_coef + P.nsec * 8 + wid * (nz + ne);
    float *s_e = s_z + nz;
    for (int i = threadIdx.x; i < P.nsec * 8; i += blockDim.x)
        s_coef[i] = P.coef[i >> 3][i & 7];
    const int c = blockIdx.x * warps + wid;
    const bool active = c < a.n_channels;
    if (active) {
        const float *gz = a.zstate + (size_t)c * nz;
        const float *ge = a.ema + (size_t)c * ne;
        for (int i = lane; i < nz; i += 32) s_z[i] = gz[i];
        for (int i = lane; i < ne; i += 32) s_e[i] = ge[i];   // e/alpha form: e = q e + y^2
    }
    __syncthreads();
    if (!active) return;

    constexpr int TILE = 32 * L0;
    const int nbands = P.n_oct * P.bpo;
    WarpCtxT<WANT_Y> w;
    channel_ctx<WANT_Y>(w, P, a, c, lane, s_z, s_e, s_coef);
    const float *xch = a.x + (size_t)c * a.x_stride;
    for (int t = 0; t < a.n_tiles; t++) {
        float xc[L0];
        load_tile<L0>(xch + (size_t)t * TILE + lane * L0, a.vec_ok, xc);
        w.energies = block_energies(a, c, t, nbands);
        w.t_off = (long long)t * TILE;
        scan_stage<L0>(xc, w, 0);
        __syncwarp();
    }
    // write the state back
    float *gz = a.zstate + (size_t)c * nz;
    float *ge = a.ema + (size_t)c * ne;
    for (int i = lane; i < nz; i += 32) gz[i] = s_z[i];
    for (int i = lane; i < ne; i += 32) ge[i] = s_e[i];
}

template <int L0, bool WANT_Y>
__global__ void __launch_bounds__(96)
bank_kernel3(const __grid_constant__ BankParams P, const BankArgs a) {
    extern __shared__ float smem[];
    const int lane = threadIdx.x & 31, role = threadIdx.x >> 5;
    const int nz = P.n_oct * P.nsec * 2, ne = P.n_oct * P.bpo;
    constexpr int TILE = 32 * L0;
    float *s_coef = smem;                        // [nsec][8]
    float *s_z = s_coef + P.nsec * 8;            // this channel's filter state
    float *s_e = s_z + nz;                       // this channel's smoothing state
    float *s_x = s_e + ne;                       // chunks of stages 1.. (TILE/2 + TILE/4 + ...)
    float *s_x32 = s_x + TILE;                   // [2][32] double-buffered input of the serial stages
    const int c = blockIdx.x;
    for (int i = threadIdx.x; i < P.nsec * 8; i += blockDim.x) s_coef[i] = P.coef[i >> 3][i & 7];
    {
        const float *gz = a.zstate + (size_t)c * nz;
        const float *ge = a.ema + (size_t)c * ne;
        for (int i = threadIdx.x; i < nz; i += blockDim.x) s_z[i] = gz[i];
        for (int i = threadIdx.x; i < ne; i += blockDim.x) s_e[i] = ge[i];
    }
    __syncthreads();
    const int nbands = P.n_oct * P.bpo;
    WarpCtxT<WANT_Y> w;
    channel_ctx<WANT_Y>(w, P, a, c, lane, s_z, s_e, s_coef);
    const float *xch = a.x + (size_t)c * a.x_stride;
    constexpr int NSCAN = Log2<L0>::v;           // scan-mode stages 0 .. NSCAN-1 (L = L0 .. 2)
    for (int t = 0; t <= a.n_tiles; t++) {
        if (role < 2 && t < a.n_tiles) {
            float xc[L0];
            load_tile<L0>(xch + (size_t)t * TILE + lane * L0, a.vec_ok, xc);
            w.energies = block_energies(a, c, t, nbands);
            w.t_off = (long long)t * TILE;
            if (role == 0) stage_D<L0>(xc, w, 0, s_x, s_x32 + (t & 1) * 32);
            else stage_B<L0>(xc, w, 0, s_x);
        } else if (role == 2 && t >= 1) {
            const int tp = t - 1;
            w.energies = block_energies(a, c, tp, nbands);
            w.t_off = (long long)tp * TILE;
            if (NSCAN < P.n_oct) serial_stages<WarpCtxT<WANT_Y>>(s_x32[(tp & 1) * 32 + lane], 32, w, NSCAN);
        }
        __syncthreads();
    }
    float *gz = a.zstate + (size_t)c * nz;
    float *ge = a.ema + (size_t)c * ne;
    for (int i = threadIdx.x; i < nz; i += blockDim.x) gz[i] = s_z[i];
    for (int i = threadIdx.x; i < ne; i += blockDim.x) ge[i] = s_e[i];
}

// ---- stand-alone N-fold decimation (decimate_multiple, friture/signal/decimate.py:45-71) ------
// The same 6-section low-pass as the bank's decimator, run NDEC times with [::2] in between, one
// warp per channel, tiles of 256 samples (L = 8, 4, ... per lane).  Used by the delay estimator
// (48 kHz -> 12 kHz with Ndec = 2, friture/delay_estimator.py:53-59,97-98).
struct DecArgs {
    const float *x;
    long long x_stride;
    float *out;
    long long out_stride;
    int n_channels, n_tiles, n_stages;
    float *zstate;   // [C][n_stages][6][2]
};

template <int L, class W>
__device__ void dec_chain(const float (&xc)[L], const W &w, int j, int n_stages, float *dst) {
    float wk[L];
    dec_of_stage<L>(xc, wk, w, j);
    if (j + 1 == n_stages) {
#pragma unroll
        for (int k = 0; k < L / 2; k++) dst[w.lane * (L / 2) + k] = wk[2 * k] * w.P->gdec;
        return;
    }
    if constexpr (L >= 4) {
        float xn[L / 2];
#pragma unroll
        for (int k = 0; k < L / 2; k++) xn[k] = wk[2 * k] * w.P->gdec;
        dec_chain<L / 2>(xn, w, j + 1, n_stages, dst);
    }
}

__global__ void __launch_bounds__(64)
decimate_kernel(const __grid_constant__ BankParams P, const DecArgs a) {
    extern __shared__ float smem[];
    constexpr int L0 = 8, TILE = 256;
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, warps = blockDim.x >> 5;
    const int nz = a.n_stages * P.nsec * 2;
    float *s_z = smem + wid * nz;
    const int c = blockIdx.x * warps + wid;
    if (c >= a.n_channels) return;
    float *gz = a.zstate + (size_t)c * nz;
    for (int i = lane; i < nz; i += 32) s_z[i] = gz[i];
    __syncwarp();
    WarpCtxT<false> w;
    w.P = &P;
    w.s_z = s_z;
    w.s_e = nullptr;
    w.s_coef = nullptr;
    w.energies = nullptr;
    w.y = nullptr;
    w.lane = lane;
    w.db = 0;
    w.weight = nullptr;
    w.t_total = 0;
    w.t_off = 0;
    const int out_tile = TILE >> a.n_stages;
    for (int t = 0; t < a.n_tiles; t++) {
        const float *xp = a.x + (size_t)c * a.x_stride + (size_t)t * TILE + lane * L0;
        float xc[L0];
#pragma unroll
        for (int k = 0; k < L0; k++) xc[k] = __ldg(xp + k);
        dec_chain<L0>(xc, w, 0, a.n_stages, a.out + (size_t)c * a.out_stride + (size_t)t * out_tile);
        __syncwarp();
    }
    for (int i = lane; i < nz; i += 32) gz[i] = s_z[i];
}

}   // namespace

void PlanDelete::operator()(BankPlan *p) const { delete p; }

static void mat2_mul(const double a[4], const double b[4], double o[4]) {
    o[0] = a[0] * b[0] + a[1] * b[2];
    o[1] = a[0] * b[1] + a[1] * b[3];
    o[2] = a[2] * b[0] + a[3] * b[2];
    o[3] = a[2] * b[1] + a[3] * b[3];
}

// Stores the SOS row s = (b0, b1, b2, a0, a1, a2) as normalised section sec of P (coefficients and
// the powers A^(2^q) the scan uses) and its gain g in *gain.  Elliptic sections have their zeros on
// the unit circle, b = g (1, c, 1); returns what is wrong with a row of another form, else NULL.
static const char *set_section(BankParams &P, int sec, const double *s, double *gain) {
    if (fabs(s[3] - 1.0) > 1e-12) return "a0 != 1";
    if (!(fabs(s[0]) > 0.0) || fabs(s[2] / s[0] - 1.0) > 1e-7) return "b2 != b0 (zeros off the unit circle)";
    *gain = s[0];
    P.coef[sec][0] = 1.f; P.coef[sec][1] = (float)(s[1] / s[0]); P.coef[sec][2] = 1.f;
    P.coef[sec][3] = (float)s[4]; P.coef[sec][4] = (float)s[5];
    // the scan must propagate the state of the float32 filter that pass 2 runs
    const double fb1 = P.coef[sec][1], fa1 = P.coef[sec][3], fa2 = P.coef[sec][4];
    P.coef[sec][5] = (float)(fb1 - fa1);
    P.coef[sec][6] = (float)(1.0 - fa2);
    double A[4] = {-fa1, 1.0, -fa2, 0.0};
    for (int q = 0; q < NQ; q++) {
        for (int i = 0; i < 4; i++) P.apow[sec][q][i] = (float)A[i];
        double A2[4];
        mat2_mul(A, A, A2);
        memcpy(A, A2, sizeof(A));
    }
    return nullptr;
}

extern "C" int frt_bank_plan(frt_handle h, int n_channels, int bands_per_octave, int n_octaves,
                             const double *sos_band, const double *sos_dec,
                             const double *alphas) {
    if (!h) return FRT_EINVAL;
    DeviceGuard g(h->device);
    FRT_CHECK_ARG(h, n_channels >= 1, "n_channels must be >= 1");
    FRT_CHECK_ARG(h, bands_per_octave >= 1 && bands_per_octave <= MAX_BPO,
                  "bands_per_octave must be in [1, 24]");
    FRT_CHECK_ARG(h, n_octaves >= 1 && n_octaves <= MAX_OCT, "n_octaves must be in [1, 10]");
    FRT_CHECK_ARG(h, sos_band && sos_dec && alphas, "NULL coefficient table");
    PlanPtr<BankPlan> pl(new (std::nothrow) BankPlan());
    if (!pl) return frt_fail(h, FRT_ENOMEM, "out of host memory");
    BankParams &P = pl->params;
    memset(&P, 0, sizeof(P));
    P.bpo = bands_per_octave;
    P.n_oct = n_octaves;
    P.nsec = 2 * bands_per_octave + 6;
    double gchain[BANK_MAX_BPO + 1];
    for (int i = 0; i <= bands_per_octave; i++) gchain[i] = 1.0;
    for (int sec = 0; sec < P.nsec; sec++) {
        const double *s = sec < 2 * bands_per_octave ? sos_band + (size_t)sec * 6
                                                     : sos_dec + (size_t)(sec - 2 * bands_per_octave) * 6;
        double g;
        if (const char *why = set_section(P, sec, s, &g))
            return frt_fail(h, FRT_EINVAL, "SOS section %d: %s", sec, why);
        gchain[sec < 2 * bands_per_octave ? sec / 2 : bands_per_octave] *= g;
    }
    for (int i = 0; i < bands_per_octave; i++) P.gband[i] = (float)gchain[i];
    P.gdec = (float)gchain[bands_per_octave];
    for (int j = 0; j < n_octaves; j++) {
        if (!(alphas[j] > 0.0 && alphas[j] <= 1.0))
            return frt_fail(h, FRT_EINVAL, "alpha[%d] must be in (0, 1]", j);
        P.alpha[j] = (float)alphas[j];
        pl->alphas[j] = alphas[j];
        double q = 1.0 - alphas[j];
        for (int k = 0; k < NQ; k++) {
            P.omq[j][k] = (float)(1.0 - q);
            q *= q;
        }
    }
    frt_pipe_prepare(pl.get());
    pl->n_channels = n_channels;
    pl->nz = (size_t)n_octaves * P.nsec * 2;
    pl->ne = (size_t)n_octaves * bands_per_octave;
    FRT_CUDA(h, pl->zstate.alloc(pl->nz * n_channels));
    FRT_CUDA(h, pl->ema.alloc(pl->ne * n_channels));
    FRT_CUDA(h, frt_sync_zero(pl->zstate.get(), sizeof(float) * pl->nz * n_channels));
    FRT_CUDA(h, frt_sync_zero(pl->ema.get(), sizeof(float) * pl->ne * n_channels));
    h->bank = std::move(pl);
    return FRT_OK;
}

extern "C" int frt_bank_reset(frt_handle h) {
    if (!h) return FRT_EINVAL;
    if (!h->bank) return frt_fail(h, FRT_ESTATE, "frt_bank_reset: no plan");
    DeviceGuard g(h->device);
    BankPlan *pl = h->bank.get();
    FRT_CUDA(h, frt_sync_zero(pl->zstate.get(), sizeof(float) * pl->nz * pl->n_channels));
    FRT_CUDA(h, frt_sync_zero(pl->ema.get(), sizeof(float) * pl->ne * pl->n_channels));
    return FRT_OK;
}

extern "C" int frt_bank_set_weighting(frt_handle h, const float *weight_db_host) {
    if (!h) return FRT_EINVAL;
    if (!h->bank) return frt_fail(h, FRT_ESTATE, "frt_bank_set_weighting: no plan");
    DeviceGuard g(h->device);
    BankPlan *pl = h->bank.get();
    const size_t nb = (size_t)pl->params.n_oct * pl->params.bpo;
    FRT_CUDA(h, cudaDeviceSynchronize());
    if (!weight_db_host) {
        pl->weight = {};
        return FRT_OK;
    }
    if (!pl->weight.get()) FRT_CUDA(h, pl->weight.alloc(nb));
    FRT_CUDA(h, frt_sync_copy(pl->weight.get(), weight_db_host, sizeof(float) * nb, cudaMemcpyHostToDevice));
    return FRT_OK;
}

extern "C" int frt_bank_schedule(int n_octaves, int log2_chunk, int64_t n_samples, int *stage_start,
                                 int *n_steps) {
    if (n_octaves < 1 || n_octaves > MAX_OCT || (log2_chunk != 5 && log2_chunk != 6) || !stage_start ||
        n_samples < 0)
        return FRT_EINVAL;
    int T[BANK_MAX_OCT + 1];
    frt_pipe_schedule(n_octaves, log2_chunk, n_samples, T, n_steps);
    for (int j = 0; j < MAX_OCT; j++) stage_start[j] = T[j];
    return FRT_OK;
}

extern "C" int frt_bank_state_size(frt_handle h, int64_t *z_floats, int64_t *ema_floats) {
    if (!h) return FRT_EINVAL;
    if (!h->bank) return frt_fail(h, FRT_ESTATE, "frt_bank_state_size: no plan");
    if (z_floats) *z_floats = (int64_t)(h->bank->nz * h->bank->n_channels);
    if (ema_floats) *ema_floats = (int64_t)(h->bank->ne * h->bank->n_channels);
    return FRT_OK;
}

extern "C" int frt_bank_get_state(frt_handle h, float *z_host, float *ema_host) {
    if (!h) return FRT_EINVAL;
    if (!h->bank) return frt_fail(h, FRT_ESTATE, "frt_bank_get_state: no plan");
    DeviceGuard g(h->device);
    BankPlan *pl = h->bank.get();
    if (z_host)
        FRT_CUDA(h, frt_sync_copy(z_host, pl->zstate.get(), sizeof(float) * pl->nz * pl->n_channels,
                                  cudaMemcpyDeviceToHost));
    if (ema_host)
        FRT_CUDA(h, frt_sync_copy(ema_host, pl->ema.get(), sizeof(float) * pl->ne * pl->n_channels,
                                  cudaMemcpyDeviceToHost));
    return FRT_OK;
}

extern "C" int frt_bank_set_state(frt_handle h, const float *z_host, const float *ema_host) {
    if (!h) return FRT_EINVAL;
    if (!h->bank) return frt_fail(h, FRT_ESTATE, "frt_bank_set_state: no plan");
    DeviceGuard g(h->device);
    BankPlan *pl = h->bank.get();
    if (z_host)
        FRT_CUDA(h, frt_sync_copy(pl->zstate.get(), z_host, sizeof(float) * pl->nz * pl->n_channels,
                                  cudaMemcpyHostToDevice));
    if (ema_host)
        FRT_CUDA(h, frt_sync_copy(pl->ema.get(), ema_host, sizeof(float) * pl->ne * pl->n_channels,
                                  cudaMemcpyHostToDevice));
    return FRT_OK;
}

// How blocks of `block` samples run for a plan: refused (`why`), or the kernel family and variant.
struct BankRoute {
    const char *why;
    enum Kind { PIPE, SCAN, SCAN3 } kind;
    int L0;            // samples per lane of the chunk-scan kernels' 32 * L0-sample tile
    int logch, pack;   // PIPE: 2^logch-sample steps, channels per lane
};

// The one statement of the filterbank's block rule and kernel choice.  It depends on the plan, the
// block and whether band outputs are wanted, not on how a stream is cut: the bits are the same.
static BankRoute bank_route(const BankPlan *pl, int block, bool want_y) {
    const BankParams &P = pl->params;
    // blocks stay even-length at every stage (decimate.py:41 restarts the [::2] phase on every call),
    // down to the chunk-scan kernels' tile: the longest of 1024, 512 and 256 samples dividing the block
    if (block <= 0 || block % 256) return {"block must be a multiple of 256 samples"};
    const int tile = block % 1024 == 0 ? 1024 : block % 512 == 0 ? 512 : 256;
    if ((tile >> (P.n_oct - 1)) < 1) return {"block too short for this many octaves"};
    const int L0 = tile / 32;
    // The lane-pipelined kernel (bank_pipe.cu) is the fast path for the fused energies of 1- and
    // 1/3-octave banks (pipe_ok): 64-sample steps up to 3072 channels, above that 32-sample steps with
    // two channels per lane.  64-sample steps start at 512-sample blocks: a 256-sample block is four
    // such steps, and its band energies would need 9 slots of the 8-slot ring at 10 octaves.
    if (pl->pipe_ok && !want_y && (block & (block - 1)) == 0) {
        const int pack = pl->n_channels > 3072 ? 2 : 1;
        const int logch = (pack == 1 && block >= PIPE_MIN_BLOCK[1]) ? 6 : 5;
        return {nullptr, BankRoute::PIPE, L0, logch, pack};
    }
    // Chunk-scan kernels: three warps per channel below 1536 channels (latency-bound); above, one warp
    // per channel saturates the schedulers with less synchronisation.  The three-warp kernel, compiled
    // for L0 <= 16, runs all log2(L0) scan-mode stages, so it needs more octaves than that.
    const bool three = L0 <= 16 && L0 < (1 << P.n_oct) && pl->n_channels < 1536;
    return {nullptr, three ? BankRoute::SCAN3 : BankRoute::SCAN, L0};
}

int frt_bank_check_block(frt_ctx *h, const BankPlan *pl, int block) {
    const char *why = bank_route(pl, block, false).why;
    return why ? frt_fail(h, FRT_EINVAL, "%s (block %d)", why, block) : FRT_OK;
}

// one warp per channel, two channels per CTA
template <int L0>
static int launch_scan(frt_handle h, const BankPlan *pl, const BankArgs &a, cudaStream_t st) {
    const BankParams &P = pl->params;
    const int warps = 2;
    const size_t smem = sizeof(float) * ((size_t)P.nsec * 8 + (size_t)warps * (pl->nz + pl->ne));
    const unsigned blocks = (unsigned)((a.n_channels + warps - 1) / warps);
    return frt_launch(h, a.y ? bank_kernel<L0, true> : bank_kernel<L0, false>, blocks, warps * 32, smem, st, P, a);
}

// one CTA of three warps per channel
template <int L0>
static int launch_scan3(frt_handle h, const BankPlan *pl, const BankArgs &a, cudaStream_t st) {
    const BankParams &P = pl->params;
    const size_t smem = sizeof(float) * ((size_t)P.nsec * 8 + pl->nz + pl->ne + 32 * L0 + 64);
    const auto kernel = a.y ? bank_kernel3<L0, true> : bank_kernel3<L0, false>;
    return frt_launch(h, kernel, (unsigned)a.n_channels, 96, smem, st, P, a);
}

static int bank_process_impl(frt_handle h, const float *x_dev, int64_t x_stride, int block,
                             int n_blocks, float *energies_dev, int64_t e_stride, float *y_dev,
                             int64_t y_stride, int db, void *stream) {
    if (!h) return FRT_EINVAL;
    if (!h->bank) return frt_fail(h, FRT_ESTATE, "frt_bank_process: call frt_bank_plan first");
    DeviceGuard g(h->device);
    BankPlan *pl = h->bank.get();
    const BankParams &P = pl->params;
    FRT_CHECK_ARG(h, n_blocks >= 0 && block >= 0, "negative shape");
    if (n_blocks == 0 || block == 0) return FRT_OK;   // empty chunk: octavespectrum.py:94-95
    const BankRoute r = bank_route(pl, block, y_dev != nullptr);
    if (r.why) return frt_fail(h, FRT_EINVAL, "%s (block %d)", r.why, block);
    FRT_CHECK_ARG(h, x_dev != nullptr, "x_dev is NULL");
    FRT_CHECK_ARG(h, x_stride >= (int64_t)block * n_blocks, "x_stride too small");
    const long long t_total = (long long)block * n_blocks;
    if (y_dev) {
        long long need = 0;
        for (int j = 0; j < P.n_oct; j++) need += (long long)P.bpo * (t_total >> j);
        FRT_CHECK_ARG(h, y_stride >= need, "y_stride smaller than the ragged output size");
    }
    BankArgs a;
    a.x = x_dev;
    a.x_stride = x_stride;
    a.n_channels = pl->n_channels;
    a.n_tiles = (int)(t_total / (32 * r.L0));
    a.tiles_per_block = block / (32 * r.L0);
    a.zstate = pl->zstate.get();
    a.ema = pl->ema.get();
    a.energies = energies_dev;
    a.e_stride = e_stride;
    a.y = y_dev;
    a.y_stride = y_stride;
    a.t_total = t_total;
    a.db = db;
    a.vec_ok = (((uintptr_t)x_dev & 15) == 0) && ((x_stride & 3) == 0);
    a.weight = db ? pl->weight.get() : nullptr;
    a.block = block;
    a.n_blocks = n_blocks;
    a.n_steps = 0;
    cudaStream_t st = (cudaStream_t)stream;
    switch (r.kind) {
    case BankRoute::PIPE: return frt_pipe_launch(h, pl, a, r.logch, r.pack, st);
    case BankRoute::SCAN3: return r.L0 == 16 ? launch_scan3<16>(h, pl, a, st) : launch_scan3<8>(h, pl, a, st);
    default:
        return r.L0 == 32 ? launch_scan<32>(h, pl, a, st)
             : r.L0 == 16 ? launch_scan<16>(h, pl, a, st) : launch_scan<8>(h, pl, a, st);
    }
}

extern "C" int frt_bank_process(frt_handle h, const float *x_dev, int64_t x_stride, int block,
                                int n_blocks, float *energies_dev, float *y_dev,
                                int64_t y_stride, int db, void *stream) {
    if (!h) return FRT_EINVAL;
    const int64_t nb = h->bank ? (int64_t)h->bank->params.n_oct * h->bank->params.bpo : 0;
    return bank_process_impl(h, x_dev, x_stride, block, n_blocks, energies_dev, (int64_t)n_blocks * nb,
                             y_dev, y_stride, db, stream);
}

extern "C" int frt_bank_process_strided(frt_handle h, const float *x_dev, int64_t x_stride, int block,
                                        int n_blocks, float *energies_dev, int64_t e_stride_c, int db,
                                        void *stream) {
    if (!h) return FRT_EINVAL;
    if (h->bank && energies_dev) {
        const int64_t nb = (int64_t)h->bank->params.n_oct * h->bank->params.bpo;
        if (e_stride_c < (int64_t)n_blocks * nb)
            return frt_fail(h, FRT_EINVAL, "e_stride_c smaller than n_blocks * nbands");
    }
    return bank_process_impl(h, x_dev, x_stride, block, n_blocks, energies_dev, e_stride_c, nullptr, 0, db,
                             stream);
}

// ---------------------------------------------------------------------------------------------
struct DecPlan {
    BankParams params;
    int n_channels = 0, n_stages = 0;
    DeviceArray<float> zstate;
};

void PlanDelete::operator()(DecPlan *p) const { delete p; }

extern "C" int frt_decimate_plan(frt_handle h, int n_channels, int n_stages, const double *sos_dec) {
    if (!h) return FRT_EINVAL;
    DeviceGuard g(h->device);
    FRT_CHECK_ARG(h, n_channels >= 1, "n_channels must be >= 1");
    FRT_CHECK_ARG(h, n_stages >= 1 && n_stages <= 2, "n_stages must be 1 or 2");
    FRT_CHECK_ARG(h, sos_dec != nullptr, "NULL coefficient table");
    PlanPtr<DecPlan> pl(new (std::nothrow) DecPlan());
    if (!pl) return frt_fail(h, FRT_ENOMEM, "out of host memory");
    BankParams &P = pl->params;
    memset(&P, 0, sizeof(P));
    P.bpo = 0;          // section index 2*bpo + s = s: the six decimator sections
    P.n_oct = n_stages;
    P.nsec = 6;
    double gdec = 1.0;
    for (int sec = 0; sec < 6; sec++) {
        double g;
        if (const char *why = set_section(P, sec, sos_dec + (size_t)sec * 6, &g))
            return frt_fail(h, FRT_EINVAL, "decimator section %d is not of the form g(1,c,1)/(1,a1,a2): %s",
                            sec, why);
        gdec *= g;
    }
    P.gdec = (float)gdec;
    pl->n_channels = n_channels;
    pl->n_stages = n_stages;
    const size_t nz = (size_t)n_stages * 6 * 2 * n_channels;
    FRT_CUDA(h, pl->zstate.alloc(nz));
    FRT_CUDA(h, frt_sync_zero(pl->zstate.get(), sizeof(float) * nz));
    h->dec = std::move(pl);
    return FRT_OK;
}

extern "C" int frt_decimate_process(frt_handle h, const float *x_dev, int64_t x_stride,
                                    int64_t n_samples, float *out_dev, int64_t out_stride,
                                    void *stream) {
    if (!h) return FRT_EINVAL;
    const DecPlan *pl = h->dec.get();
    if (!pl) return frt_fail(h, FRT_ESTATE, "frt_decimate_process: call frt_decimate_plan first");
    DeviceGuard g(h->device);
    FRT_CHECK_ARG(h, n_samples >= 0, "negative length");
    if (n_samples == 0) return FRT_OK;   // decimate_multiple returns empty input unchanged (:56-57)
    FRT_CHECK_ARG(h, n_samples % 256 == 0, "n_samples must be a multiple of 256");
    FRT_CHECK_ARG(h, x_dev && out_dev, "NULL buffer");
    FRT_CHECK_ARG(h, x_stride >= n_samples && out_stride >= (n_samples >> pl->n_stages),
                  "stride too small");
    DecArgs a;
    a.x = x_dev;
    a.x_stride = x_stride;
    a.out = out_dev;
    a.out_stride = out_stride;
    a.n_channels = pl->n_channels;
    a.n_tiles = (int)(n_samples / 256);
    a.n_stages = pl->n_stages;
    a.zstate = pl->zstate.get();
    const int warps = 2;
    const size_t smem = sizeof(float) * warps * pl->n_stages * 12;
    return frt_launch(h, decimate_kernel, (pl->n_channels + warps - 1) / warps, warps * 32, smem,
                      (cudaStream_t)stream, pl->params, a);
}
