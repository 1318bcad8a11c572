// Fused STFT for sm_90a: Hann window -> real FFT -> |X|^2/N^2 -> (10*log10(.+1e-30)), one pass
// HBM -> HBM, no cuFFT.  Stands behind audioproc.analyzelive (friture/audioproc.py:42-50), the
// framing loops of friture/spectrogram.py:131-159 / friture/spectrum.py:125-155 and
// log_spectrogram (friture/spectrogram.py:119-125).
//
// A real FFT of N points is computed as a complex FFT of M = N/2 points on
// z[n] = x[2n] + j*x[2n+1], followed by the split step
//     X[k]   = (E + T)/2,  X[M-k] = conj(E - T)/2,
//     E = Z[k] + conj(Z[M-k]),  O = Z[k] - conj(Z[M-k]),  T = (-j*W_N^k) * O.
//
// N = 64 Q, Q in {1, .., 32} (64 .. 2048 points, the benchmark's size is 2048): ONE WARP PER 32/Q
//   FRAMES (stft_small_kernel).  At N = 2048, M = 1024 = 32 x 32:
//   lane t holds z[32*n1 + t] (n1 = 0..31) in registers -> radix-32 DFT over n1 in registers
//   -> twiddle W_M^(k1*t) -> 32x32 transpose through a warp-private padded smem tile
//   -> radix-32 DFT over n2 -> lane t holds X[t + 32*k2]; the split partner X[M-k] lives in
//   lane (32-t)%32 and is fetched with warp shuffles.  Only __syncwarp(), no block barrier.
//   Complex arithmetic is written on float2 through the component-wise f2_* helpers (two FADDs
//   per complex add, one FMUL + one FFMA per component of a complex multiply).
// N = 4096 / 8192: R = 2 / 4 warps per frame, each a 1024-point FFT of a decimated sequence, radix-R
//   combine through shared memory (stft_large_kernel; stft_multi_kernel for unaligned input and 16384).
// Generic path (N = 32): one CTA per frame, Stockham radix-4 (+ one radix-2 pass when log2(M) is
//   odd) ping-ponging between two shared-memory buffers.
#include <algorithm>
#include <cmath>
#include <type_traits>
#include <utility>

#include "frt_internal.cuh"

namespace {

constexpr float kEps = 1e-30f;                        // friture/spectrogram.py:124

__device__ __forceinline__ float2 cadd(float2 a, float2 b) { return f2_add(a, b); }
__device__ __forceinline__ float2 csub(float2 a, float2 b) {
    return f2_add(a, make_float2(-b.x, -b.y));
}
// a * w
__device__ __forceinline__ float2 cmul(float2 a, float2 w) {
    float2 t = f2_mul(a, make_float2(w.x, w.x));
    return f2_fma(make_float2(-a.y, a.x), make_float2(w.y, w.y), t);
}
// a * (-j)
__device__ __forceinline__ float2 mul_mj(float2 a) { return make_float2(a.y, -a.x); }

// cos/sin(2*pi*i/32), i = 0..15
__device__ __forceinline__ constexpr float cos32(int i) {
    constexpr float t[16] = {1.0f,
                             0.98078528040323044913f,
                             0.92387953251128675613f,
                             0.83146961230254523708f,
                             0.70710678118654752440f,
                             0.55557023301960222474f,
                             0.38268343236508977173f,
                             0.19509032201612826785f,
                             0.0f,
                             -0.19509032201612826785f,
                             -0.38268343236508977173f,
                             -0.55557023301960222474f,
                             -0.70710678118654752440f,
                             -0.83146961230254523708f,
                             -0.92387953251128675613f,
                             -0.98078528040323044913f};
    return t[i];
}
__device__ __forceinline__ constexpr float sin32(int i) {
    constexpr float t[16] = {0.0f,
                             0.19509032201612826785f,
                             0.38268343236508977173f,
                             0.55557023301960222474f,
                             0.70710678118654752440f,
                             0.83146961230254523708f,
                             0.92387953251128675613f,
                             0.98078528040323044913f,
                             1.0f,
                             0.98078528040323044913f,
                             0.92387953251128675613f,
                             0.83146961230254523708f,
                             0.70710678118654752440f,
                             0.55557023301960222474f,
                             0.38268343236508977173f,
                             0.19509032201612826785f};
    return t[i];
}

__host__ __device__ constexpr int brev5(int r) {
    return ((r & 1) << 4) | ((r & 2) << 2) | (r & 4) | ((r & 8) >> 2) | ((r & 16) >> 4);
}

// LEN-point radix-2 DIF butterfly stages (spans LEN, LEN/2, .., 2) on each group of LEN consecutive
// registers.  The span is a template parameter so that every loop has a compile-time trip count and
// unrolls completely: v[] must stay in registers.
template <int LEN>
__device__ __forceinline__ void dft_stages(float2 (&v)[32]) {
    constexpr int half = LEN >> 1;
    constexpr int tstep = 32 / LEN;
#pragma unroll
    for (int base = 0; base < 32; base += LEN) {
#pragma unroll
        for (int i = 0; i < half; i++) {
            const float2 a = v[base + i], b = v[base + i + half];
            v[base + i] = cadd(a, b);
            const float2 d = csub(a, b);
            const int ti = i * tstep;
            if (ti == 0)
                v[base + i + half] = d;
            else if (ti == 8)
                v[base + i + half] = mul_mj(d);
            else
                v[base + i + half] = cmul(d, make_float2(cos32(ti), -sin32(ti)));
        }
    }
    if constexpr (LEN > 2) dft_stages<LEN / 2>(v);
}

// In-register radix-32 DFT (decimation in frequency, fully unrolled): v[r] <- bin brev5(r).
__device__ __forceinline__ void dft32(float2 (&v)[32]) { dft_stages<32>(v); }

// 32/LEN independent LEN-point DFTs on consecutive register groups (same butterflies as dft32,
// started at span LEN): v[g*LEN + r] <- bin brevq<LEN>(r) of group g.
template <int LEN>
__device__ __forceinline__ void dft_groups(float2 (&v)[32]) { dft_stages<LEN>(v); }
template <int Q>
__host__ __device__ constexpr int brevq(int r) {
    int o = 0;
    for (int b = 1, c = Q >> 1; b < Q; b <<= 1, c >>= 1)
        if (r & b) o |= c;
    return o;
}

// Fourth output of the STFT kernels (frt_spectrum_frames / _dual): each frame's power column goes
// straight into the spectrum widget's smoothing (smooth_step) and is never stored.  kModeSmoothDual
// transforms a (reference, measurement) pair per channel and smooths both.
constexpr int kModeScreen = 2;
constexpr int kModeSmooth = 3;
constexpr int kModeSmoothDual = 4;
// the smoothed states per channel: 0 for the other outputs
__host__ __device__ constexpr int smooth_nch(int mode) {
    return mode == kModeSmooth ? 1 : (mode == kModeSmoothDual ? 2 : 0);
}

template <int MODE>
__device__ __forceinline__ float finish(float mag2, float scale) {
    // mag2*scale = |X|^2/N^2 (audioproc.py:49-50); log mode: spectrogram.py:119-125.  The smoothing
    // output rounds the product on its own, so that no contraction reaches into the smoothing.
    if (smooth_nch(MODE)) return __fmul_rn(mag2, scale);
    if (MODE == FRT_STFT_POWER) return mag2 * scale;
    return kLog10Scale * lg2_fast(fmaf(mag2, scale, kEps));
}

// Third output of the STFT kernels (frt_stft_screen_rows): the frame's log-power column, computed as
// FRT_STFT_LOGPOWER computes it, stays in shared memory and only its `height` screen rows are written,
// row r = screen_value of the column (what display_kernel computes from a stored column).  Every kernel
// family takes the output as its MODE template argument and the screen tables as its last parameter,
// which the other modes leave unused (launched as ScreenRows{}).
struct ScreenRows {
    const float *weight;   // [nbins] dB or NULL
    const int *i0;         // [height] bin index of each row, 0 <= i0 <= nbins - 2
    const float *t;        // [height] its fraction toward bin i0 + 1
    float spec_min, inv_range;
    int height;
};

// Rows i, i + n, .. of one frame from its column in shared memory.  The barrier before it makes the
// column's values opaque to the compiler, so that no contraction reaches across into screen_value.
__device__ __forceinline__ void write_rows(const float *s_col, float *__restrict__ rows, const ScreenRows &s,
                                           int i, int n) {
    for (int r = i; r < s.height; r += n)
        rows[r] = screen_value<true>(s_col, s.weight, __ldg(s.i0 + r), __ldg(s.t + r), s.spec_min, s.inv_range);
}

// The smoothing outputs' arguments (the other modes launch with SmoothTicks{}).  Channel c's frames are
// those of frt_stft_process; in kModeSmoothDual frame f of its measurement row starts at
// x2 + c x_stride + f hop.  A slot walks its channel's frames as items i = NCH f + j in order (j = 1:
// the measurement), every item's power column going into state j.
struct SmoothTicks {
    const float *x2;
    const int *tick_end;   // [n_ticks] the frame at which each tick ends, strictly ascending
    int n_ticks, n_channels;
    float alpha;
    float *disp[2];        // [C][nbins] carried states, float32
    const float *weight;   // [nbins] dB or NULL (kModeSmooth)
    float *db;             // row r of channel c at db + c db_sc + r db_sr, or NULL
    long long db_sc, db_sr;
    int *imax, *ipitch;    // [n_ticks][C]
};

// One slot of a smoothing output: n threads (t = 0..n-1, whole warps) walk one channel's frames in
// order, its NCH states in shared memory in double (st: [NCH][nb]).  A state is read from disp once at
// the channel's start and written once at its end, and each tick end rounds it to float32, writes the
// tick's dB row and its two arg-maxes, as spectrum_reduce_kernel does for one tick.  s_val / s_idx:
// [n/32] scratch of the arg-maxes when the slot has more than one warp; sync() is the slot's barrier.
template <int NCH, class Sync>
struct Smoother {
    const SmoothTicks &sm;
    double *st;
    double *s_val;
    int *s_idx;
    int nb, t, n;
    Sync sync;
    double a;
    long long c = 0;
    int r = 0;

    __device__ Smoother(const SmoothTicks &sm_, double *st_, double *s_val_, int *s_idx_, int nb_, int t_, int n_,
                        Sync sync_)
        : sm(sm_), st(st_), s_val(s_val_), s_idx(s_idx_), nb(nb_), t(t_), n(n_), sync(sync_), a(sm_.alpha) {}

    __device__ void begin(long long ch) {
        c = ch;
        r = 0;
        for (int j = 0; j < NCH; j++)
            for (int k = t; k < nb; k += n) st[j * nb + k] = sm.disp[j][(size_t)c * nb + k];
        sync();
    }
    __device__ __forceinline__ void add(int j, int k, float p) { st[j * nb + k] = smooth_step(st[j * nb + k], p, a); }
    // after item i of the channel, every thread's adds made: the end of a tick?
    __device__ __forceinline__ void after(long long i) {
        if (i % NCH == NCH - 1 && r < sm.n_ticks && i / NCH + 1 == __ldg(sm.tick_end + r)) tick();
    }
    __device__ void end() {
        sync();
        for (int j = 0; j < NCH; j++)
            for (int k = t; k < nb; k += n) sm.disp[j][(size_t)c * nb + k] = (float)st[j * nb + k];
    }

    // the slot's first arg-max, in every thread
    __device__ int argmax(double best, int besti) {
        for (int o = 16; o > 0; o >>= 1) {
            const double ob = __shfl_xor_sync(0xffffffffu, best, o);
            const int oi = __shfl_xor_sync(0xffffffffu, besti, o);
            argmax_merge(best, besti, ob, oi);
        }
        if (n > 32) {
            sync();
            if ((t & 31) == 0) {
                s_val[t >> 5] = best;
                s_idx[t >> 5] = besti;
            }
            sync();
            best = -INFINITY;
            besti = 0x7fffffff;
            for (int w = 0; w < n / 32; w++) argmax_merge(best, besti, s_val[w], s_idx[w]);
        }
        return besti;
    }

    __device__ void tick() {
        sync();   // every bin has had the tick's frames
        float best = -INFINITY;
        int besti = 0x7fffffff;
        for (int k = t; k < nb; k += n) {
            const float v = (float)st[k];
            st[k] = v;
            float d;
            if constexpr (NCH == 2) {
                const float v2 = (float)st[nb + k];
                st[nb + k] = v2;
                d = db_dual(v, v2);
            } else {
                d = db_single(v, sm.weight, k);
            }
            if (sm.db) sm.db[c * sm.db_sc + r * sm.db_sr + k] = d;
            if (d > best) {   // on the float32 value, as spectrum_reduce_kernel
                best = d;
                besti = k;
            }
        }
        const int imax = argmax(best, besti);     // spectrum.py:175
        sync();   // every bin of state 0 is rounded
        double bp = -INFINITY;
        int bpi = 0x7fffffff;
        for (int k = t; k < nb / 3; k += n) {
            const double h = hps_term(st, k);
            if (h > bp) {
                bp = h;
                bpi = k;
            }
        }
        const int ipitch = argmax(bp, bpi);       // spectrum.py:180
        if (t == 0) {
            sm.imax[(size_t)r * sm.n_channels + c] = imax;
            sm.ipitch[(size_t)r * sm.n_channels + c] = ipitch;
        }
        r++;
        sync();   // the states are read before the next frame's adds
    }
};

// shared memory of one slot's states and arg-max scratch (warps: the slot's)
template <int MODE>
__host__ __device__ constexpr size_t smooth_slot_bytes(int nbins, int warps) {
    return smooth_nch(MODE)
               ? (sizeof(double) * smooth_nch(MODE) * nbins + (sizeof(double) + sizeof(int)) * warps + 15) / 16 * 16
               : 0;
}
template <int NCH, class Sync>
__device__ Smoother<NCH, Sync> slot_smoother(const SmoothTicks &sm, void *slot_smem, int nb, int t, int n, Sync sync) {
    double *st = reinterpret_cast<double *>(slot_smem);
    double *s_val = st + NCH * nb;
    return Smoother<NCH, Sync>(sm, st, s_val, reinterpret_cast<int *>(s_val + n / 32), nb, t, n, sync);
}

// frame f of channel c (in the smoothing outputs: item f of the channel)
template <int MODE>
__device__ __forceinline__ const float *frame_at(const float *x, const SmoothTicks &sm, long long x_stride, int hop,
                                                 long long c, long long f) {
    if constexpr (MODE == kModeSmoothDual) return ((f & 1) ? sm.x2 : x) + c * x_stride + (f >> 1) * hop;
    else return x + c * x_stride + f * hop;
}

// ---- TMA bulk copy (cp.async.bulk, SASS UBLKCP) + mbarrier helpers ------------------------------
__device__ __forceinline__ void mbar_init(unsigned long long *bar, unsigned count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(unsigned long long *bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)),
                 "r"(bytes)
                 : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long *bar, unsigned parity) {
    asm volatile(
        "{\n"
        ".reg .pred p;\n"
        "WAIT_LOOP:\n"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
        "@p bra WAIT_DONE;\n"
        "bra WAIT_LOOP;\n"
        "WAIT_DONE:\n"
        "}\n" ::"r"(smem_u32(bar)),
        "r"(parity)
        : "memory");
}
// global -> shared bulk copy by the TMA engine, completion signalled on the mbarrier
__device__ __forceinline__ void bulk_g2s(void *dst_smem, const void *src_gmem, unsigned bytes,
                                         unsigned long long *bar) {
    asm volatile(
        "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::
            "r"(smem_u32(dst_smem)),
        "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
        : "memory");
}
__device__ __forceinline__ void fence_proxy_async() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}

constexpr int TILE = 32 * 33;   // padded 32x32 complex tile per warp

// First half of the second radix-32 pass: twiddle W_M^(k1 t) and the transpose through the warp's
// padded tile.  Lane t holds 32/Q groups of Q bins k1 (register g*Q + r holds k1 = brevq<Q>(r) of
// group g); afterwards lane g*Q + k1 holds the 32 values over t of group g, residue k1, and the tile
// is free again.  The caller finishes the pass with dft32.
template <int Q>
__device__ __forceinline__ void twiddle_transpose(float2 (&v)[32], const float2 *s_tw, float2 *s_x,
                                                  int lane) {
#pragma unroll
    for (int r = 0; r < Q; r++) {
        const int k1 = brevq<Q>(r);
        const float2 w = s_tw[k1 * 32 + lane];
#pragma unroll
        for (int g = 0; g < 32 / Q; g++) {
            const float2 val = (k1 == 0) ? v[g * Q + r] : cmul(v[g * Q + r], w);
            s_x[(g * Q + k1) * 33 + lane] = val;
        }
    }
    __syncwarp();
#pragma unroll
    for (int n2 = 0; n2 < 32; n2++) v[n2] = s_x[lane * 33 + n2];
    __syncwarp();
}

// ------------------------------------------------------------------------------------------
// N = 4096 / 8192 (the spectrogram's and the spectrum's default sizes) and 16384: R = 2 / 4 / 8
// warps per frame.
// Warp w runs the 1024-point complex FFT of the decimated sequence z[R n + w] exactly like the
// N = 2048 kernel (radix-32 x 32 in registers, one transpose through its smem tile), leaves
// Z_w[k0] in natural order in the tile, and after one block barrier the CTA combines
//   Z[k0 + 1024 q] = sum_w W_R^(w q) W_M^(w k0) Z_w[k0]          (M = 1024 R)
// and applies the real-FFT split step.  The partner of bin k0 + 1024 q is (1024 - k0) + 1024 (R-1-q),
// so a thread that builds the groups of k0 and 1024 - k0 has all 2R bins it needs in registers.
template <int R> __device__ __forceinline__ void combine(float2 (&t)[R]);
template <> __device__ __forceinline__ void combine<2>(float2 (&t)[2]) {
    const float2 a = t[0], b = t[1];
    t[0] = cadd(a, b);
    t[1] = csub(a, b);
}
template <> __device__ __forceinline__ void combine<4>(float2 (&t)[4]) {
    const float2 s02 = cadd(t[0], t[2]), d02 = csub(t[0], t[2]);
    const float2 s13 = cadd(t[1], t[3]), d13 = mul_mj(csub(t[1], t[3]));
    t[0] = cadd(s02, s13);
    t[1] = cadd(d02, d13);
    t[2] = csub(s02, s13);
    t[3] = csub(d02, d13);
}

template <> __device__ __forceinline__ void combine<8>(float2 (&t)[8]) {
    float2 e[4] = {t[0], t[2], t[4], t[6]}, o[4] = {t[1], t[3], t[5], t[7]};
    combine<4>(e);
    combine<4>(o);
    const float h = 0.70710678118654752440f;
    // W_8^q o_q: q = 1: (1 - j)/sqrt2, q = 2: -j, q = 3: (-1 - j)/sqrt2
    const float2 o1 = make_float2(h * (o[1].x + o[1].y), h * (o[1].y - o[1].x));
    const float2 o2 = mul_mj(o[2]);
    const float2 o3 = make_float2(h * (o[3].y - o[3].x), -h * (o[3].x + o[3].y));
    t[0] = cadd(e[0], o[0]); t[4] = csub(e[0], o[0]);
    t[1] = cadd(e[1], o1);   t[5] = csub(e[1], o1);
    t[2] = cadd(e[2], o2);   t[6] = csub(e[2], o2);
    t[3] = cadd(e[3], o3);   t[7] = csub(e[3], o3);
}

// The R-warp kernels' last stage: radix-R combine of the R natural-order tiles Z_w and the split
// step of every bin of the frame, by thread t of the frame's 32 R threads.  comb(w, k0) and post(kk)
// read W_M^(w k0) and U[kk] from wherever the kernel keeps those tables.  The bins go to o, or in the
// smoothing outputs to add(k, power): a bin's value is the last one o would hold (bin M/2 is split twice).
template <int R, int MODE, class Comb, class Post, class Add>
__device__ __forceinline__ void combine_split(float *__restrict__ o, Add add, const float2 *tiles, Comb comb,
                                              Post post, int t, float scale) {
    constexpr int M = 1024 * R;
    auto load_group = [&](int k0, float2(&g)[R]) {
        g[0] = tiles[k0];
#pragma unroll
        for (int w = 1; w < R; w++) g[w] = cmul(tiles[w * TILE + k0], comb(w, k0));
        combine<R>(g);
    };
    auto split_store = [&](int kk, float2 z, float2 zp) {
        const float2 E = make_float2(z.x + zp.x, z.y - zp.y);
        const float2 O = make_float2(z.x - zp.x, z.y + zp.y);
        const float2 T = cmul(O, post(kk));
        const float2 X = cadd(E, T);
        const float2 Y = csub(E, T);
        if constexpr (smooth_nch(MODE)) {
            if (kk != M - kk) add(kk, finish<MODE>(fmaf(X.x, X.x, X.y * X.y), scale));
            add(M - kk, finish<MODE>(fmaf(Y.x, Y.x, Y.y * Y.y), scale));
        } else {
            o[kk] = finish<MODE>(fmaf(X.x, X.x, X.y * X.y), scale);
            o[M - kk] = finish<MODE>(fmaf(Y.x, Y.x, Y.y * Y.y), scale);
        }
    };
    for (int k0 = 1 + t; k0 < 512; k0 += 32 * R) {
        float2 A[R], B[R];
        load_group(k0, A);
        load_group(1024 - k0, B);
#pragma unroll
        for (int q = 0; q < R; q++) split_store(k0 + 1024 * q, A[q], B[R - 1 - q]);
    }
    if (t == 0) {          // k0 = 0: partners inside the group, q <-> R - q
        float2 A[R];
        load_group(0, A);
        split_store(0, A[0], A[0]);
#pragma unroll
        for (int q = 1; q <= R / 2; q++) split_store(1024 * q, A[q], A[R - q]);
    }
    if (t == 32) {         // k0 = 512: partners inside the group, q <-> R - 1 - q
        float2 A[R];
        load_group(512, A);
#pragma unroll
        for (int q = 0; q < R / 2; q++) split_store(512 + 1024 * q, A[q], A[R - 1 - q]);
    }
}

// kModeScreen: the frame's column goes to s_col, after the tiles, and its rows to out.  Smoothing
// outputs: one CTA per channel, its states after the tiles.
template <int R, int MODE>
__global__ void __launch_bounds__(32 * R)
stft_multi_kernel(const float *__restrict__ x, long long x_stride, long long n_frames, int hop,
                  float *__restrict__ out, long long out_stride_c, long long out_stride_f,
                  const float2 *__restrict__ win2, const float2 *__restrict__ tw32,
                  const float2 *__restrict__ comb, const float2 *__restrict__ post,
                  long long total_items, int vec_ok, const ScreenRows scr, const SmoothTicks sm) {
    constexpr int M = 1024 * R, N = 2 * M, NCH = smooth_nch(MODE);
    extern __shared__ float2 smem[];
    float2 *s_tw = smem;                       // [32][32] W_1024^(k1 t)
    float2 *s_tiles = s_tw + 1024;             // R padded tiles
    float *s_col = reinterpret_cast<float *>(s_tiles + R * TILE);   // kModeScreen: [M + 1]
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, tid = threadIdx.x;
    float2 *s_x = s_tiles + warp * TILE;
    for (int i = tid; i < 1024; i += blockDim.x) s_tw[i] = tw32[i];
    __syncthreads();
    const float scale = 1.0f / (4.0f * (float)N * (float)N);
    // the frame at p into the natural-order tiles, for the combine
    auto transform = [&](const float *p) {
        float2 v[32];
#pragma unroll
        for (int n1 = 0; n1 < 32; n1++) {
            const int idx = R * (32 * n1 + lane) + warp;      // z[idx] = x[2 idx] + j x[2 idx + 1]
            float2 xv;
            if (vec_ok) {
                xv = __ldg(reinterpret_cast<const float2 *>(p) + idx);
            } else {
                xv.x = __ldg(p + 2 * idx);
                xv.y = __ldg(p + 2 * idx + 1);
            }
            v[n1] = f2_mul(xv, __ldg(win2 + idx));
        }
        dft32(v);
        twiddle_transpose<32>(v, s_tw, s_x, lane);
        dft32(v);   // v[r] = Z_w[lane + 32*brev5(r)]
#pragma unroll
        for (int r = 0; r < 32; r++) s_x[lane + 32 * brev5(r)] = v[r];   // natural order
        __syncthreads();
    };
    auto comb_at = [=](int w, int k0) { return __ldg(comb + (w - 1) * 1024 + k0); };
    auto post_at = [=](int kk) { return __ldg(post + kk); };
    if constexpr (NCH > 0) {
        auto sync = [] { __syncthreads(); };
        auto s = slot_smoother<NCH>(sm, s_tiles + R * TILE, M + 1, tid, 32 * R, sync);
        for (long long c = blockIdx.x; c < sm.n_channels; c += gridDim.x) {
            s.begin(c);
            for (long long i = 0; i < NCH * n_frames; i++) {
                transform(frame_at<MODE>(x, sm, x_stride, hop, c, i));
                const int j = (int)(i % NCH);
                combine_split<R, MODE>(nullptr, [&](int k, float p) { s.add(j, k, p); }, s_tiles, comb_at, post_at,
                                       tid, scale);
                __syncthreads();
                s.after(i);
            }
            s.end();
        }
    } else {
        for (long long item = blockIdx.x; item < total_items; item += gridDim.x) {
            const long long c = item / n_frames;
            const long long f = item - c * n_frames;
            transform(x + c * x_stride + f * hop);
            auto no_add = [](int, float) {};
            if constexpr (MODE == kModeScreen) {
                combine_split<R, MODE>(s_col, no_add, s_tiles, comb_at, post_at, tid, scale);
                __syncthreads();
                // s_col is rewritten only after the next frame's tile barrier
                write_rows(s_col, out + c * out_stride_c + f * out_stride_f, scr, tid, 32 * R);
            } else {
                combine_split<R, MODE>(out + c * out_stride_c + f * out_stride_f, no_add, s_tiles, comb_at, post_at,
                                       tid, scale);
                __syncthreads();
            }
        }
    }
}

// ------------------------------------------------------------------------------------------
// N = 64 Q, Q in {1, 2, 4, 8, 16, 32} (64 .. 2048 points): ONE WARP PER G = 32/Q FRAMES.
// M = N/2 = 32 Q.  Lane t holds z_g[32 n1 + t] (n1 < Q) of each of the G frames in register g*Q + n1,
// so the register file is as full at every size as at N = 2048: G radix-Q DFTs in registers -> twiddle
// W_M^(k1 t) -> ONE 32x32 transpose through the warp's tile, after which lane g*Q + k1 holds the 32
// values (over t) of frame g, residue k1 -> radix-32 DFT -> that lane owns Z_g[k1 + Q k2], k2 = 0..31.
// The split partner M - (k1 + Q m) = (Q - k1) + Q (31 - m) lives in lane g*Q + (Q - k1) % Q (the
// lane itself when k1 = 0), one shuffle away.  Window, twiddle and split tables are read once per
// G frames.
// Q = 32 (N = 2048, one frame per warp) runs one CTA of 16 warps per SM, and with TMA its 16-byte
// aligned frames are staged by the TMA engine; smaller Q run two CTAs of 8 warps per SM.
// Smoothing outputs: one warp per channel, its states after the mbarriers.  At Q = 32 a lane adds the
// bins it splits (the same ones in every frame); smaller Q write the warp's G columns to its tile, as
// kModeScreen does, and add them in frame order.  Q = 32 runs 8 warps there, for the states' room.
template <int Q, int MODE = FRT_STFT_POWER> __host__ __device__ constexpr int small_warps() {
    return Q == 32 ? (smooth_nch(MODE) ? 8 : 16) : 8;
}
template <int Q, int MODE = FRT_STFT_POWER> __host__ __device__ constexpr int small_ctas_per_sm() {
    return Q == 32 || smooth_nch(MODE) ? 1 : 2;
}
// Byte offsets of stft_small_kernel's shared memory; small_smem() is its size.  kModeScreen: the warp's
// G columns go to its tile, free again after the transpose; with TMA the tile already holds the next
// frame by then, so each warp has a column buffer of its own after the mbarriers.
template <int Q, int MODE, bool TMA>
struct SmallSmem {
    static constexpr int W = small_warps<Q, MODE>(), M = 32 * Q;
    static constexpr size_t win = 0;                                    // [M]      (w[2n], w[2n+1])
    static constexpr size_t tw = win + sizeof(float2) * M;              // [Q][32]  W_M^(k1 t)
    static constexpr size_t post = tw + sizeof(float2) * M;             // [M/2]    U[k] = -j W_N^k
    static constexpr size_t tiles = post + sizeof(float2) * (M / 2);    // [W]      padded tiles
    static constexpr size_t bars = tiles + sizeof(float2) * W * TILE;   // (Q = 32) [W] mbarriers
    static constexpr size_t cols = bars + (Q == 32 ? sizeof(unsigned long long) * W : 0);   // (kModeScreen, TMA)
    static constexpr size_t slots = cols + (MODE == kModeScreen && TMA ? sizeof(float) * W * (M + 1) : 0);
    static constexpr size_t end = slots + W * smooth_slot_bytes<MODE>(M + 1, 1);   // (smoothing) [W] slots
    static_assert(tiles % 16 == 0 && TILE * sizeof(float2) % 16 == 0,
                  "the TMA engine writes each warp's tile in 16-byte units");
};
template <int Q, int MODE, bool TMA>
constexpr size_t small_smem() {
    return SmallSmem<Q, MODE, TMA>::end;
}

template <int Q, int MODE, bool TMA>
__global__ void __launch_bounds__(small_warps<Q, MODE>() * 32, small_ctas_per_sm<Q, MODE>())
stft_small_kernel(const float *__restrict__ x, long long x_stride, long long n_frames, int hop,
                  float *__restrict__ out, long long out_stride_c, long long out_stride_f,
                  const float2 *__restrict__ win2, const float2 *__restrict__ tw,
                  const float2 *__restrict__ post, long long total_items, int vec_ok, const ScreenRows scr,
                  const SmoothTicks sm) {
    static_assert(!TMA || Q == 32, "TMA staging is for one frame per warp");
    using L = SmallSmem<Q, MODE, TMA>;
    constexpr int G = 32 / Q, M = 32 * Q, N = 2 * M, WARPS = small_warps<Q, MODE>(), NCH = smooth_nch(MODE);
    extern __shared__ float2 smem[];
    float2 *s_win = smem + L::win / sizeof(float2);   // every region starts on 8 bytes
    float2 *s_tw = smem + L::tw / sizeof(float2);
    float2 *s_post = smem + L::post / sizeof(float2);
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float2 *s_x = smem + L::tiles / sizeof(float2) + warp * TILE;
    for (int i = threadIdx.x; i < M; i += blockDim.x) {
        s_win[i] = win2[i];
        s_tw[i] = tw[i];
    }
    for (int i = threadIdx.x; i < 16 * Q; i += blockDim.x) s_post[i] = post[i];
    __syncthreads();

    // The steps both loops below take.  TMA: the warp's mbarrier, before the loop's first fetch.
    unsigned long long *bar = reinterpret_cast<unsigned long long *>(smem + L::bars / sizeof(float2)) + warp;
    auto init_bar = [&] {
        if (TMA) {
            if (lane == 0) mbar_init(bar, 1);
            fence_proxy_async();
            __syncwarp();
        }
    };
    // window, first pass and transpose of the group in v: v[g*Q + r] = sum_n1 z_g[32 n1 + t] W_Q^(n1 k1),
    // k1 = brevq<Q>(r), then twiddled and transposed; the tile is free again afterwards
    auto first_pass = [&](float2(&v)[32]) {
#pragma unroll
        for (int n1 = 0; n1 < Q; n1++) {
            const float2 w = s_win[32 * n1 + lane];
#pragma unroll
            for (int g = 0; g < G; g++) v[g * Q + n1] = f2_mul(v[g * Q + n1], w);
        }
        dft_groups<Q>(v);
        twiddle_transpose<Q>(v, s_tw, s_x, lane);
    };
    // the split step of the lane's bins k = k1 + Q m, their partners M - k and (k1 = 0) bin M/2, after
    // the second pass: put(k, value of bin k), if the lane's frame exists (ok)
    auto split = [&](const float2(&v)[32], int k1, int src_lane, float scale, bool ok, auto put) {
#pragma unroll
        for (int m = 0; m < 16; m++) {
            const float2 z = v[brev5(m)];
            const float2 other = v[brev5(31 - m)];
            float2 zp;
            zp.x = __shfl_sync(0xffffffffu, other.x, src_lane);
            zp.y = __shfl_sync(0xffffffffu, other.y, src_lane);
            if (k1 == 0) zp = (m == 0) ? v[0] : v[brev5(32 - m)];
            const float2 E = make_float2(z.x + zp.x, z.y - zp.y);
            const float2 O = make_float2(z.x - zp.x, z.y + zp.y);
            const int k = k1 + Q * m;
            const float2 T = cmul(O, s_post[k]);
            const float2 X = cadd(E, T);
            const float2 Y = csub(E, T);
            const float p1 = fmaf(X.x, X.x, X.y * X.y);
            const float p2 = fmaf(Y.x, Y.x, Y.y * Y.y);
            if (ok) {
                put(k, finish<MODE>(p1, scale));
                put(M - k, finish<MODE>(p2, scale));
            }
        }
        if (k1 == 0 && ok) {
            const float2 z = v[brev5(16)];   // bin M/2: X = conj(Z)
            put(M / 2, finish<MODE>(4.0f * fmaf(z.x, z.x, z.y * z.y), scale));
        }
    };

    // Smoothing outputs: warp gw walks channels gw, gw + warps_total, ..; its items are a channel's frames
    // (kModeSmoothDual: reference and measurement in turn, frame_at).  The other outputs keep the loop below
    // to themselves, so that their code is what it was before this output existed; both loops call the
    // steps above.
    if constexpr (NCH > 0) {
        const long long warps_total = (long long)gridDim.x * WARPS;
        const float scale = 1.0f / (4.0f * (float)N * (float)N);
        const int k1 = lane & (Q - 1), gsel = lane / Q;
        const int src_lane = (lane - k1) + ((Q - k1) & (Q - 1));
        unsigned char *slot = reinterpret_cast<unsigned char *>(smem + L::slots / sizeof(float2)) +
                              warp * smooth_slot_bytes<MODE>(M + 1, 1);
        auto s = slot_smoother<NCH>(sm, slot, M + 1, lane, 32, [] { __syncwarp(); });
        unsigned parity = 0;
        init_bar();
        const long long nv = NCH * n_frames;
        for (long long ch = (long long)blockIdx.x * WARPS + warp; ch < sm.n_channels; ch += warps_total) {
            s.begin(ch);
            long long f = 0;   // the next item to load
            if (TMA && lane == 0) {
                mbar_expect_tx(bar, N * 4);
                bulk_g2s(s_x, frame_at<MODE>(x, sm, x_stride, hop, ch, 0), N * 4, bar);
            }
            for (long long item = 0; item < nv; item += G) {
                float2 v[32];
                long long myf = 0;
                bool myok = false;
#pragma unroll
                for (int g = 0; g < G; g++, f++) {
                    const bool ok = f < nv;
                    const float *p = frame_at<MODE>(x, sm, x_stride, hop, ch, f);
                    if (g == gsel) {
                        myf = f;
                        myok = ok;
                    }
                    if (TMA) {
                        mbar_wait(bar, parity);
                        parity ^= 1;
#pragma unroll
                        for (int n1 = 0; n1 < 32; n1++) v[n1] = s_x[32 * n1 + lane];
                        __syncwarp();   // every lane has its samples before the tile is reused for the exchange
                    } else if (ok && vec_ok) {
#pragma unroll
                        for (int n1 = 0; n1 < Q; n1++)
                            v[g * Q + n1] = __ldg(reinterpret_cast<const float2 *>(p) + 32 * n1 + lane);
                    } else if (ok) {
#pragma unroll
                        for (int n1 = 0; n1 < Q; n1++) {
                            v[g * Q + n1].x = __ldg(p + 64 * n1 + 2 * lane);
                            v[g * Q + n1].y = __ldg(p + 64 * n1 + 2 * lane + 1);
                        }
                    } else {
#pragma unroll
                        for (int n1 = 0; n1 < Q; n1++) v[g * Q + n1] = make_float2(0.0f, 0.0f);
                    }
                }
                first_pass(v);
                if (TMA && f < nv) {   // the tile is free: fetch the next item into it
                    fence_proxy_async();
                    if (lane == 0) {
                        mbar_expect_tx(bar, N * 4);
                        bulk_g2s(s_x, frame_at<MODE>(x, sm, x_stride, hop, ch, f), N * 4, bar);
                    }
                }
                dft32(v);   // v[r] = Z_g[k1 + Q*brev5(r)] of this lane's (g, k1)

                // G = 1: the lane's bins go straight into state j; G > 1: frame g's column to the tile
                constexpr bool direct = G == 1;
                const int j = (int)(myf % NCH);
                float *o = reinterpret_cast<float *>(s_x) + gsel * (M + 1);
                split(v, k1, src_lane, scale, myok, [&](int k, float p) {
                    if constexpr (direct) s.add(j, k, p);
                    else o[k] = p;
                });
                __syncwarp();   // every add, or the warp's G columns, complete
                if constexpr (direct) {
                    s.after(myf);
                } else {
                    const float *s_col = reinterpret_cast<const float *>(s_x);
#pragma unroll 1
                    for (int g = 0; g < G; g++) {   // in frame order; a lane adds the same bins every time
                        const long long fg = item + g;
                        if (fg >= nv) break;
                        const int jg = (int)(fg % NCH);
                        for (int k = lane; k <= M; k += 32) s.add(jg, k, s_col[g * (M + 1) + k]);
                        s.after(fg);
                    }
                    __syncwarp();   // every lane is done with the columns before the tile is written again
                }
            }
            s.end();
        }
    } else {
        // contiguous range of frames per warp, a multiple of G long
        // (consecutive frames of a channel stay on one SM, so the overlapping part of each frame is
        // re-read from L1/L2, not HBM)
        const long long warps_total = (long long)gridDim.x * WARPS;
        const long long gw = (long long)blockIdx.x * WARPS + warp;
        long long per = (total_items + warps_total - 1) / warps_total;
        per = (per + G - 1) / G * G;
        long long item = gw * per;
        long long item_end = item + per;
        if (item_end > total_items) item_end = total_items;
        const float scale = 1.0f / (4.0f * (float)N * (float)N);
        const int k1 = lane & (Q - 1), gsel = lane / Q;
        const int src_lane = (lane - k1) + ((Q - k1) & (Q - 1));

        long long c = (item < item_end) ? item / n_frames : 0;
        long long f = item - c * n_frames;
        // TMA: each frame's 8 KB are fetched by the TMA engine (cp.async.bulk) into the warp's tile
        // while the frame before it is in its second FFT pass and split step, so no warp ever waits on
        // a global load with its registers tied up.  The first frame is fetched here, each next one
        // once the transpose has freed the tile.
        unsigned parity = 0;
        init_bar();
        if (TMA && lane == 0 && item < item_end) {
            mbar_expect_tx(bar, N * 4);
            bulk_g2s(s_x, x + c * x_stride + f * hop, N * 4, bar);
        }
        for (; item < item_end; item += G) {
            float2 v[32];
            long long myc = 0, myf = 0;
            bool myok = false;
#pragma unroll
            for (int g = 0; g < G; g++) {
                const bool ok = item + g < item_end;
                const float *p = x + c * x_stride + f * hop;
                if (g == gsel) {
                    myc = c;
                    myf = f;
                    myok = ok;
                }
                if (TMA) {
                    mbar_wait(bar, parity);
                    parity ^= 1;
#pragma unroll
                    for (int n1 = 0; n1 < 32; n1++) v[n1] = s_x[32 * n1 + lane];
                    __syncwarp();   // every lane has its samples before the tile is reused for the exchange
                } else if (ok && vec_ok) {
#pragma unroll
                    for (int n1 = 0; n1 < Q; n1++)
                        v[g * Q + n1] = __ldg(reinterpret_cast<const float2 *>(p) + 32 * n1 + lane);
                } else if (ok) {
#pragma unroll
                    for (int n1 = 0; n1 < Q; n1++) {
                        v[g * Q + n1].x = __ldg(p + 64 * n1 + 2 * lane);
                        v[g * Q + n1].y = __ldg(p + 64 * n1 + 2 * lane + 1);
                    }
                } else {
#pragma unroll
                    for (int n1 = 0; n1 < Q; n1++) v[g * Q + n1] = make_float2(0.0f, 0.0f);
                }
                if (++f == n_frames) {
                    f = 0;
                    c++;
                }
            }
            first_pass(v);
            if (TMA && item + 1 < item_end) {   // the tile is free: fetch the next frame, (c, f), into it
                fence_proxy_async();
                if (lane == 0) {
                    mbar_expect_tx(bar, N * 4);
                    bulk_g2s(s_x, x + c * x_stride + f * hop, N * 4, bar);
                }
            }
            dft32(v);   // v[r] = Z_g[k1 + Q*brev5(r)] of this lane's (g, k1)

            float *o;
            if constexpr (MODE == kModeScreen) {
                float *s_col = reinterpret_cast<float *>(s_x);
                if (TMA) s_col = reinterpret_cast<float *>(smem + L::cols / sizeof(float2)) + warp * (M + 1);
                o = s_col + gsel * (M + 1);
            } else {
                o = out + myc * out_stride_c + myf * out_stride_f;
            }
            split(v, k1, src_lane, scale, myok, [&](int k, float p) { o[k] = p; });
            if constexpr (MODE == kModeScreen) {
                __syncwarp();   // the warp's G columns are complete
                const float *s_col = o - gsel * (M + 1);
#pragma unroll
                for (int g = 0; g < G; g++) {   // frame g's (channel, frame) from the lanes that hold it
                    const long long cg = __shfl_sync(0xffffffffu, myc, g * Q);
                    const long long fg = __shfl_sync(0xffffffffu, myf, g * Q);
                    if (__shfl_sync(0xffffffffu, (int)myok, g * Q))
                        write_rows(s_col + g * (M + 1), out + cg * out_stride_c + fg * out_stride_f, scr, lane, 32);
                }
                __syncwarp();   // every lane is done with the columns before the tile is written again
            }
        }
    }
}

// ------------------------------------------------------------------------------------------
// N = 4096 / 8192, 8-byte aligned input: the stft_multi_kernel decomposition (R warps per frame, each a
// 1024-point complex FFT of a decimated sequence, then a radix-R combine + split step) rebuilt
// around shared memory: one CTA of 16 warps (16/R frame groups) per SM, every table resident in shared
// memory, the frame fetched by 8-byte cp.async that DE-INTERLEAVES it on the way in (element e of the
// frame lands in warp e % R's tile at e / R, staggered by w*32/R so that the scatter is conflict
// free), named barriers per group instead of block barriers.
// The Hann window is computed on the fly (this kernel is bound by shared-memory wavefronts, not by
// the FMA pipe): w[n] = 0.5 - 0.5 cos(theta n), theta = 2 pi/(N-1), and for warp w, lane t, register
// n1, element e the sample index is n = 64 R n1 + (2 R t + 2 w + e) = A-part + B-part, so
// cos(theta n) = cos A cos B - sin A sin B with 32 (cos A, sin A)/2 pairs passed as a kernel
// argument (constant bank) and the four B factors of a lane held in registers.  Near both ends of
// the frame 0.5 - 0.5 cos(theta n) cancels (a relative error of up to 1.5e-2, and w[N-1] = 1e-8
// instead of 0), so register blocks n1 = 0 and 31 take float32(Hann) from the window table, read
// once per thread; the other blocks stay within 2.4e-6 of the exact window.
// kModeScreen: each frame group's column goes to a buffer of its own after the tiles (the tiles are read
// until the split step ends).  At R = 4 sixteen warps' tiles, tables and four such buffers exceed the
// 227 KB a CTA may hold, so that instantiation runs twelve warps (three frame groups).
// Smoothing outputs: one frame group per channel, its states after the tiles, each thread adding the bins
// it splits (the same ones in every frame).  A group's states take 16 KB (R = 2) or 32 KB (R = 4) per
// channel of the pair, so these run eight warps, and four (one group) at R = 4 in kModeSmoothDual.
template <int R, int MODE>
__host__ __device__ constexpr int large_warps() {
    if (smooth_nch(MODE)) return (R == 4 && MODE == kModeSmoothDual) ? 4 : 8;
    return (MODE == kModeScreen && R == 4) ? 12 : 16;
}
struct HannA {
    float2 v[32];     // (0.5 cos(theta 64 R n1), 0.5 sin(theta 64 R n1))
};
template <int R, int MODE>
constexpr size_t large_smem() {
    // tw [1024] + comb [R-1][1024] + post [512 R + 1 -> even] + tiles (+ kModeScreen: the groups' columns;
    // smoothing: the groups' states)
    constexpr int W = large_warps<R, MODE>();
    return sizeof(float2) * (1024 + 1024 * (R - 1) + 512 * R + 2 + (size_t)W * TILE) +
           (MODE == kModeScreen ? sizeof(float) * (size_t)(W / R) * (1024 * R + 1) : 0) +
           (W / R) * smooth_slot_bytes<MODE>(1024 * R + 1, R);
}

__device__ __forceinline__ void group_barrier(int id, int nthreads) {
    asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory");
}

// split twiddle U[kk] = -j W_N^kk for kk in [0, M] from a table of M/2 + 1 entries:
// U[kk + M/2] = -j U[kk]
__device__ __forceinline__ float2 post_lookup(const float2 *s_post, int kk, int half_m) {
    if (kk <= half_m) return s_post[kk];
    return mul_mj(s_post[kk - half_m]);
}

template <int R, int MODE>
__global__ void __launch_bounds__(large_warps<R, MODE>() * 32, 1)
stft_large_kernel(const float *__restrict__ x, long long x_stride, long long n_frames, int hop,
                  float *__restrict__ out, long long out_stride_c, long long out_stride_f,
                  const float2 *__restrict__ win2, const float4 *__restrict__ wlane,
                  const float2 *__restrict__ tw32, const float2 *__restrict__ comb,
                  const float2 *__restrict__ post, long long total_items,
                  const __grid_constant__ HannA hann_a, const ScreenRows scr, const SmoothTicks sm) {
    // STAG: 8-byte shared accesses are served per half-warp; the 16/R elements a half-warp sends to
    // each of the R tiles must fall on different banks
    constexpr int LARGE_WARPS = large_warps<R, MODE>();
    constexpr int M = 1024 * R, N = 2 * M, NG = LARGE_WARPS / R, GT = 32 * R, STAG = 16 / R, NCH = smooth_nch(MODE);
    extern __shared__ float2 smem[];
    float2 *s_tw = smem;                          // [32][32] W_1024^(k1 t)
    float2 *s_comb = s_tw + 1024;                 // [R-1][1024] W_M^(w k0)
    float2 *s_post = s_comb + 1024 * (R - 1);     // [M/2 + 1] U[k]
    float2 *s_tiles_all = s_post + 512 * R + 2;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int grp = warp / R, w = warp % R, gtid = tid - grp * GT;
    float2 *s_tiles = s_tiles_all + (size_t)grp * R * TILE;   // this group's R tiles
    float2 *s_x = s_tiles + w * TILE;
    float *s_col = reinterpret_cast<float *>(s_tiles_all + (size_t)LARGE_WARPS * TILE) + grp * (M + 1);
    for (int i = tid; i < 1024; i += blockDim.x) s_tw[i] = tw32[i];
    for (int i = tid; i < 1024 * (R - 1); i += blockDim.x) s_comb[i] = comb[i];
    for (int i = tid; i <= 512 * R; i += blockDim.x) s_post[i] = post[i];
    __syncthreads();

    const long long groups_total = (long long)gridDim.x * NG;
    const long long gg = (long long)blockIdx.x * NG + grp;
    const float scale = 1.0f / (4.0f * (float)N * (float)N);
    const float4 wb = wlane[w * 32 + lane];       // cos B (e = 0, 1), sin B (e = 0, 1)
    const float2 wcb = make_float2(wb.x, wb.y), wsb = make_float2(wb.z, wb.w);
    // (w[n], w[n+1]) of register blocks 0 and 31: z index R (32 n1 + lane) + w
    const float2 wfirst = __ldg(win2 + R * lane + w), wlast = __ldg(win2 + R * (32 * 31 + lane) + w);

    auto fetch = [&](long long cc, long long ff) {
        const float2 *p2 = reinterpret_cast<const float2 *>(frame_at<MODE>(x, sm, x_stride, hop, cc, ff));
#pragma unroll 8
        for (int e = gtid; e < M; e += GT) {
            const int ww = e % R, i = e / R;
            cp_async8(s_tiles + ww * TILE + ww * STAG + i, p2 + e);
        }
    };
    // items [item, item_end), the first one frame f of channel c, nf frames (smoothing: items) per channel;
    // s: the group's Smoother in the smoothing outputs
    auto run = [&](long long item, long long item_end, long long c, long long f, long long nf, auto &s) {
        if (item < item_end) fetch(c, f);
        for (; item < item_end; item++) {
            cp_async_commit();
            cp_async_wait<0>();
            group_barrier(1 + grp, GT);          // the whole frame has landed
            float2 v[32];
#pragma unroll
            for (int n1 = 0; n1 < 32; n1++) v[n1] = s_x[w * STAG + 32 * n1 + lane];
            __syncwarp();                        // inputs are in registers: the tile becomes the exchange buffer
#pragma unroll
            for (int n1 = 0; n1 < 32; n1++) {
                float2 wv;
                if (n1 == 0) {
                    wv = wfirst;
                } else if (n1 == 31) {
                    wv = wlast;
                } else {
                    const float ca = hann_a.v[n1].x, sa = hann_a.v[n1].y;
                    wv = f2_fma(make_float2(-ca, -ca), wcb, make_float2(0.5f, 0.5f));
                    wv = f2_fma(make_float2(sa, sa), wsb, wv);
                }
                v[n1] = f2_mul(v[n1], wv);
            }
            dft32(v);
            twiddle_transpose<32>(v, s_tw, s_x, lane);
            dft32(v);   // v[r] = Z_w[lane + 32*brev5(r)]
#pragma unroll
            for (int r = 0; r < 32; r++) s_x[lane + 32 * brev5(r)] = v[r];   // natural order
            group_barrier(1 + grp, GT);

            float *rows = out + c * out_stride_c + f * out_stride_f;
            [[maybe_unused]] const long long myf = f;
            auto add = [&](int k, float p) {
                if constexpr (NCH > 0) s.add((int)(myf % NCH), k, p);
            };
            combine_split<R, MODE>(MODE == kModeScreen ? s_col : rows, add, s_tiles,
                                   [=](int w, int k0) { return s_comb[(w - 1) * 1024 + k0]; },
                                   [=](int kk) { return post_lookup(s_post, kk, M / 2); }, gtid, scale);
            if (++f == nf) {
                f = 0;
                c++;
            }
            group_barrier(1 + grp, GT);          // every Z_w has been read: the tiles are free again
            if (item + 1 < item_end) fetch(c, f);
            // (the group's column is written again only after the next frame's first barrier)
            if constexpr (MODE == kModeScreen) write_rows(s_col, rows, scr, gtid, GT);
            if constexpr (NCH > 0) s.after(myf);
        }
    };
    if constexpr (NCH > 0) {
        unsigned char *slot = reinterpret_cast<unsigned char *>(s_tiles_all + (size_t)LARGE_WARPS * TILE) +
                              grp * smooth_slot_bytes<MODE>(M + 1, R);
        auto s = slot_smoother<NCH>(sm, slot, M + 1, gtid, GT, [grp] { group_barrier(1 + grp, GT); });
        const long long nv = NCH * n_frames;
        for (long long ch = gg; ch < sm.n_channels; ch += groups_total) {
            s.begin(ch);
            run(ch * nv, (ch + 1) * nv, ch, 0, nv, s);
            s.end();
        }
    } else {
        const long long per = (total_items + groups_total - 1) / groups_total;
        const long long item = gg * per;
        long long item_end = item + per;
        if (item_end > total_items) item_end = total_items;
        const long long c = (item < item_end) ? item / n_frames : 0;
        int none = 0;
        run(item, item_end, c, item - c * n_frames, n_frames, none);
    }
}

// ------------------------------------------------------------------------------------------
// Generic path: one CTA per frame, Stockham autosort in shared memory.
__device__ __forceinline__ void stockham_radix4(const float2 *__restrict__ in,
                                                float2 *__restrict__ outb,
                                                const float2 *__restrict__ tw, int M, int Ns,
                                                int tid, int nthreads) {
    const int quarter = M >> 2;
    const int tw_step = M / (Ns * 4);
    for (int j = tid; j < quarter; j += nthreads) {
        const int k = j & (Ns - 1);
        float2 a0 = in[j], a1 = in[j + quarter], a2 = in[j + 2 * quarter],
               a3 = in[j + 3 * quarter];
        if (Ns > 1) {
            a1 = cmul(a1, tw[k * tw_step]);
            a2 = cmul(a2, tw[2 * k * tw_step]);
            a3 = cmul(a3, tw[3 * k * tw_step]);
        }
        const float2 s02 = cadd(a0, a2), d02 = csub(a0, a2);
        const float2 s13 = cadd(a1, a3), d13 = mul_mj(csub(a1, a3));
        const int j0 = ((j - k) << 2) + k;
        outb[j0] = cadd(s02, s13);
        outb[j0 + Ns] = cadd(d02, d13);
        outb[j0 + 2 * Ns] = csub(s02, s13);
        outb[j0 + 3 * Ns] = csub(d02, d13);
    }
}

// kModeScreen: the column goes to the buffer the FFT does not end in, and the frame's rows to out.
// Smoothing outputs: one CTA per channel, its states after the two buffers.
template <int MODE>
__global__ void stft_generic_kernel(const float *__restrict__ x, long long x_stride,
                                    long long n_frames, int hop, float *__restrict__ out,
                                    long long out_stride_c, long long out_stride_f,
                                    const float *__restrict__ win,
                                    const float2 *__restrict__ tw,
                                    const float2 *__restrict__ post, int n_fft, int log2m,
                                    const ScreenRows scr, const SmoothTicks sm) {
    extern __shared__ float2 smem[];
    constexpr int NCH = smooth_nch(MODE);
    const int M = n_fft >> 1;
    float2 *buf0 = smem;
    float2 *buf1 = smem + M;
    const int tid = threadIdx.x, nthreads = blockDim.x;
    const float scale = 1.0f / (4.0f * (float)n_fft * (float)n_fft);

    // the frame at p: `in` then holds Z[0..M) and `ob` is free
    auto transform = [&](const float *p, float2 *&in, float2 *&ob) {
        for (int n = tid; n < M; n += nthreads)
            buf0[n] = make_float2(__ldg(p + 2 * n) * __ldg(win + 2 * n),
                                  __ldg(p + 2 * n + 1) * __ldg(win + 2 * n + 1));
        __syncthreads();

        in = buf0;
        ob = buf1;
        int Ns = 1;
        if (log2m & 1) {   // one radix-2 pass first (no twiddles at Ns = 1)
            const int halfm = M >> 1;
            for (int j = tid; j < halfm; j += nthreads) {
                const float2 a = in[j], b = in[j + halfm];
                ob[2 * j] = cadd(a, b);
                ob[2 * j + 1] = csub(a, b);
            }
            __syncthreads();
            float2 *t = in; in = ob; ob = t;
            Ns = 2;
        }
        for (; Ns < M; Ns <<= 2) {
            stockham_radix4(in, ob, tw, M, Ns, tid, nthreads);
            __syncthreads();
            float2 *t = in; in = ob; ob = t;
        }
    };
    // the split step: bins k and M - k to store(k, |X|^2, |Y|^2), k <= M/2
    auto split = [&](const float2 *in, auto store) {
        for (int k = tid; k <= M / 2; k += nthreads) {
            const float2 z = in[k];
            const float2 zp = in[(M - k) & (M - 1)];
            const float2 E = make_float2(z.x + zp.x, z.y - zp.y);
            const float2 O = make_float2(z.x - zp.x, z.y + zp.y);
            const float2 T = cmul(O, post[k]);
            const float2 X = cadd(E, T);
            const float2 Y = csub(E, T);
            store(k, fmaf(X.x, X.x, X.y * X.y), fmaf(Y.x, Y.x, Y.y * Y.y));
        }
    };
    if constexpr (NCH > 0) {
        auto s = slot_smoother<NCH>(sm, smem + 2 * M, M + 1, tid, nthreads, [] { __syncthreads(); });
        const long long c = blockIdx.x;
        s.begin(c);
        for (long long i = 0; i < NCH * n_frames; i++) {
            float2 *in, *ob;
            transform(frame_at<MODE>(x, sm, x_stride, hop, c, i), in, ob);
            const int j = (int)(i % NCH);
            split(in, [&](int k, float pX, float pY) {   // bin M/2 is split twice: its second value counts
                if (k != M - k) s.add(j, k, finish<MODE>(pX, scale));
                s.add(j, M - k, finish<MODE>(pY, scale));
            });
            __syncthreads();   // `in` is read before the next frame is written
            s.after(i);
        }
        s.end();
    } else {
        const long long item = blockIdx.x;
        const long long c = item / n_frames;
        const long long f = item - c * n_frames;
        float2 *in, *ob;
        transform(x + c * x_stride + f * hop, in, ob);
        float *o = MODE == kModeScreen ? reinterpret_cast<float *>(ob) : out + c * out_stride_c + f * out_stride_f;
        split(in, [&](int k, float pX, float pY) {
            o[k] = finish<MODE>(pX, scale);
            o[M - k] = finish<MODE>(pY, scale);
        });
        if constexpr (MODE == kModeScreen) {
            __syncthreads();
            write_rows(o, out + c * out_stride_c + f * out_stride_f, scr, tid, nthreads);
        }
    }
}

// the tw table and the R tiles (+ kModeScreen: the frame's column; smoothing: the channel's states)
template <int R, int MODE>
constexpr size_t multi_smem() {
    return sizeof(float2) * (1024 + (size_t)R * TILE) + (MODE == kModeScreen ? sizeof(float) * (1024 * R + 1) : 0) +
           smooth_slot_bytes<MODE>(1024 * R + 1, R);
}
// kModeScreen and smoothing: no more CTAs per SM than its 228 KB hold (1 KB of each CTA's is reserved)
template <int R, int MODE>
constexpr long long multi_ctas_per_sm() {
    constexpr long long n = R == 8 ? 2 : (R == 4 ? 4 : 8);
    return MODE == kModeScreen || smooth_nch(MODE)
               ? std::min<long long>(n, (228 * 1024) / (multi_smem<R, MODE>() + 1024))
               : n;
}

// calls launch with the output (FRT_STFT_POWER, FRT_STFT_LOGPOWER, kModeScreen, kModeSmooth or
// kModeSmoothDual) as a compile-time constant
template <class F>
int with_mode(int mode, F &&launch) {
    if (mode == FRT_STFT_POWER) return launch(std::integral_constant<int, FRT_STFT_POWER>());
    if (mode == FRT_STFT_LOGPOWER) return launch(std::integral_constant<int, FRT_STFT_LOGPOWER>());
    if (mode == kModeSmooth) return launch(std::integral_constant<int, kModeSmooth>());
    if (mode == kModeSmoothDual) return launch(std::integral_constant<int, kModeSmoothDual>());
    return launch(std::integral_constant<int, kModeScreen>());
}

// how far every frame's first sample is aligned: 2 = 16 bytes, 1 = 8 bytes, 0 = 4 bytes
int frame_alignment(const float *x, long long x_stride, int hop) {
    if ((((uintptr_t)x & 15) == 0) && ((x_stride & 3) == 0) && ((hop & 3) == 0)) return 2;
    return (((uintptr_t)x & 7) == 0) && ((x_stride & 1) == 0) && ((hop & 1) == 0);
}

// one frt_stft_process / frt_stft_screen_rows / frt_spectrum_frames(_dual) call: total = channels x
// frames items, frame f of channel c at x + c x_stride + f hop, its spectrum (or, kModeScreen, its rows)
// at out + c osc + f osf
struct Frames {
    const float *x;
    long long x_stride, n_frames;
    int hop;
    float *out;
    long long osc, osf, total;
    int mode, align;   // align: frame_alignment of the frames
    cudaStream_t st;
    ScreenRows scr;   // kModeScreen
    SmoothTicks sm;   // smoothing
};

template <int Q, bool TMA = false>
int launch_small(frt_ctx *h, const StftPlan &pl, const Frames &a) {
    return with_mode(a.mode, [&](auto m) {
        constexpr int MODE = decltype(m)::value, G = 32 / Q, WARPS = small_warps<Q, MODE>();
        const long long max_blocks = (long long)small_ctas_per_sm<Q, MODE>() * h->sm_count;
        const long long slots = smooth_nch(MODE) ? a.sm.n_channels : (a.total + G - 1) / G;
        long long blocks = (slots + WARPS - 1) / WARPS;
        if (blocks > max_blocks) blocks = max_blocks;
        return frt_launch(h, stft_small_kernel<Q, MODE, TMA>, (unsigned)blocks, WARPS * 32, small_smem<Q, MODE, TMA>(),
                          a.st, a.x, a.x_stride, a.n_frames, a.hop, a.out, a.osc, a.osf,
                          reinterpret_cast<const float2 *>(pl.win_dev.get()), pl.tw_dev.get(), pl.post_dev.get(),
                          a.total, a.align >= 1, a.scr, a.sm);
    });
}
template <int R>
int launch_large(frt_ctx *h, const StftPlan &pl, const Frames &a) {
    HannA ha;
    const double theta = 2.0 * 3.14159265358979323846 / (double)(2048 * R - 1);
    for (int n1 = 0; n1 < 32; n1++) {
        const double a = theta * 64.0 * R * n1;
        ha.v[n1] = make_float2((float)(0.5 * cos(a)), (float)(0.5 * sin(a)));
    }
    return with_mode(a.mode, [&](auto m) {
        constexpr int MODE = decltype(m)::value, NG = large_warps<R, MODE>() / R;
        const long long slots = smooth_nch(MODE) ? a.sm.n_channels : a.total;
        long long blocks = (slots + NG - 1) / NG;
        if (blocks > h->sm_count) blocks = h->sm_count;
        return frt_launch(h, stft_large_kernel<R, MODE>, (unsigned)blocks, large_warps<R, MODE>() * 32,
                          large_smem<R, MODE>(), a.st, a.x, a.x_stride, a.n_frames, a.hop, a.out, a.osc, a.osf,
                          reinterpret_cast<const float2 *>(pl.win_dev.get()), pl.wlane_dev.get(), pl.tw_dev.get(),
                          pl.comb_dev.get(), pl.post_dev.get(), a.total, ha, a.scr, a.sm);
    });
}
template <int R>
int launch_multi(frt_ctx *h, const StftPlan &pl, const Frames &a) {
    return with_mode(a.mode, [&](auto m) {
        constexpr int MODE = decltype(m)::value;
        const long long slots = smooth_nch(MODE) ? a.sm.n_channels : a.total;
        long long blocks = (long long)h->sm_count * multi_ctas_per_sm<R, MODE>();
        if (blocks > slots) blocks = slots;
        return frt_launch(h, stft_multi_kernel<R, MODE>, (unsigned)blocks, 32 * R, multi_smem<R, MODE>(), a.st, a.x,
                          a.x_stride, a.n_frames, a.hop, a.out, a.osc, a.osf,
                          reinterpret_cast<const float2 *>(pl.win_dev.get()), pl.tw_dev.get(), pl.comb_dev.get(),
                          pl.post_dev.get(), a.total, a.align >= 1, a.scr, a.sm);
    });
}

int ilog2(int v) {
    int l = 0;
    while ((1 << l) < v) l++;
    return l;
}

// [rows][32] table of W_m^(k1 t): the twiddles between the two radix-32 passes
std::vector<float2> row_twiddles(int rows, int m) {
    const double PI = 3.14159265358979323846;
    std::vector<float2> tw((size_t)rows * 32);
    for (int k1 = 0; k1 < rows; k1++)
        for (int t = 0; t < 32; t++) {
            const double a = -2.0 * PI * (double)((k1 * t) % m) / (double)m;
            tw[k1 * 32 + t] = make_float2((float)cos(a), (float)sin(a));
        }
    return tw;
}

}   // namespace

extern "C" int frt_stft_plan(frt_handle h, int n_fft) {
    if (!h) return FRT_EINVAL;
    DeviceGuard g(h->device);
    FRT_CHECK_ARG(h, n_fft >= 32 && n_fft <= 16384 && (n_fft & (n_fft - 1)) == 0,
                  "n_fft must be a power of two in [32, 16384]");
    if (h->stft && h->stft->n_fft == n_fft) return FRT_OK;
    // plans are cached per size: the spectrum (8192) and spectrogram (4096) widgets share a handle
    auto cached = h->stft_cache.find(n_fft);
    if (cached != h->stft_cache.end()) {
        h->stft = &cached->second;
        return FRT_OK;
    }
    StftPlan pl;
    const int N = n_fft, M = N / 2;
    const double PI = 3.14159265358979323846;
    // symmetric Hann, friture/audioproc.py:76-81
    pl.win_host.resize(N);
    for (int n = 0; n < N; n++)
        pl.win_host[n] = (float)(0.5 * (1.0 - cos(2.0 * PI * n / (double)(N - 1))));
    FRT_CUDA(h, pl.win_dev.upload(pl.win_host));
    const int multi_r = (N == 4096) ? 2 : ((N == 8192) ? 4 : ((N == 16384) ? 8 : 0));
    std::vector<float2> tw;
    if (multi_r) {   // each warp's 1024-point FFT, then the radix-R combine by W_M^(w k0)
        tw = row_twiddles(32, 1024);
        std::vector<float2> comb((size_t)(multi_r - 1) * 1024);
        for (int w = 1; w < multi_r; w++)
            for (int k0 = 0; k0 < 1024; k0++) {
                const double a = -2.0 * PI * (double)(w * k0) / (double)M;
                comb[(size_t)(w - 1) * 1024 + k0] = make_float2((float)cos(a), (float)sin(a));
            }
        FRT_CUDA(h, pl.comb_dev.upload(comb));
    } else if (N >= 64) {   // stft_small_kernel: [Q][32] W_M^(k1 t), M = 32 Q
        tw = row_twiddles(M / 32, M);
    } else {                // stft_generic_kernel: [M] W_M^k
        tw.resize(M);
        for (int i = 0; i < M; i++) {
            const double a = -2.0 * PI * (double)i / (double)M;
            tw[i] = make_float2((float)cos(a), (float)sin(a));
        }
    }
    FRT_CUDA(h, pl.tw_dev.upload(tw));
    // U[k] = -j * W_N^k for every k a kernel reads: k < M/2 in stft_small_kernel, k <= M/2 in
    // stft_generic_kernel and stft_large_kernel (which derives the rest), k < M - 512 in
    // stft_multi_kernel (its largest bin with a partner is k0 + 1024 (R-1), k0 < 512)
    std::vector<float2> post(multi_r ? M - 512 : M / 2 + 1);
    for (size_t k = 0; k < post.size(); k++) {
        const double a = 2.0 * PI * (double)k / (double)N;
        post[k] = make_float2((float)(-sin(a)), (float)(-cos(a)));
    }
    FRT_CUDA(h, pl.post_dev.upload(post));
    if (N == 4096 || N == 8192) {   // stft_large_kernel: per-(warp, lane) part of the Hann phase
        const int R = N / 2048;
        std::vector<float4> wl((size_t)R * 32);
        const double theta = 2.0 * PI / (double)(N - 1);
        for (int w = 0; w < R; w++)
            for (int t = 0; t < 32; t++) {
                const double b0 = theta * (2 * R * t + 2 * w), b1 = theta * (2 * R * t + 2 * w + 1);
                wl[(size_t)w * 32 + t] = make_float4((float)cos(b0), (float)cos(b1), (float)sin(b0), (float)sin(b1));
            }
        FRT_CUDA(h, pl.wlane_dev.upload(wl));
    }
    pl.n_fft = n_fft;
    h->stft = &h->stft_cache.emplace(n_fft, std::move(pl)).first->second;
    return FRT_OK;
}

extern "C" int frt_stft_window(frt_handle h, float *window_host) {
    if (!h) return FRT_EINVAL;
    if (!h->stft) return frt_fail(h, FRT_ESTATE, "frt_stft_window: no plan");
    FRT_CHECK_ARG(h, window_host != nullptr, "window_host is NULL");
    memcpy(window_host, h->stft->win_host.data(), sizeof(float) * h->stft->n_fft);
    return FRT_OK;
}

// the kernel family for the plan's size and the frames' alignment, for every output mode
static int stft_dispatch(frt_ctx *h, const StftPlan &pl, const Frames &a) {
    const int N = pl.n_fft;
    if (N >= 64 && N <= 2048) {
        switch (N / 64) {
            case 1: return launch_small<1>(h, pl, a);
            case 2: return launch_small<2>(h, pl, a);
            case 4: return launch_small<4>(h, pl, a);
            case 8: return launch_small<8>(h, pl, a);
            case 16: return launch_small<16>(h, pl, a);
            default:   // 16-byte aligned frames: the TMA engine stages them (cp.async.bulk)
                if (a.align == 2) return launch_small<32, true>(h, pl, a);
                return launch_small<32>(h, pl, a);
        }
    }
    if ((N == 4096 || N == 8192) && a.align >= 1) {
        if (N == 4096) return launch_large<2>(h, pl, a);
        return launch_large<4>(h, pl, a);
    }
    if (N >= 4096) {
        if (N == 4096) return launch_multi<2>(h, pl, a);
        if (N == 8192) return launch_multi<4>(h, pl, a);
        return launch_multi<8>(h, pl, a);
    }
    FRT_CHECK_ARG(h, a.total <= 0x7fffffffLL, "too many frames for one launch");
    const int M = N / 2;
    int threads = M / 4;
    if (threads < 32) threads = 32;
    if (threads > 512) threads = 512;
    return with_mode(a.mode, [&](auto m) {
        constexpr int MODE = decltype(m)::value;
        const long long blocks = smooth_nch(MODE) ? a.sm.n_channels : a.total;   // smoothing: one per channel
        return frt_launch(h, stft_generic_kernel<MODE>, (unsigned)blocks, threads,
                          sizeof(float2) * 2 * M + smooth_slot_bytes<MODE>(M + 1, threads / 32), a.st, a.x,
                          a.x_stride, a.n_frames, a.hop, a.out, a.osc, a.osf, pl.win_dev.get(), pl.tw_dev.get(),
                          pl.post_dev.get(), N, ilog2(M), a.scr, a.sm);
    });
}

// What frt_stft_process and frt_stft_screen_rows (mode kModeScreen) share, in order: the plan, the shape
// and hop checks, the entry point's own check on its other scalars (bad_args: why they are refused, or
// NULL), nothing to do on empty input, the buffers (tables_ok: the entry point's own ones are set), room
// for a frame's bins or screen rows at out_stride_f, and the launch.
static int stft_call(frt_ctx *h, const char *fn, const float *x, int64_t x_stride, int n_channels,
                     int64_t n_frames, int hop, float *out, int64_t out_stride_c, int64_t out_stride_f, int mode,
                     const ScreenRows &scr, const char *bad_args, bool tables_ok, void *stream) {
    if (!h->stft) return frt_fail(h, FRT_ESTATE, "%s: call frt_stft_plan first", fn);
    const StftPlan &pl = *h->stft;
    FRT_CHECK_ARG(h, n_channels >= 0 && n_frames >= 0, "negative shape");
    FRT_CHECK_ARG(h, hop >= 1, "hop must be >= 1");
    if (bad_args) return frt_fail(h, FRT_EINVAL, "%s", bad_args);
    if (n_channels == 0 || n_frames == 0) return FRT_OK;   // empty input: nothing to do
    FRT_CHECK_ARG(h, x && out && tables_ok, "NULL buffer");
    FRT_CHECK_ARG(h, out_stride_f >= (mode == kModeScreen ? scr.height : pl.n_fft / 2 + 1),
                  "frame stride smaller than a frame's bins or screen rows");
    const Frames a{x, x_stride, n_frames, hop, out, out_stride_c, out_stride_f, (long long)n_channels * n_frames,
                   mode, frame_alignment(x, x_stride, hop), (cudaStream_t)stream, scr, SmoothTicks{}};
    return stft_dispatch(h, pl, a);
}

extern "C" int frt_stft_process(frt_handle h, const float *x_dev, int64_t x_stride,
                                int n_channels, int64_t n_frames, int hop, float *out_dev,
                                int64_t out_stride_c, int64_t out_stride_f, int mode,
                                void *stream) {
    if (!h) return FRT_EINVAL;
    DeviceGuard g(h->device);
    const bool known = mode == FRT_STFT_POWER || mode == FRT_STFT_LOGPOWER;
    return stft_call(h, "frt_stft_process", x_dev, x_stride, n_channels, n_frames, hop, out_dev, out_stride_c,
                     out_stride_f, mode, ScreenRows{}, known ? nullptr : "unknown mode", true, stream);
}

extern "C" int frt_stft_screen_rows(frt_handle h, const float *x_dev, int64_t x_stride, int n_channels,
                                    int64_t n_frames, int hop, const float *weight_dev, float spec_min,
                                    float spec_max, const int *row_i0_dev, const float *row_t_dev, int height,
                                    float *rows_dev, int64_t rows_stride_c, int64_t rows_stride_f,
                                    void *stream) {
    if (!h) return FRT_EINVAL;
    DeviceGuard g(h->device);
    const char *bad = height < 1 ? "height must be >= 1" : (spec_max == spec_min ? "empty dB range" : nullptr);
    const ScreenRows scr{weight_dev, row_i0_dev, row_t_dev, spec_min, 1.0f / (spec_max - spec_min), height};
    return stft_call(h, "frt_stft_screen_rows", x_dev, x_stride, n_channels, n_frames, hop, rows_dev, rows_stride_c,
                     rows_stride_f, kModeScreen, scr, bad, row_i0_dev && row_t_dev, stream);
}

// frt_spectrum_frames and _dual (mode kModeSmooth / kModeSmoothDual; x2 and disp2 NULL in kModeSmooth): the
// checks, nothing to do on empty input, and the launch of the plan's kernel family.
static int spectrum_frames_call(frt_ctx *h, const char *fn, int mode, const float *x, const float *x2,
                                int64_t x_stride, int n_channels, int64_t n_frames, int hop, const int *tick_end,
                                int n_ticks, float alpha, float *disp, float *disp2, const float *weight, float *db,
                                int64_t db_stride_c, int64_t db_stride_r, int *imax, int *ipitch, void *stream) {
    if (!h->stft) return frt_fail(h, FRT_ESTATE, "%s: call frt_stft_plan first", fn);
    const int nbins = h->stft->n_fft / 2 + 1;
    const bool dual = mode == kModeSmoothDual;
    FRT_CHECK_ARG(h, n_channels >= 0 && n_frames >= 0, "negative shape");
    FRT_CHECK_ARG(h, hop >= 1, "hop must be >= 1");
    FRT_CHECK_ARG(h, alpha > 0.f && alpha <= 1.f, "alpha must be in (0, 1]");
    FRT_CHECK_ARG(h, n_ticks >= 0 && n_ticks <= n_frames && (n_ticks > 0 || n_frames == 0),
                  "n_ticks must be in 1..n_frames");
    if (n_channels == 0 || n_frames == 0) return FRT_OK;   // empty input: nothing to do
    FRT_CHECK_ARG(h, x && tick_end && disp && imax && ipitch && (!dual || (x2 && disp2)), "NULL buffer");
    FRT_CHECK_ARG(h, !db || (db_stride_r >= nbins && db_stride_c >= 0), "dB row stride smaller than a row's bins");
    const SmoothTicks sm{x2,     tick_end, n_ticks, n_channels,  alpha,       {disp, disp2},
                         weight, db,       db_stride_c, db_stride_r, imax,  ipitch};
    int align = frame_alignment(x, x_stride, hop);
    if (dual) align = std::min(align, frame_alignment(x2, x_stride, hop));
    const Frames a{x,    x_stride, n_frames, hop, nullptr, 0, 0, (long long)n_channels * n_frames,
                   mode, align,    (cudaStream_t)stream,   ScreenRows{}, sm};
    return stft_dispatch(h, *h->stft, a);
}

extern "C" int frt_spectrum_frames(frt_handle h, const float *x_dev, int64_t x_stride, int n_channels,
                                   int64_t n_frames, int hop, const int *tick_end_dev, int n_ticks, float alpha,
                                   float *disp_dev, const float *weight_dev, float *db_dev, int64_t db_stride_c,
                                   int64_t db_stride_r, int *imax_dev, int *ipitch_dev, void *stream) {
    if (!h) return FRT_EINVAL;
    DeviceGuard g(h->device);
    return spectrum_frames_call(h, "frt_spectrum_frames", kModeSmooth, x_dev, nullptr, x_stride, n_channels, n_frames,
                                hop, tick_end_dev, n_ticks, alpha, disp_dev, nullptr, weight_dev, db_dev, db_stride_c,
                                db_stride_r, imax_dev, ipitch_dev, stream);
}

extern "C" int frt_spectrum_frames_dual(frt_handle h, const float *x1_dev, const float *x2_dev, int64_t x_stride,
                                        int n_pairs, int64_t n_frames, int hop, const int *tick_end_dev, int n_ticks,
                                        float alpha, float *disp1_dev, float *disp2_dev, float *db_dev,
                                        int64_t db_stride_c, int64_t db_stride_r, int *imax_dev, int *ipitch_dev,
                                        void *stream) {
    if (!h) return FRT_EINVAL;
    DeviceGuard g(h->device);
    return spectrum_frames_call(h, "frt_spectrum_frames_dual", kModeSmoothDual, x1_dev, x2_dev, x_stride, n_pairs,
                                n_frames, hop, tick_end_dev, n_ticks, alpha, disp1_dev, disp2_dev, nullptr, db_dev,
                                db_stride_c, db_stride_r, imax_dev, ipitch_dev, stream);
}

extern "C" int frt_stft_process_host(frt_handle h, const float *x_host, int64_t x_stride,
                                     int n_channels, int64_t n_samples, int hop,
                                     float *out_host, int mode) {
    if (!h) return FRT_EINVAL;
    DeviceGuard g(h->device);
    if (!h->stft) return frt_fail(h, FRT_ESTATE, "frt_stft_process_host: no plan");
    const StftPlan &pl = *h->stft;
    FRT_CHECK_ARG(h, n_channels >= 0 && n_samples >= 0 && hop >= 1, "bad shape");
    const int N = pl.n_fft, nbins = N / 2 + 1;
    if (n_channels == 0 || n_samples < N) return FRT_OK;
    FRT_CHECK_ARG(h, x_host != nullptr && out_host != nullptr, "NULL buffer");
    FRT_CHECK_ARG(h, x_stride >= n_samples, "x_stride smaller than n_samples");
    const int64_t frames = (n_samples - N) / hop + 1;
    // chunk = (channel group) x (frame range), sized to ~32 MiB of output per buffer
    const size_t budget = (size_t)32 << 20, out_per_frame = sizeof(float) * nbins;
    const int64_t fchunk = (int64_t)frt_group_size(budget, out_per_frame, frames);
    const int cgroup = fchunk == frames ? (int)frt_group_size(budget, frames * out_per_frame, n_channels) : 1;
    const int64_t chunk_samples = (fchunk - 1) * (int64_t)hop + N;
    StftStaging &p = h->stft_host;
    FRT_CUDA(h, p.create());
    for (auto &d : p.d_in) FRT_CUDA(h, d.grow((size_t)cgroup * chunk_samples));
    for (auto &d : p.d_out) FRT_CUDA(h, d.grow((size_t)cgroup * fchunk * nbins));
    const cudaStream_t s_in = p.s_in.get(), s_cmp = p.s_cmp.get(), s_out = p.s_out.get();
    int rc;
    int it = 0;
    for (int c0 = 0; c0 < n_channels; c0 += cgroup) {
        const int nc = (c0 + cgroup <= n_channels) ? cgroup : (n_channels - c0);
        for (int64_t f0 = 0; f0 < frames; f0 += fchunk, it++) {
            const int64_t nf = (f0 + fchunk <= frames) ? fchunk : (frames - f0);
            const int64_t ns = (nf - 1) * (int64_t)hop + N;
            const int b = it & 1;
            // the H2D may only overwrite d_in[b] after the kernel that read it has finished
            FRT_CUDA(h, cudaStreamWaitEvent(s_in, p.ev_cmp[b].get(), 0));
            FRT_CUDA(h, cudaMemcpy2DAsync(p.d_in[b].get(), sizeof(float) * ns,
                                          x_host + (size_t)c0 * x_stride + f0 * hop,
                                          sizeof(float) * x_stride, sizeof(float) * ns, nc,
                                          cudaMemcpyHostToDevice, s_in));
            FRT_CUDA(h, cudaEventRecord(p.ev_in[b].get(), s_in));
            FRT_CUDA(h, cudaStreamWaitEvent(s_cmp, p.ev_in[b].get(), 0));
            FRT_CUDA(h, cudaStreamWaitEvent(s_cmp, p.ev_out[b].get(), 0));   // d_out[b] drained
            rc = frt_stft_process(h, p.d_in[b].get(), ns, nc, nf, hop, p.d_out[b].get(),
                                  nf * (int64_t)nbins, nbins, mode, s_cmp);
            if (rc) return rc;
            FRT_CUDA(h, cudaEventRecord(p.ev_cmp[b].get(), s_cmp));
            FRT_CUDA(h, cudaStreamWaitEvent(s_out, p.ev_cmp[b].get(), 0));
            FRT_CUDA(h, cudaMemcpy2DAsync(out_host + ((size_t)c0 * frames + f0) * nbins,
                                          sizeof(float) * frames * nbins, p.d_out[b].get(),
                                          sizeof(float) * nf * nbins,
                                          sizeof(float) * nf * nbins, nc,
                                          cudaMemcpyDeviceToHost, s_out));
            FRT_CUDA(h, cudaEventRecord(p.ev_out[b].get(), s_out));
        }
    }
    FRT_CUDA(h, cudaStreamSynchronize(s_out));
    FRT_CUDA(h, cudaStreamSynchronize(s_cmp));
    FRT_CUDA(h, cudaStreamSynchronize(s_in));
    return FRT_OK;
}
