// Lane-pipelined multi-rate IIR filterbank + exponential RMS for sm_90a (bpo = 1 or 3).
//
// Same numerics contract as bank.cu (the reference's IIR bank octave_filter_bank_decimation,
// friture/filter.py:86-118, recursion friture/signal/lfilter.py:131-139, [::2] of
// friture/signal/decimate.py:39-41, fused with exp_smoothed_value(y**2),
// friture/octavespectrum.py:104 / friture/signal/exp_smoothing.py:11-56), different schedule:
//
// A recursion is serial in time, so instead of splitting time (bank.cu: two passes + a scan per
// section) the SECTIONS are spread over lanes and every lane runs its sections serially over a chunk
// of CH samples per step, handing the chunk to the next lane of its chain through a shared-memory
// ring: the chain is a software pipeline, a lane works on the chunk its predecessor finished one
// step earlier.  Each sample of each section is computed exactly once, with the 4-operation
// normalised biquad (bank_internal.cuh).
//
// One HALF-WARP per channel (per channel pair when two channels are packed in float2: two
// independent recurrences per lane),
// NR = bpo + 3 roles per lane group, TWO CHAINED SECTIONS PER LANE (their recurrences are
// independent, which gives the in-order issue two chains to interleave):
//   role r < bpo      band r: both band-pass sections, reads the stage input
//   role bpo + d      decimator sections 2d, 2d+1 (d = 0, 1, 2); d = 0 reads the stage input
//   lanes [0, NR)     group 0: stage 0 (rate fs)
//   lanes [NR, 2 NR)  group 1: the same roles for ALL lower-rate stages, time-multiplexed: of the
//                     CH sample slots of a step, slots [CH-2 len_j, CH-len_j) belong to stage j
//                     (len_j = CH >> j) and the last slot to the one stage >= JR = log2(CH)+1 whose
//                     turn it is (stage JR + ctz(u+1): a binary-ruler schedule, every stage gets
//                     exactly its 2^-j share) -- 31/32 of these lanes' slots carry work.
//   The last decimator lane keeps the even samples (x chain gain) and writes them where the next
//   stage's chain heads read them one step later (slot i -> CH/2 + i/2 of the multiplexed input
//   vector; the single samples of the ruler stages wait in a double-buffered per-stage mailbox).
//   Smoothing of y^2 is NOT done in the section loops: after each step the 16 lanes of the
//   half-warp update one accumulator per sample slot (acc <- q^len acc + y^2, a few instructions
//   per band per step instead of two per sample); at a block end the accumulators of a stage are
//   combined with a weighted warp reduction into the band energy and collapsed back to one value, so
//   the state carried between launches is the plain smoothed energy and a stream gives the same
//   bits whether it arrives in one launch or block by block.  Decays are applied in complement
//   form (acc - (1-q^n) acc): the float32 rounding of q must not bias long time constants.
//
// tests/bank_pipeline_model.py is an executable NumPy model of exactly this schedule, checked
// against the CPU restatement of the reference; this file mirrors it phase by phase.
#include <cmath>
#include <cstdlib>
#include <type_traits>

#include "bank_internal.cuh"

namespace {

// One section per lane (a warp per channel, half the arithmetic per lane and step) was measured and
// is not faster: the step time of a warp is set by latencies spread over the whole step
// (shared-memory round trips at the segment switches, the single dependent chain of a lane,
// branches), not by the count of section samples per lane.
constexpr int HW = 16;              // lanes per channel slot
constexpr int NSLOT = 32 / HW;      // channel slots per warp
constexpr int DEC_DEPTH = 3;        // decimator chain depth in lanes = steps a stage trails its parent
constexpr int RS = 4;               // state values per role: z1A z2A z1B z2B

template <int PACK> struct VT;
template <> struct VT<1> { using t = float; };
template <> struct VT<2> { using t = float2; };

__device__ __forceinline__ float v_add(float a, float b) { return a + b; }
__device__ __forceinline__ float2 v_add(float2 a, float2 b) { return f2_add(a, b); }
__device__ __forceinline__ float v_fma(float c, float x, float z) { return fmaf(c, x, z); }
__device__ __forceinline__ float2 v_fma(float c, float2 x, float2 z) {
    return f2_fma(make_float2(c, c), x, z);
}
__device__ __forceinline__ float v_mul(float c, float x) { return c * x; }
__device__ __forceinline__ float2 v_mul(float c, float2 x) { return f2_mul(make_float2(c, c), x); }
__device__ __forceinline__ float v_sq(float a) { return a * a; }
__device__ __forceinline__ float2 v_sq(float2 a) { return f2_mul(a, a); }
__device__ __forceinline__ void v_set(float &d, float a, float) { d = a; }
__device__ __forceinline__ void v_set(float2 &d, float a, float b) { d = make_float2(a, b); }
__device__ __forceinline__ float v_x(float a) { return a; }
__device__ __forceinline__ float v_x(float2 a) { return a.x; }
__device__ __forceinline__ float v_y(float a) { return a; }
__device__ __forceinline__ float v_y(float2 a) { return a.y; }
__device__ __forceinline__ float v_sel(bool p, float a, float b) { return p ? a : b; }
__device__ __forceinline__ float2 v_sel(bool p, float2 a, float2 b) {
    return make_float2(p ? a.x : b.x, p ? a.y : b.y);
}
__device__ __forceinline__ float v_shfl_xor(float a, int d) { return __shfl_xor_sync(0xffffffffu, a, d); }
__device__ __forceinline__ float2 v_shfl_xor(float2 a, int d) {
    return make_float2(__shfl_xor_sync(0xffffffffu, a.x, d), __shfl_xor_sync(0xffffffffu, a.y, d));
}

__device__ __forceinline__ void ld4(const float *p, float (&v)[4]) {
    const float4 t = *reinterpret_cast<const float4 *>(p);
    v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
}
__device__ __forceinline__ void ld4(const float2 *p, float2 (&v)[4]) {
    const float4 a = reinterpret_cast<const float4 *>(p)[0];
    const float4 b = reinterpret_cast<const float4 *>(p)[1];
    v[0] = make_float2(a.x, a.y); v[1] = make_float2(a.z, a.w);
    v[2] = make_float2(b.x, b.y); v[3] = make_float2(b.z, b.w);
}
__device__ __forceinline__ void st4(float *p, const float (&v)[4]) {
    *reinterpret_cast<float4 *>(p) = make_float4(v[0], v[1], v[2], v[3]);
}
__device__ __forceinline__ void st4(float2 *p, const float2 (&v)[4]) {
    reinterpret_cast<float4 *>(p)[0] = make_float4(v[0].x, v[0].y, v[1].x, v[1].y);
    reinterpret_cast<float4 *>(p)[1] = make_float4(v[2].x, v[2].y, v[3].x, v[3].y);
}
__device__ __forceinline__ void st2(float *p, float a, float b) {
    *reinterpret_cast<float2 *>(p) = make_float2(a, b);
}
__device__ __forceinline__ void st2(float2 *p, float2 a, float2 b) {
    *reinterpret_cast<float4 *>(p) = make_float4(a.x, a.y, b.x, b.y);
}

// blocks of band energies staged in shared memory before the flush: a block's vector leaves fdelta
// steps after its last stage-0 chunk, meanwhile stage 0 keeps staging newer blocks
// (frt_pipe_prepare checks that the ring is deep enough for the blocks bank_route gives the kernel)
constexpr int EN_RING = 8;

// The two lane groups of a half-warp must run ONE instruction stream with per-lane predicates.
// Conditions on the (loop-invariant) group index invite the compiler to unswitch the whole
// section loop into two divergent copies, which doubles the issue slots; passing the flag through
// an empty asm makes every use a fresh value.
__device__ __forceinline__ bool opq(bool p) {
    int v = p ? 1 : 0;
    asm volatile("" : "+r"(v));
    return v != 0;
}

// normalised biquad step (bank_internal.cuh): y = x + z1; z1 = c x - a1 y + z2; z2 = x - a2 y.
// The state-space form with y substituted shortens the loop-carried path (z1 -> z1' is one FFMA) at
// the price of a fifth operation; it was measured and is not faster, the step is not bound by this
// chain alone.
template <class T>
__device__ __forceinline__ T biquad(T x, T &z1, T &z2, float b1, float na1, float na2) {
    const T y = v_add(x, z1);
    const T t = v_fma(b1 - na1, x, z2);      // c = b1 + a1
    z1 = v_fma(na1, y, t);
    z2 = v_fma(na2, y, x);
    return y;
}

// Sample slots of a step are grouped in segments (= stages of the multiplexed lanes): segment
// g < LOGCH holds the CH >> (g+1) slots starting at CH - 2 (CH >> (g+1)), segment LOGCH is the
// ruler slot CH-1.  A segment starts at slot s >= CH/2 whenever CH - s is a power of two, and is
// then segment LOGCH - log2(CH - s).
__host__ __device__ constexpr int ilog2c(int v) {
    return v >= 128 ? 7 : v >= 64 ? 6 : v >= 32 ? 5 : v >= 16 ? 4 : v >= 8 ? 3 : v >= 4 ? 2 : v >= 2 ? 1 : 0;
}
__host__ __device__ constexpr bool seg_starts_at(int slot, int ch) {
    return slot >= ch / 2 && ((ch - slot) & (ch - slot - 1)) == 0;
}

// Shared memory of one channel slot (half-warp), in units of T.  128-bit accesses are served a
// quarter-warp (8 lanes x 16 B) at a time, so the 8 lanes of a quarter must hit 8 different 16-byte
// bank groups: every writer lane hl owns a region whose base is 16*hl (mod 128) bytes, the stage
// input vectors sit in groups 5 (stage 0) and 6 (multiplexed stages), and the second half-warp's
// slot is displaced by 64 (mod 128) bytes so that the 32-bit accesses of the two halves use
// different banks.
// resident one-warp CTAs per SM the register allocation must allow (65536 / (32 * n) registers per
// thread): the small-step variant serves many channels and wants warps, the large-step variants
// serve few channels (one warp per scheduler at best) and want registers
__host__ __device__ constexpr int pipe_min_blocks(int logch, int pack) {
    return (logch == 5 && pack == 1) ? 16 : (logch == 6 && pack == 1) ? 12 : 8;
}

template <int LOGCH, int PACK, int BPO>
struct PipeLayout {
    static constexpr int CH = 1 << LOGCH;
    static constexpr int NR = BPO + 3;
    static constexpr int NWR = 12;                            // writer lanes: two groups of NR <= 6
    static constexpr int WPAD = 4;                            // 16-byte pads after the writer regions
    static constexpr int TB = 4 * PACK;                       // bytes per T
    static constexpr int PAD = 16 / TB;                       // 16 bytes
    static constexpr int XSLOT = 2 * CH + 8 * PAD;            // ring slot: 128 B of skew + 2 vectors
    static constexpr int X0 = 5 * PAD;                        // stage-0 chunk within a slot (group 5)
    static constexpr int XM = X0 + CH + PAD;                  // multiplexed vector (group 6)
    static constexpr int X = 0;                               // [RX][XSLOT]
    static constexpr int W = X + PIPE_RX * XSLOT;             // [NWR writer lanes][2 bufs][CH] + 16 B each
    static constexpr int WSTR = 2 * CH + PAD;
    static constexpr int S = W + NWR * WSTR + WPAD * PAD;     // [MAX_OCT][NR][RS]: z1A z2A z1B z2B
    static constexpr int ER = S + BANK_MAX_OCT * NR * RS;     // [MAX_OCT][4]: ruler-stage energies
    static constexpr int MB = ER + BANK_MAX_OCT * 4;          // [MAX_OCT + 2][2] mailboxes
    static constexpr int EN = MB + (BANK_MAX_OCT + 2) * 2;    // [EN_RING][32] staged band energies
    static constexpr int RAW = EN + EN_RING * 32;
    // round up to 64 (mod 128) bytes
    static constexpr int RAWB = RAW * TB;
    static constexpr int TOTALB = ((RAWB + 63) / 128) * 128 + 64;
    static constexpr int TOTAL = TOTALB / TB;
    static_assert((NWR * WSTR + WPAD * PAD) % (8 * PAD) == 0, "state rows start on a 128-byte boundary");
};

template <int LOGCH, int PACK, int BPO>
__global__ void __launch_bounds__(32, pipe_min_blocks(LOGCH, PACK))
bank_pipe_kernel(const __grid_constant__ PipeParams P, const BankArgs a) {
    using T = typename VT<PACK>::t;
    using LY = PipeLayout<LOGCH, PACK, BPO>;
    constexpr int CH = 1 << LOGCH, JR = LOGCH + 1, NR = LY::NR, NSEC = 2 * NR;
    constexpr int NSL = CH / HW;              // sample slots per lane of the channel slot (phase B)
    constexpr int NG = CH / 4;                // 4-sample groups per step
    constexpr int GB = (PACK == 1 ? 32 : 16) / 4;   // groups whose inputs are loaded ahead
    constexpr int RX = PIPE_RX, PF = PIPE_PF;
    static_assert(2 * NR <= HW, "two lane groups must fit in a channel slot");
    static_assert(LOGCH == 5 || LOGCH == 6, "steps of 32 or 64 samples");
    static_assert(NG % GB == 0, "whole load batches");

    extern __shared__ __align__(128) float4 smem4[];
    const int lane = threadIdx.x;
    const int h = lane / HW, hl = lane & (HW - 1);
    T *sm = reinterpret_cast<T *>(smem4) + h * LY::TOTAL;       // this channel slot
    int *sT = reinterpret_cast<int *>(reinterpret_cast<T *>(smem4) + NSLOT * LY::TOTAL);   // [MAX_OCT + 2]
    float *sAl = reinterpret_cast<float *>(sT + 12);            // [MAX_OCT + 2]
    T *sX = sm + LY::X, *sW = sm + LY::W, *sS = sm + LY::S, *sER = sm + LY::ER, *sMB = sm + LY::MB,
      *sEN = sm + LY::EN;

    // channels of this half-warp (clamped when the last warp is not full; `alive` gates the writes)
    const int cgrp = blockIdx.x * NSLOT + h;
    const bool alive = cgrp * PACK < a.n_channels;
    const int ch0 = alive ? cgrp * PACK : 0;
    const bool has2 = (PACK == 2) && alive && (ch0 + 1 < a.n_channels);
    const int ch1 = has2 ? ch0 + 1 : ch0;
    const int n_oct = P.n_oct;
    const int nbands = n_oct * BPO;
    const int n_chunks = (int)(a.t_total >> LOGCH);
    const int lognb = 31 - __clz(a.block) - LOGCH;          // block = CH << lognb
    const int nbmask = (1 << lognb) - 1;
    const int logblock = lognb + LOGCH;
    const bool want_e = alive && a.energies != nullptr;
    float *eout0 = a.energies ? a.energies + (size_t)ch0 * a.e_stride : nullptr;
    const int fdelta = P.fdelta;
    // dB weighting of the bands this lane emits at a flush, loaded once instead of at every flush
    constexpr int NWT = (BANK_MAX_OCT * BPO + HW - 1) / HW;
    float wreg[NWT];
#pragma unroll
    for (int t = 0; t < NWT; t++) {
        const int i = hl + HW * t;
        wreg[t] = (a.db && a.weight && i < nbands) ? __ldg(a.weight + i) : 0.f;
    }

    // ---- lane roles (phase A)
    const bool worker = hl < 2 * NR;
    const int G = (worker && hl >= NR) ? 1 : 0;
    const int r = worker ? hl - G * NR : 0;
    const bool isband = r < BPO;                             // role r < BPO: band r
    // skew = position in the lane chain (bands: one lane; decimator: DEC_DEPTH lanes)
    const int d = isband ? 0 : r - BPO;
    const bool isdec2 = worker && (r == NR - 1);
    const bool ishead = (d == 0);                            // reads the stage input
    const int maxstage = isband ? n_oct - 1 : n_oct - 2;     // the last stage's decimator is unused (filter.py:113)
    const float b1A = P.b1[2 * r], n1A = P.na1[2 * r], n2A = P.na2[2 * r];
    const float b1B = P.b1[2 * r + 1], n1B = P.na1[2 * r + 1], n2B = P.na2[2 * r + 1];
    const float gb_lane = isband ? P.gband[r] : 0.f;
    const float gdec = P.gdec;

    // ---- prologue: tables, state
    if (lane <= BANK_MAX_OCT + 1) {
        sT[lane] = lane <= BANK_MAX_OCT ? P.T[lane] : 0x3fffffff;
        sAl[lane] = lane <= BANK_MAX_OCT ? P.alpha[lane] : 1.f;
    }
    float *gz0 = a.zstate + (size_t)ch0 * n_oct * NSEC * 2;
    float *gz1 = a.zstate + (size_t)ch1 * n_oct * NSEC * 2;
    float *ge0 = a.ema + (size_t)ch0 * nbands;
    float *ge1 = a.ema + (size_t)ch1 * nbands;
    for (int i = hl; i < BANK_MAX_OCT * NSEC * 2; i += HW) {    // sS[j][r][RS] == global z[j][2 r ..][2]
        T z;
        v_set(z, 0.f, 0.f);
        if (i < n_oct * NSEC * 2) v_set(z, gz0[i], gz1[i]);
        sS[i] = z;
    }
    for (int i = hl; i < BANK_MAX_OCT * 4; i += HW) {
        const int j = i >> 2, b = i & 3;
        T e;
        v_set(e, 0.f, 0.f);
        if (j >= JR && j < n_oct && b < BPO) v_set(e, ge0[j * BPO + b], ge1[j * BPO + b]);
        sER[i] = e;
    }
    // smoothing accumulators: one per sample slot (slot = hl + HW q) of the two band-output vectors
    T acc0[BPO][NSL], accm[BPO][NSL];
    int mst[NSL];
    bool mok[NSL], lastslot[NSL];
    float om0[NSL], aqm[NSL], omm[NSL];
#pragma unroll
    for (int q = 0; q < NSL; q++) {
        const int p = hl + HW * q;
        const int j = 1 + __clz(~((unsigned)p << (32 - LOGCH)));     // stage owning slot p
        mst[q] = j;
        mok[q] = (j < JR) && (j <= n_oct - 1);
        lastslot[q] = (p == CH - (CH >> j) - 1);
        om0[q] = P.om0[p >> 5][p & 31];
        aqm[q] = P.aqm[p >> 5][p & 31];
        omm[q] = P.omm[p >> 5][p & 31];
#pragma unroll
        for (int b = 0; b < BPO; b++) {
            v_set(acc0[b][q], 0.f, 0.f);
            v_set(accm[b][q], 0.f, 0.f);
            if (p == CH - 1) v_set(acc0[b][q], ge0[b], ge1[b]);
            if (mok[q] && lastslot[q]) v_set(accm[b][q], ge0[j * BPO + b], ge1[j * BPO + b]);
        }
    }
    const float *x0 = a.x + (size_t)ch0 * a.x_stride;
    const float *x1 = a.x + (size_t)ch1 * a.x_stride;
    const bool vec16 = (PACK == 1) && a.vec_ok;
    auto prefetch = [&](int cn) {
        if (cn < n_chunks) {
            T *dst = sX + (cn & (RX - 1)) * LY::XSLOT + LY::X0;
            if (vec16) {
                if (hl < CH / 4) cp_async16(dst + 4 * hl, x0 + (size_t)cn * CH + 4 * hl);
            } else {
#pragma unroll
                for (int q = 0; q < NSL; q++) {
                    const int p = hl + HW * q;
                    float *dd = reinterpret_cast<float *>(dst + p);
                    cp_async4(dd, x0 + (size_t)cn * CH + p);
                    if (PACK == 2) cp_async4(dd + 1, x1 + (size_t)cn * CH + p);
                }
            }
        }
        cp_async_commit();
    };
#pragma unroll
    for (int cn = 0; cn < PF; cn++) prefetch(cn);
    cp_async_wait<PF - 1>();
    __syncwarp();

    // stage-0 lanes carry their section state in registers from step to step
    T zc[RS];
#pragma unroll
    for (int i = 0; i < RS; i++) zc[i] = sS[r * RS + i];
    const int n_steps = a.n_steps;
    // steps in [k_lo, k_hi) have every slot of every lane valid (pipeline full, nothing drained):
    // they run the variant without the range checks
    const int k_lo = P.T[n_oct - 1] + DEC_DEPTH;
    const int k_hi = (n_oct > JR) ? n_chunks : 0;

    // ================================================================ phase A: the section loops
    // The smoothing accumulators of step k-1 (phase B's bulk) are updated INSIDE the section loops of
    // step k: the section recurrences leave most issue slots of the warp empty, the independent
    // accumulator updates fill them.  They read the band outputs of step k-1 (buffer (k-1)&1), which
    // this step only reads as well.
    auto phaseA = [&](int k, auto check_tag) {
        constexpr bool CHECK = decltype(check_tag)::value;
        const int kp = k - 1;                      // step kp wrote the band outputs of stage-0 chunk kp
        const bool bv0 = !CHECK || (kp >= 0 && (unsigned)kp < (unsigned)n_chunks);
        bool bvm[NSL];
#pragma unroll
        for (int q = 0; q < NSL; q++) {
            bvm[q] = mok[q];
            if (CHECK) bvm[q] = bvm[q] && kp >= 0 && (unsigned)(kp - DEC_DEPTH * mst[q]) < (unsigned)n_chunks;
        }
        const T *ybuf = sW + (kp & 1) * CH;
        constexpr int NUPD = 2 * BPO * NSL;        // accumulator updates per step
        auto bupd = [&](int i) {                   // i is a compile-time constant after unrolling
            const int which = i & 1, q = (i >> 1) % NSL, b = (i >> 1) / NSL;
            const int p = hl + HW * q;
            // raw units of the normalised sections; the squared chain gain is applied on emission.
            // Band b's output is lane b's region (group 0) or lane NR + b's (group 1).
            if (which == 0) {
                const T yv = ybuf[b * LY::WSTR + p];
                if (bv0) acc0[b][q] = v_add(v_fma(-P.aq0, acc0[b][q], acc0[b][q]), v_sq(yv));
            } else {
                const T yv = ybuf[(NR + b) * LY::WSTR + p];
                if (bvm[q]) accm[b][q] = v_add(v_fma(-aqm[q], accm[b][q], accm[b][q]), v_sq(yv));
            }
        };
        const int u = k - d;
        // heads read the stage input vector, the other decimator lanes the buffer their predecessor
        // (lane hl-1) filled one step earlier; every lane writes its own region (buffer k&1)
        const T *inp = ishead ? sX + (k & (RX - 1)) * LY::XSLOT + (G ? LY::XM : LY::X0)
                              : sW + (hl - 1) * LY::WSTR + ((k - 1) & 1) * CH;
        // lanes beyond the two groups are exact clones of lane 0 (same role, same state, same
        // addresses): they run the section loops only to take part in the accumulator updates, and
        // store the same values to the same places, so no store needs a branch
        T *outp = sW + (worker ? hl : 0) * LY::WSTR + (k & 1) * CH;
        T *xn = sX + ((k + 1) & (RX - 1)) * LY::XSLOT + LY::XM + G * (CH / 2);
        const bool pv0 = !CHECK || ((unsigned)u < (unsigned)n_chunks && 0 <= maxstage);
        // ruler slot: the stage >= JR whose sample is due (group 1 only)
        const int jr = JR - 1 + __ffs(u + 1);
        const int jrc = jr < BANK_MAX_OCT - 1 ? jr : BANK_MAX_OCT - 1;
        const int Tj = sT[jrc];
        const int m = (u - Tj) >> (jrc - LOGCH);
        bool pvR = jr <= maxstage;
        if (CHECK) pvR = pvR && u >= Tj && m < (int)(a.t_total >> jrc);

        // section state: group 0 keeps it in registers (zc) for the whole step; group 1 switches
        // rows of sS at every segment start, the next row is fetched one segment ahead.  Loads are
        // unconditional (group 0 reads rows it never uses), selection is by per-lane predicate.
        const bool g1 = opq(G != 0);
        T cur[RS], nxt[RS];
        T *spc = sS + (1 * NR + r) * RS;       // state row of the segment being processed (group 1)
#pragma unroll
        for (int i = 0; i < RS; i++) cur[i] = v_sel(g1, spc[i], zc[i]);
#pragma unroll
        for (int i = 0; i < RS; i++) nxt[i] = sS[(2 * NR + r) * RS + i];
        bool pvc = !CHECK || ((unsigned)(u - DEC_DEPTH) < (unsigned)n_chunks && 1 <= maxstage);
        bool pvB = false;           // validity / chunk index of the 1-sample stage LOGCH (for the mailbox)
        int cidxB = 0;
#pragma unroll
        for (int b0 = 0; b0 < NG; b0 += GB) {
            T v[GB][4];
#pragma unroll
            for (int q = 0; q < GB; q++) ld4(inp + 4 * (b0 + q), v[q]);
            if (b0 + GB == NG) {
                // the ruler stage's sample comes from its mailbox, not from the ring
                const T mb = sMB[jrc * 2 + (m & 1)];
                v[GB - 1][3] = v_sel(opq(G != 0 && ishead), mb, v[GB - 1][3]);
            }
#pragma unroll
            for (int q = 0; q < GB; q++) {
                T y[4];
#pragma unroll
                for (int i = 0; i < 4; i++) {
                    const int slot = 4 * (b0 + q) + i;
                    if (seg_starts_at(slot, CH)) {
                        // group 1 switches to the state of the next stage; group 0 keeps its registers
                        const int g = LOGCH - ilog2c(CH - slot);
                        const bool gs = opq(G != 0);
                        if (gs && pvc) {
#pragma unroll
                            for (int e = 0; e < RS; e++) spc[e] = cur[e];
                        }
#pragma unroll
                        for (int e = 0; e < RS; e++) cur[e] = v_sel(gs, nxt[e], cur[e]);
                        spc = (g < LOGCH) ? sS + ((g + 1) * NR + r) * RS : sS + (jrc * NR + r) * RS;
                        if (g < LOGCH) {
                            const T *spn = (g + 1 < LOGCH) ? sS + ((g + 2) * NR + r) * RS
                                                           : sS + (jrc * NR + r) * RS;
#pragma unroll
                            for (int e = 0; e < RS; e++) nxt[e] = spn[e];
                            pvc = !CHECK || ((unsigned)(u - DEC_DEPTH * (g + 1)) < (unsigned)n_chunks &&
                                             (g + 1) <= maxstage);
                            if (g == LOGCH - 1) {
                                pvB = pvc;
                                cidxB = u - DEC_DEPTH * (g + 1);
                            }
                        } else {
                            pvc = pvR;
                        }
                    }
                    const T ya = biquad(v[q][i], cur[0], cur[1], b1A, n1A, n2A);
                    y[i] = biquad(ya, cur[2], cur[3], b1B, n1B, n2B);
                }
                const int gq = b0 + q;
#pragma unroll
                for (int i = gq * NUPD / NG; i < (gq + 1) * NUPD / NG; i++) bupd(i);
                if (gq < NG - 1) {
                    if (!isdec2) st4(outp + 4 * gq, y);
                    else st2(xn + 2 * gq, v_mul(gdec, y[0]), v_mul(gdec, y[2]));
                } else {
                    // last group: slots CH-4, CH-3 (a 2-sample stage), CH-2 (a 1-sample stage), CH-1 (ruler)
                    const bool gl = opq(G != 0);
                    if (!isdec2) {
                        st4(outp + 4 * gq, y);
                    } else {
                        xn[2 * gq] = v_mul(gdec, y[0]);
                        if (!gl) xn[2 * gq + 1] = v_mul(gdec, y[2]);
                        if (gl && pvB && !(cidxB & 1)) sMB[JR * 2 + ((cidxB >> 1) & 1)] = v_mul(gdec, y[2]);
                        if (gl && pvR && !(m & 1)) sMB[(jrc + 1) * 2 + ((m >> 1) & 1)] = v_mul(gdec, y[3]);
                    }
                    if (gl && isband) {
                        // exp_smoothed_value of the low-rate stages: e <- (1-alpha) e + y^2 (e/alpha form)
                        const float alj = sAl[jrc];
                        T e = sER[jrc * 4 + r];
                        e = v_add(v_fma(-alj, e, e), v_sq(y[3]));      // raw units
                        if (pvR) {
                            sER[jrc * 4 + r] = e;
                            const int bl = logblock - jrc;           // block >> jrc = 2^bl samples
                            if (((m + 1) & ((1 << bl) - 1)) == 0)
                                sEN[((((m + 1) >> bl) - 1) & (EN_RING - 1)) * 32 + (n_oct - 1 - jrc) * BPO + r] =
                                    v_mul(alj * gb_lane * gb_lane, e);
                        }
                    }
                }
            }
        }
        const bool ge = opq(G != 0);
        if (ge && pvc) {
#pragma unroll
            for (int e = 0; e < RS; e++) spc[e] = cur[e];
        }
#pragma unroll
        for (int e = 0; e < RS; e++) zc[e] = v_sel(!ge && pv0, cur[e], zc[e]);
    };

    // ================================================================ phase B of step k (run after the
    // section loops of step k+1, which carried its accumulator updates): block ends, flush
    auto phaseB = [&](int k, auto check_tag) {
        constexpr bool CHECK = decltype(check_tag)::value;
        // step k wrote the band outputs of stage-0 chunk k
        const bool valid0 = !CHECK || (k >= 0 && (unsigned)k < (unsigned)n_chunks);
        // ---- block ends (warp-uniform conditions: they depend on the step only).  The BPO bands of a
        // stage are reduced side by side, level by level, so that their shuffle latencies overlap
        // instead of adding up; each band's sum is formed in the same order as a band on its own.
        if (valid0 && (((k + 1) & nbmask) == 0)) {    // stage 0: weighted sum of its CH accumulators
            const int blk = ((k + 1) >> lognb) - 1;
            T val[BPO];
#pragma unroll
            for (int b = 0; b < BPO; b++) {
                val[b] = v_fma(-om0[0], acc0[b][0], acc0[b][0]);
#pragma unroll
                for (int q = 1; q < NSL; q++) val[b] = v_add(val[b], v_fma(-om0[q], acc0[b][q], acc0[b][q]));
            }
#pragma unroll
            for (int dlt = HW / 2; dlt >= 1; dlt >>= 1) {
#pragma unroll
                for (int b = 0; b < BPO; b++) val[b] = v_add(val[b], v_shfl_xor(val[b], dlt));
            }
#pragma unroll
            for (int b = 0; b < BPO; b++) {
#pragma unroll
                for (int q = 0; q < NSL; q++) {
                    v_set(acc0[b][q], 0.f, 0.f);
                    if (hl + HW * q == CH - 1) acc0[b][q] = val[b];
                }
            }
            if (hl == 0) {
#pragma unroll
                for (int b = 0; b < BPO; b++)
                    sEN[(blk & (EN_RING - 1)) * 32 + (n_oct - 1) * BPO + b] =
                        v_mul(P.alpha[0] * P.gband[b] * P.gband[b], val[b]);
            }
        }
#pragma unroll
        for (int j = 1; j <= LOGCH; j++) {             // chunked lower-rate stages
            const int cm = k - DEC_DEPTH * j;
            // the steps of the unchecked loop have every stage's chunk index in range
            const bool ev = j <= n_oct - 1 && (!CHECK || (unsigned)cm < (unsigned)n_chunks) &&
                            (((cm + 1) & nbmask) == 0);
            if (!ev) continue;
            const int blk = ((cm + 1) >> lognb) - 1;
            const int len = CH >> j, lo = CH - 2 * len;          // slots [lo, lo + len)
            const int kb0 = (n_oct - 1 - j) * BPO;
            const float alj = sAl[j];
            T val[BPO];
            if (len >= HW) {
                // the stage fills whole registers q in [lo/HW, (lo+len)/HW): every lane takes part
#pragma unroll
                for (int b = 0; b < BPO; b++) {
                    v_set(val[b], 0.f, 0.f);
#pragma unroll
                    for (int q = lo / HW; q < (lo + len) / HW; q++)
                        val[b] = v_add(val[b], v_fma(-omm[q], accm[b][q], accm[b][q]));
                }
#pragma unroll
                for (int dlt = HW / 2; dlt >= 1; dlt >>= 1) {
#pragma unroll
                    for (int b = 0; b < BPO; b++) val[b] = v_add(val[b], v_shfl_xor(val[b], dlt));
                }
#pragma unroll
                for (int b = 0; b < BPO; b++) {
#pragma unroll
                    for (int q = lo / HW; q < (lo + len) / HW; q++) {
                        v_set(accm[b][q], 0.f, 0.f);
                        if (hl + HW * q == lo + len - 1) accm[b][q] = val[b];
                    }
                }
                if (hl == 0) {
#pragma unroll
                    for (int b = 0; b < BPO; b++)
                        sEN[(blk & (EN_RING - 1)) * 32 + kb0 + b] = v_mul(alj * P.gband[b] * P.gband[b], val[b]);
                }
            } else {
                // the stage sits in lanes [lo % HW, lo % HW + len) of the last register
                constexpr int q = NSL - 1;
                const int l0 = lo & (HW - 1);
                const bool mine = hl >= l0 && hl < l0 + len;
#pragma unroll
                for (int b = 0; b < BPO; b++) {
                    v_set(val[b], 0.f, 0.f);
                    if (mine) val[b] = v_fma(-omm[q], accm[b][q], accm[b][q]);
                }
#pragma unroll
                for (int dlt = 1; dlt < HW / 2; dlt <<= 1) {
                    if (dlt < len) {
#pragma unroll
                        for (int b = 0; b < BPO; b++) val[b] = v_add(val[b], v_shfl_xor(val[b], dlt));
                    }
                }
                if (mine) {
#pragma unroll
                    for (int b = 0; b < BPO; b++) {
                        v_set(accm[b][q], 0.f, 0.f);
                        if (hl == l0 + len - 1) accm[b][q] = val[b];
                    }
                    if (hl == l0) {
#pragma unroll
                        for (int b = 0; b < BPO; b++)
                            sEN[(blk & (EN_RING - 1)) * 32 + kb0 + b] = v_mul(alj * P.gband[b] * P.gband[b], val[b]);
                    }
                }
            }
        }
        // ---- the band vector of the block every stage has reported goes out in one coalesced store
        {
            const int kf = k - fdelta + 1;
            if (kf > 0 && (kf & nbmask) == 0) {
                __syncwarp();
                if (want_e) {
                    const int blk = (kf >> lognb) - 1;
#pragma unroll
                    for (int t = 0; t < NWT; t++) {
                        const int i = hl + HW * t;
                        if (i < nbands) {
                            const T v = sEN[(blk & (EN_RING - 1)) * 32 + i];
                            float e0 = v_x(v), e1 = v_y(v);
                            if (a.db) {     // friture/octavespectrum.py:119-121: 10*log10(sp + 1e-30) + w
                                const float w = wreg[t];
                                e0 = fmaf(kLog10Scale, lg2_fast(e0 + 1e-30f), w);
                                e1 = fmaf(kLog10Scale, lg2_fast(e1 + 1e-30f), w);
                            }
                            float *o = eout0 + (size_t)blk * nbands + i;
                            o[0] = e0;
                            if (PACK == 2 && has2) o[a.e_stride] = e1;
                        }
                    }
                }
            }
        }
    };

    // iteration k = section loops of step k (+ accumulator updates of step k-1), block ends / flush of
    // step k-1, prefetch; one extra iteration finishes the last step.  The steps whose every slot is
    // valid (and whose predecessor's are) run in their own tight loop without the range checks.
    // Block ends and flushes happen at fixed phases of the step counter modulo the steps per block
    // (stage j's blocks end DEC_DEPTH*j steps after stage 0's, the flush fdelta steps after): one
    // bit test per step decides whether phase B has anything to do at all, instead of one compare
    // and branch per stage (each costs a lone warp ~20 cycles of branch latency).  The mask only
    // filters; phase B evaluates its own conditions.  Blocks of more than 64 steps do not fit the
    // mask and run phase B at every step.
    const int NBS = nbmask + 1;
    const bool ev_always = NBS > 64;
    unsigned long long evmask = ~0ull;
    if (!ev_always) {
        evmask = 1ull;
        for (int j = 1; j <= LOGCH && j <= n_oct - 1; j++) evmask |= 1ull << ((DEC_DEPTH * j) & nbmask);
        evmask |= 1ull << (fdelta & nbmask);
    }
    auto iteration = [&](int k, auto check_tag) {
        constexpr bool CHECK = decltype(check_tag)::value;
        phaseA(k, check_tag);
        if (CHECK || ev_always || ((evmask >> (k & nbmask)) & 1ull)) phaseB(k - 1, check_tag);
        prefetch(k + PF);
        cp_async_wait<PF - 1>();           // chunk k+1 has landed
        __syncwarp();
    };
    const int total = n_steps + 1;
    const int fast_lo = min(k_lo + 1, total);
    const int fast_hi = max(fast_lo, min(k_hi, total));
    for (int ph = 0; ph < 2; ph++) {
        const int ka = ph ? fast_hi : 0, kz = ph ? total : fast_lo;
        for (int k = ka; k < kz; k++) iteration(k, std::true_type());
        if (ph == 0)
            for (int k = fast_lo; k < fast_hi; k++) iteration(k, std::false_type());
    }

    // ---- epilogue: the pipeline is drained, every stage ended on a block boundary
    if (worker && !G) {
#pragma unroll
        for (int i = 0; i < RS; i++) sS[r * RS + i] = zc[i];
    }
    __syncwarp();
    if (alive) {
        for (int i = hl; i < n_oct * NSEC * 2; i += HW) {
            const T z = sS[i];
            gz0[i] = v_x(z);
            if (has2) gz1[i] = v_y(z);
        }
#pragma unroll
        for (int q = 0; q < NSL; q++) {
            const int p = hl + HW * q;
#pragma unroll
            for (int b = 0; b < BPO; b++) {
                if (p == CH - 1) {
                    ge0[b] = v_x(acc0[b][q]);
                    if (has2) ge1[b] = v_y(acc0[b][q]);
                }
                if (mok[q] && lastslot[q]) {
                    ge0[mst[q] * BPO + b] = v_x(accm[b][q]);
                    if (has2) ge1[mst[q] * BPO + b] = v_y(accm[b][q]);
                }
            }
        }
        for (int i = hl; i < (n_oct - JR) * BPO; i += HW) {     // ruler stages
            const int j = JR + i / BPO, b = i % BPO;
            const T e = sER[j * 4 + b];
            ge0[j * BPO + b] = v_x(e);
            if (has2) ge1[j * BPO + b] = v_y(e);
        }
    }
}

template <int LOGCH, int PACK, int BPO>
int launch_pipe(frt_ctx *h, const PipeParams &P, const BankArgs &a, cudaStream_t st) {
    using LY = PipeLayout<LOGCH, PACK, BPO>;
    const size_t smem = (size_t)LY::TB * NSLOT * LY::TOTAL + 2 * 12 * 4;
    const int per_warp = NSLOT * PACK;
    const unsigned blocks = (unsigned)((a.n_channels + per_warp - 1) / per_warp);
    return frt_launch(h, bank_pipe_kernel<LOGCH, PACK, BPO>, blocks, 32, smem, st, P, a);
}

template <int LOGCH, int PACK>
int launch_pipe_bpo(frt_ctx *h, const PipeParams &P, const BankArgs &a, cudaStream_t st) {
    if (P.bpo == 3) return launch_pipe<LOGCH, PACK, 3>(h, P, a, st);
    return launch_pipe<LOGCH, PACK, 1>(h, P, a, st);
}

}   // namespace

// Step at which the chain heads of stage j start (T[j]) and the number of steps that drains the
// pipeline for t_total samples per channel.  Stages j <= logch move a chunk of 2^logch >> j samples
// per step, DEC_DEPTH steps (the decimator chain) behind the previous stage; stage j > logch has one
// sample every P_j = 2^(j-logch) steps, at steps u = T_j (mod P_j) with T_j = P_j/2 - 1 (mod P_j),
// which makes the stages' turns disjoint (the ruler sequence JR + ctz(u+1)).
void frt_pipe_schedule(int n_oct, int logch, long long t_total, int *T, int *n_steps) {
    T[0] = 0;
    for (int j = 1; j <= BANK_MAX_OCT; j++) {
        int t = T[j - 1] + DEC_DEPTH;
        if (j > logch) {
            const int P = 1 << (j - logch), arem = P / 2 - 1;
            while (t % P != arem) t++;
        }
        T[j] = t;
    }
    if (!n_steps) return;
    const long long n_chunks = t_total >> logch;
    long long last = 0;
    for (int j = 0; j < n_oct; j++) {
        const int dmax = (j == n_oct - 1) ? 0 : DEC_DEPTH - 1;
        long long l;
        if (j <= logch) l = n_chunks - 1 + T[j] + dmax;
        else l = T[j] + (((t_total >> j) - 1) << (j - logch)) + dmax;
        if (l > last) last = l;
    }
    // block b's band vector is flushed at step (b+1)*NB - 1 + delta
    const long long flush_last = n_chunks - 1 + frt_pipe_flush_delta(n_oct, logch, T);
    if (flush_last > last) last = flush_last;
    *n_steps = (int)(last + 1);
}

// Steps after a block's last stage-0 chunk (step (b+1)*NB - 1) at which every stage has staged the
// block's band energies: chunked stage j reports T_j steps later, ruler stage j during step
// T_j - P_j of that scale (readable one phase later, hence + 1).
int frt_pipe_flush_delta(int n_oct, int logch, const int *T) {
    int delta = 0;
    for (int j = 1; j < n_oct; j++) {
        const int dj = j <= logch ? T[j] : T[j] - (1 << (j - logch)) + 1;
        if (dj > delta) delta = dj;
    }
    return delta;
}

// Builds the kernel's tables and sets pl->pipe_ok for bank_route: the kernel is compiled for 1 and 3
// bands per octave, and its energy ring must hold the shortest block bank_route runs at each step size
// (longer blocks of the same steps stage fewer); other banks run the chunk-scan kernels.
void frt_pipe_prepare(BankPlan *pl) {
    const BankParams &B = pl->params;
    pl->pipe_ok = (B.bpo == 1 || B.bpo == 3);
    if (!pl->pipe_ok) return;
    for (int v = 0; v < 2; v++) {
        const int logch = 5 + v, CH = 1 << logch;
        PipeParams &P = pl->pipe[v];
        memset(&P, 0, sizeof(P));
        P.n_oct = B.n_oct;
        P.bpo = B.bpo;
        for (int r = 0; r < B.nsec; r++) {
            P.na1[r] = -B.coef[r][3];
            P.na2[r] = -B.coef[r][4];
            P.b1[r] = B.coef[r][5];      // c - a1, rounded once from double (frt_bank_plan)
        }
        for (int b = 0; b < B.bpo; b++) P.gband[b] = B.gband[b];
        P.gdec = B.gdec;
        for (int j = 0; j <= BANK_MAX_OCT; j++) P.alpha[j] = j < B.n_oct ? (float)pl->alphas[j] : 1.f;
        frt_pipe_schedule(B.n_oct, logch, 0, P.T, nullptr);
        P.fdelta = frt_pipe_flush_delta(B.n_oct, logch, P.T);
        // blocks staged but not yet flushed when a block's vector leaves, plus the one being written
        // (+1: the section loops of the next step already stage energies while a block is flushed)
        const int nb = PIPE_MIN_BLOCK[v] >> logch;      // steps per block
        if ((P.fdelta + nb - 1) / nb + 2 > EN_RING) pl->pipe_ok = false;
        const double q0 = 1.0 - pl->alphas[0];
        P.aq0 = (float)(1.0 - pow(q0, CH));
        for (int p = 0; p < CH; p++) {
            P.om0[p >> 5][p & 31] = (float)(1.0 - pow(q0, CH - 1 - p));
            int j = 1;
            while (j <= logch && p >= CH - (CH >> j)) j++;
            if (j <= logch && j < B.n_oct) {
                const int len = CH >> j, pos = p - (CH - 2 * len);
                const double qj = 1.0 - pl->alphas[j];
                P.aqm[p >> 5][p & 31] = (float)(1.0 - pow(qj, len));
                P.omm[p >> 5][p & 31] = (float)(1.0 - pow(qj, len - 1 - pos));
            }
        }
    }
}

// Runs the variant bank_route chose; two channels per lane run 32-sample steps only.
int frt_pipe_launch(frt_ctx *h, const BankPlan *pl, BankArgs a, int logch, int pack, cudaStream_t st) {
    const PipeParams &P = pl->pipe[logch - 5];
    int T[BANK_MAX_OCT + 1];
    frt_pipe_schedule(P.n_oct, logch, a.t_total, T, &a.n_steps);
    if (pack == 2) return launch_pipe_bpo<5, 2>(h, P, a, st);
    return logch == 5 ? launch_pipe_bpo<5, 1>(h, P, a, st) : launch_pipe_bpo<6, 1>(h, P, a, st);
}
