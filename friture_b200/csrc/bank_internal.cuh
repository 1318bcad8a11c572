// Shared between bank.cu (chunk-scan kernels, plan/state management) and bank_pipe.cu (the
// lane-pipelined kernel): coefficient tables, the plan and the launch arguments.
//
// All kernels run the reference's filters (friture/generated_filters.py) as NORMALISED float32
// second-order sections: every elliptic section has its zeros on the unit circle, b = g*(1, c, 1),
// so the recursion of friture/signal/lfilter.py:131-139 becomes
//     y = x + z1;  z1 = c*x - a1*y + z2;  z2 = x - a2*y          (4 instead of 5 operations)
// and the chain gain (product of the g's) is applied once per chain: on the band output before
// squaring, on the decimator output where the even samples are kept.  The filter state the handle
// carries is the state of these normalised sections.
#pragma once

#include "frt_internal.cuh"

constexpr int BANK_MAX_BPO = 24;
constexpr int BANK_MAX_SEC = 2 * BANK_MAX_BPO + 6;
constexpr int BANK_MAX_OCT = 10;
constexpr int BANK_NQ = 10;   // A^(2^q), q = 0..9: chunk L <= 32 (q <= 5) plus 4 doublings

struct BankParams {
    float coef[BANK_MAX_SEC][8];        // 1 c 1 a1 a2 B1 B2 -, B = (c - a1, 1 - a2)
    float apow[BANK_MAX_SEC][BANK_NQ][4];    // A^(2^q), A = [[-a1, 1], [-a2, 0]], row-major
    float omq[BANK_MAX_OCT][BANK_NQ];   // 1 - (1 - alpha_j)^(2^q): decay in complement form
    float alpha[BANK_MAX_OCT];
    float gband[BANK_MAX_BPO];          // chain gain of band i (applied to its output)
    float gdec;                         // chain gain of the decimation low-pass
    int bpo, n_oct, nsec;          // nsec = 2*bpo + 6; band i section s -> 2*i+s; dec s -> 2*bpo+s
};

// ---- lane-pipelined kernel (bank_pipe.cu) -------------------------------------------------------
constexpr int PIPE_MAX_SEC = 16;    // 2*bpo + 6 <= 16: bpo in {1, 3}
constexpr int PIPE_RX = 8;          // input ring depth (chunks)
constexpr int PIPE_PF = 4;          // prefetch distance (chunks)
constexpr int PIPE_MIN_BLOCK[2] = {256, 512};   // [logch - 5]: shortest block bank_route runs in such steps

struct PipeParams {
    float na1[PIPE_MAX_SEC], na2[PIPE_MAX_SEC];   // per section: -a1, -a2
    float b1[PIPE_MAX_SEC];                       // c - a1
    float gband[4];
    float gdec;
    float alpha[BANK_MAX_OCT + 1];
    // smoothing accumulators, one per sample slot of a step (slot = lane + 32*s):
    float aq0;                  // 1 - q_0^CH
    float om0[4][32];           // 1 - q_0^(CH-1-slot)
    float aqm[4][32];           // multiplexed vector: 1 - q_j^len_j of the slot's stage j
    float omm[4][32];           // 1 - q_j^(len_j-1-pos)
    int T[BANK_MAX_OCT + 1];    // step at which stage j's chain heads start (pipe_schedule)
    int fdelta;                 // steps after a block's last chunk until every stage has staged its energies
    int n_oct, bpo;
};

struct BankArgs {
    const float *x;
    long long x_stride;
    int n_channels;
    int n_tiles;           // tiles per launch (per channel)              [scan kernels]
    int tiles_per_block;   // energies are emitted after every tiles_per_block-th tile
    float *zstate;         // [C][n_oct][nsec][2]
    float *ema;            // [C][n_oct][bpo]   smoothed energies / alpha_j (dispbuffers / alpha)
    float *energies;       // channel c, block b at energies + c*e_stride + b*nbands, or NULL
    long long e_stride;    // floats between channels (n_blocks*nbands when contiguous)
    float *y;              // ragged band outputs or NULL
    long long y_stride;
    long long t_total;     // samples per channel in this launch
    int db;                // 1: energies as 10*log10(e + 1e-30) (+ weight)
    int vec_ok;
    const float *weight;   // [nbands] dB offsets added in db mode, or NULL (octavespectrum.py:119-121)
    int block;             // samples per block                            [pipe kernel]
    int n_blocks;
    int n_steps;
};

struct BankPlan {
    BankParams params;
    PipeParams pipe[2];    // [logch - 5]: 32 / 64-sample steps
    bool pipe_ok = false;  // the lane-pipelined kernel can run this bank's blocks (frt_pipe_prepare)
    int n_channels = 0;
    DeviceArray<float> zstate, ema;
    DeviceArray<float> weight;   // device copy of the dB weighting vector, or empty
    size_t nz = 0, ne = 0;     // floats per channel
    double alphas[BANK_MAX_OCT];
};

// bank.cu: FRT_EINVAL (with the handle's error message) when the filterbank refuses blocks of
// `block` samples for this plan (bank_route); the filterbank and combined entry points refuse such a
// block before they queue anything
int frt_bank_check_block(frt_ctx *h, const BankPlan *pl, int block);

// bank_pipe.cu
void frt_pipe_prepare(BankPlan *pl);
void frt_pipe_schedule(int n_oct, int logch, long long t_total, int *T /*[BANK_MAX_OCT+1]*/, int *n_steps);
int frt_pipe_flush_delta(int n_oct, int logch, const int *T);
int frt_pipe_launch(frt_ctx *h, const BankPlan *pl, BankArgs a, int logch, int pack, cudaStream_t st);
