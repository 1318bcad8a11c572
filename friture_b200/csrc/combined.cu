// Host-buffer entry point of the combined per-hop analysis (BASELINE.json configs[4]'s unit): for
// every channel and every hop of new samples one log-power spectrogram column
// (friture/spectrogram.py:149-161 -> audioproc.analyzelive + log_spectrogram) and one vector of
// smoothed fractional-octave band levels (friture/octavespectrum.py:101-121 -> Octave_Filters.filter,
// y**2, exp_smoothed_value, 10*log10 + weighting).  The stream is cut into time segments; the H2D
// copy of segment s+1, the two kernels of segment s and the D2H copy of segment s-1 overlap.  All channels go through every launch: the filterbank's
// parallelism is the channel axis.
#include "frt_internal.cuh"

namespace {
constexpr int MAX_SEG = 32;
}

struct CombPipe {
    float *d_x = nullptr, *d_spec = nullptr, *d_bands = nullptr;
    size_t x_bytes = 0, spec_bytes = 0, bands_bytes = 0;
    cudaStream_t s_in = nullptr, s_stft = nullptr, s_bank = nullptr, s_out = nullptr;
    cudaEvent_t ev_in[MAX_SEG] = {}, ev_stft[MAX_SEG] = {}, ev_bank[MAX_SEG] = {};
};

void frt_comb_release(frt_ctx *h) {
    CombPipe *p = reinterpret_cast<CombPipe *>(h->comb);
    if (!p) return;
    if (p->d_x) cudaFree(p->d_x);
    if (p->d_spec) cudaFree(p->d_spec);
    if (p->d_bands) cudaFree(p->d_bands);
    for (int i = 0; i < MAX_SEG; i++) {
        if (p->ev_in[i]) cudaEventDestroy(p->ev_in[i]);
        if (p->ev_stft[i]) cudaEventDestroy(p->ev_stft[i]);
        if (p->ev_bank[i]) cudaEventDestroy(p->ev_bank[i]);
    }
    if (p->s_in) cudaStreamDestroy(p->s_in);
    if (p->s_stft) cudaStreamDestroy(p->s_stft);
    if (p->s_bank) cudaStreamDestroy(p->s_bank);
    if (p->s_out) cudaStreamDestroy(p->s_out);
    delete p;
    h->comb = nullptr;
}

static int comb_ensure(frt_ctx *h, size_t xb, size_t sb, size_t bb) {
    CombPipe *p = reinterpret_cast<CombPipe *>(h->comb);
    if (!p) {
        p = new (std::nothrow) CombPipe();
        if (!p) return frt_fail(h, FRT_ENOMEM, "out of host memory");
        h->comb = p;
        FRT_CUDA(h, cudaStreamCreateWithFlags(&p->s_in, cudaStreamNonBlocking));
        FRT_CUDA(h, cudaStreamCreateWithFlags(&p->s_stft, cudaStreamNonBlocking));
        FRT_CUDA(h, cudaStreamCreateWithFlags(&p->s_bank, cudaStreamNonBlocking));
        FRT_CUDA(h, cudaStreamCreateWithFlags(&p->s_out, cudaStreamNonBlocking));
        for (int i = 0; i < MAX_SEG; i++) {
            FRT_CUDA(h, cudaEventCreateWithFlags(&p->ev_in[i], cudaEventDisableTiming));
            FRT_CUDA(h, cudaEventCreateWithFlags(&p->ev_stft[i], cudaEventDisableTiming));
            FRT_CUDA(h, cudaEventCreateWithFlags(&p->ev_bank[i], cudaEventDisableTiming));
        }
    }
    if (xb > p->x_bytes) {
        if (p->d_x) cudaFree(p->d_x);
        p->d_x = nullptr;
        p->x_bytes = 0;
        FRT_CUDA(h, cudaMalloc(&p->d_x, xb));
        p->x_bytes = xb;
    }
    if (sb > p->spec_bytes) {
        if (p->d_spec) cudaFree(p->d_spec);
        p->d_spec = nullptr;
        p->spec_bytes = 0;
        FRT_CUDA(h, cudaMalloc(&p->d_spec, sb));
        p->spec_bytes = sb;
    }
    if (bb > p->bands_bytes) {
        if (p->d_bands) cudaFree(p->d_bands);
        p->d_bands = nullptr;
        p->bands_bytes = 0;
        FRT_CUDA(h, cudaMalloc(&p->d_bands, bb));
        p->bands_bytes = bb;
    }
    return FRT_OK;
}

extern "C" int frt_combined_process_host(frt_handle h, const float *x_host, int64_t x_stride,
                                         int n_channels, int64_t n_samples, int hop,
                                         float *spec_host, float *bands_host, int nbands, int db) {
    if (!h) return FRT_EINVAL;
    DeviceGuard g(h->device);
    const int N = h->stft.n_fft;
    if (!N) return frt_fail(h, FRT_ESTATE, "frt_combined_process_host: call frt_stft_plan first");
    if (!h->bank) return frt_fail(h, FRT_ESTATE, "frt_combined_process_host: call frt_bank_plan first");
    FRT_CHECK_ARG(h, n_channels >= 1 && hop >= 256 && n_samples >= 0, "bad shape");
    FRT_CHECK_ARG(h, n_samples % hop == 0, "n_samples must be a whole number of hops");
    FRT_CHECK_ARG(h, x_host && spec_host && bands_host, "NULL buffer");
    FRT_CHECK_ARG(h, x_stride >= n_samples, "x_stride smaller than n_samples");
    const int nbins = N / 2 + 1;
    const int64_t B = n_samples / hop;                                   // filterbank blocks
    const int64_t F = n_samples >= N ? (n_samples - N) / hop + 1 : 0;    // spectrogram columns
    if (B == 0) return FRT_OK;
    int rc = comb_ensure(h, sizeof(float) * (size_t)n_channels * n_samples,
                         sizeof(float) * (size_t)n_channels * (F > 0 ? F : 1) * nbins,
                         sizeof(float) * (size_t)n_channels * B * nbands);
    if (rc) return rc;
    CombPipe &p = *reinterpret_cast<CombPipe *>(h->comb);
    // the first segment's H2D and the last segment's D2H are not overlapped with anything, short
    // segments keep that exposed part small; very short ones cost more in 2-D copy rows and kernel
    // launches than they save.  Measured before the H100 port (card not recorded) at 1024 ch x 129
    // blocks (0.54 GB in, 0.55 GB out): 4 segments 14.8 ms, 8: 13.5, 12: 13.0, 16: 12.9, 24: 14.7,
    // 32: 15.0
    int nseg = B >= 128 ? 16 : (B >= 64 ? 8 : (B >= 8 ? 4 : 1));
    if (nseg > B) nseg = (int)B;
    const int64_t seg_blocks = (B + nseg - 1) / nseg;
    int64_t f_done = 0;
    int last = 0;
    for (int s = 0; s < nseg; s++) {
        const int64_t b0 = s * seg_blocks, b1 = (b0 + seg_blocks < B) ? b0 + seg_blocks : B;
        if (b0 >= b1) break;
        FRT_CUDA(h, cudaMemcpy2DAsync(p.d_x + b0 * hop, sizeof(float) * n_samples, x_host + b0 * hop,
                                      sizeof(float) * x_stride, sizeof(float) * (b1 - b0) * hop,
                                      n_channels, cudaMemcpyHostToDevice, p.s_in));
        FRT_CUDA(h, cudaEventRecord(p.ev_in[s], p.s_in));
        // spectrogram columns whose last sample has arrived
        const int64_t avail = b1 * hop;
        const int64_t f1 = avail >= N ? (avail - N) / hop + 1 : 0;
        FRT_CUDA(h, cudaStreamWaitEvent(p.s_stft, p.ev_in[s], 0));
        if (f1 > f_done) {
            rc = frt_stft_process(h, p.d_x + f_done * hop, n_samples, n_channels, f1 - f_done, hop,
                                  p.d_spec + f_done * nbins, F * (int64_t)nbins, nbins,
                                  FRT_STFT_LOGPOWER, p.s_stft);
            if (rc) return rc;
        }
        FRT_CUDA(h, cudaEventRecord(p.ev_stft[s], p.s_stft));
        // the filterbank follows the transform on the SAME stream: side by side the STFT kernel's fat
        // persistent CTAs starve the filterbank's one-warp CTAs (measured: 3.9 ms vs 3.1 ms back to back)
        rc = frt_bank_process_strided(h, p.d_x + b0 * hop, n_samples, hop, (int)(b1 - b0),
                                      p.d_bands + b0 * nbands, B * (int64_t)nbands, db, p.s_stft);
        if (rc) return rc;
        FRT_CUDA(h, cudaEventRecord(p.ev_bank[s], p.s_stft));
        // the columns leave as soon as the transform is done, the band vectors after the filterbank
        FRT_CUDA(h, cudaStreamWaitEvent(p.s_out, p.ev_stft[s], 0));
        if (f1 > f_done)
            FRT_CUDA(h, cudaMemcpy2DAsync(spec_host + f_done * nbins, sizeof(float) * F * nbins,
                                          p.d_spec + f_done * nbins, sizeof(float) * F * nbins,
                                          sizeof(float) * (f1 - f_done) * nbins, n_channels,
                                          cudaMemcpyDeviceToHost, p.s_out));
        if (f1 > f_done) f_done = f1;
        last = s;
    }
    // the band vectors (C x B x nbands, 1.5 % of the output) leave in ONE contiguous copy at the end: cut
    // per segment they are C rows of a few hundred bytes each, which costs the copy engine more time
    // than the spectrogram columns next to them
    FRT_CUDA(h, cudaStreamWaitEvent(p.s_out, p.ev_bank[last], 0));
    FRT_CUDA(h, cudaMemcpyAsync(bands_host, p.d_bands, sizeof(float) * (size_t)n_channels * B * nbands,
                                cudaMemcpyDeviceToHost, p.s_out));
    FRT_CUDA(h, cudaStreamSynchronize(p.s_out));
    FRT_CUDA(h, cudaStreamSynchronize(p.s_stft));
    FRT_CUDA(h, cudaStreamSynchronize(p.s_bank));
    FRT_CUDA(h, cudaStreamSynchronize(p.s_in));
    return FRT_OK;
}
