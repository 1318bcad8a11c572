// Host-buffer entry point of the combined per-hop analysis (BASELINE.json configs[4]'s unit): for
// every channel and every hop of new samples one log-power spectrogram column
// (friture/spectrogram.py:149-161 -> audioproc.analyzelive + log_spectrogram) and one vector of
// smoothed fractional-octave band levels (friture/octavespectrum.py:101-121 -> Octave_Filters.filter,
// y**2, exp_smoothed_value, 10*log10 + weighting).  The stream is cut into time segments; the H2D
// copy of segment s+1, the two kernels of segment s and the D2H copy of segment s-1 overlap.  All channels go through every launch: the filterbank's
// parallelism is the channel axis.
#include "bank_internal.cuh"

// Queues the segments on the staging streams; returns at the first error, with work still queued.
static int combined_segments(frt_handle h, const float *x_host, int64_t x_stride, int n_channels,
                             int64_t n_samples, int hop, float *spec_host, float *bands_host, int nbands,
                             int db) {
    const int N = h->stft->n_fft;
    const int nbins = N / 2 + 1;
    const int64_t B = n_samples / hop;                                   // filterbank blocks
    const int64_t F = n_samples >= N ? (n_samples - N) / hop + 1 : 0;    // spectrogram columns
    CombStaging &p = h->comb_host;
    FRT_CUDA(h, p.create());
    FRT_CUDA(h, p.d_x.grow((size_t)n_channels * n_samples));
    FRT_CUDA(h, p.d_spec.grow((size_t)n_channels * (F > 0 ? F : 1) * nbins));
    FRT_CUDA(h, p.d_bands.grow((size_t)n_channels * B * nbands));
    float *const d_x = p.d_x.get(), *const d_spec = p.d_spec.get(), *const d_bands = p.d_bands.get();
    const cudaStream_t s_in = p.s_in.get(), s_cmp = p.s_cmp.get(), s_out = p.s_out.get();
    int rc;
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
        FRT_CUDA(h, cudaMemcpy2DAsync(d_x + b0 * hop, sizeof(float) * n_samples, x_host + b0 * hop,
                                      sizeof(float) * x_stride, sizeof(float) * (b1 - b0) * hop,
                                      n_channels, cudaMemcpyHostToDevice, s_in));
        FRT_CUDA(h, cudaEventRecord(p.ev_in[s].get(), s_in));
        // spectrogram columns whose last sample has arrived
        const int64_t avail = b1 * hop;
        const int64_t f1 = avail >= N ? (avail - N) / hop + 1 : 0;
        FRT_CUDA(h, cudaStreamWaitEvent(s_cmp, p.ev_in[s].get(), 0));
        if (f1 > f_done) {
            rc = frt_stft_process(h, d_x + f_done * hop, n_samples, n_channels, f1 - f_done, hop,
                                  d_spec + f_done * nbins, F * (int64_t)nbins, nbins,
                                  FRT_STFT_LOGPOWER, s_cmp);
            if (rc) return rc;
        }
        FRT_CUDA(h, cudaEventRecord(p.ev_cmp[s].get(), s_cmp));
        // the filterbank follows the transform on the SAME stream: side by side the STFT kernel's fat
        // persistent CTAs starve the filterbank's one-warp CTAs (measured: 3.9 ms vs 3.1 ms back to back)
        rc = frt_bank_process_strided(h, d_x + b0 * hop, n_samples, hop, (int)(b1 - b0),
                                      d_bands + b0 * nbands, B * (int64_t)nbands, db, s_cmp);
        if (rc) return rc;
        FRT_CUDA(h, cudaEventRecord(p.ev_out[s].get(), s_cmp));   // segment s's outputs are complete
        // the columns leave as soon as the transform is done, the band vectors after the filterbank
        FRT_CUDA(h, cudaStreamWaitEvent(s_out, p.ev_cmp[s].get(), 0));
        if (f1 > f_done)
            FRT_CUDA(h, cudaMemcpy2DAsync(spec_host + f_done * nbins, sizeof(float) * F * nbins,
                                          d_spec + f_done * nbins, sizeof(float) * F * nbins,
                                          sizeof(float) * (f1 - f_done) * nbins, n_channels,
                                          cudaMemcpyDeviceToHost, s_out));
        if (f1 > f_done) f_done = f1;
        last = s;
    }
    // the band vectors (C x B x nbands, 1.5 % of the output) leave in ONE contiguous copy at the end: cut
    // per segment they are C rows of a few hundred bytes each, which costs the copy engine more time
    // than the spectrogram columns next to them
    FRT_CUDA(h, cudaStreamWaitEvent(s_out, p.ev_out[last].get(), 0));
    FRT_CUDA(h, cudaMemcpyAsync(bands_host, d_bands, sizeof(float) * (size_t)n_channels * B * nbands,
                                cudaMemcpyDeviceToHost, s_out));
    return FRT_OK;
}

extern "C" int frt_combined_process_host(frt_handle h, const float *x_host, int64_t x_stride,
                                         int n_channels, int64_t n_samples, int hop,
                                         float *spec_host, float *bands_host, int nbands, int db) {
    if (!h) return FRT_EINVAL;
    DeviceGuard g(h->device);
    if (!h->stft) return frt_fail(h, FRT_ESTATE, "frt_combined_process_host: call frt_stft_plan first");
    if (!h->bank) return frt_fail(h, FRT_ESTATE, "frt_combined_process_host: call frt_bank_plan first");
    // every refusal comes before the first copy: the bank runs over all of its plan's channels and
    // writes its plan's bands, so the staging buffers, sized from the arguments, must hold exactly those
    const BankPlan *pl = h->bank.get();
    FRT_CHECK_ARG(h, n_channels >= 1 && hop >= 256 && n_samples >= 0, "bad shape");
    FRT_CHECK_ARG(h, n_channels == pl->n_channels, "n_channels differs from the filterbank plan's channels");
    FRT_CHECK_ARG(h, nbands == pl->params.n_oct * pl->params.bpo, "nbands differs from the filterbank plan's bands");
    if (const int rc = frt_bank_check_block(h, pl, hop)) return rc;
    FRT_CHECK_ARG(h, n_samples % hop == 0, "n_samples must be a whole number of hops");
    FRT_CHECK_ARG(h, x_stride >= n_samples, "x_stride smaller than n_samples");
    if (n_samples == 0) return FRT_OK;
    // a stream shorter than one frame has band levels but no columns: spec_host may then be empty
    const bool has_columns = n_samples >= h->stft->n_fft;
    FRT_CHECK_ARG(h, x_host && bands_host && (spec_host || !has_columns), "NULL buffer");
    // the staging streams are non-blocking and wait for nothing: a device call on this handle that is
    // still queued on any stream (it reads and writes the filterbank state) must finish first
    FRT_CUDA(h, cudaDeviceSynchronize());
    int rc = combined_segments(h, x_host, x_stride, n_channels, n_samples, hop, spec_host, bands_host, nbands, db);
    // the queued copies read and write the caller's buffers: whatever happened, none is still in
    // flight when the call returns
    CombStaging &p = h->comb_host;
    for (const cudaStream_t s : {p.s_out.get(), p.s_cmp.get(), p.s_in.get()}) {
        if (!s) continue;
        const cudaError_t e = cudaStreamSynchronize(s);
        if (rc == FRT_OK && e != cudaSuccess) rc = frt_cuda_fail(h, e, "cudaStreamSynchronize", __FILE__, __LINE__);
    }
    return rc;
}
