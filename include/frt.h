/*
 * frt.h -- C ABI of friture_b200, the H100-native (sm_90a) implementation of Friture's
 * per-chunk spectral hot path.
 *
 * The reference (tlecomte/friture) is pure Python/NumPy and has no FFI: its boundary is the
 * Python call surface the widgets use.  Each entry point below names the reference interface
 * it stands behind (file:line relative to the reference root).  The host side
 * (friture_b200/*.py) binds these with ctypes and keeps the reference's class / method names.
 *
 * Conventions
 *   - plain pointers and sizes only; `*_dev` pointers are device memory on the handle's GPU,
 *     `*_host` pointers are host memory (pinned for full PCIe speed, pageable also works);
 *   - `stream` is a cudaStream_t passed as void* (NULL = the legacy default stream); device
 *     entry points are asynchronous on it, host entry points return when the result is in
 *     the caller's host buffer;
 *   - the library never owns caller buffers; plans, coefficient tables and filter / smoothing
 *     state live in the handle;
 *   - a plan call that fails leaves the handle's previous plan of that kind in place;
 *   - every function returns FRT_OK (0) or a negative FRT_E* code; frt_last_error(h) gives the
 *     message.  There is no CPU fallback anywhere: without a CUDA device frt_create fails.
 */
#ifndef FRT_H
#define FRT_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define FRT_OK 0
#define FRT_EINVAL (-1)   /* bad argument (shape, alignment, unsupported size)           */
#define FRT_ECUDA (-2)    /* CUDA runtime error (message holds cudaGetErrorString)       */
#define FRT_ENOMEM (-3)   /* host or device allocation failed: every entry point that
                             allocates (plans, setters, grow-only workspaces, staging,
                             frt_host_alloc, frt_peer_alloc) returns it when an
                             allocation fails, and leaves the handle usable            */
#define FRT_ESTATE (-4)   /* call order problem (e.g. process before plan)               */

typedef struct frt_ctx *frt_handle;

/* ---------------------------------------------------------------- lifecycle */
int frt_version(void);
/* Bind a handle to CUDA device `device`.  Fails (FRT_ECUDA) when no device is usable.       */
int frt_create(int device, frt_handle *out);
int frt_destroy(frt_handle h);
const char *frt_last_error(frt_handle h);   /* h may be NULL: last frt_create failure      */
int frt_device_sm_count(frt_handle h);
/* Number of kernels this handle has launched so far (bench.py's gpu_launches).            */
int64_t frt_launch_count(frt_handle h);
/* Pinned host memory for the *_host entry points.                                          */
int frt_host_alloc(frt_handle h, size_t bytes, void **out);
int frt_host_free(frt_handle h, void *p);

/* ---------------------------------------------------------------- STFT (audioproc)
 * Stands behind friture/audioproc.py:27-81 (`audioproc.set_fftsize`, `analyzelive`,
 * `norm_square`, `update_window`) and the framing loops that call it,
 * friture/spectrogram.py:131-159 and friture/spectrum.py:125-155, plus
 * `log_spectrogram`, friture/spectrogram.py:119-125.                                        */

#define FRT_STFT_POWER 0      /* |rfft(x*hann)|^2 / N^2           (analyzelive)             */
#define FRT_STFT_LOGPOWER 1   /* 10*log10(power + 1e-30)          (log_spectrogram)         */

/* Build the symmetric-Hann window and twiddle tables for `n_fft` (32*2^k, 32..16384;
 * friture/spectrum_settings.py:61-70).  Replaces audioproc.set_fftsize.                    */
int frt_stft_plan(frt_handle h, int n_fft);
/* Copy the plan's float32 window (n_fft values) to `window_host` (audioproc.window).        */
int frt_stft_window(frt_handle h, float *window_host);
/* Batched STFT.  Channel c, frame f is samples x[c*x_stride + f*hop .. + n_fft) and is written
 * to out[c*out_stride_c + f*out_stride_f + k], k = 0..n_fft/2.  One frame == one
 * analyzelive() call of the reference.                                                      */
int frt_stft_process(frt_handle h, const float *x_dev, int64_t x_stride, int n_channels,
                     int64_t n_frames, int hop, float *out_dev, int64_t out_stride_c,
                     int64_t out_stride_f, int mode, void *stream);
/* Same with host buffers: H2D copy, kernels and D2H copy are pipelined over channel groups
 * inside the call (bench.py's `e2e`).  n_samples is per channel; frames = (n_samples-n_fft)/hop+1,
 * out_host is [n_channels][frames][n_fft/2+1] contiguous.                                   */
int frt_stft_process_host(frt_handle h, const float *x_host, int64_t x_stride, int n_channels,
                          int64_t n_samples, int hop, float *out_host, int mode);
/* The spectrogram's screen rows straight from the frames: frame f of channel c (framed as in
 * frt_stft_process, with the frt_stft_plan'ed size) is transformed to its FRT_STFT_LOGPOWER column,
 * which stays on chip, and only its `height` rows are written,
 *   rows[c*rows_stride_c + f*rows_stride_f + r] = fmaf(t[r], b - a, a),
 *   a = (db[i0[r]] + w[i0[r]] - spec_min) / (spec_max - spec_min), b = the same at i0[r] + 1,
 * bit for bit what frt_display_columns interpolates from the stored column (w = weight_dev, or 0
 * when it is NULL).  row_i0_dev/row_t_dev are the screen-row table of frt_display_columns:
 * 0 <= i0[r] <= n_fft/2 - 1 (= nbins - 2) is the caller's precondition.  Needs height >= 1,
 * spec_max != spec_min and rows_stride_f >= height; n_channels == 0 or n_frames == 0 is a no-op.
 * Feed the rows to frt_display_rows.                                                           */
int frt_stft_screen_rows(frt_handle h, const float *x_dev, int64_t x_stride, int n_channels,
                         int64_t n_frames, int hop, const float *weight_dev, float spec_min,
                         float spec_max, const int *row_i0_dev, const float *row_t_dev, int height,
                         float *rows_dev, int64_t rows_stride_c, int64_t rows_stride_f, void *stream);

/* ---------------------------------------------------------------- filterbank (Octave_Filters)
 * Stands behind friture/octavefilters.py:37-158 (`Octave_Filters.filter`, `setbandsperoctave`)
 * with the numerics of the reference's IIR bank `octave_filter_bank_decimation`
 * (friture/filter.py:86-118, `decimate` friture/signal/decimate.py:27-42, recursion
 * friture/signal/lfilter.py:85-147), fused with the octave widget's smoothing
 * `exp_smoothed_value(kernel, alpha, y**2, old)` (friture/octavespectrum.py:104,140-156;
 * friture/signal/exp_smoothing.py:11-56) and `10*log10(sp+1e-30)` (octavespectrum.py:119-120). */

/* Build the filterbank for `n_channels` independent streams.
 *   sos_band  [bands_per_octave][2][6]  second-order sections (b0 b1 b2 1 a1 a2) of the
 *             band-passes of the top octave, band 0 = lowest (generated_filters.PARAMS[bpo])
 *   sos_dec   [6][6]                    sections of the decimation low-pass (PARAMS['dec'])
 *   alphas    [n_octaves]               smoothing factor per stage j (rate fs/2^j),
 *             octavespectrum.py:150-154
 * Filter and smoothing state start at zero (filter.py:121-133; octavespectrum.py:59).        */
int frt_bank_plan(frt_handle h, int n_channels, int bands_per_octave, int n_octaves,
                  const double *sos_band, const double *sos_dec, const double *alphas);
int frt_bank_reset(frt_handle h);
/* Per-band dB offsets added to the energies when db != 0 -- the octave widget's weighting,
 * `10*log10(sp+1e-30) + w` with w = Octave_Filters.A / .B / .C (friture/octavespectrum.py:108-121,
 * friture/octavefilters.py:76-82).  weight_db_host: nbands floats (band k as below), or NULL for
 * no weighting.  Belongs to the current plan (a new frt_bank_plan clears it).                   */
int frt_bank_set_weighting(frt_handle h, const float *weight_db_host);
/* The software-pipeline schedule of the fused-energy kernel for a stream of n_samples per channel
 * processed in steps of 2^log2_chunk (5 or 6) samples: stage_start[10] = step at which stage j
 * starts, *n_steps = steps until the pipeline has drained.  Pure host arithmetic (needs no GPU);
 * exported so that tests/bank_pipeline_model.py can check the model against the library.       */
int frt_bank_schedule(int n_octaves, int log2_chunk, int64_t n_samples, int *stage_start,
                      int *n_steps);
/* Process n_blocks consecutive blocks of `block` samples per channel
 * (x[c*x_stride + b*block + n]); block % 256 == 0 (the reference needs even lengths at every
 * stage, decimate.py:41).  State is carried across calls, so any blocking of a stream gives
 * the same result.
 *   energies_dev  [C][n_blocks][nbands] or NULL: smoothed band energies after each block
 *                 (band k = (n_octaves-1-j)*bpo + i as in filter.py:104-109); dB when db != 0
 *   y_dev         NULL, or the band outputs themselves (the literal `.filter()` contract):
 *                 channel c at y_dev + c*y_stride, bands concatenated k = 0..nbands-1, band k
 *                 holding (block*n_blocks) >> j samples                                       */
int frt_bank_process(frt_handle h, const float *x_dev, int64_t x_stride, int block, int n_blocks,
                     float *energies_dev, float *y_dev, int64_t y_stride, int db, void *stream);
/* Same with the energies of channel c, block b written to energies_dev + c*e_stride_c + b*nbands
 * (e_stride_c >= n_blocks*nbands): lets a caller that cuts one stream into several launches fill
 * one [C][all blocks][nbands] array.  No ragged band outputs.                                  */
int frt_bank_process_strided(frt_handle h, const float *x_dev, int64_t x_stride, int block,
                             int n_blocks, float *energies_dev, int64_t e_stride_c, int db,
                             void *stream);
/* State checkpoint / resume (the reference keeps its state inside the object,
 * octavefilters.py:50-56).  z: [C][n_octaves][2*bpo+6][2] section states; ema:
 * [C][n_octaves][bpo] smoothed energy divided by alpha_j (the kernel's internal form, so that a
 * get/set round trip is bit-exact).  The sections run in normalised form (numerator 1, c, 1; the
 * chain gain is applied to the chain's output), z is the state of those sections.             */
int frt_bank_state_size(frt_handle h, int64_t *z_floats, int64_t *ema_floats);
int frt_bank_get_state(frt_handle h, float *z_host, float *ema_host);
int frt_bank_set_state(frt_handle h, const float *z_host, const float *ema_host);

/* ---------------------------------------------------------------- live-path filterbank (FIR)
 * The numerics of the reference's LIVE `Octave_Filters.filter` (friture/octavefilters.py:49-58):
 * FFT overlap-add with 512-tap minimum-phase FIR approximations of the same designs
 * (friture/filter.py:136-247, taps friture/data/generated_fft.npz).  Overlap-add is an exact linear
 * convolution, which the kernel computes directly (double accumulation), carrying the last
 * n_taps-1 inputs of every stage.  Parity mode; the IIR bank above is the throughput path.
 *   fir_band [bands_per_octave][n_taps], fir_dec [n_taps]  (float64 taps)
 *   process: n_samples <= 4096 and a multiple of 2^(n_octaves-1); y_dev ragged as in frt_bank_process
 * plan and reset zero the filter history and the smoothed levels of frt_firbank_levels.
 * One CTA per channel holds the taps, every stage's history and two stage buffers in shared memory:
 *     8 ((bpo+1) n_taps) + 4 (n_octaves (n_taps-1) + 2 round4(n_taps) + 1.5 block) bytes, about,
 * which must fit the device's opt-in limit per block (227 KiB on an H100).  frt_firbank_plan refuses
 * (FRT_EINVAL) a bank that does not fit at its shortest block, 2^(n_octaves-1); process and levels
 * refuse a block that does not fit, before any launch and with the plan's state unchanged.  The
 * library's 512-tap tables fit at every block (153 728 bytes at most: bpo 24, 10 octaves, 4096).  */
int frt_firbank_plan(frt_handle h, int n_channels, int bands_per_octave, int n_octaves, int n_taps,
                     const double *fir_band, const double *fir_dec);
int frt_firbank_reset(frt_handle h);
int frt_firbank_process(frt_handle h, const float *x_dev, int64_t x_stride, int n_samples,
                        float *y_dev, int64_t y_stride, void *stream);
/* Smoothing of the live-path band levels (OctaveSpectrum_Widget.setresponsetime / setweighting,
 * friture/octavespectrum.py:136-156): alphas[n_octaves] per stage j (rate fs/2^j), weight_db
 * [nbands] dB offsets added to the dB levels, or NULL for none.  Keeps the filter history and the
 * smoothed levels, as the widget keeps its display buffers.                                     */
int frt_firbank_set_smoothing(frt_handle h, const double *alphas, const float *weight_db);
/* The octave widget's levels on the live-path bank (friture/octavespectrum.py:91-121): n_blocks
 * consecutive blocks of `block` samples per channel (x[c*x_stride + b*block + n]) in one launch,
 * no band outputs.  After every block, band k = (n_octaves-1-j)*bpo + i (N = block >> j samples):
 *     sp_k <- alpha_j * sum_n (1-alpha_j)^(N-1-n) y_k[n]^2 + sp_k * (1-alpha_j)^N     (float64)
 *   levels_dev  [C][n_blocks][nbands]: sp, or 10*log10(sp + 1e-30) + weight_db when db != 0
 * block <= 4096 and a multiple of 2^(n_octaves-1); FRT_ESTATE until frt_firbank_set_smoothing.
 * Any cut of a stream into calls gives the same bits.                                           */
int frt_firbank_levels(frt_handle h, const float *x_dev, int64_t x_stride, int block, int n_blocks,
                       float *levels_dev, int db, void *stream);

/* ---------------------------------------------------------------- combined per-hop analysis
 * What Spectrogram_Widget.handle_new_data (friture/spectrogram.py:131-169) and
 * OctaveSpectrum_Widget.handle_new_data (friture/octavespectrum.py:91-121) compute from the same
 * chunk of new samples, for n_channels independent streams held in HOST memory: the log-power
 * column of every hop (frt_stft_plan'ed size, frames as in frt_stft_process_host) and the smoothed
 * band levels after every hop-sized block (frt_bank_plan'ed bank, dB + weighting when db != 0).
 * H2D copy, the two kernels and the D2H copies are pipelined over time segments inside the call
 * (bench.py's `e2e`).  n_samples % hop == 0, hop a valid filterbank block;
 *   spec_host  [n_channels][(n_samples - n_fft)/hop + 1][n_fft/2 + 1]
 *   bands_host [n_channels][n_samples/hop][nbands]
 * spec_host may be NULL when n_samples < n_fft (no columns, only band levels).
 * FRT_EINVAL, before any copy or kernel is queued and with the filter state unchanged, unless
 * n_channels is the bank plan's channel count, nbands its n_octaves * bands_per_octave, and hop a
 * block the bank runs: a multiple of 256 whose tile (the longest of 1024, 512 and 256 samples that
 * divides it) holds 2^(n_octaves-1) samples -- so at 10 octaves 768 is refused, 512 and 1536 are not.
 * Any blocking of the stream gives the same bits as frt_stft_process and frt_bank_process_strided
 * on the same samples.  The call returns only once none of its copies is still in flight, after an
 * error too.                                                                                       */
int frt_combined_process_host(frt_handle h, const float *x_host, int64_t x_stride, int n_channels,
                              int64_t n_samples, int hop, float *spec_host, float *bands_host,
                              int nbands, int db);

/* ---------------------------------------------------------------- NVLink peer memory
 * Transport of the north-star's final all-gather of spectrogram columns: every process of the box
 * allocates its gathered buffer here (a whole cudaMalloc allocation, exportable over CUDA IPC),
 * exchanges the 64-byte handles, opens its peers' buffers and pushes its own columns into them with
 * the copy engines (cudaMemcpyAsync over NVLink/NVSwitch): no SM takes part, so the transfers do
 * not compete with the filterbank kernel for issue slots (friture_b200/peer.py).                   */
int frt_peer_alloc(frt_handle h, size_t bytes, void **out);
int frt_peer_free(frt_handle h, void *p);
int frt_peer_export(frt_handle h, void *p, void *handle64);            /* cudaIpcGetMemHandle  */
int frt_peer_import(frt_handle h, const void *handle64, void **out);   /* cudaIpcOpenMemHandle */
int frt_peer_close(frt_handle h, void *peer_ptr);
int frt_peer_copy(frt_handle h, void *dst, const void *src, size_t bytes, void *stream);
/* One-hop push of a block into the same offset of n_peers (<= 15) opened peer buffers by a small copy
 * kernel (n_ctas CTAs, 0 = 64): the block is read once from local HBM and stored to every peer
 * over NVLink with 128-bit stores.  Faster than the copy engines at 8 GPUs (not at 2 or 4).                  */
int frt_peer_push(frt_handle h, const void *src, void *const *peer_dst, int n_peers, size_t bytes,
                  int n_ctas, void *stream);

/* ---------------------------------------------------------------- GCC-PHAT (delay estimator)
 * Stands behind `generalized_cross_correlation(d0, d1)` (friture/signal/correlation.py:24-43)
 * and the smoothing + peak pick around it (friture/delay_estimator.py:129-142).               */

/* Plan for frames of `length` samples, 4 .. 24 000 000 -- every delay range the widget offers
 * (0.1 .. 1000 s, L = 2 * delayrange_s * 12 kHz, delay_estimator.py:53-54,114-117,222-226).
 * Lengths frt_gcc_fits accepts (the default 24000 among them) run with the whole frame in shared
 * memory.  All others run as Bluestein transforms over a power-of-two FFT of M = 2^m >= 2L-1
 * points in global memory, whose plan (chirps and filter spectra, built in double precision)
 * takes a few seconds of host time at the longest lengths, and whose calls use a grow-only
 * workspace of about 8*M + 4*L' bytes per pair, in groups of pairs within 2 GiB (one pair at
 * least); such a call is asynchronous on `stream` unless the workspace has to grow.  The handle
 * keeps one plan of each kind; frt_gcc_phat runs the one the last accepted length chose.        */
int frt_gcc_plan(frt_handle h, int length);
/* n_pairs independent channel pairs: d0/d1[p*stride + n].  Inputs are not modified (the
 * reference subtracts the means in place, a side effect that is not reproduced).  L' = L - 1 for
 * odd L (the reference's irfft(W*G) returns L-1 samples; the bin (L-1)/2 counts as Nyquist), else
 * L' = L.  A pair's results are the same bits whatever n_pairs and run to run.
 *   xcorr_dev     NULL or [n_pairs][L']: this frame's Xcorr (correlation.py:41)
 *   smoothed_dev  NULL or [n_pairs][L']: smoothed Xcorr (0.3*X + 0.7*old, delay_estimator.py:134-139),
 *                 written for every non-silent pair.  have_prev: 0 = first frame, nothing to blend
 *                 (a silent pair is marked "no previous" with a NaN in its slot 0); 1 = blend every
 *                 pair with the buffer; 2 = blend the pairs that have had a non-silent frame (no
 *                 NaN marker) -- the widget's `old_Xcorr is not None`; silent pairs keep their buffer
 *   idx_dev/val_dev [n_pairs]: i = argmax |Xs| and Xs[i] (delay_estimator.py:141-146); pairs
 *                 with a constant input (std == 0) give (0, 0) as in delay_estimator.py:129-131,164-167 */
int frt_gcc_phat(frt_handle h, const float *d0_dev, const float *d1_dev, int64_t stride,
                 int n_pairs, float *xcorr_dev, float *smoothed_dev, int have_prev, int *idx_dev,
                 float *val_dev, void *stream);
/* 1 when frt_gcc_plan runs `length` on the shared-memory kernel (even, 2^a 3^b 5^c, <= 28160),
 * else 0.  Pure host arithmetic (needs no GPU or handle).                                       */
int frt_gcc_fits(int length);
/* Pair table for frt_gcc_phat_pairs: pair p correlates channel pairs_host[2p] (the widget's
 * channel 0, d0) with channel pairs_host[2p+1] (d1) of an n_channels-row input.  Indices are
 * checked here (0 <= i, j < n_channels; i == j and repeated pairs are allowed); a refused call
 * keeps the previous table.  Written between device-wide synchronisations like the other setters. */
int frt_gcc_set_pairs(frt_handle h, int n_channels, const int *pairs_host, int n_pairs);
/* GCC-PHAT, smoothing and peak pick of every pair in the table, on x[c*stride + n], c < n_channels,
 * n < L (the current frt_gcc_plan length).  Outputs, have_prev, silent-pair rules and L' exactly as
 * frt_gcc_phat, indexed by pair.  Each channel is mean-removed, windowed and transformed once:
 * channels 2k and 2k+1 share one complex transform (an odd last channel is packed with zeros), so
 * with the table (0,1), (2,3), ... the outputs are the same bits as frt_gcc_phat(x[0::2], x[1::2]).
 * The per-channel spectra take a grow-only workspace of about 8 * n_channels * (L'/2+1) bytes;
 * the Bluestein route also uses frt_gcc_phat's workspace for the transforms.  FRT_ESTATE without a
 * table or a plan.                                                                                 */
int frt_gcc_phat_pairs(frt_handle h, const float *x_dev, int64_t stride, float *xcorr_dev,
                       float *smoothed_dev, int have_prev, int *idx_dev, float *val_dev, void *stream);
/* frt_gcc_phat over n_frames frames of every pair in one call, with each frame's result kept: frame f
 * of pair p is d0/d1[p*stride + f*frame_stride + n], n < L (frames may overlap; the widget's hop is
 * L/2).  The frames run in order through the smoothing: have_prev applies to frame 0 as in
 * frt_gcc_phat, and a later frame blends once its pair has had a non-silent frame (have_prev = 2's
 * rule).  smoothed_dev [n_pairs][L'] is required; it ends holding the state after the last frame.
 * Outputs, each [n_frames][n_pairs]:
 *   idx_dev/val_dev  the frame's argmax |Xs| (first maximum) and Xs there;
 *   std_dev          the population standard deviation of the frame's smoothed row, in double
 *                    (numpy.std(smoothed_Xcorr), delay_estimator.py:147).
 * A pair silent in a frame (a constant input) gives (0, 0, 0) and keeps its smoothing row.  idx, val
 * and the final smoothed buffer are the same bits as n_frames frt_gcc_phat calls, one per frame.
 * Frames run in groups within a grow-only workspace of about 4*L' + 24*ceil(L'/2048) bytes per pair
 * and frame, kept within 2 GiB (one frame at least); the Bluestein route also uses frt_gcc_phat's
 * workspace, frame by frame.  n_frames = 0 or n_pairs = 0 does nothing; frame_stride >= 1 when
 * n_frames > 1.                                                                                    */
int frt_gcc_phat_frames(frt_handle h, const float *d0_dev, const float *d1_dev, int64_t stride,
                        int64_t frame_stride, int n_frames, int n_pairs, float *smoothed_dev,
                        int have_prev, int *idx_dev, float *val_dev, double *std_dev, void *stream);
/* frt_gcc_phat_pairs over n_frames frames: frame f of channel c is x[c*stride + f*frame_stride + n].
 * Everything else as frt_gcc_phat_frames, indexed [n_frames][table entry]; each channel of each frame
 * is transformed once.  On the shared-memory route the workspace also holds the frames' spectra,
 * about 8 * n_channels * (L/2+1) bytes per frame.  With the table (0,1), (2,3), ... the results are
 * the same bits as frt_gcc_phat_frames(x[0::2], x[1::2]).                                           */
int frt_gcc_phat_pairs_frames(frt_handle h, const float *x_dev, int64_t stride, int64_t frame_stride,
                              int n_frames, float *smoothed_dev, int have_prev, int *idx_dev,
                              float *val_dev, double *std_dev, void *stream);

/* ---------------------------------------------------------------- N-fold decimation
 * Stands behind `decimate_multiple(Ndec, bdec, adec, x, zis)` (friture/signal/decimate.py:45-71),
 * the 48 kHz -> 12 kHz pre-stage of the delay estimator (friture/delay_estimator.py:53-59,97-98):
 * n_stages x (order-12 elliptic low-pass as 6 float32 sections, keep even samples), state carried
 * across calls.  n_samples % 256 == 0; out holds n_samples >> n_stages samples per channel.      */
int frt_decimate_plan(frt_handle h, int n_channels, int n_stages, const double *sos_dec);
int frt_decimate_process(frt_handle h, const float *x_dev, int64_t x_stride, int64_t n_samples,
                         float *out_dev, int64_t out_stride, void *stream);

/* ---------------------------------------------------------------- spectrum widget reductions
 * The per-tick numeric work of Spectrum_Widget.handle_new_data behind the STFT
 * (friture/spectrum.py:158-181): smoothing across the tick's frames
 * (exp_smoothed_value_2d, friture/signal/exp_smoothing.py:59-107, alpha from spectrum.py:196-218),
 * 10*log10(sp+1e-30) + weighting (spectrum.py:95-101,171), arg-max (spectrum.py:175) and the
 * 3-harmonic product spectrum arg-max (spectrum.py:103-123,179-181).
 *   power_dev [C][n_frames][nbins] (strides in floats), disp_dev [C][nbins] smoothed power in/out
 *   (the widget's dispbuffers1), weight_dev [nbins] dB offsets or NULL, db_dev [C][nbins],
 *   fmax_idx_dev / pitch_idx_dev [C].                                                          */
int frt_spectrum_reduce(frt_handle h, const float *power_dev, int64_t stride_c, int64_t stride_f,
                        int n_channels, int n_frames, int nbins, float alpha, float *disp_dev,
                        const float *weight_dev, float *db_dev, int *fmax_idx_dev,
                        int *pitch_idx_dev, void *stream);

/* The same tick in the widget's dual-channel measurement mode (friture/spectrum.py:141-182 with
 * dual_channels set and two input channels): per pair, the reference channel (channel 0, sp1) and
 * the measurement channel (channel 1, sp2) are both smoothed across the tick's frames, the output
 * is the transfer function 10*log10(sp2+1e-30) - 10*log10(sp1+1e-30) with no weighting
 * (spectrum.py:168-169), formed in double and stored as float32, fmax_idx its arg-max
 * (spectrum.py:175) and pitch_idx the harmonic-product arg-max of sp1 (spectrum.py:180-181).
 *   power1_dev / power2_dev [P][n_frames][nbins] with the same strides (in floats),
 *   disp1_dev / disp2_dev [P][nbins] smoothed power in/out (the widget's dispbuffers1 and
 *   dispbuffers2), db_dev [P][nbins], fmax_idx_dev / pitch_idx_dev [P].  Argument checks as for
 *   frt_spectrum_reduce; n_pairs == 0 does nothing.                                             */
int frt_spectrum_reduce_dual(frt_handle h, const float *power1_dev, const float *power2_dev,
                             int64_t stride_c, int64_t stride_f, int n_pairs, int n_frames,
                             int nbins, float alpha, float *disp1_dev, float *disp2_dev,
                             float *db_dev, int *fmax_idx_dev, int *pitch_idx_dev, void *stream);

/* n_ticks consecutive ticks of frames_per_tick frames each in one call, each tick's result kept: tick
 * r covers frames r*frames_per_tick .. (r+1)*frames_per_tick - 1 of power_dev [C][n_frames][nbins].
 * db_dev [C][n_ticks][nbins] (contiguous) or NULL for no dB; fmax_idx_dev / pitch_idx_dev
 * [n_ticks][C].  Every row, and disp_dev afterwards, are the same bits as n_ticks
 * frt_spectrum_reduce calls, one per tick.  Argument checks as frt_spectrum_reduce, with
 * frames_per_tick in 1..8192; n_ticks == 0 or n_channels == 0 does nothing.  The ticks run in groups
 * within a grow-only workspace of 4*C*nbins bytes per tick, kept within 256 MiB (one tick at least);
 * such a call is asynchronous on `stream` unless the workspace has to grow.                       */
int frt_spectrum_reduce_ticks(frt_handle h, const float *power_dev, int64_t stride_c,
                              int64_t stride_f, int n_channels, int frames_per_tick, int n_ticks,
                              int nbins, float alpha, float *disp_dev, const float *weight_dev,
                              float *db_dev, int *fmax_idx_dev, int *pitch_idx_dev, void *stream);

/* frt_spectrum_reduce_dual over n_ticks ticks, as frt_spectrum_reduce_ticks over
 * frt_spectrum_reduce: db_dev [P][n_ticks][nbins] or NULL, fmax_idx_dev / pitch_idx_dev
 * [n_ticks][P], disp1_dev and disp2_dev the same bits afterwards as n_ticks frt_spectrum_reduce_dual
 * calls.  The workspace holds both states' rows, 8*P*nbins bytes per tick.                       */
int frt_spectrum_reduce_dual_ticks(frt_handle h, const float *power1_dev, const float *power2_dev,
                                   int64_t stride_c, int64_t stride_f, int n_pairs,
                                   int frames_per_tick, int n_ticks, int nbins, float alpha,
                                   float *disp1_dev, float *disp2_dev, float *db_dev,
                                   int *fmax_idx_dev, int *pitch_idx_dev, void *stream);

/* The spectrum widget's ticks straight from the frames (friture/spectrum.py:125-184): frame f of
 * channel c, x_dev[c*x_stride + f*hop .. + n_fft) with the frt_stft_plan'ed size, is transformed to its
 * FRT_STFT_POWER column, which stays on chip and goes straight into the smoothing of
 * frt_spectrum_reduce; a channel's frames are smoothed in order.  Tick r ends at frame
 * tick_end_dev[r] (exclusive): tick_end_dev is int32 [n_ticks] on the device, strictly ascending,
 * tick_end_dev[n_ticks-1] == n_frames, at most 8192 frames per tick (the reference's 8192-tap kernel).
 * The library does not read it on the host: an array that breaks these rules gives rows that mean
 * nothing, not a fault.  At each tick's end the state is rounded to float32 and the tick's outputs
 * are written:
 *   db_dev[c*db_stride_c + r*db_stride_r + k] = 10*log10(sp + 1e-30) + weight[k] (db_dev may be NULL),
 *   imax_dev[r*C + c] its first arg-max, ipitch_dev[r*C + c] the harmonic-product arg-max.
 * Rows, indices and disp_dev afterwards are the same bits as frt_stft_process(FRT_STFT_POWER) on the
 * same frames followed by frt_spectrum_reduce one tick at a time.  disp_dev [C][n_fft/2+1] is read
 * once and written once; weight_dev [n_fft/2+1] dB or NULL.  Needs hop >= 1, alpha in (0, 1],
 * 1 <= n_ticks <= n_frames and, with db_dev, db_stride_r >= n_fft/2+1; n_channels == 0 or
 * n_frames == 0 is a no-op.  No workspace.                                                        */
int frt_spectrum_frames(frt_handle h, const float *x_dev, int64_t x_stride, int n_channels,
                        int64_t n_frames, int hop, const int *tick_end_dev, int n_ticks, float alpha,
                        float *disp_dev, const float *weight_dev, float *db_dev, int64_t db_stride_c,
                        int64_t db_stride_r, int *imax_dev, int *ipitch_dev, void *stream);

/* frt_spectrum_frames in the dual-channel measurement mode (friture/spectrum.py:125-184 with
 * dual_channels set): pair p's reference frames start at x1_dev + p*x_stride + f*hop, its
 * measurement frames at x2_dev + p*x_stride + f*hop; both are smoothed (disp1_dev, disp2_dev
 * [P][n_fft/2+1]), the dB row is the transfer function of frt_spectrum_reduce_dual and the pitch
 * comes from the reference.  The same bits as frt_stft_process(FRT_STFT_POWER) on both rows followed
 * by frt_spectrum_reduce_dual one tick at a time.  Checks as frt_spectrum_frames.                  */
int frt_spectrum_frames_dual(frt_handle h, const float *x1_dev, const float *x2_dev, int64_t x_stride,
                             int n_pairs, int64_t n_frames, int hop, const int *tick_end_dev,
                             int n_ticks, float alpha, float *disp1_dev, float *disp2_dev,
                             float *db_dev, int64_t db_stride_c, int64_t db_stride_r, int *imax_dev,
                             int *ipitch_dev, void *stream);

/* ---------------------------------------------------------------- plotted curves and peak hold
 * The last numeric step of the spectrum and octave widgets: SpectrumPlotWidget.setdata and
 * compute_peaks (friture/spectrumPlotWidget.py:122-200), HistPlot.setdata and compute_peaks
 * (friture/histplot.py:77-130), with the linear vertical scale of
 * friture/plotting/coordinateTransform.py:62-83.  Per channel, the peak state machine is run over
 * the n_steps dB vectors in order (rise when peak < y: peak = y, peak_int = 1, decay = d0; else
 * when peak_int < 0.2: peak += decay, decay += d0; else peak_int *= 0.975), in double.  Then, for
 * the last step only: scaled_y = 1 - (y - spec_min) / (spec_max - spec_min) (1 when the range is
 * empty), z = (y - spec_min) / (|max(y) - spec_min| + 1e-3), scaled_peak = 1 - toScreen(peak),
 * z_peak = peak_int, all rounded once to float32.
 *   y_dev [C][n_steps][nbins] dB (strides in floats, >= 0; y is only read, so rows may overlap);
 *   spec_min <= spec_max (the widget's setspecrange sorts them); d0 the decay step
 *   20*log10(1 - 3e-6)*5000, computed by the caller.
 *   peak_dev / peak_int_dev / decay_dev [C][nbins] state in/out; reset != 0 starts it from the
 *   widget's reset (-500, 0, d0) instead of reading it.  peaks == 0: compute_peaks is skipped, the
 *   state and the peak outputs are neither read nor written (they may be NULL).
 *   scaled_y_dev / z_dev / scaled_peak_dev / z_peak_dev [C][nbins] float32.                      */
int frt_plot_curves(frt_handle h, const float *y_dev, int64_t stride_c, int64_t stride_s,
                    int n_channels, int n_steps, int nbins, double spec_min, double spec_max,
                    double d0, int peaks, int reset, double *peak_dev, double *peak_int_dev,
                    double *decay_dev, float *scaled_y_dev, float *z_dev, float *scaled_peak_dev,
                    float *z_peak_dev, void *stream);

/* ---------------------------------------------------------------- spectrogram display chain
 * The Transform_Pipeline behind the spectrogram (friture/spectrogram.py:161-169): scaling of
 * dB + weighting to [0,1] (spectrogram.py:127-129), Frequency_Resampler.push
 * (friture/signal/frequency_resampler.py:67-83), Online_Linear_2D_resampler.push
 * (friture/signal/online_linear_2D_resampler.py:61-97) and Color_Transform.push
 * (friture/signal/color_tranform.py:48-51), fused.  The host supplies the screen-row table
 * (row_i0/row_t: bin index and fraction of every screen row on the chosen frequency scale) and,
 * per output column, the input column it is drawn from and the weight of the previous input
 * column (the resampler's index bookkeeping).  db_dev [C][n_frames][nbins] log-power columns,
 * old_data_dev [C][height] carried last column (in/out), lut_dev [256] 0xAARRGGBB,
 * pixels_dev [C][height][n_out].                                                              */
int frt_display_columns(frt_handle h, const float *db_dev, int64_t stride_c, int64_t stride_f,
                        int n_channels, int n_frames, int nbins, const float *weight_dev,
                        float spec_min, float spec_max, const int *row_i0_dev,
                        const float *row_t_dev, int height, const int *out_col_dev,
                        const float *out_a_dev, int n_out, float *old_data_dev,
                        const uint32_t *lut_dev, uint32_t *pixels_dev, void *stream);
/* The same time resampling, clip and colour look-up on rows already on the screen grid
 * (frt_stft_screen_rows): rows_dev [C][n_frames][height] (strides in floats), the rest as in
 * frt_display_columns.  Gives frt_display_columns' pixels and carried column bit for bit when the
 * rows come from the same frames and screen-row table.                                         */
int frt_display_rows(frt_handle h, const float *rows_dev, int64_t stride_c, int64_t stride_f,
                     int n_channels, int n_frames, int height, const int *out_col_dev,
                     const float *out_a_dev, int n_out, float *old_data_dev, const uint32_t *lut_dev,
                     uint32_t *pixels_dev, void *stream);

/* ---------------------------------------------------------------- level meter
 * Levels_Widget.handle_new_data (friture/levels.py:84-131) for every one of C channels, with the
 * ballistic peak of its display (BallisticPeak.peak_iec, friture/ballistic_peak.py:43-66, of
 * dB_to_IEC(max(level_max, level_rms)), friture/iec.py).  Each buffer of `buffer` samples is one
 * handle_new_data call.  frt_levels_plan takes the buffer length, the tail of the widget's
 * smoothing kernel, weights_host[j] = kernel[Nk - buffer + j] (exp_smoothing.py:41-51), alpha, decay =
 * (1 - alpha)^buffer and keep = 1 - alpha2 (levels.py:58-74), all computed by the caller as the widget
 * does.  The per-channel state (old_rms, old_max, the ballistic peak, its decay factor and hold
 * counter) starts from the widget's (1e-30, 1e-30, 0, 1 - 3e-6/500, 0); a plan with the planned
 * channel count keeps it.  frt_levels_reset starts it again.                                  */
int frt_levels_plan(frt_handle h, int n_channels, int buffer, const double *weights_host, double alpha,
                    double decay, double keep);
int frt_levels_reset(frt_handle h);
/* The state after the last call: state_host [4][C] double (old_rms, old_max, peak, decay factor),
 * hold_host [C] int.  Waits for the device.                                                     */
int frt_levels_state(frt_handle h, double *state_host, int *hold_host);
/* n_buffers consecutive buffers of every channel, x_dev[c*x_stride + r*buffer .. + buffer), in one
 * launch: rms_db_dev / max_db_dev / peak_iec_dev [C][n_buffers] double get level_rms, level_max and
 * peak_iec after each buffer.  max|x|, the peak state and the ballistic peak are the widget's
 * double arithmetic bit for bit; the weighted sum of x^2 and log10 may differ from NumPy's by
 * rounding.  A NaN sample acts as in the widget: max|x| is NaN, so old_max takes its decay step,
 * and old_rms and level_rms become NaN.  x_stride >= n_buffers*buffer unless C == 1.            */
int frt_levels_process(frt_handle h, const float *x_dev, int64_t x_stride, int n_buffers, double *rms_db_dev,
                       double *max_db_dev, double *peak_iec_dev, void *stream);

/* ---------------------------------------------------------------- long-term levels
 * LongLevelWidget.handle_new_data and setresptime (friture/longlevels.py:150-230) for C channels:
 * per block of 2^n_dec samples, x^2 through n_dec stages of decimate (friture/signal/decimate.py:
 * 27-42: bdec_host, the 11 taps of gauss(11, 2), then every other output) and the 41-tap FIR
 * bfir_host = gauss(41, 8), one linear level per block, and 10*log10(max(level, 1e-150)).  The
 * filters are lfilter_float64_1D with a = [1, 0, ...] (friture/signal/lfilter.py:132-139) evaluated in
 * its order, so the linear level is the same bits.  The plan and frt_longlevels_reset zero the
 * filter state, as setresptime does (longlevels.py:207-221).  n_dec in 1..13.                   */
int frt_longlevels_plan(frt_handle h, int n_channels, int n_dec, const double *bdec_host,
                        const double *bfir_host);
int frt_longlevels_reset(frt_handle h);
/* n_blocks consecutive blocks, x_dev[c*x_stride + b*2^n_dec .. + 2^n_dec), in one launch:
 * level_dev / db_dev [C][n_blocks] double get each block's linear level and dB, and
 * ring_dev[c*ring_len + (ring_pos + b) % ring_len] (float32) its dB: the widget's level ring
 * buffer (friture/ringbuffer.py:39-61) whose offset is ring_pos.  A NaN or infinite sample acts as
 * in the widget: its transposed-form filters take y*0 into their state, so from the sample's block
 * on the channel's levels are NaN (max(level, 1e-150) keeps NaN) until the next plan or reset.
 * x_stride >= n_blocks*2^n_dec unless C == 1.                                                  */
int frt_longlevels_process(frt_handle h, const float *x_dev, int64_t x_stride, int n_blocks, double *level_dev,
                           double *db_dev, float *ring_dev, int64_t ring_len, int64_t ring_pos, void *stream);
/* The plotted curve (longlevels.py:181-187): scaled_dev [C][length] float32 = clip(1 - (l -
 * level_min) / (level_max - level_min), 0, 1) of the last `length` ring values before offset
 * ring_pos (RingBuffer.data, ringbuffer.py:63-78), in double.  length <= ring_len.              */
int frt_longlevels_history(frt_handle h, const float *ring_dev, int64_t ring_len, int64_t ring_pos,
                           int n_channels, int length, double level_min, double level_max,
                           float *scaled_dev, void *stream);

/* ---------------------------------------------------------------- scope
 * Scope_Widget.handle_new_data (friture/scope.py:78-133) for n_scopes scopes of n_ch (1 or 2)
 * channels: row s*n_ch + k of x_dev is channel k of scope s, x_stride floats apart.  Tick r (0 <=
 * r < n_ticks) reads the `need` samples that end at column lead + (r+1)*buffer, need = 2*width in
 * trigger mode (trigger != 0) and width in scrolling mode; lead + buffer >= need.  The caller stages
 * each row as the widget's ring buffer reads it, so column c is stream index origin + c.
 *   trigger: level = max(s) * 2 / 3 of the search window s = d[width/2 .. width/2 + width) of
 *     channel 0, a NaN anywhere making it NaN; the first i with s[i] < level <= s[i+1], compared in
 *     double; the tick draws 2*(width/2) samples from d[i].  No such i: the tick draws nothing.
 *   scrolling: the tick draws the last width samples.
 * start_dev [n_scopes][n_ticks] int64 gets the stream index each tick's drawn window starts at
 * (negative when it reaches into the zeros before the stream), or INT64_MIN when it drew nothing.
 * For each scope whose ticks drew, the last one that drew gives curve_dev[(s*n_ch + k)*curve_stride
 * + j] = float32(1 - (y + 1) / 2) in double (scope.py:128-133), j < its point count, and drawn_dev[s]
 * = timerange; the other scopes' curves and drawn_dev are left alone.  Two launches; every
 * refusal comes before the first.  x_stride >= lead + n_ticks*buffer and curve_stride >= the point
 * count unless n_scopes*n_ch == 1.  In trigger mode width/buffer is at most 25 000.             */
int frt_scope_process(frt_handle h, const float *x_dev, int64_t x_stride, int n_scopes, int n_ch, int64_t lead,
                      int n_ticks, int buffer, int width, int trigger, int64_t origin, int64_t *start_dev,
                      float *curve_dev, int64_t curve_stride, double timerange, double *drawn_dev,
                      void *stream);

#ifdef __cplusplus
}
#endif
#endif /* FRT_H */
