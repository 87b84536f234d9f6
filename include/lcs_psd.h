/* lcs_psd.h - C ABI of the Welch power spectrum of a wideband recording (DESIGN.md section 4.8), liblcs_psd.so.
 *
 * The spectrum is a module of its own on top of liblcs_b200.so: it takes an lcs_ctx of that library (device, stream,
 * launch count, error text) and follows its conventions (plain C, every function returns an lcs_status and never throws,
 * lcs_last_error() gives the message, no CPU fallback).  Link with -llcs_psd -llcs_b200.
 */
#ifndef LCS_PSD_H
#define LCS_PSD_H

#include "lcs_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* An lcs_psd accumulates Welch's power spectral density over a stream pushed in pieces of any size.
 *   fs_in   an integer number of Hz (within 1e-6), 0 < fs_in <= 250 MHz.
 *   input   iq_format LCS_IQ_CI16, CS8, CU8 or CF32, converted as in section 4.7; sample m counted from the stream start.
 *   nfft    N, a power of two, 64 <= N <= 65536.  Segment s covers samples [s*N/2, s*N/2 + N) (hop N/2, 50 % overlap)
 *           and counts once its last sample has been pushed; the host keeps at most N - 1 samples of carry.
 *   window  periodic Hann w[n] = 0.5 - 0.5 cos(2 pi n/N), computed in double and kept as float.
 *   estimate P[k] = sum_s |X_s[k]|^2 / (S * fs_in * sum_n w[n]^2), X_s[k] = sum_n w[n] x[s*N/2 + n] exp(-j2pi kn/N), over
 *           the S segments accumulated; full-scale^2 per Hz.  This is scipy.signal.welch(x, fs, window='hann',
 *           nperseg=N, noverlap=N//2, detrend=False, return_onesided=False, scaling='density') followed by fftshift.
 *   order   psd[i] is bin k = (i + N/2) mod N, at frequency fc_in + (i - N/2) * fs_in / N (fftshift order).
 *   sums    each segment's |X_s[k]|^2 (FP32 FFT) is added to an FP64 accumulator per bin in segment order, so any
 *           sequence of pushes gives bitwise the PSD of one push. */
typedef struct lcs_psd lcs_psd;
lcs_status lcs_psd_create(lcs_ctx* ctx, double fs_in, int iq_format, uint32_t nfft, lcs_psd** out);
void lcs_psd_destroy(lcs_psd* psd);
/* Push n_in samples ([n_in][2] in the handle's format, host memory).  Every segment they complete is computed; large
 * pushes run in launches that bound the device scratch. */
lcs_status lcs_psd_push(lcs_psd* psd, const void* iq_host, uint32_t n_in);
/* P over the segments completed since the last read (psd [nfft], fftshift order) and their number S; then the
 * accumulator restarts (the carry stays).  S = 0 gives zeros.  Reading once at the end gives the PSD of the whole stream,
 * reading every few segments the rows of a spectrogram. */
lcs_status lcs_psd_read(lcs_psd* psd, double* out, uint64_t* n_segments);
/* Summed device time of the spectrum's kernels (CUDA events around the kernels of each launch chunk, ms) and the number
 * of kernels launched since the last read; resets both. */
lcs_status lcs_psd_timing_read(lcs_psd* psd, double* kernel_ms, uint64_t* launches);

#ifdef __cplusplus
}
#endif
#endif /* LCS_PSD_H */
