/* lcs_cir.h - C ABI of the power delay profile of found cells over their whole carrier (DESIGN.md section 4.11),
 * liblcs_cir.so.
 *
 * The measurement is a module of its own on top of liblcs_b200.so: it takes an lcs_ctx of that library (device, stream,
 * launch count, error text) and follows its conventions (plain C, every function returns an lcs_status and never throws,
 * lcs_last_error() gives the message, no CPU fallback).  Link with -llcs_cir -llcs_b200.
 *
 * It transforms the CRS of each cell's whole OFDM grid, the grid of lcs_carrier.h, into the cell's channel impulse
 * response, and reports per antenna port the power delay profile (PDP), the delay of its strongest and of its first
 * path, its mean delay and RMS delay spread, and the arrival time of the cell's frame in the recording.  All cells of one
 * recording share its sample clock, so the difference of two cells' frame_arrival is their timing offset.
 */
#ifndef LCS_CIR_H
#define LCS_CIR_H

#include "lcs_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Cells per chunk of one lcs_cir_cells call; each chunk makes LCS_CIR_LAUNCHES_PER_CHUNK kernel launches (the carrier
 * grid, then the delay transform with the statistics), so a call with n cells launches 2 * ceil(n / 32) kernels. */
#define LCS_CIR_CHUNK 32
#define LCS_CIR_LAUNCHES_PER_CHUNK 2
/* The delay grid: tap j < LCS_CIR_TAPS is tau_j = (j - 64) T_s, T_s = 1 / 30.72 MHz, so -2.083 us .. +8.301 us. */
#define LCS_CIR_TAPS 320
/* Taps within this many dB of the PDP's peak enter the statistics. */
#define LCS_CIR_RANGE_DB 20.0

/* What one found cell measures.  With R = n_rb_dl and the grid Y[t][c] of lcs_carrier.h (the same windows, mixer and
 * scaling):
 *   1. For port p and each OFDM symbol t that carries its CRS, h_t[m] = Y[t][6 m + s_t] conj(r_t[m]) for m < 2R, s_t the
 *      port's shift in that symbol; b_t[m] is the subcarrier of that column (c - 6R below DC, c - 6R + 1 above).
 *   2. The taper w[m] = sin^2(pi (m + 1/2) / 2R); its sum is R, and its -31 dB sidelobes stay out of a 20 dB range.
 *   3. c_t(tau_j) = sum_m w[m] h_t[m] exp(+j2pi b_t[m] (j - 64) / 2048), j < LCS_CIR_TAPS: a direct DFT at the true
 *      subcarriers (15 kHz T_s = 1/2048, so every twiddle is an exact 2048-th root of unity, and the DC gap needs nothing).
 *   4. Pairs as in lcs_carrier.h: the same port and symbol of the slot, two slots (1 ms) apart, n_pairs of them per tap.
 *      S_j = |mean c_a conj(c_b)|, T_j = mean (|c_a|^2 + |c_b|^2) / 2, pdp[p][j] = S_j / (128 R^2): a single path of
 *      power P on a tap reads P, as lcs_carrier_meas.rsrp reads it on a flat channel.  |.| makes the PDP blind to a
 *      residual frequency offset; the mean of the products has no noise term, but its |.| over a finite number of pairs
 *      leaves a small positive floor that falls as 1/sqrt(n_pairs), and floor[p] is the noise per tap beside it: the mean
 *      over taps of (T_j - S_j) / (128 R^2).
 *   5. Statistics per port, FP64, in ascending j: j* is the first arg-max of pdp and peak_delay = tau_j*; K = {j : pdp_j
 *      >= pdp_j* 10^(-LCS_CIR_RANGE_DB / 10)}, n_taps = |K|; first_delay is the smallest j in K that is a local maximum
 *      (not below either neighbour, neighbours outside the grid counting as -inf), refined by the parabolic vertex
 *      offset delta = (p- - p+) / (2 (p- - 2 p0 + p+)) clipped to +-1/2 (0 at the grid's ends or when the three are
 *      equal): tau_j + delta T_s; mean_delay and rms_spread are the pdp-weighted mean and RMS spread (two passes) of tau
 *      over K.
 *   6. frame_arrival = D frame_start / fs_in + first_delay[0], D = fs_in / 1.92 MHz: seconds from the recording's first
 *      sample.  The DFT windows start frame_start plus one cyclic prefix into the frame, so a path d after frame_start
 *      sits at tau = d, and frame_arrival does not depend on where the search put frame_start.  The search's frame_start
 *      carries a 2-sample advance at 1.92 Msps, so a found cell's first path reads about +1.04 us.
 *   7. Ports at or above n_ports are NaN, with counts 0.
 * Limits: a path outside [-2.083, 8.301) us folds into the window, since one port's CRS comb in one symbol repeats in
 * delay every 1 / 90 kHz = 11.1 us.  A single path's rms_spread is not zero: it is the width of the taper's main lobe
 * inside the 20 dB range, which shrinks as 1 / R. */
typedef struct lcs_cir_meas {
  double pdp[4][LCS_CIR_TAPS];                 /* per port, in the units of lcs_carrier_meas.rsrp */
  double floor[4];                             /* mean over taps of (T_j - S_j) / (128 R^2) */
  double peak_delay[4], first_delay[4], mean_delay[4], rms_spread[4];   /* seconds */
  double frame_arrival;                        /* seconds from recording sample 0, from port 0 */
  uint32_t n_pairs[4];                         /* symbol pairs per tap: 240 for ports 0-1, 120 for ports 2-3 */
  uint32_t n_taps[4];                          /* |K| */
} lcs_cir_meas;

typedef struct lcs_cir lcs_cir;
lcs_status lcs_cir_create(lcs_ctx* ctx, lcs_cir** out);
void lcs_cir_destroy(lcs_cir* cir);
/* Measure n_cells found cells on the wideband recording they were found in, chunk by chunk, then wait for them.  The
 * arguments, the accepted formats and rates, the rules a cell must fit and the errors are those of lcs_carrier_cells
 * (include/lcs_carrier.h): iq [n_in][2] in LCS_IQ_CI16, CS8, CU8 or CF32 at fs_in = D * 1.92 MHz, D in {2, 4, 8, 16, 32},
 * in device memory when on_device is non-zero (16-byte aligned), host memory otherwise.  Every argument is checked before
 * any launch; a bad one returns LCS_ERR_ARG (naming the cell).  out[i] is that of cells[i]; n_cells = 0 launches nothing.
 * A cell's record is bitwise the same whatever else the call measures. */
lcs_status lcs_cir_cells(lcs_cir* cir, const void* iq, int iq_format, int on_device, uint64_t n_in, double fs_in,
                         double fc_in, const lcs_cell* cells, uint32_t n_cells, double fs_programmed, lcs_cir_meas* out);
/* Summed device time of the measurement's kernels (CUDA events around the launches of each chunk, ms) and the number of
 * kernels launched since the last read; resets both. */
lcs_status lcs_cir_timing_read(lcs_cir* cir, double* kernel_ms, uint64_t* launches);

#ifdef __cplusplus
}
#endif
#endif /* LCS_CIR_H */
