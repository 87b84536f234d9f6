/* lcs_carrier.h - C ABI of the full-carrier RSRP / RSRQ / SINR measurement of found cells (DESIGN.md section 4.10),
 * liblcs_carrier.so.
 *
 * The measurement is a module of its own on top of liblcs_b200.so: it takes an lcs_ctx of that library (device, stream,
 * launch count, error text) and follows its conventions (plain C, every function returns an lcs_status and never throws,
 * lcs_last_error() gives the message, no CPU fallback).  Link with -llcs_carrier -llcs_b200.
 *
 * Where lcs_meas.h measures a cell from the central six resource blocks of a 1.92 Msps channel, this module takes the
 * cell's whole OFDM grid, all n_rb_dl resource blocks, straight from the wideband recording the cell was found in.
 */
#ifndef LCS_CARRIER_H
#define LCS_CARRIER_H

#include "lcs_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Cells per chunk of one lcs_carrier_cells call; each chunk makes LCS_CARRIER_LAUNCHES_PER_CHUNK kernel launches (the
 * grid and the measurement), so a call with n cells launches 2 * ceil(n / 32) kernels.  The device scratch of a call is
 * the recording (host input only) and one chunk's grids, at most 32 * 366 * 1200 float2 (112 MB). */
#define LCS_CARRIER_CHUNK 32
#define LCS_CARRIER_LAUNCHES_PER_CHUNK 2

/* What one found cell measures from the cell-specific reference signals (CRS) of all its R = n_rb_dl resource blocks.
 * With D = fs_in / 1.92 MHz and N = 128 D:
 *   windows loc_t (t < n_ofdm) are the DFT-window positions of lcs_extract_tfg for the cell with freq_fine =
 *           freq_superfine, in 1.92 Msps samples; window t starts at recording sample q_t = rint(D loc_t), late by
 *           late_t = q_t - D loc_t.
 *   mixer   x~[m] = x[m] exp(-j2pi ((m delta) mod fs_in) / fs_in) exp(j kappa m), m counted from the recording's first
 *           sample, delta = fc_requested - fc_in (an integer number of Hz), kappa = -2pi freq_superfine /
 *           (D fs_programmed k_factor), k_factor = (fc_requested - freq_superfine) / fc_programmed.
 *   grid    Y[t][c] = (sqrt(128) / N) sum_{n<N} x~[q_t + n] exp(-j2pi b n / N) exp(-j2pi late_t b / N), c < 12 R, with
 *           subcarrier b = c - 6R for c < 6R and c - 6R + 1 above (DC skipped), so |Y|^2 / 128 is the per-sample power of
 *           a resource element in the recording's full-scale^2, and the central 72 columns are lcs_meas.h's grid.
 *           Only the OFDM symbols that carry CRS are made: 0 and n_symb - 3 of every slot, and 1 for four ports.
 *   pairs   for port p, h = Y conj(r) at each of its 2R CRS per symbol, r(m') with m' = 110 - R + m on subcarrier
 *           6 m + shift (36.211 6.10.1), paired with the RE of the same port, symbol and subcarrier two slots (1 ms)
 *           later: n_pairs = 480 R for ports 0 and 1 and 240 R for ports 2 and 3.
 *   sums    C = mean h_a conj(h_b), T = mean (|h_a|^2 + |h_b|^2) / 2, S = |C|, N = T - S, over the whole carrier and
 *           over each resource block b (columns 12b .. 12b + 11; RB 0 is the lowest in frequency).  Every sum is FP64 in
 *           one fixed order: a cell's record is bitwise the same on every run, whatever else the call measures, and the
 *           carrier's sums are its RBs' sums added in RB order.
 *   results rsrp[p] = S / 128, noise[p] = N / 128, sinr[p] = S / N (+inf when N <= 0); rssi = the mean, over the symbols
 *           that carry port-0 CRS, of sum_{c<12R} |Y_c|^2 / 128; rsrq = R rsrp[0] / rssi (36.214 5.1.3).  rb_rsrp,
 *           rb_noise and rb_rssi are the same per resource block.  Ports at or above n_ports and RBs at or above R are
 *           NaN, and their pair counts 0. */
typedef struct lcs_carrier_meas {
  double rsrp[4];
  double noise[4];
  double sinr[4];
  double rssi, rsrq;
  double rb_rsrp[4][100];
  double rb_noise[4][100];
  double rb_rssi[100];
  uint32_t n_pairs[4];
  uint32_t n_rb;
} lcs_carrier_meas;

typedef struct lcs_carrier lcs_carrier;
lcs_status lcs_carrier_create(lcs_ctx* ctx, lcs_carrier** out);
void lcs_carrier_destroy(lcs_carrier* carrier);
/* Measure n_cells found cells on the wideband recording they were found in, chunk by chunk, then wait for them.
 *   iq          [n_in][2] samples at fs_in centred on fc_in, in iq_format LCS_IQ_CI16, CS8, CU8 or CF32; in device memory
 *               when on_device is non-zero (16-byte aligned, read in place; writes of other streams must be complete),
 *               host memory otherwise (the span the cells' windows cover is copied to the device).
 *   fs_in       D * 1.92 MHz with D in {2, 4, 8, 16, 32} (3.84 to 61.44 Msps).
 *   cells[i]    as the search returns it: cp_type 1 or 2, n_id_1 in [0, 167], n_id_2 in [0, 2], n_ports 1, 2 or 4,
 *               n_rb_dl in {6, 15, 25, 50, 75, 100}, frame_start and freq_superfine finite, fc_requested and
 *               fc_programmed finite and positive, fc_requested - fc_in an integer number of Hz (within 1e-6).  The cell
 *               must fit: every q_t >= 0 and q_t + N <= n_in, 6 R < 64 D and |fc_requested - fc_in| + 90 kHz R <= fs_in / 2.
 *   out         [n_cells] results, in the order of cells.
 * Every argument is checked before any launch: a null pointer, an unknown format, n_in 0, a rate outside the list, a
 * non-finite fc_in, a non-positive fs_programmed, or a cell out of range or that does not fit returns LCS_ERR_ARG
 * (naming the cell).  n_cells = 0 launches nothing. */
lcs_status lcs_carrier_cells(lcs_carrier* carrier, const void* iq, int iq_format, int on_device, uint64_t n_in,
                             double fs_in, double fc_in, const lcs_cell* cells, uint32_t n_cells, double fs_programmed,
                             lcs_carrier_meas* out);
/* Summed device time of the measurement's kernels (CUDA events around the launches of each chunk, ms) and the number of
 * kernels launched since the last read; resets both. */
lcs_status lcs_carrier_timing_read(lcs_carrier* carrier, double* kernel_ms, uint64_t* launches);

#ifdef __cplusplus
}
#endif
#endif /* LCS_CARRIER_H */
