/* lcs_meas.h - C ABI of the per-cell RSRP / RSRQ / SINR measurement (DESIGN.md section 4.9), liblcs_meas.so.
 *
 * The measurement is a module of its own on top of liblcs_b200.so: it takes an lcs_ctx of that library (device, stream,
 * launch count, error text) and follows its conventions (plain C, every function returns an lcs_status and never throws,
 * lcs_last_error() gives the message, no CPU fallback).  Link with -llcs_meas -llcs_b200.
 */
#ifndef LCS_MEAS_H
#define LCS_MEAS_H

#include "lcs_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* What one found cell measures from the cell-specific reference signals (CRS) of its central six resource blocks.
 *   grid    Y [n_ofdm][72] is what lcs_extract_tfg returns for a copy of the cell whose freq_fine is freq_superfine, at
 *           the cell's fc_requested / fc_programmed and the call's fs_programmed.  Its 1/sqrt(128) DFT scaling makes
 *           |Y|^2 / 128 the per-sample power of one resource element.  Row s is symbol s mod n_symb of slot s / n_symb.
 *   pairs   for port p, h = Y conj(r) at each of its CRS resource elements, r the cell's CRS (36.211 6.10.1, 6 RB).  Each
 *           is paired with the RE of the same port, symbol within the slot and subcarrier two slots (1 ms) later, the one
 *           interval at which ports 0-3 all repeat on the same subcarriers; every pair wholly inside the grid is used:
 *           n_pairs = 2880 for ports 0 and 1 and 1440 for ports 2 and 3 (the grid has 122 slots in either CP).
 *   sums    C_p = mean h_a conj(h_b), T_p = mean (|h_a|^2 + |h_b|^2) / 2, S_p = |C_p|, N_p = T_p - S_p, in FP64 in one fixed
 *           order, so a cell's result does not depend on the other cells of the call or on the run.  |C_p| makes the
 *           estimate blind to a residual frequency offset and to a common phase.
 *   results rsrp[p] = S_p / 128 and noise[p] = N_p / 128, in capture full-scale^2 per resource element; rssi = the mean,
 *           over the grid's OFDM symbols that carry port-0 CRS, of sum_{k<72} |Y_k|^2 / 128; rsrq = 6 rsrp[0] / rssi;
 *           sinr[p] = S_p / N_p, or +inf when N_p <= 0.  Ports at or above n_ports give NaN and n_pairs 0.
 *   model   the channel is taken as quasi-static over 1 ms: Doppler decorrelation lowers S and counts as noise.  Other
 *           cells' CRS that collide with this cell's (equal PCI mod 3) count as noise too, which is what SINR means here. */
typedef struct lcs_cell_meas {
  double rsrp[4];
  double noise[4];
  double sinr[4];
  double rssi, rsrq;
  uint32_t n_pairs[4];
} lcs_cell_meas;

typedef struct lcs_meas lcs_meas;
lcs_status lcs_meas_create(lcs_ctx* ctx, lcs_meas** out);
void lcs_meas_destroy(lcs_meas* meas);
/* Measure n_cells found cells in one grid launch and one measurement launch, then wait for them.
 *   iq          [n_ch][n_cap][2] in iq_format LCS_IQ_CU8, CF32 or C128; in device memory when on_device is non-zero
 *               (16-byte aligned, read in place; writes of other streams must be complete), host memory otherwise.
 *   cells[i]    as the search returns it: cp_type 1 or 2, n_id_1 in [0, 167], n_id_2 in [0, 2], n_ports 1, 2 or 4,
 *               frame_start and freq_superfine finite, fc_requested and fc_programmed finite and positive.
 *   ch[i]       the channel (row of iq) cell i was found in, < n_ch.
 *   out         [n_cells] results, in the order of cells.
 * Every argument is checked before any launch: a null pointer, an unknown format, n_ch or n_cap 0, n_cap > 2^31 - 1, a
 * non-positive fs_programmed, or a cell whose fields are out of range or whose grid does not fit in [0, n_cap) returns
 * LCS_ERR_ARG (naming the cell).  n_cells = 0 launches nothing. */
lcs_status lcs_meas_cells(lcs_meas* meas, const void* iq, int iq_format, int on_device, uint32_t n_ch, uint32_t n_cap,
                          const lcs_cell* cells, const uint32_t* ch, uint32_t n_cells, double fs_programmed,
                          lcs_cell_meas* out);
/* Summed device time of the measurement's kernels (CUDA events around both launches of each call, ms) and the number of
 * kernels launched since the last read (two per call with cells); resets both. */
lcs_status lcs_meas_timing_read(lcs_meas* meas, double* kernel_ms, uint64_t* launches);

#ifdef __cplusplus
}
#endif
#endif /* LCS_MEAS_H */
