/* lcs_pcfich.h - C ABI of the control format indicator (CFI) of found cells in every subframe, decoded from their PCFICH
 * over the whole carrier (DESIGN.md section 4.12), liblcs_pcfich.so.
 *
 * The decoder is a module of its own on top of liblcs_b200.so: it takes an lcs_ctx of that library (device, stream,
 * launch count, error text) and follows its conventions (plain C, every function returns an lcs_status and never throws,
 * lcs_last_error() gives the message, no CPU fallback).  Link with -llcs_pcfich -llcs_b200.
 *
 * It reads OFDM symbol 0 of every subframe of each cell's whole OFDM grid, the grid of lcs_carrier.h, equalises the
 * PCFICH's 16 QPSK symbols with the cell's CRS, and decides the subframe's CFI: the size of its control region, 1 to 3
 * OFDM symbols (2 to 4 at 1.4 MHz), and the first thing to know before PHICH, PDCCH or any SIB can be read.
 */
#ifndef LCS_PCFICH_H
#define LCS_PCFICH_H

#include "lcs_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Cells per chunk of one lcs_pcfich_cells call; each chunk makes LCS_PCFICH_LAUNCHES_PER_CHUNK kernel launches (the
 * carrier grid, then the decoder), so a call with n cells launches 2 * ceil(n / 32) kernels. */
#define LCS_PCFICH_CHUNK 32
#define LCS_PCFICH_LAUNCHES_PER_CHUNK 2
/* Subframes of the grid: its 122 slots. */
#define LCS_PCFICH_SUBFRAMES 61

/* What one found cell decodes.  With R = n_rb_dl, N_ID = n_id_cell, the grid Y[t][c] of lcs_carrier.h (the same windows,
 * mixer and scaling; grid column c is subcarrier k = c of 36.211, since the grid skips DC) and references to 36.211 /
 * 36.212:
 *   1. Subframes.  Grid subframe s < 61 is grid slots 2s and 2s + 1; its number in the frame is s mod 10, the frame
 *      alignment of the CRS of lcs_carrier.h.  Each subframe is decoded on its own: nothing is averaged over time.
 *   2. REs (6.7.4, 6.2.4).  kbar = 6 (N_ID mod 2R).  Quadruplet i < 4 goes to the REG starting at column
 *      (kbar + 6 floor(i R / 2)) mod 12 R of symbol 0 of slot 2s, onto the 4 columns k of that REG with
 *      k mod 3 != N_ID mod 3, in increasing k (the REs the CRS of ports 0 and 1 leave free, whatever n_ports is).
 *      RE n < 16 holds symbol n: quadruplet n / 4, position n mod 4.
 *   3. Channel.  For port p at column k, hhat_p(k) interpolates linearly in k between the port's two CRS products
 *      h[m] = Y[6 m + s][..] conj(r[m]) (36.211 6.10.1, as in lcs_carrier.h; m < 2R, s the port's shift) on either side of
 *      k, and holds h[0] below the first CRS and h[2R - 1] above the last: with d = k - s, hhat = h[0] for d <= 0,
 *      h[2R - 1] for d >= 6 (2R - 1), else (1 - f) h[m] + f h[m + 1], m = floor(d / 6), f = (d - 6m) / 6.  Ports 0 and 1
 *      use symbol 0 of slot 2s, ports 2 and 3 symbol 1 of slot 2s.
 *   4. Combining (6.3.3.3, 6.3.4.3), y the 16 REs of rule 2.  One port: xhat_n = y_n conj(hhat_0) / |hhat_0|^2.  Two and
 *      four ports: pair j < 8 is REs (2j, 2j + 1) and uses ports (a, b) = (0, 1) for two ports; for four ports (0, 2) when
 *      j is even and (1, 3) when j is odd (SFBC-FSTD: each quadruplet's first pair on ports 0 and 2, its second on 1
 *      and 3).  H_a = (hhat_a(k_2j) + hhat_a(k_2j+1)) / 2, H_b the same, g = |H_a|^2 + |H_b|^2;
 *        xhat_2j   = sqrt(2) (conj(H_a) y_2j + H_b conj(y_2j+1)) / g,
 *        xhat_2j+1 = sqrt(2) (conj(H_a) y_2j+1 - H_b conj(y_2j)) / g.
 *      A clean reception gives unit-power QPSK: xhat_n = x_n.
 *   5. Decision.  Soft bits soft_2n = Re xhat_n, soft_2n+1 = Im xhat_n (the QPSK of 7.1.2).  c_b, b < 32, are the bits of
 *      36.211 7.2 with c_init = ((s mod 10) + 1)(2 N_ID + 1) 2^9 + N_ID (6.7.1).  cw_k, k = 1..3, are the codewords of
 *      36.212 Table 5.3.4-1: cw_k[b] = 0 where b mod 3 = k - 1, else 1.
 *        metric[s][k - 1] = sqrt(2) / 32 sum_b soft_b (1 - 2 c_b) (1 - 2 cw_k[b]), b ascending: a noiseless match reads 1;
 *        cfi[s] = the k with the largest metric, the smallest on ties;
 *        sinr[s] = 16 / sum_n |xhat_n - xref_n|^2, n ascending, xref the decided codeword scrambled and QPSK-mapped
 *        ((1 - 2 e_2n) + j (1 - 2 e_2n+1)) / sqrt(2), e_b = cw[b] xor c_b; +inf when the sum is 0.
 *   6. Per cell: count[k] the subframes decided k (count[0] = 0); cfi_mode the k with the largest count, the smallest on
 *      ties; n_ctrl_symbols = cfi_mode + 1 when R <= 10, else cfi_mode (36.211 Table 6.7-1); n_subframes = 61.
 * Everything after the grid is FP64 in a fixed order: a cell's record is bitwise the same whatever else the call decodes. */
typedef struct lcs_pcfich_meas {
  double metric[LCS_PCFICH_SUBFRAMES][3];      /* metric[s][k - 1] of CFI k */
  double sinr[LCS_PCFICH_SUBFRAMES];           /* linear, of the equalised PCFICH symbols */
  uint32_t cfi[LCS_PCFICH_SUBFRAMES];          /* 1, 2 or 3 */
  uint32_t count[4];                           /* count[k]: subframes decided k; count[0] = 0 */
  uint32_t cfi_mode;
  uint32_t n_ctrl_symbols;                     /* OFDM symbols of the control region at cfi_mode */
  uint32_t n_subframes;
} lcs_pcfich_meas;

typedef struct lcs_pcfich lcs_pcfich;
lcs_status lcs_pcfich_create(lcs_ctx* ctx, lcs_pcfich** out);
void lcs_pcfich_destroy(lcs_pcfich* pcfich);
/* Decode n_cells found cells on the wideband recording they were found in, chunk by chunk, then wait for them.  The
 * arguments, the accepted formats and rates, the rules a cell must fit and the errors are those of lcs_carrier_cells
 * (include/lcs_carrier.h): iq [n_in][2] in LCS_IQ_CI16, CS8, CU8 or CF32 at fs_in = D * 1.92 MHz, D in {2, 4, 8, 16, 32},
 * in device memory when on_device is non-zero (16-byte aligned), host memory otherwise.  Every argument is checked before
 * any launch; a bad one returns LCS_ERR_ARG (naming the cell).  out[i] is that of cells[i]; n_cells = 0 launches nothing.
 * A cell's record is bitwise the same whatever else the call decodes. */
lcs_status lcs_pcfich_cells(lcs_pcfich* pcfich, const void* iq, int iq_format, int on_device, uint64_t n_in, double fs_in,
                            double fc_in, const lcs_cell* cells, uint32_t n_cells, double fs_programmed,
                            lcs_pcfich_meas* out);
/* Summed device time of the decoder's kernels (CUDA events around the launches of each chunk, ms) and the number of
 * kernels launched since the last read; resets both. */
lcs_status lcs_pcfich_timing_read(lcs_pcfich* pcfich, double* kernel_ms, uint64_t* launches);

#ifdef __cplusplus
}
#endif
#endif /* LCS_PCFICH_H */
