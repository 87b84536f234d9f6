/* lcs_pdcch.h - C ABI of the common-search-space DCIs of found cells in every subframe, decoded from their PDCCH over the
 * whole carrier (DESIGN.md section 4.13), liblcs_pdcch.so.
 *
 * The decoder is a module of its own on top of liblcs_b200.so: it takes an lcs_ctx of that library (device, stream,
 * launch count, error text) and follows its conventions (plain C, every function returns an lcs_status and never throws,
 * lcs_last_error() gives the message, no CPU fallback).  Link with -llcs_pdcch -llcs_b200.
 *
 * It reads the control region of every subframe of each cell's whole OFDM grid, the grid of lcs_carrier.h, sized by the
 * CFI of lcs_pcfich.h, and blind-decodes the common search space: DCI formats 1A and 1C addressed to SI-RNTI (where SIB1
 * and the SI messages sit), P-RNTI (paging) and RA-RNTI (random-access responses).
 */
#ifndef LCS_PDCCH_H
#define LCS_PDCCH_H

#include "lcs_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Cells per chunk of one lcs_pdcch_cells call; each chunk makes LCS_PDCCH_LAUNCHES_PER_CHUNK kernel launches (the
 * carrier grid, the PCFICH decoder of lcs_pcfich.h, then the PDCCH decoder), so a call with n cells launches
 * 3 * ceil(n / 32) kernels. */
#define LCS_PDCCH_CHUNK 32
#define LCS_PDCCH_LAUNCHES_PER_CHUNK 3
/* Subframes of the grid: its 122 slots. */
#define LCS_PDCCH_SUBFRAMES 61
/* DCIs reported per subframe at most: 2 candidates of 8 CCEs and 4 of 4 CCEs. */
#define LCS_PDCCH_MAX_DCI 6
/* lcs_pdcch_dci.format */
#define LCS_DCI_1A 1
#define LCS_DCI_1C 2
/* RNTIs of the common search space (36.321 Table 7.1-1); RA-RNTIs are 1 to 60. */
#define LCS_RNTI_SI 0xFFFF
#define LCS_RNTI_P 0xFFFE

/* What one found cell decodes.  With R = n_rb_dl, N_ID = n_id_cell, grid subframe s < 61 (slots 2s and 2s + 1 of the grid
 * Y[t][c] of lcs_carrier.h: the same windows, mixer and scaling), subframe number u = s mod 10, grid column c = subcarrier
 * k = c, and references to 36.211, 36.212, 36.213 and 36.321 Rel-8, FDD:
 *   1. Control region.  cfi[s] is the decision of lcs_pcfich.h rules 1-5, bitwise what lcs_pcfich_cells returns for the
 *      cell.  n_ctrl[s] = cfi[s] + (R <= 10), raised to 3 when phich_duration is 2 (extended).  The control region is
 *      symbols 0 to n_ctrl - 1 of slot 2s.  Every subframe is non-MBSFN and is decoded on its own.
 *   2. REGs (6.2.4).  In symbol l = 0, l = 1 with four ports, or l = 3 with extended CP, REGs are 6 REs starting at
 *      columns 6m and their data REs are the 4 columns with k mod 3 != N_ID mod 3; otherwise REGs are 4 REs starting at
 *      4m, all data.  Data REs are taken in increasing k.
 *   3. PCFICH REGs are the four of lcs_pcfich.h rule 2.
 *   4. PHICH REGs (6.9.3).  N_g = 1/6, 1/2, 1, 2 for phich_resource 1 to 4; M_u = ceil(N_g R / 8) mapping units (extended
 *      CP has twice the groups, two to a unit: the same REG count).  n_l is the number of REGs of symbol l not used by the
 *      PCFICH, numbered from 0 in increasing frequency.  Unit m' < M_u, i < 3, goes to symbol l_i = 0 (normal duration)
 *      or l_i = i (extended duration), REG number (floor(N_ID n_li / n_0) + m' + floor(i n_li / 3)) mod n_li.
 *   5. PDCCH REG order (6.8.5).  For k' = 0 .. 12R - 1, and for each l < n_ctrl in turn, a REG of symbol l that starts at
 *      k' and is neither PCFICH nor PHICH is the next REG m'.  n_reg[s] is their count, n_cce[s] = floor(n_reg / 9).
 *   6. Quadruplets (6.8.5).  Quadruplet j is symbols 4j .. 4j + 3 of the PDCCH sequence; CCE n is quadruplets 9n .. 9n + 8.
 *      The n_reg quadruplets go through the sub-block interleaver of 36.212 5.1.4.2.1 (32 columns, its column permutation,
 *      ceil(n_reg / 32) rows, dummies first, read column by column, dummies dropped): w'.  REG m' carries
 *      w'((m' + N_ID) mod n_reg), its positions 0-3 on the REG's data REs.
 *   7. Equalisation: lcs_pcfich.h rules 3-4 on each REG's 4 data REs, pairs (0, 1) and (2, 3); with four ports the first
 *      pair on ports (0, 2), the second on (1, 3).  hhat comes from symbol 0 (ports 0 and 1) and symbol 1 (ports 2 and 3)
 *      of slot 2s, whichever symbol the REG is in.  This gives xhat and the gain g: |hhat_0|^2 for one port, rule 4's g
 *      for two or four.
 *   8. Candidates (36.213 9.1.1, common search space, Y = 0): L = 8 at CCE 8m, m < min(2, floor(n_cce / 8)); L = 4 at
 *      CCE 4m, m < min(4, floor(n_cce / 4)).  Each is tried at both sizes of rule 9.
 *   9. Sizes (36.212 5.3.3.1.3-4).  N_RA = ceil(log2(R (R + 1) / 2)).  1A: 15 + N_RA bits, one zero bit appended when that
 *      is in {12, 14, 16, 20, 24, 26, 32, 40, 44, 56}: 21, 22, 25, 27, 27, 28 bits for R = 6, 15, 25, 50, 75, 100.  1C:
 *      [R >= 50] + ceil(log2(floor(N_VRB,gap1 / N_step) (floor(N_VRB,gap1 / N_step) + 1) / 2)) + 5 bits: 8, 10, 12, 13, 14,
 *      15.  K = size + 16.
 *  10. Decoding.  Soft bits u_2n = sqrt(2) Re xhat_n, u_2n+1 = sqrt(2) Im xhat_n over the candidate's 36 L symbols.  c is
 *      the sequence of 36.211 7.2 with c_init = u 2^9 + N_ID (6.8.2), bit b of CCE n at 72 n + b.  v_b = (1 - 2 c) u_b g.
 *      De-rate-matching averages the repetitions (36.212 5.1.4.2 inverted, as for the MIB); the decoder is the exact ML
 *      tail-biting Viterbi over all 64 start states of the MIB decoder, with its tie rules (the even predecessor on equal
 *      metrics, the lowest start state on equal totals).
 *  11. Acceptance.  p = CRC16 (x^16 + x^12 + x^5 + 1, zero init) of a_0 .. a_size-1; rnti = sum (p_i xor a_size+i)
 *      2^(15 - i).  Accepted when rnti is 0xFFFF (SI), 0xFFFE (P) or 1 to 60 (RA), a_0 = 1 for 1A, and q >= 0.8, where
 *      q = sum u_b (1 - 2 e_b) / sqrt(72 L sum u_b^2), b < 72 L, e_b the decoded word re-encoded, rate-matched and
 *      scrambled (a noiseless match reads 1; an L = 8 candidate whose second half is empty reads at most 1/sqrt(2)).
 *  12. Duplicates.  A candidate accepted at both sizes keeps the larger q, 1A on ties.  An accepted L = 4 candidate inside
 *      an accepted L = 8 candidate with the same format, rnti and payload is dropped.  dci[s] holds the L = 8 candidates
 *      first, then L = 4, CCEs ascending: n_dci[s] <= 6.
 *  13. Record.  Per DCI format, agg (L), cce, rnti, n_bits (size), quality (q) and payload = sum a_i 2^(size - 1 - i),
 *      and the fields parsed from it on the host: for 1A (36.212 5.3.3.1.3) localized (the raw localized/distributed
 *      VRB assignment flag: 1 means distributed), the resource block assignment as
 *      riv and decoded on R to rb_start and n_rb (36.213 7.1.6.3; -1 when riv is not a valid RIV), mcs, harq, ndi, rv and
 *      tpc; for 1C (5.3.3.1.4) gap, riv (raw) and tbs_index.  Fields a format does not have are 0 (rb_start, n_rb -1).
 *      Per subframe cfi, n_ctrl, n_reg, n_cce and n_dci.  Per cell count[] the DCIs with SI-, P- and RA-RNTI,
 *      si_subframes (bit u set when an SI-RNTI DCI was found in a subframe numbered u) and n_subframes = 61.
 * Everything after the grid is FP64 in a fixed order: a cell's record is bitwise the same whatever else the call decodes. */
typedef struct lcs_pdcch_dci {
  double quality;                              /* q of rule 11 */
  uint64_t payload;                            /* a_0 is the most significant of n_bits bits */
  uint32_t format;                             /* LCS_DCI_1A or LCS_DCI_1C */
  uint32_t agg;                                /* 4 or 8 CCEs */
  uint32_t cce;                                /* first CCE */
  uint32_t rnti;
  uint32_t n_bits;                             /* payload size */
  uint32_t riv;                                /* resource block assignment field */
  int32_t rb_start, n_rb;                      /* 1A: riv decoded on R; -1 otherwise */
  uint32_t localized, mcs, harq, ndi, rv, tpc; /* 1A; localized is the raw flag: 1 means distributed VRBs */
  uint32_t gap, tbs_index;                     /* 1C */
} lcs_pdcch_dci;

typedef struct lcs_pdcch_meas {
  lcs_pdcch_dci dci[LCS_PDCCH_SUBFRAMES][LCS_PDCCH_MAX_DCI];   /* dci[s][i], i < n_dci[s] */
  uint32_t cfi[LCS_PDCCH_SUBFRAMES];
  uint32_t n_ctrl[LCS_PDCCH_SUBFRAMES];        /* OFDM symbols of the control region */
  uint32_t n_reg[LCS_PDCCH_SUBFRAMES];
  uint32_t n_cce[LCS_PDCCH_SUBFRAMES];
  uint32_t n_dci[LCS_PDCCH_SUBFRAMES];
  uint32_t count[3];                           /* DCIs with SI-RNTI, P-RNTI, RA-RNTI */
  uint32_t si_subframes;                       /* bit u: an SI-RNTI DCI in a subframe numbered u */
  uint32_t n_subframes;
} lcs_pdcch_meas;

typedef struct lcs_pdcch lcs_pdcch;
lcs_status lcs_pdcch_create(lcs_ctx* ctx, lcs_pdcch** out);
void lcs_pdcch_destroy(lcs_pdcch* pdcch);
/* Decode n_cells found cells on the wideband recording they were found in, chunk by chunk, then wait for them.  The
 * arguments, the accepted formats and rates, the rules a cell must fit and the errors are those of lcs_carrier_cells
 * (include/lcs_carrier.h), and a cell must also have phich_duration 1 or 2 and phich_resource 1 to 4: iq [n_in][2] in
 * LCS_IQ_CI16, CS8, CU8 or CF32 at fs_in = D * 1.92 MHz, D in {2, 4, 8, 16, 32}, in device memory when on_device is
 * non-zero (16-byte aligned), host memory otherwise.  Every argument is checked before any launch; a bad one returns
 * LCS_ERR_ARG (naming the cell).  out[i] is that of cells[i]; n_cells = 0 launches nothing.  A cell's record is bitwise
 * the same whatever else the call decodes. */
lcs_status lcs_pdcch_cells(lcs_pdcch* pdcch, const void* iq, int iq_format, int on_device, uint64_t n_in, double fs_in,
                           double fc_in, const lcs_cell* cells, uint32_t n_cells, double fs_programmed,
                           lcs_pdcch_meas* out);
/* Summed device time of the decoder's kernels (CUDA events around the launches of each chunk, ms) and the number of
 * kernels launched since the last read; resets both. */
lcs_status lcs_pdcch_timing_read(lcs_pdcch* pdcch, double* kernel_ms, uint64_t* launches);

#ifdef __cplusplus
}
#endif
#endif /* LCS_PDCCH_H */
