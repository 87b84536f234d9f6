/* lcs_sib1.h - C ABI of SystemInformationBlockType1 (SIB1) of found cells, decoded from the PDSCH their SI-RNTI DCIs
 * schedule over the whole carrier (DESIGN.md section 4.14), liblcs_sib1.so.
 *
 * The decoder is a module of its own on top of liblcs_b200.so: it takes an lcs_ctx of that library (device, stream,
 * launch count, error text) and follows its conventions (plain C, every function returns an lcs_status and never throws,
 * lcs_last_error() gives the message, no CPU fallback).  Link with -llcs_sib1 -llcs_b200.
 *
 * SIB1 names the networks a cell belongs to (MCC-MNC), its tracking area code and its 28-bit cell identity.  The decoder
 * reads the three SIB1 occasions of each cell's grid: their control region and SI-RNTI DCI as lcs_pdcch.h decodes them,
 * then the PDSCH that DCI schedules, through a turbo decoder, into the transport block, whose SIB1 fields it parses.
 */
#ifndef LCS_SIB1_H
#define LCS_SIB1_H

#include "lcs_pdcch.h"

#ifdef __cplusplus
extern "C" {
#endif

/* Cells per chunk of one lcs_sib1_cells call; each chunk makes LCS_SIB1_LAUNCHES_PER_CHUNK kernel launches (the carrier
 * grid, the PCFICH decoder of lcs_pcfich.h, the PDCCH decoder of lcs_pdcch.h on the occasions only, the PDSCH front end
 * and the turbo decoder), so a call with n cells launches 5 * ceil(n / 32) kernels. */
#define LCS_SIB1_CHUNK 32
#define LCS_SIB1_LAUNCHES_PER_CHUNK 5
#define LCS_SIB1_OCCASIONS 3
#define LCS_SIB1_TB_BYTES 280
#define LCS_SIB1_MAX_PLMN 6
#define LCS_SIB1_MAX_SI 32

/* What one found cell decodes.  With R = n_rb_dl, N_ID = n_id_cell, n_symb = 7 (normal CP) or 6 (extended), the grid
 * Y[t][c] of lcs_carrier.h (grid column c = subcarrier k = c) and references to 36.211, 36.212, 36.213, 36.321 and 36.331
 * Rel-8, FDD:
 *   1. Occasions.  cell.sfn (0 to 1023) is the SFN of grid frame 0, as lcs_decode_mib reports it.  Grid subframe
 *      s = 10 f + 5, f = 0 .. 5 with (sfn + f) even, is a SIB1 occasion (36.331 5.2.1.2): exactly 3 per cell, whose SFN
 *      is (sfn + f) mod 1024.
 *   2. Control region and DCI.  cfi, n_ctrl and the DCIs of an occasion are bitwise what lcs_pdcch_cells reports for
 *      that subframe.  The occasion uses its SI-RNTI DCI of the largest quality, the first in record order on ties;
 *      without one it is found = 0 and nothing else is decoded.
 *   3. Allocation.  1A (the DCI's localized field is the raw flag: 1 means distributed): the RIV is decoded on R (rule 13
 *      of lcs_pdcch.h) to VRBs rb_start .. rb_start + n_rb - 1; localized VRBs are the PRBs of the same numbers,
 *      distributed ones use N_gap,1.  1C: N_step = 2 (R < 50) or 4, gap = the DCI's gap bit (R >= 50, else 0); the RIV
 *      is decoded on floor(N_VRB,gap / N_step) and its start and length are scaled by N_step; the VRBs are
 *      distributed.  Distributed VRB n is PRB vrb_to_prb(n, slot) of 36.211 6.2.3.2 in each slot: prb[slot] lists the
 *      PRBs of each slot, ascending.  An invalid RIV, VRBs beyond N_VRB, or a 1A mcs above 26 leaves n_re = 0.
 *   4. Transport block (QPSK).  1A: I_TBS = mcs, N_PRB^1A = 2 when the TPC field's LSB is 0, else 3 (36.213 7.1.7);
 *      1C: 36.213 Table 7.1.7.2.3-1 at tbs_index.  rv = ceil(3k / 2) mod 4, k = (SFN / 2) mod 4 (36.321 5.3.1), whatever
 *      the 1A rv field says.  One code block of K = the smallest turbo block size >= TBS + 24 (K <= 2240), whose first
 *      F = K - TBS - 24 bits are filler bits, known zeros.
 *   5. REs (36.211 6.3.5).  The data REs are those of the PRBs of rule 3 in symbols l = n_ctrl .. 2 n_symb - 1 of the
 *      subframe, taken k first, then l, slot 0's PRBs in its symbols and slot 1's in its, leaving out the CRS REs of
 *      every port below n_ports, and in symbols n_symb - 2 and n_symb - 1 (PSS and SSS) the columns 6R - 36 <= c < 6R + 36.
 *      Every PRB keeps an even number of REs in each symbol, so transmit-diversity pairs stay in a symbol.  n_re of them.
 *   6. Equalisation.  Port p's estimate at column k in CRS symbol l of the port is rule 3 of lcs_pcfich.h on that
 *      symbol; in the data symbol l it is the linear interpolation in l between the port's CRS symbols either side,
 *      (1 - w) h_a + w h_b with w = (l - l_a) / (l_b - l_a), and the nearest one's value outside them.  The CRS symbols
 *      of ports 0 and 1 are 0, n_symb - 3, n_symb and 2 n_symb - 3; of ports 2 and 3, 1 and n_symb + 1.  Combining is
 *      rule 4 of lcs_pcfich.h on consecutive RE pairs in mapping order (one port: ZF per RE; four ports: pair i on ports
 *      (0, 2) when i is even, (1, 3) when odd, i counted over the subframe), giving xhat and its gain g.
 *      u_2n = sqrt(2) Re xhat_n, u_2n+1 = sqrt(2) Im xhat_n; v_b = (1 - 2 c_b) u_b g, c of 36.211 7.2 with
 *      c_init = 0xFFFF 2^14 + 5 2^9 + N_ID (6.3.1).  sinr = n_re / sum |xhat - slice(xhat)|^2, slice the nearest QPSK
 *      point (+inf when the sum is 0).
 *   7. De-rate-matching (36.212 5.1.4.1).  E = 2 n_re.  The circular buffer w of K_w = 96 ceil((K + 4) / 32) positions
 *      (the 32-column sub-block interleaver, the third stream's offset permutation), N_cb = K_w, read from
 *      k0 = R_sub (2 ceil(N_cb / (8 R_sub)) rv + 2), NULLs skipped, gives e_j the bit at its j-th non-NULL position;
 *      each coded bit d[i][k] is the sum of v_j over the e_j that carry it, in increasing j, 0 when none does.  Filler
 *      bits read +1e6 in d[0] and 0 in d[1].
 *   8. Turbo decoding (36.212 5.1.3.2, QPP of Table 5.1.3-3, the 12 tail bits of 5.1.3.2.2).  LLRs are log P(0) / P(1).
 *      Max-log-MAP in FP64: the branch metric of input u and parity z is ((1 - 2u)(L_s + L_a) + (1 - 2z) L_p) / 2;
 *      decoder 1 runs the natural order on d[0], d[1], decoder 2 the interleaved order (L_s = d[0][pi(k)]) on d[2]; one
 *      iteration is decoder 1 then decoder 2.  Each half-iteration cuts the K steps into windows of 32: the first
 *      window starts from state 0, the last ends on the tail's metrics (the 3 termination steps summed from state 0
 *      backwards), and every other boundary starts from the metrics that window's neighbour reached there in the same
 *      decoder's previous half-iteration (0 for every state on the first).  Extrinsic = L_app - L_s - L_a, times 0.75,
 *      is the other decoder's L_a.  After each iteration the hard decision (bit 0 when decoder 2's L_app >= 0) is
 *      checked with CRC24A; decoding stops at the first pass or after 8 iterations.  iterations counts them; tb holds
 *      the decided TBS bits (most significant bit first), crc_ok whether the CRC passed.
 *   9. SIB1 (on the host).  The first occasion that passes CRC is read as UPER BCCH-DL-SCH-Message, c1,
 *      systemInformationBlockType1 (36.331 Rel-8), up to systemInfoValueTag and the presence of nonCriticalExtension.
 *      parse_ok = 0 when no occasion passed CRC, or it is another message, or its bits run out; the parsed fields (n_plmn
 *      on) are then all 0.  A PLMN without MCC takes the previous one's.  consistent = 1 when at least one occasion
 *      passed CRC and every occasion that passed carries the same bytes, else 0.
 *  10. Record: per occasion below; per cell n_found, n_crc_ok, consistent and the parsed fields.
 * Everything after the grid is FP64 in a fixed order: a cell's record is bitwise the same whatever else the call decodes. */
typedef struct lcs_sib1_occasion {
  double sinr;                                 /* linear, of the equalised PDSCH symbols */
  lcs_pdcch_dci dci;                           /* the SI-RNTI DCI used (its fields parsed as lcs_pdcch.h rule 13) */
  uint32_t subframe;                           /* grid subframe */
  uint32_t sfn;
  uint32_t found;                              /* an SI-RNTI DCI was found */
  uint32_t cfi, n_ctrl;
  uint32_t format;                             /* LCS_DCI_1A or LCS_DCI_1C */
  uint32_t distributed, gap;
  int32_t vrb_start, n_vrb;                    /* the VRBs; -1 when the allocation is invalid */
  uint32_t n_prb;                              /* PRBs per slot */
  uint8_t prb[2][100];                         /* prb[slot][i], i < n_prb, ascending */
  uint32_t tbs, K, F, rv;
  uint32_t n_re;
  uint32_t crc_ok, iterations;
  uint8_t tb[LCS_SIB1_TB_BYTES];
} lcs_sib1_occasion;

typedef struct lcs_sib1_plmn {
  uint32_t mcc;                                /* three digits, e.g. 310 */
  uint32_t mnc;
  uint32_t mnc_digits;                         /* 2 or 3 */
  uint32_t reserved;                           /* cellReservedForOperatorUse: 1 reserved */
} lcs_sib1_plmn;

typedef struct lcs_sib1_meas {
  lcs_sib1_occasion occ[LCS_SIB1_OCCASIONS];
  uint32_t n_found, n_crc_ok, consistent;
  uint32_t parse_ok;
  uint32_t n_plmn;
  lcs_sib1_plmn plmn[LCS_SIB1_MAX_PLMN];
  uint32_t tac;                                /* trackingAreaCode */
  uint32_t cell_identity;                      /* 28 bits */
  uint32_t cell_barred;                        /* 1 barred */
  uint32_t intra_freq_reselection;             /* 1 allowed */
  uint32_t csg_indication, csg_identity_present, csg_identity;
  int32_t q_rx_lev_min;                        /* the IE's value (-70 .. -22; dBm / 2) */
  uint32_t q_rx_lev_min_offset;                /* 1 .. 8, 0 when absent */
  uint32_t p_max_present;
  int32_t p_max;                               /* dBm */
  uint32_t freq_band_indicator;
  uint32_t n_si;
  uint32_t si_periodicity[LCS_SIB1_MAX_SI];    /* radio frames: 8 .. 512 */
  uint32_t si_sib_mask[LCS_SIB1_MAX_SI];       /* bit n: SIB type n (3 .. 11) is in SI message i */
  uint32_t tdd_present, tdd_subframe_assignment, tdd_special_subframe_patterns;
  uint32_t si_window_ms;
  uint32_t system_info_value_tag;
  uint32_t non_critical_extension;
} lcs_sib1_meas;

typedef struct lcs_sib1 lcs_sib1;
lcs_status lcs_sib1_create(lcs_ctx* ctx, lcs_sib1** out);
void lcs_sib1_destroy(lcs_sib1* sib1);
/* Decode n_cells found cells on the wideband recording they were found in, chunk by chunk, then wait for them.  The
 * arguments, formats, rates, the rules a cell must fit and the errors are those of lcs_pdcch_cells (include/lcs_pdcch.h),
 * and a cell's sfn must be 0 to 1023.  Every argument is checked before any launch; a bad one returns LCS_ERR_ARG (naming
 * the cell).  out[i] is that of cells[i]; n_cells = 0 launches nothing.  A cell's record is bitwise the same whatever
 * else the call decodes. */
lcs_status lcs_sib1_cells(lcs_sib1* sib1, const void* iq, int iq_format, int on_device, uint64_t n_in, double fs_in,
                          double fc_in, const lcs_cell* cells, uint32_t n_cells, double fs_programmed, lcs_sib1_meas* out);
/* Summed device time of the decoder's kernels (CUDA events around the launches of each chunk, ms) and the number of
 * kernels launched since the last read; resets both. */
lcs_status lcs_sib1_timing_read(lcs_sib1* sib1, double* kernel_ms, uint64_t* launches);

#ifdef __cplusplus
}
#endif
#endif /* LCS_SIB1_H */
