// searcher_dropin.hpp - host-side mirror of the reference's search interface.
//
// Same names, argument order, argument meaning and in-band error conventions as
// include/searcher.h:22-124, include/common.h.in:101-129 (class Cell) and the RS_DL handle of
// include/lte_lib.h - but every function forwards to the C ABI of include/lcs_b200.h, i.e. to the
// CUDA kernels.  A maintainer of the reference replaces src/searcher.cpp by searcher_dropin.cpp
// and links liblcs_b200.so (INTEGRATION.md).
//
// Error behaviour: like the reference, "not found" is in-band (n_id_1==-1, n_rb_dl==-1); states the
// reference answers with `throw("...")` (unknown cp_type, searcher.cpp:786,883) and any failure of
// the CUDA layer throw a `const char*` here as well.
#pragma once
#include <list>
#include <string>
#include <vector>

#ifdef LCS_USE_REAL_ITPP
#include <itpp/itbase.h>
#else
#include "itpp_min.hpp"
#endif
#include "../../include/lcs_b200.h"
#include "../../include/lcs_meas.h"
#include "../../include/lcs_carrier.h"
#include "../../include/lcs_cir.h"
#include "../../include/lcs_pcfich.h"
#include "../../include/lcs_pdcch.h"
#include "../../include/lcs_sib1.h"

// --- include/common.h.in ---
typedef char int8;
typedef unsigned char uint8;
typedef short int16;
typedef unsigned short uint16;
typedef int int32;
typedef unsigned int uint32;
typedef std::vector<std::vector<std::vector<std::complex<float> > > > vcf3d;
typedef std::vector<std::vector<std::vector<float> > > vf3d;
namespace cp_type_t { enum cp_type_t { UNKNOWN = 0, NORMAL, EXTENDED }; }
namespace phich_duration_t { enum phich_duration_t { UNKNOWN = 0, NORMAL, EXTENDED }; }
namespace phich_resource_t { enum phich_resource_t { UNKNOWN = 0, oneSixth, half, one, two }; }

class Cell {   // include/common.h.in:101-129
 public:
  double fc_requested, fc_programmed, pss_pow;
  int32 ind;
  double freq;
  int8 n_id_2;
  int16 n_id_1;
  cp_type_t::cp_type_t cp_type;
  double frame_start, freq_fine, freq_superfine;
  int8 n_ports, n_rb_dl;
  phich_duration_t::phich_duration_t phich_duration;
  phich_resource_t::phich_resource_t phich_resource;
  int16 sfn;
  Cell();
  int16 n_id_cell() const;
  int8 n_symb_dl() const;
};

// Opaque stand-in for the reference's RS_DL (include/lte_lib.h): the CUDA library builds the
// reference-signal tables itself from (n_id_cell, cp_type); the object only carries those.
class RS_DL {
 public:
  RS_DL(const uint16& n_id_cell, const uint8& n_rb_dl, const cp_type_t::cp_type_t& cp_type)
      : n_id_cell_(n_id_cell), n_rb_dl_(n_rb_dl), cp_type_(cp_type) {}
  uint16 n_id_cell_;
  uint8 n_rb_dl_;
  cp_type_t::cp_type_t cp_type_;
};

// --- include/searcher.h:22-124 (verbatim signatures) ---
void xcorr_pss(const itpp::cvec& capbuf, const itpp::vec& f_search_set, const uint8& ds_comb_arm,
               const double& fc_requested, const double& fc_programmed, const double& fs_programmed,
               itpp::mat& xc_incoherent_collapsed_pow, itpp::imat& xc_incoherent_collapsed_frq,
               vf3d& xc_incoherent_single, vf3d& xc_incoherent, itpp::vec& sp_incoherent, vcf3d& xc, itpp::vec& sp,
               uint16& n_comb_xc, uint16& n_comb_sp);
void peak_search(const itpp::mat& xc_incoherent_collapsed_pow, const itpp::imat& xc_incoherent_collapsed_frq,
                 const itpp::vec& Z_th1, const itpp::vec& f_search_set, const double& fc_requested,
                 const double& fc_programmed, const vf3d& xc_incoherent_single, const uint8& ds_comb_arm,
                 std::list<Cell>& cells);
Cell sss_detect(const Cell& cell, const itpp::cvec& capbuf, const double& thresh2_n_sigma, const double& fc_requested,
                const double& fc_programmed, const double& fs_programmed, itpp::vec& sss_h1_np_est,
                itpp::vec& sss_h2_np_est, itpp::cvec& sss_h1_nrm_est, itpp::cvec& sss_h2_nrm_est,
                itpp::cvec& sss_h1_ext_est, itpp::cvec& sss_h2_ext_est, itpp::mat& log_lik_nrm, itpp::mat& log_lik_ext);
Cell pss_sss_foe(const Cell& cell_in, const itpp::cvec& capbuf, const double& fc_requested,
                 const double& fc_programmed, const double& fs_programmed);
void extract_tfg(const Cell& cell, const itpp::cvec& capbuf_raw, const double& fc_requested, const double& fc_programmed,
                 const double& fs_programmed, itpp::cmat& tfg, itpp::vec& tfg_timestamp);
Cell tfoec(const Cell& cell, const itpp::cmat& tfg, const itpp::vec& tfg_timestamp, const double& fc_requested,
           const double& fc_programmed, const RS_DL& rs_dl, itpp::cmat& tfg_comp, itpp::vec& tfg_comp_timestamp);
Cell decode_mib(const Cell& cell, const itpp::cmat& tfg, const RS_DL& rs_dl);
void del_oob(itpp::ivec& v);

// --- glue of src/CellSearch.cpp the CLI needs ---
void dedup(const std::vector<std::list<Cell> >& detected_cells, std::list<Cell>& cells_final);   // CellSearch.cpp:285-319
itpp::vec calc_Z_th1(const itpp::vec& sp_incoherent, uint16 n_comb_xc, uint8 ds_comb_arm);         // CellSearch.cpp:500-503
// CUDA device used by the drop-in (default 0, or env LCS_DEVICE); created lazily, process-wide.
lcs_ctx* lcs_dropin_ctx();
void xcorr_pss_skip_debug_outputs(bool skip);
// The whole per-centre-frequency loop of CellSearch.cpp:465-558 for raw 8-bit capture buffers (cu8 [n_fc][n_cap][2]) in one call:
// lcs_sweep_search_cu8 (one plan per centre frequency, one correlator launch per 64 channels).  detected_cells as in :469.
void sweep_search_cu8(const std::vector<unsigned char>& iq, uint32_t n_cap, const std::vector<double>& fc_requested,
                      const itpp::vec& f_search_set, const double& fs_programmed, std::vector<std::list<Cell> >& detected_cells);
// The same sweep fed from one wideband ci16 recording (iq [n][2] at fs_in, centred on fc_in): lcs_chan auto gain, every
// channel channelized into device memory (153 600 samples each), then lcs_sweep_search_cu8_device.  With meas, every
// found cell is also measured (lcs_meas_cells) on the channelized buffer in place, with rsrp, noise and rssi divided by
// the channel's gain^2 so that they are in the recording's full scale: meas[c][k] is that of detected_cells[c]'s k-th.
void wideband_search_ci16(const int16_t* iq, uint32_t n, double fs_in, double fc_in, const std::vector<double>& fc_requested,
                          const itpp::vec& f_search_set, const double& fs_programmed, std::vector<std::list<Cell> >& detected_cells,
                          std::vector<std::vector<lcs_cell_meas> >* meas = nullptr);
// The same at any rate lcs_chan_create_rational allows, iq [n][2] in iq_format (LCS_IQ_CI16, CS8, CU8 or CF32).
void wideband_search_rational(const void* iq, int iq_format, uint32_t n, double fs_in, double fc_in,
                              const std::vector<double>& fc_requested, const itpp::vec& f_search_set,
                              const double& fs_programmed, std::vector<std::list<Cell> >& detected_cells,
                              std::vector<std::vector<lcs_cell_meas> >* meas = nullptr);
// RSRP / RSRQ / SINR (lcs_meas of liblcs_meas.so, DESIGN.md section 4.9) of every cell of detected_cells[c], found in
// capture buffer c of iq ([detected_cells.size()][n_cap][2] in iq_format LCS_IQ_CU8, CF32 or C128, host memory), in one
// call: meas[c][k] is that of detected_cells[c]'s k-th cell.
void measure_cells(const void* iq, int iq_format, uint32_t n_cap, const std::vector<std::list<Cell> >& detected_cells,
                   const double& fs_programmed, std::vector<std::vector<lcs_cell_meas> >& meas);
   // skip the 136 MB `xc`/`sp`/`xc_incoherent` debug outputs (CLI does)
// Full-carrier RSRP / RSRQ / SINR (lcs_carrier of liblcs_carrier.so, DESIGN.md section 4.10) of every cell of `cells`,
// found in the wideband recording iq ([n][2] in iq_format at fs_in, centred on fc_in, host memory): meas[i] is that of
// cells[i], and ok[i] is false for a cell lcs_carrier_cells rejects (one the recording does not hold whole).
void measure_carriers(const void* iq, int iq_format, uint64_t n, double fs_in, double fc_in, const std::vector<Cell>& cells,
                      const double& fs_programmed, std::vector<lcs_carrier_meas>& meas, std::vector<bool>& ok);
// The power delay profile (lcs_cir of liblcs_cir.so, DESIGN.md section 4.11) of every cell of `cells`, as
// measure_carriers: meas[i] is that of cells[i], and ok[i] is false for a cell lcs_cir_cells rejects.
void measure_cirs(const void* iq, int iq_format, uint64_t n, double fs_in, double fc_in, const std::vector<Cell>& cells,
                  const double& fs_programmed, std::vector<lcs_cir_meas>& meas, std::vector<bool>& ok);
// The control format indicator in every subframe (lcs_pcfich of liblcs_pcfich.so, DESIGN.md section 4.12) of every cell
// of `cells`, as measure_carriers: meas[i] is that of cells[i], and ok[i] is false for a cell lcs_pcfich_cells rejects.
void measure_pcfich(const void* iq, int iq_format, uint64_t n, double fs_in, double fc_in, const std::vector<Cell>& cells,
                    const double& fs_programmed, std::vector<lcs_pcfich_meas>& meas, std::vector<bool>& ok);
// The common-search-space DCIs in every subframe (lcs_pdcch of liblcs_pdcch.so, DESIGN.md section 4.13) of every cell of
// `cells`, as measure_carriers: meas[i] is that of cells[i], and ok[i] is false for a cell lcs_pdcch_cells rejects.
void measure_pdcch(const void* iq, int iq_format, uint64_t n, double fs_in, double fc_in, const std::vector<Cell>& cells,
                   const double& fs_programmed, std::vector<lcs_pdcch_meas>& meas, std::vector<bool>& ok);
// SIB1 (lcs_sib1 of liblcs_sib1.so, DESIGN.md section 4.14) of every cell of `cells`, each with the SFN its MIB decode
// gave, as measure_carriers: meas[i] is that of cells[i], and ok[i] is false for a cell lcs_sib1_cells rejects.
void measure_sib1(const void* iq, int iq_format, uint64_t n, double fs_in, double fc_in, const std::vector<Cell>& cells,
                  const double& fs_programmed, std::vector<lcs_sib1_meas>& meas, std::vector<bool>& ok);
// Welch power spectral density (lcs_psd of liblcs_psd.so, DESIGN.md section 4.8) of the whole recording in `path` ([n][2] in iq_format,
// sample_bytes per sample, at fs_in, read in blocks): psd [nfft] in fftshift order, full-scale^2 per Hz, over n_segments segments.
void wideband_psd(const std::string& path, int iq_format, size_t sample_bytes, double fs_in, uint32_t nfft,
                  std::vector<double>& psd, uint64_t& n_segments);
