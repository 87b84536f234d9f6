// chain_host.hpp - host-side stages of the cell-search chain (see chain_host.cpp).
#pragma once
#include <functional>
#include <vector>

#include "lcs_internal.hpp"

namespace lcs {

struct RsDl {   // cell-specific reference signals of the 6 centre RBs (lte_lib.cpp:354-405)
  int n_id_cell, n_symb;
  std::vector<cd> rs;   // [slot][sym in {0,1,n_symb-3}][12]
  RsDl(int n_id_cell, int cp_type);
  const cd* get(int slot, int sym) const;
  int shift(int slot, int sym, int port) const;
};

void calc_z_th1(const double* sp_incoherent, uint32_t n, uint16_t n_comb_xc, uint8_t arm, double* z);
void peak_search(const double* pow_rowmajor, const int32_t* frq_rowmajor, const double* z_th1, const double* f_search_set,
                 double fc_requested, double fc_programmed, const std::function<float(int, int, int)>& single_at,
                 uint8_t arm, std::vector<lcs_cell>& cells);
void tfoec(const lcs_cell& cell, const cd* tfg, const double* ts, int n_ofdm, double fc_requested, double fc_programmed,
           const RsDl& rs, cd* tfg_comp, double* ts_comp, lcs_cell& out);
void chan_est(const RsDl& rs, const cd* tfg, int n_ofdm, int port, std::vector<cd>& ce, double& np);
void decode_mib(const lcs_cell& cell, const cd* tfg, int n_ofdm, const RsDl& rs, lcs_cell& out);
void dedup(const lcs_cell* cells, uint32_t n, std::vector<lcs_cell>& fin);
std::vector<double> f_search_set_for(double freq_start, double ppm);
// position in the 3 x 40 coded block of every rate-matched PBCH bit e[k] (lte_lib.cpp:409-463)
void pbch_ratematch_positions(int n_e, std::vector<int>& pos);

}  // namespace lcs
