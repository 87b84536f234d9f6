// carrier_plan.hpp - host planning of the full-carrier measurement (carrier.cu): one cell checked against the contract of
// include/lcs_carrier.h and its CRS windows laid out, with no device work.
#pragma once
#include <string>
#include <vector>

#include "../../include/lcs_b200.h"

namespace lcs {
namespace carrier {

constexpr int N_SLOT = 122;          // slots of the grid in either CP (lcs_extract_tfg's 854 or 732 symbols)

struct CellPlan {
  std::vector<long long> q;          // [N_SLOT][nw] first recording sample of each CRS window
  std::vector<double> late;          // q - D loc_t
  long long step = 0;                // (delta mod fs_in)
  double kpi = 0;                    // kappa / pi
  int R = 0, n_ports = 0, nw = 0, n_id_cell = 0, cp_type = 0;   // nw: windows per slot (2, or 3 for four ports)
};

// Check cell c (rules 1-5 of lcs_carrier.h for a recording of n_in samples at fs_in = D * 1.92 MHz, centred on fc_in) and
// fill `plan`; "" when it is measurable, else why not.  The window order within a slot is symbol 0, symbol 1 (four ports
// only), symbol n_symb - 3.
std::string plan_cell(const lcs_cell& c, uint64_t n_in, int D, double fs_in, double fc_in, double fs_programmed,
                      CellPlan& plan);

}  // namespace carrier
}  // namespace lcs
