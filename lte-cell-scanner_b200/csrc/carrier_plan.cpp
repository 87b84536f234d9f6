// carrier_plan.cpp - host planning of the full-carrier measurement (see carrier_plan.hpp).  Host code only, so that it
// can be checked on its own (tests/test_carrier_meas_host.py builds it with AddressSanitizer).
#include "carrier_plan.hpp"

#include <cmath>
#include <cstdlib>

#include "chain_gpu.hpp"

namespace lcs {
namespace carrier {

std::string plan_cell(const lcs_cell& c, uint64_t n_in, int D, double fs_in, double fc_in, double fs_programmed,
                      CellPlan& plan) {
  if (c.cp_type != 1 && c.cp_type != 2) return "cp_type must be 1 (normal) or 2 (extended)";
  if (c.n_id_1 < 0 || c.n_id_1 > 167 || c.n_id_2 < 0 || c.n_id_2 > 2) return "n_id_1 / n_id_2 out of range";
  if (c.n_ports != 1 && c.n_ports != 2 && c.n_ports != 4) return "n_ports must be 1, 2 or 4";
  const int R = c.n_rb_dl;
  if (R != 6 && R != 15 && R != 25 && R != 50 && R != 75 && R != 100) return "n_rb_dl must be 6, 15, 25, 50, 75 or 100";
  if (!(std::isfinite(c.frame_start) && std::isfinite(c.freq_superfine))) return "frame_start and freq_superfine must be finite";
  if (!(std::isfinite(c.fc_requested) && c.fc_requested > 0 && std::isfinite(c.fc_programmed) && c.fc_programmed > 0))
    return "fc_requested and fc_programmed must be finite and positive";
  const double delta = c.fc_requested - fc_in;
  if (!(std::fabs(delta - std::rint(delta)) <= 1e-6)) return "fc_requested - fc_in must be an integer number of Hz";
  const long long di = std::llround(delta), fs = std::llround(fs_in);
  if (6 * R >= 64 * D) return "6 n_rb_dl must be below 64 D: the carrier is wider than fs_in allows";
  if (2 * (std::llabs(di) + 90000ll * R) > fs) return "the carrier does not lie inside the recording's band";
  lcs_cell gc = c;
  gc.freq_fine = c.freq_superfine;
  // tfg_geometry's tables for this one cell, in host memory the call owns
  std::vector<int> pos(TFG_MAX);
  std::vector<double> late(TFG_MAX), ts(TFG_MAX);
  double k = 0;
  int n_ofdm = 0;
  const GridTables g(pos.data(), late.data(), &k, &n_ofdm);
  const char* why = "";
  if (tfg_geometry(gc, c.fc_requested, c.fc_programmed, fs_programmed, 0xffffffffu, g, 0, ts.data(), &why) != LCS_OK)
    return std::string("no grid (") + why + ")";
  const int n_symb = c.cp_type == 1 ? 7 : 6, N = 128 * D;
  const int nw = c.n_ports == 4 ? 3 : 2;
  plan.q.assign((size_t)N_SLOT * nw, 0);
  plan.late.assign(plan.q.size(), 0.0);
  for (int t = 0; t < n_ofdm; t++) {
    const double dl = D * ts[t], q = std::rint(dl);
    if (q < 0 || q + N > (double)n_in) return "a DFT window falls outside the recording";
    const int slot = t / n_symb, sym = t % n_symb;
    const int w = sym == 0 ? 0 : (sym == n_symb - 3 ? nw - 1 : (sym == 1 && nw == 3 ? 1 : -1));
    if (w < 0) continue;
    plan.q[(size_t)slot * nw + w] = (long long)q;
    plan.late[(size_t)slot * nw + w] = q - dl;
  }
  const double k_factor = (c.fc_requested - c.freq_superfine) / c.fc_programmed;
  plan.step = (di % fs + fs) % fs;
  plan.kpi = -2.0 * c.freq_superfine / (D * fs_programmed * k_factor);
  plan.R = R;
  plan.n_ports = c.n_ports;
  plan.nw = nw;
  plan.n_id_cell = c.n_id_2 + 3 * c.n_id_1;
  plan.cp_type = c.cp_type;
  return "";
}

}  // namespace carrier
}  // namespace lcs
