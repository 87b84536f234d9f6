// pdcch_plan.cpp - host planning of the PDCCH decoder (see pdcch_plan.hpp).  Host code only, so that it can be checked on
// its own (tests/test_pdcch_host.py builds it with AddressSanitizer).
#include "pdcch_plan.hpp"

#include <algorithm>
#include <cmath>

#include "chain_gpu.hpp"
#include "lcs_internal.hpp"

namespace lcs {
namespace pdcch {

namespace {
const int kPerm[32] = {1, 17, 9, 25, 5, 21, 13, 29, 3, 19, 11, 27, 7, 23, 15, 31,
                       0, 16, 8, 24, 4, 20, 12, 28, 2, 18, 10, 26, 6, 22, 14, 30};   // 36.212 Table 5.1.4-2
}  // namespace

std::string plan_pdcch(const lcs_cell& c, uint64_t n_in, int D, double fs_in, double fc_in, double fs_programmed,
                       carrier::CellPlan& plan) {
  std::string why = carrier::plan_cell(c, n_in, D, fs_in, fc_in, fs_programmed, plan);
  if (!why.empty()) return why;
  if (c.phich_duration != 1 && c.phich_duration != 2) return "phich_duration must be 1 (normal) or 2 (extended)";
  if (c.phich_resource < 1 || c.phich_resource > 4) return "phich_resource must be 1 to 4";
  lcs_cell gc = c;                   // the positions plan_cell took its windows from
  gc.freq_fine = c.freq_superfine;
  std::vector<int> pos(TFG_MAX);
  std::vector<double> late(TFG_MAX), ts(TFG_MAX);
  double k = 0;
  int n_ofdm = 0;
  const GridTables g(pos.data(), late.data(), &k, &n_ofdm);
  const char* what = "";
  if (tfg_geometry(gc, c.fc_requested, c.fc_programmed, fs_programmed, 0xffffffffu, g, 0, ts.data(), &what) != LCS_OK)
    return std::string("no grid (") + what + ")";
  const int n_symb = c.cp_type == 1 ? 7 : 6, nm = n_max(plan.R);
  plan.q.clear();
  plan.late.clear();
  for (int t = 0; t < carrier::N_SLOT; t += 2)
    for (int l = 0; l < nm; l++) {   // inside the span of the slot's CRS windows, which plan_cell checked
      const double dl = D * ts[t * n_symb + l], q = std::rint(dl);
      plan.q.push_back((long long)q);
      plan.late.push_back(q - dl);
    }
  plan.nw = nm;
  return "";
}

int size_1a(int R) {
  const int s = 15 + ceil_log2((long long)R * (R + 1) / 2);
  for (int a : {12, 14, 16, 20, 24, 26, 32, 40, 44, 56})
    if (s == a) return s + 1;
  return s;
}

int size_1c(int R) {
  const int gap = R <= 10 ? (R + 1) / 2 : R == 11 ? 4 : R <= 19 ? 8 : R <= 26 ? 12 : R <= 44 ? 18 : R <= 63 ? 27 : R <= 79 ? 32 : 48;
  const int n = 2 * std::min(gap, R - gap) / (R < 50 ? 2 : 4);
  return (R >= 50) + ceil_log2((long long)n * (n + 1) / 2) + 5;
}

CtrlTable control_table(int R, int n_ports, int cp_type, int n_id, int phich_duration, int phich_resource, int n_ctrl) {
  const int W = 12 * R;
  auto six = [&](int l) { return l == 0 || (l == 1 && n_ports == 4) || (l == 3 && cp_type == 2); };
  // used[l][k0]: the REG of symbol l starting at k0 is the PCFICH's or the PHICH's
  std::vector<std::vector<char>> used(4, std::vector<char>(W, 0));
  for (int i = 0; i < 4; i++) used[0][(6 * (n_id % (2 * R)) + 6 * (i * R / 2)) % W] = 1;
  std::vector<std::vector<int>> avail(4);       // REG starts of symbol l not used by the PCFICH, in increasing frequency
  for (int l = 0; l < 4; l++)
    for (int k0 = 0; k0 < W; k0 += six(l) ? 6 : 4)
      if (!used[l][k0]) avail[l].push_back(k0);
  const int num[4] = {1, 1, 1, 2}, den[4] = {6, 2, 1, 1};
  const int m_u = (num[phich_resource - 1] * R + 8 * den[phich_resource - 1] - 1) / (8 * den[phich_resource - 1]);
  const int n0 = (int)avail[0].size();
  for (int m = 0; m < m_u; m++)
    for (int i = 0; i < 3; i++) {
      const int l = phich_duration == 2 ? i : 0, nl = (int)avail[l].size();
      used[l][avail[l][(n_id * nl / n0 + m + i * nl / 3) % nl]] = 1;
    }
  std::vector<std::pair<int, int>> regs;        // rule 5: (l, k0) of REG m'
  for (int k0 = 0; k0 < W; k0++)
    for (int l = 0; l < n_ctrl; l++)
      if (k0 % (six(l) ? 6 : 4) == 0 && !used[l][k0]) regs.push_back({l, k0});
  CtrlTable t;
  t.n_reg = (int)regs.size();
  t.n_cce = t.n_reg / 9;
  const int rows = (t.n_reg + 31) / 32, nd = 32 * rows - t.n_reg;
  std::vector<int> w;                           // rule 6: w'
  for (int col = 0; col < 32; col++)
    for (int r = 0; r < rows; r++) {
      const int y = r * 32 + kPerm[col];
      if (y >= nd) w.push_back(y - nd);
    }
  std::vector<int> reg_of(t.n_reg);
  for (int m = 0; m < t.n_reg; m++) reg_of[w[(m + n_id) % t.n_reg]] = m;
  const int nq = std::min(MAX_QUAD, 9 * t.n_cce);
  for (int j = 0; j < nq; j++) t.quad.push_back((uint16_t)((regs[reg_of[j]].first << 12) | regs[reg_of[j]].second));
  return t;
}

void scrambling(int n_id, int u, uint32_t* w) {
  const std::vector<uint8_t> c = lte_pn((uint32_t)u * 512 + n_id, 32 * SCR_WORDS);
  for (int i = 0; i < SCR_WORDS; i++) w[i] = 0;
  for (int b = 0; b < 32 * SCR_WORDS; b++) w[b / 32] |= (uint32_t)(c[b] & 1) << (b % 32);
}

std::vector<uint8_t> ratematch_positions(int K) {
  const int rows = (K + 31) / 32, nd = 32 * rows - K;
  std::vector<uint8_t> pos;
  for (int s = 0; s < 3; s++)
    for (int col = 0; col < 32; col++)
      for (int r = 0; r < rows; r++) {
        const int y = r * 32 + kPerm[col];
        if (y >= nd) pos.push_back((uint8_t)(s * K + y - nd));
      }
  return pos;
}

}  // namespace pdcch
}  // namespace lcs
