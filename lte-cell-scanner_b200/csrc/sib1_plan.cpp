// sib1_plan.cpp - host planning of the SIB1 decoder (see sib1_plan.hpp).  Host code only, so that it can be checked on its
// own with AddressSanitizer.
#include "sib1_plan.hpp"

#include <cstddef>
#include <cstring>
#include <vector>

#include "chain_gpu.hpp"
#include "lcs_internal.hpp"
#include "pdcch_plan.hpp"

namespace lcs {
namespace sib1 {

void occasions(int sfn, int* sf) {
  for (int f = 0, n = 0; f < 6; f++)
    if ((sfn + f) % 2 == 0) sf[n++] = 10 * f + 5;
}

std::string plan_sib1(const lcs_cell& c, uint64_t n_in, int D, double fs_in, double fc_in, double fs_programmed,
                      carrier::CellPlan& plan) {
  std::string why = pdcch::plan_pdcch(c, n_in, D, fs_in, fc_in, fs_programmed, plan);
  if (!why.empty()) return why;
  if (c.sfn < 0 || c.sfn > 1023) return "sfn must be 0 to 1023";
  lcs_cell gc = c;                   // the positions plan_pdcch took its windows from
  gc.freq_fine = c.freq_superfine;
  std::vector<int> pos(TFG_MAX);
  std::vector<double> late(TFG_MAX), ts(TFG_MAX);
  double k = 0;
  int n_ofdm = 0;
  const GridTables g(pos.data(), late.data(), &k, &n_ofdm);
  const char* what = "";
  if (tfg_geometry(gc, c.fc_requested, c.fc_programmed, fs_programmed, 0xffffffffu, g, 0, ts.data(), &what) != LCS_OK)
    return std::string("no grid (") + what + ")";
  const int n_symb = c.cp_type == 1 ? 7 : 6;
  int sf[LCS_SIB1_OCCASIONS];
  occasions(c.sfn, sf);
  for (int o = 0; o < LCS_SIB1_OCCASIONS; o++)
    for (int l = 0; l < 2 * n_symb; l++) {   // plan_cell checked every symbol's window against the recording
      const double dl = D * ts[2 * sf[o] * n_symb + l], q = std::rint(dl);
      plan.q.push_back((long long)q);
      plan.late.push_back(q - dl);
    }
  return "";
}

void scrambling(int n_id, uint32_t* w) {
  const std::vector<uint8_t> c = lte_pn(0xFFFFu * 16384u + 5u * 512u + (uint32_t)n_id, 32 * SCR_WORDS);
  for (int i = 0; i < SCR_WORDS; i++) w[i] = 0;
  for (int b = 0; b < 32 * SCR_WORDS; b++) w[b / 32] |= (uint32_t)(c[b] & 1) << (b % 32);
}

namespace {
// An MSB-first bit reader that records running out instead of reading past the end.
struct Bits {
  const uint8_t* p;
  int n, at = 0;
  bool over = false;
  uint32_t get(int w) {
    uint32_t v = 0;
    for (int i = 0; i < w; i++, at++) {
      if (at >= n) {
        over = true;
        return 0;
      }
      v = (v << 1) | ((p[at >> 3] >> (7 - (at & 7))) & 1u);
    }
    return v;
  }
};
}  // namespace

namespace {
bool parse_fields(const uint8_t* tb, int n_bytes, lcs_sib1_meas& m) {
  Bits b{tb, 8 * n_bytes};
  if (b.get(1) != 0 || b.get(1) != 1) return false;            // BCCH-DL-SCH-MessageType: c1, systemInformationBlockType1
  const uint32_t has_pmax = b.get(1), has_tdd = b.get(1), has_nce = b.get(1);
  m.csg_identity_present = b.get(1);                           // cellAccessRelatedInfo
  m.n_plmn = b.get(3) + 1;
  if (m.n_plmn > LCS_SIB1_MAX_PLMN) return false;
  uint32_t mcc = 0;
  for (uint32_t i = 0; i < m.n_plmn; i++) {
    lcs_sib1_plmn& p = m.plmn[i];
    if (b.get(1)) {
      mcc = 0;
      for (int d = 0; d < 3; d++) mcc = 10 * mcc + b.get(4);
    }
    p.mcc = mcc;
    p.mnc_digits = b.get(1) + 2;
    p.mnc = 0;
    for (uint32_t d = 0; d < p.mnc_digits; d++) p.mnc = 10 * p.mnc + b.get(4);
    p.reserved = b.get(1) == 0;
  }
  m.tac = b.get(16);
  m.cell_identity = b.get(28);
  m.cell_barred = b.get(1) == 0;
  m.intra_freq_reselection = b.get(1) == 0;
  m.csg_indication = b.get(1);
  m.csg_identity = m.csg_identity_present ? b.get(27) : 0;
  const uint32_t has_offset = b.get(1);                        // cellSelectionInfo
  m.q_rx_lev_min = (int32_t)b.get(6) - 70;
  m.q_rx_lev_min_offset = has_offset ? b.get(3) + 1 : 0;
  m.p_max_present = has_pmax;
  m.p_max = has_pmax ? (int32_t)b.get(6) - 30 : 0;
  m.freq_band_indicator = b.get(6) + 1;
  m.n_si = b.get(5) + 1;                                       // schedulingInfoList
  for (uint32_t i = 0; i < m.n_si; i++) {
    const uint32_t per = b.get(3);
    if (per > 6) return false;
    m.si_periodicity[i] = 8u << per;
    m.si_sib_mask[i] = 0;
    const uint32_t n = b.get(5);
    for (uint32_t j = 0; j < n; j++) {
      if (b.get(1)) return false;                              // SIB-Type beyond the Rel-8 root
      m.si_sib_mask[i] |= 1u << (b.get(4) + 3);
    }
  }
  m.tdd_present = has_tdd;
  if (has_tdd) {
    m.tdd_subframe_assignment = b.get(3);
    m.tdd_special_subframe_patterns = b.get(4);
  }
  const int win[8] = {1, 2, 5, 10, 15, 20, 40, 0};
  m.si_window_ms = (uint32_t)win[b.get(3)];
  m.system_info_value_tag = b.get(5);
  m.non_critical_extension = has_nce;
  return !b.over && m.si_window_ms != 0 && m.q_rx_lev_min <= -22 && m.freq_band_indicator <= 64;
}
}  // namespace

bool parse_sib1(const uint8_t* tb, int n_bytes, lcs_sib1_meas& m) {
  lcs_sib1_meas t;                               // the parsed fields, n_plmn on, all 0 unless the whole parse succeeds
  std::memset(&t, 0, sizeof t);
  const bool ok = tb && n_bytes > 0 && parse_fields(tb, n_bytes, t);
  const size_t at = offsetof(lcs_sib1_meas, n_plmn);
  if (ok)
    std::memcpy(reinterpret_cast<char*>(&m) + at, reinterpret_cast<const char*>(&t) + at, sizeof m - at);
  else
    std::memset(reinterpret_cast<char*>(&m) + at, 0, sizeof m - at);
  return ok;
}

}  // namespace sib1
}  // namespace lcs
