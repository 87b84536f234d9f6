// sib1_plan.hpp - host planning of the SIB1 decoder (sib1.cu, contract in include/lcs_sib1.h): a cell's windows and
// occasions, its PDSCH scrambling, and the parsing of a decoded SIB1, with no device work.
#pragma once
#include <cstdint>
#include <string>

#include "../../include/lcs_sib1.h"
#include "carrier_plan.hpp"

namespace lcs {
namespace sib1 {

constexpr int SCR_WORDS = 100 * 12 * 14 * 2 / 32;    // the scrambling bits of the largest allocation

// Rule 1: the grid subframes of the occasions of a cell whose grid frame 0 has SFN sfn.
void occasions(int sfn, int* sf);

// plan_pdcch's checks and windows, the sfn check, then the windows of all 2 n_symb symbols of each occasion after them,
// occasion by occasion: "" or why not.
std::string plan_sib1(const lcs_cell& c, uint64_t n_in, int D, double fs_in, double fc_in, double fs_programmed,
                      carrier::CellPlan& plan);

// Rule 6's scrambling: bit b at bit b % 32 of w[b / 32], b < 32 SCR_WORDS.
void scrambling(int n_id, uint32_t* w);

// Rule 9: the SIB1 fields of tb [n_bytes] into m (n_plmn and every field after it); false (parse_ok = 0) when it is not
// SIB1 or its bits run out, and then those fields are all 0.
bool parse_sib1(const uint8_t* tb, int n_bytes, lcs_sib1_meas& m);

}  // namespace sib1
}  // namespace lcs
