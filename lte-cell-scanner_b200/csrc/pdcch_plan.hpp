// pdcch_plan.hpp - host planning of the PDCCH decoder (pdcch.cu, contract in include/lcs_pdcch.h): a cell's windows, its
// control-region tables, its DCI sizes and scrambling, with no device work (a decoded DCI's fields: dci_fields.hpp).
#pragma once
#include <cstdint>
#include <string>
#include <vector>

#include "../../include/lcs_pdcch.h"
#include "carrier_plan.hpp"
#include "dci_fields.hpp"

namespace lcs {
namespace pdcch {

constexpr int MAX_QUAD = 144;        // the common search space: 16 CCEs of 9 quadruplets
constexpr int MAX_K = 44;            // the longest 1A (28 bits) plus its CRC
constexpr int SCR_WORDS = 36;        // 72 * 16 scrambling bits per subframe number

// Rule 1's largest control region: 4 symbols when R <= 10, else 3.
inline int n_max(int R) { return R <= 10 ? 4 : 3; }

// plan_cell's checks and the PHICH fields' (rules of lcs_pdcch.h), then the windows of symbols 0 to n_max - 1 of every
// even slot, in that order: "" or why not.  Symbol 0 (and 1) equal those of the PCFICH decoder.
std::string plan_pdcch(const lcs_cell& c, uint64_t n_in, int D, double fs_in, double fc_in, double fs_programmed,
                       carrier::CellPlan& plan);

// Rule 9: DCI sizes in bits.
int size_1a(int R);
int size_1c(int R);

// Rules 2-6 for a control region of n_ctrl symbols.  quad[j], j < min(MAX_QUAD, 9 n_cce), is (l << 12) | k0: the symbol
// and first column of the REG carrying quadruplet j.
struct CtrlTable {
  int n_reg = 0, n_cce = 0;
  std::vector<uint16_t> quad;
};
CtrlTable control_table(int R, int n_ports, int cp_type, int n_id, int phich_duration, int phich_resource, int n_ctrl);

// Rule 10's scrambling of subframe number u: bit b of the 72 * 16 bits at bit b % 32 of w[b / 32].
void scrambling(int n_id, int u, uint32_t* w);

// 36.212 5.1.4.2: pos[i], i < 3K, the coded bit (row j * K + column k of the [3][K] block) of rate-matched bit i; bit
// i + 3K m is the same coded bit again.
std::vector<uint8_t> ratematch_positions(int K);

}  // namespace pdcch
}  // namespace lcs
