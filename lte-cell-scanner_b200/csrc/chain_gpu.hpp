// chain_gpu.hpp - drivers of the companion kernels (chain_gpu.cu) on a device-resident capture buffer.
#pragma once
#include "chain_host.hpp"
#include "lcs_ctx.hpp"

namespace lcs {

// One call of the per-peak stages: the capture buffer on the device, the configuration its peaks were found with, and
// the stream the stage's copies and kernels run on.  The stages use the context's scratch (ctx->chain).
struct StageCall {
  lcs_ctx* ctx;
  const void* d_cap;
  int fmt;
  uint32_t n_cap;
  const PlanCfg& cfg;              // fc_req, fc_prog, fs_prog
  cudaStream_t st;
};

struct SssDebugHost {
  std::vector<double> est;  // [h1_np 62][h2_np 62][h1_nrm 124][h2_nrm 124][h1_ext 124][h2_ext 124]
  std::vector<double> ll;   // [nrm col0 168][nrm col1][ext col0][ext col1]
};

// The stages for ALL peaks / cells of a capture buffer with one launch set and one synchronisation per stage.
// status[i] == LCS_ERR_RANGE marks an entry the reference would read outside the buffer for (callers skip it).
lcs_status dev_sss_detect_batch(const StageCall& sc, const std::vector<lcs_cell>& cells, double thresh2_n_sigma,
                                std::vector<lcs_cell>& out, std::vector<lcs_status>& status, SssDebugHost* dbg);
lcs_status dev_pss_sss_foe_batch(const StageCall& sc, const std::vector<lcs_cell>& cells, std::vector<lcs_cell>& out);
lcs_status dev_extract_tfg_batch(const StageCall& sc, const std::vector<lcs_cell>& cells,
                                 std::vector<std::vector<cd>>& tfg_rowmajor, std::vector<std::vector<double>>& ts,
                                 std::vector<lcs_status>& status);
// sss_detect -> pss_sss_foe -> extract_tfg -> tfoec -> decode_mib for the PSS peaks pk of one capture buffer.
lcs_status cell_chain_dev(const StageCall& sc, const std::vector<lcs_cell>& pk, lcs_cell* cells, uint32_t max_cells,
                          uint32_t* n_cells, const int32_t* tracked = nullptr, uint32_t n_tracked = 0, bool tracker_cycle = false);

// extract_tfg's grid: at most 854 OFDM symbols (122 slots of 7, or 732 of 6 for the extended CP) of 72 subcarriers.
constexpr int TFG_MAX = 854;
// The host tables of a grid launch, slices of a Staging: pos / late [cell][TFG_MAX], k / n_ofdm [cell], filled through
// tfg_geometry, and base [cell] (NULL: all 0), the sample of the device buffer at which the cell's capture buffer starts.
struct GridTables {
  int* pos;
  double* late;
  double* k;
  int* n_ofdm;
  uint64_t* base;
  static size_t bytes(size_t n_cells) { return n_cells * (TFG_MAX * 12 + 20) + 5 * 16; }   // Staging::reset
  GridTables(Staging& up, size_t n_cells, bool with_base);
  // Over caller-owned host arrays, for geometry that is not uploaded: pos / late [n_cells][TFG_MAX], k / n_ofdm [n_cells].
  GridTables(int* pos_, double* late_, double* k_, int* n_ofdm_) : pos(pos_), late(late_), k(k_), n_ofdm(n_ofdm_), base(nullptr) {}
};
// The host geometry of extract_tfg (searcher.cpp:871-928) for one cell, into slot `slot` of g: pos / late and ts [n_ofdm]
// of every DFT window, the FOC constant k and n_ofdm.  LCS_ERR_ARG (cp_type unknown, frame_start / freq_fine not finite)
// or LCS_ERR_RANGE (a window outside [0, n_cap)), with the reason in *why; the slot's k and n_ofdm are not written then.
lcs_status tfg_geometry(const lcs_cell& cell, double fc_req, double fc_prog, double fs_prog, uint32_t n_cap, const GridTables& g,
                        size_t slot, double* ts, const char** why);
// One tfg_kernel launch over the first n_cells cells of g, once `up` has been uploaded on st (asynchronous); the grids
// land in d_tfg [cell][TFG_MAX][72] (1/sqrt(128) DFT scaling).  A format other than cu8, cf32 or c128 launches nothing
// and fails with LCS_ERR_ARG and the message bad_fmt.
lcs_status launch_grids(lcs_ctx* ctx, const Staging& up, const GridTables& g, uint32_t n_cells, const void* d_cap, int fmt,
                        double2* d_tfg, cudaStream_t st, const char* bad_fmt);

}  // namespace lcs
