// chain_gpu.hpp - drivers of the companion kernels (chain_gpu.cu) on a device-resident capture buffer.
#pragma once
#include "chain_host.hpp"
#include "lcs_ctx.hpp"

namespace lcs {

struct ChainScratch {
  DevBuf<signed char> d_sss_tab;   // [168][3][2][62] +-1
  DevBuf<double2> d_pss_fd;        // [3][62]
  DevBuf<int> d_starts;
  DevBuf<double> d_kseg;           // per-segment / per-cell frequency-shift constant
  DevBuf<int3> d_par;              // per-peak {first segment, n_pss, n_id_2}
  DevBuf<int> d_nofdm;
  PinBuf<unsigned char> h_up, h_up2, h_down;   // page-locked staging (asynchronous copies, one sync per stage)
  DevBuf<double2> d_psss;          // [n_seg][62]
  DevBuf<double> d_est;            // [124] np + 4x62 complex
  DevBuf<double> d_ll;             // [4][168]
  DevBuf<double> d_late;
  DevBuf<double2> d_tfg;           // [n_ofdm][72]
};
ChainScratch& chain_scratch(lcs_ctx* ctx);

struct SssDebugHost {
  std::vector<double> est;  // [h1_np 62][h2_np 62][h1_nrm 124][h2_nrm 124][h1_ext 124][h2_ext 124]
  std::vector<double> ll;   // [nrm col0 168][nrm col1][ext col0][ext col1]
};

lcs_status dev_sss_detect(lcs_ctx* ctx, ChainScratch& cs, const void* d_cap, int fmt, uint32_t n_cap, const lcs_cell& cell,
                          double thresh2_n_sigma, double fc_req, double fc_prog, double fs_prog, lcs_cell& out,
                          SssDebugHost* dbg);
lcs_status dev_pss_sss_foe(lcs_ctx* ctx, ChainScratch& cs, const void* d_cap, int fmt, uint32_t n_cap, const lcs_cell& cell,
                           double fc_req, double fc_prog, double fs_prog, lcs_cell& out);
lcs_status dev_extract_tfg(lcs_ctx* ctx, ChainScratch& cs, const void* d_cap, int fmt, uint32_t n_cap, const lcs_cell& cell,
                           double fc_req, double fc_prog, double fs_prog, std::vector<cd>& tfg_rowmajor,
                           std::vector<double>& ts);
// The same stages for ALL peaks / cells of a capture buffer with one launch set and one synchronisation per stage.
// status[i] == LCS_ERR_RANGE marks an entry the reference would read outside the buffer for (callers skip it).
lcs_status dev_sss_detect_batch(lcs_ctx* ctx, ChainScratch& cs, const void* d_cap, int fmt, uint32_t n_cap,
                                const std::vector<lcs_cell>& cells, double thresh2_n_sigma, double fc_req, double fc_prog,
                                double fs_prog, std::vector<lcs_cell>& out, std::vector<lcs_status>& status, SssDebugHost* dbg);
lcs_status dev_pss_sss_foe_batch(lcs_ctx* ctx, ChainScratch& cs, const void* d_cap, int fmt, uint32_t n_cap,
                                 const std::vector<lcs_cell>& cells, double fc_req, double fc_prog, double fs_prog,
                                 std::vector<lcs_cell>& out);
// extract_tfg's grid: at most 854 OFDM symbols (122 slots of 7, or 732 of 6 for the extended CP) of 72 subcarriers.
constexpr int TFG_MAX = 854;
// The host geometry of extract_tfg (searcher.cpp:871-928) for one cell: pos / late / ts [n_ofdm] of every DFT window, the
// FOC constant kcell and n_ofdm.  LCS_ERR_ARG (cp_type unknown, frame_start / freq_fine not finite) or LCS_ERR_RANGE (a
// window outside [0, n_cap)), with the reason in *why; nothing else is written then.
lcs_status tfg_geometry(const lcs_cell& cell, double fc_req, double fc_prog, double fs_prog, uint32_t n_cap, int* pos,
                        double* late, double* ts, double* kcell, int* n_ofdm, const char** why);
// One tfg_kernel launch over n_cells cells (asynchronous on st): d_pos / d_late [cell][TFG_MAX] from tfg_geometry, d_k and
// d_nofdm [cell]; the grids land in d_tfg [cell][TFG_MAX][72] (1/sqrt(128) DFT scaling).  d_base [cell] (NULL: all 0) is
// the sample index in d_cap at which the cell's capture buffer starts.  A format other than cu8, cf32 or c128 launches
// nothing and returns LCS_ERR_ARG.
lcs_status launch_tfg(const void* d_cap, int fmt, const uint64_t* d_base, const int* d_pos, const double* d_late,
                      const double* d_k, const int* d_nofdm, uint32_t n_cells, double2* d_tfg, cudaStream_t st);
lcs_status dev_extract_tfg_batch(lcs_ctx* ctx, ChainScratch& cs, const void* d_cap, int fmt, uint32_t n_cap,
                                 const std::vector<lcs_cell>& cells, double fc_req, double fc_prog, double fs_prog,
                                 std::vector<std::vector<cd>>& tfg_rowmajor, std::vector<std::vector<double>>& ts,
                                 std::vector<lcs_status>& status);

}  // namespace lcs
