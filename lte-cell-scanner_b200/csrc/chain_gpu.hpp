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
lcs_status dev_extract_tfg_batch(lcs_ctx* ctx, ChainScratch& cs, const void* d_cap, int fmt, uint32_t n_cap,
                                 const std::vector<lcs_cell>& cells, double fc_req, double fc_prog, double fs_prog,
                                 std::vector<std::vector<cd>>& tfg_rowmajor, std::vector<std::vector<double>>& ts,
                                 std::vector<lcs_status>& status);

}  // namespace lcs
