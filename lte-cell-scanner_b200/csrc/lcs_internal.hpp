// lcs_internal.hpp - shared declarations between the C-ABI layer (lcs_api.cu) and the kernels.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>

#include <complex>
#include <string>
#include <vector>

#include "../../include/lcs_b200.h"

namespace lcs {

typedef std::complex<double> cd;

// ---- geometry of the fused FP32 correlator (xcorr_fp32.cu) ----
constexpr int XC_R = 7;                 // lags per lane (7*8 B stride is LDS.64 bank-conflict free)
constexpr int XC_TI = 32 * XC_R;        // 224 fold positions per block
constexpr int XC_FW = 8;                // warps per block: fw frequency hypotheses x (8/fw) lag sub-tiles, fw = 8 or 1
constexpr int XC_NTAP_PAD = 140;        // 137 taps zero-padded to a multiple of XC_R
constexpr int XC_THREADS = 32 * XC_FW;
constexpr int XC_TAP_BLOCK = 28;        // taps per partial sum of the two-level accumulation (4 x XC_R)

// Geometry shared by all plans of a plan set (one capture-buffer shape, one ds_comb_arm).  Arrays that depend on the
// plan (templates, fold offsets) are indexed [plan][...][n_f_stride]; a plan with fewer hypotheses leaves the tail unused.
struct XcorrGeom {
  uint32_t n_cap, n_comb_xc, n_comb_sp, ds_comb_arm;
  uint32_t n_f_stride;      // hypotheses per plan the arrays are laid out for (max over the plans)
  uint32_t n_fchunk;        // ceil(n_f_stride / fw)
  uint32_t fw;              // hypotheses per block of the FP32 correlator: 8, or 1 for the single-hypothesis (tracker) shape
  uint32_t tile_len;        // staged samples per (block, half-frame)
  uint32_t max_spread;
};

// Per-launch view of a plan set for the kernels that follow the correlator.
struct PlanView {
  const int* d_nf;            // [n_plans] hypotheses of each plan
  const uint32_t* d_buf_plan; // [batch] plan of each capture buffer (NULL: every buffer uses plan 0)
};

// Launchers (all asynchronous on `st`); return the number of kernel launches they issued.  The caller checks iq_format
// first (SearchFormats::has): for any other format they launch nothing and return 0.
int launch_xcorr_fold_fp32(const XcorrGeom& g, const PlanView& pv, const void* d_iq, int iq_format, uint32_t batch,
                           const float4* d_w01, const float2* d_w2, const int* d_soff, const int* d_smin,
                           float* d_single_planar, cudaStream_t st);
int launch_sp_fold(const XcorrGeom& g, const void* d_iq, int iq_format, uint32_t batch, double* d_sp_incoherent,
                   cudaStream_t st);
int launch_epilogue(const XcorrGeom& g, const PlanView& pv, uint32_t batch, const float* d_single_planar, double* d_pow,
                    int32_t* d_frq, float* d_incoherent_planar, cudaStream_t st);
// ref-layout conversions for the drop-in host call
int launch_planar_to_ref(const XcorrGeom& g, const float* d_planar, float* d_ref, cudaStream_t st);
int launch_xc_debug(const XcorrGeom& g, const void* d_iq, int iq_format, const float4* d_w01, const float2* d_w2,
                    float2* d_xc, cudaStream_t st);
int launch_sp_debug(const XcorrGeom& g, const void* d_iq, int iq_format, double* d_sp, cudaStream_t st);
void xcorr_fp32_init();   // one-time function attributes

// ---- host-side tables (lte_tables.cpp) ----
void pss_fd(int n_id_2, cd out[62]);            // lte_lib.cpp:155-161
void pss_td(int n_id_2, cd out[137]);           // lte_lib.cpp:177-188
void sss_fd(int n_id_1, int n_id_2, int slot, int out[62]);  // lte_lib.cpp:199-257
std::vector<uint8_t> lte_pn(uint32_t c_init, uint32_t len);  // lte_lib.cpp:41-147
double chi2cdf_inv(double p, double k);         // dsp.h:188-193

}  // namespace lcs
