// xcorr_fp32.cu - fused PSS correlator on the FP32 CUDA cores (general-input path).
//
// Replaces xc_correlate + xc_combine + xc_delay_spread + sp_est + xc_peak_freq of the reference
// (src/searcher.cpp:113-383) with three kernels:
//
//   xcorr_fold_fp32   correlate the capture buffer against 3 PSS roots x n_f frequency hypotheses
//                     (137 complex taps) and accumulate |xc|^2 over the n_comb half frames IN
//                     REGISTERS - the 3 x (n_cap-136) x n_f complex `xc` array of the reference
//                     (136 MB at n_f=37) is never materialised.  Output: xc_incoherent_single,
//                     planar layout [batch][3][n_f][9600].
//   sp_partial        sliding 274-sample signal power per half frame (sp_est), FP64.
//   epilogue          delay-spread box filter (same float summation order as searcher.cpp:330-343),
//                     strict-> first-max over f (searcher.cpp:369-382), sp fold + 137-sample shift.
//
// Work decomposition of xcorr_fold_fp32: a block owns 224 consecutive fold positions (idx) and 8
// frequency hypotheses (one per warp); each lane owns 7 consecutive idx x 3 roots.  For every half
// frame m the block stages the samples it needs into shared memory once (coalesced 128-bit loads /
// byte loads converted in flight), then each lane slides a 7-sample register window across the
// 137 taps: per tap 1 LDS.64 (new sample) + LDS.128 + LDS.64 (3 template taps, warp broadcast) feed
// 21 complex MACs = 84 FFMA.  The k_factor-dependent fold offsets round_i(m*.005*k_f*fs)
// (searcher.cpp:298) differ per hypothesis; each warp simply offsets its window into the shared
// tile.  A 7-sample (56 B) lane stride makes the LDS.64 window loads bank-conflict free.
#include <assert.h>

#include "iq_format.cuh"
#include "lcs_internal.hpp"

namespace lcs {

__device__ __forceinline__ void cmac(float2& acc, const float wx, const float wy, const float2 x) {
  acc.x = fmaf(wx, x.x, acc.x);
  acc.x = fmaf(-wy, x.y, acc.x);
  acc.y = fmaf(wx, x.y, acc.y);
  acc.y = fmaf(wy, x.x, acc.y);
}

template <int FMT, int FW>
__global__ void __launch_bounds__(XC_THREADS, 2)
xcorr_fold_fp32_kernel(const void* __restrict__ iq, const float4* __restrict__ w01g_all, const float2* __restrict__ w2g_all,
                       const int* __restrict__ soff_all, const int* __restrict__ smin_all, float* __restrict__ single_planar,
                       const int* __restrict__ plan_nf, const uint32_t* __restrict__ buf_plan,
                       const uint32_t n_cap, const uint32_t n_f_stride, const uint32_t n_comb, const uint32_t n_fchunk,
                       const uint32_t tile_len) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float4* w01s = reinterpret_cast<float4*>(smem_raw);                        // [FW][NTAP_PAD] roots 0,1
  float2* w2s = reinterpret_cast<float2*>(w01s + FW * XC_NTAP_PAD);          // [FW][NTAP_PAD] root 2
  float* part = reinterpret_cast<float*>(w2s + FW * XC_NTAP_PAD);            // [42][XC_THREADS] second-level partial sums
  float2* tile = reinterpret_cast<float2*>(part + 6 * XC_R * XC_THREADS);    // [tile_len]

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const uint32_t fchunk = blockIdx.y, b = blockIdx.z;
  // operands of this buffer's plan
  const uint32_t plan = buf_plan ? __ldg(buf_plan + b) : 0u;
  const uint32_t n_f = (uint32_t)__ldg(plan_nf + plan);
  if (fchunk * FW >= n_f) return;                                            // block-uniform: this plan has fewer hypotheses
  const float4* w01g = w01g_all + (size_t)plan * n_f_stride * XC_NTAP_PAD;
  const float2* w2g = w2g_all + (size_t)plan * n_f_stride * XC_NTAP_PAD;
  const int* soff = soff_all + (size_t)plan * n_comb * n_f_stride;
  const int* smin_tab = smin_all + (size_t)plan * n_comb * n_fchunk;
  // warp -> (hypothesis fsub of the chunk, lag sub-tile lsub of the block)
  const int fsub = warp % FW, lsub = warp / FW;
  const uint32_t f = fchunk * FW + fsub;
  const bool f_ok = f < n_f;
  const uint32_t fcl = f_ok ? f : n_f - 1;
  const uint32_t i0_blk = blockIdx.x * (XC_TI * (XC_FW / FW));
  const uint32_t i0 = i0_blk + lsub * XC_TI;
  const size_t iq_base = (size_t)b * n_cap;

  for (int i = tid; i < FW * XC_NTAP_PAD; i += XC_THREADS) {
    const uint32_t fw = i / XC_NTAP_PAD, tap = i - fw * XC_NTAP_PAD;
    uint32_t ff = fchunk * FW + fw;
    ff = ff < n_f ? ff : n_f - 1;
    w01s[i] = __ldg(w01g + (size_t)ff * XC_NTAP_PAD + tap);
    w2s[i] = __ldg(w2g + (size_t)ff * XC_NTAP_PAD + tap);
  }

  float pw[3][XC_R];
#pragma unroll
  for (int t = 0; t < 3; t++)
#pragma unroll
    for (int j = 0; j < XC_R; j++) pw[t][j] = 0.f;

  const float4* w01w = w01s + fsub * XC_NTAP_PAD;
  const float2* w2w = w2s + fsub * XC_NTAP_PAD;

  for (uint32_t m = 0; m < n_comb; m++) {
    const int smin = __ldg(smin_tab + m * n_fchunk + fchunk);
    const int off = __ldg(soff + m * n_f_stride + fcl) - smin;
    __syncthreads();  // everyone is done with the previous tile (and, for m==0, the W stores are issued)
    for (uint32_t e = tid; e < tile_len; e += XC_THREADS) {
      const size_t g = (size_t)i0_blk + smin + e;
      tile[e] = g < n_cap ? load_iq<FMT>(iq, iq_base + g) : make_float2(0.f, 0.f);
    }
    __syncthreads();

    const float2* xp = tile + off + lsub * XC_TI + lane * XC_R;
    float2 acc[3][XC_R];
#pragma unroll
    for (int t = 0; t < 3; t++)
#pragma unroll
      for (int j = 0; j < XC_R; j++) acc[t][j] = make_float2(0.f, 0.f);
    float2 win[XC_R];
#pragma unroll
    for (int j = 0; j < XC_R - 1; j++) win[j] = xp[j];

    // Two-level summation: the 140 taps are accumulated in blocks of XC_TAP_BLOCK = 28; after each block the 42 register
    // accumulators are added into per-thread partial sums in shared memory and cleared.  The rounding error of an FP32
    // chain grows with the magnitude of its running sum, so five short chains plus five adds are ~2x more accurate than
    // one chain of 274 FMAs (measured margin to the 1e-6 contract in DESIGN.md) for ~5 % more instructions.
    float* mypart = part + tid;
#pragma unroll 1
    for (int tb0 = 0; tb0 < XC_NTAP_PAD; tb0 += XC_TAP_BLOCK) {
#pragma unroll 1
      for (int tb = tb0; tb < tb0 + XC_TAP_BLOCK; tb += XC_R) {
#pragma unroll
        for (int u = 0; u < XC_R; u++) {
          win[(u + XC_R - 1) % XC_R] = xp[tb + u + XC_R - 1];
          const float4 wa = w01w[tb + u];
          const float2 wb = w2w[tb + u];
#pragma unroll
          for (int j = 0; j < XC_R; j++) {
            const float2 x = win[(u + j) % XC_R];
            cmac(acc[0][j], wa.x, wa.y, x);
            cmac(acc[1][j], wa.z, wa.w, x);
            cmac(acc[2][j], wb.x, wb.y, x);
          }
        }
      }
      const bool first = tb0 == 0, last = tb0 + XC_TAP_BLOCK >= XC_NTAP_PAD;
#pragma unroll
      for (int t = 0; t < 3; t++)
#pragma unroll
        for (int j = 0; j < XC_R; j++) {
          float* q = mypart + ((t * XC_R + j) * 2) * XC_THREADS;
          float2 s = acc[t][j];
          if (!first) { s.x = __fadd_rn(q[0], s.x); s.y = __fadd_rn(q[XC_THREADS], s.y); }
          if (!last) { q[0] = s.x; q[XC_THREADS] = s.y; acc[t][j] = make_float2(0.f, 0.f); }
          else acc[t][j] = s;
        }
    }
    // IT++ sqr(complex<float>) then float += : re*re+im*im, un-fused  (searcher.cpp:300)
#pragma unroll
    for (int t = 0; t < 3; t++)
#pragma unroll
      for (int j = 0; j < XC_R; j++)
        pw[t][j] = __fadd_rn(pw[t][j], __fadd_rn(__fmul_rn(acc[t][j].x, acc[t][j].x), __fmul_rn(acc[t][j].y, acc[t][j].y)));
  }

  if (f_ok) {
    const float ncf = (float)n_comb;
#pragma unroll
    for (int t = 0; t < 3; t++) {
      float* dst = single_planar + (((size_t)b * 3 + t) * n_f_stride + f) * LCS_N_FOLD;
#pragma unroll
      for (int j = 0; j < XC_R; j++) {
        const uint32_t idx = i0 + lane * XC_R + j;
        if (idx < LCS_N_FOLD) dst[idx] = __fdiv_rn(pw[t][j], ncf);  // searcher.cpp:304
      }
    }
  }
}

static size_t fp32_smem(uint32_t fw, uint32_t tile_len) {
  return (size_t)fw * XC_NTAP_PAD * (sizeof(float4) + sizeof(float2)) + (size_t)6 * XC_R * XC_THREADS * sizeof(float) +
         (size_t)tile_len * sizeof(float2);
}
void xcorr_fp32_init() {
  const int cap = 100 * 1024;     // planset_build rejects grids that would need more
  SearchFormats::each([&](auto FMT) {
    cudaFuncSetAttribute(xcorr_fold_fp32_kernel<FMT, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, cap);
    cudaFuncSetAttribute(xcorr_fold_fp32_kernel<FMT, XC_FW>, cudaFuncAttributeMaxDynamicSharedMemorySize, cap);
  });
}

int launch_xcorr_fold_fp32(const XcorrGeom& g, const PlanView& pv, const void* d_iq, int iq_format, uint32_t batch,
                           const float4* d_w01, const float2* d_w2, const int* d_soff, const int* d_smin,
                           float* d_single_planar, cudaStream_t st) {
  const size_t smem = fp32_smem(g.fw, g.tile_len);
  const uint32_t ti_blk = XC_TI * (XC_FW / g.fw);
  dim3 grid((LCS_N_FOLD + ti_blk - 1) / ti_blk, g.n_fchunk, batch), block(XC_THREADS);
  const auto launch = [&](auto kernel) {
    kernel<<<grid, block, smem, st>>>(d_iq, d_w01, d_w2, d_soff, d_smin, d_single_planar, pv.d_nf, pv.d_buf_plan, g.n_cap,
                                      g.n_f_stride, g.n_comb_xc, g.n_fchunk, g.tile_len);
  };
  return SearchFormats::dispatch(iq_format, [&](auto FMT) {
    if (g.fw == 1) launch(xcorr_fold_fp32_kernel<FMT, 1>);
    else launch(xcorr_fold_fp32_kernel<FMT, XC_FW>);
  }) == LCS_OK;
}

// ------------------------------------------------------------------------------------------
// sp_est  (searcher.cpp:185-221): sp[t] = mean_{j<274} |x[t+j]|^2 for t < n_comb_sp*9600, folded by 9600, averaged and
// shifted right by 137 (:213-220).  FP64 like the reference.
// One block = 1024 consecutive fold positions: for every half frame m the 1024+273 sample powers are summed with a
// block-wide FP64 prefix scan, sp[t] = (S[t+274]-S[t])/274, and the fold  sp[0][i] + sp[1][i] + ...  is accumulated in
// registers in the reference's order - only sp_incoherent is written.  For 8-bit IQ every term is a multiple of 2^-14
// and every partial sum (< 2^7) is exact in double, so sp[t] is the exactly rounded quotient.
// ------------------------------------------------------------------------------------------
constexpr int SP_TILE = 1024;
constexpr int SP_THREADS = 256;
constexpr int SP_ITEMS = 6;        // 256*6 = 1536 >= 1024+273

template <int FMT>
__device__ __forceinline__ double pwr(const void* __restrict__ iq, size_t i) {
  if constexpr (FMT == LCS_IQ_C128) {  // keep the IT++ doubles: sp_est is an FP64 routine in the reference
    const double2 v = load_c<FMT>(iq, i);
    return v.x * v.x + v.y * v.y;
  }
  const float2 v = load_iq<FMT>(iq, i);
  return (double)v.x * (double)v.x + (double)v.y * (double)v.y;
}

// Element type of the prefix scan: for raw 8-bit IQ the sample power (I-127)^2 + (Q-127)^2 is an integer <= 2*128^2 and a
// prefix sum over a tile (< 2^26) fits int32, so the scan runs in integers (exact, a third of the FP64 instructions);
// sp = isum * 2^-14 / 274 is then the same exactly rounded quotient the reference's double recursion produces.
template <int FMT> struct SpAcc { typedef double T; };
template <> struct SpAcc<LCS_IQ_CU8> { typedef int T; };
template <int FMT>
__device__ __forceinline__ typename SpAcc<FMT>::T sp_term(const void* __restrict__ iq, size_t i) { return pwr<FMT>(iq, i); }
template <>
__device__ __forceinline__ int sp_term<LCS_IQ_CU8>(const void* __restrict__ iq, size_t i) {
  const int2 v = load_cu8(iq, i);
  return v.x * v.x + v.y * v.y;
}

template <int FMT>
__global__ void __launch_bounds__(SP_THREADS) sp_fold_kernel(const void* __restrict__ iq, double* __restrict__ sp_incoherent,
                                                             const uint32_t n_cap, const uint32_t n_comb_sp) {
  typedef typename SpAcc<FMT>::T T;
  __shared__ T ps[SP_THREADS * SP_ITEMS + 1];   // exclusive prefix sums
  __shared__ T wsum[SP_THREADS / 32];
  const uint32_t b = blockIdx.y, tid = threadIdx.x;
  const uint32_t i_base = blockIdx.x * SP_TILE;
  const uint32_t n_pos = min((uint32_t)SP_TILE, LCS_N_FOLD - i_base);
  const uint32_t n_need = n_pos + 273;               // samples this block touches per half frame (all < n_cap)
  const double unit = FMT == LCS_IQ_CU8 ? 1.0 / 16384.0 : 1.0;
  double acc[SP_TILE / SP_THREADS];
  // the loads of half frame m+1 are issued before the scan of half frame m (the scan's barriers would otherwise expose the
  // full global-memory latency fifteen times per block)
  T nxt[SP_ITEMS];
#pragma unroll
  for (int k = 0; k < SP_ITEMS; k++) {
    const uint32_t e = tid * SP_ITEMS + k;
    nxt[k] = e < n_need ? sp_term<FMT>(iq, (size_t)b * n_cap + i_base + e) : (T)0;
  }
  for (uint32_t m = 0; m < n_comb_sp; m++) {
    T v[SP_ITEMS], run = 0;
#pragma unroll
    for (int k = 0; k < SP_ITEMS; k++) {
      v[k] = nxt[k];
      run += v[k];
    }
    if (m + 1 < n_comb_sp) {
      const size_t base = (size_t)b * n_cap + (size_t)(m + 1) * LCS_N_FOLD + i_base;
#pragma unroll
      for (int k = 0; k < SP_ITEMS; k++) {
        const uint32_t e = tid * SP_ITEMS + k;
        nxt[k] = e < n_need ? sp_term<FMT>(iq, base + e) : (T)0;
      }
    }
    // block exclusive scan of the per-thread totals
    T incl = run;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const T t = __shfl_up_sync(0xffffffffu, incl, o);
      if ((tid & 31) >= (uint32_t)o) incl += t;
    }
    __syncthreads();                                 // the previous half frame's prefix sums have been consumed
    if ((tid & 31) == 31) wsum[tid >> 5] = incl;
    __syncthreads();
    T woff = 0;
    for (uint32_t w = 0; w < (tid >> 5); w++) woff += wsum[w];
    T a = woff + incl - run;
#pragma unroll
    for (int k = 0; k < SP_ITEMS; k++) {
      ps[tid * SP_ITEMS + k] = a;
      a += v[k];
    }
    if (tid == SP_THREADS - 1) ps[SP_THREADS * SP_ITEMS] = a;
    __syncthreads();
#pragma unroll
    for (int k = 0; k < SP_TILE / SP_THREADS; k++) {
      const uint32_t i = tid + k * SP_THREADS;
      const double sp = ((double)(ps[i + 274] - ps[i]) * unit) / 274;
      acc[k] = m == 0 ? sp : acc[k] + sp;            // searcher.cpp:213-216: sp_incoherent = sp(0..9599) + sp(9600..) + ...
    }
  }
#pragma unroll
  for (int k = 0; k < SP_TILE / SP_THREADS; k++) {
    const uint32_t i = tid + k * SP_THREADS;
    if (i < n_pos) sp_incoherent[(size_t)b * LCS_N_FOLD + (i_base + i + 137) % LCS_N_FOLD] = acc[k] / n_comb_sp;   // :217-220
  }
}

int launch_sp_fold(const XcorrGeom& g, const void* d_iq, int iq_format, uint32_t batch, double* d_sp_incoherent, cudaStream_t st) {
  dim3 grid((LCS_N_FOLD + SP_TILE - 1) / SP_TILE, batch);
  return SearchFormats::dispatch(iq_format, [&](auto FMT) {
    sp_fold_kernel<FMT><<<grid, SP_THREADS, 0, st>>>(d_iq, d_sp_incoherent, g.n_cap, g.n_comb_sp);
  }) == LCS_OK;
}

// ------------------------------------------------------------------------------------------
// Epilogue: xc_delay_spread (searcher.cpp:312-347) + xc_peak_freq (:353-383).  One thread per (t, idx); planar reads
// are coalesced along idx.  HBM-bound: every value of xc_incoherent_single is read once.
// ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) epilogue_kernel(const float* __restrict__ single_planar, double* __restrict__ pow_out,
                                                       int32_t* __restrict__ frq_out, float* __restrict__ incoherent_planar,
                                                       const uint32_t n_f_stride, const int* __restrict__ plan_nf,
                                                       const uint32_t* __restrict__ buf_plan, const uint32_t arm) {
  const uint32_t idx = blockIdx.x * 256 + threadIdx.x, t = blockIdx.y, b = blockIdx.z;
  if (idx >= LCS_N_FOLD) return;
  const uint32_t n_f = (uint32_t)__ldg(plan_nf + (buf_plan ? __ldg(buf_plan + b) : 0u));
  const float* s = single_planar + ((size_t)b * 3 + t) * n_f_stride * LCS_N_FOLD;
  float* inc_out = incoherent_planar ? incoherent_planar + ((size_t)b * 3 + t) * n_f_stride * LCS_N_FOLD : nullptr;
  const float denom = (float)(2 * arm + 1);
  float best = 0.f;
  int best_f = 0;
#pragma unroll 4
  for (uint32_t f = 0; f < n_f; f++) {
    const float* sf = s + (size_t)f * LCS_N_FOLD;
    float v = __ldg(sf + idx);
    for (uint32_t a = 1; a <= arm; a++) {
      const uint32_t lo = idx >= a ? idx - a : idx + LCS_N_FOLD - a;
      const uint32_t hi = idx + a < LCS_N_FOLD ? idx + a : idx + a - LCS_N_FOLD;
      v = __fadd_rn(v, __fadd_rn(__ldg(sf + lo), __ldg(sf + hi)));  // searcher.cpp:336: += single[idx-t]+single[idx+t]
    }
    v = __fdiv_rn(v, denom);  // :343
    if (inc_out) inc_out[(size_t)f * LCS_N_FOLD + idx] = v;
    if (f == 0 || v > best) { best = v; best_f = (int)f; }  // :371-377 strict >, first max wins
  }
  pow_out[((size_t)b * 3 + t) * LCS_N_FOLD + idx] = (double)best;
  frq_out[((size_t)b * 3 + t) * LCS_N_FOLD + idx] = best_f;
}

// x / (2*arm+1) for the box filter: q = RN(x*r); q += RN(x - n*q) * r equals the IEEE quotient for every non-negative float
// when n is 1, 3, 5, 7 or 9 (exhaustive check, tools/divchk.c) - three instructions instead of the division sequence.
template <int N>
__device__ __forceinline__ float div_small_odd(float x) {
  if (N == 1) return x;
  constexpr float r = 1.0f / (float)N;
  const float q = __fmul_rn(x, r);
  return __fmaf_rn(__fmaf_rn(-(float)N, q, x), r, q);
}

// Vectorised variant for ds_comb_arm <= 4: one thread = 4 consecutive fold positions, three 128-bit loads per hypothesis
// (previous / own / next quad; the neighbours' quads are L1 hits; 9600 % 4 == 0 so the circular wrap is a quad index
// wrap).  HBM-bound.
template <int ARM>
__global__ void __launch_bounds__(128) epilogue4_kernel(const float* __restrict__ single_planar, double* __restrict__ pow_out,
                                                        int32_t* __restrict__ frq_out, float* __restrict__ incoherent_planar,
                                                        const uint32_t n_f_stride, const int* __restrict__ plan_nf,
                                                        const uint32_t* __restrict__ buf_plan) {
  constexpr uint32_t NQ = LCS_N_FOLD / 4;
  const uint32_t q = blockIdx.x * 128 + threadIdx.x, t = blockIdx.y, b = blockIdx.z;
  if (q >= NQ) return;
  const uint32_t n_f = (uint32_t)__ldg(plan_nf + (buf_plan ? __ldg(buf_plan + b) : 0u));
  const uint32_t qp = q == 0 ? NQ - 1 : q - 1, qn = q == NQ - 1 ? 0 : q + 1;
  const float4* s = reinterpret_cast<const float4*>(single_planar + ((size_t)b * 3 + t) * n_f_stride * LCS_N_FOLD);
  float4* inc_out = incoherent_planar ? reinterpret_cast<float4*>(incoherent_planar + ((size_t)b * 3 + t) * n_f_stride * LCS_N_FOLD) : nullptr;
  float best[4] = {0.f, 0.f, 0.f, 0.f};
  int best_f[4] = {0, 0, 0, 0};
#pragma unroll 4
  for (uint32_t f = 0; f < n_f; f++) {
    const float4* sf = s + (size_t)f * NQ;
    const float4 c = __ldg(sf + q);
    float w[12];
    if (ARM > 0) {
      const float4 pv = __ldg(sf + qp), nx = __ldg(sf + qn);
      w[0] = pv.x; w[1] = pv.y; w[2] = pv.z; w[3] = pv.w;
      w[8] = nx.x; w[9] = nx.y; w[10] = nx.z; w[11] = nx.w;
    }
    w[4] = c.x; w[5] = c.y; w[6] = c.z; w[7] = c.w;
    float v[4];
#pragma unroll
    for (int o = 0; o < 4; o++) {
      float x = w[4 + o];
#pragma unroll
      for (int a = 1; a <= ARM; a++) x = __fadd_rn(x, __fadd_rn(w[4 + o - a], w[4 + o + a]));  // searcher.cpp:336
      x = div_small_odd<2 * ARM + 1>(x);                                                    // :343
      v[o] = x;
      if (f == 0 || x > best[o]) { best[o] = x; best_f[o] = (int)f; }                      // :371-377
    }
    if (inc_out) inc_out[(size_t)f * NQ + q] = make_float4(v[0], v[1], v[2], v[3]);
  }
  const size_t o0 = ((size_t)b * 3 + t) * LCS_N_FOLD + 4 * q;
  reinterpret_cast<double2*>(pow_out + o0)[0] = make_double2((double)best[0], (double)best[1]);
  reinterpret_cast<double2*>(pow_out + o0)[1] = make_double2((double)best[2], (double)best[3]);
  *reinterpret_cast<int4*>(frq_out + o0) = make_int4(best_f[0], best_f[1], best_f[2], best_f[3]);
}

int launch_epilogue(const XcorrGeom& g, const PlanView& pv, uint32_t batch, const float* d_single_planar, double* d_pow,
                    int32_t* d_frq, float* d_incoherent_planar, cudaStream_t st) {
  if (g.ds_comb_arm <= 4) {
    dim3 grid((LCS_N_FOLD / 4 + 127) / 128, 3, batch);
#define EPI(A) epilogue4_kernel<A><<<grid, 128, 0, st>>>(d_single_planar, d_pow, d_frq, d_incoherent_planar, g.n_f_stride, pv.d_nf, pv.d_buf_plan)
    switch (g.ds_comb_arm) {
      case 0: EPI(0); break;
      case 1: EPI(1); break;
      case 2: EPI(2); break;
      case 3: EPI(3); break;
      default: EPI(4); break;
    }
#undef EPI
    return 1;
  }
  dim3 grid((LCS_N_FOLD + 255) / 256, 3, batch);
  epilogue_kernel<<<grid, 256, 0, st>>>(d_single_planar, d_pow, d_frq, d_incoherent_planar, g.n_f_stride, pv.d_nf, pv.d_buf_plan, g.ds_comb_arm);
  return 1;
}

// ------------------------------------------------------------------------------------------
// Layout / format helpers for the drop-in host call.
// ------------------------------------------------------------------------------------------
// planar [3][n_f][9600] -> ref vf3d [3][9600][n_f]; 32x32 shared-memory transpose.
__global__ void planar_to_ref_kernel(const float* __restrict__ planar, float* __restrict__ ref, const uint32_t n_f) {
  __shared__ float tilebuf[32][33];
  const uint32_t t = blockIdx.z, i0 = blockIdx.x * 32, f0 = blockIdx.y * 32;
  for (int r = threadIdx.y; r < 32; r += blockDim.y) {
    const uint32_t f = f0 + r, i = i0 + threadIdx.x;
    tilebuf[r][threadIdx.x] = (f < n_f && i < LCS_N_FOLD) ? planar[((size_t)t * n_f + f) * LCS_N_FOLD + i] : 0.f;
  }
  __syncthreads();
  for (int r = threadIdx.y; r < 32; r += blockDim.y) {
    const uint32_t i = i0 + r, f = f0 + threadIdx.x;
    if (f < n_f && i < LCS_N_FOLD) ref[((size_t)t * LCS_N_FOLD + i) * n_f + f] = tilebuf[threadIdx.x][r];
  }
}
int launch_planar_to_ref(const XcorrGeom& g, const float* d_planar, float* d_ref, cudaStream_t st) {
  dim3 grid((LCS_N_FOLD + 31) / 32, (g.n_f_stride + 31) / 32, 3), block(32, 8);
  planar_to_ref_kernel<<<grid, block, 0, st>>>(d_planar, d_ref, g.n_f_stride);
  return 1;
}

// Debug-only materialisation of xc (searcher.h:37, vcf3d [t][k][f]) with the same FP32 arithmetic
// order as the fused kernel; one thread per (k, f).
template <int FMT>
__global__ void __launch_bounds__(128) xc_debug_kernel(const void* __restrict__ iq, const float4* __restrict__ w01g,
                                                       const float2* __restrict__ w2g, float2* __restrict__ xc,
                                                       const uint32_t n_cap, const uint32_t n_f) {
  const uint32_t n_lag = n_cap - 136;
  const uint32_t k = blockIdx.x * 128 + threadIdx.x, f = blockIdx.y;
  if (k >= n_lag) return;
  float2 a0 = make_float2(0.f, 0.f), a1 = a0, a2 = a0;
  for (int m = 0; m < LCS_N_TAPS; m++) {
    const float2 x = load_iq<FMT>(iq, (size_t)k + m);
    const float4 wa = __ldg(w01g + (size_t)f * XC_NTAP_PAD + m);
    const float2 wb = __ldg(w2g + (size_t)f * XC_NTAP_PAD + m);
    cmac(a0, wa.x, wa.y, x);
    cmac(a1, wa.z, wa.w, x);
    cmac(a2, wb.x, wb.y, x);
  }
  xc[((size_t)0 * n_lag + k) * n_f + f] = a0;
  xc[((size_t)1 * n_lag + k) * n_f + f] = a1;
  xc[((size_t)2 * n_lag + k) * n_f + f] = a2;
}
int launch_xc_debug(const XcorrGeom& g, const void* d_iq, int iq_format, const float4* d_w01, const float2* d_w2,
                    float2* d_xc, cudaStream_t st) {
  dim3 grid((g.n_cap - 136 + 127) / 128, g.n_f_stride);
  return SearchFormats::dispatch(iq_format, [&](auto FMT) {
    xc_debug_kernel<FMT><<<grid, 128, 0, st>>>(d_iq, d_w01, d_w2, d_xc, g.n_cap, g.n_f_stride);
  }) == LCS_OK;
}

// Debug-only `sp` (searcher.h:38): [n_comb_sp*9600] doubles.
template <int FMT>
__global__ void sp_debug_kernel(const void* __restrict__ iq, double* __restrict__ sp, const uint32_t n_sp) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= n_sp) return;
  double s = 0;
  for (int j = 0; j < 274; j++) s += pwr<FMT>(iq, (size_t)t + j);
  sp[t] = s / 274;
}
int launch_sp_debug(const XcorrGeom& g, const void* d_iq, int iq_format, double* d_sp, cudaStream_t st) {
  const uint32_t n_sp = g.n_comb_sp * LCS_N_FOLD;
  return SearchFormats::dispatch(iq_format, [&](auto FMT) {
    sp_debug_kernel<FMT><<<(n_sp + 255) / 256, 256, 0, st>>>(d_iq, d_sp, n_sp);
  }) == LCS_OK;
}

}  // namespace lcs
