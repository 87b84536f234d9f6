// planset.cu - search plans: everything xcorr_pss needs besides the capture buffer, built for MANY search configurations
// at once (one per centre frequency of a sweep, one per tracked channel) and kept resident in HBM.
//
//   host   integer geometry: k_factor fold offsets round_i(m*.005*k_factor*fs) (searcher.cpp:298), their range check,
//          per-pass staging starts / column offsets of the tensor-core correlator, tile geometry of the FP32 correlator
//   device plan_build_kernel: the pre-rotated templates conj(fshift(pss_td[t], f_off, fs*k_factor))/137
//          (searcher.cpp:145-151 with dsp.h:40-53) in double precision, rounded once to FP32 for the CUDA-core
//          correlator and to 24-bit fixed point, split in three balanced int8 digit planes in wgmma core-matrix order,
//          for the tensor-core correlator, plus the per-template additive constants of the v-128 sample representation.
#include <cmath>
#include <cstring>

#include "iq_format.cuh"
#include "lcs_ctx.hpp"

namespace lcs {

constexpr int CFG_HDR = 4;   // doubles before the f list of a plan's builder record

// ---------------------------------------------------------------------------------------------------------------------
// One block per (hypothesis, plan); thread = tap.
// ---------------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(160) plan_build_kernel(const double* __restrict__ cfg, const double2* __restrict__ pss_td,
                                                         const uint32_t n_f_stride, float4* __restrict__ w01,
                                                         float2* __restrict__ w2, unsigned char* __restrict__ b_img,
                                                         float* __restrict__ corr, int* __restrict__ flag, const double S,
                                                         const tc::Layout lay, const uint32_t n_pass,
                                                         const uint32_t hyp_per_pass_used) {
  const uint32_t f = blockIdx.x, p = blockIdx.y, tap = threadIdx.x;
  const double* c = cfg + (size_t)p * (CFG_HDR + n_f_stride);
  const uint32_t n_f = (uint32_t)c[3];
  __shared__ long long s_all[3], s_even[3], s_abs2[3];
  if (tap < 3) { s_all[tap] = 0; s_even[tap] = 0; s_abs2[tap] = 0; }
  __syncthreads();
  const bool live = f < n_f && tap < LCS_N_TAPS;
  double wre[3] = {0, 0, 0}, wim[3] = {0, 0, 0};
  if (live) {
    const double fc_req = c[0], fc_prog = c[1], fs_prog = c[2], f_off = c[CFG_HDR + f];
    const double k_factor = __ddiv_rn(__dsub_rn(fc_req, f_off), fc_prog);                               // searcher.cpp:147
    const double k = __ddiv_rn(__dmul_rn(3.14159265358979323846, f_off), __ddiv_rn(__dmul_rn(fs_prog, k_factor), 2.0));   // dsp.h:42
    double sn, cs;
    sincos(__dmul_rn(k, (double)tap), &sn, &cs);
#pragma unroll
    for (int t = 0; t < 3; t++) {
      const double2 td = pss_td[t * LCS_N_TAPS + tap];
      // conj(td * rot) / 137, products and sums rounded separately like std::complex on the host
      const double re = __dsub_rn(__dmul_rn(td.x, cs), __dmul_rn(td.y, sn));
      const double im = __dadd_rn(__dmul_rn(td.x, sn), __dmul_rn(td.y, cs));
      wre[t] = __ddiv_rn(re, 137.0);
      wim[t] = __ddiv_rn(-im, 137.0);
    }
  }
  if (w01 && tap < XC_NTAP_PAD) {
    const size_t o = ((size_t)p * n_f_stride + f) * XC_NTAP_PAD + tap;
    w01[o] = make_float4((float)wre[0], (float)wim[0], (float)wre[1], (float)wim[1]);
    w2[o] = make_float2((float)wre[2], (float)wim[2]);
  }
  if (b_img && live) {
    const uint32_t pass = f / hyp_per_pass_used, fl = f - pass * hyp_per_pass_used;
    unsigned char* img = b_img + ((size_t)p * n_pass + pass) * lay.b_bytes();
    const int C = lay.c();
#pragma unroll
    for (int t = 0; t < 3; t++) {
      const int col = (int)fl * 3 + t, g = col / C, r0 = col % C;
      unsigned char* job = img + (size_t)g * lay.b_job_bytes();
      const long long wr = llrint(__dmul_rn(wre[t], S)), wi = llrint(__dmul_rn(wim[t], S));
      const long long v[2] = {wr, -wi};     // multiplies the I byte / the Q byte (re) resp. the ~I byte (im)
      long long a2sum = 0;
#pragma unroll
      for (int e = 0; e < 2; e++) {
        // balanced base-256 digits: v = 65536 d0 + 256 d1 + d2, d1, d2 in [-128, 127]
        long long d2 = ((v[e] % 256) + 256) % 256; if (d2 > 127) d2 -= 256;
        const long long r1 = (v[e] - d2) / 256;
        long long d1 = ((r1 % 256) + 256) % 256; if (d1 > 127) d1 -= 256;
        const long long d0 = (r1 - d1) / 256;
        const int k = 2 * (int)tap + e;
        job[tc::b_offset(0 * C + r0, k)] = (unsigned char)(signed char)d0;
        job[tc::b_offset(1 * C + r0, k)] = (unsigned char)(signed char)d1;
        job[tc::b_offset(2 * C + r0, k)] = (unsigned char)(signed char)d2;
        a2sum += d2 < 0 ? -d2 : d2;
        if (d0 < -128 || d0 > 127) atomicOr(flag, 1);
      }
      atomicAdd((unsigned long long*)&s_all[t], (unsigned long long)(wr - wi));     // x = x'+1 :  + sum_j a[j]
      atomicAdd((unsigned long long*)&s_even[t], (unsigned long long)wr);           // (Q', ~I') stream:  + sum_m a[2m]
      atomicAdd((unsigned long long*)&s_abs2[t], (unsigned long long)a2sum);
    }
  }
  __syncthreads();
  if (corr && tap < 3 && f < n_f) {
    const uint32_t pass = f / hyp_per_pass_used, fl = f - pass * hyp_per_pass_used;
    const int col = (int)fl * 3 + (int)tap, npad = lay.npad();
    float* cc = corr + ((size_t)p * n_pass + pass) * 2 * npad;
    // the epilogue adds the low digit plane as the float (MAGIC_VAL + a2): fold -MAGIC_VAL into the constants
    cc[col] = (float)((double)s_all[tap] - tc::MAGIC_VAL);
    cc[npad + col] = (float)((double)s_even[tap] - tc::MAGIC_VAL);
    if (s_abs2[tap] * 128 >= (1ll << 22)) atomicOr(flag, 2);     // |a2| could leave the exact range of the magic-number conversion
  }
}

static tc::Layout pick_layout(uint32_t n_f, uint32_t& n_pass) {
  // one consumer warpgroup per job: two jobs let one warpgroup's epilogue overlap the other one's MMAs
  n_pass = 1;
  if (n_f <= 5) return tc::Layout{16, 1};          // tracker shape (one offset): N = 48, one consumer warpgroup
  if (n_f <= 16) return tc::Layout{24, 2};         // N = 80
  if (n_f <= 21) return tc::Layout{32, 2};         // N = 96
  if (n_f <= 32) return tc::Layout{48, 2};         // N = 144
  if (n_f <= 42) { n_pass = 2; return tc::Layout{32, 2}; }
  n_pass = (n_f + 31) / 32;
  return tc::Layout{48, 2};
}

lcs_status planset_build(lcs_ctx* ctx, PlanSet& ps, uint32_t n_cap, uint8_t arm, const std::vector<PlanCfg>& cfgs,
                         bool want_fp32, cudaStream_t st) {
  if (cfgs.empty()) return fail(ctx, LCS_ERR_ARG, "xcorr plan: no search configuration");
  if (n_cap < 136 + 100 + LCS_N_FOLD || n_cap < 273 + LCS_N_FOLD)
    return fail(ctx, LCS_ERR_ARG, "xcorr plan: capture buffer shorter than one 5 ms half frame + margins");
  if (arm > 64) return fail(ctx, LCS_ERR_ARG, "xcorr plan: ds_comb_arm out of range");
  uint32_t n_f_stride = 0;
  for (const PlanCfg& c : cfgs) {
    if (c.f.empty() || c.f.size() > 4096) return fail(ctx, LCS_ERR_ARG, "xcorr plan: n_f out of range");
    n_f_stride = std::max<uint32_t>(n_f_stride, (uint32_t)c.f.size());
  }
  LCS_CUDA(ctx, cudaSetDevice(ctx->device));
  ps.ctx = ctx;
  const uint32_t P = (uint32_t)cfgs.size();
  ps.n_plans = P;
  ps.cfg = cfgs;
  ps.h_nf.resize(P);
  XcorrGeom& g = ps.geom;
  g.n_cap = n_cap;
  g.ds_comb_arm = arm;
  g.n_f_stride = n_f_stride;
  const uint32_t n_lag = n_cap - 136;
  g.n_comb_xc = (n_lag - 100) / LCS_N_FOLD;        // searcher.cpp:276
  g.n_comb_sp = (n_cap - 136 - 137) / LCS_N_FOLD;  // searcher.cpp:194
  g.fw = n_f_stride == 1 ? 1 : XC_FW;              // searcher_thread.cpp:97-98 searches a single offset
  g.n_fchunk = (n_f_stride + g.fw - 1) / g.fw;
  const uint32_t M = g.n_comb_xc;

  // ---- tensor-core pass structure ----
  uint32_t n_pass = 1;
  ps.lay = pick_layout(n_f_stride, n_pass);
  ps.n_pass = n_pass;
  const uint32_t hpp = (n_f_stride + n_pass - 1) / n_pass;      // hypotheses per pass actually used (balanced)
  const int npad = ps.lay.npad();
  ps.tc_ready = true;
  ps.tc_why.clear();
  if (n_pass > (uint32_t)tc::MAX_PASS) { ps.tc_ready = false; ps.tc_why = "more than 256 frequency hypotheses"; }
  if (M > (uint32_t)tc::M_MAX) { ps.tc_ready = false; ps.tc_why = "capture buffer longer than 24 half frames"; }

  // ---- host staging: [cfg doubles][nf ints][soff ints][smin ints][geo][dsh] ----
  const size_t n_cfg = (size_t)P * (CFG_HDR + n_f_stride);
  const size_t n_soff = (size_t)P * M * n_f_stride, n_smin = (size_t)P * M * g.n_fchunk;
  const size_t n_geo = (size_t)P * n_pass, n_dsh = (size_t)P * n_pass * tc::M_MAX * npad;
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off = (off + bytes + 255) & ~(size_t)255; return o; };
  const size_t o_cfg = take(n_cfg * 8), o_nf = take(P * 4), o_soff = take(n_soff * 4), o_smin = take(n_smin * 4),
               o_geo = take(n_geo * sizeof(tc::PassGeo)), o_dsh = take(n_dsh * 2);
  if (!ps.staged) LCS_CUDA(ctx, cudaEventCreateWithFlags(&ps.staged, cudaEventDisableTiming));
  else LCS_CUDA(ctx, cudaEventSynchronize(ps.staged));         // the previous upload out of the staging buffer is done
  LCS_CUDA(ctx, ps.h_stage.ensure(off));
  unsigned char* hs = ps.h_stage.p;
  std::memset(hs, 0, off);
  double* h_cfg = reinterpret_cast<double*>(hs + o_cfg);
  int* h_nf = reinterpret_cast<int*>(hs + o_nf);
  int* h_soff = reinterpret_cast<int*>(hs + o_soff);
  int* h_smin = reinterpret_cast<int*>(hs + o_smin);
  tc::PassGeo* h_geo = reinterpret_cast<tc::PassGeo*>(hs + o_geo);
  int16_t* h_dsh = reinterpret_cast<int16_t*>(hs + o_dsh);

  uint32_t max_spread = 0;
  for (uint32_t p = 0; p < P; p++) {
    const PlanCfg& c = cfgs[p];
    const uint32_t n_f = (uint32_t)c.f.size();
    ps.h_nf[p] = h_nf[p] = (int)n_f;
    double* hc = h_cfg + (size_t)p * (CFG_HDR + n_f_stride);
    hc[0] = c.fc_req; hc[1] = c.fc_prog; hc[2] = c.fs_prog; hc[3] = (double)n_f;
    int* so = h_soff + (size_t)p * M * n_f_stride;
    for (uint32_t f = 0; f < n_f; f++) {
      hc[CFG_HDR + f] = c.f[f];
      const double k_factor = (c.fc_req - c.f[f]) / c.fc_prog;      // :147
      for (uint32_t m = 0; m < M; m++) {
        const double s = std::rint(m * .005 * k_factor * c.fs_prog);  // :298 (IT++ round_i == rint)
        if (!(s >= 0) || s + (LCS_N_FOLD - 1) >= (double)n_lag)
          return fail(ctx, LCS_ERR_RANGE, "xcorr plan: fold offset runs past the correlation buffer (reference would read out of bounds)");
        so[(size_t)m * n_f_stride + f] = (int)s;
      }
    }
    for (uint32_t f = n_f; f < n_f_stride; f++)                       // unused tail: repeat the last hypothesis
      for (uint32_t m = 0; m < M; m++) so[(size_t)m * n_f_stride + f] = so[(size_t)m * n_f_stride + n_f - 1];
    // FP32 correlator: minimum / spread per block of fw hypotheses
    for (uint32_t m = 0; m < M; m++)
      for (uint32_t ch = 0; ch < g.n_fchunk; ch++) {
        int lo = INT32_MAX, hi = INT32_MIN;
        for (uint32_t f = ch * g.fw; f < std::min(n_f_stride, (ch + 1) * g.fw); f++) {
          lo = std::min(lo, so[(size_t)m * n_f_stride + f]);
          hi = std::max(hi, so[(size_t)m * n_f_stride + f]);
        }
        h_smin[((size_t)p * M + m) * g.n_fchunk + ch] = lo;
        max_spread = std::max(max_spread, (uint32_t)(hi - lo));
      }
    // tensor-core correlator: per pass staging start smin[m] and per-column offsets dsh = offset - smin[m].  The kernel
    // adds half frame m of a fold position in tile (position - run start + dsh) / 256 of its run, half frames of one tile
    // in order.  smin[m] advances by the smallest step of the pass' offsets from half frame m - 1 to m, so dsh is
    // non-decreasing in m for every column: the half frames of a position are then added in ascending m, whatever tile
    // phase its run starts at (so at every batch size and SM count).  smin[m] <= every offset of half frame m, so dsh >= 0.
    for (uint32_t ps_i = 0; ps_i < n_pass && ps.tc_ready; ps_i++) {
      tc::PassGeo& pg = h_geo[(size_t)p * n_pass + ps_i];
      const uint32_t f0 = ps_i * hpp, f1 = std::min(n_f, f0 + hpp);
      pg.f0 = (int)f0;
      pg.n_f = f1 > f0 ? (int)(f1 - f0) : 0;
      int16_t* dsh = h_dsh + ((size_t)p * n_pass + ps_i) * tc::M_MAX * npad;
      int start = 0;
      for (uint32_t m = 0; m < M; m++) {
        int lo = INT32_MAX, hi = INT32_MIN, step = INT32_MAX;
        for (uint32_t f = f0; f < f1; f++) {
          const int s = so[(size_t)m * n_f_stride + f];
          lo = std::min(lo, s);
          hi = std::max(hi, s);
          if (m > 0) step = std::min(step, s - so[(size_t)(m - 1) * n_f_stride + f]);
        }
        if (f1 <= f0) start = hi = so[(size_t)m * n_f_stride + n_f - 1];     // an empty pass: no column to order
        else start = m == 0 ? lo : start + step;
        pg.smin[m] = start;
        if (hi - start > tc::HALO) {
          ps.tc_ready = false;
          ps.tc_why = "frequency grid too sparse for the tensor-core tiling (fold offsets more than 32 samples above the staging start)";
          break;
        }
        for (uint32_t f = f0; f < f1; f++)
          for (int t = 0; t < 3; t++) dsh[(size_t)m * npad + (f - f0) * 3 + t] = (int16_t)(so[(size_t)m * n_f_stride + f] - start);
      }
    }
  }
  g.max_spread = max_spread;
  g.tile_len = XC_TI * (XC_FW / g.fw) + XC_NTAP_PAD + max_spread + 8;
  const size_t smem = (size_t)g.fw * XC_NTAP_PAD * 24 + (size_t)g.tile_len * 8 + (want_fp32 ? (size_t)XC_THREADS * 42 * 4 : 0);
  if (want_fp32 && smem > 100 * 1024)
    return fail(ctx, LCS_ERR_RANGE, "xcorr plan: frequency grid too sparse for one shared-memory tile (spread too large)");

  // ---- uploads (one staged copy per table) ----
  LCS_CUDA(ctx, ps.d_cfg.ensure(n_cfg));
  LCS_CUDA(ctx, ps.d_nf.ensure(P));
  LCS_CUDA(ctx, ps.d_soff.ensure(n_soff));
  LCS_CUDA(ctx, ps.d_smin.ensure(n_smin));
  LCS_CUDA(ctx, cudaMemcpyAsync(ps.d_cfg.p, h_cfg, n_cfg * 8, cudaMemcpyHostToDevice, st));
  LCS_CUDA(ctx, cudaMemcpyAsync(ps.d_nf.p, h_nf, P * 4, cudaMemcpyHostToDevice, st));
  LCS_CUDA(ctx, cudaMemcpyAsync(ps.d_soff.p, h_soff, n_soff * 4, cudaMemcpyHostToDevice, st));
  LCS_CUDA(ctx, cudaMemcpyAsync(ps.d_smin.p, h_smin, n_smin * 4, cudaMemcpyHostToDevice, st));
  if (ps.tc_ready) {
    LCS_CUDA(ctx, ps.d_geo.ensure(n_geo));
    LCS_CUDA(ctx, ps.d_dsh.ensure(n_dsh));
    LCS_CUDA(ctx, ps.d_b.ensure((size_t)P * n_pass * ps.lay.b_bytes()));
    LCS_CUDA(ctx, ps.d_corr.ensure((size_t)P * n_pass * 2 * npad));
    LCS_CUDA(ctx, cudaMemcpyAsync(ps.d_geo.p, h_geo, n_geo * sizeof(tc::PassGeo), cudaMemcpyHostToDevice, st));
    LCS_CUDA(ctx, cudaMemcpyAsync(ps.d_dsh.p, h_dsh, n_dsh * 2, cudaMemcpyHostToDevice, st));
    LCS_CUDA(ctx, cudaMemsetAsync(ps.d_b.p, 0, (size_t)P * n_pass * ps.lay.b_bytes(), st));
    LCS_CUDA(ctx, cudaMemsetAsync(ps.d_corr.p, 0, (size_t)P * n_pass * 2 * npad * 4, st));
  }
  LCS_CUDA(ctx, cudaEventRecord(ps.staged, st));
  if (!ps.d_flag.p) LCS_CUDA(ctx, ps.d_flag.alloc(1));
  LCS_CUDA(ctx, cudaMemsetAsync(ps.d_flag.p, 0, 4, st));         // diagnostics of THIS build
  if (want_fp32) {
    LCS_CUDA(ctx, ps.d_w01.ensure((size_t)P * n_f_stride * XC_NTAP_PAD));
    LCS_CUDA(ctx, ps.d_w2.ensure((size_t)P * n_f_stride * XC_NTAP_PAD));
  }
  ps.inv_scale = (float)(1.0 / (ctx->tc_scale * 128.0));
  dim3 grid(n_f_stride, P);
  plan_build_kernel<<<grid, 160, 0, st>>>(ps.d_cfg.p, reinterpret_cast<const double2*>(ctx->d_pss_td.p), n_f_stride,
                                          want_fp32 ? ps.d_w01.p : nullptr, want_fp32 ? ps.d_w2.p : nullptr,
                                          ps.tc_ready ? ps.d_b.p : nullptr, ps.tc_ready ? ps.d_corr.p : nullptr, ps.d_flag.p,
                                          ctx->tc_scale, ps.lay, n_pass, hpp);
  ctx->launches++;
  LCS_CUDA(ctx, cudaGetLastError());
  ps.has_fp32 = want_fp32;
  return LCS_OK;
}

lcs_status planset_finish(lcs_ctx* ctx, PlanSet& ps, cudaStream_t st) {
  int flag = 0;
  LCS_CUDA(ctx, cudaMemcpyAsync(&flag, ps.d_flag.p, 4, cudaMemcpyDeviceToHost, st));
  LCS_CUDA(ctx, cudaStreamSynchronize(st));
  if (flag) { ps.tc_ready = false; ps.tc_why = "template digits outside the exact range of the integer formulation"; }
  return LCS_OK;
}

int planset_resolve_kernel(const PlanSet& ps, int kernel, int iq_format) {
  if (kernel == LCS_KERNEL_FP32) return LCS_KERNEL_FP32;
  if (kernel == LCS_KERNEL_TC) return LCS_KERNEL_TC;
  // AUTO: the tensor-core kernel is exact only for 8-bit IQ, so it serves that format (the single-offset tracker shape
  // included: one N = 48 job per part); other formats go to the FP32 correlator.
  return (iq_format == LCS_IQ_CU8 && ps.tc_ready) ? LCS_KERNEL_TC : LCS_KERNEL_FP32;
}

lcs_status planset_run(PlanSet& ps, int kernel, const void* d_iq, int iq_format, uint32_t batch, const uint32_t* d_buf_plan,
                       float* d_single, double* d_pow, int32_t* d_frq, double* d_spi, float* d_inc, cudaStream_t st,
                       const std::pair<cudaEvent_t, cudaEvent_t>* ev) {
  lcs_ctx* ctx = ps.ctx;
  if (!d_iq || !d_single || !d_pow || !d_frq || !d_spi) return fail(ctx, LCS_ERR_ARG, "xcorr_pss_device: null pointer");
  if (batch == 0) return fail(ctx, LCS_ERR_ARG, "xcorr_pss_device: empty batch");
  if (!SearchFormats::has(iq_format)) return fail(ctx, LCS_ERR_ARG, "xcorr_pss_device: bad iq_format");
  // every kernel loads a whole sample at a time (uchar2 / float2 / double2); the epilogue reads `single` as float4 and
  // writes incoherent / pow / frq as float4 / double2 / int4; sp_fold_kernel stores single doubles
  if ((uintptr_t)d_iq % sample_bytes(iq_format) != 0)
    return fail(ctx, LCS_ERR_ARG, "xcorr_pss_device: IQ pointer not aligned to its sample size");
  if ((((uintptr_t)d_single | (uintptr_t)d_pow | (uintptr_t)d_frq | (uintptr_t)d_inc) & 15) != 0)
    return fail(ctx, LCS_ERR_ARG, "xcorr_pss_device: single, pow, frq and incoherent need 16-byte aligned pointers");
  if (((uintptr_t)d_spi & 7) != 0) return fail(ctx, LCS_ERR_ARG, "xcorr_pss_device: sp_incoherent needs an 8-byte aligned pointer");
  int kern = planset_resolve_kernel(ps, kernel, iq_format);
  // the tensor-core kernel stages raw bytes with 16-byte bulk copies: an unaligned base pointer goes to the FP32 kernel
  if (kern == LCS_KERNEL_TC && kernel == LCS_KERNEL_AUTO && ((uintptr_t)d_iq & 15) != 0) kern = LCS_KERNEL_FP32;
  if (kern == LCS_KERNEL_TC) {
    if (iq_format != LCS_IQ_CU8) return fail(ctx, LCS_ERR_ARG, "tensor-core correlator needs LCS_IQ_CU8 input");
    if (!ps.tc_ready) return fail(ctx, LCS_ERR_STATE, "tensor-core correlator not available for this plan: " + ps.tc_why);
    if (((uintptr_t)d_iq & 15) != 0) return fail(ctx, LCS_ERR_ARG, "tensor-core correlator needs a 16-byte aligned IQ pointer");
  } else if (!ps.has_fp32) {
    return fail(ctx, LCS_ERR_STATE, "this plan set was built without the FP32 correlator's templates");
  }
  const PlanView pv{ps.d_nf.p, d_buf_plan};
  if (ev) LCS_CUDA(ctx, cudaEventRecord(ev->first, st));
  if (kern == LCS_KERNEL_TC)
    ctx->launches += launch_xcorr_fold_tc(ps, d_iq, batch, d_buf_plan, d_single, st);
  else
    ctx->launches += launch_xcorr_fold_fp32(ps.geom, pv, d_iq, iq_format, batch, ps.d_w01.p, ps.d_w2.p, ps.d_soff.p, ps.d_smin.p,
                                            d_single, st);
  if (ev) LCS_CUDA(ctx, cudaEventRecord(ev->second, st));
  ctx->launches += launch_sp_fold(ps.geom, d_iq, iq_format, batch, d_spi, st);
  ctx->launches += launch_epilogue(ps.geom, pv, batch, d_single, d_pow, d_frq, d_inc, st);
  LCS_CUDA(ctx, cudaGetLastError());
  return LCS_OK;
}

}  // namespace lcs
