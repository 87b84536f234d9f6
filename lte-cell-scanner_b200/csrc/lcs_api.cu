// lcs_api.cu - context, xcorr plan and the xcorr_pss entry points of the C ABI (include/lcs_b200.h).
#include <cmath>
#include <cstdio>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <mutex>

#include "iq_format.cuh"
#include "lcs_ctx.hpp"

namespace lcs {

static std::string g_last_error;
static std::mutex g_err_mu;

lcs_status fail(lcs_ctx* ctx, lcs_status st, const std::string& msg) {
  {
    std::lock_guard<std::mutex> lk(g_err_mu);
    g_last_error = msg;
  }
  if (ctx) ctx->last_error = msg;
  return st;
}

// ---------------------------------------------------------------------------------------------
// Plan construction: one search configuration wrapped around a plan set (planset.cu).
// ---------------------------------------------------------------------------------------------
static lcs_status build_plan(lcs_ctx* ctx, uint32_t n_cap, const double* f_search_set, uint32_t n_f, uint8_t arm,
                             double fc_req, double fc_prog, double fs_prog, uint32_t max_batch, int kernel,
                             lcs_xcorr_plan** out) {
  if (!ctx || !f_search_set || !out) return fail(ctx, LCS_ERR_ARG, "xcorr plan: null argument");
  if (n_f == 0 || n_f > 4096) return fail(ctx, LCS_ERR_ARG, "xcorr plan: n_f out of range");
  if (max_batch == 0) max_batch = 1;
  std::unique_ptr<lcs_xcorr_plan> p(new lcs_xcorr_plan());
  p->ctx = ctx;
  p->max_batch = max_batch;
  p->kernel = kernel;
  std::vector<PlanCfg> cfg(1);
  cfg[0].fc_req = fc_req;
  cfg[0].fc_prog = fc_prog;
  cfg[0].fs_prog = fs_prog;
  cfg[0].f.assign(f_search_set, f_search_set + n_f);
  cudaStream_t st = ctx->streams[0];
  lcs_status rc = planset_build(ctx, p->ps, n_cap, arm, cfg, true, st);
  if (rc == LCS_OK) rc = planset_finish(ctx, p->ps, st);
  if (rc != LCS_OK) return rc;
  *out = p.release();
  return LCS_OK;
}

static lcs_status run_device(lcs_xcorr_plan* p, const void* d_iq, int iq_format, uint32_t batch, float* d_single,
                             double* d_pow, int32_t* d_frq, double* d_spi, float* d_inc, cudaStream_t st) {
  lcs_ctx* ctx = p->ctx;
  if (batch == 0 || batch > p->max_batch) return fail(ctx, LCS_ERR_ARG, "xcorr_pss_device: batch exceeds plan max_batch");
  if (!p->timing)
    return planset_run(p->ps, p->kernel, d_iq, iq_format, batch, nullptr, d_single, d_pow, d_frq, d_spi, d_inc, st);
  const KernelClock::Pair* ev = nullptr;
  LCS_CUDA(ctx, p->clock.open(&ev));
  lcs_status rc = planset_run(p->ps, p->kernel, d_iq, iq_format, batch, nullptr, d_single, d_pow, d_frq, d_spi, d_inc, st, ev);
  if (rc != LCS_OK) return rc;
  LCS_CUDA(ctx, p->clock.commit(1));
  return LCS_OK;
}

// ---------------------------------------------------------------------------------------------
// 8-bit exactness probe of the c128 drop-in call: a capture read from an rtl-sdr dump holds exactly (u8-127)/128
// (src/capbuf.cpp:172-175).  If every component of the buffer is such a value the raw bytes are reconstructed and the
// tensor-core correlator (exact for 8-bit IQ) serves the call; anything else stays on the FP32 correlator.
// ---------------------------------------------------------------------------------------------
__global__ void c128_to_cu8_kernel(const double* __restrict__ cap, const uint32_t n, unsigned char* __restrict__ cu8, int* __restrict__ inexact) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double v = cap[i] * 128.0 + 127.0;         // exact for the values in question
  const double r = rint(v);
  if (!(v == r) || r < 0.0 || r > 255.0) { atomicOr(inexact, 1); return; }
  cu8[i] = (unsigned char)(int)r;
}

}  // namespace lcs

using namespace lcs;

extern "C" {

const char* lcs_version(void) { return "lcs_b200 0.3 (sm_90a)"; }

lcs_status lcs_ctx_create(int device, lcs_ctx** out) {
  if (!out) return fail(nullptr, LCS_ERR_ARG, "ctx_create: null out pointer");
  *out = nullptr;
  int n = 0;
  cudaError_t e = cudaGetDeviceCount(&n);
  if (e != cudaSuccess || n == 0)
    return fail(nullptr, LCS_ERR_CUDA, std::string("no CUDA device (there is no CPU fallback): ") + cudaGetErrorString(e));
  if (device < 0 || device >= n) return fail(nullptr, LCS_ERR_ARG, "ctx_create: device index out of range");
  cudaDeviceProp prop;
  e = cudaGetDeviceProperties(&prop, device);
  if (e != cudaSuccess) return fail(nullptr, LCS_ERR_CUDA, cudaGetErrorString(e));
  if (prop.major != 9 || prop.minor != 0)
    return fail(nullptr, LCS_ERR_CUDA, "device is not compute capability 9.0 (kernels are built for sm_90a only)");
  e = cudaSetDevice(device);
  if (e != cudaSuccess) return fail(nullptr, LCS_ERR_CUDA, cudaGetErrorString(e));
  std::unique_ptr<lcs_ctx> c(new lcs_ctx());
  c->device = device;
  c->n_sm = prop.multiProcessorCount;
  for (int i = 0; i < lcs_ctx::N_STREAMS; i++)
    if (cudaStreamCreateWithFlags(&c->streams[i], cudaStreamNonBlocking) != cudaSuccess) {
      for (int k = 0; k < i; k++) cudaStreamDestroy(c->streams[k]);
      return fail(nullptr, LCS_ERR_CUDA, "stream creation failed");
    }
  // constants of the plan builder: the three time-domain PSS (lte_lib.cpp:177-188) and the fixed-point scale of the
  // tensor-core templates.  A frequency shift only rotates a tap, so |component| <= |pss_td tap| / 137 for every offset:
  // one power of two S serves all plans.
  cd td[3][137];
  double maxmag = 0;
  for (int t = 0; t < 3; t++) {
    pss_td(t, td[t]);
    for (int k = 0; k < 137; k++) maxmag = std::max(maxmag, std::abs(td[t][k]) / 137.0);
  }
  const double limit = 127.0 * 65536 + 127 * 256 + 127;
  int ex = (int)std::floor(std::log2(limit / maxmag));
  while (std::ldexp(maxmag, ex) > limit) ex--;
  c->tc_scale = std::ldexp(1.0, ex);
  if (c->d_pss_td.alloc(3 * 137 * 2) != cudaSuccess ||
      cudaMemcpy(c->d_pss_td.p, &td[0][0], sizeof(td), cudaMemcpyHostToDevice) != cudaSuccess) {
    for (int i = 0; i < lcs_ctx::N_STREAMS; i++) cudaStreamDestroy(c->streams[i]);
    return fail(nullptr, LCS_ERR_CUDA, "pss_td upload failed");
  }
  xcorr_fp32_init();
  lcs_status rc = tc_init(c.get());
  if (rc != LCS_OK) {
    for (int i = 0; i < lcs_ctx::N_STREAMS; i++) cudaStreamDestroy(c->streams[i]);
    return rc;
  }
  *out = c.release();
  return LCS_OK;
}

void lcs_ctx_destroy(lcs_ctx* ctx) {
  if (!ctx) return;
  cudaSetDevice(ctx->device);
  cudaDeviceSynchronize();
  for (auto* p : ctx->cached_plans) lcs_xcorr_plan_destroy(p);
  ctx->cached_plans.clear();
  for (int i = 0; i < lcs_ctx::N_STREAMS; i++)
    if (ctx->streams[i]) cudaStreamDestroy(ctx->streams[i]);
  delete ctx;
}

const char* lcs_last_error(const lcs_ctx* ctx) {
  if (ctx) return ctx->last_error.c_str();
  std::lock_guard<std::mutex> lk(g_err_mu);
  static thread_local std::string copy;
  copy = g_last_error;
  return copy.c_str();
}

uint64_t lcs_launch_count(const lcs_ctx* ctx) { return ctx ? ctx->launches : 0; }

void lcs_cell_init(lcs_cell* c) {  // Cell::Cell(), reference src/common.cpp:36-56
  if (!c) return;
  c->fc_requested = c->fc_programmed = c->pss_pow = NAN;
  c->ind = -1;
  c->freq = NAN;
  c->n_id_2 = -1;
  c->n_id_1 = -1;
  c->cp_type = 0;
  c->frame_start = c->freq_fine = c->freq_superfine = NAN;
  c->n_ports = c->n_rb_dl = -1;
  c->phich_duration = c->phich_resource = 0;
  c->sfn = -1;
}

lcs_status lcs_xcorr_plan_create(lcs_ctx* ctx, uint32_t n_cap, const double* f_search_set, uint32_t n_f,
                                 uint8_t ds_comb_arm, double fc_requested, double fc_programmed, double fs_programmed,
                                 uint32_t max_batch, int kernel, lcs_xcorr_plan** plan) {
  return build_plan(ctx, n_cap, f_search_set, n_f, ds_comb_arm, fc_requested, fc_programmed, fs_programmed, max_batch,
                    kernel, plan);
}

void lcs_xcorr_plan_destroy(lcs_xcorr_plan* plan) {
  if (!plan) return;
  cudaSetDevice(plan->ctx->device);
  cudaDeviceSynchronize();
  delete plan;
}

lcs_status lcs_xcorr_plan_timing_enable(lcs_xcorr_plan* p, int enable) {
  if (!p) return fail(nullptr, LCS_ERR_ARG, "timing_enable: null plan");
  p->timing = enable != 0;
  return LCS_OK;
}
lcs_status lcs_xcorr_plan_timing_read(lcs_xcorr_plan* p, double* kernel_ms, uint64_t* launches) {
  if (!p || !kernel_ms || !launches) return fail(nullptr, LCS_ERR_ARG, "timing_read: null argument");
  LCS_CUDA(p->ctx, p->clock.read(kernel_ms, launches));
  return LCS_OK;
}

uint16_t lcs_xcorr_plan_n_comb_xc(const lcs_xcorr_plan* p) { return p ? (uint16_t)p->ps.geom.n_comb_xc : 0; }
uint16_t lcs_xcorr_plan_n_comb_sp(const lcs_xcorr_plan* p) { return p ? (uint16_t)p->ps.geom.n_comb_sp : 0; }
int lcs_xcorr_plan_kernel(const lcs_xcorr_plan* p, int iq_format) { return p ? planset_resolve_kernel(p->ps, p->kernel, iq_format) : 0; }

lcs_status lcs_xcorr_pss_device(lcs_xcorr_plan* plan, const void* d_iq, int iq_format, uint32_t batch,
                                float* d_single_planar, double* d_pow, int32_t* d_frq, double* d_sp_incoherent,
                                float* d_incoherent_planar, void* stream) {
  if (!plan) return fail(nullptr, LCS_ERR_ARG, "xcorr_pss_device: null plan");
  return run_device(plan, d_iq, iq_format, batch, d_single_planar, d_pow, d_frq, d_sp_incoherent, d_incoherent_planar,
                    (cudaStream_t)stream);
}

// Host-buffer batched call: chunks of the batch rotate over the context's streams (rotate_chunks), so that the copies
// of the neighbouring chunks overlap the kernels of a chunk; the host waits only once, for every stream at the end.
lcs_status lcs_xcorr_pss_batch_host(lcs_xcorr_plan* p, const void* h_iq, int iq_format, uint32_t batch,
                                    float* h_single, double* h_pow, int32_t* h_frq, double* h_spi) {
  if (!p) return fail(nullptr, LCS_ERR_ARG, "xcorr_pss_batch_host: null plan");
  lcs_ctx* ctx = p->ctx;
  if (!h_iq || !h_pow || !h_frq || !h_spi) return fail(ctx, LCS_ERR_ARG, "xcorr_pss_batch_host: null pointer");
  if (batch == 0) return LCS_OK;
  const XcorrGeom& g = p->ps.geom;
  if (!SearchFormats::has(iq_format)) return fail(ctx, LCS_ERR_ARG, "xcorr_pss_batch_host: bad iq_format");
  const size_t samp_bytes = sample_bytes(iq_format);
  LCS_CUDA(ctx, cudaSetDevice(ctx->device));
  const uint32_t chunk = std::min<uint32_t>(std::min<uint32_t>(p->max_batch, BATCH_CHUNK), batch);
  const size_t n_single = (size_t)3 * g.n_f_stride * LCS_N_FOLD;
  for (auto& hb : p->hb) LCS_CUDA(ctx, hb.ensure(g, chunk, samp_bytes, true, false));
  auto issue = [&](uint32_t b0, int s) -> lcs_status {
    const uint32_t nb = std::min(chunk, batch - b0);
    cudaStream_t st = ctx->streams[s];
    auto& hb = p->hb[s];
    LCS_CUDA(ctx, cudaMemcpyAsync(hb.iq.p, (const char*)h_iq + (size_t)b0 * g.n_cap * samp_bytes,
                                  (size_t)nb * g.n_cap * samp_bytes, cudaMemcpyHostToDevice, st));
    lcs_status rc = run_device(p, hb.iq.p, iq_format, nb, hb.single.p, hb.pow.p, hb.frq.p, hb.spi.p, nullptr, st);
    if (rc != LCS_OK) return rc;
    if (h_single)
      LCS_CUDA(ctx, cudaMemcpyAsync(h_single + (size_t)b0 * n_single, hb.single.p, (size_t)nb * n_single * 4, cudaMemcpyDeviceToHost, st));
    LCS_CUDA(ctx, cudaMemcpyAsync(h_pow + (size_t)b0 * 3 * LCS_N_FOLD, hb.pow.p, (size_t)nb * 3 * LCS_N_FOLD * 8, cudaMemcpyDeviceToHost, st));
    LCS_CUDA(ctx, cudaMemcpyAsync(h_frq + (size_t)b0 * 3 * LCS_N_FOLD, hb.frq.p, (size_t)nb * 3 * LCS_N_FOLD * 4, cudaMemcpyDeviceToHost, st));
    LCS_CUDA(ctx, cudaMemcpyAsync(h_spi + (size_t)b0 * LCS_N_FOLD, hb.spi.p, (size_t)nb * LCS_N_FOLD * 8, cudaMemcpyDeviceToHost, st));
    return LCS_OK;
  };
  lcs_status rc = rotate_chunks(batch, chunk, issue, [](uint32_t, int) { return LCS_OK; });
  if (rc != LCS_OK) return rc;
  for (cudaStream_t st : ctx->streams) LCS_CUDA(ctx, cudaStreamSynchronize(st));
  return LCS_OK;
}

// Drop-in for searcher.h:22-41.
lcs_status lcs_xcorr_pss(lcs_ctx* ctx, const double* capbuf, uint32_t n_cap, const double* f_search_set, uint32_t n_f,
                         uint8_t ds_comb_arm, double fc_requested, double fc_programmed, double fs_programmed,
                         double* pow, int32_t* frq, float* single, float* incoherent, double* sp_incoherent, float* xc,
                         double* sp, uint16_t* n_comb_xc, uint16_t* n_comb_sp) {
  if (!ctx) return fail(nullptr, LCS_ERR_ARG, "xcorr_pss: null context");
  if (!capbuf || !f_search_set || !pow || !frq || !single || !sp_incoherent)
    return fail(ctx, LCS_ERR_ARG, "xcorr_pss: null pointer");
  lcs_xcorr_plan* p = nullptr;
  lcs_status rc = get_cached_plan(ctx, n_cap, f_search_set, n_f, ds_comb_arm, fc_requested, fc_programmed, fs_programmed, &p);
  if (rc != LCS_OK) return rc;
  const XcorrGeom& g = p->ps.geom;
  cudaStream_t st = ctx->streams[0];
  const size_t n_single = (size_t)3 * n_f * LCS_N_FOLD;
  auto& hb = p->hb[0];
  rc = upload_c128(ctx, capbuf, n_cap, st);
  if (rc != LCS_OK) return rc;
  LCS_CUDA(ctx, hb.ensure(g, 1, 0, false, false));
  LCS_CUDA(ctx, ctx->d_ref.ensure(n_single));
  LCS_CUDA(ctx, ctx->d_inc.ensure(n_single));
  // 8-bit exact input (an rtl-sdr capture, capbuf.cpp:172-175) goes to the tensor-core correlator
  const void* d_in = ctx->d_capbuf.p;
  int fmt = LCS_IQ_C128;
  if (planset_resolve_kernel(p->ps, p->kernel, LCS_IQ_CU8) == LCS_KERNEL_TC) {
    int inexact = 0;
    LCS_CUDA(ctx, ctx->d_cu8.ensure((size_t)n_cap * 2 + 16));
    LCS_CUDA(ctx, ctx->d_flag8.ensure(1));
    LCS_CUDA(ctx, cudaMemsetAsync(ctx->d_flag8.p, 0, 4, st));
    c128_to_cu8_kernel<<<(2 * n_cap + 255) / 256, 256, 0, st>>>(ctx->d_capbuf.p, 2 * n_cap, ctx->d_cu8.p, ctx->d_flag8.p);
    ctx->launches++;
    LCS_CUDA(ctx, cudaMemcpyAsync(&inexact, ctx->d_flag8.p, 4, cudaMemcpyDeviceToHost, st));
    LCS_CUDA(ctx, cudaStreamSynchronize(st));
    if (!inexact) { d_in = ctx->d_cu8.p; fmt = LCS_IQ_CU8; }
  }
  rc = run_device(p, d_in, fmt, 1, hb.single.p, hb.pow.p, hb.frq.p, hb.spi.p, incoherent ? ctx->d_inc.p : nullptr, st);
  if (rc != LCS_OK) return rc;
  // reference layouts: vf3d [t][idx][f]; mat(3,9600) column-major
  ctx->launches += launch_planar_to_ref(g, hb.single.p, ctx->d_ref.p, st);
  LCS_CUDA(ctx, cudaMemcpyAsync(single, ctx->d_ref.p, n_single * 4, cudaMemcpyDeviceToHost, st));
  if (incoherent) {
    LCS_CUDA(ctx, cudaStreamSynchronize(st));
    ctx->launches += launch_planar_to_ref(g, ctx->d_inc.p, ctx->d_ref.p, st);
    LCS_CUDA(ctx, cudaMemcpyAsync(incoherent, ctx->d_ref.p, n_single * 4, cudaMemcpyDeviceToHost, st));
  }
  std::vector<double> hpow(3 * LCS_N_FOLD);
  std::vector<int32_t> hfrq(3 * LCS_N_FOLD);
  LCS_CUDA(ctx, cudaMemcpyAsync(hpow.data(), hb.pow.p, hpow.size() * 8, cudaMemcpyDeviceToHost, st));
  LCS_CUDA(ctx, cudaMemcpyAsync(hfrq.data(), hb.frq.p, hfrq.size() * 4, cudaMemcpyDeviceToHost, st));
  LCS_CUDA(ctx, cudaMemcpyAsync(sp_incoherent, hb.spi.p, LCS_N_FOLD * 8, cudaMemcpyDeviceToHost, st));
  if (xc) {
    const size_t n_xc = (size_t)3 * (n_cap - 136) * n_f;
    DevBuf<float2> d_xc;
    LCS_CUDA(ctx, d_xc.alloc(n_xc));
    ctx->launches += launch_xc_debug(g, ctx->d_capbuf.p, LCS_IQ_C128, p->ps.d_w01.p, p->ps.d_w2.p, d_xc.p, st);
    LCS_CUDA(ctx, cudaMemcpyAsync(xc, d_xc.p, n_xc * 8, cudaMemcpyDeviceToHost, st));
    LCS_CUDA(ctx, cudaStreamSynchronize(st));
  }
  if (sp) {
    DevBuf<double> d_sp;
    LCS_CUDA(ctx, d_sp.alloc((size_t)g.n_comb_sp * LCS_N_FOLD));
    ctx->launches += launch_sp_debug(g, ctx->d_capbuf.p, LCS_IQ_C128, d_sp.p, st);
    LCS_CUDA(ctx, cudaMemcpyAsync(sp, d_sp.p, (size_t)g.n_comb_sp * LCS_N_FOLD * 8, cudaMemcpyDeviceToHost, st));
    LCS_CUDA(ctx, cudaStreamSynchronize(st));
  }
  LCS_CUDA(ctx, cudaStreamSynchronize(st));
  for (int t = 0; t < 3; t++)
    for (int k = 0; k < LCS_N_FOLD; k++) {
      pow[(size_t)k * 3 + t] = hpow[(size_t)t * LCS_N_FOLD + k];
      frq[(size_t)k * 3 + t] = hfrq[(size_t)t * LCS_N_FOLD + k];
    }
  if (n_comb_xc) *n_comb_xc = (uint16_t)g.n_comb_xc;
  if (n_comb_sp) *n_comb_sp = (uint16_t)g.n_comb_sp;
  return LCS_OK;
}

}  // extern "C"

namespace lcs {
lcs_status upload_c128(lcs_ctx* ctx, const double* capbuf, uint32_t n_cap, cudaStream_t st) {
  LCS_CUDA(ctx, cudaSetDevice(ctx->device));
  LCS_CUDA(ctx, ctx->d_capbuf.ensure((size_t)n_cap * 2));
  LCS_CUDA(ctx, cudaMemcpyAsync(ctx->d_capbuf.p, capbuf, (size_t)n_cap * 16, cudaMemcpyHostToDevice, st));
  return LCS_OK;
}

lcs_status get_cached_plan(lcs_ctx* ctx, uint32_t n_cap, const double* f_search_set, uint32_t n_f, uint8_t arm,
                           double fc_req, double fc_prog, double fs_prog, lcs_xcorr_plan** out) {
  for (auto* q : ctx->cached_plans) {
    const PlanCfg& c = q->ps.cfg[0];
    if (q->ps.geom.n_cap == n_cap && c.f.size() == n_f && q->ps.geom.ds_comb_arm == arm && c.fc_req == fc_req &&
        c.fc_prog == fc_prog && c.fs_prog == fs_prog && std::memcmp(c.f.data(), f_search_set, n_f * sizeof(double)) == 0) {
      *out = q;
      return LCS_OK;
    }
  }
  lcs_xcorr_plan* p = nullptr;
  lcs_status rc = build_plan(ctx, n_cap, f_search_set, n_f, arm, fc_req, fc_prog, fs_prog, 1, LCS_KERNEL_AUTO, &p);
  if (rc != LCS_OK) return rc;
  if (ctx->cached_plans.size() >= 8) {
    lcs_xcorr_plan_destroy(ctx->cached_plans.front());
    ctx->cached_plans.erase(ctx->cached_plans.begin());
  }
  ctx->cached_plans.push_back(p);
  *out = p;
  return LCS_OK;
}
}  // namespace lcs
