// chain_gpu.cu - companion kernels of the correlator (FP64): batched PSS/SSS symbol extraction
// (fshift + 2-sample rotate + 128-point FFT), SSS channel-estimate combining, SSS maximum-likelihood
// detection over the 168 x {h1h2,h2h1} x {normal,extended} hypotheses, and OFDM time/frequency-grid
// extraction (whole-buffer FOC fused into 854 FFT-128).  Reference: src/searcher.cpp:516-935.
#include <cmath>
#include <cstring>

#include "chain_gpu.hpp"
#include "fft128.cuh"

namespace lcs {

static const double kPi = 3.14159265358979323846;
static const double kFsLte = 30720000.0;

// ---------------------------------------------------------------------------------------------
// extract_psss (searcher.cpp:516-530), batched: one block per 128-sample segment.
//   out[seg][62] = bins [-31..-1, 1..31] of dft( rotate_left_2( x[start..start+127] * e^{j k n} ) )
// with k = pi*foc_freq/(fs/2), n = 0..127 local (the reference shifts each segment from phase 0).
// ---------------------------------------------------------------------------------------------
template <int FMT>
__global__ void __launch_bounds__(64) psss_kernel(const void* __restrict__ cap, const int* __restrict__ start,
                                                  const double* __restrict__ kseg, double2* __restrict__ out) {
  __shared__ double2 buf[128];
  __shared__ double2 tw[64];
  const int tid = threadIdx.x, seg = blockIdx.x;
  make_twiddles(tw, tid);
  const size_t s0 = (size_t)start[seg];
  const double k = kseg[seg];
  for (int n = tid; n < 128; n += 64) {
    double sn, cs;
    sincos(k * (double)n, &sn, &cs);
    const double2 x = cmul(load_c<FMT>(cap, s0 + n), make_double2(cs, sn));
    const int dst = (n + 126) & 127;  // rotate left by 2: b[i] = a[i+2]
    buf[bitrev7(dst)] = x;
  }
  __syncthreads();
  fft128_inplace(buf, tw, tid);
  const double sc = 1.0 / sqrt(128.0);
  if (tid < 62) {
    const int bin = tid < 31 ? 97 + tid : 1 + (tid - 31);
    out[(size_t)seg * 62 + tid] = make_double2(buf[bin].x * sc, buf[bin].y * sc);
  }
}

// ---------------------------------------------------------------------------------------------
// sss_detect_getce_sss (searcher.cpp:577-631) after the FFTs.  psss: [n_pss][3][62] =
// {PSS symbol, SSS symbol assuming extended CP, SSS symbol assuming normal CP}.  One block per peak, thread t
// owns subcarrier t.  est: [h1_np 62][h2_np 62] doubles then c128 [h1_nrm][h2_nrm][h1_ext][h2_ext].
// par[peak] = {first segment of the peak in psss, n_pss, n_id_2}.
// ---------------------------------------------------------------------------------------------
constexpr int MAX_PSS = 64;
constexpr int EST_LEN = 124 + 4 * 124;     // doubles per peak
__global__ void __launch_bounds__(64) sss_getce_kernel(const double2* __restrict__ psss_all, const int3* __restrict__ par,
                                                       const double2* __restrict__ pss_fd_all, double* __restrict__ est_all,
                                                       const int max_pss) {
  extern __shared__ double2 sm[];
  const int3 pp = par[blockIdx.x];
  const int n_pss = pp.y;
  const double2* psss = psss_all + (size_t)pp.x * 62;
  const double2* pss_fd = pss_fd_all + pp.z * 62;
  double* est = est_all + (size_t)blockIdx.x * EST_LEN;
  double2* h_raw = sm;                 // [n_pss][62]
  double2* h_sm = sm + max_pss * 62;   // [n_pss][62]
  __shared__ double np[MAX_PSS];
  const int t = threadIdx.x;
  if (t < 62) {
    const double2 pc = make_double2(pss_fd[t].x, -pss_fd[t].y);
    for (int k = 0; k < n_pss; k++) h_raw[k * 62 + t] = cmul(psss[((size_t)k * 3 + 0) * 62 + t], pc);
  }
  __syncthreads();
  if (t < 62) {
    const int lt = max(0, t - 6), rt = min(61, t + 6);
    for (int k = 0; k < n_pss; k++) {
      double2 s = make_double2(0, 0);
      for (int i = lt; i <= rt; i++) { s.x += h_raw[k * 62 + i].x; s.y += h_raw[k * 62 + i].y; }
      const double n = (double)(rt - lt + 1);
      h_sm[k * 62 + t] = make_double2(s.x / n, s.y / n);
    }
  }
  __syncthreads();
  if (t < n_pss) {  // noise power of PSS k (sigpower, dsp.h:23-29)
    double r = 0;
    for (int i = 0; i < 62; i++) {
      const double dx = h_sm[t * 62 + i].x - h_raw[t * 62 + i].x, dy = h_sm[t * 62 + i].y - h_raw[t * 62 + i].y;
      r += dx * dx + dy * dy;
    }
    np[t] = r / 62;
  }
  __syncthreads();
  if (t < 62) {
    double2* estc = reinterpret_cast<double2*>(est + 124);
    for (int half = 0; half < 2; half++) {
      double den = 0;
      double2 nrm = make_double2(0, 0), ext = make_double2(0, 0);
      for (int k = half; k < n_pss; k += 2) {
        const double inv = 1.0 / np[k];
        const double2 h = h_sm[k * 62 + t];
        den += (h.x * h.x + h.y * h.y) * inv;
        const double2 hc = make_double2(h.x * inv, -h.y * inv);
        const double2 a = cmul(hc, psss[((size_t)k * 3 + 2) * 62 + t]);
        const double2 b = cmul(hc, psss[((size_t)k * 3 + 1) * 62 + t]);
        nrm.x += a.x; nrm.y += a.y;
        ext.x += b.x; ext.y += b.y;
      }
      const double npe = 1.0 / (1.0 + den);
      est[half * 62 + t] = npe;
      estc[(0 + half) * 62 + t] = make_double2(npe * nrm.x, npe * nrm.y);
      estc[(2 + half) * 62 + t] = make_double2(npe * ext.x, npe * ext.y);
    }
  }
}

// ---------------------------------------------------------------------------------------------
// sss_detect_ml (searcher.cpp:636-693): block = n_id_1, warp = hypothesis
// {nrm h1h2, nrm h2h1, ext h1h2, ext h2h1}.  sss_tab: int8 [168][3][2][62].
// ll: [4][168] = {nrm col0, nrm col1, ext col0, ext col1}.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__global__ void __launch_bounds__(128) sss_ml_kernel(const double* __restrict__ est_all, const signed char* __restrict__ sss_tab,
                                                     const int3* __restrict__ par, double* __restrict__ ll_all) {
  const int n1 = blockIdx.x, hyp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const double* est = est_all + (size_t)blockIdx.y * EST_LEN;
  double* ll = ll_all + (size_t)blockIdx.y * 4 * 168;
  const int n_id_2 = par[blockIdx.y].z;
  const bool swap = hyp & 1, is_ext = hyp >> 1;
  const double2* estc = reinterpret_cast<const double2*>(est + 124) + (is_ext ? 2 * 62 : 0);  // [h1][h2]
  const signed char* s0 = sss_tab + (((size_t)n1 * 3 + n_id_2) * 2 + 0) * 62;
  const signed char* s10 = s0 + 62;
  double ax = 0, ay = 0;
  for (int i = lane; i < 124; i += 32) {
    const int half = i >= 62, j = i - 62 * half;
    const double tr = (double)((half ^ swap) ? s10[j] : s0[j]);
    const double2 e = estc[i];
    ax += e.x * tr;   // conj(est)*try
    ay += -e.y * tr;
  }
  ax = warp_sum(ax);
  ay = warp_sum(ay);
  const double ang = atan2(ay, ax);
  double sn, cs;
  sincos(-ang, &sn, &cs);
  double sre = 0, sim = 0;
  for (int i = lane; i < 124; i += 32) {
    const int half = i >= 62, j = i - 62 * half;
    const double tr = (double)((half ^ swap) ? s10[j] : s0[j]);
    const double2 e = estc[i];
    const double dx = tr * cs - e.x, dy = tr * sn - e.y;
    const double npv = est[i];  // [h1_np][h2_np]
    sre += dx * dx / npv;
    sim += dy * dy / npv;
  }
  sre = warp_sum(sre);
  sim = warp_sum(sim);
  if (lane == 0) ll[hyp * 168 + n1] = -sre - sim;
}

// ---------------------------------------------------------------------------------------------
// extract_tfg (searcher.cpp:892-931): FOC of the whole buffer fused into the per-symbol FFT.
//   tfg[t][72] = bins [-36..-1,1..36] of dft( x[pos_t + n] * e^{j k (pos_t+n)} ) * e^{-j 2 pi late_t cn/128}
// ---------------------------------------------------------------------------------------------
// Grid (854, cells): pos / late / tfg are [cell][854], kcell[cell], n_ofdm[cell] (732 for the extended CP).
constexpr int TFG_MAX = 854;
template <int FMT>
__global__ void __launch_bounds__(64) tfg_kernel(const void* __restrict__ cap, const int* __restrict__ pos_all,
                                                 const double* __restrict__ late_all, const double* __restrict__ kcell,
                                                 const int* __restrict__ n_ofdm, double2* __restrict__ tfg_all) {
  __shared__ double2 buf[128];
  __shared__ double2 tw[64];
  const int tid = threadIdx.x, sym = blockIdx.x, cell = blockIdx.y;
  if (sym >= n_ofdm[cell]) return;
  const int* pos = pos_all + (size_t)cell * TFG_MAX;
  const double* late = late_all + (size_t)cell * TFG_MAX;
  double2* tfg = tfg_all + (size_t)cell * TFG_MAX * 72;
  const double k = kcell[cell];
  make_twiddles(tw, tid);
  const size_t p0 = (size_t)pos[sym];
  for (int n = tid; n < 128; n += 64) {
    double sn, cs;
    sincos(k * (double)(p0 + n), &sn, &cs);
    buf[bitrev7(n)] = cmul(load_c<FMT>(cap, p0 + n), make_double2(cs, sn));
  }
  __syncthreads();
  fft128_inplace(buf, tw, tid);
  const double sc = 1.0 / sqrt(128.0);
  const double lt = late[sym];
  for (int i = tid; i < 72; i += 64) {
    const int bin = i < 36 ? 92 + i : 1 + (i - 36);
    const int cn = i < 36 ? i - 36 : i - 35;
    double sn, cs;
    sincos((-2.0 * kPi * lt / 128.0) * (double)cn, &sn, &cs);
    const double2 v = make_double2(buf[bin].x * sc, buf[bin].y * sc);
    tfg[(size_t)sym * 72 + i] = cmul(v, make_double2(cs, sn));
  }
}

#define DISPATCH(fmt, CALL)                               \
  do {                                                    \
    if ((fmt) == LCS_IQ_CU8) { CALL(LCS_IQ_CU8); }        \
    else if ((fmt) == LCS_IQ_CF32) { CALL(LCS_IQ_CF32); } \
    else { CALL(LCS_IQ_C128); }                           \
  } while (0)

// =============================================================================================
// Host drivers (device-resident capture buffer)
// =============================================================================================
static const signed char* sss_table_dev(lcs_ctx* ctx, ChainScratch& cs) {
  if (cs.d_sss_tab.p) return cs.d_sss_tab.p;
  std::vector<signed char> tab((size_t)168 * 3 * 2 * 62);
  int v[62];
  for (int n1 = 0; n1 < 168; n1++)
    for (int n2 = 0; n2 < 3; n2++)
      for (int s = 0; s < 2; s++) {
        sss_fd(n1, n2, s * 10, v);
        for (int i = 0; i < 62; i++) tab[(((size_t)n1 * 3 + n2) * 2 + s) * 62 + i] = (signed char)v[i];
      }
  if (cs.d_sss_tab.alloc(tab.size()) != cudaSuccess) return nullptr;
  cudaMemcpy(cs.d_sss_tab.p, tab.data(), tab.size(), cudaMemcpyHostToDevice);
  cd fd[62];
  cs.d_pss_fd.alloc(3 * 62);
  for (int t = 0; t < 3; t++) {
    pss_fd(t, fd);
    cudaMemcpy(cs.d_pss_fd.p + t * 62, fd, 62 * 16, cudaMemcpyHostToDevice);
  }
  (void)ctx;
  return cs.d_sss_tab.p;
}

static std::vector<double> mrange(double first, double incr, double last) {  // itpp_ext.cpp:97-108
  std::vector<double> r;
  auto sg = [](double x) { return (x > 0) - (x < 0); };
  if (sg(last - first) * sg(incr) >= 0) {
    const int n = (int)std::floor((last - first) / incr) + 1;
    for (int t = 0; t < n; t++) r.push_back(first + t * incr);
  }
  return r;
}
static inline double wrapd(double x, double sm, double lg) {  // macros.h:49 with itpp_ext.h:40-42
  const double n = lg - sm, k = x - sm;
  return (n == 0 ? k : k - n * (int)std::floor(k / n)) + sm;
}

// page-locked staging of the small per-peak tables and results: the copies are truly asynchronous and a whole batch of
// peaks needs one synchronisation per stage
struct Stage {
  unsigned char* base;
  size_t off = 0;
  explicit Stage(unsigned char* b) : base(b) {}
  template <class T> T* take(size_t n) {
    off = (off + 15) & ~(size_t)15;
    T* p = reinterpret_cast<T*>(base + off);
    off += n * sizeof(T);
    return p;
  }
};

// all 128-sample segments of a stage through one psss launch; bins land in cs.d_psss
static lcs_status run_psss(lcs_ctx* ctx, ChainScratch& cs, const void* d_cap, int fmt, const std::vector<int>& starts,
                           const std::vector<double>& kseg, cudaStream_t st) {
  const size_t n = starts.size();
  LCS_CUDA(ctx, cs.h_up.ensure(n * 12 + 64));
  LCS_CUDA(ctx, cs.d_starts.ensure(n));
  LCS_CUDA(ctx, cs.d_kseg.ensure(n));
  LCS_CUDA(ctx, cs.d_psss.ensure(n * 62));
  Stage up(cs.h_up.p);
  int* hs = up.take<int>(n);
  double* hk = up.take<double>(n);
  std::memcpy(hs, starts.data(), n * 4);
  std::memcpy(hk, kseg.data(), n * 8);
  LCS_CUDA(ctx, cudaMemcpyAsync(cs.d_starts.p, hs, n * 4, cudaMemcpyHostToDevice, st));
  LCS_CUDA(ctx, cudaMemcpyAsync(cs.d_kseg.p, hk, n * 8, cudaMemcpyHostToDevice, st));
#define CALL(F) psss_kernel<F><<<(unsigned)n, 64, 0, st>>>(d_cap, cs.d_starts.p, cs.d_kseg.p, cs.d_psss.p)
  DISPATCH(fmt, CALL);
#undef CALL
  ctx->launches++;
  LCS_CUDA(ctx, cudaGetLastError());
  return LCS_OK;
}

// sss_detect (searcher.cpp:696-761) for all PSS peaks of a capture buffer: one FFT launch over every (peak, PSS position,
// {PSS, SSS-ext, SSS-nrm}) segment, one channel-estimate block and 168 x 4 likelihood warps per peak, ONE synchronisation.
// st[i] = LCS_ERR_RANGE marks a peak for which the reference would index outside the buffer (the caller skips it).
lcs_status dev_sss_detect_batch(lcs_ctx* ctx, ChainScratch& cs, const void* d_cap, int fmt, uint32_t n_cap,
                                const std::vector<lcs_cell>& cells, double thresh2_n_sigma, double fc_req, double fc_prog,
                                double fs_prog, std::vector<lcs_cell>& out, std::vector<lcs_status>& status, SssDebugHost* dbg) {
  cudaStream_t st = ctx->chain_stream ? ctx->chain_stream : ctx->streams[0];
  const size_t P = cells.size();
  out.assign(cells.begin(), cells.end());
  status.assign(P, LCS_OK);
  if (P == 0) return LCS_OK;
  if (!sss_table_dev(ctx, cs)) return fail(ctx, LCS_ERR_CUDA, "sss table upload failed");
  std::vector<int> starts;
  std::vector<double> kseg;
  std::vector<int3> par;
  std::vector<size_t> live;      // peaks that take part in the launches
  int max_pss = 1;
  for (size_t i = 0; i < P; i++) {
    const lcs_cell& cell = cells[i];
    if (cell.n_id_2 < 0 || cell.n_id_2 > 2) return fail(ctx, LCS_ERR_ARG, "sss_detect: n_id_2 out of range");
    // PSS positions with an SSS in front of them (searcher.cpp:549-563)
    double peak_loc = cell.ind;
    const double k_factor = (fc_req - cell.freq) / fc_prog;
    if (peak_loc + 9 < 162) peak_loc += 9600 * k_factor;
    const std::vector<double> locs = mrange(peak_loc, k_factor * 9600, (double)n_cap - 125 - 9);
    const int n_pss = (int)locs.size();
    if (n_pss < 1 || n_pss > MAX_PSS) { status[i] = LCS_ERR_RANGE; continue; }
    const size_t seg0 = starts.size();
    bool ok = true;
    for (int k = 0; k < n_pss && ok; k++) {
      const long pss_dft = (long)std::rint(locs[k]) + 9 - 2;
      const long sg[3] = {pss_dft, pss_dft - 128 - 32, pss_dft - 128 - 9};  // :579,:594,:596
      for (long v : sg) {
        if (v < 0 || v + 128 > (long)n_cap) { ok = false; break; }
        starts.push_back((int)v);
      }
    }
    if (!ok) { starts.resize(seg0); status[i] = LCS_ERR_RANGE; continue; }   // DFT window outside the capture buffer
    const double kk = kPi * -cell.freq / ((fs_prog * k_factor) / 2);         // dsp.h:42
    kseg.resize(starts.size(), kk);
    par.push_back(make_int3((int)seg0, n_pss, cell.n_id_2));
    live.push_back(i);
    max_pss = std::max(max_pss, n_pss);
  }
  if (live.empty()) return LCS_OK;
  const size_t L = live.size();
  lcs_status rc = run_psss(ctx, cs, d_cap, fmt, starts, kseg, st);
  if (rc != LCS_OK) return rc;
  LCS_CUDA(ctx, cs.d_par.ensure(L));
  LCS_CUDA(ctx, cs.d_est.ensure(L * EST_LEN));
  LCS_CUDA(ctx, cs.d_ll.ensure(L * 4 * 168));
  LCS_CUDA(ctx, cs.h_up2.ensure(L * sizeof(int3) + 64));
  LCS_CUDA(ctx, cs.h_down.ensure(L * (4 * 168 + EST_LEN) * 8 + 64));
  std::memcpy(cs.h_up2.p, par.data(), L * sizeof(int3));
  LCS_CUDA(ctx, cudaMemcpyAsync(cs.d_par.p, cs.h_up2.p, L * sizeof(int3), cudaMemcpyHostToDevice, st));
  if (!cs.getce_attr_set) {
    LCS_CUDA(ctx, cudaFuncSetAttribute(sss_getce_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * MAX_PSS * 62 * (int)sizeof(double2)));
    cs.getce_attr_set = true;
  }
  sss_getce_kernel<<<(unsigned)L, 64, (size_t)2 * max_pss * 62 * sizeof(double2), st>>>(cs.d_psss.p, cs.d_par.p, cs.d_pss_fd.p, cs.d_est.p, max_pss);
  sss_ml_kernel<<<dim3(168, (unsigned)L), 128, 0, st>>>(cs.d_est.p, cs.d_sss_tab.p, cs.d_par.p, cs.d_ll.p);
  ctx->launches += 2;
  LCS_CUDA(ctx, cudaGetLastError());
  double* h_ll = reinterpret_cast<double*>(cs.h_down.p);
  double* h_est = h_ll + L * 4 * 168;
  LCS_CUDA(ctx, cudaMemcpyAsync(h_ll, cs.d_ll.p, L * 4 * 168 * 8, cudaMemcpyDeviceToHost, st));
  if (dbg) LCS_CUDA(ctx, cudaMemcpyAsync(h_est, cs.d_est.p, L * EST_LEN * 8, cudaMemcpyDeviceToHost, st));
  LCS_CUDA(ctx, cudaStreamSynchronize(st));
  for (size_t li = 0; li < L; li++) {
    const lcs_cell& cell = cells[live[li]];
    const double* ll = h_ll + li * 4 * 168;
    const double k_factor = (fc_req - cell.freq) / fc_prog;
    // decisions (searcher.cpp:719-758)
    const double* nrm0 = &ll[0], *nrm1 = &ll[168], *ext0 = &ll[336], *ext1 = &ll[504];
    auto mx = [](const double* v) { return *std::max_element(v, v + 168); };
    const bool normal = std::max(mx(nrm0), mx(nrm1)) > std::max(mx(ext0), mx(ext1));
    const double* c0 = normal ? nrm0 : ext0, *c1 = normal ? nrm1 : ext1;
    const double fs_ratio = 16 / kFsLte * fs_prog;
    double frame_start = cell.ind + (128 + 9 - 960 - 2) * fs_ratio * k_factor;  // :735
    const double* col;
    if (mx(c0) > mx(c1)) col = c0;
    else { col = c1; frame_start += 9600 * k_factor * fs_ratio * k_factor; }  // :741
    frame_start = wrapd(frame_start, -0.5, (2 * 9600.0 - 0.5) * fs_ratio * k_factor);  // :743
    const int n_id_1 = (int)(std::max_element(col, col + 168) - col);
    const double lik_final = col[n_id_1];
    double sum = 0, sq = 0;  // IT++ mean / variance (N-1) over all 672 likelihoods
    for (int i = 0; i < 672; i++) { sum += ll[i]; sq += ll[i] * ll[i]; }
    const double mean = sum / 672, var = (sq - sum * sum / 672) / 671;
    lcs_cell& o = out[live[li]];
    if (lik_final >= mean + std::pow(var, 0.5) * thresh2_n_sigma) {
      o.n_id_1 = n_id_1;
      o.cp_type = normal ? 1 : 2;
      o.frame_start = frame_start;
    }
    if (dbg && li == 0) {
      dbg->est.assign(h_est, h_est + EST_LEN);
      dbg->ll.assign(ll, ll + 4 * 168);
    }
  }
  return LCS_OK;
}

lcs_status dev_sss_detect(lcs_ctx* ctx, ChainScratch& cs, const void* d_cap, int fmt, uint32_t n_cap, const lcs_cell& cell,
                          double thresh2_n_sigma, double fc_req, double fc_prog, double fs_prog, lcs_cell& out,
                          SssDebugHost* dbg) {
  std::vector<lcs_cell> o;
  std::vector<lcs_status> st;
  lcs_status rc = dev_sss_detect_batch(ctx, cs, d_cap, fmt, n_cap, std::vector<lcs_cell>(1, cell), thresh2_n_sigma, fc_req, fc_prog,
                                       fs_prog, o, st, dbg);
  if (rc != LCS_OK) return rc;
  if (st[0] != LCS_OK) return fail(ctx, st[0], "sss_detect: DFT window outside the capture buffer / unsupported number of PSS positions");
  out = o[0];
  return LCS_OK;
}

// pss_sss_foe (searcher.cpp:767-850) for several cells: one FFT launch, one synchronisation.
lcs_status dev_pss_sss_foe_batch(lcs_ctx* ctx, ChainScratch& cs, const void* d_cap, int fmt, uint32_t n_cap,
                                 const std::vector<lcs_cell>& cells, double fc_req, double fc_prog, double fs_prog,
                                 std::vector<lcs_cell>& out) {
  cudaStream_t st = ctx->chain_stream ? ctx->chain_stream : ctx->streams[0];
  const size_t P = cells.size();
  out.assign(cells.begin(), cells.end());
  if (P == 0) return LCS_OK;
  struct Geo { int dist, n_sss, sn; size_t seg0; };
  std::vector<Geo> geo(P);
  std::vector<int> starts;
  std::vector<double> kseg;
  for (size_t i = 0; i < P; i++) {
    const lcs_cell& cell = cells[i];
    if (cell.n_id_1 < 0 || cell.n_id_1 > 167 || cell.n_id_2 < 0 || cell.n_id_2 > 2)
      return fail(ctx, LCS_ERR_ARG, "pss_sss_foe: cell id not set");
    const double k_factor = (fc_req - cell.freq) / fc_prog;
    const double fs_ratio = 16 / kFsLte * fs_prog;
    int dist;
    double first;
    if (cell.cp_type == 1) {
      dist = (int)std::rint((128 + 9) * fs_ratio * k_factor);  // :780
      first = cell.frame_start + (960 - 128 - 9 - 128) * fs_ratio * k_factor;
    } else if (cell.cp_type == 2) {
      dist = (int)std::rint((128 + 32) * k_factor);  // :783
      first = cell.frame_start + (960 - 128 - 32 - 128) * fs_ratio * k_factor;
    } else {
      return fail(ctx, LCS_ERR_ARG, "pss_sss_foe: cp_type unknown (reference throws \"Error... check code...\")");
    }
    int sn;
    first = wrapd(first, -0.5, 9600 * 2 - 0.5);
    if (first - 9600 * k_factor > -0.5) { first -= 9600 * k_factor; sn = 10; } else sn = 0;
    const std::vector<double> locs = mrange(first, 9600 * fs_ratio * k_factor, (double)((long)n_cap - 127 - dist - 100));
    geo[i] = Geo{dist, (int)locs.size(), sn, starts.size()};
    for (size_t k = 0; k < locs.size(); k++) {
      const long sg = (long)std::rint(locs[k]);
      if (sg < 0 || sg + dist + 128 > (long)n_cap) return fail(ctx, LCS_ERR_RANGE, "pss_sss_foe: DFT window outside the capture buffer");
      starts.push_back((int)(sg + dist));  // PSS
      starts.push_back((int)sg);           // SSS
    }
    kseg.resize(starts.size(), kPi * -cell.freq / ((fs_prog * k_factor) / 2));
  }
  const cd* bins = nullptr;
  if (!starts.empty()) {
    lcs_status rc = run_psss(ctx, cs, d_cap, fmt, starts, kseg, st);
    if (rc != LCS_OK) return rc;
    LCS_CUDA(ctx, cs.h_down.ensure(starts.size() * 62 * 16 + 64));
    LCS_CUDA(ctx, cudaMemcpyAsync(cs.h_down.p, cs.d_psss.p, starts.size() * 62 * 16, cudaMemcpyDeviceToHost, st));
    LCS_CUDA(ctx, cudaStreamSynchronize(st));
    bins = reinterpret_cast<const cd*>(cs.h_down.p);
  }
  for (size_t i = 0; i < P; i++) {
    const lcs_cell& cell = cells[i];
    const Geo& g = geo[i];
    if (g.n_sss < 1) { out[i].freq_fine = cell.freq; continue; }   // reference: M stays 0, arg(0) = 0 (searcher.cpp:806,848)
    const double k_factor = (fc_req - cell.freq) / fc_prog;
    cd pfd[62];
    pss_fd(cell.n_id_2, pfd);
    int sn = (1 - (g.sn / 10)) * 10;  // :800
    const double pa = kPi * -cell.freq / (kFsLte / 16 / 2) * -(double)g.dist;  // :832
    const cd ph(std::cos(pa), std::sin(pa));
    cd M = 0;
    for (int k = 0; k < g.n_sss; k++) {
      sn = (1 - (sn / 10)) * 10;
      const cd* bp = bins + (g.seg0 + 2 * k) * 62;
      cd h_raw[62], h_sm[62];
      for (int t = 0; t < 62; t++) h_raw[t] = bp[t] * std::conj(pfd[t]);
      for (int t = 0; t < 62; t++) {
        const int lt = std::max(0, t - 6), rt = std::min(61, t + 6);
        cd sm = 0;
        for (int j = lt; j <= rt; j++) sm += h_raw[j];
        h_sm[t] = sm / (double)(rt - lt + 1);
      }
      double np = 0;
      for (int t = 0; t < 62; t++) np += std::norm(h_sm[t] - h_raw[t]);
      np /= 62;
      int sfd[62];
      sss_fd(cell.n_id_1, cell.n_id_2, sn, sfd);
      cd sm = 0;
      for (int t = 0; t < 62; t++) {
        const cd sss = bp[62 + t] * ph * (double)sfd[t];
        const double a2 = std::norm(h_sm[t]);
        sm += std::conj(sss) * h_raw[t] * (a2 / (2 * a2 * np + np * np));  // :836-843
      }
      M += sm;
    }
    out[i].freq_fine = cell.freq + std::arg(M) / (2 * kPi) / (1 / (fs_prog * k_factor) * g.dist);  // :848
  }
  return LCS_OK;
}

lcs_status dev_pss_sss_foe(lcs_ctx* ctx, ChainScratch& cs, const void* d_cap, int fmt, uint32_t n_cap, const lcs_cell& cell,
                           double fc_req, double fc_prog, double fs_prog, lcs_cell& out) {
  std::vector<lcs_cell> o;
  lcs_status rc = dev_pss_sss_foe_batch(ctx, cs, d_cap, fmt, n_cap, std::vector<lcs_cell>(1, cell), fc_req, fc_prog, fs_prog, o);
  if (rc == LCS_OK) out = o[0];
  return rc;
}

// extract_tfg (searcher.cpp:857-935) for several cells: one launch of (854 symbols x cells) FFT blocks, one copy back.
// status[i] = LCS_ERR_RANGE: a DFT window of that cell falls outside the capture buffer (the caller skips it).
lcs_status dev_extract_tfg_batch(lcs_ctx* ctx, ChainScratch& cs, const void* d_cap, int fmt, uint32_t n_cap,
                                 const std::vector<lcs_cell>& cells, double fc_req, double fc_prog, double fs_prog,
                                 std::vector<std::vector<cd>>& tfg, std::vector<std::vector<double>>& ts,
                                 std::vector<lcs_status>& status) {
  cudaStream_t st = ctx->chain_stream ? ctx->chain_stream : ctx->streams[0];
  const size_t P = cells.size();
  tfg.assign(P, std::vector<cd>());
  ts.assign(P, std::vector<double>());
  status.assign(P, LCS_OK);
  if (P == 0) return LCS_OK;
  LCS_CUDA(ctx, cs.h_up.ensure(P * (TFG_MAX * 12 + 16) + 64));
  Stage up(cs.h_up.p);
  int* h_pos = up.take<int>(P * TFG_MAX);
  double* h_late = up.take<double>(P * TFG_MAX);
  double* h_k = up.take<double>(P);
  int* h_n = up.take<int>(P);
  std::vector<size_t> live;
  for (size_t i = 0; i < P; i++) {
    const lcs_cell& cell = cells[i];
    const double k_factor = (fc_req - cell.freq_fine) / fc_prog;  // :875
    const double fs_ratio = 16 / kFsLte * fs_prog;
    int n_symb;
    double loc;
    if (cell.cp_type == 1) { n_symb = 7; loc = cell.frame_start + 10 * fs_ratio * k_factor; }
    else if (cell.cp_type == 2) { n_symb = 6; loc = cell.frame_start + 32 * fs_ratio * k_factor; }
    else return fail(ctx, LCS_ERR_ARG, "extract_tfg: cp_type unknown (reference throws \"Check code...\")");
    if (!(std::isfinite(loc) && std::isfinite(cell.freq_fine))) return fail(ctx, LCS_ERR_ARG, "extract_tfg: frame_start / freq_fine not set");
    if (loc - .01 * fs_prog * k_factor > -0.5) loc -= .01 * fs_prog * k_factor;  // :887-889
    const int n_ofdm = 6 * 10 * 2 * n_symb + 2 * n_symb;
    const size_t li = live.size();
    ts[i].resize(n_ofdm);
    int sym_num = 0;
    bool ok = true;
    for (int t = 0; t < n_ofdm; t++) {  // :903-920 (same running sum as the reference)
      const double r = std::rint(loc);
      if (r < 0 || r + 128 > (double)n_cap) { ok = false; break; }
      h_pos[li * TFG_MAX + t] = (int)r;
      ts[i][t] = loc;
      h_late[li * TFG_MAX + t] = r - loc;  // :925-928
      if (n_symb == 6) loc += (128 + 32) * fs_ratio * k_factor;
      else {
        loc += (sym_num == 6 ? (128 + 10) : (128 + 9)) * fs_ratio * k_factor;
        sym_num = (sym_num + 1) % 7;
      }
    }
    if (!ok) { status[i] = LCS_ERR_RANGE; ts[i].clear(); continue; }
    h_k[li] = kPi * -cell.freq_fine / ((fs_prog * k_factor) / 2);  // :892 via dsp.h:42
    h_n[li] = n_ofdm;
    live.push_back(i);
  }
  const size_t L = live.size();
  if (L == 0) return LCS_OK;
  LCS_CUDA(ctx, cs.d_starts.ensure(L * TFG_MAX));
  LCS_CUDA(ctx, cs.d_late.ensure(L * TFG_MAX));
  LCS_CUDA(ctx, cs.d_kseg.ensure(L));
  LCS_CUDA(ctx, cs.d_nofdm.ensure(L));
  LCS_CUDA(ctx, cs.d_tfg.ensure(L * TFG_MAX * 72));
  LCS_CUDA(ctx, cs.h_down.ensure(L * TFG_MAX * 72 * 16 + 64));
  LCS_CUDA(ctx, cudaMemcpyAsync(cs.d_starts.p, h_pos, L * TFG_MAX * 4, cudaMemcpyHostToDevice, st));
  LCS_CUDA(ctx, cudaMemcpyAsync(cs.d_late.p, h_late, L * TFG_MAX * 8, cudaMemcpyHostToDevice, st));
  LCS_CUDA(ctx, cudaMemcpyAsync(cs.d_kseg.p, h_k, L * 8, cudaMemcpyHostToDevice, st));
  LCS_CUDA(ctx, cudaMemcpyAsync(cs.d_nofdm.p, h_n, L * 4, cudaMemcpyHostToDevice, st));
#define CALL(F) tfg_kernel<F><<<dim3(TFG_MAX, (unsigned)L), 64, 0, st>>>(d_cap, cs.d_starts.p, cs.d_late.p, cs.d_kseg.p, cs.d_nofdm.p, cs.d_tfg.p)
  DISPATCH(fmt, CALL);
#undef CALL
  ctx->launches++;
  LCS_CUDA(ctx, cudaGetLastError());
  LCS_CUDA(ctx, cudaMemcpyAsync(cs.h_down.p, cs.d_tfg.p, L * TFG_MAX * 72 * 16, cudaMemcpyDeviceToHost, st));
  LCS_CUDA(ctx, cudaStreamSynchronize(st));
  const cd* h_tfg = reinterpret_cast<const cd*>(cs.h_down.p);
  for (size_t li = 0; li < L; li++) {
    const size_t i = live[li];
    tfg[i].assign(h_tfg + li * TFG_MAX * 72, h_tfg + li * TFG_MAX * 72 + ts[i].size() * 72);
  }
  return LCS_OK;
}

lcs_status dev_extract_tfg(lcs_ctx* ctx, ChainScratch& cs, const void* d_cap, int fmt, uint32_t n_cap, const lcs_cell& cell,
                           double fc_req, double fc_prog, double fs_prog, std::vector<cd>& tfg, std::vector<double>& ts) {
  std::vector<std::vector<cd>> g;
  std::vector<std::vector<double>> t;
  std::vector<lcs_status> st;
  lcs_status rc = dev_extract_tfg_batch(ctx, cs, d_cap, fmt, n_cap, std::vector<lcs_cell>(1, cell), fc_req, fc_prog, fs_prog, g, t, st);
  if (rc != LCS_OK) return rc;
  if (st[0] != LCS_OK) return fail(ctx, st[0], "extract_tfg: DFT window outside the capture buffer");
  tfg.swap(g[0]);
  ts.swap(t[0]);
  return LCS_OK;
}

}  // namespace lcs
