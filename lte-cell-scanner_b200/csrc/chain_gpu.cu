// chain_gpu.cu - companion kernels of the correlator (FP64): batched PSS/SSS symbol extraction
// (fshift + 2-sample rotate + 128-point FFT), SSS channel-estimate combining, SSS maximum-likelihood
// detection over the 168 x {h1h2,h2h1} x {normal,extended} hypotheses, and OFDM time/frequency-grid
// extraction (whole-buffer FOC fused into 854 FFT-128).  Reference: src/searcher.cpp:516-935.
#include <cmath>

#include "chain_gpu.hpp"
#include "fft128.cuh"
#include "iq_format.cuh"

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
// Any n_pss: the PSS positions pass through shared memory GETCE_CHUNK at a time, and each thread keeps the sums of both
// halves (even / odd k) in registers.  Every sum runs in the order of the whole-buffer form: per half k ascending, the
// noise power of one PSS over i ascending by one thread.
// ---------------------------------------------------------------------------------------------
constexpr int GETCE_CHUNK = 16;            // even: position k of a chunk is in half k & 1
constexpr int EST_LEN = 124 + 4 * 124;     // doubles per peak
struct GetceAcc {
  double den = 0;
  double2 nrm = make_double2(0, 0), ext = make_double2(0, 0);
};
__device__ __forceinline__ void getce_add(GetceAcc& acc, double npk, double2 h, double2 sss_nrm, double2 sss_ext) {
  const double inv = 1.0 / npk;
  acc.den += (h.x * h.x + h.y * h.y) * inv;
  const double2 hc = make_double2(h.x * inv, -h.y * inv);
  const double2 a = cmul(hc, sss_nrm);
  const double2 b = cmul(hc, sss_ext);
  acc.nrm.x += a.x; acc.nrm.y += a.y;
  acc.ext.x += b.x; acc.ext.y += b.y;
}
__global__ void __launch_bounds__(64) sss_getce_kernel(const double2* __restrict__ psss_all, const int3* __restrict__ par,
                                                       const double2* __restrict__ pss_fd_all, double* __restrict__ est_all) {
  __shared__ double2 h_raw[GETCE_CHUNK * 62];
  __shared__ double2 h_sm[GETCE_CHUNK * 62];
  __shared__ double np[GETCE_CHUNK];
  const int3 pp = par[blockIdx.x];
  const int n_pss = pp.y;
  const double2* psss = psss_all + (size_t)pp.x * 62;
  const double2* pss_fd = pss_fd_all + pp.z * 62;
  double* est = est_all + (size_t)blockIdx.x * EST_LEN;
  const int t = threadIdx.x;
  const double2 pc = t < 62 ? make_double2(pss_fd[t].x, -pss_fd[t].y) : make_double2(0, 0);
  GetceAcc acc[2];   // [half], indexed with constants only
  for (int k0 = 0; k0 < n_pss; k0 += GETCE_CHUNK) {
    const int nk = min(GETCE_CHUNK, n_pss - k0);
    const double2* pk = psss + (size_t)k0 * 3 * 62;
    if (t < 62)
      for (int k = 0; k < nk; k++) h_raw[k * 62 + t] = cmul(pk[((size_t)k * 3 + 0) * 62 + t], pc);
    __syncthreads();
    if (t < 62) {
      const int lt = max(0, t - 6), rt = min(61, t + 6);
      for (int k = 0; k < nk; k++) {
        double2 s = make_double2(0, 0);
        for (int i = lt; i <= rt; i++) { s.x += h_raw[k * 62 + i].x; s.y += h_raw[k * 62 + i].y; }
        const double n = (double)(rt - lt + 1);
        h_sm[k * 62 + t] = make_double2(s.x / n, s.y / n);
      }
    }
    __syncthreads();
    if (t < nk) {  // noise power of PSS k0 + t (sigpower, dsp.h:23-29)
      double r = 0;
      for (int i = 0; i < 62; i++) {
        const double dx = h_sm[t * 62 + i].x - h_raw[t * 62 + i].x, dy = h_sm[t * 62 + i].y - h_raw[t * 62 + i].y;
        r += dx * dx + dy * dy;
      }
      np[t] = r / 62;
    }
    __syncthreads();
    if (t < 62) {
      for (int k = 0; k < nk; k += 2) {
        getce_add(acc[0], np[k], h_sm[k * 62 + t], pk[((size_t)k * 3 + 2) * 62 + t], pk[((size_t)k * 3 + 1) * 62 + t]);
        if (k + 1 < nk)
          getce_add(acc[1], np[k + 1], h_sm[(k + 1) * 62 + t], pk[((size_t)(k + 1) * 3 + 2) * 62 + t],
                    pk[((size_t)(k + 1) * 3 + 1) * 62 + t]);
      }
    }
    __syncthreads();   // the next chunk overwrites h_raw, h_sm and np
  }
  if (t < 62) {
    double2* estc = reinterpret_cast<double2*>(est + 124);
#pragma unroll
    for (int half = 0; half < 2; half++) {
      const double npe = 1.0 / (1.0 + acc[half].den);
      est[half * 62 + t] = npe;
      estc[(0 + half) * 62 + t] = make_double2(npe * acc[half].nrm.x, npe * acc[half].nrm.y);
      estc[(2 + half) * 62 + t] = make_double2(npe * acc[half].ext.x, npe * acc[half].ext.y);
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
// Grid (854, cells): pos / late / tfg are [cell][854], kcell[cell], n_ofdm[cell] (732 for the extended CP).  base[cell]
// (NULL: 0) is the first sample of the cell's capture buffer in cap; positions and the FOC phase count from there.
template <int FMT>
__global__ void __launch_bounds__(64) tfg_kernel(const void* __restrict__ cap, const uint64_t* __restrict__ base,
                                                 const int* __restrict__ pos_all, const double* __restrict__ late_all,
                                                 const double* __restrict__ kcell, const int* __restrict__ n_ofdm,
                                                 double2* __restrict__ tfg_all) {
  __shared__ double2 buf[128];
  __shared__ double2 tw[64];
  const int tid = threadIdx.x, sym = blockIdx.x, cell = blockIdx.y;
  if (sym >= n_ofdm[cell]) return;
  const int* pos = pos_all + (size_t)cell * TFG_MAX;
  const double* late = late_all + (size_t)cell * TFG_MAX;
  double2* tfg = tfg_all + (size_t)cell * TFG_MAX * 72;
  const double k = kcell[cell];
  const size_t b0 = base ? (size_t)base[cell] : 0;
  make_twiddles(tw, tid);
  const size_t p0 = (size_t)pos[sym];
  for (int n = tid; n < 128; n += 64) {
    double sn, cs;
    sincos(k * (double)(p0 + n), &sn, &cs);
    buf[bitrev7(n)] = cmul(load_c<FMT>(cap, b0 + p0 + n), make_double2(cs, sn));
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

// =============================================================================================
// Host drivers (device-resident capture buffer)
// =============================================================================================
// The SSS and PSS tables of the detector, uploaded by the first call.  A failed upload keeps neither table, so the next
// call builds both again.
static cudaError_t sss_tables(ChainScratch& cs) {
  if (cs.d_sss_tab.p) return cudaSuccess;
  std::vector<signed char> tab((size_t)168 * 3 * 2 * 62);
  int v[62];
  for (int n1 = 0; n1 < 168; n1++)
    for (int n2 = 0; n2 < 3; n2++)
      for (int s = 0; s < 2; s++) {
        sss_fd(n1, n2, s * 10, v);
        for (int i = 0; i < 62; i++) tab[(((size_t)n1 * 3 + n2) * 2 + s) * 62 + i] = (signed char)v[i];
      }
  cd fd[3][62];
  for (int t = 0; t < 3; t++) pss_fd(t, fd[t]);
  DevBuf<signed char> d_sss;
  DevBuf<double2> d_pss;
  cudaError_t e = d_sss.alloc(tab.size());
  if (e == cudaSuccess) e = d_pss.alloc(3 * 62);
  if (e == cudaSuccess) e = cudaMemcpy(d_sss.p, tab.data(), tab.size(), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(d_pss.p, fd, sizeof(fd), cudaMemcpyHostToDevice);
  if (e != cudaSuccess) return e;
  cs.d_sss_tab.swap(d_sss);
  cs.d_pss_fd.swap(d_pss);
  return cudaSuccess;
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
// n LTE samples (at FS_LTE/16) in capture samples: n*16/FS_LTE*fs_programmed*k_factor, rounded left to right as
// searcher.cpp writes it everywhere.  Another grouping moves timestamps by ulps off the nominal clock.
static inline double cap_samples(double n, double fs_prog, double k_factor) { return n * 16 / kFsLte * fs_prog * k_factor; }
static inline double wrapd(double x, double sm, double lg) {  // macros.h:49 with itpp_ext.h:40-42
  const double n = lg - sm, k = x - sm;
  return (n == 0 ? k : k - n * (int)std::floor(k / n)) + sm;
}

// All 128-sample segments of a stage through one psss launch; bins land in cs.d_psss.  starts and kseg go to ctx->chain.up
// after the slices the caller took since its reset (which counts them too), and one copy uploads all of them.
static lcs_status run_psss(const StageCall& sc, const std::vector<int>& starts, const std::vector<double>& kseg) {
  lcs_ctx* ctx = sc.ctx;
  ChainScratch& cs = ctx->chain;
  const size_t n = starts.size();
  LCS_CUDA(ctx, cs.d_psss.ensure(n * 62));
  const int* hs = cs.up.put(starts);
  const double* hk = cs.up.put(kseg);
  LCS_CUDA(ctx, cs.up.upload(sc.st));
  if (SearchFormats::dispatch(sc.fmt, [&](auto FMT) {
        psss_kernel<FMT><<<(unsigned)n, 64, 0, sc.st>>>(sc.d_cap, cs.up.dev(hs), cs.up.dev(hk), cs.d_psss.p);
      }) != LCS_OK)
    return fail(ctx, LCS_ERR_ARG, "psss: bad iq_format");
  ctx->launches++;
  LCS_CUDA(ctx, cudaGetLastError());
  return LCS_OK;
}

// sss_detect (searcher.cpp:696-761) for all PSS peaks of a capture buffer: one FFT launch over every (peak, PSS position,
// {PSS, SSS-ext, SSS-nrm}) segment, one channel-estimate block and 168 x 4 likelihood warps per peak, ONE synchronisation.
// st[i] = LCS_ERR_RANGE marks a peak for which the reference would index outside the buffer (the caller skips it).
lcs_status dev_sss_detect_batch(const StageCall& sc, const std::vector<lcs_cell>& cells, double thresh2_n_sigma,
                                std::vector<lcs_cell>& out, std::vector<lcs_status>& status, SssDebugHost* dbg) {
  lcs_ctx* ctx = sc.ctx;
  ChainScratch& cs = ctx->chain;
  const double fc_req = sc.cfg.fc_req, fc_prog = sc.cfg.fc_prog, fs_prog = sc.cfg.fs_prog;
  const size_t P = cells.size();
  out.assign(cells.begin(), cells.end());
  status.assign(P, LCS_OK);
  if (P == 0) return LCS_OK;
  if (sss_tables(cs) != cudaSuccess) return fail(ctx, LCS_ERR_CUDA, "sss table upload failed");
  std::vector<int> starts;
  std::vector<double> kseg;
  std::vector<int3> par;
  std::vector<size_t> live;      // peaks that take part in the launches
  for (size_t i = 0; i < P; i++) {
    const lcs_cell& cell = cells[i];
    if (cell.n_id_2 < 0 || cell.n_id_2 > 2) return fail(ctx, LCS_ERR_ARG, "sss_detect: n_id_2 out of range");
    // PSS positions with an SSS in front of them (searcher.cpp:549-563)
    double peak_loc = cell.ind;
    const double k_factor = (fc_req - cell.freq) / fc_prog;
    if (peak_loc + 9 < 162) peak_loc += 9600 * k_factor;
    const std::vector<double> locs = mrange(peak_loc, k_factor * 9600, (double)sc.n_cap - 125 - 9);
    const int n_pss = (int)locs.size();
    if (n_pss < 1) { status[i] = LCS_ERR_RANGE; continue; }
    const size_t seg0 = starts.size();
    bool ok = true;
    for (int k = 0; k < n_pss && ok; k++) {
      const long pss_dft = (long)std::rint(locs[k]) + 9 - 2;
      const long sg[3] = {pss_dft, pss_dft - 128 - 32, pss_dft - 128 - 9};  // :579,:594,:596
      for (long v : sg) {
        if (v < 0 || v + 128 > (long)sc.n_cap) { ok = false; break; }
        starts.push_back((int)v);
      }
    }
    if (!ok) { starts.resize(seg0); status[i] = LCS_ERR_RANGE; continue; }   // DFT window outside the capture buffer
    const double kk = kPi * -cell.freq / ((fs_prog * k_factor) / 2);         // dsp.h:42
    kseg.resize(starts.size(), kk);
    par.push_back(make_int3((int)seg0, n_pss, cell.n_id_2));
    live.push_back(i);
  }
  if (live.empty()) return LCS_OK;
  const size_t L = live.size();
  LCS_CUDA(ctx, cs.up.reset(L * sizeof(int3) + starts.size() * 12 + 3 * 16));
  const int3* h_par = cs.up.put(par);
  lcs_status rc = run_psss(sc, starts, kseg);
  if (rc != LCS_OK) return rc;
  LCS_CUDA(ctx, cs.d_est.ensure(L * EST_LEN));
  LCS_CUDA(ctx, cs.d_ll.ensure(L * 4 * 168));
  LCS_CUDA(ctx, cs.h_down.ensure(L * (4 * 168 + EST_LEN) * 8 + 64));
  const int3* d_par = cs.up.dev(h_par);
  sss_getce_kernel<<<(unsigned)L, 64, 0, sc.st>>>(cs.d_psss.p, d_par, cs.d_pss_fd.p, cs.d_est.p);
  sss_ml_kernel<<<dim3(168, (unsigned)L), 128, 0, sc.st>>>(cs.d_est.p, cs.d_sss_tab.p, d_par, cs.d_ll.p);
  ctx->launches += 2;
  LCS_CUDA(ctx, cudaGetLastError());
  double* h_ll = reinterpret_cast<double*>(cs.h_down.p);
  double* h_est = h_ll + L * 4 * 168;
  LCS_CUDA(ctx, cudaMemcpyAsync(h_ll, cs.d_ll.p, L * 4 * 168 * 8, cudaMemcpyDeviceToHost, sc.st));
  if (dbg) LCS_CUDA(ctx, cudaMemcpyAsync(h_est, cs.d_est.p, L * EST_LEN * 8, cudaMemcpyDeviceToHost, sc.st));
  LCS_CUDA(ctx, cudaStreamSynchronize(sc.st));
  for (size_t li = 0; li < L; li++) {
    const lcs_cell& cell = cells[live[li]];
    const double* ll = h_ll + li * 4 * 168;
    const double k_factor = (fc_req - cell.freq) / fc_prog;
    // decisions (searcher.cpp:719-758)
    const double* nrm0 = &ll[0], *nrm1 = &ll[168], *ext0 = &ll[336], *ext1 = &ll[504];
    auto mx = [](const double* v) { return *std::max_element(v, v + 168); };
    const bool normal = std::max(mx(nrm0), mx(nrm1)) > std::max(mx(ext0), mx(ext1));
    const double* c0 = normal ? nrm0 : ext0, *c1 = normal ? nrm1 : ext1;
    double frame_start = cell.ind + cap_samples(128 + 9 - 960 - 2, fs_prog, k_factor);  // :735
    const double* col;
    if (mx(c0) > mx(c1)) col = c0;
    else { col = c1; frame_start += cap_samples(9600 * k_factor, fs_prog, k_factor); }  // :741
    frame_start = wrapd(frame_start, -0.5, cap_samples(2 * 9600.0 - 0.5, fs_prog, k_factor));  // :743
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

// pss_sss_foe (searcher.cpp:767-850) for several cells: one FFT launch, one synchronisation.
lcs_status dev_pss_sss_foe_batch(const StageCall& sc, const std::vector<lcs_cell>& cells, std::vector<lcs_cell>& out) {
  lcs_ctx* ctx = sc.ctx;
  ChainScratch& cs = ctx->chain;
  const double fc_req = sc.cfg.fc_req, fc_prog = sc.cfg.fc_prog, fs_prog = sc.cfg.fs_prog;
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
    int dist;
    double first;
    if (cell.cp_type == 1) {
      dist = (int)std::rint(cap_samples(128 + 9, fs_prog, k_factor));  // :780
      first = cell.frame_start + cap_samples(960 - 128 - 9 - 128, fs_prog, k_factor);
    } else if (cell.cp_type == 2) {
      dist = (int)std::rint((128 + 32) * k_factor);  // :783
      first = cell.frame_start + cap_samples(960 - 128 - 32 - 128, fs_prog, k_factor);
    } else {
      return fail(ctx, LCS_ERR_ARG, "pss_sss_foe: cp_type unknown (reference throws \"Error... check code...\")");
    }
    int sn;
    first = wrapd(first, -0.5, 9600 * 2 - 0.5);
    if (first - 9600 * k_factor > -0.5) { first -= 9600 * k_factor; sn = 10; } else sn = 0;
    const std::vector<double> locs = mrange(first, cap_samples(9600, fs_prog, k_factor), (double)((long)sc.n_cap - 127 - dist - 100));
    geo[i] = Geo{dist, (int)locs.size(), sn, starts.size()};
    for (size_t k = 0; k < locs.size(); k++) {
      const long sg = (long)std::rint(locs[k]);
      if (sg < 0 || sg + dist + 128 > (long)sc.n_cap) return fail(ctx, LCS_ERR_RANGE, "pss_sss_foe: DFT window outside the capture buffer");
      starts.push_back((int)(sg + dist));  // PSS
      starts.push_back((int)sg);           // SSS
    }
    kseg.resize(starts.size(), kPi * -cell.freq / ((fs_prog * k_factor) / 2));
  }
  const cd* bins = nullptr;
  if (!starts.empty()) {
    LCS_CUDA(ctx, cs.up.reset(starts.size() * 12 + 2 * 16));
    lcs_status rc = run_psss(sc, starts, kseg);
    if (rc != LCS_OK) return rc;
    LCS_CUDA(ctx, cs.h_down.ensure(starts.size() * 62 * 16 + 64));
    LCS_CUDA(ctx, cudaMemcpyAsync(cs.h_down.p, cs.d_psss.p, starts.size() * 62 * 16, cudaMemcpyDeviceToHost, sc.st));
    LCS_CUDA(ctx, cudaStreamSynchronize(sc.st));
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

GridTables::GridTables(Staging& up, size_t n_cells, bool with_base)
    : pos(up.take<int>(n_cells * TFG_MAX)), late(up.take<double>(n_cells * TFG_MAX)), k(up.take<double>(n_cells)),
      n_ofdm(up.take<int>(n_cells)), base(with_base ? up.take<uint64_t>(n_cells) : nullptr) {}

lcs_status tfg_geometry(const lcs_cell& cell, double fc_req, double fc_prog, double fs_prog, uint32_t n_cap, const GridTables& g,
                        size_t slot, double* ts, const char** why) {
  int* pos = g.pos + slot * TFG_MAX;
  double* late = g.late + slot * TFG_MAX;
  const double k_factor = (fc_req - cell.freq_fine) / fc_prog;  // :875
  int n_symb;
  double loc;
  if (cell.cp_type == 1) { n_symb = 7; loc = cell.frame_start + cap_samples(10, fs_prog, k_factor); }
  else if (cell.cp_type == 2) { n_symb = 6; loc = cell.frame_start + cap_samples(32, fs_prog, k_factor); }
  else { *why = "cp_type unknown (reference throws \"Check code...\")"; return LCS_ERR_ARG; }
  if (!(std::isfinite(loc) && std::isfinite(cell.freq_fine))) { *why = "frame_start / freq_fine not set"; return LCS_ERR_ARG; }
  if (loc - .01 * fs_prog * k_factor > -0.5) loc -= .01 * fs_prog * k_factor;  // :887-889
  const int n_ofdm = 6 * 10 * 2 * n_symb + 2 * n_symb;
  int sym_num = 0;
  for (int t = 0; t < n_ofdm; t++) {  // :903-920 (same running sum as the reference)
    const double r = std::rint(loc);
    if (r < 0 || r + 128 > (double)n_cap) { *why = "DFT window outside the capture buffer"; return LCS_ERR_RANGE; }
    pos[t] = (int)r;
    ts[t] = loc;
    late[t] = r - loc;  // :925-928
    if (n_symb == 6) loc += cap_samples(128 + 32, fs_prog, k_factor);
    else {
      loc += cap_samples(sym_num == 6 ? (128 + 10) : (128 + 9), fs_prog, k_factor);
      sym_num = (sym_num + 1) % 7;
    }
  }
  g.k[slot] = kPi * -cell.freq_fine / ((fs_prog * k_factor) / 2);  // :892 via dsp.h:42
  g.n_ofdm[slot] = n_ofdm;
  return LCS_OK;
}

lcs_status launch_grids(lcs_ctx* ctx, const Staging& up, const GridTables& g, uint32_t n_cells, const void* d_cap, int fmt,
                        double2* d_tfg, cudaStream_t st, const char* bad_fmt) {
  const uint64_t* d_base = g.base ? up.dev(g.base) : nullptr;
  if (SearchFormats::dispatch(fmt, [&](auto FMT) {
        tfg_kernel<FMT><<<dim3(TFG_MAX, n_cells), 64, 0, st>>>(d_cap, d_base, up.dev(g.pos), up.dev(g.late), up.dev(g.k),
                                                               up.dev(g.n_ofdm), d_tfg);
      }) != LCS_OK)
    return fail(ctx, LCS_ERR_ARG, bad_fmt);
  ctx->launches++;
  LCS_CUDA(ctx, cudaGetLastError());
  return LCS_OK;
}

// extract_tfg (searcher.cpp:857-935) for several cells: one launch of (854 symbols x cells) FFT blocks, one copy back.
// status[i] = LCS_ERR_RANGE: a DFT window of that cell falls outside the capture buffer (the caller skips it).
lcs_status dev_extract_tfg_batch(const StageCall& sc, const std::vector<lcs_cell>& cells, std::vector<std::vector<cd>>& tfg,
                                 std::vector<std::vector<double>>& ts, std::vector<lcs_status>& status) {
  lcs_ctx* ctx = sc.ctx;
  ChainScratch& cs = ctx->chain;
  const size_t P = cells.size();
  tfg.assign(P, std::vector<cd>());
  ts.assign(P, std::vector<double>());
  status.assign(P, LCS_OK);
  if (P == 0) return LCS_OK;
  LCS_CUDA(ctx, cs.up.reset(GridTables::bytes(P)));
  const GridTables g(cs.up, P, false);
  std::vector<size_t> live;
  std::vector<double> t(TFG_MAX);
  for (size_t i = 0; i < P; i++) {
    const size_t li = live.size();
    const char* why = "";
    const lcs_status rc = tfg_geometry(cells[i], sc.cfg.fc_req, sc.cfg.fc_prog, sc.cfg.fs_prog, sc.n_cap, g, li, t.data(), &why);
    if (rc == LCS_ERR_ARG) return fail(ctx, rc, std::string("extract_tfg: ") + why);
    if (rc != LCS_OK) { status[i] = rc; continue; }
    ts[i].assign(t.begin(), t.begin() + g.n_ofdm[li]);
    live.push_back(i);
  }
  const size_t L = live.size();
  if (L == 0) return LCS_OK;
  LCS_CUDA(ctx, cs.d_tfg.ensure(L * TFG_MAX * 72));
  LCS_CUDA(ctx, cs.h_down.ensure(L * TFG_MAX * 72 * 16 + 64));
  LCS_CUDA(ctx, cs.up.upload(sc.st));
  lcs_status rc = launch_grids(ctx, cs.up, g, (uint32_t)L, sc.d_cap, sc.fmt, cs.d_tfg.p, sc.st, "extract_tfg: bad iq_format");
  if (rc != LCS_OK) return rc;
  LCS_CUDA(ctx, cudaMemcpyAsync(cs.h_down.p, cs.d_tfg.p, L * TFG_MAX * 72 * 16, cudaMemcpyDeviceToHost, sc.st));
  LCS_CUDA(ctx, cudaStreamSynchronize(sc.st));
  const cd* h_tfg = reinterpret_cast<const cd*>(cs.h_down.p);
  for (size_t li = 0; li < L; li++) {
    const size_t i = live[li];
    tfg[i].assign(h_tfg + li * TFG_MAX * 72, h_tfg + li * TFG_MAX * 72 + ts[i].size() * 72);
  }
  return LCS_OK;
}

}  // namespace lcs
