// search_batch.cu - threshold + peak_search on the device and every search entry point, all built on one driver
// (SURVEY 8f rank 2: no host round trip between xcorr_pss and the per-peak stages of a sweep).
//
//   peak_search_kernel          src/searcher.cpp:422-510 with Z_th1 of src/CellSearch.cpp:500-503 folded in
//   lcs_xcorr_peaks_batch_host  xcorr_pss + threshold + peak_search for a batch of host capture buffers
//   lcs_cell_search_batch_cu8   the whole chain of CellSearch.cpp:497-558 per buffer of a batch
//   lcs_cell_search[_cu8], lcs_kalibrate_cu8, lcs_tracker_search_cu8
//                               the same for one buffer, as a batch of one on the context's cached plan
//   lcs_sweep_*                 one plan per channel, all channels of a chunk in one correlator launch
#include <cmath>
#include <cstring>
#include <vector>

#include "chain_gpu.hpp"
#include "chain_host.hpp"
#include "iq_format.cuh"
#include "lcs_ctx.hpp"

namespace lcs {

struct DevPeak {
  double pss_pow;
  int32_t ind;      // refined index (-1: the reference's uint16 wrap, searcher.cpp:459)
  int32_t fi;       // index into f_search_set
  int32_t row;      // n_id_2
  int32_t col;      // peak column before refinement
};

constexpr int PK_THREADS = 512;

// Length of a buffer's device peak list.  After each peak the kernel zeroes every position of its row within circular
// distance 274, and a position holding 0 is never taken (!(v > 0) stops the search).  So the peaks of one row are
// pairwise at least 275 apart on a circle of LCS_N_FOLD positions: at most 9600 / 275 = 34 per row, 102 per buffer, and
// the list cannot overflow.
constexpr int SEARCH_MAX_PEAKS = 3 * (LCS_N_FOLD / 275);
static_assert(SEARCH_MAX_PEAKS == 102, "peak list length");

// (value, flat index) arg-max with the reference's tie rule: first maximum of each row, rows compared with a strict
// '>' in order 0,1,2 (searcher.cpp:441-445)  ==  largest value, smallest flat index row*9600+col among equals.
__device__ __forceinline__ void argmax_combine(double& v, int& i, double v2, int i2) {
  if (v2 > v || (v2 == v && i2 < i)) { v = v2; i = i2; }
}

// One CTA per capture buffer.  `work` ([batch][3][9600] double scratch) is written only once a peak has been found:
// buffers without a PSS above threshold cost a single pass over `pow`.
__global__ void __launch_bounds__(PK_THREADS) peak_search_kernel(const double* __restrict__ pow_all, const int32_t* __restrict__ frq_all,
                                                                 const double* __restrict__ spi_all, const float* __restrict__ single_all,
                                                                 double* __restrict__ work_all, DevPeak* __restrict__ peaks_all,
                                                                 int32_t* __restrict__ npeaks_all, uint32_t n_f /* stride */, double r_th1,
                                                                 double rx_cutoff, double n_comb, double box, int arm, double cancel) {
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int N = 3 * LCS_N_FOLD;
  const double* pw = pow_all + (size_t)b * N;
  const int32_t* frq = frq_all + (size_t)b * N;
  const double* spi = spi_all + (size_t)b * LCS_N_FOLD;
  const float* single = single_all + (size_t)b * 3 * n_f * LCS_N_FOLD;
  double* work = work_all + (size_t)b * N;
  __shared__ double s_v[PK_THREADS / 32];
  __shared__ int s_i[PK_THREADS / 32];
  __shared__ double s_best;
  __shared__ int s_besti;
  __shared__ bool s_stop;
  const double* src = pw;
  int n_found = 0;
  for (;;) {
    double v = -INFINITY;
    int vi = 0x7fffffff;
    for (int i = tid; i < N; i += PK_THREADS) argmax_combine(v, vi, src[i], i);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const double v2 = __shfl_xor_sync(0xffffffffu, v, o);
      const int i2 = __shfl_xor_sync(0xffffffffu, vi, o);
      argmax_combine(v, vi, v2, i2);
    }
    if (lane == 0) { s_v[warp] = v; s_i[warp] = vi; }
    __syncthreads();
    if (tid == 0) {
      for (int w = 1; w < PK_THREADS / 32; w++) argmax_combine(v, vi, s_v[w], s_i[w]);
      const int row = vi / LCS_N_FOLD, col = vi - row * LCS_N_FOLD;
      // Z_th1 (CellSearch.cpp:500-503), same operation order as the host code
      const double z = r_th1 * spi[col] / rx_cutoff / 137 / 2 / n_comb / box;
      const bool stop = (v < z) || !(v > 0);                             // searcher.cpp:446 (+ all-zero guard as on the host)
      if (!stop) {
        const int fi = frq[vi];
        int ind = -1;                                                     // searcher.cpp:457-465 incl. the uint16 wrap
        if (col >= arm) {
          float bp = -INFINITY;
          for (int t = col - arm; t <= col + arm; t++) {
            const int tw = t % LCS_N_FOLD;
            const float sv = single[((size_t)row * n_f + fi) * LCS_N_FOLD + tw];
            if (sv > bp) { bp = sv; ind = tw; }
          }
        }
        DevPeak pk;
        pk.pss_pow = v; pk.ind = ind; pk.fi = fi; pk.row = row; pk.col = col;
        peaks_all[(size_t)b * SEARCH_MAX_PEAKS + n_found] = pk;
      }
      s_best = v; s_besti = vi; s_stop = stop;
    }
    __syncthreads();
    if (s_stop) {
      if (tid == 0) npeaks_all[b] = n_found;
      return;
    }
    n_found++;
    const double best = s_best;
    const int row = s_besti / LCS_N_FOLD, col = s_besti - row * LCS_N_FOLD;
    const double th = best * cancel;                                      // searcher.cpp:501
    // no second peak of the same PSS within +-274 samples (:481-484); drop everything 12 dB below this peak (:501-508)
    for (int i = tid; i < N; i += PK_THREADS) {
      double x = src[i];
      const int r = i / LCS_N_FOLD, c = i - r * LCS_N_FOLD;
      if (r == row) {
        int d = c - col;
        if (d < 0) d = -d;
        if (d > LCS_N_FOLD / 2) d = LCS_N_FOLD - d;                       // circular distance
        if (d <= 274) x = 0;
      }
      if (x < th) x = 0;
      work[i] = x;
    }
    src = work;
    __syncthreads();
  }
}

static lcs_status launch_peak_search(lcs_ctx* ctx, const XcorrGeom& g, uint32_t nb, const double* d_pow, const int32_t* d_frq,
                                     const double* d_spi, const float* d_single, double* d_work, DevPeak* d_peaks, int32_t* d_npeaks,
                                     cudaStream_t st) {
  const double r_th1 = chi2cdf_inv(1 - std::pow(10.0, -12.0), 2.0 * g.n_comb_xc * (2 * g.ds_comb_arm + 1));
  const double rx_cutoff = (6 * 12 * 15e3 / 2 + 4 * 15e3) / ((30720000.0 / 16) / 2);
  const double cancel = std::pow(10.0, -12.0 / 10.0);
  peak_search_kernel<<<nb, PK_THREADS, 0, st>>>(d_pow, d_frq, d_spi, d_single, d_work, d_peaks, d_npeaks, g.n_f_stride, r_th1, rx_cutoff,
                                                (double)g.n_comb_xc, (double)(2 * g.ds_comb_arm + 1), (int)g.ds_comb_arm, cancel);
  ctx->launches++;
  LCS_CUDA(ctx, cudaGetLastError());
  return LCS_OK;
}

// Shared driver: xcorr_pss + threshold + peak_search for `batch` host capture buffers in chunks on the context's streams
// (rotate_chunks); `per_buffer(buffer index, StageCall of the buffer, its PSS peaks)` runs on the host after the chunk's
// kernels finished while the next chunks are already in flight on the other streams.  The StageCall names the buffer's
// IQ bytes on the device, its PlanCfg and the chunk's stream, which is idle by then: the per-peak kernels do not queue
// behind later chunks.
// d_buf_plan == NULL: every buffer is searched with plan 0 of `ps`; otherwise buffer b uses plan d_buf_plan[b] and
// h_buf_plan[b] names the same plan on the host.
// device_input: h_iq is device memory; each chunk is searched in place there (no host-to-device copy).
template <class F>
static lcs_status search_chunks(lcs_ctx* ctx, PlanSet& ps, int kernel, lcs_xcorr_plan::HostBatchBufs (&hbs)[lcs_ctx::N_STREAMS], const void* h_iq,
                                int iq_format, uint32_t batch, uint32_t chunk, const uint32_t* d_buf_plan, const uint32_t* h_buf_plan,
                                F&& per_buffer, bool device_input = false) {
  const XcorrGeom& g = ps.geom;
  if (!SearchFormats::has(iq_format)) return fail(ctx, LCS_ERR_ARG, "search_batch: bad iq_format");
  const size_t samp_bytes = sample_bytes(iq_format);
  if (batch == 0) return LCS_OK;
  LCS_CUDA(ctx, cudaSetDevice(ctx->device));
  chunk = std::max<uint32_t>(1, std::min<uint32_t>(chunk, batch));
  const uint32_t n_chunks = (batch + chunk - 1) / chunk;
  // buffers only for the streams that get a chunk (a single-buffer search uses one stream)
  for (int s = 0; s < (int)std::min<uint32_t>(lcs_ctx::N_STREAMS, n_chunks); s++)
    LCS_CUDA(ctx, hbs[s].ensure(g, chunk, samp_bytes, !device_input, true));
  // device IQ of the chunk starting at buffer b0 on stream s
  auto chunk_iq = [&](uint32_t b0, int s) -> const unsigned char* {
    return device_input ? (const unsigned char*)h_iq + (size_t)b0 * g.n_cap * samp_bytes : hbs[s].iq.p;
  };
  auto issue = [&](uint32_t b0, int s) -> lcs_status {
    const uint32_t nb = std::min(chunk, batch - b0);
    cudaStream_t st = ctx->streams[s];
    auto& hb = hbs[s];
    if (!device_input)
      LCS_CUDA(ctx, cudaMemcpyAsync(hb.iq.p, (const char*)h_iq + (size_t)b0 * g.n_cap * samp_bytes, (size_t)nb * g.n_cap * samp_bytes,
                                    cudaMemcpyHostToDevice, st));
    lcs_status rc = planset_run(ps, kernel, chunk_iq(b0, s), iq_format, nb, d_buf_plan ? d_buf_plan + b0 : nullptr, hb.single.p, hb.pow.p,
                                hb.frq.p, hb.spi.p, nullptr, st);
    if (rc != LCS_OK) return rc;
    rc = launch_peak_search(ctx, g, nb, hb.pow.p, hb.frq.p, hb.spi.p, hb.single.p, hb.work.p, reinterpret_cast<DevPeak*>(hb.peaks.p),
                            hb.npeaks.p, st);
    if (rc != LCS_OK) return rc;
    LCS_CUDA(ctx, cudaMemcpyAsync(hb.h_npeaks.p, hb.npeaks.p, nb * 4, cudaMemcpyDeviceToHost, st));
    LCS_CUDA(ctx, cudaMemcpyAsync(hb.h_peaks.p, hb.peaks.p, (size_t)nb * SEARCH_MAX_PEAKS * sizeof(DevPeak), cudaMemcpyDeviceToHost, st));
    return LCS_OK;
  };
  auto finish = [&](uint32_t b0, int s) -> lcs_status {
    const uint32_t nb = std::min(chunk, batch - b0);
    auto& hb = hbs[s];
    const DevPeak* h_peaks = reinterpret_cast<const DevPeak*>(hb.h_peaks.p);
    LCS_CUDA(ctx, cudaStreamSynchronize(ctx->streams[s]));
    std::vector<lcs_cell> pk;
    for (uint32_t i = 0; i < nb; i++) {
      const PlanCfg& cfg = ps.cfg[h_buf_plan ? h_buf_plan[b0 + i] : 0];
      pk.clear();
      for (int k = 0; k < hb.h_npeaks.p[i]; k++) {
        const DevPeak& d = h_peaks[(size_t)i * SEARCH_MAX_PEAKS + k];
        lcs_cell c;
        lcs_cell_init(&c);
        c.fc_requested = cfg.fc_req;
        c.fc_programmed = cfg.fc_prog;
        c.pss_pow = d.pss_pow;
        c.ind = d.ind;
        c.freq = cfg.f[d.fi];
        c.n_id_2 = (int8_t)d.row;
        pk.push_back(c);
      }
      const StageCall sc{ctx, chunk_iq(b0, s) + (size_t)i * g.n_cap * samp_bytes, iq_format, g.n_cap, cfg, ctx->streams[s]};
      lcs_status rc = per_buffer(b0 + i, sc, pk);
      if (rc != LCS_OK) return rc;
    }
    return LCS_OK;
  };
  return rotate_chunks(batch, chunk, issue, finish);
}

// What a searcher cycle of a tracked channel (src/searcher_thread.cpp:95-232) adds to a cell search.
struct TrackerCycle {
  const int32_t* tracked;    // n_id_cell of the channel's tracked cells: skipped
  uint32_t n_tracked;
  double late;               // lateness of the buffer, from the framer
  double* frame_timing;      // [batch][max_cells]: the timing handed to each new cell's tracker
};

// The per-buffer step of the cell-search entry points: the per-peak chain (CellSearch.cpp:510-558) on buffer b of a
// search_chunks call; writes cells[b * max_cells ...] and n_cells[b].
static lcs_status chain_step(uint32_t b, const StageCall& sc, const std::vector<lcs_cell>& pk, lcs_cell* cells, uint32_t max_cells,
                             uint32_t* n_cells, const TrackerCycle* tc = nullptr) {
  lcs_cell* out = cells ? cells + (size_t)b * max_cells : nullptr;
  uint32_t found = 0;
  const lcs_status rc = cell_chain_dev(sc, pk, out, max_cells, &found, tc ? tc->tracked : nullptr, tc ? tc->n_tracked : 0, tc != nullptr);
  n_cells[b] = found;
  if (tc) {
    const PlanCfg& cfg = sc.cfg;
    const double k_factor = (cfg.fc_req - cfg.f[0]) / cfg.fc_prog;
    for (uint32_t i = 0; i < found && i < max_cells; i++)                                  // searcher_thread.cpp:214
      tc->frame_timing[(size_t)b * max_cells + i] = out[i].frame_start * (30720000.0 / 16) / (cfg.fs_prog * k_factor) + tc->late;
  }
  return rc;
}

// One capture buffer through search_chunks as a batch of one, on the context's cached plan for its configuration.
static lcs_status search_one(lcs_ctx* ctx, const void* capbuf, int fmt, uint32_t n_cap, const double* f_search_set, uint32_t n_f,
                             double fc_req, double fc_prog, double fs_prog, lcs_cell* cells, uint32_t max_cells, uint32_t* n_cells,
                             lcs_cell* peaks, uint32_t* n_peaks, const TrackerCycle* tc = nullptr) {
  const uint8_t DS_COMB_ARM = 2;        // CellSearch.cpp:484
  lcs_xcorr_plan* p = nullptr;
  lcs_status rc = get_cached_plan(ctx, n_cap, f_search_set, n_f, DS_COMB_ARM, fc_req, fc_prog, fs_prog, &p);
  if (rc != LCS_OK) return rc;
  uint32_t found = 0;
  rc = search_chunks(ctx, p->ps, p->kernel, p->hb, capbuf, fmt, 1, 1, nullptr, nullptr,
                     [&](uint32_t b, const StageCall& sc, const std::vector<lcs_cell>& pk) {
                       if (n_peaks) *n_peaks = (uint32_t)pk.size();
                       for (size_t i = 0; peaks && i < pk.size() && i < max_cells; i++) peaks[i] = pk[i];
                       return chain_step(b, sc, pk, cells, max_cells, &found, tc);
                     });
  if (n_cells) *n_cells = found;
  return rc;
}

}  // namespace lcs

using namespace lcs;

cudaError_t lcs_xcorr_plan::HostBatchBufs::ensure(const XcorrGeom& g, uint32_t chunk, size_t samp_bytes, bool host_iq, bool with_peaks) {
  const size_t n_pow = (size_t)chunk * 3 * LCS_N_FOLD;
  cudaError_t e = cudaSuccess;
  // only the base of a chunk needs 16-byte alignment (the correlator aligns absolute addresses), not the buffer stride
  if (host_iq) e = iq.ensure((size_t)chunk * g.n_cap * samp_bytes + 16);
  if (e == cudaSuccess) e = single.ensure(n_pow * g.n_f_stride);
  if (e == cudaSuccess) e = pow.ensure(n_pow);
  if (e == cudaSuccess) e = frq.ensure(n_pow);
  if (e == cudaSuccess) e = spi.ensure((size_t)chunk * LCS_N_FOLD);
  if (!with_peaks) return e;
  if (e == cudaSuccess) e = work.ensure(n_pow);
  if (e == cudaSuccess) e = peaks.ensure((size_t)chunk * SEARCH_MAX_PEAKS * sizeof(DevPeak));
  if (e == cudaSuccess) e = npeaks.ensure(chunk);
  // page-locked: with pageable memory cudaMemcpyAsync would block the host until the chunk's kernels are done and the
  // next chunk could not be queued behind it
  if (e == cudaSuccess) e = h_peaks.ensure((size_t)chunk * SEARCH_MAX_PEAKS * sizeof(DevPeak));
  if (e == cudaSuccess) e = h_npeaks.ensure(chunk);
  return e;
}

// Multi-channel searcher: one plan per channel (planset.cu builds them in one launch), all channels of a chunk in one
// correlator launch.
struct lcs_sweep {
  lcs_ctx* ctx = nullptr;
  uint32_t n_cap = 0;
  PlanSet ps;
  lcs_xcorr_plan::HostBatchBufs hb[lcs_ctx::N_STREAMS];
  DevBuf<uint32_t> d_ident;              // 0, 1, 2, ...: plan of buffer b is b
  std::vector<uint32_t> h_ident;
};

static lcs_status sweep_prepare(lcs_sweep* sw, const std::vector<PlanCfg>& cfgs, uint8_t arm, bool want_fp32) {
  lcs_ctx* ctx = sw->ctx;
  cudaStream_t st = ctx->streams[0];
  // the previous call's kernels on the other streams may still read the old plans
  for (int i = 1; i < lcs_ctx::N_STREAMS; i++) LCS_CUDA(ctx, cudaStreamSynchronize(ctx->streams[i]));
  lcs_status rc = planset_build(ctx, sw->ps, sw->n_cap, arm, cfgs, want_fp32, st);
  if (rc != LCS_OK) return rc;
  if (!want_fp32 && planset_resolve_kernel(sw->ps, LCS_KERNEL_AUTO, LCS_IQ_CU8) != LCS_KERNEL_TC) {
    rc = planset_build(ctx, sw->ps, sw->n_cap, arm, cfgs, true, st);       // this grid runs on the FP32 correlator
    if (rc != LCS_OK) return rc;
  }
  const uint32_t n = (uint32_t)cfgs.size();
  if (sw->h_ident.size() < n) {
    sw->h_ident.resize(n);
    for (uint32_t i = 0; i < n; i++) sw->h_ident[i] = i;
    LCS_CUDA(ctx, sw->d_ident.ensure(n));
    LCS_CUDA(ctx, cudaMemcpyAsync(sw->d_ident.p, sw->h_ident.data(), n * 4, cudaMemcpyHostToDevice, st));
  }
  return planset_finish(ctx, sw->ps, st);
}

extern "C" {

lcs_status lcs_xcorr_peaks_batch_host(lcs_xcorr_plan* p, const void* iq_host, int iq_format, uint32_t batch, lcs_cell* peaks,
                                      uint32_t max_peaks, uint32_t* n_peaks) {
  if (!p) return fail(nullptr, LCS_ERR_ARG, "xcorr_peaks_batch_host: null plan");
  if (!iq_host || !n_peaks || (!peaks && max_peaks)) return fail(p->ctx, LCS_ERR_ARG, "xcorr_peaks_batch_host: null pointer");
  return search_chunks(p->ctx, p->ps, p->kernel, p->hb, iq_host, iq_format, batch, std::min<uint32_t>(p->max_batch, BATCH_CHUNK), nullptr,
                       nullptr, [&](uint32_t b, const StageCall&, const std::vector<lcs_cell>& pk) {
                         n_peaks[b] = (uint32_t)pk.size();
                         for (size_t k = 0; k < pk.size() && k < max_peaks; k++) peaks[(size_t)b * max_peaks + k] = pk[k];
                         return LCS_OK;
                       });
}

lcs_status lcs_cell_search_batch_cu8(lcs_xcorr_plan* p, const uint8_t* iq_host, uint32_t batch, lcs_cell* cells, uint32_t max_cells,
                                     uint32_t* n_cells) {
  if (!p) return fail(nullptr, LCS_ERR_ARG, "cell_search_batch_cu8: null plan");
  if (!iq_host || !n_cells || (!cells && max_cells)) return fail(p->ctx, LCS_ERR_ARG, "cell_search_batch_cu8: null pointer");
  return search_chunks(p->ctx, p->ps, p->kernel, p->hb, iq_host, LCS_IQ_CU8, batch, std::min<uint32_t>(p->max_batch, BATCH_CHUNK), nullptr,
                       nullptr, [&](uint32_t b, const StageCall& sc, const std::vector<lcs_cell>& pk) {
                         return chain_step(b, sc, pk, cells, max_cells, n_cells);
                       });
}

lcs_status lcs_cell_search(lcs_ctx* ctx, const double* capbuf, uint32_t n_cap, const double* f_search_set, uint32_t n_f,
                           double fc_requested, double fc_programmed, double fs_programmed, lcs_cell* cells,
                           uint32_t max_cells, uint32_t* n_cells, lcs_cell* peaks, uint32_t* n_peaks) {
  if (!ctx || !capbuf || !f_search_set) return fail(ctx, LCS_ERR_ARG, "cell_search: null argument");
  return search_one(ctx, capbuf, LCS_IQ_C128, n_cap, f_search_set, n_f, fc_requested, fc_programmed, fs_programmed, cells, max_cells,
                    n_cells, peaks, n_peaks);
}

lcs_status lcs_cell_search_cu8(lcs_ctx* ctx, const uint8_t* capbuf_cu8, uint32_t n_cap, const double* f_search_set,
                               uint32_t n_f, double fc_requested, double fc_programmed, double fs_programmed,
                               lcs_cell* cells, uint32_t max_cells, uint32_t* n_cells, lcs_cell* peaks, uint32_t* n_peaks) {
  if (!ctx || !capbuf_cu8 || !f_search_set) return fail(ctx, LCS_ERR_ARG, "cell_search_cu8: null argument");
  return search_one(ctx, capbuf_cu8, LCS_IQ_CU8, n_cap, f_search_set, n_f, fc_requested, fc_programmed, fs_programmed, cells, max_cells,
                    n_cells, peaks, n_peaks);
}

// kalibrate (src/LTE-Tracker.cpp:565-741): an initial full search whose only purpose is the oscillator's residual offset.
// The frequency grid is centred on the offset implied by the current correction factor (:586-587); the strongest
// surviving cell after dedup (:703-716) gives freq_superfine and the residual correction factor (:719-726).  The
// reference loops until a cell is found (new data every iteration); here one buffer is examined and *n_cells = 0 reports
// "nothing found, try the next buffer".
lcs_status lcs_kalibrate_cu8(lcs_ctx* ctx, const uint8_t* capbuf_cu8, uint32_t n_cap, double fc_requested, double fc_programmed,
                             double fs_programmed, double ppm, double correction, lcs_cell* best, double* correction_residual,
                             uint32_t* n_cells) {
  if (!ctx || !capbuf_cu8 || !best || !n_cells) return fail(ctx, LCS_ERR_ARG, "kalibrate_cu8: null argument");
  std::vector<double> f = f_search_set_for(fc_requested, ppm);                          // :586
  for (double& v : f) v = (fc_requested * correction - fc_requested) + v;               // :587
  std::vector<lcs_cell> cells(64);
  uint32_t found = 0;
  lcs_status rc = search_one(ctx, capbuf_cu8, LCS_IQ_CU8, n_cap, f.data(), (uint32_t)f.size(), fc_requested, fc_programmed,
                             fs_programmed, cells.data(), (uint32_t)cells.size(), &found, nullptr, nullptr);
  if (rc != LCS_OK) return rc;
  std::vector<lcs_cell> fin;
  dedup(cells.data(), std::min<uint32_t>(found, (uint32_t)cells.size()), fin);           // :703-705
  *n_cells = (uint32_t)fin.size();
  lcs_cell_init(best);
  if (fin.empty()) return LCS_OK;
  double bp = -INFINITY;
  for (const lcs_cell& c : fin)                                                         // :709-716
    if (c.pss_pow > bp) { bp = c.pss_pow; *best = c; }
  if (correction_residual) {
    const double true_location = fc_requested;                                          // :720
    const double crystal_freq_actual = fc_programmed - best->freq_superfine;            // :722
    *correction_residual = (true_location / fc_requested * fc_programmed) / crystal_freq_actual;   // :724
  }
  return LCS_OK;
}

// One cycle of the tracker's searcher thread (src/searcher_thread.cpp:95-232) on a capture buffer delivered by the framer.
lcs_status lcs_tracker_search_cu8(lcs_ctx* ctx, const uint8_t* capbuf_cu8, uint32_t n_cap, double frequency_offset,
                                  double fc_requested, double fc_programmed, double fs_programmed, double late,
                                  const int32_t* tracked_n_id_cell, uint32_t n_tracked, lcs_cell* cells, double* frame_timing,
                                  uint32_t max_cells, uint32_t* n_cells) {
  if (!ctx || !capbuf_cu8 || !n_cells || (n_tracked && !tracked_n_id_cell) || (max_cells && (!cells || !frame_timing)))
    return fail(ctx, LCS_ERR_ARG, "tracker_search_cu8: null argument");
  const double f_search_set[1] = {frequency_offset};                                   // searcher_thread.cpp:96-98
  const TrackerCycle tc{tracked_n_id_cell, n_tracked, late, frame_timing};
  return search_one(ctx, capbuf_cu8, LCS_IQ_CU8, n_cap, f_search_set, 1, fc_requested, fc_programmed, fs_programmed, cells, max_cells,
                    n_cells, nullptr, nullptr, &tc);
}

// ---- multi-channel searcher -------------------------------------------------------------------------------------------
lcs_status lcs_sweep_create(lcs_ctx* ctx, uint32_t n_cap, lcs_sweep** out) {
  if (!ctx || !out) return fail(ctx, LCS_ERR_ARG, "sweep_create: null argument");
  if (n_cap < 136 + 100 + LCS_N_FOLD || n_cap < 273 + LCS_N_FOLD)
    return fail(ctx, LCS_ERR_ARG, "sweep_create: capture buffer shorter than one 5 ms half frame + margins");
  lcs_sweep* sw = new lcs_sweep();
  sw->ctx = ctx;
  sw->n_cap = n_cap;
  *out = sw;
  return LCS_OK;
}

void lcs_sweep_destroy(lcs_sweep* sw) {
  if (!sw) return;
  cudaSetDevice(sw->ctx->device);
  cudaDeviceSynchronize();
  delete sw;
}

}  // extern "C"

// The per-centre-frequency loop of CellSearch (src/CellSearch.cpp:465-558) for n_ch capture buffers at once (host or
// device memory).
static lcs_status sweep_search(lcs_sweep* sw, const uint8_t* iq, bool device_input, uint32_t n_ch, const double* fc_requested,
                               const double* fc_programmed, double fs_programmed, const double* f_search_set, uint32_t n_f,
                               lcs_cell* cells, uint32_t max_cells, uint32_t* n_cells) {
  lcs_ctx* ctx = sw->ctx;
  if (n_ch == 0) return LCS_OK;
  std::vector<PlanCfg> cfgs(n_ch);
  for (uint32_t c = 0; c < n_ch; c++) {
    cfgs[c].fc_req = fc_requested[c];
    cfgs[c].fc_prog = fc_programmed ? fc_programmed[c] : fc_requested[c];
    cfgs[c].fs_prog = fs_programmed;
    cfgs[c].f.assign(f_search_set, f_search_set + n_f);
  }
  const uint8_t DS_COMB_ARM = 2;        // CellSearch.cpp:484
  lcs_status rc = sweep_prepare(sw, cfgs, DS_COMB_ARM, false);
  if (rc != LCS_OK) return rc;
  // chunks of 64 channels: 128 units of 38+ tiles keep every persistent correlator CTA busy for >30 tiles
  return search_chunks(ctx, sw->ps, LCS_KERNEL_AUTO, sw->hb, iq, LCS_IQ_CU8, n_ch, BATCH_CHUNK, sw->d_ident.p, sw->h_ident.data(),
                       [&](uint32_t b, const StageCall& sc, const std::vector<lcs_cell>& pk) {
                         return chain_step(b, sc, pk, cells, max_cells, n_cells);
                       },
                       device_input);
}

extern "C" {

lcs_status lcs_sweep_search_cu8(lcs_sweep* sw, const uint8_t* iq_host, uint32_t n_ch, const double* fc_requested,
                                const double* fc_programmed, double fs_programmed, const double* f_search_set, uint32_t n_f,
                                lcs_cell* cells, uint32_t max_cells, uint32_t* n_cells) {
  if (!sw) return fail(nullptr, LCS_ERR_ARG, "sweep_search_cu8: null handle");
  if (!iq_host || !fc_requested || !f_search_set || !n_cells || (!cells && max_cells)) return fail(sw->ctx, LCS_ERR_ARG, "sweep_search_cu8: null pointer");
  return sweep_search(sw, iq_host, false, n_ch, fc_requested, fc_programmed, fs_programmed, f_search_set, n_f, cells, max_cells, n_cells);
}

lcs_status lcs_sweep_search_cu8_device(lcs_sweep* sw, const uint8_t* d_iq, uint32_t n_ch, const double* fc_requested,
                                       const double* fc_programmed, double fs_programmed, const double* f_search_set, uint32_t n_f,
                                       lcs_cell* cells, uint32_t max_cells, uint32_t* n_cells) {
  if (!sw) return fail(nullptr, LCS_ERR_ARG, "sweep_search_cu8_device: null handle");
  if (!d_iq || !fc_requested || !f_search_set || !n_cells || (!cells && max_cells))
    return fail(sw->ctx, LCS_ERR_ARG, "sweep_search_cu8_device: null pointer");
  // the tensor-core correlator reads the buffers with 16-byte bulk copies (64-buffer chunks keep that alignment)
  if (((uintptr_t)d_iq & 15) != 0) return fail(sw->ctx, LCS_ERR_ARG, "sweep_search_cu8_device: d_iq must be 16-byte aligned");
  return sweep_search(sw, d_iq, true, n_ch, fc_requested, fc_programmed, fs_programmed, f_search_set, n_f, cells, max_cells, n_cells);
}

// One searcher cycle (src/searcher_thread.cpp:95-232) for n_ch tracked channels at once: every channel is searched at its
// own single frequency offset.
lcs_status lcs_sweep_track_cu8(lcs_sweep* sw, const uint8_t* iq_host, uint32_t n_ch, const double* frequency_offset,
                               const double* fc_requested, const double* fc_programmed, double fs_programmed, const double* late,
                               const int32_t* tracked_n_id_cell, const uint32_t* n_tracked, uint32_t tracked_stride, lcs_cell* cells,
                               double* frame_timing, uint32_t max_cells, uint32_t* n_cells) {
  if (!sw) return fail(nullptr, LCS_ERR_ARG, "sweep_track_cu8: null handle");
  lcs_ctx* ctx = sw->ctx;
  if (!iq_host || !frequency_offset || !fc_requested || !n_cells || (max_cells && (!cells || !frame_timing)) ||
      (n_tracked && !tracked_n_id_cell))
    return fail(ctx, LCS_ERR_ARG, "sweep_track_cu8: null pointer");
  if (n_ch == 0) return LCS_OK;
  std::vector<PlanCfg> cfgs(n_ch);
  for (uint32_t c = 0; c < n_ch; c++) {
    cfgs[c].fc_req = fc_requested[c];
    cfgs[c].fc_prog = fc_programmed ? fc_programmed[c] : fc_requested[c];
    cfgs[c].fs_prog = fs_programmed;
    cfgs[c].f.assign(1, frequency_offset[c]);                                          // searcher_thread.cpp:96-98
  }
  lcs_status rc = sweep_prepare(sw, cfgs, 2, true);
  if (rc != LCS_OK) return rc;
  return search_chunks(ctx, sw->ps, LCS_KERNEL_AUTO, sw->hb, iq_host, LCS_IQ_CU8, n_ch, BATCH_CHUNK, sw->d_ident.p, sw->h_ident.data(),
                       [&](uint32_t b, const StageCall& sc, const std::vector<lcs_cell>& pk) {
                         const TrackerCycle tc{n_tracked ? tracked_n_id_cell + (size_t)b * tracked_stride : nullptr,
                                               n_tracked ? n_tracked[b] : 0, late ? late[b] : 0.0, frame_timing};
                         return chain_step(b, sc, pk, cells, max_cells, n_cells, &tc);
                       });
}

}  // extern "C"
