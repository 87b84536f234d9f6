// carrier_grid.cuh - the full-bandwidth OFDM grid of found cells, from the wideband recording they were found in: the grid
// Y[t][c] of include/lcs_carrier.h, built for the CRS symbols only, and the one host path of every module on it:
// liblcs_carrier.so (carrier.cu), liblcs_cir.so (cir.cu), liblcs_pcfich.so (pcfich.cu), liblcs_pdcch.so (pdcch.cu) and
// liblcs_sib1.so (sib1.cu).
// Each module's handle is a GridModule, and its lcs_X_cells is grid_cells with the module's planner, slices and kernels.
#pragma once
#include <cmath>
#include <limits>
#include <new>
#include <string>
#include <vector>

#include "carrier_plan.hpp"
#include "chain_gpu.hpp"
#include "fft_tile.cuh"
#include "iq_format.cuh"

namespace lcs {
namespace carrier {

using namespace fft;
constexpr int N_SLOT_TAB = 20;       // CRS tables repeat every frame: [20 slots][3 symbols {0, 1, n_symb-3}]
constexpr int MAX_RB = 100;

struct Win {                         // one DFT window
  long long q;                       // first sample in the recording
  double late;                       // q - D loc_t
  unsigned long long out;            // its grid row (float2 index)
  int cell;                          // in the chunk
  int pad;
};
struct GridCell {
  long long step;                    // (delta mod fs_in): the mixer phase advances by step / fs_in cycles per sample
  double kpi;                        // kappa / pi
  int R;
  int pad;
};

struct GridParams {
  const unsigned char* in;           // the recording from sample `base` on
  long long base;
  long long fs;
  const Win* win;
  const GridCell* cell;
  int n_win;
  int lg;                            // log2 N
  float scale;                       // sqrt(128) / N
  const float2* tw;                  // [N] exp(-j2pi m/N)
  float2* grid;
};

template <int FMT>
__global__ void __launch_bounds__(THREADS) carrier_grid_kernel(GridParams P) {
  __shared__ float2 a[TILE];
  __shared__ Win sw[TILE / 256];
  __shared__ GridCell sc[TILE / 256];
  const int lg = P.lg, N = 1 << lg, per = TILE >> lg;
  const int w0 = blockIdx.x * per;
  if (threadIdx.x < per && w0 + (int)threadIdx.x < P.n_win) {
    sw[threadIdx.x] = P.win[w0 + threadIdx.x];
    sc[threadIdx.x] = P.cell[sw[threadIdx.x].cell];
  }
  __syncthreads();
  for (int e = threadIdx.x; e < TILE; e += THREADS) {
    const int b = e >> lg, n = e & (N - 1);
    float2 v = make_float2(0.f, 0.f);
    if (w0 + b < P.n_win) {
      const long long m = sw[b].q + n;
      const long long p = ((m % P.fs) * sc[b].step) % P.fs;         // exact mixer phase, in cycles * fs
      double sn, cs;
      sincospi(sc[b].kpi * (double)m - 2.0 * (double)p / (double)P.fs, &sn, &cs);
      v = cmul(load_iq<FMT>(P.in, (size_t)(m - P.base)), make_float2((float)cs, (float)sn));
    }
    a[swz((b << lg) + bitrev(n, lg))] = v;
  }
  __syncthreads();
  fft_tile(a, lg, P.tw, lg);
  for (int e = threadIdx.x; e < TILE; e += THREADS) {
    const int b = e >> lg, c = e & (N - 1);
    if (w0 + b >= P.n_win) continue;
    const int R = sc[b].R;
    if (c >= 12 * R) continue;
    const int k = c < 6 * R ? c - 6 * R : c - 6 * R + 1;              // subcarrier, DC skipped
    const float2 x = a[swz((b << lg) + (k & (N - 1)))];
    double sn, cs;
    sincospi(-2.0 * sw[b].late * (double)k / (double)N, &sn, &cs);
    P.grid[sw[b].out + c] = cmul(make_float2(x.x * P.scale, x.y * P.scale), make_float2((float)cs, (float)sn));
  }
}

// ---- host side ------------------------------------------------------------------------------------------------------------
// The arguments of a call other than its cells, against lcs_carrier.h: "" when they are valid (D then set), else why not.
inline std::string check_call(const void* iq, int iq_format, int on_device, uint64_t n_in, double fs_in, double fc_in,
                              uint32_t n_cells, const lcs_cell* cells, const void* out, double fs_programmed, int& D) {
  if (!iq || (n_cells && (!cells || !out))) return "null pointer";
  if (!StreamFormats::has(iq_format)) return "iq_format must be LCS_IQ_CI16, CS8, CU8 or CF32";
  if (on_device && ((uintptr_t)iq & 15)) return "device iq must be 16-byte aligned";
  const char* rate = "fs_in must be D * 1.92 MHz with D in {2, 4, 8, 16, 32}";
  if (!(std::isfinite(fs_in) && fs_in > 0 && fs_in < 100e6)) return rate;
  D = (int)std::lround(fs_in / 1.92e6);
  if (!((D == 2 || D == 4 || D == 8 || D == 16 || D == 32) && std::fabs(fs_in - D * 1.92e6) <= 1e-6)) return rate;
  if (!n_in || n_in / D >= (1ull << 31)) return "n_in must be positive and below 2^31 D";
  if (!std::isfinite(fc_in)) return "fc_in must be finite";
  if (!(std::isfinite(fs_programmed) && fs_programmed > 0)) return "fs_programmed must be finite and positive";
  return "";
}

// What a module keeps between calls to build grids: the recording's span (host input), the staged tables of a chunk, the
// FFT twiddles of the last N used and one chunk's grids.
struct GridScratch {
  DevBuf<unsigned char> d_iq;
  Staging up;
  DevBuf<float2> d_tw;                     // [N] twiddles of the last N used
  uint32_t tw_n = 0;
  DevBuf<float2> d_grid;

  // The recording as the grid kernel reads it (uploading the span [lo, hi) of host input on st) and the twiddles of N.
  cudaError_t prepare(const void* iq, size_t esz, int on_device, long long lo, long long hi, int N, cudaStream_t st,
                      const unsigned char** d_in, long long* base) {
    *d_in = static_cast<const unsigned char*>(iq);
    *base = 0;
    if (!on_device) {
      cudaError_t e = d_iq.ensure((size_t)(hi - lo) * esz);
      if (e == cudaSuccess)
        e = cudaMemcpyAsync(d_iq.p, static_cast<const unsigned char*>(iq) + (size_t)lo * esz, (size_t)(hi - lo) * esz,
                            cudaMemcpyHostToDevice, st);
      if (e != cudaSuccess) return e;
      *d_in = d_iq.p;
      *base = lo;
    }
    if (tw_n != (uint32_t)N) {
      std::vector<float2> tw(N);
      for (int n = 0; n < N; n++) {
        const double ang = -2 * M_PI * (double)n / (double)N;
        tw[n] = make_float2((float)std::cos(ang), (float)std::sin(ang));
      }
      tw_n = 0;
      cudaError_t e = d_tw.ensure(N);
      if (e == cudaSuccess) e = cudaMemcpy(d_tw.p, tw.data(), N * sizeof(float2), cudaMemcpyHostToDevice);
      if (e != cudaSuccess) return e;
      tw_n = N;
    }
    return cudaSuccess;
  }
};

// One chunk's tables in a GridScratch's staging: the windows and cells carrier_grid_kernel reads, and the CRS of every
// cell, rs [cell][20][3][2 MAX_RB] (the signs of r = (s.x + j s.y) / sqrt(2)) and shift [cell][20][3][4].  off[i] is
// cell i's grid [N_SLOT][nw][12 R] (float2 index) and n_grid all the chunk's grids.
struct ChunkTables {
  Win* win = nullptr;
  GridCell* gc = nullptr;
  char2* rs = nullptr;
  unsigned char* shift = nullptr;
  size_t n_win = 0, n_grid = 0;
  std::vector<unsigned long long> off;
};

// Resets g.up with room for these tables of cells ch[0 .. nc) and `extra` more bytes (the caller's own slices, 16 bytes of
// alignment each included), fills them, and makes room for the chunk's grids; the caller takes its slices and uploads.
inline cudaError_t stage_chunk(GridScratch& g, const CellPlan* ch, uint32_t nc, size_t extra, ChunkTables& t) {
  t.n_win = t.n_grid = 0;
  for (uint32_t i = 0; i < nc; i++) t.n_win += ch[i].q.size();
  const size_t n_tab = (size_t)nc * N_SLOT_TAB * 3;
  cudaError_t e = g.up.reset(t.n_win * sizeof(Win) + nc * sizeof(GridCell) + n_tab * (2 * MAX_RB * sizeof(char2) + 4) +
                             4 * 16 + extra);
  if (e != cudaSuccess) return e;
  t.win = g.up.take<Win>(t.n_win);
  t.gc = g.up.take<GridCell>(nc);
  t.rs = g.up.take<char2>(n_tab * 2 * MAX_RB);
  t.shift = g.up.take<unsigned char>(n_tab * 4);
  t.off.assign(nc, 0);
  size_t w = 0;
  for (uint32_t i = 0; i < nc; i++) {
    const CellPlan& c = ch[i];
    const size_t W = 12 * (size_t)c.R;
    t.gc[i] = GridCell{c.step, c.kpi, c.R, 0};
    t.off[i] = t.n_grid;
    for (size_t j = 0; j < c.q.size(); j++, w++) t.win[w] = Win{c.q[j], c.late[j], t.n_grid + j * W, (int)i, 0};
    t.n_grid += c.q.size() * W;
    const RsDl rs(c.n_id_cell, c.cp_type, c.R);
    for (int sl = 0; sl < N_SLOT_TAB; sl++)
      for (int s3 = 0; s3 < 3; s3++) {
        const int sym = s3 == 2 ? rs.n_symb - 3 : s3;
        const cd* r = rs.get(sl, sym);
        char2* tr = t.rs + ((i * N_SLOT_TAB + sl) * 3 + s3) * 2 * MAX_RB;
        for (int m = 0; m < 2 * MAX_RB; m++)
          tr[m] = m < 2 * c.R ? make_char2(r[m].real() > 0 ? 1 : -1, r[m].imag() > 0 ? 1 : -1) : make_char2(0, 0);
        for (int p = 0; p < 4; p++) t.shift[((i * N_SLOT_TAB + sl) * 3 + s3) * 4 + p] = (unsigned char)rs.shift(sl, sym, p);
      }
  }
  return g.d_grid.ensure(t.n_grid);
}

// carrier_grid_kernel on a staged chunk (one launch on st); false when no kernel takes iq_format.
inline bool launch_grid(const GridScratch& g, const ChunkTables& t, int iq_format, const unsigned char* d_in,
                        long long base, double fs_in, int D, cudaStream_t st) {
  const int N = 128 * D;
  GridParams P;
  P.in = d_in;
  P.base = base;
  P.fs = std::llround(fs_in);
  P.win = g.up.dev(t.win);
  P.cell = g.up.dev(t.gc);
  P.n_win = (int)t.n_win;
  P.lg = 7 + __builtin_ctz(D);
  P.scale = (float)(std::sqrt(128.0) / N);
  P.tw = g.d_tw.p;
  P.grid = g.d_grid.p;
  const int per = TILE / N;
  return StreamFormats::dispatch(iq_format, [&](auto FMT) {
           carrier_grid_kernel<FMT><<<(unsigned)((t.n_win + per - 1) / per), THREADS, 0, st>>>(P);
         }) == LCS_OK;
}

// ---- the host path of every module on the grid ------------------------------------------------------------------------
// What a module's handle keeps between calls; each module's opaque handle type derives from it.
template <class Meas>
struct GridModule {
  lcs_ctx* ctx = nullptr;
  GridScratch g;                     // the recording's span, the staged tables and one chunk's grids
  DevBuf<Meas> d_out;                // one chunk's records
  KernelClock clock;                 // the launches of each chunk
};

// lcs_X_create, lcs_X_destroy and lcs_X_timing_read of a module's handle type H; fn is the C function's name.
template <class H>
lcs_status grid_create(lcs_ctx* ctx, H** out, const char* fn) {
  if (!ctx || !out) return fail(ctx, LCS_ERR_ARG, std::string(fn) + ": null argument");
  H* h = new (std::nothrow) H();
  if (!h) return fail(ctx, LCS_ERR_STATE, std::string(fn) + ": out of memory");
  h->ctx = ctx;
  *out = h;
  return LCS_OK;
}

template <class H>
void grid_destroy(H* h) {
  if (!h) return;
  cudaSetDevice(h->ctx->device);     // its buffers and events belong to the context's device
  delete h;
}

template <class H>
lcs_status grid_timing_read(H* h, double* kernel_ms, uint64_t* launches, const char* fn) {
  if (!h) return LCS_ERR_ARG;
  if (!kernel_ms || !launches) return fail(h->ctx, LCS_ERR_ARG, std::string(fn) + ": null pointer");
  LCS_CUDA(h->ctx, h->clock.read(kernel_ms, launches));
  return LCS_OK;
}

// One chunk of a call, as a module's fill and launch see it.
struct GridChunk {
  ChunkTables t;                     // its staged tables and grids
  const CellPlan* plan = nullptr;    // its cells' plans
  const lcs_cell* cell = nullptr;    // and its cells
  uint32_t n = 0;
  int D = 0;
  cudaStream_t st = nullptr;
};

struct NoHostStep {
  template <class Meas> void operator()(Meas&, const CellPlan&) const {}
};

// lcs_X_cells of a module (fn its name, `chunk` cells per chunk, `launches` kernels per chunk).  The call's arguments are
// checked, and every cell planned by plan (plan_cell's signature) before any device work; the span of the recording its
// windows cover is uploaded.  Then each chunk, on the context's stream 0, is staged with bytes(n) more bytes for the
// module's slices, which fill(chunk) takes and fills (readying the module's own device scratch too); it is uploaded, its
// records zeroed, and carrier_grid_kernel and launch(chunk) run between the clock's events; its records are copied out,
// the stream synchronised and done(record, plan) run on each.
template <class H, class Meas, class Plan, class Bytes, class Fill, class Launch, class Done = NoHostStep>
lcs_status grid_cells(H* h, const char* fn, uint32_t chunk, uint64_t launches, const void* iq, int iq_format,
                      int on_device, uint64_t n_in, double fs_in, double fc_in, const lcs_cell* cells, uint32_t n_cells,
                      double fs_programmed, Meas* out, Plan plan, Bytes bytes, Fill fill, Launch launch,
                      Done done = Done()) {
  if (!h) return LCS_ERR_ARG;
  lcs_ctx* ctx = h->ctx;
  const std::string pre = std::string(fn) + ": ";
  int D = 0;
  const std::string bad = check_call(iq, iq_format, on_device, n_in, fs_in, fc_in, n_cells, cells, out, fs_programmed, D);
  if (!bad.empty()) return fail(ctx, LCS_ERR_ARG, pre + bad);
  if (!n_cells) return LCS_OK;
  LCS_CUDA(ctx, cudaSetDevice(ctx->device));
  std::vector<CellPlan> ch(n_cells);
  long long lo = std::numeric_limits<long long>::max(), hi = 0;
  for (uint32_t i = 0; i < n_cells; i++) {
    const std::string why = plan(cells[i], n_in, D, fs_in, fc_in, fs_programmed, ch[i]);
    if (!why.empty()) return fail(ctx, LCS_ERR_ARG, pre + "cell " + std::to_string(i) + ": " + why);
    lo = std::min(lo, ch[i].q.front());
    hi = std::max(hi, ch[i].q.back() + 128ll * D);
  }
  GridChunk c;
  c.D = D;
  c.st = ctx->streams[0];
  const unsigned char* d_in;
  long long base;
  LCS_CUDA(ctx, h->g.prepare(iq, sample_bytes(iq_format), on_device, lo, hi, 128 * D, c.st, &d_in, &base));
  LCS_CUDA(ctx, h->d_out.ensure(std::min(n_cells, chunk)));
  for (uint32_t c0 = 0; c0 < n_cells; c0 += chunk) {
    c.n = std::min(chunk, n_cells - c0);
    c.plan = &ch[c0];
    c.cell = cells + c0;
    LCS_CUDA(ctx, stage_chunk(h->g, c.plan, c.n, bytes(c.n), c.t));
    LCS_CUDA(ctx, fill(c));
    LCS_CUDA(ctx, h->g.up.upload(c.st));
    LCS_CUDA(ctx, cudaMemsetAsync(h->d_out.p, 0, c.n * sizeof(Meas), c.st));   // the records' padding too
    LCS_CUDA(ctx, h->clock.begin(c.st));
    if (!launch_grid(h->g, c.t, iq_format, d_in, base, fs_in, D, c.st))
      return fail(ctx, LCS_ERR_ARG, pre + "no grid kernel for this iq_format");
    launch(c);
    ctx->launches += launches;
    LCS_CUDA(ctx, cudaGetLastError());
    LCS_CUDA(ctx, h->clock.end(c.st, launches));
    LCS_CUDA(ctx, cudaMemcpyAsync(out + c0, h->d_out.p, c.n * sizeof(Meas), cudaMemcpyDeviceToHost, c.st));
    LCS_CUDA(ctx, cudaStreamSynchronize(c.st));
    for (uint32_t i = 0; i < c.n; i++) done(out[c0 + i], ch[c0 + i]);
  }
  return LCS_OK;
}

}  // namespace carrier
}  // namespace lcs
