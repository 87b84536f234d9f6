// carrier.cu - RSRP, RSRQ and SINR of found cells over all their resource blocks, from the wideband recording they were
// found in (DESIGN.md section 4.10; contract in include/lcs_carrier.h).  Built into liblcs_carrier.so.
//
// A call is cut into chunks of LCS_CARRIER_CHUNK cells; each chunk makes two launches on the context's stream:
//   1. carrier_grid_kernel: one N-point window (N = 128 D) per OFDM symbol that carries CRS, 4096 / N windows per CTA.
//      Each sample is staged with load_iq, rotated once by the cell's mixer (the channelizer's exact integer phase plus
//      the FOC phase, in FP64), the windows go through the FP32 FFT of fft_tile.cuh, and the 12 R used bins, scaled and
//      turned by the window's lateness ramp, are written as float2.
//   2. carrier_meas_kernel: one CTA per cell.  Each (port, CRS index) has its pairs summed over the grid in slot order by
//      one thread, and threads sum the RSSI of the columns in slot order; each RB then adds its two CRS indices
//      (and twelve columns) in order, and thread 0 adds the RBs in order.  All sums are FP64, so a cell's record is the
//      same on every run and independent of the other cells of the call.
// Each cell is checked and its windows laid out on the host first (plan_cell, carrier_plan.cpp, from tfg_geometry); the
// CRS signs and shifts come from RsDl (chain_host.cpp).
#include <cmath>
#include <limits>
#include <new>
#include <string>
#include <vector>

#include "../../include/lcs_carrier.h"
#include "carrier_plan.hpp"
#include "chain_gpu.hpp"
#include "fft_tile.cuh"
#include "iq_format.cuh"

namespace lcs {
namespace carrier {

using namespace fft;
constexpr int N_SLOT_TAB = 20;       // CRS tables repeat every frame: [20 slots][3 symbols {0, 1, n_symb-3}]
constexpr int MAX_RB = 100;
constexpr int MEAS_THREADS = 512;
constexpr uint32_t CHUNK = LCS_CARRIER_CHUNK;

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
struct MeasCell {
  unsigned long long off;            // the cell's grid [N_SLOT][nw][12 R]
  int R, n_ports, nw, pad;           // nw: windows per slot (2, or 3 for four ports)
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

// rs_all [cell][20][3][2 MAX_RB] holds the signs of the CRS r = (s.x + j s.y) / sqrt(2); shift_all [cell][20][3][4].
__global__ void __launch_bounds__(MEAS_THREADS) carrier_meas_kernel(const float2* __restrict__ grid,
                                                                    const char2* __restrict__ rs_all,
                                                                    const unsigned char* __restrict__ shift_all,
                                                                    const MeasCell* __restrict__ par,
                                                                    lcs_carrier_meas* __restrict__ out) {
  __shared__ double pm[4][2 * MAX_RB][3];      // per (port, CRS index): C (re, im) and T sums
  __shared__ double col[12 * MAX_RB];          // per column: the RSSI sum
  __shared__ double rbs[4][MAX_RB][3];         // per (port, RB)
  __shared__ double rbr[MAX_RB];
  const int tid = threadIdx.x, cell = blockIdx.x;
  const MeasCell mc = par[cell];
  const int R = mc.R, n_ports = mc.n_ports, nw = mc.nw, W = 12 * R;
  const float2* G = grid + mc.off;
  const char2* rs = rs_all + (size_t)cell * N_SLOT_TAB * 3 * 2 * MAX_RB;
  const unsigned char* shift = shift_all + (size_t)cell * N_SLOT_TAB * 3 * 4;
  for (int j = tid; j < n_ports * 2 * R; j += MEAS_THREADS) {
    const int p = j / (2 * R), m = j % (2 * R);
    const int nsp = p < 2 ? 2 : 1;                 // CRS symbols of the port per slot
    double cre = 0, cim = 0, T = 0;
    for (int t = 0; t < N_SLOT - 2; t++)
      for (int si = 0; si < nsp; si++) {
        const int s3 = p < 2 ? (si ? 2 : 0) : 1;
        const int k = s3 == 0 ? 0 : (s3 == 2 ? nw - 1 : 1);
        const int ta = t % N_SLOT_TAB, tb = (t + 2) % N_SLOT_TAB;
        const float2 ya = G[(size_t)(t * nw + k) * W + 6 * m + shift[(ta * 3 + s3) * 4 + p]];
        const float2 yb = G[(size_t)((t + 2) * nw + k) * W + 6 * m + shift[(tb * 3 + s3) * 4 + p]];
        const char2 ra = rs[(ta * 3 + s3) * 2 * MAX_RB + m], rb = rs[(tb * 3 + s3) * 2 * MAX_RB + m];
        // sqrt(2) y conj(r); the factor 1/2 of both products is applied to the sums
        const double hax = (double)ya.x * ra.x + (double)ya.y * ra.y, hay = (double)ya.y * ra.x - (double)ya.x * ra.y;
        const double hbx = (double)yb.x * rb.x + (double)yb.y * rb.y, hby = (double)yb.y * rb.x - (double)yb.x * rb.y;
        cre += hax * hbx + hay * hby;               // h_a conj(h_b)
        cim += hay * hbx - hax * hby;
        T += (hax * hax + hay * hay) + (hbx * hbx + hby * hby);
      }
    pm[p][m][0] = cre;
    pm[p][m][1] = cim;
    pm[p][m][2] = T;
  }
  for (int c = tid; c < W; c += MEAS_THREADS) {    // the port-0 CRS symbols {0, n_symb-3} of every slot
    double s = 0;
    for (int t = 0; t < N_SLOT; t++)
      for (int k = 0; k < nw; k += nw - 1) {
        const float2 y = G[(size_t)(t * nw + k) * W + c];
        s += (double)y.x * y.x + (double)y.y * y.y;
      }
    col[c] = s;
  }
  __syncthreads();
  const double nan = __longlong_as_double(0x7ff8000000000000ll), inf = __longlong_as_double(0x7ff0000000000000ll);
  lcs_carrier_meas* o = out + cell;
  if (tid < MAX_RB) {
    const int b = tid;
    for (int p = 0; p < 4; p++) {
      if (p < n_ports && b < R) {
        const int n = 2 * (p < 2 ? 2 : 1) * (N_SLOT - 2);   // pairs per RB
        for (int v = 0; v < 3; v++) rbs[p][b][v] = pm[p][2 * b][v] + pm[p][2 * b + 1][v];
        const double S = hypot(0.5 * rbs[p][b][0] / n, 0.5 * rbs[p][b][1] / n), Tm = 0.5 * rbs[p][b][2] / (2.0 * n);
        o->rb_rsrp[p][b] = S / 128;
        o->rb_noise[p][b] = (Tm - S) / 128;
      } else {
        o->rb_rsrp[p][b] = o->rb_noise[p][b] = nan;
      }
    }
    if (b < R) {
      double s = col[12 * b];
      for (int k = 1; k < 12; k++) s += col[12 * b + k];
      rbr[b] = s;
      o->rb_rssi[b] = s / (2.0 * N_SLOT) / 128;
    } else {
      o->rb_rssi[b] = nan;
    }
  }
  __syncthreads();
  if (tid) return;
  for (int p = 0; p < 4; p++) {
    if (p < n_ports) {
      double s[3] = {rbs[p][0][0], rbs[p][0][1], rbs[p][0][2]};
      for (int b = 1; b < R; b++)
        for (int v = 0; v < 3; v++) s[v] += rbs[p][b][v];
      const int n = R * 2 * (p < 2 ? 2 : 1) * (N_SLOT - 2);   // 480 R or 240 R
      const double S = hypot(0.5 * s[0] / n, 0.5 * s[1] / n), Tm = 0.5 * s[2] / (2.0 * n), Nn = Tm - S;
      o->rsrp[p] = S / 128;
      o->noise[p] = Nn / 128;
      o->sinr[p] = Nn > 0 ? S / Nn : inf;
      o->n_pairs[p] = (uint32_t)n;
    } else {
      o->rsrp[p] = o->noise[p] = o->sinr[p] = nan;
      o->n_pairs[p] = 0;
    }
  }
  double r = rbr[0];
  for (int b = 1; b < R; b++) r += rbr[b];
  o->rssi = r / (2.0 * N_SLOT) / 128;
  o->rsrq = R * o->rsrp[0] / o->rssi;
  o->n_rb = (uint32_t)R;
}

}  // namespace carrier
}  // namespace lcs

using namespace lcs;
using namespace lcs::carrier;

struct lcs_carrier {
  lcs_ctx* ctx = nullptr;
  DevBuf<unsigned char> d_iq;              // host input: the span of the recording the cells' windows cover
  Staging up;                              // per chunk: windows, cell parameters, CRS signs and shifts
  DevBuf<float2> d_tw;                     // [N] twiddles of the last N used
  uint32_t tw_n = 0;
  DevBuf<float2> d_grid;                   // one chunk's grids
  DevBuf<lcs_carrier_meas> d_out;
  KernelClock clock;                       // both launches of each chunk
};

namespace {

lcs_status cfail(const lcs_carrier* h, const std::string& msg) {
  return fail(h->ctx, LCS_ERR_ARG, "lcs_carrier_cells: " + msg);
}

}  // namespace

extern "C" {

lcs_status lcs_carrier_create(lcs_ctx* ctx, lcs_carrier** out) {
  if (!ctx || !out) return fail(ctx, LCS_ERR_ARG, "lcs_carrier_create: null argument");
  lcs_carrier* h = new (std::nothrow) lcs_carrier();
  if (!h) return fail(ctx, LCS_ERR_STATE, "lcs_carrier_create: out of memory");
  h->ctx = ctx;
  *out = h;
  return LCS_OK;
}

void lcs_carrier_destroy(lcs_carrier* h) {
  if (!h) return;
  cudaSetDevice(h->ctx->device);             // its buffers and events belong to the context's device
  delete h;
}

lcs_status lcs_carrier_cells(lcs_carrier* h, const void* iq, int iq_format, int on_device, uint64_t n_in, double fs_in,
                             double fc_in, const lcs_cell* cells, uint32_t n_cells, double fs_programmed,
                             lcs_carrier_meas* out) {
  if (!h) return LCS_ERR_ARG;
  if (!iq || (n_cells && (!cells || !out))) return cfail(h, "null pointer");
  if (!StreamFormats::has(iq_format)) return cfail(h, "iq_format must be LCS_IQ_CI16, CS8, CU8 or CF32");
  const size_t esz = sample_bytes(iq_format);
  if (on_device && ((uintptr_t)iq & 15)) return cfail(h, "device iq must be 16-byte aligned");
  if (!(std::isfinite(fs_in) && fs_in > 0 && fs_in < 100e6))
    return cfail(h, "fs_in must be D * 1.92 MHz with D in {2, 4, 8, 16, 32}");
  const int D = (int)std::lround(fs_in / 1.92e6);
  if (!((D == 2 || D == 4 || D == 8 || D == 16 || D == 32) && std::fabs(fs_in - D * 1.92e6) <= 1e-6))
    return cfail(h, "fs_in must be D * 1.92 MHz with D in {2, 4, 8, 16, 32}");
  if (!n_in || n_in / D >= (1ull << 31)) return cfail(h, "n_in must be positive and below 2^31 D");
  if (!std::isfinite(fc_in)) return cfail(h, "fc_in must be finite");
  if (!(std::isfinite(fs_programmed) && fs_programmed > 0)) return cfail(h, "fs_programmed must be finite and positive");
  if (!n_cells) return LCS_OK;
  lcs_ctx* ctx = h->ctx;
  LCS_CUDA(ctx, cudaSetDevice(ctx->device));
  // every cell checked, and its windows laid out, before any device work
  std::vector<CellPlan> ch(n_cells);
  long long lo = std::numeric_limits<long long>::max(), hi = 0;
  const int N = 128 * D, lg = 7 + __builtin_ctz(D);
  for (uint32_t i = 0; i < n_cells; i++) {
    const std::string why = plan_cell(cells[i], n_in, D, fs_in, fc_in, fs_programmed, ch[i]);
    if (!why.empty()) return cfail(h, "cell " + std::to_string(i) + ": " + why);
    lo = std::min(lo, ch[i].q.front());
    hi = std::max(hi, ch[i].q.back() + N);
  }
  cudaStream_t st = ctx->streams[0];
  const unsigned char* d_in = static_cast<const unsigned char*>(iq);
  long long base = 0;
  if (!on_device) {
    LCS_CUDA(ctx, h->d_iq.ensure((size_t)(hi - lo) * esz));
    LCS_CUDA(ctx, cudaMemcpyAsync(h->d_iq.p, static_cast<const unsigned char*>(iq) + (size_t)lo * esz, (size_t)(hi - lo) * esz,
                                  cudaMemcpyHostToDevice, st));
    d_in = h->d_iq.p;
    base = lo;
  }
  if (h->tw_n != (uint32_t)N) {
    std::vector<float2> tw(N);
    for (int n = 0; n < N; n++) {
      const double ang = -2 * M_PI * (double)n / (double)N;
      tw[n] = make_float2((float)std::cos(ang), (float)std::sin(ang));
    }
    h->tw_n = 0;
    LCS_CUDA(ctx, h->d_tw.ensure(N));
    LCS_CUDA(ctx, cudaMemcpy(h->d_tw.p, tw.data(), N * sizeof(float2), cudaMemcpyHostToDevice));
    h->tw_n = N;
  }
  LCS_CUDA(ctx, h->d_out.ensure(std::min(n_cells, CHUNK)));
  for (uint32_t c0 = 0; c0 < n_cells; c0 += CHUNK) {
    const uint32_t nc = std::min(CHUNK, n_cells - c0);
    size_t n_win = 0, n_grid = 0;
    for (uint32_t i = 0; i < nc; i++) n_win += ch[c0 + i].q.size();
    const size_t n_tab = (size_t)nc * N_SLOT_TAB * 3;
    LCS_CUDA(ctx, h->up.reset(n_win * sizeof(Win) + nc * (sizeof(GridCell) + sizeof(MeasCell)) +
                              n_tab * (2 * MAX_RB * sizeof(char2) + 4) + 5 * 16));
    Win* win = h->up.take<Win>(n_win);
    GridCell* gc = h->up.take<GridCell>(nc);
    MeasCell* mc = h->up.take<MeasCell>(nc);
    char2* rs_tab = h->up.take<char2>(n_tab * 2 * MAX_RB);
    unsigned char* shift_tab = h->up.take<unsigned char>(n_tab * 4);
    size_t w = 0;
    for (uint32_t i = 0; i < nc; i++) {
      const CellPlan& c = ch[c0 + i];
      const size_t W = 12 * (size_t)c.R;
      gc[i] = GridCell{c.step, c.kpi, c.R, 0};
      mc[i] = MeasCell{n_grid, c.R, c.n_ports, c.nw, 0};
      for (size_t j = 0; j < c.q.size(); j++, w++) win[w] = Win{c.q[j], c.late[j], n_grid + j * W, (int)i, 0};
      n_grid += c.q.size() * W;
      const RsDl rs(c.n_id_cell, c.cp_type, c.R);
      for (int sl = 0; sl < N_SLOT_TAB; sl++)
        for (int s3 = 0; s3 < 3; s3++) {
          const int sym = s3 == 2 ? rs.n_symb - 3 : s3;
          const cd* r = rs.get(sl, sym);
          char2* t = rs_tab + ((i * N_SLOT_TAB + sl) * 3 + s3) * 2 * MAX_RB;
          for (int m = 0; m < 2 * MAX_RB; m++)
            t[m] = m < 2 * c.R ? make_char2(r[m].real() > 0 ? 1 : -1, r[m].imag() > 0 ? 1 : -1) : make_char2(0, 0);
          for (int p = 0; p < 4; p++) shift_tab[((i * N_SLOT_TAB + sl) * 3 + s3) * 4 + p] = (unsigned char)rs.shift(sl, sym, p);
        }
    }
    LCS_CUDA(ctx, h->d_grid.ensure(n_grid));
    LCS_CUDA(ctx, h->up.upload(st));
    LCS_CUDA(ctx, cudaMemsetAsync(h->d_out.p, 0, nc * sizeof(lcs_carrier_meas), st));   // the records' padding too
    GridParams P;
    P.in = d_in;
    P.base = base;
    P.fs = std::llround(fs_in);
    P.win = h->up.dev(win);
    P.cell = h->up.dev(gc);
    P.n_win = (int)n_win;
    P.lg = lg;
    P.scale = (float)(std::sqrt(128.0) / N);
    P.tw = h->d_tw.p;
    P.grid = h->d_grid.p;
    const int per = TILE / N;
    LCS_CUDA(ctx, h->clock.begin(st));
    if (StreamFormats::dispatch(iq_format, [&](auto FMT) {
          carrier_grid_kernel<FMT><<<(unsigned)((n_win + per - 1) / per), THREADS, 0, st>>>(P);
        }) != LCS_OK)
      return cfail(h, "no grid kernel for this iq_format");
    carrier_meas_kernel<<<nc, MEAS_THREADS, 0, st>>>(h->d_grid.p, h->up.dev(rs_tab), h->up.dev(shift_tab), h->up.dev(mc),
                                                     h->d_out.p);
    ctx->launches += LCS_CARRIER_LAUNCHES_PER_CHUNK;
    LCS_CUDA(ctx, cudaGetLastError());
    LCS_CUDA(ctx, h->clock.end(st, LCS_CARRIER_LAUNCHES_PER_CHUNK));
    LCS_CUDA(ctx, cudaMemcpyAsync(out + c0, h->d_out.p, nc * sizeof(lcs_carrier_meas), cudaMemcpyDeviceToHost, st));
    LCS_CUDA(ctx, cudaStreamSynchronize(st));
  }
  return LCS_OK;
}

lcs_status lcs_carrier_timing_read(lcs_carrier* h, double* kernel_ms, uint64_t* launches) {
  if (!h) return LCS_ERR_ARG;
  if (!kernel_ms || !launches) return fail(h->ctx, LCS_ERR_ARG, "lcs_carrier_timing_read: null pointer");
  LCS_CUDA(h->ctx, h->clock.read(kernel_ms, launches));
  return LCS_OK;
}

}  // extern "C"
