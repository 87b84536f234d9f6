// meas.cu - RSRP, RSRQ and SINR of found cells from the CRS of their central six resource blocks (DESIGN.md section 4.9;
// contract in include/lcs_meas.h).
//
// One call measures every cell it is given with two launches on the context's stream:
//   1. tfg_kernel (chain_gpu.cu, through launch_grids): each cell's 72-subcarrier grid, exactly as lcs_extract_tfg makes it
//      for the cell with freq_fine = freq_superfine; the cells may sit in different channels of one [n_ch][n_cap] buffer.
//   2. meas_kernel: one CTA per cell.  Each thread sums a fixed, strided subset of the cell's CRS pairs (and of its RSSI
//      resource elements) in FP64; the warps then reduce with a fixed shuffle tree and thread 0 adds the warps in order.
//      The result is thus the same on every run and independent of the other cells of the call.
// The CRS values and their subcarrier shifts come from the host tables (RsDl, chain_host.cpp), staged with the grid
// geometry and uploaded with it in one copy per call.
#include <cmath>
#include <limits>
#include <new>
#include <string>
#include <vector>

#include "../../include/lcs_meas.h"
#include "chain_gpu.hpp"
#include "iq_format.cuh"

namespace lcs {
namespace meas {

constexpr int THREADS = 256;
constexpr int WARPS = THREADS / 32;
constexpr int N_SUM = 13;          // C_p (re, im) and T_p for 4 ports, and the RSSI sum
constexpr int N_SLOT_TAB = 20;     // CRS tables repeat every frame: [20 slots][3 symbols {0, 1, n_symb-3}]

// Per cell: n_symb, n_ports, n_ofdm.
__global__ void __launch_bounds__(THREADS) meas_kernel(const double2* __restrict__ tfg_all, const double2* __restrict__ rs_all,
                                                       const unsigned char* __restrict__ shift_all,
                                                       const int4* __restrict__ par, lcs_cell_meas* __restrict__ out) {
  __shared__ double part[WARPS][N_SUM];
  const int tid = threadIdx.x, cell = blockIdx.x;
  const int4 pc = par[cell];
  const int n_symb = pc.x, n_ports = pc.y, n_slot = pc.z / n_symb;
  const double2* Y = tfg_all + (size_t)cell * TFG_MAX * 72;
  const double2* rs = rs_all + (size_t)cell * N_SLOT_TAB * 3 * 12;        // [slot][s3][12]
  const unsigned char* shift = shift_all + (size_t)cell * N_SLOT_TAB * 3 * 4;   // [slot][s3][port]
  double acc[N_SUM];
#pragma unroll
  for (int v = 0; v < N_SUM; v++) acc[v] = 0;
#pragma unroll
  for (int p = 0; p < 4; p++) {
    if (p >= n_ports) break;
    const int nsp = p < 2 ? 2 : 1;                 // CRS symbols of the port per slot
    const int n_pairs = nsp * 12 * (n_slot - 2);
    for (int j = tid; j < n_pairs; j += THREADS) {
      const int i = j % 12, q = j / 12, si = q % nsp, t = q / nsp;
      const int s3 = p < 2 ? (si ? 2 : 0) : 1;
      const int sym = s3 == 2 ? n_symb - 3 : s3;
      const int ta = t % N_SLOT_TAB, tb = (t + 2) % N_SLOT_TAB;
      const int col = shift[(ta * 3 + s3) * 4 + p] + 6 * i;
      const double2 ya = Y[(size_t)(t * n_symb + sym) * 72 + col], yb = Y[(size_t)((t + 2) * n_symb + sym) * 72 + col];
      const double2 ra = rs[(ta * 3 + s3) * 12 + i], rb = rs[(tb * 3 + s3) * 12 + i];
      const double2 ha = make_double2(ya.x * ra.x + ya.y * ra.y, ya.y * ra.x - ya.x * ra.y);   // y conj(r)
      const double2 hb = make_double2(yb.x * rb.x + yb.y * rb.y, yb.y * rb.x - yb.x * rb.y);
      acc[3 * p] += ha.x * hb.x + ha.y * hb.y;                                                 // h_a conj(h_b)
      acc[3 * p + 1] += ha.y * hb.x - ha.x * hb.y;
      acc[3 * p + 2] += (ha.x * ha.x + ha.y * ha.y) + (hb.x * hb.x + hb.y * hb.y);
    }
  }
  const int n_rssi = 2 * n_slot * 72;              // the port-0 CRS symbols {0, n_symb-3} of every slot, all 72 REs
  for (int j = tid; j < n_rssi; j += THREADS) {
    const int k = j % 72, q = j / 72;
    const double2 y = Y[(size_t)((q >> 1) * n_symb + ((q & 1) ? n_symb - 3 : 0)) * 72 + k];
    acc[12] += y.x * y.x + y.y * y.y;
  }
#pragma unroll
  for (int v = 0; v < N_SUM; v++)
    for (int o = 16; o > 0; o >>= 1) acc[v] += __shfl_down_sync(0xffffffffu, acc[v], o);
  if ((tid & 31) == 0)
#pragma unroll
    for (int v = 0; v < N_SUM; v++) part[tid >> 5][v] = acc[v];
  __syncthreads();
  if (tid) return;
  double s[N_SUM];
  for (int v = 0; v < N_SUM; v++) {
    s[v] = part[0][v];
    for (int w = 1; w < WARPS; w++) s[v] += part[w][v];
  }
  lcs_cell_meas m;
  const double nan = __longlong_as_double(0x7ff8000000000000ll), inf = __longlong_as_double(0x7ff0000000000000ll);
  for (int p = 0; p < 4; p++) {
    if (p < n_ports) {
      const int n = (p < 2 ? 2 : 1) * 12 * (n_slot - 2);
      const double cre = s[3 * p] / n, cim = s[3 * p + 1] / n, T = s[3 * p + 2] / (2.0 * n);
      const double S = hypot(cre, cim), N = T - S;
      m.rsrp[p] = S / 128;
      m.noise[p] = N / 128;
      m.sinr[p] = N > 0 ? S / N : inf;
      m.n_pairs[p] = (uint32_t)n;
    } else {
      m.rsrp[p] = m.noise[p] = m.sinr[p] = nan;
      m.n_pairs[p] = 0;
    }
  }
  m.rssi = s[12] / (2.0 * n_slot) / 128;
  m.rsrq = 6 * m.rsrp[0] / m.rssi;
  out[cell] = m;
}

}  // namespace meas
}  // namespace lcs

using namespace lcs;

struct lcs_meas {
  lcs_ctx* ctx = nullptr;
  DevBuf<unsigned char> d_iq;              // host input, uploaded
  Staging up;                              // per call: the grid geometry, the CRS and shift tables and the cell parameters
  DevBuf<double2> d_tfg;                   // [cell][TFG_MAX][72]
  DevBuf<lcs_cell_meas> d_out;
  KernelClock clock;                       // both launches of each call
};

namespace {

lcs_status mfail(const lcs_meas* m, const std::string& msg) { return fail(m->ctx, LCS_ERR_ARG, "lcs_meas_cells: " + msg); }

}  // namespace

extern "C" {

lcs_status lcs_meas_create(lcs_ctx* ctx, lcs_meas** out) {
  if (!ctx || !out) return fail(ctx, LCS_ERR_ARG, "lcs_meas_create: null argument");
  lcs_meas* m = new (std::nothrow) lcs_meas();
  if (!m) return fail(ctx, LCS_ERR_STATE, "lcs_meas_create: out of memory");
  m->ctx = ctx;
  *out = m;
  return LCS_OK;
}

void lcs_meas_destroy(lcs_meas* m) {
  if (!m) return;
  cudaSetDevice(m->ctx->device);             // its buffers and events belong to the context's device
  delete m;
}

lcs_status lcs_meas_cells(lcs_meas* m, const void* iq, int iq_format, int on_device, uint32_t n_ch, uint32_t n_cap,
                          const lcs_cell* cells, const uint32_t* ch, uint32_t n_cells, double fs_programmed,
                          lcs_cell_meas* out) {
  if (!m) return LCS_ERR_ARG;
  if (!iq || (n_cells && (!cells || !ch || !out))) return mfail(m, "null pointer");
  if (!SearchFormats::has(iq_format)) return mfail(m, "iq_format must be LCS_IQ_CU8, CF32 or C128");
  const size_t esz = sample_bytes(iq_format);
  if (on_device && ((uintptr_t)iq & 15)) return mfail(m, "device iq must be 16-byte aligned");
  if (!n_ch || !n_cap || n_cap > 0x7fffffffu) return mfail(m, "n_ch and n_cap must be positive, n_cap < 2^31");
  if (!(std::isfinite(fs_programmed) && fs_programmed > 0)) return mfail(m, "fs_programmed must be finite and positive");
  if (!n_cells) return LCS_OK;
  // host tables of every cell, and every argument checked, before any device work
  lcs_ctx* ctx = m->ctx;
  LCS_CUDA(ctx, cudaSetDevice(ctx->device));
  const size_t L = n_cells;
  const size_t n_tab = L * meas::N_SLOT_TAB * 3;
  LCS_CUDA(ctx, m->up.reset(GridTables::bytes(L) + n_tab * (12 * sizeof(cd) + 4) + L * sizeof(int4) + 3 * 16));
  const GridTables g(m->up, L, true);
  cd* rs_tab = m->up.take<cd>(n_tab * 12);                         // [cell][20][3][12]
  unsigned char* shift_tab = m->up.take<unsigned char>(n_tab * 4);  // [cell][20][3][4]
  int4* par = m->up.take<int4>(L);
  std::vector<double> ts(TFG_MAX);
  for (size_t i = 0; i < L; i++) {
    const lcs_cell& c = cells[i];
    const std::string who = "cell " + std::to_string(i) + ": ";
    if (ch[i] >= n_ch) return mfail(m, who + "ch >= n_ch");
    if (c.cp_type != 1 && c.cp_type != 2) return mfail(m, who + "cp_type must be 1 (normal) or 2 (extended)");
    if (c.n_id_1 < 0 || c.n_id_1 > 167 || c.n_id_2 < 0 || c.n_id_2 > 2) return mfail(m, who + "n_id_1 / n_id_2 out of range");
    if (c.n_ports != 1 && c.n_ports != 2 && c.n_ports != 4) return mfail(m, who + "n_ports must be 1, 2 or 4");
    if (!(std::isfinite(c.frame_start) && std::isfinite(c.freq_superfine)))
      return mfail(m, who + "frame_start and freq_superfine must be finite");
    if (!(std::isfinite(c.fc_requested) && c.fc_requested > 0 && std::isfinite(c.fc_programmed) && c.fc_programmed > 0))
      return mfail(m, who + "fc_requested and fc_programmed must be finite and positive");
    lcs_cell gc = c;
    gc.freq_fine = c.freq_superfine;
    const char* why = "";
    if (tfg_geometry(gc, c.fc_requested, c.fc_programmed, fs_programmed, n_cap, g, i, ts.data(), &why) != LCS_OK)
      return mfail(m, who + "grid does not fit in the capture buffer (" + why + ")");
    g.base[i] = (uint64_t)ch[i] * n_cap;
    const RsDl rs(c.n_id_2 + 3 * c.n_id_1, c.cp_type);
    for (int sl = 0; sl < meas::N_SLOT_TAB; sl++)
      for (int s3 = 0; s3 < 3; s3++) {
        const int sym = s3 == 2 ? rs.n_symb - 3 : s3;
        const cd* r = rs.get(sl, sym);
        for (int k = 0; k < 12; k++) rs_tab[((i * meas::N_SLOT_TAB + sl) * 3 + s3) * 12 + k] = r[k];
        for (int p = 0; p < 4; p++) shift_tab[((i * meas::N_SLOT_TAB + sl) * 3 + s3) * 4 + p] = (unsigned char)rs.shift(sl, sym, p);
      }
    par[i] = make_int4(rs.n_symb, c.n_ports, g.n_ofdm[i], 0);
  }
  cudaStream_t st = ctx->streams[0];
  const void* d_iq = iq;
  if (!on_device) {
    const size_t bytes = (size_t)n_ch * n_cap * esz;
    LCS_CUDA(ctx, m->d_iq.ensure(bytes));
    LCS_CUDA(ctx, cudaMemcpyAsync(m->d_iq.p, iq, bytes, cudaMemcpyHostToDevice, st));
    d_iq = m->d_iq.p;
  }
  LCS_CUDA(ctx, m->d_tfg.ensure(L * TFG_MAX * 72));
  LCS_CUDA(ctx, m->d_out.ensure(L));
  LCS_CUDA(ctx, m->up.upload(st));
  LCS_CUDA(ctx, m->clock.begin(st));
  lcs_status rc = launch_grids(ctx, m->up, g, n_cells, d_iq, iq_format, m->d_tfg.p, st, "lcs_meas_cells: no grid kernel for this iq_format");
  if (rc != LCS_OK) return rc;
  meas::meas_kernel<<<n_cells, meas::THREADS, 0, st>>>(m->d_tfg.p, reinterpret_cast<const double2*>(m->up.dev(rs_tab)),
                                                       m->up.dev(shift_tab), m->up.dev(par), m->d_out.p);
  ctx->launches++;
  LCS_CUDA(ctx, cudaGetLastError());
  LCS_CUDA(ctx, m->clock.end(st, 2));
  LCS_CUDA(ctx, cudaMemcpyAsync(out, m->d_out.p, L * sizeof(lcs_cell_meas), cudaMemcpyDeviceToHost, st));
  LCS_CUDA(ctx, cudaStreamSynchronize(st));
  return LCS_OK;
}

lcs_status lcs_meas_timing_read(lcs_meas* m, double* kernel_ms, uint64_t* launches) {
  if (!m) return LCS_ERR_ARG;
  if (!kernel_ms || !launches) return fail(m->ctx, LCS_ERR_ARG, "lcs_meas_timing_read: null pointer");
  LCS_CUDA(m->ctx, m->clock.read(kernel_ms, launches));
  return LCS_OK;
}

}  // extern "C"
