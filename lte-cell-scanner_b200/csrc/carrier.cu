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
// CRS signs and shifts come from RsDl (chain_host.cpp).  The grid and the host path of a call (grid_cells) are
// carrier_grid.cuh's, which every module on the grid shares.
#include "../../include/lcs_carrier.h"
#include "carrier_grid.cuh"

namespace lcs {
namespace carrier {

constexpr int MEAS_THREADS = 512;
constexpr uint32_t CHUNK = LCS_CARRIER_CHUNK;

struct MeasCell {
  unsigned long long off;            // the cell's grid [N_SLOT][nw][12 R]
  int R, n_ports, nw, pad;           // nw: windows per slot (2, or 3 for four ports)
};

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

struct lcs_carrier : GridModule<lcs_carrier_meas> {};

extern "C" {

lcs_status lcs_carrier_create(lcs_ctx* ctx, lcs_carrier** out) { return grid_create(ctx, out, "lcs_carrier_create"); }

void lcs_carrier_destroy(lcs_carrier* h) { grid_destroy(h); }

lcs_status lcs_carrier_cells(lcs_carrier* h, const void* iq, int iq_format, int on_device, uint64_t n_in, double fs_in,
                             double fc_in, const lcs_cell* cells, uint32_t n_cells, double fs_programmed,
                             lcs_carrier_meas* out) {
  MeasCell* mc = nullptr;
  return grid_cells(
      h, "lcs_carrier_cells", CHUNK, LCS_CARRIER_LAUNCHES_PER_CHUNK, iq, iq_format, on_device, n_in, fs_in, fc_in, cells,
      n_cells, fs_programmed, out, plan_cell, [](uint32_t n) { return n * sizeof(MeasCell) + 16; },
      [&](const GridChunk& c) {
        mc = h->g.up.take<MeasCell>(c.n);
        for (uint32_t i = 0; i < c.n; i++) mc[i] = MeasCell{c.t.off[i], c.plan[i].R, c.plan[i].n_ports, c.plan[i].nw, 0};
        return cudaSuccess;
      },
      [&](const GridChunk& c) {
        carrier_meas_kernel<<<c.n, MEAS_THREADS, 0, c.st>>>(h->g.d_grid.p, h->g.up.dev(c.t.rs), h->g.up.dev(c.t.shift),
                                                            h->g.up.dev(mc), h->d_out.p);
      });
}

lcs_status lcs_carrier_timing_read(lcs_carrier* h, double* kernel_ms, uint64_t* launches) {
  return grid_timing_read(h, kernel_ms, launches, "lcs_carrier_timing_read");
}

}  // extern "C"
