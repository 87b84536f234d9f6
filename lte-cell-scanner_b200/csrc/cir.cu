// cir.cu - the power delay profile of found cells over their whole carrier, from the wideband recording they were found
// in (DESIGN.md section 4.11; contract in include/lcs_cir.h).  Built into liblcs_cir.so.
//
// A call is cut into chunks of LCS_CIR_CHUNK cells; each chunk makes two launches on the context's stream:
//   1. carrier_grid_kernel (carrier_grid.cuh): the CRS symbols of every cell's full-bandwidth grid, as lcs_carrier makes
//      them.
//   2. cir_kernel: one CTA per (cell, port, block of TAPS_PER_CTA taps).  The CTA stages the 2048 twiddles exp(j2pi i /
//      2048) and, slot by slot, w h of the port's 2R CRS in each of its symbols; four threads evaluate each tap, each over
//      every fourth m, and add their parts by shuffles.  Each tap keeps the c of the two slots before the current one, so
//      a pair (slot t, slot t + 2) is summed as soon as its second symbol is transformed, in slot order, in FP64.  The
//      last CTA of a (cell, port) to finish, which a device counter behind a fence tells it is last, walks the complete
//      pdp in ascending tap order for the statistics.  Nothing depends on the order CTAs finish in, so a cell's record is
//      bitwise the same whatever else the call measures.
#include "../../include/lcs_cir.h"
#include "carrier_grid.cuh"

namespace lcs {
namespace cir {

using namespace lcs::carrier;
constexpr int TAPS = LCS_CIR_TAPS;
constexpr int TAP0 = 64;                         // tau_j = (j - TAP0) T_s
constexpr int CIR_THREADS = 256;
constexpr int SPLIT = 4;                         // threads per tap
constexpr int TAPS_PER_CTA = CIR_THREADS / SPLIT;
constexpr int TAP_BLOCKS = TAPS / TAPS_PER_CTA;
constexpr int N_TW = 2048;                       // 15 kHz T_s = 1 / 2048
constexpr double T_S = 1.0 / 30.72e6;
constexpr uint32_t CHUNK = LCS_CIR_CHUNK;
static_assert(TAPS % TAPS_PER_CTA == 0, "whole tap blocks");

struct CirCell {
  unsigned long long off;                        // the cell's grid [N_SLOT][nw][12 R]
  double t_frame;                                // D frame_start / fs_in
  int R, n_ports, nw, pad;                       // nw: windows per slot (2, or 3 for four ports)
};

__device__ __forceinline__ double tau(int j) { return (double)(j - TAP0) * T_S; }

// The statistics of rule 5 of lcs_cir.h from the complete pdp and per-tap noise of one (cell, port), by one thread.
__device__ void cir_stats(const double* pdp, const double* noise, int p, int n_pairs, double t_frame, lcs_cir_meas* o) {
  int js = 0;
  for (int j = 1; j < TAPS; j++)
    if (pdp[j] > pdp[js]) js = j;
  const double thr = pdp[js] * 0.01;             // 10^(-LCS_CIR_RANGE_DB / 10)
  double fl = 0, w = 0, wt = 0;
  int nk = 0, jf = -1;
  for (int j = 0; j < TAPS; j++) {
    fl += noise[j];
    if (!(pdp[j] >= thr)) continue;
    nk++;
    w += pdp[j];
    wt += pdp[j] * tau(j);
    if (jf < 0 && (j == 0 || pdp[j] >= pdp[j - 1]) && (j == TAPS - 1 || pdp[j] >= pdp[j + 1])) jf = j;
  }
  const double mean = wt / w;
  double v = 0;
  for (int j = 0; j < TAPS; j++)
    if (pdp[j] >= thr) {
      const double d = tau(j) - mean;
      v += pdp[j] * d * d;
    }
  double delta = 0;
  if (jf > 0 && jf < TAPS - 1) {
    const double pm = pdp[jf - 1], p0 = pdp[jf], pp = pdp[jf + 1], den = pm - 2 * p0 + pp;
    if (den != 0) delta = fmin(0.5, fmax(-0.5, (pm - pp) / (2 * den)));
  }
  o->floor[p] = fl / TAPS;
  o->peak_delay[p] = tau(js);
  o->first_delay[p] = tau(jf) + delta * T_S;
  o->mean_delay[p] = mean;
  o->rms_spread[p] = sqrt(v / w);
  o->n_pairs[p] = (uint32_t)n_pairs;
  o->n_taps[p] = (uint32_t)nk;
  if (p == 0) o->frame_arrival = t_frame + o->first_delay[0];
}

// rs_all [cell][20][3][2 MAX_RB] holds the signs of the CRS r = (s.x + j s.y) / sqrt(2); shift_all [cell][20][3][4].
// noise [cell][4][TAPS] and count [cell][4] are scratch; count starts at 0.
__global__ void __launch_bounds__(CIR_THREADS) cir_kernel(const float2* __restrict__ grid, const char2* __restrict__ rs_all,
                                                          const unsigned char* __restrict__ shift_all,
                                                          const CirCell* __restrict__ par, double* noise,
                                                          unsigned int* count, lcs_cir_meas* out) {
  __shared__ double2 tw[N_TW];                   // exp(+j2pi i / 2048)
  __shared__ double2 v[2][2 * MAX_RB];           // w h of the slot's (up to two) CRS symbols of the port
  __shared__ double ws[2 * MAX_RB];              // w[m] / sqrt(2)
  __shared__ int sb[2];                          // the subcarrier shift s_t of each staged symbol
  __shared__ bool last;
  const int tid = threadIdx.x, p = blockIdx.y, cell = blockIdx.z;
  const CirCell cc = par[cell];
  const int R = cc.R, M = 2 * R, W = 12 * R, nw = cc.nw;
  lcs_cir_meas* o = out + cell;
  const double nan = __longlong_as_double(0x7ff8000000000000ll);
  if (p >= cc.n_ports) {                         // rule 7, by the port's first tap block
    if (blockIdx.x) return;
    for (int j = tid; j < TAPS; j += CIR_THREADS) o->pdp[p][j] = nan;
    if (!tid) {
      o->floor[p] = o->peak_delay[p] = o->first_delay[p] = o->mean_delay[p] = o->rms_spread[p] = nan;
      o->n_pairs[p] = o->n_taps[p] = 0;
    }
    return;
  }
  for (int i = tid; i < N_TW; i += CIR_THREADS) {
    double s, c;
    sincospi((double)i / (N_TW / 2), &s, &c);
    tw[i] = make_double2(c, s);
  }
  for (int m = tid; m < M; m += CIR_THREADS) {
    const double s = sinpi((m + 0.5) / M);
    ws[m] = s * s * M_SQRT1_2;
  }
  const float2* G = grid + cc.off;
  const char2* rs = rs_all + (size_t)cell * N_SLOT_TAB * 3 * 2 * MAX_RB;
  const unsigned char* shift = shift_all + (size_t)cell * N_SLOT_TAB * 3 * 4;
  const int nsp = p < 2 ? 2 : 1;                 // CRS symbols of the port per slot
  const int k = tid % SPLIT, j = blockIdx.x * TAPS_PER_CTA + tid / SPLIT, dj = j - TAP0;
  double2 prev1[2], prev2[2];                    // c of slots t - 1 and t - 2
  double cre = 0, cim = 0, T = 0;
  for (int t = 0; t < N_SLOT; t++) {
    __syncthreads();                             // the previous slot's v is consumed (and tw, ws written)
    for (int e = tid; e < nsp * M; e += CIR_THREADS) {
      const int si = e / M, m = e % M;
      const int s3 = p < 2 ? (si ? 2 : 0) : 1;
      const int kw = s3 == 0 ? 0 : (s3 == 2 ? nw - 1 : 1);
      const int tab = (t % N_SLOT_TAB) * 3 + s3;
      const int sh = shift[tab * 4 + p];
      const float2 y = G[(size_t)(t * nw + kw) * W + 6 * m + sh];
      const char2 r = rs[tab * 2 * MAX_RB + m];
      v[si][m] = make_double2(ws[m] * ((double)y.x * r.x + (double)y.y * r.y), ws[m] * ((double)y.y * r.x - (double)y.x * r.y));
      if (m == 0) sb[si] = sh;
    }
    __syncthreads();
    double2 cur[2];
#pragma unroll
    for (int si = 0; si < 2; si++) {
      if (si >= nsp) break;
      double x = 0, y = 0;
      const int s = sb[si];
      for (int m = k; m < M; m += SPLIT) {
        const int c = 6 * m + s, b = c < 6 * R ? c - 6 * R : c - 6 * R + 1;
        const double2 a = v[si][m], e = tw[(b * dj) & (N_TW - 1)];
        x = fma(a.x, e.x, fma(-a.y, e.y, x));
        y = fma(a.x, e.y, fma(a.y, e.x, y));
      }
      x += __shfl_xor_sync(0xffffffffu, x, 1);
      y += __shfl_xor_sync(0xffffffffu, y, 1);
      x += __shfl_xor_sync(0xffffffffu, x, 2);
      y += __shfl_xor_sync(0xffffffffu, y, 2);
      cur[si] = make_double2(x, y);
      if (t >= 2) {                              // the pair (slot t - 2, slot t): c_a conj(c_b)
        const double2 a = prev2[si];
        cre += a.x * x + a.y * y;
        cim += a.y * x - a.x * y;
        T += (a.x * a.x + a.y * a.y) + (x * x + y * y);
      }
      prev2[si] = prev1[si];
      prev1[si] = cur[si];
    }
  }
  const int n = nsp * (N_SLOT - 2);
  const double S = hypot(cre / n, cim / n), Tm = T / (2.0 * n), scale = 1.0 / (128.0 * R * R);
  double* nz = noise + ((size_t)cell * 4 + p) * TAPS;
  if (k == 0) {
    o->pdp[p][j] = S * scale;
    nz[j] = (Tm - S) * scale;
  }
  __threadfence();                               // this CTA's taps visible before it counts itself done
  __syncthreads();
  if (!tid) last = atomicAdd(&count[cell * 4 + p], 1u) == TAP_BLOCKS - 1;
  __syncthreads();
  if (!last) return;
  __threadfence();
  // the last CTA of the (cell, port): the complete pdp and noise, then the statistics in ascending tap order
  double* pd = &v[0][0].x;                       // 2 * 2 MAX_RB double2 = 800 doubles >= 2 TAPS
  for (int i = tid; i < TAPS; i += CIR_THREADS) {
    pd[i] = __ldcg(&o->pdp[p][i]);
    pd[TAPS + i] = __ldcg(&nz[i]);
  }
  __syncthreads();
  if (!tid) cir_stats(pd, pd + TAPS, p, n, cc.t_frame, o);
}

}  // namespace cir
}  // namespace lcs

using namespace lcs;
using namespace lcs::carrier;
using namespace lcs::cir;

struct lcs_cir : GridModule<lcs_cir_meas> {
  DevBuf<double> d_noise;                        // [CHUNK][4][TAPS] noise per tap
  DevBuf<unsigned int> d_count;                  // [CHUNK][4] finished tap blocks
};

extern "C" {

lcs_status lcs_cir_create(lcs_ctx* ctx, lcs_cir** out) { return grid_create(ctx, out, "lcs_cir_create"); }

void lcs_cir_destroy(lcs_cir* h) { grid_destroy(h); }

lcs_status lcs_cir_cells(lcs_cir* h, const void* iq, int iq_format, int on_device, uint64_t n_in, double fs_in,
                         double fc_in, const lcs_cell* cells, uint32_t n_cells, double fs_programmed, lcs_cir_meas* out) {
  CirCell* cc = nullptr;
  return grid_cells(
      h, "lcs_cir_cells", CHUNK, LCS_CIR_LAUNCHES_PER_CHUNK, iq, iq_format, on_device, n_in, fs_in, fc_in, cells, n_cells,
      fs_programmed, out, plan_cell, [](uint32_t n) { return n * sizeof(CirCell) + 16; },
      [&](const GridChunk& c) {
        cc = h->g.up.take<CirCell>(c.n);
        for (uint32_t i = 0; i < c.n; i++) {
          const CellPlan& p = c.plan[i];
          cc[i] = CirCell{c.t.off[i], c.D * c.cell[i].frame_start / fs_in, p.R, p.n_ports, p.nw, 0};
        }
        // the first chunk is the largest: it sizes the scratch for the call
        cudaError_t e = h->d_noise.ensure((size_t)c.n * 4 * TAPS);
        if (e == cudaSuccess) e = h->d_count.ensure((size_t)c.n * 4);
        return e == cudaSuccess ? cudaMemsetAsync(h->d_count.p, 0, c.n * 4 * sizeof(unsigned int), c.st) : e;
      },
      [&](const GridChunk& c) {
        cir_kernel<<<dim3(TAP_BLOCKS, 4, c.n), CIR_THREADS, 0, c.st>>>(h->g.d_grid.p, h->g.up.dev(c.t.rs),
                                                                       h->g.up.dev(c.t.shift), h->g.up.dev(cc),
                                                                       h->d_noise.p, h->d_count.p, h->d_out.p);
      });
}

lcs_status lcs_cir_timing_read(lcs_cir* h, double* kernel_ms, uint64_t* launches) {
  return grid_timing_read(h, kernel_ms, launches, "lcs_cir_timing_read");
}

}  // extern "C"
