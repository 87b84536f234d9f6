// pcfich_kernel.cuh - the PCFICH decoder's kernel and its device helpers (contract in include/lcs_pcfich.h), shared by
// liblcs_pcfich.so (pcfich.cu) and liblcs_pdcch.so (pdcch.cu), whose control region starts from the same decisions.
//
// pcfich_kernel runs one CTA per cell.  Thread (s, j) equalises pair j of subframe s (rules 2-4) into shared memory; then
// one thread per subframe decides it (rule 5) and one thread counts the decisions (rule 6), every sum in FP64 in a fixed
// order, so a cell's record is bitwise the same whatever else the call decodes.  pcfich_fill and pcfich_launch stage and
// launch it in a chunk of either module.
#pragma once
#include "../../include/lcs_pcfich.h"
#include "carrier_grid.cuh"

namespace lcs {
namespace pcfich {

using namespace lcs::carrier;
constexpr int N_SF = LCS_PCFICH_SUBFRAMES;
constexpr int PAIRS = 8;                         // 16 PCFICH symbols
constexpr int PC_THREADS = 512;                  // >= N_SF * PAIRS
constexpr uint32_t CHUNK = LCS_PCFICH_CHUNK;
static_assert(N_SF * PAIRS <= PC_THREADS, "one thread per (subframe, pair)");
static_assert(2 * N_SF == N_SLOT, "subframes of the grid");

struct PcfichCell {
  unsigned long long off;                        // the cell's grid [N_SF][nw][12 R]
  int R, n_ports, nw, n_id;                      // nw: windows per subframe (1, or 2 for four ports)
};

__device__ __forceinline__ double2 cmul_d(double2 a, double2 b) { return make_double2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }
__device__ __forceinline__ double2 conj_d(double2 a) { return make_double2(a.x, -a.y); }

// h[m] = Y[6 m + sh] conj(r[m]), r = (rs.x + j rs.y) / sqrt(2)
__device__ __forceinline__ double2 crs_h(const float2* row, const char2* r, int sh, int m) {
  const float2 y = row[6 * m + sh];
  const char2 s = r[m];
  return make_double2(((double)y.x * s.x + (double)y.y * s.y) * M_SQRT1_2, ((double)y.y * s.x - (double)y.x * s.y) * M_SQRT1_2);
}

// Rule 3: hhat of a port at column k from its CRS in grid row `row` (shift sh, signs r).
__device__ double2 chan(const float2* row, const char2* r, int sh, int R, int k) {
  const int d = k - sh, M = 2 * R;
  if (d <= 0) return crs_h(row, r, sh, 0);
  if (d >= 6 * (M - 1)) return crs_h(row, r, sh, M - 1);
  const int m = d / 6;
  const double f = (double)(d - 6 * m) / 6.0;
  const double2 a = crs_h(row, r, sh, m), b = crs_h(row, r, sh, m + 1);
  return make_double2((1 - f) * a.x + f * b.x, (1 - f) * a.y + f * b.y);
}

// Rule 2: the column of PCFICH RE n < 16.
__device__ __forceinline__ int re_col(int n, int R, int n_id) {
  const int i = n >> 2, v = n_id % 3;
  int o = n & 3;
  if (o >= v) o++;
  if (o >= v + 3) o++;
  return (6 * (n_id % (2 * R)) + 6 * ((i * R) / 2)) % (12 * R) + o;
}

// rs_all [cell][20][3][2 MAX_RB] holds the signs of the CRS r = (s.x + j s.y) / sqrt(2); shift_all [cell][20][3][4];
// scr [cell][10] the scrambling bits c_b of each subframe number, bit b of the word.
__global__ void __launch_bounds__(PC_THREADS) pcfich_kernel(const float2* __restrict__ grid, const char2* __restrict__ rs_all,
                                                            const unsigned char* __restrict__ shift_all,
                                                            const PcfichCell* __restrict__ par,
                                                            const uint32_t* __restrict__ scr, lcs_pcfich_meas* out) {
  __shared__ double2 xs[N_SF][2 * PAIRS];        // xhat
  __shared__ unsigned char dec[N_SF];
  const int tid = threadIdx.x, cell = blockIdx.x;
  const PcfichCell cc = par[cell];
  const int R = cc.R, W = 12 * R;
  lcs_pcfich_meas* o = out + cell;
  if (tid < N_SF * PAIRS) {                      // rules 2-4: pair j of subframe s
    const int s = tid / PAIRS, j = tid % PAIRS;
    const float2* G = grid + cc.off + (size_t)s * cc.nw * W;
    const int sl = (2 * s) % N_SLOT_TAB;
    const char2* rs = rs_all + (size_t)cell * N_SLOT_TAB * 3 * 2 * MAX_RB;
    const unsigned char* shift = shift_all + (size_t)cell * N_SLOT_TAB * 3 * 4;
    const int k0 = re_col(2 * j, R, cc.n_id), k1 = re_col(2 * j + 1, R, cc.n_id);
    const double2 y0 = make_double2(G[k0].x, G[k0].y), y1 = make_double2(G[k1].x, G[k1].y);
    const int pa = cc.n_ports == 4 ? (j & 1) : 0, pb = cc.n_ports == 4 ? 2 + (j & 1) : 1;
    auto est = [&](int p, int k) {               // ports 0 and 1 from symbol 0, ports 2 and 3 from symbol 1
      const int s3 = p < 2 ? 0 : 1, tab = sl * 3 + s3;
      return chan(G + (size_t)s3 * W, rs + tab * 2 * MAX_RB, shift[tab * 4 + p], R, k);
    };
    double2 x0, x1;
    if (cc.n_ports == 1) {
      const double2 h0 = est(0, k0), h1 = est(0, k1);
      const double g0 = h0.x * h0.x + h0.y * h0.y, g1 = h1.x * h1.x + h1.y * h1.y;
      const double2 a = cmul_d(y0, conj_d(h0)), b = cmul_d(y1, conj_d(h1));
      x0 = make_double2(a.x / g0, a.y / g0);
      x1 = make_double2(b.x / g1, b.y / g1);
    } else {
      const double2 a0 = est(pa, k0), a1 = est(pa, k1), b0 = est(pb, k0), b1 = est(pb, k1);
      const double2 ha = make_double2((a0.x + a1.x) / 2, (a0.y + a1.y) / 2), hb = make_double2((b0.x + b1.x) / 2, (b0.y + b1.y) / 2);
      const double g = (ha.x * ha.x + ha.y * ha.y) + (hb.x * hb.x + hb.y * hb.y);
      const double2 n0 = cmul_d(conj_d(ha), y0), m0 = cmul_d(hb, conj_d(y1));
      const double2 n1 = cmul_d(conj_d(ha), y1), m1 = cmul_d(hb, conj_d(y0));
      x0 = make_double2(M_SQRT2 * (n0.x + m0.x) / g, M_SQRT2 * (n0.y + m0.y) / g);
      x1 = make_double2(M_SQRT2 * (n1.x - m1.x) / g, M_SQRT2 * (n1.y - m1.y) / g);
    }
    xs[s][2 * j] = x0;
    xs[s][2 * j + 1] = x1;
  }
  __syncthreads();
  if (tid < N_SF) {                              // rule 5: subframe tid
    const int s = tid;
    const uint32_t c = scr[cell * 10 + s % 10];
    double met[3] = {0, 0, 0};
    for (int n = 0; n < 2 * PAIRS; n++) {
      const double2 x = xs[s][n];
#pragma unroll
      for (int h = 0; h < 2; h++) {
        const int b = 2 * n + h;
        const double d = (h ? x.y : x.x) * ((c >> b) & 1 ? -1.0 : 1.0);
#pragma unroll
        for (int k = 0; k < 3; k++) met[k] += b % 3 == k ? d : -d;       // cw_k+1[b] = 0 where b mod 3 = k
      }
    }
    int best = 0;
    double top = 0;
#pragma unroll
    for (int k = 0; k < 3; k++) {
      met[k] *= M_SQRT2 / 32;
      if (k == 0 || met[k] > top) {
        best = k;
        top = met[k];
      }
    }
    double e = 0;
    for (int n = 0; n < 2 * PAIRS; n++) {
      const double2 x = xs[s][n];
      const int b = 2 * n;
      const int e0 = (b % 3 != best) ^ ((c >> b) & 1), e1 = ((b + 1) % 3 != best) ^ ((c >> (b + 1)) & 1);
      const double re = x.x - (e0 ? -M_SQRT1_2 : M_SQRT1_2), im = x.y - (e1 ? -M_SQRT1_2 : M_SQRT1_2);
      e += re * re + im * im;
    }
#pragma unroll
    for (int k = 0; k < 3; k++) o->metric[s][k] = met[k];
    o->sinr[s] = 16.0 / e;
    o->cfi[s] = best + 1;
    dec[s] = (unsigned char)(best + 1);
  }
  __syncthreads();
  if (!tid) {                                    // rule 6
    uint32_t n1 = 0, n2 = 0, n3 = 0;
    for (int s = 0; s < N_SF; s++) {
      n1 += dec[s] == 1;
      n2 += dec[s] == 2;
      n3 += dec[s] == 3;
    }
    const int mode = n3 > n1 && n3 > n2 ? 3 : (n2 > n1 ? 2 : 1);
    o->count[0] = 0;
    o->count[1] = n1;
    o->count[2] = n2;
    o->count[3] = n3;
    o->cfi_mode = mode;
    o->n_ctrl_symbols = mode + (R <= 10);
    o->n_subframes = N_SF;
  }
}

// scr [10] of pcfich_kernel for cell n_id: the scrambling bits of each subframe number (36.211 6.7.1).
inline void pcfich_scrambling(int n_id, uint32_t* scr) {
  for (int sf = 0; sf < 10; sf++) {
    const uint32_t c_init = (uint32_t)(sf + 1) * (2 * n_id + 1) * 512 + n_id;
    const std::vector<uint8_t> bits = lte_pn(c_init, 32);
    uint32_t w = 0;
    for (int b = 0; b < 32; b++) w |= (uint32_t)(bits[b] & 1) << b;
    scr[sf] = w;
  }
}

// The PCFICH stage of a chunk of grid_cells: pcfich_kernel's slices of the staging (pcfich_bytes of them for n cells),
// taken and filled by pcfich_fill, and its launch on the chunk's grids into out [n].
struct PcfichSlices {
  PcfichCell* cell;
  uint32_t* scr;                                 // [cell][10]
};

inline size_t pcfich_bytes(uint32_t n) { return n * sizeof(PcfichCell) + 16 + n * 10 * sizeof(uint32_t) + 16; }

inline PcfichSlices pcfich_fill(GridScratch& g, const GridChunk& c) {
  const PcfichSlices s{g.up.take<PcfichCell>(c.n), g.up.take<uint32_t>(c.n * 10)};
  for (uint32_t i = 0; i < c.n; i++) {
    const CellPlan& p = c.plan[i];
    s.cell[i] = PcfichCell{c.t.off[i], p.R, p.n_ports, p.nw, p.n_id_cell};
    pcfich_scrambling(p.n_id_cell, s.scr + i * 10);
  }
  return s;
}

inline void pcfich_launch(const GridScratch& g, const GridChunk& c, const PcfichSlices& s, lcs_pcfich_meas* out) {
  pcfich_kernel<<<c.n, PC_THREADS, 0, c.st>>>(g.d_grid.p, g.up.dev(c.t.rs), g.up.dev(c.t.shift), g.up.dev(s.cell),
                                              g.up.dev(s.scr), out);
}

}  // namespace pcfich
}  // namespace lcs
