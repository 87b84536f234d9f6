// pdcch_kernel.cuh - the PDCCH decoder's kernel (contract in include/lcs_pdcch.h), shared by liblcs_pdcch.so (pdcch.cu),
// which decodes every subframe of the grid, and liblcs_sib1.so (sib1.cu), which decodes only its SIB1 occasions.
//
// pdcch_kernel runs one CTA per (cell, listed subframe).  Thread (j, h) equalises pair h of quadruplet j of the common
// search space into shared memory (rule 7); then warp w runs decode w: candidate w / 2 at size w % 2 (rules 8-11), lanes
// over trellis states; then one thread resolves the duplicates and writes the subframe's record (rule 12).  Every sum is
// FP64 in a fixed order, so a cell's record is bitwise the same whatever else the call decodes.
#pragma once
#include "../../include/lcs_pdcch.h"
#include "pcfich_kernel.cuh"
#include "pdcch_plan.hpp"

namespace lcs {
namespace pdcch {

using namespace lcs::carrier;
using pcfich::chan;
using pcfich::cmul_d;
using pcfich::conj_d;
constexpr int N_SF = LCS_PDCCH_SUBFRAMES;
constexpr int N_DEC = 12;                        // 6 candidates x 2 sizes
constexpr int PD_THREADS = 32 * N_DEC;
constexpr uint32_t CHUNK = LCS_PDCCH_CHUNK;
static_assert(2 * MAX_QUAD <= PD_THREADS, "one thread per pair of the common search space");
static_assert(N_SF == LCS_PCFICH_SUBFRAMES, "subframes of the grid");

struct PdcchCell {
  unsigned long long off;                        // the cell's grid [N_SF][nw][12 R]
  int R, n_ports, nw, n_id, cp_type, phich_duration;
  int sf0;                                       // the first grid subframe the cell's CTAs decode
  int size[2], K[2];                             // format 1A, 1C
  int n_reg[4], n_cce[4];                        // by n_ctrl - 1
  uint32_t scr[10][SCR_WORDS];                   // rule 10's c of each subframe number
  uint16_t quad[4][MAX_QUAD];                    // by n_ctrl - 1: (l << 12) | k0 of the REG carrying quadruplet j
  uint8_t pos[2][3 * MAX_K];                     // by format: the coded bit of rate-matched bit i < 3K
  uint8_t inv[2][3 * MAX_K];                     // by format: the first rate-matched bit of coded bit x < 3K
};

__device__ __forceinline__ int conv_out(int s, int b) {         // the 3 output bits of input b in state s
  const int r = (b << 6) | s;
  return (__popc(0133 & r) & 1) | ((__popc(0171 & r) & 1) << 1) | ((__popc(0165 & r) & 1) << 2);
}

// Rule 1: the symbols of the control region of subframe s.
__device__ __forceinline__ int ctrl_symbols(const PdcchCell& cc, const lcs_pcfich_meas& pc, int s) {
  const int n = (int)pc.cfi[s] + (cc.R <= 10);
  return cc.phich_duration == 2 && n < 3 ? 3 : n;
}

// x with its sign flipped when the sign bit of `flip` is set: an exact negation.
__device__ __forceinline__ double flip_sign(double x, int flip) {
  return __hiloint2double(__double2hiint(x) ^ flip, __double2loint(x));
}

// rs_all [cell][20][3][2 MAX_RB] and shift_all [cell][20][3][4] as for pcfich_kernel; pc [cell] its records.  The CTAs
// of a cell decode grid subframes sf0 + STEP i, i < N_LIST (every subframe when N_LIST is 61: sf0 is not read), and only
// those are written in out [cell].
template <int N_LIST, int STEP>
__global__ void __launch_bounds__(PD_THREADS) pdcch_kernel(const float2* __restrict__ grid, const char2* __restrict__ rs_all,
                                                           const unsigned char* __restrict__ shift_all,
                                                           const PdcchCell* __restrict__ par,
                                                           const lcs_pcfich_meas* __restrict__ pc,
                                                           lcs_pdcch_meas* out) {
  __shared__ double su[MAX_QUAD * 8];            // u_b, bit b of quadruplet j at 8 j + b
  __shared__ double sv[MAX_QUAD * 8];            // u_b g
  __shared__ double sg[N_DEC][MAX_K][4];         // each decode's branch gains of outputs 0-3 (output o ^ 7 gains minus o's)
  __shared__ unsigned long long surv[N_DEC][2][MAX_K];   // survivor bits of the current and of the best start state
  __shared__ double rq[N_DEC];
  __shared__ unsigned long long ra[N_DEC];
  __shared__ int rok[N_DEC];
  __shared__ uint32_t rrnti[N_DEC];
  const int tid = threadIdx.x, cell = blockIdx.x / N_LIST;
  const int s = (N_LIST == N_SF ? 0 : par[cell].sf0) + STEP * (int)(blockIdx.x % N_LIST);
  const PdcchCell& cc = par[cell];
  const int R = cc.R, W = 12 * R, P = cc.n_ports;
  const int n_ctrl = ctrl_symbols(cc, pc[cell], s);
  const int n_cce = cc.n_cce[n_ctrl - 1], nq = min(MAX_QUAD, 9 * n_cce);
  const float2* G = grid + cc.off + (size_t)s * cc.nw * W;
  if (tid < 2 * nq) {                            // rules 2 and 7: pair h of quadruplet j
    const int j = tid >> 1, h = tid & 1;
    const int l = cc.quad[n_ctrl - 1][j] >> 12, k0 = cc.quad[n_ctrl - 1][j] & 0xfff;
    const bool six = l == 0 || (l == 1 && P == 4) || (l == 3 && cc.cp_type == 2);
    int k[2] = {k0 + 2 * h, k0 + 2 * h + 1};
    if (six) {
      const int v = cc.n_id % 3;
      for (int o = 0, n = 0; o < 6; o++)
        if ((k0 + o) % 3 != v) {
          if (n == 2 * h) k[0] = k0 + o;
          if (n == 2 * h + 1) k[1] = k0 + o;
          n++;
        }
    }
    const float2* Y = G + (size_t)l * W;
    const double2 y0 = make_double2(Y[k[0]].x, Y[k[0]].y), y1 = make_double2(Y[k[1]].x, Y[k[1]].y);
    const int sl = (2 * s) % N_SLOT_TAB;
    const char2* rs = rs_all + (size_t)cell * N_SLOT_TAB * 3 * 2 * MAX_RB;
    const unsigned char* shift = shift_all + (size_t)cell * N_SLOT_TAB * 3 * 4;
    auto est = [&](int p, int kk) {              // ports 0 and 1 from symbol 0, ports 2 and 3 from symbol 1
      const int s3 = p < 2 ? 0 : 1, tab = sl * 3 + s3;
      return chan(G + (size_t)s3 * W, rs + tab * 2 * MAX_RB, shift[tab * 4 + p], R, kk);
    };
    double2 x0, x1;
    double g0, g1;
    if (P == 1) {
      const double2 h0 = est(0, k[0]), h1 = est(0, k[1]);
      g0 = h0.x * h0.x + h0.y * h0.y;
      g1 = h1.x * h1.x + h1.y * h1.y;
      const double2 a = cmul_d(y0, conj_d(h0)), b = cmul_d(y1, conj_d(h1));
      x0 = make_double2(a.x / g0, a.y / g0);
      x1 = make_double2(b.x / g1, b.y / g1);
    } else {
      const int pa = P == 4 ? h : 0, pb = P == 4 ? 2 + h : 1;
      const double2 a0 = est(pa, k[0]), a1 = est(pa, k[1]), b0 = est(pb, k[0]), b1 = est(pb, k[1]);
      const double2 ha = make_double2((a0.x + a1.x) / 2, (a0.y + a1.y) / 2), hb = make_double2((b0.x + b1.x) / 2, (b0.y + b1.y) / 2);
      const double g = (ha.x * ha.x + ha.y * ha.y) + (hb.x * hb.x + hb.y * hb.y);
      const double2 n0 = cmul_d(conj_d(ha), y0), m0 = cmul_d(hb, conj_d(y1));
      const double2 n1 = cmul_d(conj_d(ha), y1), m1 = cmul_d(hb, conj_d(y0));
      x0 = make_double2(M_SQRT2 * (n0.x + m0.x) / g, M_SQRT2 * (n0.y + m0.y) / g);
      x1 = make_double2(M_SQRT2 * (n1.x - m1.x) / g, M_SQRT2 * (n1.y - m1.y) / g);
      g0 = g1 = g;
    }
    const double u[4] = {M_SQRT2 * x0.x, M_SQRT2 * x0.y, M_SQRT2 * x1.x, M_SQRT2 * x1.y};
    const int b0 = 8 * j + 4 * h;
#pragma unroll
    for (int i = 0; i < 4; i++) {
      su[b0 + i] = u[i];
      sv[b0 + i] = u[i] * (i < 2 ? g0 : g1);
    }
  }
  __syncthreads();
  const int warp = tid >> 5, lane = tid & 31;
  const int cand = warp >> 1, f = warp & 1;      // candidates 0, 1: L = 8; 2 .. 5: L = 4 (rule 8)
  const int L = cand < 2 ? 8 : 4, m = cand < 2 ? cand : cand - 2, cce = L * m;
  int ok = 0;
  double q = 0;
  unsigned long long A = 0;
  uint32_t rnti = 0;
  if (m < min(cand < 2 ? 2 : 4, n_cce / L)) {    // uniform over the warp
    const int K = cc.K[f], N3 = 3 * K, E = 72 * L, size = cc.size[f];
    const uint32_t* scr = cc.scr[s % 10];
    double* d = &sg[warp][0][0];                 // first the de-rate-matched input d [3][K], then the gains in its place
    for (int x = lane; x < N3; x += 32) {        // rule 10: descramble, weigh, average the repetitions
      double acc = 0;
      int cnt = 0;
      for (int t = cc.inv[f][x]; t < E; t += N3) {
        const int b = 72 * cce + t;
        acc += (scr[b >> 5] >> (b & 31)) & 1 ? -sv[b] : sv[b];
        cnt++;
      }
      d[x] = cnt > 1 ? acc / cnt : acc;
    }
    __syncwarp();
    double dl[2][3];                             // the gain of output o at step l: sum_j (bit j of o ? -d[j][l] : d[j][l])
#pragma unroll
    for (int i = 0; i < 2; i++)
#pragma unroll
      for (int j = 0; j < 3; j++) dl[i][j] = lane + 32 * i < K ? d[j * K + lane + 32 * i] : 0.0;
    __syncwarp();
#pragma unroll
    for (int i = 0; i < 2; i++)
      if (lane + 32 * i < K)
#pragma unroll
        for (int o = 0; o < 4; o++) {
          double g = 0;
          g += (o & 1) ? -dl[i][0] : dl[i][0];
          g += (o & 2) ? -dl[i][1] : dl[i][1];
          g += dl[i][2];
          sg[warp][lane + 32 * i][o] = g;
        }
    __syncwarp();
    // exact ML tail-biting Viterbi, one start state at a time: lane owns states lane (input 0) and lane + 32 (input 1),
    // whose predecessors are p0 = 2 lane mod 64 and p0 + 1; the odd one wins only when strictly better
    const int p0 = (2 * lane) & 63, src0 = p0 & 31, src1 = src0 + 1;
    const bool from_hi = lane >= 16;
    const int o0 = conv_out(p0, 0), o1 = conv_out(p0 + 1, 0);    // input 1 flips all three outputs: o ^ 7
    const int i0 = o0 < 4 ? o0 : 7 - o0, i1 = o1 < 4 ? o1 : 7 - o1;
    const int f0 = o0 < 4 ? 0 : (int)0x80000000, f1 = o1 < 4 ? 0 : (int)0x80000000;
    double best = -INFINITY;
    int best_ss = -1, cur = 0, best_buf = 1;
    for (int ss = 0; ss < 64; ss++) {
      double mlo = lane == ss ? 0.0 : -INFINITY, mhi = lane + 32 == ss ? 0.0 : -INFINITY;
      for (int l = 0; l < K; l++) {
        const double a0l = __shfl_sync(0xffffffffu, mlo, src0), a0h = __shfl_sync(0xffffffffu, mhi, src0);
        const double a1l = __shfl_sync(0xffffffffu, mlo, src1), a1h = __shfl_sync(0xffffffffu, mhi, src1);
        const double m0 = from_hi ? a0h : a0l, m1 = from_hi ? a1h : a1l;
        const double g0 = flip_sign(sg[warp][l][i0], f0), g1 = flip_sign(sg[warp][l][i1], f1);
        const double c00 = m0 + g0, c10 = m1 + g1, c01 = m0 - g0, c11 = m1 - g1;
        const bool hi0 = c10 > c00, hi1 = c11 > c01;
        mlo = hi0 ? c10 : c00;
        mhi = hi1 ? c11 : c01;
        const unsigned bl = __ballot_sync(0xffffffffu, hi0), bh = __ballot_sync(0xffffffffu, hi1);
        if (!lane) surv[warp][cur][l] = (unsigned long long)bl | ((unsigned long long)bh << 32);
      }
      const double fin = __shfl_sync(0xffffffffu, ss < 32 ? mlo : mhi, ss & 31);
      if (fin > best) {
        best = fin;
        best_ss = ss;
        best_buf = cur;
        cur ^= 1;
      }
      __syncwarp();
    }
    int st = best_ss < 0 ? 0 : best_ss;
    for (int l = K - 1; l >= 0; l--) {
      A |= (unsigned long long)(st >> 5) << l;
      st = ((st << 1) & 63) | (int)((surv[warp][best_buf][l] >> st) & 1);
    }
    uint32_t reg = 0;                            // rule 11: CRC16, zero init, and the RNTI it is masked with
    for (int i = 0; i < size; i++) {
      const uint32_t fb = ((reg >> 15) & 1u) ^ (uint32_t)((A >> i) & 1);
      reg = (reg << 1) & 0xffffu;
      if (fb) reg ^= 0x1021u;
    }
    uint32_t mask = 0;
    for (int i = 0; i < 16; i++) mask |= (uint32_t)((A >> (size + i)) & 1) << (15 - i);
    rnti = reg ^ mask;
    const bool common = rnti == LCS_RNTI_SI || rnti == LCS_RNTI_P || (rnti >= 1 && rnti <= 60);
    if (common && (f == 1 || (A & 1))) {         // q: the decoded word re-encoded, rate-matched and scrambled
      double num = 0, den = 0;
      for (int b = lane; b < E; b += 32) {
        const int x = cc.pos[f][b % N3], j = x / K, k = x % K;
        int sr = 0;
#pragma unroll
        for (int t = 0; t < 7; t++) sr |= (int)((A >> ((k - t + K) % K)) & 1) << (6 - t);
        const int gen = j == 0 ? 0133 : (j == 1 ? 0171 : 0165), bb = 72 * cce + b;
        const int e = (__popc(gen & sr) & 1) ^ (int)((scr[bb >> 5] >> (bb & 31)) & 1);
        const double ub = su[bb];
        num += e ? -ub : ub;
        den += ub * ub;
      }
#pragma unroll
      for (int o = 16; o; o >>= 1) {             // every lane ends with the same sums
        num += __shfl_xor_sync(0xffffffffu, num, o);
        den += __shfl_xor_sync(0xffffffffu, den, o);
      }
      q = num / sqrt((double)E * den);
      ok = q >= 0.8;
    }
  }
  if (!lane) {
    rok[warp] = ok;
    rq[warp] = q;
    ra[warp] = A;
    rrnti[warp] = rnti;
  }
  __syncthreads();
  if (tid) return;
  lcs_pdcch_meas* o = out + cell;                // rule 12
  int sel[6];
  unsigned long long pay[6];
  for (int c = 0; c < 6; c++) {
    const int a = rok[2 * c], b = rok[2 * c + 1];
    sel[c] = a && b ? (rq[2 * c] >= rq[2 * c + 1] ? 0 : 1) : (a ? 0 : (b ? 1 : -1));
    pay[c] = 0;
    if (sel[c] >= 0) {
      const int w = 2 * c + sel[c], size = cc.size[sel[c]];
      for (int i = 0; i < size; i++) pay[c] = (pay[c] << 1) | ((ra[w] >> i) & 1);
    }
  }
  for (int c = 2; c < 6; c++) {
    const int p = (c - 2) / 2;                   // the L = 8 candidate holding CCEs 4 (c - 2) .. + 3
    if (sel[c] >= 0 && sel[p] == sel[c] && rrnti[2 * p + sel[p]] == rrnti[2 * c + sel[c]] && pay[p] == pay[c]) sel[c] = -1;
  }
  int n = 0;
  for (int c = 0; c < 6; c++) {
    if (sel[c] < 0) continue;
    const int w = 2 * c + sel[c];
    lcs_pdcch_dci r = {};
    r.quality = rq[w];
    r.payload = pay[c];
    r.format = sel[c] ? LCS_DCI_1C : LCS_DCI_1A;
    r.agg = c < 2 ? 8 : 4;
    r.cce = c < 2 ? 8 * c : 4 * (c - 2);
    r.rnti = rrnti[w];
    r.n_bits = cc.size[sel[c]];
    o->dci[s][n++] = r;
  }
  for (int i = n; i < LCS_PDCCH_MAX_DCI; i++) o->dci[s][i] = lcs_pdcch_dci{};
  const int nc = ctrl_symbols(cc, pc[cell], s);  // read again: nothing stays live through the decodes
  o->cfi[s] = pc[cell].cfi[s];
  o->n_ctrl[s] = nc;
  o->n_reg[s] = cc.n_reg[nc - 1];
  o->n_cce[s] = cc.n_cce[nc - 1];
  o->n_dci[s] = n;
}

// One cell's PdcchCell (rules 1-10 of lcs_pdcch.h): its control region tables for every n_ctrl, the DCI sizes,
// rate-matching positions and scrambling words.
inline PdcchCell pdcch_cell(const CellPlan& c, const lcs_cell& cell, unsigned long long off) {
  PdcchCell p = {};
  p.off = off;
  p.R = c.R;
  p.n_ports = c.n_ports;
  p.nw = c.nw;
  p.n_id = c.n_id_cell;
  p.cp_type = c.cp_type;
  p.phich_duration = cell.phich_duration;
  p.size[0] = size_1a(c.R);
  p.size[1] = size_1c(c.R);
  for (int f = 0; f < 2; f++) {
    p.K[f] = p.size[f] + 16;
    const std::vector<uint8_t> pos = ratematch_positions(p.K[f]);
    for (size_t b = 0; b < pos.size(); b++) {
      p.pos[f][b] = pos[b];
      p.inv[f][pos[b]] = (uint8_t)b;
    }
  }
  for (int n = 1; n <= n_max(c.R); n++) {
    const CtrlTable ct = control_table(c.R, c.n_ports, c.cp_type, c.n_id_cell, cell.phich_duration, cell.phich_resource, n);
    p.n_reg[n - 1] = ct.n_reg;
    p.n_cce[n - 1] = ct.n_cce;
    std::copy(ct.quad.begin(), ct.quad.end(), p.quad[n - 1]);
  }
  for (int u = 0; u < 10; u++) scrambling(c.n_id_cell, u, p.scr[u]);
  return p;
}

}  // namespace pdcch
}  // namespace lcs

