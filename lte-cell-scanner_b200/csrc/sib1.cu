// sib1.cu - SIB1 of found cells, decoded from the PDSCH their SI-RNTI DCIs schedule over the whole carrier, from the
// wideband recording they were found in (DESIGN.md section 4.14; contract in include/lcs_sib1.h).  Built into
// liblcs_sib1.so.
//
// A call is cut into chunks of LCS_SIB1_CHUNK cells; each chunk makes five launches on the context's stream:
//   1. carrier_grid_kernel (carrier_grid.cuh) on plan_pdcch's windows, then all symbols of the 3 occasions
//      (sib1_plan.cpp).
//   2. pcfich_kernel (pcfich_kernel.cuh), unchanged: the CFI of every subframe.
//   3. pdcch_kernel (pdcch_kernel.cuh) on the 3 occasion subframes only.
//   4. pdsch_kernel: one CTA per (cell, occasion).  It picks the SI-RNTI DCI, resolves the allocation and transport block
//      (rules 2-4), counts the data REs of each (symbol, PRB) (rule 5), equalises and descrambles them into the soft bits
//      v (rule 6, a global scratch), and de-rate-matches v into the soft inputs d [3][K + 4] (rule 7).
//   5. turbo_kernel: one CTA per (cell, occasion), thread (w, s) the state s of trellis window w (rule 8): the windows
//      run in parallel, state metrics move between the 8 lanes of a window by shuffles, the forward metrics of every
//      step stay in shared memory for the backward pass.  It iterates, checks CRC24A and packs the transport block.
// The host then parses SIB1 from the first occasion that passed its CRC (rules 9-10).
#include "../../include/lcs_sib1.h"
#include "pdcch_kernel.cuh"
#include "sib1_plan.hpp"
#include "sib1_rules.hpp"

#include <cstring>

namespace lcs {
namespace sib1 {

using namespace lcs::carrier;
using pcfich::chan;
using pcfich::cmul_d;
using pcfich::conj_d;
constexpr int N_OCC = LCS_SIB1_OCCASIONS;
constexpr uint32_t CHUNK = LCS_SIB1_CHUNK;
constexpr int PX_THREADS = 512;
constexpr int MAX_SYM = 14;                      // data symbols of a subframe at most
constexpr int MAX_ENT = MAX_SYM * MAX_RB;        // (symbol, PRB) entries at most
constexpr int V_STRIDE = 2 * 12 * MAX_RB * MAX_SYM;   // soft bits of an occasion at most
constexpr int D_STRIDE = 3 * (MAX_K + 4);
constexpr int WIN = 32;                          // trellis steps per window
constexpr int MAX_WIN = (MAX_K + WIN - 1) / WIN;
constexpr int TB_THREADS = (8 * MAX_WIN + 31) / 32 * 32;   // whole warps: the shuffles use the full mask
constexpr int MAX_ITER = 8;
static_assert(32 * SCR_WORDS >= V_STRIDE, "scrambling bits for the largest allocation");
static_assert(TB_THREADS <= 1024, "one thread per (window, state)");

struct Sib1Cell {
  unsigned long long occ_off[N_OCC];             // grid row of symbol 0 of each occasion
  int R, n_ports, n_id, n_symb, sfn;
  int sf[N_OCC];
};

// Rule 5: whether column k of subframe symbol l is a data RE (in an allocated PRB) of grid subframe s.
__device__ __forceinline__ bool data_re(const Sib1Cell& cc, const unsigned char* shift, int s, int l, int k) {
  const int n_symb = cc.n_symb, sl = l / n_symb, ls = l % n_symb, tab = ((2 * s + sl) % N_SLOT_TAB) * 3;
  const int P = cc.n_ports;
  if (ls == 0 || ls == n_symb - 3) {
    const int s3 = ls == 0 ? 0 : 2;
    for (int p = 0; p < min(P, 2); p++)
      if ((k - shift[(tab + s3) * 4 + p] + 6) % 6 == 0) return false;
  }
  if (ls == 1 && P == 4)
    for (int p = 2; p < 4; p++)
      if ((k - shift[(tab + 1) * 4 + p] + 6) % 6 == 0) return false;
  if (sl == 0 && ls >= n_symb - 2 && k >= 6 * cc.R - 36 && k < 6 * cc.R + 36) return false;
  return true;
}

// Rule 6: port p's estimate at column k in subframe symbol l of the occasion whose symbol 0 is grid row G.
__device__ double2 port_h(const Sib1Cell& cc, const float2* G, const char2* rs, const unsigned char* shift, int s, int p,
                          int l, int k) {
  const int n = cc.n_symb, W = 12 * cc.R;
  int ls[4], m;
  if (p < 2) {
    ls[0] = 0, ls[1] = n - 3, ls[2] = n, ls[3] = 2 * n - 3, m = 4;
  } else {
    ls[0] = 1, ls[1] = n + 1, m = 2;
  }
  auto at = [&](int lc) {
    const int tab = ((2 * s + lc / n) % N_SLOT_TAB) * 3 + (lc % n == 0 ? 0 : (lc % n == 1 ? 1 : 2));
    return chan(G + (size_t)lc * W, rs + tab * 2 * MAX_RB, shift[tab * 4 + p], cc.R, k);
  };
  if (l <= ls[0]) return at(ls[0]);
  if (l >= ls[m - 1]) return at(ls[m - 1]);
  int i = 0;
  while (ls[i + 1] < l) i++;
  if (ls[i + 1] == l) return at(l);
  const double2 a = at(ls[i]), b = at(ls[i + 1]);
  const double w = (double)(l - ls[i]) / (double)(ls[i + 1] - ls[i]);
  return make_double2((1 - w) * a.x + w * b.x, (1 - w) * a.y + w * b.y);
}

// rs_all [cell][20][3][2 MAX_RB], shift_all [cell][20][3][4] as for pcfich_kernel; scr [cell][SCR_WORDS]; pd [cell] the
// PDCCH records of the occasions; v [cell * 3 + o][V_STRIDE] scratch; d [cell * 3 + o][3][K + 4] the soft inputs.
__global__ void __launch_bounds__(PX_THREADS) pdsch_kernel(const float2* __restrict__ grid, const char2* __restrict__ rs_all,
                                                           const unsigned char* __restrict__ shift_all,
                                                           const Sib1Cell* __restrict__ par, const uint32_t* __restrict__ scr_all,
                                                           const lcs_pdcch_meas* __restrict__ pd, double* __restrict__ vbuf,
                                                           double* __restrict__ dbuf, lcs_sib1_meas* out) {
  __shared__ int s_prb[2][MAX_RB];
  __shared__ int s_cnt[MAX_ENT + 1];             // REs of entry (symbol, PRB), then their first RE
  __shared__ double s_err[MAX_ENT];
  __shared__ int s_wc[PX_THREADS + 1];
  __shared__ int s_ok, s_np, s_nent;
  const int tid = threadIdx.x, cell = blockIdx.x / N_OCC, o = blockIdx.x % N_OCC;
  const Sib1Cell& cc = par[cell];
  const int R = cc.R, W = 12 * R, s = cc.sf[o], n_symb = cc.n_symb;
  lcs_sib1_occasion* rec = &out[cell].occ[o];
  const lcs_pdcch_meas& pm = pd[cell];
  const char2* rs = rs_all + (size_t)cell * N_SLOT_TAB * 3 * 2 * MAX_RB;
  const unsigned char* shift = shift_all + (size_t)cell * N_SLOT_TAB * 3 * 4;
  if (!tid) {                                    // rules 1-4
    rec->subframe = s;
    rec->sfn = (cc.sfn + s / 10) % 1024;
    rec->cfi = pm.cfi[s];
    rec->n_ctrl = pm.n_ctrl[s];
    rec->vrb_start = rec->n_vrb = -1;
    int best = -1;
    for (int i = 0; i < (int)pm.n_dci[s]; i++)
      if (pm.dci[s][i].rnti == LCS_RNTI_SI && (best < 0 || pm.dci[s][i].quality > pm.dci[s][best].quality)) best = i;
    int ok = best >= 0, np = 0;
    if (ok) {
      lcs_pdcch_dci d = pm.dci[s][best];
      pdcch::parse_dci(d, R);
      rec->dci = d;
      rec->found = 1;
      rec->format = d.format;
      int vs = -1, nv = -1, tbs = 0, gap = 0, dist = 1;
      if (d.format == LCS_DCI_1A) {
        dist = d.localized;
        vs = d.rb_start;
        nv = d.n_rb;
        tbs = d.mcs <= 26 ? tbs_1a(d.mcs, (d.tpc & 1) ? 3 : 2) : 0;
        ok = nv >= 1 && (!dist || vs + nv <= n_vrb_gap(R, 0));
      } else {
        gap = d.gap;
        const int step = R < 50 ? 2 : 4, nvp = n_vrb_gap(R, gap) / step;
        int st, len;
        ok = pdcch::riv_decode(nvp, d.riv, st, len);
        if (ok) {
          vs = st * step;
          nv = len * step;
        }
        tbs = tbs_1c(d.tbs_index);
      }
      rec->distributed = dist;
      rec->gap = gap;
      ok = ok && tbs > 0;
      if (ok) {
        rec->vrb_start = vs;
        rec->n_vrb = nv;
        np = nv;
        for (int ns = 0; ns < 2; ns++) {
          for (int i = 0; i < nv; i++) {          // insertion sort: at most 100 PRBs
            int p = dist ? vrb_to_prb(R, gap, vs + i, ns) : vs + i, j = i;
            while (j > 0 && s_prb[ns][j - 1] > p) {
              s_prb[ns][j] = s_prb[ns][j - 1];
              j--;
            }
            s_prb[ns][j] = p;
          }
          for (int i = 0; i < nv; i++) rec->prb[ns][i] = (uint8_t)s_prb[ns][i];
        }
        rec->n_prb = nv;
        const int K = k_plus(tbs + 24);
        rec->tbs = tbs;
        rec->K = K;
        rec->F = K - tbs - 24;
        rec->rv = sib1_rv((int)rec->sfn);
      }
    }
    s_ok = ok;
    s_np = np;
    s_nent = (2 * n_symb - (int)pm.n_ctrl[s]) * np;
  }
  __syncthreads();
  if (!s_ok) return;
  const int np = s_np, n_ent = s_nent, n_ctrl = (int)pm.n_ctrl[s], P = cc.n_ports;
  for (int e = tid; e < n_ent; e += PX_THREADS) {   // rule 5: the REs of each (symbol, PRB)
    const int l = n_ctrl + e / np, prb = s_prb[l / n_symb][e % np];
    int n = 0;
    for (int i = 0; i < 12; i++) n += data_re(cc, shift, s, l, 12 * prb + i);
    s_cnt[e] = n;
  }
  __syncthreads();
  if (!tid) {
    int acc = 0;
    for (int e = 0; e < n_ent; e++) {
      const int n = s_cnt[e];
      s_cnt[e] = acc;
      acc += n;
    }
    s_cnt[n_ent] = acc;
    rec->n_re = acc;
  }
  __syncthreads();
  const int n_re = s_cnt[n_ent], E = 2 * n_re;
  const float2* G = grid + cc.occ_off[o];
  const uint32_t* scr = scr_all + (size_t)cell * SCR_WORDS;
  double* v = vbuf + (size_t)blockIdx.x * V_STRIDE;
  for (int e = tid; e < n_ent; e += PX_THREADS) {   // rule 6, pair by pair
    const int l = n_ctrl + e / np, prb = s_prb[l / n_symb][e % np];
    int k[12], n = 0;
    for (int i = 0; i < 12; i++)
      if (data_re(cc, shift, s, l, 12 * prb + i)) k[n++] = 12 * prb + i;
    const float2* Y = G + (size_t)l * W;
    double err = 0;
    for (int j = 0; j < n; j += 2) {
      const int r = s_cnt[e] + j;                 // the pair's first RE in mapping order
      const double2 y0 = make_double2(Y[k[j]].x, Y[k[j]].y), y1 = make_double2(Y[k[j + 1]].x, Y[k[j + 1]].y);
      double2 x0, x1;
      double g0, g1;
      if (P == 1) {
        const double2 h0 = port_h(cc, G, rs, shift, s, 0, l, k[j]), h1 = port_h(cc, G, rs, shift, s, 0, l, k[j + 1]);
        g0 = h0.x * h0.x + h0.y * h0.y;
        g1 = h1.x * h1.x + h1.y * h1.y;
        const double2 a = cmul_d(y0, conj_d(h0)), b = cmul_d(y1, conj_d(h1));
        x0 = make_double2(a.x / g0, a.y / g0);
        x1 = make_double2(b.x / g1, b.y / g1);
      } else {
        const int odd = (r / 2) & 1, pa = P == 4 ? odd : 0, pb = P == 4 ? 2 + odd : 1;
        const double2 a0 = port_h(cc, G, rs, shift, s, pa, l, k[j]), a1 = port_h(cc, G, rs, shift, s, pa, l, k[j + 1]);
        const double2 b0 = port_h(cc, G, rs, shift, s, pb, l, k[j]), b1 = port_h(cc, G, rs, shift, s, pb, l, k[j + 1]);
        const double2 ha = make_double2((a0.x + a1.x) / 2, (a0.y + a1.y) / 2), hb = make_double2((b0.x + b1.x) / 2, (b0.y + b1.y) / 2);
        const double g = (ha.x * ha.x + ha.y * ha.y) + (hb.x * hb.x + hb.y * hb.y);
        const double2 n0 = cmul_d(conj_d(ha), y0), m0 = cmul_d(hb, conj_d(y1));
        const double2 n1 = cmul_d(conj_d(ha), y1), m1 = cmul_d(hb, conj_d(y0));
        x0 = make_double2(M_SQRT2 * (n0.x + m0.x) / g, M_SQRT2 * (n0.y + m0.y) / g);
        x1 = make_double2(M_SQRT2 * (n1.x - m1.x) / g, M_SQRT2 * (n1.y - m1.y) / g);
        g0 = g1 = g;
      }
      const double u[4] = {M_SQRT2 * x0.x, M_SQRT2 * x0.y, M_SQRT2 * x1.x, M_SQRT2 * x1.y};
#pragma unroll
      for (int i = 0; i < 4; i++) {
        const int b = 2 * r + i;
        const double vb = u[i] * (i < 2 ? g0 : g1);
        v[b] = (scr[b >> 5] >> (b & 31)) & 1 ? -vb : vb;
      }
      const double2 xs[2] = {x0, x1};
#pragma unroll
      for (int i = 0; i < 2; i++) {
        const double ex = xs[i].x - (xs[i].x >= 0 ? M_SQRT1_2 : -M_SQRT1_2), ey = xs[i].y - (xs[i].y >= 0 ? M_SQRT1_2 : -M_SQRT1_2);
        err += ex * ex + ey * ey;
      }
    }
    s_err[e] = err;
  }
  __syncthreads();                               // v is complete: the block's global writes are visible to it
  if (!tid) {
    double acc = 0;
    for (int e = 0; e < n_ent; e++) acc += s_err[e];
    rec->sinr = acc > 0 ? (double)n_re / acc : INFINITY;
  }
  // rule 7: position i of the circular buffer carries e_j for j = rank(i) + m N_valid < E
  const int K = (int)rec->K, F = (int)rec->F, Dk = K + 4, kw = 96 * ((Dk + 31) / 32), k0 = k0_of(K, (int)rec->rv);
  const int ch = (kw + PX_THREADS - 1) / PX_THREADS, lo = min(kw, tid * ch), hi = min(kw, lo + ch);
  double* d = dbuf + (size_t)blockIdx.x * D_STRIDE;
  int c = 0;
  for (int i = lo; i < hi; i++) c += wbuf_pos(K, F, i) >= 0;
  s_wc[tid] = c;
  for (int k = tid; k < F; k += PX_THREADS) {
    d[k] = KNOWN_ZERO;
    d[Dk + k] = 0;
  }
  __syncthreads();
  if (!tid) {
    int acc = 0;
    for (int t = 0; t < PX_THREADS; t++) {
      const int n = s_wc[t];
      s_wc[t] = acc;
      acc += n;
    }
    s_wc[PX_THREADS] = acc;
  }
  __syncthreads();
  const int nv = s_wc[PX_THREADS];
  int pk0 = s_wc[k0 / ch];
  for (int i = (k0 / ch) * ch; i < k0; i++) pk0 += wbuf_pos(K, F, i) >= 0;
  int pc = s_wc[tid];
  for (int i = lo; i < hi; i++) {
    const int x = wbuf_pos(K, F, i);
    if (x < 0) continue;
    const int rank = i >= k0 ? pc - pk0 : nv - pk0 + pc;
    double acc = 0;
    for (int j = rank; j < E; j += nv) acc += v[j];
    d[x] = acc;
    pc++;
  }
}

// Rule 8's branch metric.
__device__ __forceinline__ double gam(int u, int z, double lsa, double lp) {
  return ((u ? -lsa : lsa) + (z ? -lp : lp)) * 0.5;
}

struct TurboSmem {
  double alpha[MAX_K][8];                        // forward metrics before each step
  double ext[2][MAX_K];                          // each decoder's scaled extrinsic, natural order
  double ab[2][MAX_WIN + 1][8];                  // each decoder's window-start forward metrics from its last pass
  double bb[2][MAX_WIN + 1][8];                  // and window-end backward metrics
  uint8_t bits[MAX_K];
  int pass;
};

__global__ void __launch_bounds__(TB_THREADS) turbo_kernel(const double* __restrict__ dbuf, lcs_sib1_meas* out) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  TurboSmem& S = *reinterpret_cast<TurboSmem*>(smem_raw);
  const int tid = threadIdx.x, cell = blockIdx.x / N_OCC, o = blockIdx.x % N_OCC;
  lcs_sib1_occasion* rec = &out[cell].occ[o];
  if (!rec->n_re) return;                        // nothing to decode (uniform over the block)
  const int K = (int)rec->K, F = (int)rec->F, Dk = K + 4, nwin = (K + WIN - 1) / WIN;
  int ki = 0;
  while (k_of(ki) != K) ki++;
  int f1, f2;
  qpp_params(ki, f1, f2);
  const double* d0 = dbuf + (size_t)blockIdx.x * D_STRIDE;
  const double *d1 = d0 + Dk, *d2 = d1 + Dk;
  const int w = tid >> 3, st = tid & 7, base = (tid & 31) & ~7;
  const bool act_w = w < nwin;
  for (int i = tid; i < 2 * (MAX_WIN + 1) * 8; i += TB_THREADS) {
    (&S.ab[0][0][0])[i] = 0;
    (&S.bb[0][0][0])[i] = 0;
  }
  for (int i = tid; i < 2 * MAX_K; i += TB_THREADS) (&S.ext[0][0])[i] = 0;
  double beta_k[2];                              // the tail's backward metrics at step K of state st
  for (int dec = 0; dec < 2; dec++) {
    const double* t = dec ? d0 + K + 2 : d0 + K;  // x, z of the 3 termination steps (36.212 5.1.3.2.2)
    const double xs[3] = {t[0], t[2 * Dk], t[Dk + 1]}, zs[3] = {t[Dk], t[1], t[2 * Dk + 1]};
    int sa = st, u[3], z[3];
    for (int j = 0; j < 3; j++) {
      const int a1 = (sa >> 2) & 1, a2 = (sa >> 1) & 1, a3 = sa & 1;
      u[j] = a2 ^ a3;
      z[j] = a1 ^ a3;
      sa = (a1 << 1) | a2;
    }
    double b = 0;
    for (int j = 2; j >= 0; j--) b = gam(u[j], z[j], xs[j], zs[j]) + b;
    beta_k[dec] = b;
  }
  __syncthreads();
  int it = 0, pass = 0;
  while (it < MAX_ITER && !pass) {
    it++;
    for (int dec = 0; dec < 2; dec++) {
      const double* lp = dec ? d2 : d1;
      const double* la_src = S.ext[1 - dec];
      auto inputs = [&](int t, double& lsa, double& lpar, double& ls, double& la) {
        const int q = dec ? qpp(K, f1, f2, t) : t;
        ls = d0[q];
        la = la_src[q];
        lsa = ls + la;
        lpar = lp[t];
      };
      double a = w == 0 ? (st == 0 ? 0.0 : -INFINITY) : (act_w ? S.ab[dec][w][st] : 0.0);
      double b = w == nwin - 1 ? beta_k[dec] : (act_w ? S.bb[dec][w][st] : 0.0);
      __syncthreads();
      const int t0 = WIN * w;
      // forward: state st as the next state; its predecessors differ in their oldest register bit
      const int n1 = (st >> 1) & 1, n2 = st & 1, na = st >> 2;
      for (int j = 0; j < WIN; j++) {
        const int t = t0 + j;
        const bool act = act_w && t < K;
        double lsa = 0, lpar = 0, ls, la;
        if (act) {
          S.alpha[t][st] = a;
          inputs(t, lsa, lpar, ls, la);
        }
        const double ap0 = __shfl_sync(0xffffffffu, a, base + ((n1 << 2) | (n2 << 1))),
                     ap1 = __shfl_sync(0xffffffffu, a, base + ((n1 << 2) | (n2 << 1) | 1));
        if (act) {
          const double c0 = ap0 + gam(na ^ n2, na ^ n1, lsa, lpar), c1 = ap1 + gam(na ^ n2 ^ 1, na ^ n1 ^ 1, lsa, lpar);
          a = fmax(c0, c1);
        }
      }
      const double a_end = a;
      // backward, with the a-posteriori LLR of each step
      const int s1 = (st >> 2) & 1, s2 = (st >> 1) & 1, s3 = st & 1;
      for (int j = WIN - 1; j >= 0; j--) {
        const int t = t0 + j;
        const bool act = act_w && t < K;
        double lsa = 0, lpar = 0, ls = 0, la = 0;
        if (act) inputs(t, lsa, lpar, ls, la);
        const int a0 = s2 ^ s3, a1 = a0 ^ 1;
        const double bn0 = __shfl_sync(0xffffffffu, b, base + ((a0 << 2) | (s1 << 1) | s2));
        const double bn1 = __shfl_sync(0xffffffffu, b, base + ((a1 << 2) | (s1 << 1) | s2));
        const double g0 = gam(0, a0 ^ s1 ^ s3, lsa, lpar) + bn0, g1 = gam(1, a1 ^ s1 ^ s3, lsa, lpar) + bn1;
        const double al = act ? S.alpha[t][st] : 0.0;
        double m0 = al + g0, m1 = al + g1;
#pragma unroll
        for (int x = 1; x < 8; x <<= 1) {
          m0 = fmax(m0, __shfl_xor_sync(0xffffffffu, m0, x));
          m1 = fmax(m1, __shfl_xor_sync(0xffffffffu, m1, x));
        }
        if (act) {
          b = fmax(g0, g1);
          if (st == 0) {
            const double lapp = m0 - m1;
            const int q = dec ? qpp(K, f1, f2, t) : t;
            S.ext[dec][q] = 0.75 * (lapp - ls - la);
            if (dec) S.bits[q] = lapp < 0;
          }
        }
      }
      __syncthreads();
      if (act_w && w + 1 < nwin) S.ab[dec][w + 1][st] = a_end;
      if (act_w && w >= 1) S.bb[dec][w - 1][st] = b;
      __syncthreads();
    }
    if (!tid) S.pass = crc24a(S.bits + F, K - F) == 0;
    __syncthreads();
    pass = S.pass;
  }
  const int tbs = (int)rec->tbs;
  for (int i = tid; i < LCS_SIB1_TB_BYTES; i += TB_THREADS) {
    uint32_t byte = 0;
    if (8 * i < tbs)
      for (int j = 0; j < 8; j++) byte = (byte << 1) | S.bits[F + 8 * i + j];
    rec->tb[i] = (uint8_t)byte;
  }
  if (!tid) {
    rec->crc_ok = pass;
    rec->iterations = it;
  }
}

}  // namespace sib1
}  // namespace lcs

using namespace lcs;
using namespace lcs::carrier;
using namespace lcs::sib1;

struct lcs_sib1 : GridModule<lcs_sib1_meas> {
  DevBuf<lcs_pcfich_meas> d_pc;                  // one chunk's CFI decisions
  DevBuf<lcs_pdcch_meas> d_pd;                   // its DCIs (the occasions' subframes only)
  DevBuf<double> d_v, d_d;                       // its soft bits and soft inputs
};

namespace {

// Rules 9-10 on the host: the cell's counts, consistency and SIB1 fields.
void finish(lcs_sib1_meas& m) {
  m.n_found = m.n_crc_ok = 0;
  bool same = true;
  int first = -1;
  for (int o = 0; o < N_OCC; o++) {
    const lcs_sib1_occasion& x = m.occ[o];
    m.n_found += x.found;
    if (!x.crc_ok) continue;
    m.n_crc_ok++;
    if (first < 0)
      first = o;
    else if (x.tbs != m.occ[first].tbs || std::memcmp(x.tb, m.occ[first].tb, LCS_SIB1_TB_BYTES) != 0)
      same = false;
  }
  m.consistent = first >= 0 && same;
  m.parse_ok = parse_sib1(first >= 0 ? m.occ[first].tb : nullptr, first >= 0 ? (int)(m.occ[first].tbs / 8) : 0, m);
}

}  // namespace

extern "C" {

lcs_status lcs_sib1_create(lcs_ctx* ctx, lcs_sib1** out) { return grid_create(ctx, out, "lcs_sib1_create"); }

void lcs_sib1_destroy(lcs_sib1* h) { grid_destroy(h); }

lcs_status lcs_sib1_cells(lcs_sib1* h, const void* iq, int iq_format, int on_device, uint64_t n_in, double fs_in,
                          double fc_in, const lcs_cell* cells, uint32_t n_cells, double fs_programmed,
                          lcs_sib1_meas* out) {
  pcfich::PcfichSlices s{};
  pdcch::PdcchCell* pd = nullptr;
  Sib1Cell* sc = nullptr;
  uint32_t* scr = nullptr;
  return grid_cells(
      h, "lcs_sib1_cells", CHUNK, LCS_SIB1_LAUNCHES_PER_CHUNK, iq, iq_format, on_device, n_in, fs_in, fc_in, cells,
      n_cells, fs_programmed, out, plan_sib1,
      [](uint32_t n) {
        return pcfich::pcfich_bytes(n) + n * sizeof(pdcch::PdcchCell) + 16 + n * sizeof(Sib1Cell) + 16 +
               (size_t)n * SCR_WORDS * sizeof(uint32_t) + 16;
      },
      [&](const GridChunk& c) {
        s = pcfich::pcfich_fill(h->g, c);
        pd = h->g.up.take<pdcch::PdcchCell>(c.n);
        sc = h->g.up.take<Sib1Cell>(c.n);
        scr = h->g.up.take<uint32_t>((size_t)c.n * SCR_WORDS);
        for (uint32_t i = 0; i < c.n; i++) {
          const CellPlan& p = c.plan[i];
          pd[i] = pdcch::pdcch_cell(p, c.cell[i], c.t.off[i]);
          Sib1Cell& x = sc[i];
          x = Sib1Cell{};
          x.R = p.R;
          x.n_ports = p.n_ports;
          x.n_id = p.n_id_cell;
          x.n_symb = p.cp_type == 1 ? 7 : 6;
          x.sfn = c.cell[i].sfn;
          occasions(x.sfn, x.sf);
          pd[i].sf0 = x.sf[0];                   // the occasions are sf0, sf0 + 20, sf0 + 40
          for (int o = 0; o < N_OCC; o++)
            x.occ_off[o] = c.t.off[i] + ((size_t)pdcch::N_SF * p.nw + (size_t)o * 2 * x.n_symb) * 12 * p.R;
          scrambling(p.n_id_cell, scr + (size_t)i * SCR_WORDS);
        }
        cudaError_t e = h->d_pc.ensure(c.n);     // the first chunk is the largest: it sizes the buffers for the call
        if (e == cudaSuccess) e = h->d_pd.ensure(c.n);
        if (e == cudaSuccess) e = h->d_v.ensure((size_t)c.n * N_OCC * V_STRIDE);
        if (e == cudaSuccess) e = h->d_d.ensure((size_t)c.n * N_OCC * D_STRIDE);
        if (e == cudaSuccess)
          e = cudaFuncSetAttribute(turbo_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(TurboSmem));
        return e;
      },
      [&](const GridChunk& c) {
        pcfich::pcfich_launch(h->g, c, s, h->d_pc.p);
        pdcch::pdcch_kernel<N_OCC, 20><<<c.n * N_OCC, pdcch::PD_THREADS, 0, c.st>>>(h->g.d_grid.p, h->g.up.dev(c.t.rs),
                                                                         h->g.up.dev(c.t.shift), h->g.up.dev(pd),
                                                                         h->d_pc.p, h->d_pd.p);
        pdsch_kernel<<<c.n * N_OCC, PX_THREADS, 0, c.st>>>(h->g.d_grid.p, h->g.up.dev(c.t.rs), h->g.up.dev(c.t.shift),
                                                           h->g.up.dev(sc), h->g.up.dev(scr), h->d_pd.p, h->d_v.p,
                                                           h->d_d.p, h->d_out.p);
        turbo_kernel<<<c.n * N_OCC, TB_THREADS, sizeof(TurboSmem), c.st>>>(h->d_d.p, h->d_out.p);
      },
      [](lcs_sib1_meas& m, const CellPlan&) { finish(m); });
}

lcs_status lcs_sib1_timing_read(lcs_sib1* h, double* kernel_ms, uint64_t* launches) {
  return grid_timing_read(h, kernel_ms, launches, "lcs_sib1_timing_read");
}

}  // extern "C"
