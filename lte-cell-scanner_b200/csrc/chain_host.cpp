// chain_host.cpp - host-side stages of the cell-search chain (product code).
//
// These are the small, branchy, sequential stages that follow the GPU kernels: threshold,
// peak_search, tfoec, chan_est, decode_mib, dedup.  They mirror the reference's behaviour
// (file:line cited per function) but are written independently of oracle/ - nothing here
// includes or links the oracle.
#include <algorithm>
#include <cmath>
#include <cstring>
#include <thread>

#include "chain_host.hpp"

namespace lcs {

static const double kPi = 3.14159265358979323846;
static const double kFsLte16 = 30720000.0 / 16;

static inline int fmod_floor_i(int k, int n) { return k - n * (int)std::floor((double)k / n); }

// ---------------------------------------------------------------------------------------------
// Z_th1  (src/CellSearch.cpp:500-503)
// ---------------------------------------------------------------------------------------------
void calc_z_th1(const double* sp_incoherent, uint32_t n, uint16_t n_comb_xc, uint8_t arm, double* z) {
  const double R_th1 = chi2cdf_inv(1 - std::pow(10.0, -12.0), 2.0 * n_comb_xc * (2 * arm + 1));
  const double rx_cutoff = (6 * 12 * 15e3 / 2 + 4 * 15e3) / (kFsLte16 / 2);
  for (uint32_t i = 0; i < n; i++) z[i] = R_th1 * sp_incoherent[i] / rx_cutoff / 137 / 2 / n_comb_xc / (2 * arm + 1);
}

// ---------------------------------------------------------------------------------------------
// peak_search  (src/searcher.cpp:422-510).  `single_at(t, f, idx)` fetches xc_incoherent_single.
// ---------------------------------------------------------------------------------------------
void peak_search(const double* pow_in, const int32_t* frq, const double* z_th1, const double* f_search_set,
                 double fc_requested, double fc_programmed, const std::function<float(int, int, int)>& single_at,
                 uint8_t arm, std::vector<lcs_cell>& cells) {
  std::vector<double> work(pow_in, pow_in + 3 * LCS_N_FOLD);
  const double cancel_db12 = std::pow(10.0, -12.0 / 10.0);  // udb10(-12.0), :501
  for (;;) {
    // global maximum: first maximum of each row, then first maximum over rows (:441-445)
    int best_row = 0, best_col = 0;
    double best = -INFINITY;
    for (int r = 0; r < 3; r++) {
      const double* row = &work[(size_t)r * LCS_N_FOLD];
      int c = (int)(std::max_element(row, row + LCS_N_FOLD) - row);  // max_element returns the first maximum
      if (row[c] > best) { best = row[c]; best_row = r; best_col = c; }
    }
    if (best < z_th1[best_col]) break;  // :446
    if (!(best > 0)) break;             // all-zero input: the reference's loop would never end (0 < 0 is false)
    const int fi = frq[(size_t)best_row * LCS_N_FOLD + best_col];
    // refine the index inside +-arm (:457-465).  The reference iterates with a uint16 that wraps when
    // peak_ind < arm, in which case its loop body never runs and ind stays -1; reproduce that.
    int ind = -1;
    if (best_col >= (int)arm) {
      float bp = -INFINITY;
      for (int t = best_col - arm; t <= best_col + arm; t++) {
        const int tw = t % LCS_N_FOLD;
        const float v = single_at(best_row, fi, tw);
        if (v > bp) { bp = v; ind = tw; }
      }
    }
    lcs_cell c;
    lcs_cell_init(&c);
    c.fc_requested = fc_requested;
    c.fc_programmed = fc_programmed;
    c.pss_pow = best;
    c.ind = ind;
    c.freq = f_search_set[fi];
    c.n_id_2 = best_row;
    cells.push_back(c);
    // no second peak of the same PSS within +-274 samples (:481-484)
    for (int t = -274; t <= 274; t++) work[(size_t)best_row * LCS_N_FOLD + fmod_floor_i(best_col + t, LCS_N_FOLD)] = 0;
    // (:487-497 of the reference re-tests the row just zeroed - a no-op at HEAD - so nothing to do.)
    // CRS-induced ghosts: drop everything 12 dB below this peak (:501-508)
    const double th = best * cancel_db12;
    for (double& v : work)
      if (v < th) v = 0;
  }
}

// ---------------------------------------------------------------------------------------------
// Downlink cell-specific reference signals for the n_rb_dl centre RBs (src/lte_lib.cpp:305-405).
// ---------------------------------------------------------------------------------------------
RsDl::RsDl(int n_id_cell_, int cp_type, int n_rb_dl) : n_id_cell(n_id_cell_), n_symb(cp_type == 2 ? 6 : 7), n_rb(n_rb_dl) {
  const int n_cp = cp_type == 1 ? 1 : 0;
  rs.assign((size_t)20 * 3 * 2 * n_rb, cd(0, 0));
  const double a = 1 / std::sqrt(2.0);
  for (int slot = 0; slot < 20; slot++)
    for (int s3 = 0; s3 < 3; s3++) {
      const int sym = s3 == 2 ? n_symb - 3 : s3;
      const uint32_t c_init = (1u << 10) * (7 * (slot + 1) + sym + 1) * (2 * n_id_cell + 1) + 2 * n_id_cell + n_cp;
      std::vector<uint8_t> c = lte_pn(c_init, 440);
      for (int i = 0; i < 2 * n_rb; i++) {
        const int m = 110 - n_rb + i;  // centre n_rb RBs out of N_RB_MAXDL=110
        rs[((size_t)slot * 3 + s3) * 2 * n_rb + i] = a * cd(1 - 2 * c[2 * m], 1 - 2 * c[2 * m + 1]);
      }
    }
}
const cd* RsDl::get(int slot, int sym) const {
  const int s3 = sym == 0 ? 0 : (sym == 1 ? 1 : 2);
  return &rs[((size_t)slot * 3 + s3) * 2 * n_rb];
}
int RsDl::shift(int slot, int sym, int port) const {  // src/lte_lib.cpp:327-351
  int v = 0;
  if (port == 0) v = sym == 0 ? 0 : 3;
  else if (port == 1) v = sym == 0 ? 3 : 0;
  else if (port == 2) v = 3 * (slot & 1);
  else v = 3 + 3 * (slot & 1);
  return (v + n_id_cell) % 6;
}

static inline int cn_of(int i) { return i < 36 ? i - 36 : i - 35; }  // subcarrier numbers [-36..-1, 1..36]

// ---------------------------------------------------------------------------------------------
// tfoec  (src/searcher.cpp:952-1069).  tfg/tfg_comp are row-major [n_ofdm][72].
// ---------------------------------------------------------------------------------------------
void tfoec(const lcs_cell& cell, const cd* tfg, const double* ts, int n_ofdm, double fc_requested, double fc_programmed,
           const RsDl& rs, cd* tfg_comp, double* ts_comp, lcs_cell& out) {
  const int n = rs.n_symb;
  const int n_slot = n_ofdm / n;
  // residual frequency offset from CRS pairs one slot (0.5 ms) apart (:969-989)
  cd foe = 0;
  for (int pass = 0; pass < 2; pass++) {
    const int sym = pass == 0 ? 0 : n - 3;
    for (int i = 0; i < 12; i++) {
      cd s = 0, prev = 0;
      for (int t = 0; t < n_slot; t++) {
        const int sl = t % 20;
        const cd cur = tfg[(size_t)(t * n + sym) * 72 + rs.shift(sl, sym, 0) + 6 * i] * std::conj(rs.get(sl, sym)[i]);
        if (t > 0) s += std::conj(prev) * cur;
        prev = cur;
      }
      foe += s;
    }
  }
  const double residual_f = std::arg(foe) / (2 * kPi) / 0.0005;
  const double k_res = (fc_requested - residual_f) / fc_programmed;  // :992
  for (int t = 0; t < n_ofdm; t++) {  // FOC + lateness (:997-1005)
    ts_comp[t] = k_res * ts[t];
    const double ph = 2 * kPi * -residual_f * ts_comp[t] / kFsLte16;
    const cd rot(std::cos(ph), std::sin(ph));
    const double late = ts[t] - ts_comp[t];
    // lateness ramp e^{-j 2 pi late cn / 128}, cn = -36..-1, 1..36: one sincos per symbol, the other 35 powers by
    // repeated multiplication (error growth ~4e-15, against a 72-fold sincos cost), negative cn by conjugation
    const double a1 = -2 * kPi * late / 128;
    const cd step(std::cos(a1), std::sin(a1));
    cd pw[37];
    pw[1] = step;
    for (int c = 2; c <= 36; c++) pw[c] = pw[c - 1] * step;
    for (int i = 0; i < 72; i++) {
      const int cn = cn_of(i);
      tfg_comp[(size_t)t * 72 + i] = (tfg[(size_t)t * 72 + i] * rot) * (cn > 0 ? pw[cn] : std::conj(pw[-cn]));
    }
  }
  // time offset from CRS on subcarriers k and k+3 of adjacent RS symbols (:1012-1058)
  cd toe = 0;
  for (int t = 0; t < 2 * n_slot - 1; t++) {
    int sym[2], slot[2], row[2], sh[2];
    for (int q = 0; q < 2; q++) {
      const int tt = t + q;
      sym[q] = (tt & 1) ? n - 3 : 0;
      slot[q] = (tt >> 1) % 20;
      row[q] = (tt >> 1) * n + sym[q];
      sh[q] = rs.shift(0, sym[q], 0);
    }
    const int lo = sh[0] < sh[1] ? 0 : 1, hi = 1 - lo;  // r1 = the symbol with the smaller shift
    cd r1[12], r2[12];
    for (int i = 0; i < 12; i++) {
      r1[i] = tfg_comp[(size_t)row[lo] * 72 + sh[lo] + 6 * i] * std::conj(rs.get(slot[lo], sym[lo])[i]);
      r2[i] = tfg_comp[(size_t)row[hi] * 72 + sh[hi] + 6 * i] * std::conj(rs.get(slot[hi], sym[hi])[i]);
    }
    cd a = 0, b = 0;
    for (int i = 0; i < 12; i++) a += std::conj(r1[i]) * r2[i];
    for (int i = 0; i < 11; i++) b += std::conj(r2[i]) * r1[i + 1];
    toe += a + b;
  }
  const double delay = -std::arg(toe) / 3 / (2 * kPi / 128);
  cd comp[72];
  for (int i = 0; i < 72; i++) {
    const double a = 2 * kPi / 128 * delay * cn_of(i);
    comp[i] = cd(std::cos(a), std::sin(a));
  }
  for (int t = 0; t < n_ofdm; t++)
    for (int i = 0; i < 72; i++) tfg_comp[(size_t)t * 72 + i] *= comp[i];
  out = cell;
  out.freq_superfine = cell.freq_fine + residual_f;  // :1067
}

// ---------------------------------------------------------------------------------------------
// chan_est  (src/searcher.cpp:1369-1477) with the hexagonal planar interpolation of :1223-1362.
// ---------------------------------------------------------------------------------------------
namespace {
struct Vtx { double x, y; cd v; };

// one RS row padded so that it has vertices at subcarriers 0 and 71 (:1200-1213)
void padded_row(int shift, const cd* vals, std::vector<double>& x, std::vector<cd>& v) {
  x.clear(); v.clear();
  for (int i = 0; i < 12; i++) { x.push_back(shift + 6 * i); v.push_back(vals[i]); }
  if (x.front() != 0) {
    const cd e = v[0] - x[0] * (v[1] - v[0]) / (x[1] - x[0]);
    x.insert(x.begin(), 0.0);
    v.insert(v.begin(), e);
  }
  if (x.back() != 71) {
    const size_t L = v.size();
    const cd e = v[L - 1] + (71 - x[L - 1]) * (v[L - 1] - v[L - 2]) / (x[L - 1] - x[L - 2]);
    x.push_back(71.0);
    v.push_back(e);
  }
}
cd lerp_row(const std::vector<double>& X, const std::vector<cd>& Y, double x) {  // include/dsp.h:152-185
  size_t l = 0, r = X.size() - 1;
  while (r - l > 1) {
    const size_t mid = (size_t)std::rint((r + l) / 2.0);
    if (x >= X[mid]) l = mid; else r = mid;
  }
  return Y[l] + (x - X[l]) * (Y[r] - Y[l]) / (X[r] - X[l]);
}
}  // namespace

void chan_est(const RsDl& rs, const cd* tfg, int n_ofdm, int port, std::vector<cd>& ce, double& np) {
  const int n = rs.n_symb;
  std::vector<int> rows;  // OFDM symbols carrying RS for this port (:1383-1392)
  if (port <= 1) {
    for (int s = 0; s < n_ofdm; s++)
      if (s % n == 0 || s % n == n - 3) rows.push_back(s);
  } else {
    for (int s = 1; s < n_ofdm; s += n) rows.push_back(s);
  }
  const int nr = (int)rows.size();
  std::vector<cd> raw((size_t)nr * 12), filt((size_t)nr * 12);
  int shift2[2] = {-1000, -1000};
  {  // raw LS estimates (:1401-1419)
    int slot = 0;
    for (int t = 0; t < nr; t++) {
      const int sym = rows[t] % n;
      const int sh = rs.shift(slot % 20, sym, port);
      if (t <= 1) shift2[t] = sh;
      const cd* r = rs.get(slot, sym);
      for (int i = 0; i < 12; i++) raw[(size_t)t * 12 + i] = tfg[(size_t)rows[t] * 72 + sh + 6 * i] * std::conj(r[i]);
      if ((t & 1) || port >= 2) slot = (slot + 1) % 20;
    }
  }
  {  // 7-point hexagonal neighbourhood mean (:1421-1467)
    bool leftmost = shift2[0] < shift2[1];
    for (int t = 0; t < nr; t++) {
      for (int k = 0; k < 12; k++) {
        cd tot = 0;
        int cnt = 0;
        for (int i = std::max(0, k - 1); i <= std::min(11, k + 1); i++) { tot += raw[(size_t)t * 12 + i]; cnt++; }
        int lo = k - 1, hi = k + 1;
        if (shift2[0] != shift2[1]) { if (leftmost) hi = k; else lo = k; }
        lo = std::max(lo, 0);
        hi = std::min(hi, 11);
        for (int dt = -1; dt <= 1; dt += 2) {
          const int tt = t + dt;
          if (tt < 0 || tt >= nr) continue;
          cd s = 0;
          for (int i = lo; i <= hi; i++) { s += raw[(size_t)tt * 12 + i]; cnt++; }
          tot += s;
        }
        filt[(size_t)t * 12 + k] = tot / (double)cnt;
      }
      leftmost = !leftmost;
    }
  }
  {  // noise power (:1470)
    double acc = 0;
    for (int k = 0; k < 12; k++)
      for (int t = 0; t < nr; t++) acc += std::norm(filt[(size_t)t * 12 + k] - raw[(size_t)t * 12 + k]);
    np = acc / ((double)nr * 12);
  }
  // planar interpolation over the strip of triangles between consecutive RS rows (:1223-1362)
  ce.assign((size_t)n_ofdm * 72, cd(0, 0));
  std::vector<double> xt, xb;
  std::vector<cd> vt, vb;
  for (int t = 0; t + 1 < nr; t++) {
    padded_row((t & 1) ? shift2[1] : shift2[0], &filt[(size_t)t * 12], xt, vt);
    padded_row((t & 1) ? shift2[0] : shift2[1], &filt[(size_t)(t + 1) * 12], xb, vb);
    const double yt = rows[t], yb = rows[t + 1];
    if (t == 0)
      for (int x = 0; x < 72; x++) ce[(size_t)rows[0] * 72 + x] = lerp_row(xt, vt, x);
    // vertices alternate between the two rows, starting with the row whose 2nd vertex is further left
    std::vector<Vtx> seq;
    {
      size_t it = 0, ib = 0;
      bool top = xt[1] < xb[1];
      while (it < xt.size() || ib < xb.size()) {
        if (top && it < xt.size()) seq.push_back({xt[it], yt, vt[it]}), it++;
        else if (!top && ib < xb.size()) seq.push_back({xb[ib], yb, vb[ib]}), ib++;
        else break;
        top = !top;
      }
    }
    const int spacing = rows[t + 1] - rows[t];
    std::vector<int> next_x(spacing + 1, 0);
    for (size_t k = 0; k + 2 < seq.size(); k++) {
      const Vtx &A = seq[k], &B = seq[k + 1], &C = seq[k + 2];
      // plane through A,B,C:  v = a*x + b*y + c   (Cramer's rule on the real 3x3 system)
      const double det = A.x * (B.y - C.y) - A.y * (B.x - C.x) + (B.x * C.y - C.x * B.y);
      const cd a = (A.v * (B.y - C.y) - A.y * (B.v - C.v) + (B.v * C.y - C.v * B.y)) / det;
      const cd b = (A.x * (B.v - C.v) - A.v * (B.x - C.x) + (B.x * C.v - C.x * B.v)) / det;
      const cd c = (A.x * (B.y * C.v - C.y * B.v) - A.y * (B.x * C.v - C.x * B.v) + A.v * (B.x * C.y - C.x * B.y)) / det;
      // right edge of the triangle: x = al*y + bl through B and C (:1317-1322)
      const double al = (B.x - C.x) / (B.y - C.y), bl = (B.y * C.x - C.y * B.x) / (B.y - C.y);
      for (int r = 1; r <= spacing; r++) {
        const double y = yt + r;
        while (next_x[r] < 72 && next_x[r] <= al * y + bl) {
          ce[(size_t)(rows[t] + r) * 72 + next_x[r]] = a * (double)next_x[r] + b * y + c;
          next_x[r]++;
        }
      }
      if (next_x[1] == 72 && next_x[spacing] == 72) break;
    }
  }
  for (int t = 0; t < rows[0]; t++) std::copy(&ce[(size_t)rows[0] * 72], &ce[(size_t)rows[0] * 72] + 72, &ce[(size_t)t * 72]);
  for (int t = rows.back() + 1; t < n_ofdm; t++)
    std::copy(&ce[(size_t)rows.back() * 72], &ce[(size_t)rows.back() * 72] + 72, &ce[(size_t)t * 72]);
}

// ---------------------------------------------------------------------------------------------
// PBCH channel decoding helpers (src/lte_lib.cpp:409-663)
// ---------------------------------------------------------------------------------------------
namespace {
const int kGen[3] = {0133, 0171, 0165};
inline int par(int x) { return __builtin_parity((unsigned)x); }

// exact maximum-likelihood tail-biting Viterbi: best path over all 64 (start==end) states.
// llr > 0 means bit 0 (lte_lib.cpp:465-468, 535-537).
// The 64 constrained decodes (one per start state) are independent: their path metrics are kept side by side,
// m[state][start], so that the add-compare-select of one trellis branch is a 64-wide element-wise operation the compiler
// vectorises (AVX2 / AVX-512 clones are selected at load time).  Every metric is the same sequence of double additions
// and every decision the same strict comparison as in a start-state-at-a-time decoder, so the decoded bits are identical.
#if defined(__x86_64__) && defined(__GNUC__) && !defined(__CUDACC__)
#define LCS_SIMD_CLONES __attribute__((target_clones("avx512f", "avx2", "default")))
#else
#define LCS_SIMD_CLONES
#endif
LCS_SIMD_CLONES
void viterbi_tailbite(const double* llr /*[3][40]*/, uint8_t* bits /*[40]*/) {
  constexpr int L = 40, S = 64;
  int out[64][2];
  for (int s = 0; s < S; s++)
    for (int b = 0; b < 2; b++) {
      const int reg = (b << 6) | s;
      out[s][b] = par(kGen[0] & reg) | (par(kGen[1] & reg) << 1) | (par(kGen[2] & reg) << 2);
    }
  double gain[40][8];  // correlation of each 3-bit output with the LLRs (to maximise)
  for (int l = 0; l < L; l++)
    for (int o = 0; o < 8; o++) {
      double g = 0;
      for (int j = 0; j < 3; j++) g += ((o >> j) & 1) ? -llr[j * L + l] : llr[j * L + l];
      gain[l][o] = g;
    }
  alignas(64) static thread_local double ma[64][64], mb[64][64];
  alignas(64) static thread_local uint8_t dec[40][64][64];   // [step][state][start]: 1 = the odd predecessor won
  double (*m)[64] = ma, (*m2)[64] = mb;
  for (int s = 0; s < S; s++)
    for (int s0 = 0; s0 < S; s0++) m[s][s0] = s == s0 ? 0.0 : -INFINITY;
  for (int l = 0; l < L; l++) {
    for (int ns = 0; ns < S; ns++) {
      const int b = ns >> 5;                       // input bit that leads into ns
      const int p0 = (ns << 1) & 63, p1 = p0 | 1;  // predecessors: (reg>>1)==ns
      const double g0 = gain[l][out[p0][b]], g1 = gain[l][out[p1][b]];
      const double* __restrict__ a0 = m[p0];
      const double* __restrict__ a1 = m[p1];
      double* __restrict__ o = m2[ns];
      uint8_t* __restrict__ d = dec[l][ns];
      for (int s0 = 0; s0 < S; s0++) {
        const double c0 = a0[s0] + g0, c1 = a1[s0] + g1;
        const bool hi = c1 > c0;
        o[s0] = hi ? c1 : c0;
        d[s0] = (uint8_t)hi;
      }
    }
    std::swap(m, m2);
  }
  double best = -INFINITY;
  int best_s0 = -1;
  for (int s0 = 0; s0 < S; s0++)
    if (m[s0][s0] > best) { best = m[s0][s0]; best_s0 = s0; }
  if (best_s0 < 0) best_s0 = 0;     // all metrics NaN / -inf: the start-state-at-a-time decoder would leave `bits` untouched
  int s = best_s0;
  for (int l = L - 1; l >= 0; l--) {
    bits[l] = (uint8_t)(s >> 5);
    s = ((s << 1) & 63) | (int)dec[l][s][best_s0];
  }
}

void crc16(const uint8_t* a, int n, uint8_t* p) {  // x^16+x^12+x^5+1, zero init (lte_lib.cpp:637-663)
  unsigned reg = 0;
  for (int i = 0; i < n; i++) {
    const unsigned fb = ((reg >> 15) & 1u) ^ (a[i] & 1u);
    reg = (reg << 1) & 0xffffu;
    if (fb) reg ^= 0x1021u;
  }
  for (int i = 0; i < 16; i++) p[i] = (reg >> (15 - i)) & 1u;
}
}  // namespace

// position of every rate-matched bit e[k] in the 3 x 40 coded block (36.212 5.1.4.2; lte_lib.cpp:409-463)
void pbch_ratematch_positions(int n_e, std::vector<int>& pos) {
  static const int perm[32] = {1,17,9,25,5,21,13,29,3,19,11,27,7,23,15,31,0,16,8,24,4,20,12,28,2,18,10,26,6,22,14,30};
  const int D = 40, C = 32, R = 2, K = R * C, ND = K - D;
  std::vector<int> w;  // circular buffer of d positions, -1 = <NULL>
  for (int s = 0; s < 3; s++)
    for (int col = 0; col < C; col++)
      for (int r = 0; r < R; r++) {
        const int y = r * C + perm[col];
        w.push_back(y < ND ? -1 : s * D + (y - ND));
      }
  pos.clear();
  for (size_t j = 0; (int)pos.size() < n_e; j = (j + 1) % w.size())
    if (w[j] >= 0) pos.push_back(w[j]);
}


// ---------------------------------------------------------------------------------------------
// decode_mib  (src/searcher.cpp:1526-1692).  tfg row-major [n_ofdm][72].
// ---------------------------------------------------------------------------------------------
void decode_mib(const lcs_cell& cell, const cd* tfg, int n_ofdm, const RsDl& rs, lcs_cell& out) {
  out = cell;
  const int n = rs.n_symb;
  const int n_id_cell = cell.n_id_2 + 3 * cell.n_id_1;
  // channel estimates of the four candidate antenna ports: independent, one thread each
  std::vector<cd> ce[4];
  double npv[4];
  {
    std::thread th[3];
    for (int p = 1; p < 4; p++) th[p - 1] = std::thread([&, p] { chan_est(rs, tfg, n_ofdm, p, ce[p], npv[p]); });
    chan_est(rs, tfg, n_ofdm, 0, ce[0], npv[0]);
    for (auto& t : th) t.join();
  }
  const int n_sym = cell.cp_type == 1 ? 960 : 864;
  const std::vector<uint8_t> scr = lte_pn((uint32_t)n_id_cell, 2 * n_sym);
  std::vector<int> pos;
  pbch_ratematch_positions(2 * n_sym, pos);
  std::vector<cd> y(n_sym), h[4];
  for (auto& v : h) v.resize(n_sym);
  std::vector<double> llr(2 * n_sym);
  // The reference tries 4 frame-timing guesses x {1, 2, 4} ports in this order and stops at the first CRC match
  // (:1560-1640).  The soft bits of all 12 attempts are prepared first, the 12 tail-biting decodes (the expensive part) run
  // on parallel threads, and the first attempt IN THE REFERENCE'S ORDER whose CRC matches is taken: same result.
  struct Attempt { double d[120]; uint8_t c[40]; bool ok; int guess, n_ports; };
  std::vector<Attempt> att;
  att.reserve(12);
  for (int guess = 0; guess < 4; guess++) {
    // PBCH resource elements of 4 consecutive frames (:1482-1522)
    int q = 0;
    for (int fr = 0; fr < 4; fr++)
      for (int sym = 0; sym < 4; sym++) {
        const int row = guess * 20 * n + fr * 20 * n + n + sym;
        const bool has_rs = sym == 0 || sym == 1 || (sym == 3 && n == 6);
        for (int sc = 0; sc < 72; sc++) {
          if (has_rs && (sc % 3 == n_id_cell % 3)) continue;
          y[q] = tfg[(size_t)row * 72 + sc];
          for (int p = 0; p < 4; p++) h[p][q] = ce[p][(size_t)row * 72 + sc];
          q++;
        }
      }
    for (int n_ports : {1, 2, 4}) {
      // equalise + per-symbol noise power (:1571-1612), then QPSK LLRs (lte_lib.cpp:612-634:
      // exact log-MAP of the Gray-mapped QPSK reduces to 2*sqrt(2)*Re/Im(sym)/np)
      if (n_ports == 1) {
        for (int t = 0; t < n_sym; t++) {
          const cd g = std::conj(h[0][t] / std::norm(h[0][t]));
          const cd s = y[t] * g;
          const double np = npv[0] * std::norm(g);
          llr[2 * t] = 2 * std::sqrt(2.0) * s.real() / np;
          llr[2 * t + 1] = 2 * std::sqrt(2.0) * s.imag() / np;
        }
      } else {
        for (int t = 0; t < n_sym; t += 2) {
          int pa = 0, pb = 1;
          if (n_ports == 4) { if (t % 4 == 0) { pa = 0; pb = 2; } else { pa = 1; pb = 3; } }
          const cd h1 = (h[pa][t] + h[pa][t + 1]) / 2.0, h2 = (h[pb][t] + h[pb][t + 1]) / 2.0;
          const double npt = (npv[pa] + npv[pb]) / 2;
          const double scale = std::norm(h1) + std::norm(h2);
          const cd s0 = (std::conj(h1) * y[t] + h2 * std::conj(y[t + 1])) / scale * std::sqrt(2.0);
          const cd s1 = std::conj((-std::conj(h2) * y[t] + h1 * std::conj(y[t + 1])) / scale) * std::sqrt(2.0);
          const double np = (std::norm(h1) + std::norm(h2)) / (scale * scale) * npt;
          llr[2 * t] = 2 * std::sqrt(2.0) * s0.real() / np;
          llr[2 * t + 1] = 2 * std::sqrt(2.0) * s0.imag() / np;
          llr[2 * t + 2] = 2 * std::sqrt(2.0) * s1.real() / np;
          llr[2 * t + 3] = 2 * std::sqrt(2.0) * s1.imag() / np;
        }
      }
      // descramble, undo rate matching (average the 16 repetitions) (:1617-1630)
      Attempt a;
      a.guess = guess;
      a.n_ports = n_ports;
      a.ok = false;
      int cnt[120] = {0};
      for (int i = 0; i < 120; i++) a.d[i] = 0;
      for (int k = 0; k < 2 * n_sym; k++) {
        a.d[pos[k]] += scr[k] ? -llr[k] : llr[k];
        cnt[pos[k]]++;
      }
      for (int i = 0; i < 120; i++)
        if (cnt[i] > 1) a.d[i] /= cnt[i];
      att.push_back(a);
    }
  }
  auto decode = [](Attempt& a) {   // Viterbi + CRC with the port-count mask (:1631-1636)
    uint8_t crc[16];
    viterbi_tailbite(a.d, a.c);
    crc16(a.c, 24, crc);
    if (a.n_ports == 2) for (int i = 0; i < 16; i++) crc[i] ^= 1;
    if (a.n_ports == 4) for (int i = 1; i < 16; i += 2) crc[i] ^= 1;
    a.ok = std::memcmp(crc, a.c + 24, 16) == 0;
  };
  {
    std::vector<std::thread> th;
    for (size_t i = 1; i < att.size(); i++) th.emplace_back([&, i] { decode(att[i]); });
    decode(att[0]);
    for (auto& t : th) t.join();
  }
  for (const Attempt& a : att) {
    if (!a.ok) continue;
    const uint8_t* c = a.c;
    out.n_ports = a.n_ports;
    static const int bw[6] = {6, 15, 25, 50, 75, 100};
    const int bwi = c[0] * 4 + c[1] * 2 + c[2];
    if (bwi < 6) out.n_rb_dl = bw[bwi];
    out.phich_duration = c[3] ? 2 : 1;
    out.phich_resource = 1 + c[4] * 2 + c[5];
    int sfn8 = 0;
    for (int i = 0; i < 8; i++) sfn8 = (sfn8 << 1) | c[6 + i];
    out.sfn = fmod_floor_i(sfn8 * 4 - a.guess, 1024);  // :1684-1685 (int8 wrap is a multiple of 1024 after *4)
    return;
  }
}

// ---------------------------------------------------------------------------------------------
// dedup  (src/CellSearch.cpp:285-319)
// ---------------------------------------------------------------------------------------------
void dedup(const lcs_cell* cells, uint32_t n, std::vector<lcs_cell>& fin) {
  fin.clear();
  auto id = [](const lcs_cell& c) { return (c.n_id_1 >= 0 && c.n_id_2 >= 0) ? c.n_id_2 + 3 * c.n_id_1 : -1; };
  for (uint32_t i = 0; i < n; i++) {
    const lcs_cell& c = cells[i];
    bool match = false;
    for (lcs_cell& f : fin) {
      if (id(c) == id(f) && std::fabs((c.fc_requested + c.freq_superfine) - (f.fc_requested + f.freq_superfine)) < 1e6) {
        match = true;
        if (c.pss_pow > f.pss_pow) f = c;
        break;
      }
    }
    if (!match) fin.push_back(c);
  }
}

std::vector<double> f_search_set_for(double freq_start, double ppm) {  // src/CellSearch.cpp:463-464
  const int n_extra = (int)(uint16_t)std::floor((freq_start * ppm / 1e6 + 2.5e3) / 5e3);
  std::vector<double> f;
  for (int i = -n_extra; i <= n_extra; i++) f.push_back(5000.0 * i);
  return f;
}

}  // namespace lcs
