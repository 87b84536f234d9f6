// track.cu - the cell tracker of LTE-Tracker on the device (FP64): per-cell slicing of each channel's stream
// (src/producer_thread.cpp:163-250) and the per-cell tracker loop (src/tracker_thread.cpp:856-1067) for every cell of
// every channel, one launch per push.  The schedule is the one of DESIGN.md section 4.5.
//
// One CTA per channel walks the channel's complete blocks in order; inside a block:
//   1. thread 0 runs the time-stamp recurrence (the same double additions as lcs_framer_push) into shared memory;
//   2. one thread per cell slices the block: slice positions, `late`, the block's offset / timing snapshots and the
//      bulk phase offset (a scalar prefix over the cell's symbols);
//   3. all symbols of all cells: FOC, FFT-128, the 72 bins, late and bulk phase correction (64 threads per symbol);
//   4. one warp per cell runs the tracker loop over its symbols: warp-uniform scalar recurrences, 72-wide work split
//      over the lanes, and the tail-biting Viterbi of a MIB attempt over the warp;
//   5. thread 0 applies the FOE updates to the channel's frequency offset in cell order, then symbol order, then port
//      order.
#include <cmath>
#include <cstring>
#include <new>
#include <vector>

#include "chain_host.hpp"
#include "fft128.cuh"
#include "lcs_ctx.hpp"

namespace lcs {
namespace trk {

constexpr int BLOCK = LCS_TRACK_BLOCK;
constexpr int THREADS = 256;
constexpr int WARPS = THREADS / 32;
constexpr int GROUPS = THREADS / 64;        // FFT groups
constexpr int MAX_PDU = 80;                 // symbols one cell completes in a block (<= 10000/137 + 1)
constexpr int RING = 32;                    // data / interpolated-CE ring depth
constexpr int TAIL = 128;                   // samples of the previous block kept in front of a push
constexpr double kPi = 3.14159265358979323846;
constexpr double kFs16 = 30720000.0 / 16;

struct CeRaw { double shift, fo, ft; int slot, sym; double2 ce[12]; };
struct CeFilt { double shift, tp, sp, sp_raw, np; int slot, sym; double2 ce[12]; };
struct CeInterp { double tp, sp, sp_raw, np; int slot, sym; double2 ce[72]; };
struct DataEnt { int slot, sym; double2 syms[72]; };
struct MibEnt { double2 syms[72]; double2 ce[4][72]; double np[4]; };

struct Pdu {            // one completed symbol of the current block
  int pos;              // first sample in the launch buffer
  int slot, sym;
  double late, fo, ft, bpo;
  long long start;      // stream sample
};

struct Hdr {
  int slot, sym;
  int n_raw[4], n_filt[4], interp_init[4];
  int ih[4], in_[4];        // interpolated-CE ring head / count
  int dh, dn;               // data ring
  int mh, mn, mib_sync;     // MIB ring
  int n_foe;                // FOE updates queued in this block
  double frame_timing;
};

struct CellState {
  // configuration
  int active, n_id_cell, n_id_1, n_id_2, n_ports, cp_type, n_symb, n_rb_dl, phich_dur, phich_res;
  // slicer (cell_local_t)
  unsigned target;
  int filling, buffer_offset, pslot, psym;
  double plate, pfo, pft;
  long long pstart;
  double bpo;
  Hdr h;                    // tracker scalars (each lane of the cell's warp works on a copy)
  CeRaw raw[4][3];
  CeFilt filt[4][2];
  CeInterp interp[4][RING];
  DataEnt data[RING];
  MibEnt mib[16];
  double2 sss_sym[72];
  lcs_track_cell out;
};

struct ChanState {
  double fc_req, fc_prog, fo, sample_time;
  long long n_done;
};

struct Tables {                 // per cell: CRS values, scrambling bits, rate-matching positions
  double2 rs[20][3][12];        // [slot][sym in {0, 1, n_symb-3}][12]
  unsigned char scr[1920];
  short inv[120][16];           // rate-matched bits e[k] of each coded bit, ascending k (lte_lib.cpp:469-518)
  unsigned char n_inv[120];
  int sss[2][62];
  double2 pss[62];
};

struct Scratch {                // per cell, per block
  Pdu pdu[MAX_PDU];
  int n_pdu;
  int n_foe;
  double2 foe[MAX_PDU * 4];     // (target offset, 1/np) in processing order
  double2 sr[62], pr[62], sm[62];   // PSS/SSS channel estimates of do_pss_sss_sigpower_ce
  double2 syms[MAX_PDU][72];
  double2 y[960], h[4][960];
  double npv[4][960];
  double llr[1920];
  double d[120];
  double m[2][64][64];
  unsigned char dec[40][64][64];
};

struct Params {
  int n_ch, max_cells, n_blocks, stride;   // stride: samples per channel in the launch buffer
  double fs_prog;
  const unsigned char* iq;                 // [n_ch][stride][2]
  ChanState* ch;
  CellState* cells;                        // [n_ch][max_cells]
  const Tables* tab;
  Scratch* scr;
};

__device__ __forceinline__ double wrapd(double x, double sm, double lg) {   // macros.h:49, itpp_ext.h:40-42
  const double n = lg - sm, k = x - sm;
  return (n == 0 ? k : k - n * floor(k / n)) + sm;
}
__device__ __forceinline__ double mmod(double k, double n) { return n == 0 ? k : k - n * floor(k / n); }
__device__ __forceinline__ double2 cadd(double2 a, double2 b) { return make_double2(a.x + b.x, a.y + b.y); }
__device__ __forceinline__ double2 csub(double2 a, double2 b) { return make_double2(a.x - b.x, a.y - b.y); }
__device__ __forceinline__ double2 cscale(double2 a, double s) { return make_double2(a.x * s, a.y * s); }
__device__ __forceinline__ double2 cdiv(double2 a, double s) { return make_double2(a.x / s, a.y / s); }
__device__ __forceinline__ double2 conj2(double2 a) { return make_double2(a.x, -a.y); }
__device__ __forceinline__ double nrm(double2 a) { return a.x * a.x + a.y * a.y; }
__device__ __forceinline__ double carg(double2 a) { return atan2(a.y, a.x); }
__device__ __forceinline__ void sym_inc(int n_symb, int& slot, int& sym) {
  if (++sym == n_symb) { sym = 0; slot = (slot + 1) % 20; }
}
__device__ __forceinline__ bool has_rs(const CellState& c, int sym, int port) {
  return port < 2 ? (sym == 0 || sym == c.n_symb - 3) : sym == 1;
}
__device__ __forceinline__ int rs_shift(const CellState& c, int slot, int sym, int port) {   // lte_lib.cpp:327-351
  int v;
  if (port == 0) v = sym == 0 ? 0 : 3;
  else if (port == 1) v = sym == 0 ? 3 : 0;
  else if (port == 2) v = 3 * (slot & 1);
  else v = 3 + 3 * (slot & 1);
  return (v + c.n_id_cell) % 6;
}

// interp72 of a filtered CE at subcarrier t (tracker_thread.cpp:372-393)
__device__ double2 interp72_at(const CeFilt& rs, int t) {
  int l_x = (int)rs.shift, r_x = (int)rs.shift + 6, ptr = 1;
  double2 l_y = rs.ce[0], r_y = rs.ce[1];
  for (int u = 0; u <= t; u++)
    if (u > r_x && ptr < 11) { l_x = r_x; l_y = r_y; r_x += 6; ptr++; r_y = rs.ce[ptr]; }
  const double2 sl = cdiv(csub(r_y, l_y), (double)(r_x - l_x));
  return cadd(cscale(sl, (double)(t - l_x)), l_y);
}

// MIB attempt on the 16 queued symbols (tracker_thread.cpp:494-749), executed by one whole warp.
// Returns 1 on a CRC + MIB match.
__device__ int mib_attempt(const CellState& c, const Hdr& h, const Tables& tb, Scratch& s, int lane) {
  const int n_syms = c.cp_type == 1 ? 960 : 864, v3 = c.n_id_cell % 3, P = c.n_ports;
  // pbch_extract_rt
  for (int e = lane; e < 16 * 72; e += 32) {
    const int q = e / 72, sc = e % 72, symn = q % 4;
    int base = 0;
    for (int k = 0; k < q; k++) {
      const int sn = k % 4;
      base += (sn == 0 || sn == 1 || (sn == 3 && c.cp_type == 2)) ? 48 : 72;
    }
    const bool skip_sym = symn == 0 || symn == 1 || (symn == 3 && c.cp_type == 2);
    if (skip_sym && sc % 3 == v3) continue;
    const int idx = base + (skip_sym ? sc - (sc - v3 + 2) / 3 : sc);
    const MibEnt& m = c.mib[(h.mh + q) % 16];
    s.y[idx] = m.syms[sc];
    for (int p = 0; p < P; p++) { s.h[p][idx] = m.ce[p][sc]; s.npv[p][idx] = m.np[p]; }
  }
  __syncwarp();
  // equalisation and QPSK LLRs (lte_demodulate: 2*sqrt(2)*Re/Im / np)
  const double k2 = 2 * sqrt(2.0);
  if (P == 1) {
    for (int t = lane; t < n_syms; t += 32) {
      const double2 h = s.h[0][t];
      const double2 g = conj2(cdiv(h, nrm(h)));
      const double2 v = cmul(s.y[t], g);
      const double np = s.npv[0][t] * nrm(g);
      s.llr[2 * t] = k2 * v.x / np;
      s.llr[2 * t + 1] = k2 * v.y / np;
    }
  } else {
    for (int t = 2 * lane; t < n_syms; t += 64) {
      int pa = 0, pb = 1;
      if (P == 4) { if (t % 4 == 0) { pa = 0; pb = 2; } else { pa = 1; pb = 3; } }
      const double2 h1 = cdiv(cadd(s.h[pa][t], s.h[pa][t + 1]), 2.0), h2 = cdiv(cadd(s.h[pb][t], s.h[pb][t + 1]), 2.0);
      const double npt = (s.npv[pa][t] + s.npv[pb][t]) / 2;
      const double2 x1 = s.y[t], x2 = s.y[t + 1];
      const double scale = nrm(h1) + nrm(h2);
      const double r2 = sqrt(2.0);
      const double2 s0 = cscale(cdiv(cadd(cmul(conj2(h1), x1), cmul(h2, conj2(x2))), scale), r2);
      const double2 s1 = cscale(conj2(cdiv(cadd(cmul(make_double2(-h2.x, h2.y), x1), cmul(h1, conj2(x2))), scale)), r2);
      const double a1 = sqrt(nrm(h1)) / scale, a2 = sqrt(nrm(h2)) / scale;
      const double np = (a1 * a1 + a2 * a2) * npt;
      s.llr[2 * t] = k2 * s0.x / np;
      s.llr[2 * t + 1] = k2 * s0.y / np;
      s.llr[2 * t + 2] = k2 * s1.x / np;
      s.llr[2 * t + 3] = k2 * s1.y / np;
    }
  }
  __syncwarp();
  // descramble and undo rate matching (average the repetitions)
  for (int i = lane; i < 120; i += 32) {
    double acc = 0;
    const int cnt = tb.n_inv[i];
    for (int j = 0; j < cnt; j++) {
      const int k = tb.inv[i][j];
      acc += tb.scr[k] ? -s.llr[k] : s.llr[k];
    }
    s.d[i] = cnt > 1 ? acc / cnt : acc;
  }
  __syncwarp();
  // exact ML tail-biting Viterbi over all 64 start states (chain_host.cpp viterbi_tailbite): lane owns starts lane, lane+32
  const int G[3] = {0133, 0171, 0165};
  for (int st = lane; st < 64; st += 32)
    for (int s2 = 0; s2 < 64; s2++) s.m[0][s2][st] = s2 == st ? 0.0 : -INFINITY;
  __syncwarp();
  int cur = 0;
  for (int l = 0; l < 40; l++) {
    double gain[8];
    for (int o = 0; o < 8; o++) {
      double g = 0;
      for (int j = 0; j < 3; j++) g += ((o >> j) & 1) ? -s.d[j * 40 + l] : s.d[j * 40 + l];
      gain[o] = g;
    }
    for (int ns = 0; ns < 64; ns++) {
      const int b = ns >> 5, p0 = (ns << 1) & 63, p1 = p0 | 1;
      const int r0 = (b << 6) | p0, r1 = (b << 6) | p1;
      const int o0 = __popc(G[0] & r0) & 1 | ((__popc(G[1] & r0) & 1) << 1) | ((__popc(G[2] & r0) & 1) << 2);
      const int o1 = __popc(G[0] & r1) & 1 | ((__popc(G[1] & r1) & 1) << 1) | ((__popc(G[2] & r1) & 1) << 2);
      for (int st = lane; st < 64; st += 32) {
        const double c0 = s.m[cur][p0][st] + gain[o0], c1 = s.m[cur][p1][st] + gain[o1];
        const bool hi = c1 > c0;
        s.m[cur ^ 1][ns][st] = hi ? c1 : c0;
        s.dec[l][ns][st] = (unsigned char)hi;
      }
    }
    cur ^= 1;
    __syncwarp();
  }
  int ok = 0;
  if (lane == 0) {
    double best = -INFINITY;
    int b0 = -1;
    for (int st = 0; st < 64; st++)
      if (s.m[cur][st][st] > best) { best = s.m[cur][st][st]; b0 = st; }
    if (b0 < 0) b0 = 0;
    unsigned char bits[40];
    int st = b0;
    for (int l = 39; l >= 0; l--) {
      bits[l] = (unsigned char)(st >> 5);
      st = ((st << 1) & 63) | (int)s.dec[l][st][b0];
    }
    unsigned reg = 0;   // CRC16 x^16+x^12+x^5+1, zero init
    for (int i = 0; i < 24; i++) {
      const unsigned fb = ((reg >> 15) & 1u) ^ bits[i];
      reg = (reg << 1) & 0xffffu;
      if (fb) reg ^= 0x1021u;
    }
    unsigned char crc[16];
    for (int i = 0; i < 16; i++) crc[i] = (reg >> (15 - i)) & 1u;
    if (P == 2) for (int i = 0; i < 16; i++) crc[i] ^= 1;
    else if (P == 4) for (int i = 1; i < 16; i += 2) crc[i] ^= 1;
    bool match = true;
    for (int i = 0; i < 16; i++) match = match && crc[i] == bits[24 + i];
    const int bw[6] = {6, 15, 25, 50, 75, 100};
    const int bwi = bits[0] * 4 + bits[1] * 2 + bits[2];
    const int n_rb = bwi < 6 ? bw[bwi] : 0;
    ok = match && n_rb == c.n_rb_dl && (bits[3] ? 2 : 1) == c.phich_dur && 1 + bits[4] * 2 + bits[5] == c.phich_res;
  }
  return __shfl_sync(0xffffffffu, ok, 0);
}

// The tracker loop for one symbol (tracker_thread.cpp:870-1066), one whole warp.  Returns 1 when the cell is dropped.
__device__ int tracker_step(CellState& c, Hdr& h, const Tables& tb, Scratch& s, const ChanState& chn, double fs_prog, int k,
                            int lane) {
  const Pdu& pd = s.pdu[k];
  const double2* syms = s.syms[k];
  const int P = c.n_ports, slot = h.slot, sym = h.sym;
  // data fifo
  {
    DataEnt& d = c.data[(h.dh + h.dn) % RING];
    for (int t = lane; t < 72; t += 32) d.syms[t] = syms[t];
    if (lane == 0) { d.slot = slot; d.sym = sym; }
  }
  __syncwarp();
  h.dn++;
  // raw CRS estimates
  const int s3 = sym == 0 ? 0 : (sym == 1 ? 1 : 2);
  for (int p = 0; p < P; p++) {
    if (!has_rs(c, sym, p)) continue;
    const int sh = rs_shift(c, slot, sym, p);
    CeRaw& r = c.raw[p][h.n_raw[p]];
    if (lane < 12) r.ce[lane] = cmul(syms[sh + 6 * lane], conj2(tb.rs[slot][s3][lane]));
    if (lane == 0) { r.shift = sh; r.slot = slot; r.sym = sym; r.fo = pd.fo; r.ft = pd.ft; }
    __syncwarp();
    h.n_raw[p]++;
  }
  // filter, powers, FOE, TOE (warp-uniform scalar code)
  for (int p = 0; p < P; p++) {
    if (h.n_raw[p] != 3) continue;
    const CeRaw& rp = c.raw[p][0];
    const CeRaw& rc = c.raw[p][1];
    const CeRaw& rn = c.raw[p][2];
    double2 f[12];
    for (int t = 0; t < 12; t++) {
      double2 tot = make_double2(0, 0);
      int n_tot = 0;
      for (int i = t - 1; i <= t + 1; i++)
        if (i >= 0 && i < 12) { tot = cadd(tot, rc.ce[i]); n_tot++; }
      const int lo = rp.shift < rc.shift ? t : t - 1;
      double2 sp_ = make_double2(0, 0), sn_ = make_double2(0, 0);
      int len = 0;
      for (int i = lo; i <= lo + 1; i++)
        if (i >= 0 && i < 12) { sp_ = cadd(sp_, rp.ce[i]); sn_ = cadd(sn_, rn.ce[i]); len++; }
      tot = cadd(cadd(tot, sp_), sn_);
      f[t] = cdiv(tot, (double)(n_tot + 2 * len));
    }
    double npa = 0, tpa = 0;
    for (int t = 0; t < 12; t++) { npa += nrm(csub(rc.ce[t], f[t])); tpa += nrm(f[t]); }
    const double np = npa / 12 * 7 / 6, tp = tpa / 12;
    const double sp_raw = tp - np / 7, sp = fmax(.00001, sp_raw);
    // do_foe
    double2 fc = make_double2(0, 0);
    double fnp = 0, den = 0;
    for (int t = 0; t < 12; t++) {
      const double2 foe = cmul(conj2(rp.ce[t]), rn.ce[t]);
      const double a = nrm(f[t]);
      const double foe_np = np * np + 2 * np * a;
      const double w = a / foe_np;
      fc = cadd(fc, cscale(foe, w));
      fnp += foe_np * w * w;
      den += a * w;
    }
    const double scale = 1 / den;
    fc = cscale(fc, scale);
    fnp = fnp * scale * scale;
    const double kf = (chn.fc_req - rp.fo) / chn.fc_prog;
    const double res = carg(fc) / (2 * kPi) / (0.0005 + wrapd(rn.ft - rp.ft, -9600.0, 9600.0) * (1 / (fs_prog * kf)));
    const double res_np = fmax(fnp / 2, .001);
    if (lane == 0) s.foe[h.n_foe] = make_double2(rp.fo + res, 1 / res_np);
    h.n_foe++;
    // do_toe_v2
    const CeRaw& x = rp.shift < rc.shift ? rp : rc;
    const CeRaw& y = rp.shift < rc.shift ? rc : rp;
    double2 t1 = make_double2(0, 0), a2 = make_double2(0, 0), b2 = make_double2(0, 0);
    for (int t = 0; t < 12; t++) t1 = cadd(t1, cmul(conj2(x.ce[t]), y.ce[t]));
    for (int t = 0; t < 5; t++) a2 = cadd(a2, cmul(conj2(y.ce[t]), x.ce[t + 1]));
    for (int t = 6; t < 11; t++) b2 = cadd(b2, cmul(conj2(y.ce[t]), x.ce[t + 1]));
    t1 = cdiv(cdiv(t1, 12.0), sqrt(sp));
    const double2 t2 = cdiv(cdiv(cadd(a2, b2), 10.0), sqrt(sp));
    const double delay = -(carg(t1) + carg(t2)) / 2 / 3 / (2 * kPi / 128);
    const double delay_np = fmax(np / sp / 2 / 12, .001);
    double diff = wrapd((rc.ft + delay) - h.frame_timing, -9600.0, 9600.0);
    diff = (0 * (1 / .0001) + diff * (1 / delay_np)) / (1 / .0001 + 1 / delay_np);
    const double ft_new = mmod(h.frame_timing + diff, 19200.0);
    // push the filtered estimate, pop the oldest raw one
    CeFilt& fl = c.filt[p][h.n_filt[p]];
    if (lane < 12) fl.ce[lane] = f[lane];
    if (lane == 0) {
      fl.shift = rc.shift; fl.slot = rc.slot; fl.sym = rc.sym;
      fl.tp = tp; fl.sp = sp; fl.sp_raw = sp_raw; fl.np = np;
    }
    __syncwarp();
    CeRaw r1 = c.raw[p][1], r2 = c.raw[p][2];
    __syncwarp();
    if (lane == 0) { c.raw[p][0] = r1; c.raw[p][1] = r2; }
    __syncwarp();
    h.frame_timing = ft_new;
    h.n_raw[p] = 2;
    h.n_filt[p]++;
  }
  // interp2d
  for (int p = 0; p < P; p++) {
    if (h.n_filt[p] != 2) continue;
    const CeFilt& fp = c.filt[p][0];
    const CeFilt& fcu = c.filt[p][1];
    double time_diff;
    if (p > 2) time_diff = 0.0005;
    else if (c.cp_type == 2) time_diff = 3 * (128 + 32) * (1 / kFs16);
    else if (fp.sym == 0) time_diff = 4 * (128 + 9) * (1 / kFs16);
    else time_diff = (2 * (128 + 9) + (128 + 10)) * (1 / kFs16);
    double2 pi[3], ci[3];
    for (int j = 0; j < 3; j++) {
      const int t = lane + 32 * j;
      if (t < 72) { pi[j] = interp72_at(fp, t); ci[j] = interp72_at(fcu, t); }
    }
    int sl = fp.slot, sy = fp.sym;
    double toff = 0;
    while (sl != fcu.slot || sy != fcu.sym) {
      const double fr = toff / time_diff;
      const double tp = fp.tp + (fcu.tp - fp.tp) * fr, sp = fp.sp + (fcu.sp - fp.sp) * fr;
      const double spr = fp.sp_raw + (fcu.sp_raw - fp.sp_raw) * fr, np = fp.np + (fcu.np - fp.np) * fr;
      int nfill = 1;
      int tsl = 0, tsy = 0;
      if (!h.interp_init[p]) {   // repeat the first estimate back to slot 0 symbol 0
        h.interp_init[p] = 1;
        nfill = 1;
        for (int a = 0, b = 0; a != sy || b != sl; sym_inc(c.n_symb, b, a)) nfill++;
      }
      for (int e = 0; e < nfill; e++) {
        const int esl = e == nfill - 1 ? sl : tsl, esy = e == nfill - 1 ? sy : tsy;
        CeInterp& ci_ = c.interp[p][(h.ih[p] + h.in_[p]) % RING];
        for (int j = 0; j < 3; j++) {
          const int t = lane + 32 * j;
          if (t < 72) ci_.ce[t] = cadd(pi[j], cscale(csub(ci[j], pi[j]), fr));
        }
        if (lane == 0) { ci_.tp = tp; ci_.sp = sp; ci_.sp_raw = spr; ci_.np = np; ci_.slot = esl; ci_.sym = esy; }
        h.in_[p]++;
        sym_inc(c.n_symb, tsl, tsy);
      }
      __syncwarp();
      toff += (c.cp_type == 2 ? 128 + 32 : (sy == 6 ? 128 + 10 : 128 + 9)) * (1 / kFs16);
      sym_inc(c.n_symb, sl, sy);
    }
    CeFilt f1 = c.filt[p][1];
    __syncwarp();
    if (lane == 0) c.filt[p][0] = f1;
    __syncwarp();
    h.n_filt[p] = 1;
  }
  // process the data symbols whose channel estimates are complete
  int dropped = 0;
  lcs_track_cell& o = c.out;
  while (h.dn > 0) {
    bool ready = true;
    for (int p = 0; p < P; p++) ready = ready && h.in_[p] > 0;
    if (!ready) break;
    const DataEnt& d = c.data[h.dh];
    double tp[4], spr[4], np[4];
    for (int p = 0; p < P; p++) {
      const CeInterp& e = c.interp[p][h.ih[p]];
      tp[p] = e.tp; spr[p] = e.sp_raw; np[p] = e.np;
      for (int t = lane; t < 72; t += 32) { o.ce[p][t][0] = e.ce[t].x; o.ce[p][t][1] = e.ce[t].y; }
    }
    const bool first = isnan(o.crs_sp_raw_av[0]);
    const bool avg = (d.slot == 0 || d.slot == 10) && (d.sym == 5 || d.sym == 6);
    __syncwarp();
    if (lane == 0)
      for (int p = 0; p < P; p++) {
        o.crs_tp[p] = tp[p]; o.crs_sp_raw[p] = spr[p]; o.crs_np[p] = np[p];
        if (first) { o.crs_tp_av[p] = tp[p]; o.crs_sp_raw_av[p] = spr[p]; o.crs_np_av[p] = np[p]; }
        else if (avg) {
          o.crs_tp_av[p] = 0.999 * o.crs_tp_av[p] + .001 * tp[p];
          o.crs_sp_raw_av[p] = 0.999 * o.crs_sp_raw_av[p] + .001 * spr[p];
          o.crs_np_av[p] = 0.999 * o.crs_np_av[p] + .001 * np[p];
        }
      }
    __syncwarp();
    // do_pss_sss_sigpower_ce (tracker_thread.cpp:754-820)
    if ((d.slot == 0 || d.slot == 10) && (d.sym == c.n_symb - 2 || d.sym == c.n_symb - 1)) {
      if (d.sym == c.n_symb - 2) {
        for (int t = lane; t < 72; t += 32) c.sss_sym[t] = d.syms[t];
        __syncwarp();
      } else if (lane == 0) {
        const double2* ps = d.syms;
        double b1 = 0, b2 = 0, b3 = 0, b4 = 0;
        for (int t = 0; t < 5; t++) {
          b1 += nrm(c.sss_sym[t]); b2 += nrm(c.sss_sym[67 + t]); b3 += nrm(ps[t]); b4 += nrm(ps[67 + t]);
        }
        const double np_blank = (b1 / 5 + b2 / 5 + b3 / 5 + b4 / 5) / 4;
        const int* sss = tb.sss[d.slot == 0 ? 0 : 1];
        double2* sr = s.sr;
        double2* pr = s.pr;
        double2* sm = s.sm;
        for (int t = 0; t < 62; t++) {
          sr[t] = cscale(c.sss_sym[5 + t], (double)sss[t]);
          pr[t] = cmul(ps[5 + t], conj2(tb.pss[t]));
        }
        double n1 = 0, n2 = 0, tpa = 0;
        for (int t = 0; t < 62; t++) {
          const int lt = max(0, t - 6), rt = min(t + 6, 61);
          double2 a = make_double2(0, 0), b = make_double2(0, 0);
          for (int i = lt; i <= rt; i++) { a = cadd(a, sr[i]); b = cadd(b, pr[i]); }
          sm[t] = cdiv(cadd(a, b), (double)(2 * (rt - lt + 1)));
        }
        for (int t = 0; t < 62; t++) { n1 += nrm(csub(sm[t], sr[t])); n2 += nrm(csub(sm[t], pr[t])); tpa += nrm(sm[t]); }
        const double snp = (n1 / 62 * 13 / 12 + n2 / 62 * 13 / 12) / 2, stp = tpa / 62, ssp = stp - snp / 13;
        o.sync_tp = stp; o.sync_sp = ssp; o.sync_np = snp; o.sync_np_blank = np_blank;
        for (int t = 0; t < 72; t++) {
          const double2 v = (t >= 5 && t < 67) ? sm[t - 5] : make_double2(0, 0);
          o.sync_ce[t][0] = v.x; o.sync_ce[t][1] = v.y;
        }
        if (isnan(o.sync_sp_av)) { o.sync_tp_av = stp; o.sync_sp_av = ssp; o.sync_np_av = snp; o.sync_np_blank_av = np_blank; }
        else {
          o.sync_tp_av = 0.999 * o.sync_tp_av + .001 * stp;
          o.sync_sp_av = 0.999 * o.sync_sp_av + .001 * ssp;
          o.sync_np_av = 0.999 * o.sync_np_av + .001 * snp;
          o.sync_np_blank_av = 0.999 * o.sync_np_blank_av + .001 * np_blank;
        }
      }
      __syncwarp();
    }
    // do_mib_decode (tracker_thread.cpp:531-749)
    if (d.slot == 1 && d.sym <= 3) {
      MibEnt& m = c.mib[(h.mh + h.mn) % 16];
      for (int t = lane; t < 72; t += 32) {
        m.syms[t] = d.syms[t];
        for (int p = 0; p < P; p++) m.ce[p][t] = c.interp[p][h.ih[p]].ce[t];
      }
      if (lane == 0) for (int p = 0; p < P; p++) m.np[p] = np[p];
      __syncwarp();
      h.mn++;
    }
    if (h.mn == 16) {
      const int ok = mib_attempt(c, h, tb, s, lane);
      double fails = o.mib_decode_failures;
      int pop;
      if (ok) { h.mib_sync = 1; fails = 0; pop = 16; }
      else if (h.mib_sync) { fails += 1; pop = 16; }
      else { fails += 0.25; pop = 4; }
      __syncwarp();
      if (lane == 0) {
        o.mib_attempts++;
        if (ok) o.mib_successes++;
        o.mib_decode_failures = fails;
      }
      __syncwarp();
      h.mh = (h.mh + pop) % 16;
      h.mn -= pop;
      if (fails >= 400) { dropped = 1; break; }
    }
    h.dh = (h.dh + 1) % RING;
    h.dn--;
    for (int p = 0; p < P; p++) { h.ih[p] = (h.ih[p] + 1) % RING; h.in_[p]--; }
  }
  sym_inc(c.n_symb, h.slot, h.sym);
  return dropped;
}

// The tracker loop over the symbols one cell completed in this block (one whole warp).
__device__ void run_cell(CellState& c, const Tables& tb, Scratch& s, const ChanState& chn, double fs_prog, int lane) {
  Hdr h = c.h;
  h.n_foe = 0;
  for (int k = 0; k < s.n_pdu; k++) {
    const int dropped = tracker_step(c, h, tb, s, chn, fs_prog, k, lane);
    __syncwarp();
    if (lane == 0) {
      c.out.last_slice_start = s.pdu[k].start;
      c.out.n_symbols++;
      c.out.frame_timing = h.frame_timing;
      if (dropped) { c.out.dropped = 1; c.out.drop_sample = s.pdu[k].start + 128; }
    }
    __syncwarp();
    if (dropped) break;
  }
  if (lane == 0) {
    c.h = h;
    s.n_foe = h.n_foe;
  }
}

// Per-cell slicer for one block (producer_thread.cpp:199-247), one thread.  Completed symbols go to s.pdu with their
// position in the launch buffer and the bulk phase offset of get_fd (tracker_thread.cpp:151-162).
__device__ void slice_cell(CellState& c, Scratch& s, const double* ts, double fo, long long n_done, long long base) {
  const double ft = c.h.frame_timing;
  int t = 0;
  while (t < BLOCK) {
    if (!c.filling) {
      const double tdiff = wrapd(ts[t] - (ft + c.target), -19200.0 / 2, 19200.0 / 2);
      if (fabs(tdiff) < 0.5 || (tdiff > 0 && tdiff < 3)) {
        c.filling = 1;
        c.plate = tdiff;
        c.buffer_offset = 0;
        c.pfo = fo;
        c.pft = ft;
        c.pstart = n_done + t;
      } else {
        t++;
        continue;
      }
    }
    const int take = min(128 - c.buffer_offset, BLOCK - t);
    c.buffer_offset += take;
    t += take;
    if (c.buffer_offset == 128) {
      const int n_el = c.cp_type == 2 ? 128 + 32 : (c.psym == 0 ? 128 + 10 : 128 + 9);
      c.bpo = wrapd(c.bpo + 2 * kPi * n_el * (1 / kFs16) * -c.pfo, -kPi, kPi);
      Pdu& p = s.pdu[s.n_pdu++];
      p.pos = (int)(c.pstart - base);
      p.slot = c.pslot;
      p.sym = c.psym;
      p.late = c.plate;
      p.fo = c.pfo;
      p.ft = c.pft;
      p.bpo = c.bpo;
      p.start = c.pstart;
      c.filling = 0;
      c.target += c.cp_type == 2 ? 32 + 128 : (c.psym == 6 ? 128 + 10 : 128 + 9);
      c.target %= 19200;
      sym_inc(c.n_symb, c.pslot, c.psym);
    }
  }
}

__global__ void __launch_bounds__(THREADS) track_kernel(Params P) {
  extern __shared__ double ts[];                 // [BLOCK] time stamps of the block
  __shared__ double2 fbuf[GROUPS][128];
  __shared__ double2 tw[64];
  __shared__ int pref[33];
  const int ch = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  ChanState& chn = P.ch[ch];
  CellState* cells = P.cells + (size_t)ch * P.max_cells;
  Scratch* scr = P.scr + (size_t)ch * P.max_cells;
  const Tables* tab = P.tab + (size_t)ch * P.max_cells;
  const unsigned char* iq = P.iq + (size_t)ch * P.stride * 2;
  const long long base = chn.n_done - TAIL;      // stream sample of launch-buffer position 0
  if (tid < 64) make_twiddles(tw, tid);
  for (int b = 0; b < P.n_blocks; b++) {
    __syncthreads();
    const double fo = chn.fo;
    const long long n_done = chn.n_done;
    const double kf = (chn.fc_req - fo) / chn.fc_prog;
    if (tid == 0) {                              // producer_thread.cpp:130-136
      double st = chn.sample_time;
      for (int t = 0; t < BLOCK; t++) {
        st += kFs16 / (P.fs_prog * kf);
        if (st > 19200.0) st -= 19200.0;
        ts[t] = st;
      }
      chn.sample_time = st;
    }
    __syncthreads();
    if (tid < P.max_cells) {
      CellState& c = cells[tid];
      scr[tid].n_pdu = 0;
      scr[tid].n_foe = 0;
      if (c.active && !c.out.dropped) slice_cell(c, scr[tid], ts, fo, n_done, base);
    }
    __syncthreads();
    if (tid == 0) {
      pref[0] = 0;
      for (int i = 0; i < P.max_cells; i++) pref[i + 1] = pref[i] + scr[i].n_pdu;
    }
    __syncthreads();
    // get_fd for every symbol of every cell: FOC, 2-sample rotation, FFT-128, 72 bins, late and bulk phase correction
    const int total = pref[P.max_cells], g = tid >> 6, gt = tid & 63;
    for (int r0 = 0; r0 < total; r0 += GROUPS) {
      const int k = r0 + g;
      int ci = 0;
      if (k < total) {
        while (pref[ci + 1] <= k) ci++;
        const Pdu& p = scr[ci].pdu[k - pref[ci]];
        const double kf2 = (chn.fc_req - p.fo) / chn.fc_prog;
        const double kk = kPi * -p.fo / ((P.fs_prog * kf2) / 2);   // fshift_inplace, dsp.h:58-69
        for (int n = gt; n < 128; n += 64) {
          double sn, cs;
          sincos(kk * n, &sn, &cs);
          const double2 x = cmul(load_c<LCS_IQ_CU8>(iq, (size_t)(p.pos + n)), make_double2(cs, sn));
          fbuf[g][bitrev7((n + 126) & 127)] = x;
        }
      }
      __syncthreads();
      fft128_inplace(fbuf[g], tw, gt);
      if (k < total) {
        const Pdu& p = scr[ci].pdu[k - pref[ci]];
        const double sc = 1.0 / sqrt(128.0);
        const double kl = 2 * kPi * p.late / 128;
        double bs, bc;
        sincos(p.bpo, &bs, &bc);
        for (int i = gt; i < 72; i += 64) {
          const int bin = i < 36 ? 92 + i : 1 + (i - 36);
          const int t = i < 36 ? 36 - i : i - 35;
          double sn, cs;
          sincos(-kl * t, &sn, &cs);
          const double2 coeff = make_double2(cs, i < 36 ? -sn : sn);
          const double2 v = make_double2(fbuf[g][bin].x * sc, fbuf[g][bin].y * sc);
          scr[ci].syms[k - pref[ci]][i] = cmul(v, cmul(make_double2(bc, bs), coeff));
        }
      }
      __syncthreads();
    }
    // the tracker loops, one warp per cell
    for (int ci = warp; ci < P.max_cells; ci += WARPS) {
      CellState& c = cells[ci];
      if (c.active && !c.out.dropped && scr[ci].n_pdu > 0) run_cell(c, tab[ci], scr[ci], chn, P.fs_prog, lane);
    }
    __syncthreads();
    if (tid == 0) {                              // FOE updates (tracker_thread.cpp:239-242) in schedule order
      double f = chn.fo;
      for (int ci = 0; ci < P.max_cells; ci++)
        for (int i = 0; i < scr[ci].n_foe; i++) {
          const double2 u = scr[ci].foe[i];
          f = (f * (1 / .000001) + u.x * u.y) / (1 / .000001 + u.y);
        }
      chn.fo = f;
      chn.n_done = n_done + BLOCK;
    }
  }
}

}  // namespace trk
}  // namespace lcs

using namespace lcs;
using namespace lcs::trk;

struct lcs_track {
  lcs_ctx* ctx = nullptr;
  uint32_t n_ch = 0, max_cells = 0;
  double fs_prog = 0;
  std::vector<uint32_t> n_cells;               // cells per channel (slots [0, n) are in use, in the order added)
  std::vector<unsigned char> carry;            // [n_ch][carry_n][2] bytes of the incomplete block
  uint32_t carry_n = 0;
  std::vector<unsigned char> tail;             // [n_ch][TAIL][2] last samples of the processed stream
  DevBuf<ChanState> d_ch;
  DevBuf<CellState> d_cells;
  DevBuf<Tables> d_tab;
  DevBuf<Scratch> d_scr;
  DevBuf<unsigned char> d_iq;
  PinBuf<unsigned char> h_iq;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;    // around each launch
  double kernel_ms = 0;                        // accumulated since the last lcs_track_timing_read
  uint64_t kernel_launches = 0;
  ~lcs_track() {
    if (ev0) cudaEventDestroy(ev0);
    if (ev1) cudaEventDestroy(ev1);
  }
};

static lcs_status tfail(lcs_track* t, lcs_status st, const char* msg) {
  return t ? fail(t->ctx, st, msg) : st;
}

extern "C" {

lcs_status lcs_track_create(lcs_ctx* ctx, uint32_t n_ch, const double* fc_requested, const double* fc_programmed,
                            double fs_programmed, const double* frequency_offset, uint32_t max_cells, lcs_track** out) {
  if (!ctx || !out || !fc_requested || !frequency_offset || n_ch == 0 || max_cells == 0 || max_cells > 32 ||
      !(fs_programmed > 0))
    return ctx ? fail(ctx, LCS_ERR_ARG, "lcs_track_create: bad argument") : LCS_ERR_ARG;
  lcs_track* t = new (std::nothrow) lcs_track();
  if (!t) return fail(ctx, LCS_ERR_STATE, "lcs_track_create: out of memory");
  t->ctx = ctx;
  t->n_ch = n_ch;
  t->max_cells = max_cells;
  t->fs_prog = fs_programmed;
  t->n_cells.assign(n_ch, 0);
  t->tail.assign((size_t)n_ch * TAIL * 2, 127);
  std::vector<ChanState> h(n_ch);
  for (uint32_t c = 0; c < n_ch; c++) {
    h[c].fc_req = fc_requested[c];
    h[c].fc_prog = fc_programmed ? fc_programmed[c] : fc_requested[c];
    h[c].fo = frequency_offset[c];
    h[c].sample_time = -1;                     // producer_thread.cpp:76
    h[c].n_done = 0;
  }
  const size_t nc = (size_t)n_ch * max_cells;
  cudaError_t e = t->d_ch.alloc(n_ch);
  if (e == cudaSuccess) e = t->d_cells.alloc(nc);
  if (e == cudaSuccess) e = t->d_tab.alloc(nc);
  if (e == cudaSuccess) e = t->d_scr.alloc(nc);
  if (e == cudaSuccess) e = cudaMemcpy(t->d_ch.p, h.data(), n_ch * sizeof(ChanState), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemset(t->d_cells.p, 0, nc * sizeof(CellState));
  if (e == cudaSuccess) e = cudaEventCreate(&t->ev0);
  if (e == cudaSuccess) e = cudaEventCreate(&t->ev1);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(track_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, BLOCK * (int)sizeof(double));
  if (e != cudaSuccess) {
    delete t;
    return fail(ctx, LCS_ERR_CUDA, std::string("lcs_track_create: ") + cudaGetErrorString(e));
  }
  *out = t;
  return LCS_OK;
}

void lcs_track_destroy(lcs_track* t) { delete t; }

lcs_status lcs_track_add_cell(lcs_track* t, uint32_t ch, const lcs_cell* cell, double frame_timing) {
  if (!t) return LCS_ERR_ARG;
  if (!cell || ch >= t->n_ch) return tfail(t, LCS_ERR_ARG, "lcs_track_add_cell: bad channel or null cell");
  if (!(cell->n_ports == 1 || cell->n_ports == 2 || cell->n_ports == 4))
    return tfail(t, LCS_ERR_ARG, "lcs_track_add_cell: n_ports must be 1, 2 or 4");
  if (cell->cp_type != 1 && cell->cp_type != 2) return tfail(t, LCS_ERR_ARG, "lcs_track_add_cell: cp_type must be normal or extended");
  if (cell->n_id_1 < 0 || cell->n_id_1 > 167 || cell->n_id_2 < 0 || cell->n_id_2 > 2)
    return tfail(t, LCS_ERR_ARG, "lcs_track_add_cell: cell id out of range");
  if (!(frame_timing >= 0 && frame_timing < 19200)) return tfail(t, LCS_ERR_ARG, "lcs_track_add_cell: frame_timing outside [0, 19200)");
  if (t->n_cells[ch] >= t->max_cells) return tfail(t, LCS_ERR_ARG, "lcs_track_add_cell: channel already tracks max_cells cells");
  std::vector<unsigned char> raw(sizeof(CellState), 0);
  CellState& c = *reinterpret_cast<CellState*>(raw.data());
  c.active = 1;
  c.n_id_1 = cell->n_id_1;
  c.n_id_2 = cell->n_id_2;
  c.n_id_cell = cell->n_id_2 + 3 * cell->n_id_1;
  c.n_ports = cell->n_ports;
  c.cp_type = cell->cp_type;
  c.n_symb = cell->cp_type == 1 ? 7 : 6;
  c.n_rb_dl = cell->n_rb_dl;
  c.phich_dur = cell->phich_duration;
  c.phich_res = cell->phich_resource;
  c.target = cell->cp_type == 1 ? 10 : 32;     // producer_thread.cpp:184
  c.h.frame_timing = frame_timing;
  lcs_track_cell& o = c.out;
  o.n_id_cell = c.n_id_cell;
  o.n_ports = c.n_ports;
  o.cp_type = c.cp_type;
  o.drop_sample = -1;
  o.last_slice_start = -1;
  o.frame_timing = frame_timing;
  double* m = o.crs_tp;
  for (int i = 0; i < 6 * 4 + 8; i++) m[i] = NAN;
  Tables tb;
  std::memset(&tb, 0, sizeof(tb));
  RsDl rs(c.n_id_cell, c.cp_type);
  for (int sl = 0; sl < 20; sl++)
    for (int s3 = 0; s3 < 3; s3++) {
      const cd* v = rs.get(sl, s3 == 2 ? c.n_symb - 3 : s3);
      for (int i = 0; i < 12; i++) tb.rs[sl][s3][i] = make_double2(v[i].real(), v[i].imag());
    }
  const int n_e = c.cp_type == 1 ? 1920 : 1728;
  const std::vector<uint8_t> scr = lte_pn((uint32_t)c.n_id_cell, n_e);   // tracker_thread.cpp:832
  std::vector<int> pos;
  pbch_ratematch_positions(n_e, pos);
  for (int k = 0; k < n_e; k++) {
    tb.scr[k] = scr[k];
    tb.inv[pos[k]][tb.n_inv[pos[k]]++] = (short)k;   // at most ceil(1920 / 120) = 16 repetitions
  }
  sss_fd(c.n_id_1, c.n_id_2, 0, tb.sss[0]);
  sss_fd(c.n_id_1, c.n_id_2, 10, tb.sss[1]);
  cd pfd[62];
  pss_fd(c.n_id_2, pfd);
  for (int i = 0; i < 62; i++) tb.pss[i] = make_double2(pfd[i].real(), pfd[i].imag());
  const size_t slot = (size_t)ch * t->max_cells + t->n_cells[ch];
  LCS_CUDA(t->ctx, cudaMemcpy(t->d_cells.p + slot, raw.data(), sizeof(CellState), cudaMemcpyHostToDevice));
  LCS_CUDA(t->ctx, cudaMemcpy(t->d_tab.p + slot, &tb, sizeof(Tables), cudaMemcpyHostToDevice));
  t->n_cells[ch]++;
  return LCS_OK;
}

lcs_status lcs_track_push_cu8(lcs_track* t, const uint8_t* iq_host, uint32_t n) {
  if (!t) return LCS_ERR_ARG;
  if (!iq_host && n) return tfail(t, LCS_ERR_ARG, "lcs_track_push_cu8: null samples");
  const size_t have = (size_t)t->carry_n + n;
  const uint32_t n_blocks = (uint32_t)(have / BLOCK);
  const size_t rest = have - (size_t)n_blocks * BLOCK;
  const size_t stride = TAIL + (size_t)n_blocks * BLOCK;
  std::vector<unsigned char> carry((size_t)t->n_ch * rest * 2);
  if (n_blocks) {
    LCS_CUDA(t->ctx, t->h_iq.ensure((size_t)t->n_ch * stride * 2));
    LCS_CUDA(t->ctx, t->d_iq.ensure((size_t)t->n_ch * stride * 2));
  }
  for (uint32_t c = 0; c < t->n_ch; c++) {
    // the channel's virtual stream for this push: tail | carried samples | new samples
    const unsigned char* cold = t->carry.data() + (size_t)c * t->carry_n * 2;
    const unsigned char* cnew = iq_host + (size_t)c * n * 2;
    // copy samples [j0, j0 + len) of carried | new into dst
    auto copy = [&](unsigned char* dst, size_t j0, size_t len) {
      const size_t a = j0 < t->carry_n ? std::min(len, (size_t)t->carry_n - j0) : 0;
      if (a) std::memcpy(dst, cold + 2 * j0, 2 * a);
      if (len > a) std::memcpy(dst + 2 * a, cnew + 2 * (j0 + a - t->carry_n), 2 * (len - a));
    };
    if (n_blocks) {
      unsigned char* dst = t->h_iq.p + (size_t)c * stride * 2;
      std::memcpy(dst, t->tail.data() + (size_t)c * TAIL * 2, TAIL * 2);
      copy(dst + 2 * TAIL, 0, (size_t)n_blocks * BLOCK);
      std::memcpy(t->tail.data() + (size_t)c * TAIL * 2, dst + (stride - TAIL) * 2, TAIL * 2);
    }
    copy(carry.data() + (size_t)c * rest * 2, (size_t)n_blocks * BLOCK, rest);
  }
  if (n_blocks) {
    cudaStream_t st = t->ctx->streams[0];
    LCS_CUDA(t->ctx, cudaMemcpyAsync(t->d_iq.p, t->h_iq.p, (size_t)t->n_ch * stride * 2, cudaMemcpyHostToDevice, st));
    Params P;
    P.n_ch = (int)t->n_ch;
    P.max_cells = (int)t->max_cells;
    P.n_blocks = (int)n_blocks;
    P.stride = (int)stride;
    P.fs_prog = t->fs_prog;
    P.iq = t->d_iq.p;
    P.ch = t->d_ch.p;
    P.cells = t->d_cells.p;
    P.tab = t->d_tab.p;
    P.scr = t->d_scr.p;
    LCS_CUDA(t->ctx, cudaEventRecord(t->ev0, st));
    track_kernel<<<t->n_ch, THREADS, BLOCK * sizeof(double), st>>>(P);
    t->ctx->launches++;
    LCS_CUDA(t->ctx, cudaGetLastError());
    LCS_CUDA(t->ctx, cudaEventRecord(t->ev1, st));
    LCS_CUDA(t->ctx, cudaStreamSynchronize(st));
    float ms = 0;
    LCS_CUDA(t->ctx, cudaEventElapsedTime(&ms, t->ev0, t->ev1));
    t->kernel_ms += ms;
    t->kernel_launches++;
  }
  t->carry.swap(carry);
  t->carry_n = (uint32_t)rest;
  return LCS_OK;
}

lcs_status lcs_track_timing_read(lcs_track* t, double* kernel_ms, uint64_t* launches) {
  if (!t) return LCS_ERR_ARG;
  if (!kernel_ms || !launches) return tfail(t, LCS_ERR_ARG, "lcs_track_timing_read: null pointer");
  *kernel_ms = t->kernel_ms;
  *launches = t->kernel_launches;
  t->kernel_ms = 0;
  t->kernel_launches = 0;
  return LCS_OK;
}

lcs_status lcs_track_frequency_offset(const lcs_track* t, double* fo) {
  if (!t) return LCS_ERR_ARG;
  if (!fo) return fail(t->ctx, LCS_ERR_ARG, "lcs_track_frequency_offset: null pointer");
  std::vector<ChanState> h(t->n_ch);
  LCS_CUDA(t->ctx, cudaMemcpy(h.data(), t->d_ch.p, t->n_ch * sizeof(ChanState), cudaMemcpyDeviceToHost));
  for (uint32_t c = 0; c < t->n_ch; c++) fo[c] = h[c].fo;
  return LCS_OK;
}

lcs_status lcs_track_sample_time(const lcs_track* t, uint32_t ch, double* sample_time) {
  if (!t) return LCS_ERR_ARG;
  if (!sample_time || ch >= t->n_ch) return fail(t->ctx, LCS_ERR_ARG, "lcs_track_sample_time: bad channel or null pointer");
  ChanState h;
  LCS_CUDA(t->ctx, cudaMemcpy(&h, t->d_ch.p + ch, sizeof(ChanState), cudaMemcpyDeviceToHost));
  *sample_time = h.sample_time;
  return LCS_OK;
}

lcs_status lcs_track_read(lcs_track* t, uint32_t ch, lcs_track_cell* out, uint32_t max, uint32_t* n) {
  if (!t) return LCS_ERR_ARG;
  if (ch >= t->n_ch || !n || (!out && max)) return tfail(t, LCS_ERR_ARG, "lcs_track_read: bad argument");
  const size_t base = (size_t)ch * t->max_cells;
  const uint32_t nc = t->n_cells[ch];
  std::vector<lcs_track_cell> o(nc);
  for (uint32_t i = 0; i < nc; i++)
    LCS_CUDA(t->ctx, cudaMemcpy(&o[i], &t->d_cells.p[base + i].out, sizeof(lcs_track_cell), cudaMemcpyDeviceToHost));
  uint32_t k = 0, keep = 0;
  for (uint32_t i = 0; i < nc; i++) {
    const bool written = k < max;
    if (written) out[k++] = o[i];
    if (o[i].dropped && written) continue;   // reported once: its slot is freed
    if (keep != i) {                          // keep the order in which the cells were added
      LCS_CUDA(t->ctx, cudaMemcpy(t->d_cells.p + base + keep, t->d_cells.p + base + i, sizeof(CellState), cudaMemcpyDeviceToDevice));
      LCS_CUDA(t->ctx, cudaMemcpy(t->d_tab.p + base + keep, t->d_tab.p + base + i, sizeof(Tables), cudaMemcpyDeviceToDevice));
    }
    keep++;
  }
  for (uint32_t i = keep; i < nc; i++) LCS_CUDA(t->ctx, cudaMemset(&t->d_cells.p[base + i].active, 0, sizeof(int)));
  t->n_cells[ch] = keep;
  *n = k;
  return LCS_OK;
}

}  // extern "C"
