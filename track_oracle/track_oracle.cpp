// track_oracle.cpp - CPU ORACLE of the cell tracker (lcs_track_*).  TEST INFRASTRUCTURE ONLY.
//
// A scalar, loop-for-loop restatement of the reference's per-cell slicer (src/producer_thread.cpp:163-250) and tracker
// loop (src/tracker_thread.cpp:89-1068), run under the deterministic schedule of DESIGN.md section 4.5: blocks of 10000
// samples per channel; at each block start the channel's frequency offset and every cell's frame timing are sampled;
// after a block is sliced every cell (in the order added) runs the tracker loop over the symbols completed in that
// block.  It is compiled together with the searcher oracle (oracle/lcs_oracle.cpp), whose tables, FFT, rate matching,
// Viterbi, CRC and QPSK demodulator it uses.  It lives apart from oracle/, whose restatement of the searcher is pinned
// by the reference's golden vectors and left as it is.  Nothing under lte-cell-scanner_b200/ uses this file.
#include <array>
#include <cmath>
#include <cstring>
#include <deque>
#include <vector>

#include "../include/lcs_b200.h"
#include "../oracle/lcs_oracle.hpp"

using namespace lcso;

namespace {

const double kPi = 3.14159265358979323846;
const double kFs16 = 30720000.0 / 16;     // FS_LTE/16
const int kBlock = 10000;                 // BLOCK_SIZE, producer_thread.cpp:95
const double kDrop = 400;                 // CELL_DROP_THRESHOLD, constants.h:35

double sigpower(const cd* v, int n) {     // dsp.h:23-29
  double r = 0;
  for (int t = 0; t < n; t++) r += std::pow(v[t].real(), 2) + std::pow(v[t].imag(), 2);
  return r / n;
}
double sqr(cd v) { return v.real() * v.real() + v.imag() * v.imag(); }
void slot_sym_inc(int n_symb, int& slot, int& sym) {
  if (++sym == n_symb) { sym = 0; slot = (slot + 1) % 20; }
}

struct TdPdu {        // td_fifo_pdu_t
  int slot, sym;
  double late, frequency_offset, frame_timing;
  int64_t start;
  cd data[128];
};
struct CeRaw { double shift; int slot, sym; cd ce[12]; double frequency_offset, frame_timing; };
struct CeFilt { double shift; int slot, sym; double tp, sp, sp_raw, np; cd ce_filt[12]; };
struct CeInterp { int slot, sym; double tp, sp, sp_raw, np; cd ce[72]; };
struct DataPdu { int slot, sym; cd syms[72]; };
struct MibPdu { cd syms[72]; cd ce[4][72]; double sp[4], np[4]; };

struct TCell {
  lcs_cell info;
  int n_id_cell, n_id_1, n_id_2, n_ports, cp_type, n_symb;
  double frame_timing;
  lcs_track_cell out;
  // producer-side slicer state (cell_local_t)
  uint32_t target;
  bool filling = false;
  int buffer_offset = 0;
  TdPdu pdu;
  // tracker state
  RS_DL rs;
  std::vector<uint8_t> scr;
  int slot = 0, sym = 0;
  double bpo = 0;
  std::deque<DataPdu> data_fifo;
  std::deque<CeRaw> raw[4];
  std::deque<CeFilt> filt[4];
  std::deque<CeInterp> interp[4];
  bool interp_init[4] = {false, false, false, false};
  std::deque<MibPdu> mib_fifo;
  bool mib_sync = false;
  cd sss_sym[72];
  std::deque<std::array<cd, 12>> ce_history[4];   // tracker_thread.cpp:850
  TCell(const lcs_cell& c, double ft)
      : info(c), n_id_cell(c.n_id_2 + 3 * c.n_id_1), n_id_1(c.n_id_1), n_id_2(c.n_id_2), n_ports(c.n_ports),
        cp_type(c.cp_type), n_symb(c.cp_type == 1 ? 7 : 6), frame_timing(ft), rs(n_id_cell, 6, c.cp_type) {
    scr = lte_pn((uint32_t)n_id_cell, cp_type == 1 ? 1920 : 1728);   // tracker_thread.cpp:832
    target = cp_type == 1 ? 10 : 32;                                  // producer_thread.cpp:184
    pdu.slot = pdu.sym = 0;
    std::memset(&out, 0, sizeof(out));
    out.n_id_cell = n_id_cell;
    out.n_ports = n_ports;
    out.cp_type = cp_type;
    out.drop_sample = -1;
    out.last_slice_start = -1;
    double* m = out.crs_tp;
    for (int i = 0; i < 6 * 4 + 8; i++) m[i] = NAN;
    out.frame_timing = ft;
    for (auto& s : sss_sym) s = 0;
  }
};

struct Channel {
  double fc_req, fc_prog, fo;
  double sample_time = -1;
  int64_t n_done = 0;                // samples of complete blocks processed
  std::vector<uint8_t> pend;         // bytes of the incomplete block
  std::vector<TCell*> cells;
};

}  // namespace

struct to_track {
  double fs_prog;
  uint32_t max_cells;
  std::vector<Channel> ch;
  ~to_track() {
    for (auto& c : ch)
      for (TCell* p : c.cells) delete p;
  }
};

namespace {

// get_fd, tracker_thread.cpp:91-174
void get_fd(TCell& c, const Channel& chn, double fs_prog, const TdPdu& pdu, cd syms[72]) {
  const double fo = pdu.frequency_offset;
  const double k_factor = (chn.fc_req - fo) / chn.fc_prog;
  cd d[128];
  const double k = kPi * -fo / ((fs_prog * k_factor) / 2);            // fshift_inplace, dsp.h:58-69
  for (int t = 0; t < 128; t++) d[t] = pdu.data[t] * cd(std::cos(k * t), std::sin(k * t));
  cd in[128], o[128];
  for (int t = 0; t < 126; t++) in[t] = d[t + 2];
  in[126] = d[0];
  in[127] = d[1];
  fft128(in, o);
  for (int t = 0; t < 128; t++) o[t] /= std::sqrt(128.0);             // dft = fft/sqrt(N), dsp.h:34
  for (int t = 0; t < 36; t++) { syms[t + 36] = o[t + 1]; syms[t] = o[92 + t]; }
  const int n_el = c.cp_type == 2 ? 128 + 32 : (pdu.sym == 0 ? 128 + 10 : 128 + 9);
  const double kk = 2 * kPi * pdu.late / 128;
  c.bpo = wrap(c.bpo + 2 * kPi * n_el * (1 / kFs16) * -fo, -kPi, kPi);
  const cd bpo(std::cos(c.bpo), std::sin(c.bpo));
  for (int t = 1; t <= 36; t++) {
    const double ph = -kk * t;
    cd coeff(std::cos(ph), std::sin(ph));
    syms[35 + t] *= bpo * coeff;
    coeff = std::conj(coeff);
    syms[36 - t] *= bpo * coeff;
  }
}

// filter_ce, tracker_thread.cpp:176-202
void filter_ce(const CeRaw& p, const CeRaw& c, const CeRaw& n, cd out[12]) {
  for (int t = 0; t < 12; t++) {
    cd total = 0;
    int n_total = 0;
    cd s = 0;
    for (int i = t - 1; i <= t + 1; i++)
      if (i >= 0 && i < 12) { s += c.ce[i]; n_total++; }
    total = s;
    const int lo = p.shift < c.shift ? t : t - 1, hi = lo + 1;
    cd sp = 0, sn = 0;
    int len = 0;
    for (int i = lo; i <= hi; i++)
      if (i >= 0 && i < 12) { sp += p.ce[i]; sn += n.ce[i]; len++; }
    total = total + sp;
    total = total + sn;
    n_total += 2 * len;
    out[t] = total / (double)n_total;
  }
}

// do_foe, tracker_thread.cpp:204-243
void do_foe(Channel& chn, double fs_prog, const CeRaw& p, const CeRaw& n, double np, const cd* ce_filt) {
  cd foe_comb = 0;
  double foe_comb_np = 0, den = 0;
  for (int t = 0; t < 12; t++) {
    const cd foe = std::conj(p.ce[t]) * n.ce[t];
    const double foe_np = np * np + 2 * np * sqr(ce_filt[t]);
    const double w = sqr(ce_filt[t]) / foe_np;
    foe_comb += foe * cd(w, 0);
    foe_comb_np += foe_np * w * w;
    den += sqr(ce_filt[t]) * w;
  }
  const double scale = 1 / den;
  foe_comb = foe_comb * scale;
  foe_comb_np = foe_comb_np * scale * scale;
  const double fo = p.frequency_offset;
  const double k_factor = (chn.fc_req - fo) / chn.fc_prog;
  const double residual_f = std::arg(foe_comb) / (2 * kPi) /
                            (0.0005 + wrap(n.frame_timing - p.frame_timing, -19200.0 / 2, 19200.0 / 2) * (1 / (fs_prog * k_factor)));
  const double residual_f_np = std::max(foe_comb_np / 2, .001);
  chn.fo = (chn.fo * (1 / .000001) + (fo + residual_f) * (1 / residual_f_np)) / (1 / .000001 + 1 / residual_f_np);
}

// do_toe_v2, tracker_thread.cpp:245-279
void do_toe_v2(TCell& c, const CeRaw& p, const CeRaw& cu, double sp, double np) {
  cd toe1 = 0, toe2 = 0, a = 0, b = 0;
  const CeRaw& x = p.shift < cu.shift ? p : cu;   // conj() operand of toe1
  const CeRaw& y = p.shift < cu.shift ? cu : p;
  for (int t = 0; t < 12; t++) toe1 += std::conj(x.ce[t]) * y.ce[t];
  toe1 = toe1 / 12.0;
  // toe2 pairs conj(y[t]) with x[t+1]
  for (int t = 0; t < 5; t++) a += std::conj(y.ce[t]) * x.ce[t + 1];
  for (int t = 6; t < 11; t++) b += std::conj(y.ce[t]) * x.ce[t + 1];
  toe2 = (a + b) / 10.0;
  toe1 = toe1 / std::sqrt(sp);
  toe2 = toe2 / std::sqrt(sp);
  const double delay = -(std::arg(toe1) + std::arg(toe2)) / 2 / 3 / (2 * kPi / 128);
  const double delay_np = std::max(np / sp / 2 / 12, .001);
  double diff = wrap((cu.frame_timing + delay) - c.frame_timing, -19200.0 / 2, 19200.0 / 2);
  diff = (0 * (1 / .0001) + diff * (1 / delay_np)) / (1 / .0001 + 1 / delay_np);
  c.frame_timing = matlab_mod(c.frame_timing + diff, 19200.0);
}

// do_ac_fd, tracker_thread.cpp:318-340
void do_ac_fd(TCell& c, const CeRaw& cu, double sp, double np) {
  cd ac[12];
  for (int d = 0; d < 12; d++) {
    ac[d] = 0;
    for (int t = 0; t < 12 - d; t++) ac[d] += std::conj(cu.ce[t]) * cu.ce[t + d];
    ac[d] = ac[d] / (double)(12 - d);
  }
  for (int d = 0; d < 12; d++) ac[d] = ac[d] / sp;
  for (int d = 0; d < 12; d++) {
    const double ac_np = (np * np / (sp * sp) + 2 * np / sp) / (12 - d);   // matlab_range(12.0, -1.0, 1.0)
    double* o = c.out.ac_fd[d];
    const double w = 1.0 / ac_np;
    o[0] = (o[0] * (1 / .00001) + ac[d].real() * w) / (1 / .00001 + w);
    o[1] = (o[1] * (1 / .00001) + ac[d].imag() * w) / (1 / .00001 + w);
  }
}

// do_ac_td, tracker_thread.cpp:343-370
void do_ac_td(TCell& c, const CeRaw& cu, double sp, std::deque<std::array<cd, 12>>& ce_history) {
  std::array<cd, 12> v;
  for (int i = 0; i < 12; i++) v[i] = cu.ce[i];
  ce_history.push_back(v);
  if (ce_history.size() > 72) ce_history.pop_front();
  if (ce_history.size() != 72) return;
  cd xc[72];
  for (int t = 0; t < 72; t++) {
    cd s = 0;
    for (int i = 0; i < 12; i++) s += std::conj(ce_history[71][i]) * ce_history[71 - t][i];
    xc[t] = s / 12.0;
  }
  for (int t = 0; t < 72; t++) xc[t] = xc[t] / sp;
  for (int t = 0; t < 72; t++) {
    double* o = c.out.ac_td[t];
    o[0] = (o[0] * (1 / .00001) + xc[t].real() * 1 / 1) / (1 / .00001 + 1);
    o[1] = (o[1] * (1 / .00001) + xc[t].imag() * 1 / 1) / (1 / .00001 + 1);
  }
}

// interp72, tracker_thread.cpp:372-393
void interp72(const CeFilt& rs, cd out[72]) {
  int l_x = (int)rs.shift, r_x = (int)rs.shift + 6, ptr = 1;
  cd l_y = rs.ce_filt[0], r_y = rs.ce_filt[1];
  for (int t = 0; t < 72; t++) {
    if (t > r_x && ptr < 11) { l_x = r_x; l_y = r_y; r_x += 6; ptr++; r_y = rs.ce_filt[ptr]; }
    out[t] = (r_y - l_y) / (double)(r_x - l_x) * (double)(t - l_x) + l_y;
  }
}

// interp2d, tracker_thread.cpp:395-477
void interp2d(TCell& c, const CeFilt& p, const CeFilt& cu, int port) {
  cd pi[72], ci[72];
  interp72(p, pi);
  interp72(cu, ci);
  int slot = p.slot, sym = p.sym;
  double time_diff;
  if (port > 2) time_diff = 0.0005;
  else if (c.cp_type == 2) time_diff = 3 * (128 + 32) * (1 / kFs16);
  else if (p.sym == 0) time_diff = 4 * (128 + 9) * (1 / kFs16);
  else time_diff = (2 * (128 + 9) + (128 + 10)) * (1 / kFs16);
  double time_offset = 0;
  while (slot != cu.slot || sym != cu.sym) {
    const double f = time_offset / time_diff;
    CeInterp e;
    for (int t = 0; t < 72; t++) e.ce[t] = pi[t] + (ci[t] - pi[t]) * f;
    e.tp = p.tp + (cu.tp - p.tp) * f;
    e.sp = p.sp + (cu.sp - p.sp) * f;
    e.sp_raw = p.sp_raw + (cu.sp_raw - p.sp_raw) * f;
    e.np = p.np + (cu.np - p.np) * f;
    if (!c.interp_init[port]) {
      c.interp_init[port] = true;
      int tsy = 0, tsl = 0;
      while (tsy != sym || tsl != slot) {
        e.sym = tsy;
        e.slot = tsl;
        c.interp[port].push_back(e);
        slot_sym_inc(c.n_symb, tsl, tsy);
      }
    }
    e.slot = slot;
    e.sym = sym;
    c.interp[port].push_back(e);
    if (c.cp_type == 2) time_offset += (128 + 32) * (1 / kFs16);
    else time_offset += (sym == 6 ? 128 + 10 : 128 + 9) * (1 / kFs16);
    slot_sym_inc(c.n_symb, slot, sym);
  }
}

// do_pss_sss_sigpower_ce, tracker_thread.cpp:754-820
void do_pss_sss(TCell& c, const cd* syms, int slot, int sym) {
  if ((slot != 0 && slot != 10) || (sym != c.n_symb - 2 && sym != c.n_symb - 1)) return;
  if (sym == c.n_symb - 2) {
    for (int t = 0; t < 72; t++) c.sss_sym[t] = syms[t];
    return;
  }
  const cd* pss = syms;
  const double np_blank = (sigpower(c.sss_sym, 5) + sigpower(c.sss_sym + 67, 5) + sigpower(pss, 5) + sigpower(pss + 67, 5)) / 4;
  const std::vector<int> sss = sss_fd_calc(c.n_id_1, c.n_id_2, slot == 0 ? 0 : 10);
  const std::vector<cd> pfd = pss_fd_calc(c.n_id_2);
  cd sr[62], pr[62], sm[62], d1[62], d2[62];
  for (int t = 0; t < 62; t++) {
    sr[t] = c.sss_sym[5 + t] * cd(sss[t], 0);
    pr[t] = pss[5 + t] * std::conj(pfd[t]);
  }
  for (int t = 0; t < 62; t++) {
    const int lt = std::max(0, t - 6), rt = std::min(t + 6, 61);
    cd a = 0, b = 0;
    for (int i = lt; i <= rt; i++) { a += sr[i]; b += pr[i]; }
    sm[t] = (a + b) / (double)(2 * (rt - lt + 1));
  }
  for (int t = 0; t < 62; t++) { d1[t] = sm[t] - sr[t]; d2[t] = sm[t] - pr[t]; }
  const double np = (sigpower(d1, 62) * 13 / 12 + sigpower(d2, 62) * 13 / 12) / 2;
  const double tp = sigpower(sm, 62);
  const double sp = tp - np / 13;
  lcs_track_cell& o = c.out;
  o.sync_tp = tp;
  o.sync_sp = sp;
  o.sync_np = np;
  o.sync_np_blank = np_blank;
  for (int t = 0; t < 72; t++) {
    const cd v = (t >= 5 && t < 67) ? sm[t - 5] : cd(0, 0);
    o.sync_ce[t][0] = v.real();
    o.sync_ce[t][1] = v.imag();
  }
  if (std::isnan(o.sync_sp_av)) {
    o.sync_tp_av = tp; o.sync_sp_av = sp; o.sync_np_av = np; o.sync_np_blank_av = np_blank;
  } else {
    o.sync_tp_av = 0.999 * o.sync_tp_av + .001 * tp;
    o.sync_sp_av = 0.999 * o.sync_sp_av + .001 * sp;
    o.sync_np_av = 0.999 * o.sync_np_av + .001 * np;
    o.sync_np_blank_av = 0.999 * o.sync_np_blank_av + .001 * np_blank;
  }
}

// do_mib_decode with pbch_extract_rt, tracker_thread.cpp:494-749.  Returns true when the cell is dropped.
bool do_mib(TCell& c, const cd* syms, const cd ce[4][72], const double* sp, const double* np, int slot, int sym) {
  if (slot == 1 && sym <= 3) {
    MibPdu m;
    for (int t = 0; t < 72; t++) m.syms[t] = syms[t];
    for (int p = 0; p < c.n_ports; p++) {
      for (int t = 0; t < 72; t++) m.ce[p][t] = ce[p][t];
      m.sp[p] = sp[p];
      m.np[p] = np[p];
    }
    c.mib_fifo.push_back(m);
  }
  if (c.mib_fifo.size() != 16) return false;
  const int n_syms = c.cp_type == 1 ? 960 : 864;
  std::vector<cd> y(n_syms), h[4];
  std::vector<double> npp[4];
  for (int p = 0; p < 4; p++) { h[p].resize(n_syms); npp[p].resize(n_syms); }
  const int v3 = c.n_id_cell % 3;
  int idx = 0;
  for (int fr = 0; fr < 4; fr++)
    for (int symn = 0; symn < 4; symn++)
      for (int sc = 0; sc < 72; sc++) {
        if (sc % 3 == v3 && (symn == 0 || symn == 1 || (symn == 3 && c.cp_type == 2))) continue;
        const MibPdu& m = c.mib_fifo[fr * 4 + symn];
        y[idx] = m.syms[sc];
        for (int p = 0; p < c.n_ports; p++) { h[p][idx] = m.ce[p][sc]; npp[p][idx] = m.np[p]; }
        idx++;
      }
  std::vector<cd> s(n_syms);
  std::vector<double> nm(n_syms);
  if (c.n_ports == 1) {
    for (int t = 0; t < n_syms; t++) {
      const cd gain = std::conj(h[0][t] / cd(sqr(h[0][t]), 0));
      s[t] = y[t] * gain;
      nm[t] = npp[0][t] * sqr(gain);
    }
  } else {
    for (int t = 0; t < n_syms; t += 2) {
      cd h1, h2;
      double npt;
      if (c.n_ports == 2) {
        h1 = (h[0][t] + h[0][t + 1]) / 2.0; h2 = (h[1][t] + h[1][t + 1]) / 2.0; npt = (npp[0][t] + npp[1][t]) / 2;
      } else if (t % 4 == 0) {
        h1 = (h[0][t] + h[0][t + 1]) / 2.0; h2 = (h[2][t] + h[2][t + 1]) / 2.0; npt = (npp[0][t] + npp[2][t]) / 2;
      } else {
        h1 = (h[1][t] + h[1][t + 1]) / 2.0; h2 = (h[3][t] + h[3][t + 1]) / 2.0; npt = (npp[1][t] + npp[3][t]) / 2;
      }
      const cd x1 = y[t], x2 = y[t + 1];
      const double scale = std::pow(h1.real(), 2) + std::pow(h1.imag(), 2) + std::pow(h2.real(), 2) + std::pow(h2.imag(), 2);
      s[t] = (std::conj(h1) * x1 + h2 * std::conj(x2)) / scale;
      s[t + 1] = std::conj((-std::conj(h2) * x1 + h1 * std::conj(x2)) / scale);
      nm[t] = (std::pow(std::abs(h1) / scale, 2) + std::pow(std::abs(h2) / scale, 2)) * npt;
      nm[t + 1] = nm[t];
    }
    for (auto& v : s) v *= std::pow(2, 0.5);
  }
  std::vector<double> e = lte_demodulate_qpsk(s, nm);
  for (size_t t = 0; t < e.size(); t++)
    if (c.scr[t]) e[t] = -e[t];
  const std::vector<double> d = lte_conv_deratematch(e, 40);
  const std::vector<uint8_t> bits = lte_conv_decode(d, 40);
  std::vector<uint8_t> crc = lte_calc_crc16(std::vector<uint8_t>(bits.begin(), bits.begin() + 24));
  if (c.n_ports == 2) for (int t = 0; t < 16; t++) crc[t] = 1 - crc[t];
  else if (c.n_ports == 4) for (int t = 1; t < 16; t += 2) crc[t] = 1 - crc[t];
  static const int bw[6] = {6, 15, 25, 50, 75, 100};
  const int bwi = bits[0] * 4 + bits[1] * 2 + bits[2];
  const int n_rb = bwi < 6 ? bw[bwi] : 0;
  const int phich_dur = bits[3] ? 2 : 1;
  const int phich_res = 1 + bits[4] * 2 + bits[5];
  const bool ok = std::memcmp(crc.data(), bits.data() + 24, 16) == 0 && n_rb == c.info.n_rb_dl &&
                  phich_dur == c.info.phich_duration && phich_res == c.info.phich_resource;
  c.out.mib_attempts++;
  int pop;
  if (ok) {
    c.mib_sync = true;
    c.out.mib_decode_failures = 0;
    c.out.mib_successes++;
    pop = 16;
  } else if (c.mib_sync) {
    c.out.mib_decode_failures++;
    pop = 16;
  } else {
    c.out.mib_decode_failures += 0.25;
    pop = 4;
  }
  for (int t = 0; t < pop; t++) c.mib_fifo.pop_front();
  return c.out.mib_decode_failures >= kDrop;
}

// One iteration of the tracker loop (tracker_thread.cpp:856-1067) for one sliced symbol.  Returns true on a drop.
bool tracker_step(TCell& c, Channel& chn, double fs_prog, const TdPdu& pdu) {
  DataPdu dp;
  dp.slot = c.slot;
  dp.sym = c.sym;
  get_fd(c, chn, fs_prog, pdu, dp.syms);
  c.data_fifo.push_back(dp);
  for (int p = 0; p < c.n_ports; p++) {
    const double shift = c.rs.get_shift(c.slot, c.sym, p);
    if (std::isnan(shift)) continue;
    CeRaw r;
    r.shift = shift;
    r.slot = c.slot;
    r.sym = c.sym;
    const std::vector<cd>& rsv = c.rs.get_rs(c.slot, c.sym);
    for (int i = 0; i < 12; i++) r.ce[i] = dp.syms[round_i(shift) + 6 * i] * std::conj(rsv[i]);
    r.frequency_offset = pdu.frequency_offset;
    r.frame_timing = pdu.frame_timing;
    c.raw[p].push_back(r);
  }
  for (int p = 0; p < c.n_ports; p++) {
    if (c.raw[p].size() != 3) continue;
    const CeRaw& rp = c.raw[p][0];
    const CeRaw& rc = c.raw[p][1];
    const CeRaw& rn = c.raw[p][2];
    CeFilt f;
    filter_ce(rp, rc, rn, f.ce_filt);
    cd diff[12];
    for (int t = 0; t < 12; t++) diff[t] = rc.ce[t] - f.ce_filt[t];
    const double np = sigpower(diff, 12) * 7 / 6;
    const double tp = sigpower(f.ce_filt, 12);
    const double sp_raw = tp - np / 7;
    const double sp = std::max(.00001, sp_raw);
    f.shift = rc.shift; f.slot = rc.slot; f.sym = rc.sym;
    f.tp = tp; f.sp = sp; f.sp_raw = sp_raw; f.np = np;
    c.filt[p].push_back(f);
    do_foe(chn, fs_prog, rp, rn, np, f.ce_filt);
    do_toe_v2(c, rp, rc, sp, np);
    do_ac_fd(c, rc, sp, np);                  // tracker_thread.cpp:955
    do_ac_td(c, rc, sp, c.ce_history[p]);     // tracker_thread.cpp:958
    c.raw[p].pop_front();
  }
  for (int p = 0; p < c.n_ports; p++) {
    if (c.filt[p].size() != 2) continue;
    interp2d(c, c.filt[p][0], c.filt[p][1], p);
    c.filt[p].pop_front();
  }
  auto ce_ready = [&] {
    for (int p = 0; p < c.n_ports; p++)
      if (c.interp[p].empty()) return false;
    return true;
  };
  bool dropped = false;
  while (!c.data_fifo.empty() && ce_ready()) {
    const DataPdu& d = c.data_fifo.front();
    cd ce[4][72];
    double tp[4], sp[4], sp_raw[4], np[4];
    lcs_track_cell& o = c.out;
    for (int p = 0; p < c.n_ports; p++) {
      const CeInterp& e = c.interp[p].front();
      for (int t = 0; t < 72; t++) { ce[p][t] = e.ce[t]; o.ce[p][t][0] = e.ce[t].real(); o.ce[p][t][1] = e.ce[t].imag(); }
      tp[p] = e.tp; sp[p] = e.sp; sp_raw[p] = e.sp_raw; np[p] = e.np;
    }
    // tracker_thread.cpp:1021-1045
    const bool first = std::isnan(o.crs_sp_raw_av[0]);
    const bool avg = (d.slot == 0 || d.slot == 10) && (d.sym == 5 || d.sym == 6);
    for (int p = 0; p < c.n_ports; p++) {
      o.crs_tp[p] = tp[p];
      o.crs_sp_raw[p] = sp_raw[p];
      o.crs_np[p] = np[p];
      if (first) {
        o.crs_tp_av[p] = tp[p]; o.crs_sp_raw_av[p] = sp_raw[p]; o.crs_np_av[p] = np[p];
      } else if (avg) {
        o.crs_tp_av[p] = 0.999 * o.crs_tp_av[p] + .001 * tp[p];
        o.crs_sp_raw_av[p] = 0.999 * o.crs_sp_raw_av[p] + .001 * sp_raw[p];
        o.crs_np_av[p] = 0.999 * o.crs_np_av[p] + .001 * np[p];
      }
    }
    do_pss_sss(c, d.syms, d.slot, d.sym);
    if (do_mib(c, d.syms, ce, sp, np, d.slot, d.sym)) { dropped = true; break; }
    c.data_fifo.pop_front();
    for (int p = 0; p < c.n_ports; p++) c.interp[p].pop_front();
  }
  c.out.n_symbols++;
  c.out.frame_timing = c.frame_timing;
  slot_sym_inc(c.n_symb, c.slot, c.sym);
  return dropped;
}

// One block of one channel: time stamps, per-cell slicing (producer_thread.cpp:199-247), then the tracker loops.
void run_block(to_track* tr, Channel& chn, const uint8_t* iq) {
  const double fo = chn.fo;
  const double k_factor = (chn.fc_req - fo) / chn.fc_prog;
  std::vector<double> ts(kBlock);
  for (int t = 0; t < kBlock; t++) {
    chn.sample_time += kFs16 / (tr->fs_prog * k_factor);
    if (chn.sample_time > 19200.0) chn.sample_time -= 19200.0;
    ts[t] = chn.sample_time;
  }
  std::vector<std::vector<TdPdu>> done(chn.cells.size());
  for (size_t ci = 0; ci < chn.cells.size(); ci++) {
    TCell& c = *chn.cells[ci];
    if (c.out.dropped) continue;
    const double ft = c.frame_timing;
    for (int t = 0; t < kBlock; t++) {
      if (!c.filling) {
        const double tdiff = wrap(ts[t] - (ft + c.target), -19200.0 / 2, 19200.0 / 2);
        if (std::fabs(tdiff) < 0.5 || (tdiff > 0 && tdiff < 3)) {
          c.filling = true;
          c.pdu.late = tdiff;
          c.buffer_offset = 0;
          c.pdu.frequency_offset = fo;
          c.pdu.frame_timing = ft;
          c.pdu.start = chn.n_done + t;
        }
      }
      if (c.filling) {
        c.pdu.data[c.buffer_offset++] = cd((iq[2 * t] - 127.0) / 128.0, (iq[2 * t + 1] - 127.0) / 128.0);
        if (c.buffer_offset == 128) {
          done[ci].push_back(c.pdu);
          c.filling = false;
          c.target += c.cp_type == 2 ? 32 + 128 : (c.pdu.sym == 6 ? 128 + 10 : 128 + 9);
          c.target %= 19200;
          slot_sym_inc(c.n_symb, c.pdu.slot, c.pdu.sym);
        }
      }
    }
  }
  for (size_t ci = 0; ci < chn.cells.size(); ci++) {
    TCell& c = *chn.cells[ci];
    for (const TdPdu& p : done[ci]) {
      c.out.last_slice_start = p.start;
      if (tracker_step(c, chn, tr->fs_prog, p)) {
        c.out.dropped = 1;
        c.out.drop_sample = p.start + 128;
        break;
      }
    }
  }
  chn.n_done += kBlock;
}

}  // namespace

extern "C" {

to_track* to_create(uint32_t n_ch, const double* fc_req, const double* fc_prog, double fs_prog, const double* fo,
                    uint32_t max_cells) {
  to_track* t = new to_track();
  t->fs_prog = fs_prog;
  t->max_cells = max_cells;
  t->ch.resize(n_ch);
  for (uint32_t c = 0; c < n_ch; c++) {
    t->ch[c].fc_req = fc_req[c];
    t->ch[c].fc_prog = fc_prog ? fc_prog[c] : fc_req[c];
    t->ch[c].fo = fo[c];
  }
  return t;
}
void to_destroy(to_track* t) { delete t; }
int to_add_cell(to_track* t, uint32_t ch, const lcs_cell* cell, double frame_timing) {
  if (ch >= t->ch.size() || t->ch[ch].cells.size() >= t->max_cells) return LCS_ERR_ARG;
  t->ch[ch].cells.push_back(new TCell(*cell, frame_timing));
  return LCS_OK;
}
int to_push_cu8(to_track* t, const uint8_t* iq, uint32_t n) {
  for (size_t c = 0; c < t->ch.size(); c++) {
    Channel& chn = t->ch[c];
    const uint8_t* src = iq + (size_t)c * n * 2;
    chn.pend.insert(chn.pend.end(), src, src + (size_t)n * 2);
    size_t off = 0;
    while (chn.pend.size() - off >= (size_t)kBlock * 2) {
      run_block(t, chn, chn.pend.data() + off);
      off += (size_t)kBlock * 2;
    }
    chn.pend.erase(chn.pend.begin(), chn.pend.begin() + off);
  }
  return LCS_OK;
}
void to_frequency_offset(const to_track* t, double* fo) {
  for (size_t c = 0; c < t->ch.size(); c++) fo[c] = t->ch[c].fo;
}
double to_sample_time(const to_track* t, uint32_t ch) { return t->ch[ch].sample_time; }
int to_read(to_track* t, uint32_t ch, lcs_track_cell* out, uint32_t max, uint32_t* n) {
  if (ch >= t->ch.size()) return LCS_ERR_ARG;
  std::vector<TCell*>& cells = t->ch[ch].cells;
  uint32_t k = 0;
  std::vector<TCell*> keep;
  for (TCell* c : cells) {
    const bool written = k < max;
    if (written) out[k++] = c->out;
    if (c->out.dropped && written) delete c;   // a dropped cell is reported once, then frees its slot
    else keep.push_back(c);
  }
  cells.swap(keep);
  *n = k;
  return LCS_OK;
}

}  // extern "C"
