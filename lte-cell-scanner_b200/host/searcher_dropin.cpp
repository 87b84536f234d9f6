// searcher_dropin.cpp - replacement for the reference's src/searcher.cpp: identical signatures
// (include/searcher.h:22-124), bodies marshal the IT++ containers to the C ABI of
// include/lcs_b200.h and back.  No numerical work happens here.
#include "searcher_dropin.hpp"
#include "../../include/lcs_meas.h"
#include "../../include/lcs_psd.h"

#include <cmath>
#include <cstdlib>
#include <cstring>

#include <cuda_runtime.h>

using namespace itpp;
using std::complex;

static lcs_ctx* g_ctx = nullptr;
static bool g_skip_debug = false;
static char g_err[512];

void xcorr_pss_skip_debug_outputs(bool skip) { g_skip_debug = skip; }

static void check(lcs_status rc, const char* where) {
  if (rc == LCS_OK) return;
  snprintf(g_err, sizeof(g_err), "%s: %s", where, lcs_last_error(g_ctx));
  throw((const char*)g_err);   // the reference throws const char* (searcher.cpp:786,883)
}

lcs_ctx* lcs_dropin_ctx() {
  if (!g_ctx) {
    const char* d = std::getenv("LCS_DEVICE");
    lcs_status rc = lcs_ctx_create(d ? std::atoi(d) : 0, &g_ctx);
    if (rc != LCS_OK) {
      snprintf(g_err, sizeof(g_err), "lcs_ctx_create: %s", lcs_last_error(nullptr));
      throw((const char*)g_err);
    }
  }
  return g_ctx;
}

// ---- Cell (src/common.cpp:29-56) ----
Cell::Cell()
    : fc_requested(NAN), fc_programmed(NAN), pss_pow(NAN), ind(-1), freq(NAN), n_id_2(-1), n_id_1(-1),
      cp_type(cp_type_t::UNKNOWN), frame_start(NAN), freq_fine(NAN), freq_superfine(NAN), n_ports(-1), n_rb_dl(-1),
      phich_duration(phich_duration_t::UNKNOWN), phich_resource(phich_resource_t::UNKNOWN), sfn(-1) {}
int16 Cell::n_id_cell() const { return ((n_id_1 >= 0) && (n_id_2 >= 0)) ? (n_id_2 + 3 * n_id_1) : -1; }
int8 Cell::n_symb_dl() const { return (cp_type == cp_type_t::NORMAL) ? 7 : ((cp_type == cp_type_t::EXTENDED) ? 6 : -1); }

static lcs_cell to_pod(const Cell& c) {
  lcs_cell p;
  p.fc_requested = c.fc_requested; p.fc_programmed = c.fc_programmed; p.pss_pow = c.pss_pow;
  p.ind = c.ind; p.freq = c.freq; p.n_id_2 = c.n_id_2; p.n_id_1 = c.n_id_1; p.cp_type = (int)c.cp_type;
  p.frame_start = c.frame_start; p.freq_fine = c.freq_fine; p.freq_superfine = c.freq_superfine;
  p.n_ports = c.n_ports; p.n_rb_dl = c.n_rb_dl; p.phich_duration = (int)c.phich_duration;
  p.phich_resource = (int)c.phich_resource; p.sfn = c.sfn;
  return p;
}
static Cell from_pod(const lcs_cell& p) {
  Cell c;
  c.fc_requested = p.fc_requested; c.fc_programmed = p.fc_programmed; c.pss_pow = p.pss_pow;
  c.ind = p.ind; c.freq = p.freq; c.n_id_2 = (int8)p.n_id_2; c.n_id_1 = (int16)p.n_id_1;
  c.cp_type = (cp_type_t::cp_type_t)p.cp_type;
  c.frame_start = p.frame_start; c.freq_fine = p.freq_fine; c.freq_superfine = p.freq_superfine;
  c.n_ports = (int8)p.n_ports; c.n_rb_dl = (int8)p.n_rb_dl;
  c.phich_duration = (phich_duration_t::phich_duration_t)p.phich_duration;
  c.phich_resource = (phich_resource_t::phich_resource_t)p.phich_resource; c.sfn = (int16)p.sfn;
  return c;
}

// lcs_meas_cells on every cell of cells[c], found in channel c of iq ([cells.size()][n_cap][2]); meas[c][k] is the k-th
// cell's.  Returns the status and sets *where for check().
static lcs_status measure_lists(const void* iq, int iq_format, int on_device, uint32_t n_cap,
                                const std::vector<std::list<Cell> >& cells, double fs_programmed,
                                std::vector<std::vector<lcs_cell_meas> >& meas, const char** where) {
  std::vector<lcs_cell> flat;
  std::vector<uint32_t> ch;
  for (size_t c = 0; c < cells.size(); c++)
    for (const Cell& cell : cells[c]) {
      flat.push_back(to_pod(cell));
      ch.push_back((uint32_t)c);
    }
  std::vector<lcs_cell_meas> out(flat.size());
  lcs_meas* m = nullptr;
  *where = "lcs_meas_create";
  lcs_status rc = lcs_meas_create(lcs_dropin_ctx(), &m);
  if (rc == LCS_OK) {
    rc = lcs_meas_cells(m, iq, iq_format, on_device, (uint32_t)cells.size(), n_cap, flat.data(), ch.data(),
                        (uint32_t)flat.size(), fs_programmed, out.data());
    *where = "lcs_meas_cells";
  }
  if (m) lcs_meas_destroy(m);
  meas.assign(cells.size(), std::vector<lcs_cell_meas>());
  for (size_t i = 0; i < flat.size(); i++) meas[ch[i]].push_back(out[i]);
  return rc;
}

void measure_cells(const void* iq, int iq_format, uint32_t n_cap, const std::vector<std::list<Cell> >& detected_cells,
                   const double& fs_programmed, std::vector<std::vector<lcs_cell_meas> >& meas) {
  const char* where = "";
  check(measure_lists(iq, iq_format, 0, n_cap, detected_cells, fs_programmed, meas, &where), where);
}

// One measurement of the wideband recording (lcs_carrier_cells, lcs_cir_cells, lcs_pcfich_cells, lcs_pdcch_cells or
// lcs_sib1_cells, through
// handle type H) of every cell of `cells`: all in one call, and when a cell is rejected each on its own, so that only the rejected ones go
// unmeasured.
template <class H, class M, class Create, class Cells, class Destroy>
static void measure_recording(Create create, Cells cells_fn, Destroy destroy, const char* what, const void* iq, int iq_format,
                              uint64_t n, double fs_in, double fc_in, const std::vector<Cell>& cells,
                              const double& fs_programmed, std::vector<M>& meas, std::vector<bool>& ok) {
  std::vector<lcs_cell> flat;
  for (const Cell& c : cells) flat.push_back(to_pod(c));
  meas.assign(flat.size(), M());
  ok.assign(flat.size(), true);
  if (flat.empty()) return;
  H* h = nullptr;
  check(create(lcs_dropin_ctx(), &h), (std::string(what) + "_create").c_str());
  lcs_status rc = cells_fn(h, iq, iq_format, 0, n, fs_in, fc_in, flat.data(), (uint32_t)flat.size(), fs_programmed,
                           meas.data());
  if (rc == LCS_ERR_ARG) {
    rc = LCS_OK;
    for (size_t i = 0; i < flat.size() && rc == LCS_OK; i++) {
      const lcs_status r = cells_fn(h, iq, iq_format, 0, n, fs_in, fc_in, &flat[i], 1, fs_programmed, &meas[i]);
      ok[i] = r == LCS_OK;
      if (r != LCS_ERR_ARG) rc = r;
    }
  }
  destroy(h);
  check(rc, (std::string(what) + "_cells").c_str());
}

void measure_carriers(const void* iq, int iq_format, uint64_t n, double fs_in, double fc_in, const std::vector<Cell>& cells,
                      const double& fs_programmed, std::vector<lcs_carrier_meas>& meas, std::vector<bool>& ok) {
  measure_recording<lcs_carrier>(lcs_carrier_create, lcs_carrier_cells, lcs_carrier_destroy, "lcs_carrier", iq, iq_format, n,
                                 fs_in, fc_in, cells, fs_programmed, meas, ok);
}

void measure_cirs(const void* iq, int iq_format, uint64_t n, double fs_in, double fc_in, const std::vector<Cell>& cells,
                  const double& fs_programmed, std::vector<lcs_cir_meas>& meas, std::vector<bool>& ok) {
  measure_recording<lcs_cir>(lcs_cir_create, lcs_cir_cells, lcs_cir_destroy, "lcs_cir", iq, iq_format, n, fs_in, fc_in, cells,
                             fs_programmed, meas, ok);
}

void measure_pcfich(const void* iq, int iq_format, uint64_t n, double fs_in, double fc_in, const std::vector<Cell>& cells,
                    const double& fs_programmed, std::vector<lcs_pcfich_meas>& meas, std::vector<bool>& ok) {
  measure_recording<lcs_pcfich>(lcs_pcfich_create, lcs_pcfich_cells, lcs_pcfich_destroy, "lcs_pcfich", iq, iq_format, n, fs_in,
                                fc_in, cells, fs_programmed, meas, ok);
}

void measure_pdcch(const void* iq, int iq_format, uint64_t n, double fs_in, double fc_in, const std::vector<Cell>& cells,
                   const double& fs_programmed, std::vector<lcs_pdcch_meas>& meas, std::vector<bool>& ok) {
  measure_recording<lcs_pdcch>(lcs_pdcch_create, lcs_pdcch_cells, lcs_pdcch_destroy, "lcs_pdcch", iq, iq_format, n, fs_in,
                               fc_in, cells, fs_programmed, meas, ok);
}

void measure_sib1(const void* iq, int iq_format, uint64_t n, double fs_in, double fc_in, const std::vector<Cell>& cells,
                  const double& fs_programmed, std::vector<lcs_sib1_meas>& meas, std::vector<bool>& ok) {
  measure_recording<lcs_sib1>(lcs_sib1_create, lcs_sib1_cells, lcs_sib1_destroy, "lcs_sib1", iq, iq_format, n, fs_in, fc_in,
                              cells, fs_programmed, meas, ok);
}

void sweep_search_cu8(const std::vector<unsigned char>& iq, uint32_t n_cap, const std::vector<double>& fc_requested,
                      const vec& f_search_set, const double& fs_programmed, std::vector<std::list<Cell> >& detected_cells) {
  const uint32_t n_ch = (uint32_t)fc_requested.size(), max_cells = 16;
  if (iq.size() < (size_t)n_ch * n_cap * 2) throw("sweep_search_cu8: capture data shorter than n_fc buffers");
  lcs_sweep* sw = nullptr;
  check(lcs_sweep_create(lcs_dropin_ctx(), n_cap, &sw), "lcs_sweep_create");
  std::vector<lcs_cell> cells((size_t)n_ch * max_cells);
  std::vector<uint32_t> n(n_ch, 0);
  lcs_status rc = lcs_sweep_search_cu8(sw, iq.data(), n_ch, fc_requested.data(), nullptr, fs_programmed, f_search_set._data(),
                                       (uint32_t)f_search_set.length(), cells.data(), max_cells, n.data());
  lcs_sweep_destroy(sw);
  check(rc, "lcs_sweep_search_cu8");
  detected_cells.assign(n_ch, std::list<Cell>());
  for (uint32_t c = 0; c < n_ch; c++)
    for (uint32_t k = 0; k < n[c] && k < max_cells; k++) detected_cells[c].push_back(from_pod(cells[(size_t)c * max_cells + k]));
}

// iq_format < 0: lcs_chan_create (ci16 at D * 1.92 MHz); otherwise lcs_chan_create_rational with that format
static void wideband_search(const void* iq, int iq_format, uint32_t n, double fs_in, double fc_in,
                            const std::vector<double>& fc_requested, const vec& f_search_set, const double& fs_programmed,
                            std::vector<std::list<Cell> >& detected_cells, std::vector<std::vector<lcs_cell_meas> >* meas) {
  const uint32_t n_ch = (uint32_t)fc_requested.size(), max_cells = 16, n_cap = 153600;
  lcs_ctx* ctx = lcs_dropin_ctx();
  lcs_chan* ch = nullptr;
  lcs_sweep* sw = nullptr;
  uint8_t* d_iq = nullptr;
  std::vector<lcs_cell> cells((size_t)n_ch * max_cells);
  std::vector<uint32_t> found(n_ch, 0);
  uint32_t n_out = 0;
  lcs_status rc;
  const char* where;
  if (iq_format < 0) {
    rc = lcs_chan_create(ctx, fs_in, fc_in, n_ch, fc_requested.data(), nullptr, &ch);
    where = "lcs_chan_create";
  } else {
    rc = lcs_chan_create_rational(ctx, fs_in, iq_format, fc_in, n_ch, fc_requested.data(), nullptr, &ch);
    where = "lcs_chan_create_rational";
  }
  if (rc == LCS_OK) { rc = lcs_chan_auto_gain(ch, iq, n); where = "lcs_chan_auto_gain"; }
  if (rc == LCS_OK && cudaMalloc((void**)&d_iq, (size_t)n_ch * n_cap * 2) != cudaSuccess) {
    d_iq = nullptr;
    rc = LCS_ERR_CUDA;
    where = "cudaMalloc";
  }
  if (rc == LCS_OK) { rc = lcs_chan_push(ch, iq, n, d_iq, n_cap, 1, &n_out, nullptr); where = "lcs_chan_push"; }
  if (rc == LCS_OK && n_out != n_cap) { rc = LCS_ERR_ARG; where = "lcs_chan_push (recording too short)"; }
  if (rc == LCS_OK) { rc = lcs_sweep_create(ctx, n_cap, &sw); where = "lcs_sweep_create"; }
  if (rc == LCS_OK) {
    rc = lcs_sweep_search_cu8_device(sw, d_iq, n_ch, fc_requested.data(), nullptr, fs_programmed, f_search_set._data(),
                                     (uint32_t)f_search_set.length(), cells.data(), max_cells, found.data());
    where = "lcs_sweep_search_cu8_device";
  }
  if (rc == LCS_OK) {
    detected_cells.assign(n_ch, std::list<Cell>());
    for (uint32_t c = 0; c < n_ch; c++)
      for (uint32_t k = 0; k < found[c] && k < max_cells; k++) detected_cells[c].push_back(from_pod(cells[(size_t)c * max_cells + k]));
  }
  // measured on the channelized buffers in place, then brought back to the recording's full scale: channel c's bytes
  // carry gain[c] times the recording
  std::vector<float> gain(n_ch);
  if (rc == LCS_OK && meas) rc = measure_lists(d_iq, LCS_IQ_CU8, 1, n_cap, detected_cells, fs_programmed, *meas, &where);
  if (rc == LCS_OK && meas) { rc = lcs_chan_gain(ch, gain.data()); where = "lcs_chan_gain"; }
  if (rc == LCS_OK && meas)
    for (uint32_t c = 0; c < n_ch; c++)
      for (lcs_cell_meas& m : (*meas)[c]) {
        const double g2 = (double)gain[c] * gain[c];
        for (int p = 0; p < 4; p++) { m.rsrp[p] /= g2; m.noise[p] /= g2; }
        m.rssi /= g2;
      }
  if (sw) lcs_sweep_destroy(sw);
  if (d_iq) cudaFree(d_iq);
  if (ch) lcs_chan_destroy(ch);
  check(rc, where);
}

void wideband_search_ci16(const int16_t* iq, uint32_t n, double fs_in, double fc_in, const std::vector<double>& fc_requested,
                          const vec& f_search_set, const double& fs_programmed, std::vector<std::list<Cell> >& detected_cells,
                          std::vector<std::vector<lcs_cell_meas> >* meas) {
  wideband_search(iq, -1, n, fs_in, fc_in, fc_requested, f_search_set, fs_programmed, detected_cells, meas);
}

void wideband_search_rational(const void* iq, int iq_format, uint32_t n, double fs_in, double fc_in,
                              const std::vector<double>& fc_requested, const vec& f_search_set,
                              const double& fs_programmed, std::vector<std::list<Cell> >& detected_cells,
                              std::vector<std::vector<lcs_cell_meas> >* meas) {
  wideband_search(iq, iq_format, n, fs_in, fc_in, fc_requested, f_search_set, fs_programmed, detected_cells, meas);
}

void wideband_psd(const std::string& path, int iq_format, size_t es, double fs_in, uint32_t nfft, std::vector<double>& psd,
                  uint64_t& n_segments) {
  const size_t block = (size_t)1 << 22;                              // samples per push
  FILE* f = std::fopen(path.c_str(), "rb");
  if (!f) throw("wideband_psd: cannot read the recording");
  lcs_psd* p = nullptr;
  lcs_status rc = lcs_psd_create(lcs_dropin_ctx(), fs_in, iq_format, nfft, &p);
  const char* where = "lcs_psd_create";
  std::vector<unsigned char> buf(block * es);
  while (rc == LCS_OK) {
    const size_t got = std::fread(buf.data(), es, block, f);
    if (!got) break;
    rc = lcs_psd_push(p, buf.data(), (uint32_t)got);
    where = "lcs_psd_push";
  }
  std::fclose(f);
  psd.assign(nfft, 0.0);
  if (rc == LCS_OK) { rc = lcs_psd_read(p, psd.data(), &n_segments); where = "lcs_psd_read"; }
  if (p) lcs_psd_destroy(p);
  check(rc, where);
}

// ---- searcher.h:22-41 ----
void xcorr_pss(const cvec& capbuf, const vec& f_search_set, const uint8& ds_comb_arm, const double& fc_requested,
               const double& fc_programmed, const double& fs_programmed, mat& xc_incoherent_collapsed_pow,
               imat& xc_incoherent_collapsed_frq, vf3d& xc_incoherent_single, vf3d& xc_incoherent, vec& sp_incoherent,
               vcf3d& xc, vec& sp, uint16& n_comb_xc, uint16& n_comb_sp) {
  lcs_ctx* ctx = lcs_dropin_ctx();
  const uint32_t n_cap = (uint32_t)capbuf.length(), n_f = (uint32_t)f_search_set.length();
  xc_incoherent_collapsed_pow.set_size(3, LCS_N_FOLD);
  xc_incoherent_collapsed_frq.set_size(3, LCS_N_FOLD);
  sp_incoherent.set_size(LCS_N_FOLD);
  std::vector<float> single((size_t)3 * LCS_N_FOLD * n_f), inc, xcf;
  std::vector<double> spv;
  if (!g_skip_debug) {
    inc.resize(single.size());
    xcf.resize((size_t)3 * (n_cap - 136) * n_f * 2);
    spv.resize((size_t)((n_cap - 273) / LCS_N_FOLD) * LCS_N_FOLD);
  }
  check(lcs_xcorr_pss(ctx, reinterpret_cast<const double*>(capbuf._data()), n_cap, f_search_set._data(), n_f, ds_comb_arm,
                      fc_requested, fc_programmed, fs_programmed, xc_incoherent_collapsed_pow._data(),
                      xc_incoherent_collapsed_frq._data(), single.data(), g_skip_debug ? nullptr : inc.data(),
                      sp_incoherent._data(), g_skip_debug ? nullptr : xcf.data(), g_skip_debug ? nullptr : spv.data(),
                      &n_comb_xc, &n_comb_sp),
        "xcorr_pss");
  auto unpack = [&](const std::vector<float>& src, vf3d& dst) {
    dst.assign(3, std::vector<std::vector<float> >(LCS_N_FOLD, std::vector<float>(n_f)));
    for (int t = 0; t < 3; t++)
      for (int i = 0; i < LCS_N_FOLD; i++)
        std::memcpy(dst[t][i].data(), &src[((size_t)t * LCS_N_FOLD + i) * n_f], n_f * sizeof(float));
  };
  unpack(single, xc_incoherent_single);
  if (!g_skip_debug) {
    unpack(inc, xc_incoherent);
    const uint32_t n_lag = n_cap - 136;
    xc.assign(3, std::vector<std::vector<complex<float> > >(n_lag, std::vector<complex<float> >(n_f)));
    for (int t = 0; t < 3; t++)
      for (uint32_t k = 0; k < n_lag; k++)
        std::memcpy(static_cast<void*>(xc[t][k].data()), &xcf[(((size_t)t * n_lag + k) * n_f) * 2], n_f * 2 * sizeof(float));
    sp.set_size((int)spv.size());
    std::memcpy(sp._data(), spv.data(), spv.size() * 8);
  }
}

// ---- searcher.h:44-56 ----
void peak_search(const mat& pow, const imat& frq, const vec& Z_th1, const vec& f_search_set, const double& fc_requested,
                 const double& fc_programmed, const vf3d& xc_incoherent_single, const uint8& ds_comb_arm,
                 std::list<Cell>& cells) {
  const uint32_t n_f = (uint32_t)f_search_set.length();
  std::vector<double> pw((size_t)3 * LCS_N_FOLD);
  std::vector<int32_t> fq((size_t)3 * LCS_N_FOLD);
  std::vector<float> planar((size_t)3 * n_f * LCS_N_FOLD);
  for (int t = 0; t < 3; t++)
    for (int i = 0; i < LCS_N_FOLD; i++) {
      pw[(size_t)t * LCS_N_FOLD + i] = pow(t, i);
      fq[(size_t)t * LCS_N_FOLD + i] = frq(t, i);
      for (uint32_t f = 0; f < n_f; f++) planar[((size_t)t * n_f + f) * LCS_N_FOLD + i] = xc_incoherent_single[t][i][f];
    }
  std::vector<lcs_cell> out(256);
  uint32_t n = 0;
  check(lcs_peak_search(pw.data(), fq.data(), Z_th1._data(), f_search_set._data(), n_f, fc_requested, fc_programmed,
                        planar.data(), ds_comb_arm, out.data(), (uint32_t)out.size(), &n),
        "peak_search");
  for (uint32_t i = 0; i < n && i < out.size(); i++) cells.push_back(from_pod(out[i]));   // appends (searcher.cpp:476)
}

// ---- searcher.h:59-76 ----
Cell sss_detect(const Cell& cell, const cvec& capbuf, const double& thresh2_n_sigma, const double& fc_requested,
                const double& fc_programmed, const double& fs_programmed, vec& h1_np, vec& h2_np, cvec& h1_nrm,
                cvec& h2_nrm, cvec& h1_ext, cvec& h2_ext, mat& log_lik_nrm, mat& log_lik_ext) {
  h1_np.set_size(62); h2_np.set_size(62);
  h1_nrm.set_size(62); h2_nrm.set_size(62); h1_ext.set_size(62); h2_ext.set_size(62);
  log_lik_nrm.set_size(168, 2); log_lik_ext.set_size(168, 2);
  lcs_cell in = to_pod(cell), out;
  check(lcs_sss_detect(lcs_dropin_ctx(), &in, reinterpret_cast<const double*>(capbuf._data()), (uint32_t)capbuf.length(),
                       thresh2_n_sigma, fc_requested, fc_programmed, fs_programmed, &out, h1_np._data(), h2_np._data(),
                       reinterpret_cast<double*>(h1_nrm._data()), reinterpret_cast<double*>(h2_nrm._data()),
                       reinterpret_cast<double*>(h1_ext._data()), reinterpret_cast<double*>(h2_ext._data()),
                       log_lik_nrm._data(), log_lik_ext._data()),
        "sss_detect");
  return from_pod(out);
}

// ---- searcher.h:79-85 ----
Cell pss_sss_foe(const Cell& cell_in, const cvec& capbuf, const double& fc_requested, const double& fc_programmed,
                 const double& fs_programmed) {
  if (cell_in.cp_type == cp_type_t::UNKNOWN) throw("Error... check code...");   // searcher.cpp:786
  lcs_cell in = to_pod(cell_in), out;
  check(lcs_pss_sss_foe(lcs_dropin_ctx(), &in, reinterpret_cast<const double*>(capbuf._data()), (uint32_t)capbuf.length(),
                        fc_requested, fc_programmed, fs_programmed, &out),
        "pss_sss_foe");
  return from_pod(out);
}

// ---- searcher.h:88-98 ----
void extract_tfg(const Cell& cell, const cvec& capbuf_raw, const double& fc_requested, const double& fc_programmed,
                 const double& fs_programmed, cmat& tfg, vec& tfg_timestamp) {
  if (cell.cp_type == cp_type_t::UNKNOWN) throw("Check code...");   // searcher.cpp:883
  const int n_ofdm = 6 * 10 * 2 * cell.n_symb_dl() + 2 * cell.n_symb_dl();
  tfg.set_size(n_ofdm, 72);
  tfg_timestamp.set_size(n_ofdm);
  lcs_cell in = to_pod(cell);
  uint32_t n = 0;
  check(lcs_extract_tfg(lcs_dropin_ctx(), &in, reinterpret_cast<const double*>(capbuf_raw._data()),
                        (uint32_t)capbuf_raw.length(), fc_requested, fc_programmed, fs_programmed,
                        reinterpret_cast<double*>(tfg._data()), tfg_timestamp._data(), &n),
        "extract_tfg");
}

// ---- searcher.h:101-112 ----
Cell tfoec(const Cell& cell, const cmat& tfg, const vec& tfg_timestamp, const double& fc_requested,
           const double& fc_programmed, const RS_DL& rs_dl, cmat& tfg_comp, vec& tfg_comp_timestamp) {
  (void)rs_dl;   // tables are rebuilt inside the library from (n_id_cell, cp_type)
  tfg_comp.set_size(tfg.rows(), 72);
  tfg_comp_timestamp.set_size(tfg.rows());
  lcs_cell in = to_pod(cell), out;
  check(lcs_tfoec(lcs_dropin_ctx(), &in, reinterpret_cast<const double*>(tfg._data()), tfg_timestamp._data(),
                  (uint32_t)tfg.rows(), fc_requested, fc_programmed, reinterpret_cast<double*>(tfg_comp._data()),
                  tfg_comp_timestamp._data(), &out),
        "tfoec");
  return from_pod(out);
}

// ---- searcher.h:115-119 ----
Cell decode_mib(const Cell& cell, const cmat& tfg, const RS_DL& rs_dl) {
  (void)rs_dl;
  lcs_cell in = to_pod(cell), out;
  check(lcs_decode_mib(lcs_dropin_ctx(), &in, reinterpret_cast<const double*>(tfg._data()), (uint32_t)tfg.rows(), &out),
        "decode_mib");
  return from_pod(out);
}

// ---- searcher.h:122-124 (searcher.cpp:1072-1083) ----
void del_oob(ivec& v) {
  ivec r(v.length());
  int n = 0;
  for (int t = 0; t < v.length(); t++)
    if (!(v(t) < 0 || v(t) > 11)) r(n++) = v(t);
  v.set_size(n);
  for (int t = 0; t < n; t++) v(t) = r(t);
}

// ---- CellSearch.cpp glue ----
void dedup(const std::vector<std::list<Cell> >& detected_cells, std::list<Cell>& cells_final) {
  std::vector<lcs_cell> flat;
  for (const auto& l : detected_cells)
    for (const Cell& c : l) flat.push_back(to_pod(c));
  std::vector<lcs_cell> out(flat.size() + 1);
  uint32_t n = 0;
  check(lcs_dedup(flat.data(), (uint32_t)flat.size(), out.data(), &n), "dedup");
  cells_final.clear();
  for (uint32_t i = 0; i < n; i++) cells_final.push_back(from_pod(out[i]));
}

vec calc_Z_th1(const vec& sp_incoherent, uint16 n_comb_xc, uint8 ds_comb_arm) {
  vec z(sp_incoherent.length());
  check(lcs_calc_z_th1(sp_incoherent._data(), (uint32_t)sp_incoherent.length(), n_comb_xc, ds_comb_arm, z._data()), "calc_Z_th1");
  return z;
}
