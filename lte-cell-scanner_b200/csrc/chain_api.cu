// chain_api.cu - C-ABI entry points for the stages after xcorr_pss (include/lcs_b200.h).
#include <algorithm>
#include <atomic>
#include <cmath>
#include <cstring>
#include <thread>

#include "chain_gpu.hpp"

namespace lcs {

static void to_colmajor(const std::vector<cd>& rowmajor, int n_rows, int n_cols, double* out) {
  cd* o = reinterpret_cast<cd*>(out);
  for (int r = 0; r < n_rows; r++)
    for (int c = 0; c < n_cols; c++) o[(size_t)c * n_rows + r] = rowmajor[(size_t)r * n_cols + c];
}
static std::vector<cd> from_colmajor(const double* in, int n_rows, int n_cols) {
  const cd* i = reinterpret_cast<const cd*>(in);
  std::vector<cd> r((size_t)n_rows * n_cols);
  for (int a = 0; a < n_rows; a++)
    for (int c = 0; c < n_cols; c++) r[(size_t)a * n_cols + c] = i[(size_t)c * n_rows + a];
  return r;
}

// Per-peak stages of CellSearch.cpp:510-558 (sss_detect -> pss_sss_foe -> extract_tfg -> tfoec -> decode_mib) on a
// device-resident capture buffer; cells that fail the SSS or MIB tests are dropped like in the reference.
// Two phases: the device stages run on sc.st, each for all peaks at once; the host stages (tfoec, chan_est, PBCH decoding
// with its 12 tail-biting Viterbi attempts - milliseconds per cell) of all surviving peaks then run on parallel threads.
lcs_status cell_chain_dev(const StageCall& sc, const std::vector<lcs_cell>& pk, lcs_cell* cells, uint32_t max_cells,
                          uint32_t* n_cells, const int32_t* tracked, uint32_t n_tracked, bool tracker_cycle) {
  const double THRESH2_N_SIGMA = 3;     // CellSearch.cpp:528
  lcs_status rc = LCS_OK;
  if (n_cells) *n_cells = 0;
  if (pk.empty()) return LCS_OK;
  struct Pending {
    lcs_cell c;                      // after pss_sss_foe
    std::vector<cd> tfg;
    std::vector<double> ts;
    lcs_cell out{};                  // after decode_mib
  };
  // device stages, each for all peaks at once
  std::vector<lcs_cell> det;
  std::vector<lcs_status> st1;
  rc = dev_sss_detect_batch(sc, pk, THRESH2_N_SIGMA, det, st1, nullptr);
  if (rc != LCS_OK) return rc;
  std::vector<lcs_cell> surv;
  for (size_t i = 0; i < pk.size(); i++) {
    if (st1[i] == LCS_ERR_RANGE) continue;   // the reference would index outside the buffer here
    if (det[i].n_id_1 == -1) continue;       // CellSearch.cpp:530-534
    // searcher_thread.cpp:153-174: cells that are being tracked are not examined further
    bool already_tracked = false;
    for (uint32_t k = 0; k < n_tracked; k++) already_tracked |= tracked[k] == det[i].n_id_2 + 3 * det[i].n_id_1;
    if (already_tracked) continue;
    surv.push_back(det[i]);
  }
  std::vector<lcs_cell> foe;
  rc = dev_pss_sss_foe_batch(sc, surv, foe);
  if (rc != LCS_OK) return rc;
  std::vector<std::vector<cd>> tfgs;
  std::vector<std::vector<double>> tss;
  std::vector<lcs_status> st3;
  rc = dev_extract_tfg_batch(sc, foe, tfgs, tss, st3);
  if (rc != LCS_OK) return rc;
  std::vector<Pending> pend;
  pend.reserve(foe.size());
  for (size_t i = 0; i < foe.size(); i++) {
    if (st3[i] == LCS_ERR_RANGE) continue;
    Pending q;
    q.c = foe[i];
    q.tfg.swap(tfgs[i]);
    q.ts.swap(tss[i]);
    pend.push_back(std::move(q));
  }
  auto host_stage = [&](Pending& q) {
    RsDl rs(q.c.n_id_2 + 3 * q.c.n_id_1, q.c.cp_type);  // CellSearch.cpp:545
    std::vector<cd> tfg_comp(q.tfg.size());
    std::vector<double> ts_comp(q.ts.size());
    lcs_cell o;
    tfoec(q.c, q.tfg.data(), q.ts.data(), (int)q.ts.size(), sc.cfg.fc_req, sc.cfg.fc_prog, rs, tfg_comp.data(), ts_comp.data(), o);
    decode_mib(o, tfg_comp.data(), (int)q.ts.size(), rs, q.out);
  };
  if (pend.size() <= 1) {
    for (Pending& q : pend) host_stage(q);
  } else {
    const unsigned hw = std::max(1u, std::thread::hardware_concurrency());
    const size_t n_thr = std::min<size_t>(pend.size(), hw);
    std::atomic<size_t> next{0};
    std::vector<std::thread> pool;
    for (size_t t = 0; t < n_thr; t++)
      pool.emplace_back([&] {
        for (size_t i = next.fetch_add(1); i < pend.size(); i = next.fetch_add(1)) host_stage(pend[i]);
      });
    for (std::thread& th : pool) th.join();
  }
  // In tracker mode the reference appends every new cell to tracked_cell_list inside its peak loop
  // (searcher_thread.cpp:216-219): a later peak of the same buffer that decodes to an id accepted earlier is skipped.
  uint32_t found = 0;
  std::vector<int> accepted_ids;
  for (Pending& q : pend) {
    if (q.out.n_rb_dl == -1) continue;  // CellSearch.cpp:554-558
    const int id = q.out.n_id_2 + 3 * q.out.n_id_1;
    if (tracker_cycle && std::find(accepted_ids.begin(), accepted_ids.end(), id) != accepted_ids.end()) continue;
    if (found < max_cells && cells) cells[found] = q.out;
    found++;
    accepted_ids.push_back(id);
  }
  if (n_cells) *n_cells = found;
  return LCS_OK;
}

}  // namespace lcs

using namespace lcs;

extern "C" {

lcs_status lcs_calc_z_th1(const double* sp_incoherent, uint32_t n, uint16_t n_comb_xc, uint8_t ds_comb_arm, double* z) {
  if (!sp_incoherent || !z || n_comb_xc == 0) return fail(nullptr, LCS_ERR_ARG, "calc_z_th1: bad argument");
  calc_z_th1(sp_incoherent, n, n_comb_xc, ds_comb_arm, z);
  return LCS_OK;
}

lcs_status lcs_peak_search(const double* pow, const int32_t* frq, const double* z_th1, const double* f_search_set,
                           uint32_t n_f, double fc_requested, double fc_programmed, const float* single_planar,
                           uint8_t ds_comb_arm, lcs_cell* cells, uint32_t max_cells, uint32_t* n_cells) {
  if (!pow || !frq || !z_th1 || !f_search_set || !single_planar || !n_cells || n_f == 0)
    return fail(nullptr, LCS_ERR_ARG, "peak_search: bad argument");
  for (uint32_t i = 0; i < 3 * LCS_N_FOLD; i++)
    if (frq[i] < 0 || (uint32_t)frq[i] >= n_f) return fail(nullptr, LCS_ERR_ARG, "peak_search: frq index out of range");
  std::vector<lcs_cell> v;
  auto at = [&](int t, int f, int idx) { return single_planar[((size_t)t * n_f + f) * LCS_N_FOLD + idx]; };
  peak_search(pow, frq, z_th1, f_search_set, fc_requested, fc_programmed, at, ds_comb_arm, v);
  for (size_t i = 0; i < v.size() && i < max_cells && cells; i++) cells[i] = v[i];
  *n_cells = (uint32_t)v.size();
  return LCS_OK;
}

lcs_status lcs_sss_detect(lcs_ctx* ctx, const lcs_cell* cell, const double* capbuf, uint32_t n_cap, double thresh2_n_sigma,
                          double fc_requested, double fc_programmed, double fs_programmed, lcs_cell* cell_out,
                          double* h1_np, double* h2_np, double* h1_nrm, double* h2_nrm, double* h1_ext, double* h2_ext,
                          double* log_lik_nrm, double* log_lik_ext) {
  if (!ctx || !cell || !capbuf || !cell_out) return fail(ctx, LCS_ERR_ARG, "sss_detect: null argument");
  const cudaStream_t st = ctx->streams[0];
  lcs_status rc = upload_c128(ctx, capbuf, n_cap, st);
  if (rc != LCS_OK) return rc;
  const PlanCfg cfg{fc_requested, fc_programmed, fs_programmed};
  std::vector<lcs_cell> out;
  std::vector<lcs_status> status;
  SssDebugHost d;
  rc = dev_sss_detect_batch(StageCall{ctx, ctx->d_capbuf.p, LCS_IQ_C128, n_cap, cfg, st}, {*cell}, thresh2_n_sigma, out, status, &d);
  if (rc != LCS_OK) return rc;
  if (status[0] != LCS_OK) return fail(ctx, status[0], "sss_detect: DFT window outside the capture buffer");
  *cell_out = out[0];
  if (h1_np) std::memcpy(h1_np, &d.est[0], 62 * 8);
  if (h2_np) std::memcpy(h2_np, &d.est[62], 62 * 8);
  if (h1_nrm) std::memcpy(h1_nrm, &d.est[124], 62 * 16);
  if (h2_nrm) std::memcpy(h2_nrm, &d.est[248], 62 * 16);
  if (h1_ext) std::memcpy(h1_ext, &d.est[372], 62 * 16);
  if (h2_ext) std::memcpy(h2_ext, &d.est[496], 62 * 16);
  if (log_lik_nrm) std::memcpy(log_lik_nrm, &d.ll[0], 336 * 8);    // mat(168,2) column-major = [col0][col1]
  if (log_lik_ext) std::memcpy(log_lik_ext, &d.ll[336], 336 * 8);
  return LCS_OK;
}

lcs_status lcs_pss_sss_foe(lcs_ctx* ctx, const lcs_cell* cell_in, const double* capbuf, uint32_t n_cap, double fc_requested,
                           double fc_programmed, double fs_programmed, lcs_cell* cell_out) {
  if (!ctx || !cell_in || !capbuf || !cell_out) return fail(ctx, LCS_ERR_ARG, "pss_sss_foe: null argument");
  const cudaStream_t st = ctx->streams[0];
  lcs_status rc = upload_c128(ctx, capbuf, n_cap, st);
  if (rc != LCS_OK) return rc;
  const PlanCfg cfg{fc_requested, fc_programmed, fs_programmed};
  std::vector<lcs_cell> out;
  rc = dev_pss_sss_foe_batch(StageCall{ctx, ctx->d_capbuf.p, LCS_IQ_C128, n_cap, cfg, st}, {*cell_in}, out);
  if (rc != LCS_OK) return rc;
  *cell_out = out[0];
  return LCS_OK;
}

lcs_status lcs_extract_tfg(lcs_ctx* ctx, const lcs_cell* cell, const double* capbuf, uint32_t n_cap, double fc_requested,
                           double fc_programmed, double fs_programmed, double* tfg, double* tfg_timestamp,
                           uint32_t* n_ofdm_out) {
  if (!ctx || !cell || !capbuf || !tfg || !tfg_timestamp) return fail(ctx, LCS_ERR_ARG, "extract_tfg: null argument");
  const cudaStream_t st = ctx->streams[0];
  lcs_status rc = upload_c128(ctx, capbuf, n_cap, st);
  if (rc != LCS_OK) return rc;
  const PlanCfg cfg{fc_requested, fc_programmed, fs_programmed};
  std::vector<std::vector<cd>> g;
  std::vector<std::vector<double>> ts;
  std::vector<lcs_status> status;
  rc = dev_extract_tfg_batch(StageCall{ctx, ctx->d_capbuf.p, LCS_IQ_C128, n_cap, cfg, st}, {*cell}, g, ts, status);
  if (rc != LCS_OK) return rc;
  if (status[0] != LCS_OK) return fail(ctx, status[0], "extract_tfg: DFT window outside the capture buffer");
  to_colmajor(g[0], (int)ts[0].size(), 72, tfg);
  std::memcpy(tfg_timestamp, ts[0].data(), ts[0].size() * 8);
  if (n_ofdm_out) *n_ofdm_out = (uint32_t)ts[0].size();
  return LCS_OK;
}

lcs_status lcs_tfoec(lcs_ctx* ctx, const lcs_cell* cell, const double* tfg, const double* tfg_timestamp, uint32_t n_ofdm,
                     double fc_requested, double fc_programmed, double* tfg_comp, double* tfg_comp_timestamp,
                     lcs_cell* cell_out) {
  if (!cell || !tfg || !tfg_timestamp || !tfg_comp || !tfg_comp_timestamp || !cell_out)
    return fail(ctx, LCS_ERR_ARG, "tfoec: null argument");
  if (cell->cp_type != 1 && cell->cp_type != 2) return fail(ctx, LCS_ERR_ARG, "tfoec: cp_type unknown");
  if (cell->n_id_1 < 0 || cell->n_id_2 < 0) return fail(ctx, LCS_ERR_ARG, "tfoec: cell id not set");
  const int n_symb = cell->cp_type == 1 ? 7 : 6;
  if (n_ofdm < (uint32_t)(2 * n_symb)) return fail(ctx, LCS_ERR_ARG, "tfoec: grid too short");
  std::vector<cd> g = from_colmajor(tfg, (int)n_ofdm, 72), gc(g.size());
  RsDl rs(cell->n_id_2 + 3 * cell->n_id_1, cell->cp_type);
  tfoec(*cell, g.data(), tfg_timestamp, (int)n_ofdm, fc_requested, fc_programmed, rs, gc.data(), tfg_comp_timestamp, *cell_out);
  to_colmajor(gc, (int)n_ofdm, 72, tfg_comp);
  return LCS_OK;
}

lcs_status lcs_decode_mib(lcs_ctx* ctx, const lcs_cell* cell, const double* tfg, uint32_t n_ofdm, lcs_cell* cell_out) {
  if (!cell || !tfg || !cell_out) return fail(ctx, LCS_ERR_ARG, "decode_mib: null argument");
  if (cell->cp_type != 1 && cell->cp_type != 2) return fail(ctx, LCS_ERR_ARG, "decode_mib: cp_type unknown");
  if (cell->n_id_1 < 0 || cell->n_id_2 < 0) return fail(ctx, LCS_ERR_ARG, "decode_mib: cell id not set");
  const int n_symb = cell->cp_type == 1 ? 7 : 6;
  if (n_ofdm < (uint32_t)(6 * 20 * n_symb + 2 * n_symb)) return fail(ctx, LCS_ERR_ARG, "decode_mib: grid shorter than 6 frames + 2 slots");
  std::vector<cd> g = from_colmajor(tfg, (int)n_ofdm, 72);
  RsDl rs(cell->n_id_2 + 3 * cell->n_id_1, cell->cp_type);
  decode_mib(*cell, g.data(), (int)n_ofdm, rs, *cell_out);
  return LCS_OK;
}

lcs_status lcs_dedup(const lcs_cell* cells, uint32_t n, lcs_cell* out, uint32_t* n_out) {
  if ((!cells && n) || !out || !n_out) return fail(nullptr, LCS_ERR_ARG, "dedup: null argument");
  std::vector<lcs_cell> fin;
  dedup(cells, n, fin);
  for (size_t i = 0; i < fin.size(); i++) out[i] = fin[i];
  *n_out = (uint32_t)fin.size();
  return LCS_OK;
}

lcs_status lcs_f_search_set(double freq_start, double ppm, double* out, uint32_t* n_f) {
  if (!n_f) return fail(nullptr, LCS_ERR_ARG, "f_search_set: null n_f");
  std::vector<double> f = f_search_set_for(freq_start, ppm);
  if (out) std::memcpy(out, f.data(), f.size() * 8);
  *n_f = (uint32_t)f.size();
  return LCS_OK;
}

}  // extern "C"
