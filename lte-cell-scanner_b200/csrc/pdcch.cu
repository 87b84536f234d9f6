// pdcch.cu - the common-search-space DCIs of found cells in every subframe, decoded from their PDCCH over the whole
// carrier, from the wideband recording they were found in (DESIGN.md section 4.13; contract in include/lcs_pdcch.h).
// Built into liblcs_pdcch.so.
//
// A call is cut into chunks of LCS_PDCCH_CHUNK cells; each chunk makes three launches on the context's stream:
//   1. carrier_grid_kernel (carrier_grid.cuh) on symbols 0 to n_max - 1 of every even slot (pdcch_plan.cpp).
//   2. pcfich_kernel (pcfich_kernel.cuh), unchanged, on the same grid into a device buffer: the CFI of every subframe.
//   3. pdcch_kernel (pdcch_kernel.cuh) on all 61 subframes: one CTA per (cell, subframe).
// The host then parses each DCI's fields and counts the cell's DCIs (rule 13).
#include "pdcch_kernel.cuh"

using namespace lcs;
using namespace lcs::carrier;
using namespace lcs::pdcch;

struct lcs_pdcch : GridModule<lcs_pdcch_meas> {
  DevBuf<lcs_pcfich_meas> d_pc;                  // one chunk's CFI decisions
};

namespace {

// Rule 13 on the host: each DCI's fields and the cell's counts.
void finish(lcs_pdcch_meas& m, int R) {
  m.count[0] = m.count[1] = m.count[2] = 0;
  m.si_subframes = 0;
  for (int s = 0; s < N_SF; s++)
    for (uint32_t i = 0; i < m.n_dci[s]; i++) {
      lcs_pdcch_dci& d = m.dci[s][i];
      parse_dci(d, R);
      if (d.rnti == LCS_RNTI_SI) {
        m.count[0]++;
        m.si_subframes |= 1u << (s % 10);
      } else {
        m.count[d.rnti == LCS_RNTI_P ? 1 : 2]++;
      }
    }
  m.n_subframes = N_SF;
}

}  // namespace

extern "C" {

lcs_status lcs_pdcch_create(lcs_ctx* ctx, lcs_pdcch** out) { return grid_create(ctx, out, "lcs_pdcch_create"); }

void lcs_pdcch_destroy(lcs_pdcch* h) { grid_destroy(h); }

lcs_status lcs_pdcch_cells(lcs_pdcch* h, const void* iq, int iq_format, int on_device, uint64_t n_in, double fs_in,
                           double fc_in, const lcs_cell* cells, uint32_t n_cells, double fs_programmed,
                           lcs_pdcch_meas* out) {
  pcfich::PcfichSlices s{};
  PdcchCell* pd = nullptr;
  return grid_cells(
      h, "lcs_pdcch_cells", CHUNK, LCS_PDCCH_LAUNCHES_PER_CHUNK, iq, iq_format, on_device, n_in, fs_in, fc_in, cells,
      n_cells, fs_programmed, out, plan_pdcch,
      [](uint32_t n) { return pcfich::pcfich_bytes(n) + n * sizeof(PdcchCell) + 16; },
      [&](const GridChunk& c) {
        s = pcfich::pcfich_fill(h->g, c);
        pd = h->g.up.take<PdcchCell>(c.n);
        for (uint32_t i = 0; i < c.n; i++) pd[i] = pdcch_cell(c.plan[i], c.cell[i], c.t.off[i]);
        return h->d_pc.ensure(c.n);              // the first chunk is the largest: it sizes d_pc for the call
      },
      [&](const GridChunk& c) {
        pcfich::pcfich_launch(h->g, c, s, h->d_pc.p);
        pdcch_kernel<N_SF, 1><<<c.n * N_SF, PD_THREADS, 0, c.st>>>(h->g.d_grid.p, h->g.up.dev(c.t.rs), h->g.up.dev(c.t.shift),
                                                          h->g.up.dev(pd), h->d_pc.p, h->d_out.p);
      },
      [](lcs_pdcch_meas& m, const CellPlan& c) { finish(m, c.R); });
}

lcs_status lcs_pdcch_timing_read(lcs_pdcch* h, double* kernel_ms, uint64_t* launches) {
  return grid_timing_read(h, kernel_ms, launches, "lcs_pdcch_timing_read");
}

}  // extern "C"
