// pcfich.cu - the control format indicator of found cells in every subframe, decoded from their PCFICH over the whole
// carrier, from the wideband recording they were found in (DESIGN.md section 4.12; contract in include/lcs_pcfich.h).
// Built into liblcs_pcfich.so.
//
// A call is cut into chunks of LCS_PCFICH_CHUNK cells; each chunk makes two launches on the context's stream:
//   1. carrier_grid_kernel (carrier_grid.cuh) on the windows the decoder reads only: symbol 0 of every even slot, and
//      symbol 1 of it for four ports (a filtered copy of each cell's plan).
//   2. pcfich_kernel (pcfich_kernel.cuh): one CTA per cell, every sum in FP64 in a fixed order, so a cell's record is
//      bitwise the same whatever else the call decodes.
#include "pcfich_kernel.cuh"

using namespace lcs;
using namespace lcs::carrier;
using namespace lcs::pcfich;

struct lcs_pcfich : GridModule<lcs_pcfich_meas> {};

namespace {

// The windows pcfich_kernel reads out of a cell's plan (window order symbol 0, symbol 1 for four ports, symbol
// n_symb - 3): symbol 0 of each even slot, and symbol 1 of it for four ports.
CellPlan pcfich_windows(const CellPlan& c) {
  CellPlan f = c;
  const int keep = c.nw == 3 ? 2 : 1;
  f.q.clear();
  f.late.clear();
  for (int t = 0; t < N_SLOT; t += 2)
    for (int w = 0; w < keep; w++) {
      f.q.push_back(c.q[(size_t)t * c.nw + w]);
      f.late.push_back(c.late[(size_t)t * c.nw + w]);
    }
  f.nw = keep;
  return f;
}

}  // namespace

extern "C" {

lcs_status lcs_pcfich_create(lcs_ctx* ctx, lcs_pcfich** out) { return grid_create(ctx, out, "lcs_pcfich_create"); }

void lcs_pcfich_destroy(lcs_pcfich* h) { grid_destroy(h); }

lcs_status lcs_pcfich_cells(lcs_pcfich* h, const void* iq, int iq_format, int on_device, uint64_t n_in, double fs_in,
                            double fc_in, const lcs_cell* cells, uint32_t n_cells, double fs_programmed,
                            lcs_pcfich_meas* out) {
  PcfichSlices s{};
  return grid_cells(
      h, "lcs_pcfich_cells", CHUNK, LCS_PCFICH_LAUNCHES_PER_CHUNK, iq, iq_format, on_device, n_in, fs_in, fc_in, cells,
      n_cells, fs_programmed, out,
      [](const lcs_cell& cell, uint64_t n_in, int D, double fs_in, double fc_in, double fs_prog, CellPlan& plan) {
        const std::string why = plan_cell(cell, n_in, D, fs_in, fc_in, fs_prog, plan);   // the full plan's checks
        if (why.empty()) plan = pcfich_windows(plan);
        return why;
      },
      pcfich_bytes,
      [&](const GridChunk& c) {
        s = pcfich_fill(h->g, c);
        return cudaSuccess;
      },
      [&](const GridChunk& c) { pcfich_launch(h->g, c, s, h->d_out.p); });
}

lcs_status lcs_pcfich_timing_read(lcs_pcfich* h, double* kernel_ms, uint64_t* launches) {
  return grid_timing_read(h, kernel_ms, launches, "lcs_pcfich_timing_read");
}

}  // extern "C"
