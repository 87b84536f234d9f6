// pcfich.cu - the control format indicator of found cells in every subframe, decoded from their PCFICH over the whole
// carrier, from the wideband recording they were found in (DESIGN.md section 4.12; contract in include/lcs_pcfich.h).
// Built into liblcs_pcfich.so.
//
// A call is cut into chunks of LCS_PCFICH_CHUNK cells; each chunk makes two launches on the context's stream:
//   1. carrier_grid_kernel (carrier_grid.cuh) on the windows the decoder reads only: symbol 0 of every even slot, and
//      symbol 1 of it for four ports (a filtered copy of each cell's plan).
//   2. pcfich_kernel (pcfich_kernel.cuh): one CTA per cell, every sum in FP64 in a fixed order, so a cell's record is
//      bitwise the same whatever else the call decodes.
#include <new>

#include "pcfich_kernel.cuh"

using namespace lcs;
using namespace lcs::carrier;
using namespace lcs::pcfich;

struct lcs_pcfich {
  lcs_ctx* ctx = nullptr;
  GridScratch g;                                 // the recording's span, the staged tables and one chunk's grids
  DevBuf<lcs_pcfich_meas> d_out;
  KernelClock clock;                             // both launches of each chunk
};

namespace {

lcs_status pfail(const lcs_pcfich* h, const std::string& msg) {
  return fail(h->ctx, LCS_ERR_ARG, "lcs_pcfich_cells: " + msg);
}

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

lcs_status lcs_pcfich_create(lcs_ctx* ctx, lcs_pcfich** out) {
  if (!ctx || !out) return fail(ctx, LCS_ERR_ARG, "lcs_pcfich_create: null argument");
  lcs_pcfich* h = new (std::nothrow) lcs_pcfich();
  if (!h) return fail(ctx, LCS_ERR_STATE, "lcs_pcfich_create: out of memory");
  h->ctx = ctx;
  *out = h;
  return LCS_OK;
}

void lcs_pcfich_destroy(lcs_pcfich* h) {
  if (!h) return;
  cudaSetDevice(h->ctx->device);                 // its buffers and events belong to the context's device
  delete h;
}

lcs_status lcs_pcfich_cells(lcs_pcfich* h, const void* iq, int iq_format, int on_device, uint64_t n_in, double fs_in,
                            double fc_in, const lcs_cell* cells, uint32_t n_cells, double fs_programmed,
                            lcs_pcfich_meas* out) {
  if (!h) return LCS_ERR_ARG;
  int D = 0;
  const std::string bad = check_call(iq, iq_format, on_device, n_in, fs_in, fc_in, n_cells, cells, out, fs_programmed, D);
  if (!bad.empty()) return pfail(h, bad);
  if (!n_cells) return LCS_OK;
  lcs_ctx* ctx = h->ctx;
  LCS_CUDA(ctx, cudaSetDevice(ctx->device));
  std::vector<CellPlan> ch;                      // every cell checked, and its windows laid out, before any device work
  long long lo, hi;
  const std::string why = plan_cells(cells, n_cells, n_in, D, fs_in, fc_in, fs_programmed, ch, lo, hi);
  if (!why.empty()) return pfail(h, why);
  lo = std::numeric_limits<long long>::max();    // the span of the windows the decoder reads
  hi = 0;
  for (CellPlan& c : ch) {
    c = pcfich_windows(c);
    lo = std::min(lo, c.q.front());
    hi = std::max(hi, c.q.back() + 128ll * D);
  }
  cudaStream_t st = ctx->streams[0];
  const unsigned char* d_in;
  long long base;
  LCS_CUDA(ctx, h->g.prepare(iq, sample_bytes(iq_format), on_device, lo, hi, 128 * D, st, &d_in, &base));
  LCS_CUDA(ctx, h->d_out.ensure(std::min(n_cells, CHUNK)));
  ChunkTables t;
  for (uint32_t c0 = 0; c0 < n_cells; c0 += CHUNK) {
    const uint32_t nc = std::min(CHUNK, n_cells - c0);
    LCS_CUDA(ctx, stage_chunk(h->g, &ch[c0], nc, nc * sizeof(PcfichCell) + 16 + nc * 10 * sizeof(uint32_t) + 16, t));
    PcfichCell* pc = h->g.up.take<PcfichCell>(nc);
    uint32_t* scr = h->g.up.take<uint32_t>(nc * 10);
    for (uint32_t i = 0; i < nc; i++) {
      const CellPlan& c = ch[c0 + i];
      pc[i] = PcfichCell{t.off[i], c.R, c.n_ports, c.nw, c.n_id_cell};
      pcfich_scrambling(c.n_id_cell, scr + i * 10);
    }
    LCS_CUDA(ctx, h->g.up.upload(st));
    LCS_CUDA(ctx, h->clock.begin(st));
    if (!launch_grid(h->g, t, iq_format, d_in, base, fs_in, D, st)) return pfail(h, "no grid kernel for this iq_format");
    pcfich_kernel<<<nc, PC_THREADS, 0, st>>>(h->g.d_grid.p, h->g.up.dev(t.rs), h->g.up.dev(t.shift), h->g.up.dev(pc),
                                             h->g.up.dev(scr), h->d_out.p);
    ctx->launches += LCS_PCFICH_LAUNCHES_PER_CHUNK;
    LCS_CUDA(ctx, cudaGetLastError());
    LCS_CUDA(ctx, h->clock.end(st, LCS_PCFICH_LAUNCHES_PER_CHUNK));
    LCS_CUDA(ctx, cudaMemcpyAsync(out + c0, h->d_out.p, nc * sizeof(lcs_pcfich_meas), cudaMemcpyDeviceToHost, st));
    LCS_CUDA(ctx, cudaStreamSynchronize(st));
  }
  return LCS_OK;
}

lcs_status lcs_pcfich_timing_read(lcs_pcfich* h, double* kernel_ms, uint64_t* launches) {
  if (!h) return LCS_ERR_ARG;
  if (!kernel_ms || !launches) return fail(h->ctx, LCS_ERR_ARG, "lcs_pcfich_timing_read: null pointer");
  LCS_CUDA(h->ctx, h->clock.read(kernel_ms, launches));
  return LCS_OK;
}

}  // extern "C"
