// pcfich.cu - the control format indicator of found cells in every subframe, decoded from their PCFICH over the whole
// carrier, from the wideband recording they were found in (DESIGN.md section 4.12; contract in include/lcs_pcfich.h).
// Built into liblcs_pcfich.so.
//
// A call is cut into chunks of LCS_PCFICH_CHUNK cells; each chunk makes two launches on the context's stream:
//   1. carrier_grid_kernel (carrier_grid.cuh) on the windows the decoder reads only: symbol 0 of every even slot, and
//      symbol 1 of it for four ports (a filtered copy of each cell's plan).
//   2. pcfich_kernel: one CTA per cell.  Thread (s, j) equalises pair j of subframe s (rules 2-4) into shared memory;
//      then one thread per subframe decides it (rule 5) and one thread counts the decisions (rule 6), every sum in FP64
//      in a fixed order, so a cell's record is bitwise the same whatever else the call decodes.
#include <new>

#include "../../include/lcs_pcfich.h"
#include "carrier_grid.cuh"

namespace lcs {
namespace pcfich {

using namespace lcs::carrier;
constexpr int N_SF = LCS_PCFICH_SUBFRAMES;
constexpr int PAIRS = 8;                         // 16 PCFICH symbols
constexpr int PC_THREADS = 512;                  // >= N_SF * PAIRS
constexpr uint32_t CHUNK = LCS_PCFICH_CHUNK;
static_assert(N_SF * PAIRS <= PC_THREADS, "one thread per (subframe, pair)");
static_assert(2 * N_SF == N_SLOT, "subframes of the grid");

struct PcfichCell {
  unsigned long long off;                        // the cell's grid [N_SF][nw][12 R]
  int R, n_ports, nw, n_id;                      // nw: windows per subframe (1, or 2 for four ports)
};

__device__ __forceinline__ double2 cmul_d(double2 a, double2 b) { return make_double2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }
__device__ __forceinline__ double2 conj_d(double2 a) { return make_double2(a.x, -a.y); }

// h[m] = Y[6 m + sh] conj(r[m]), r = (rs.x + j rs.y) / sqrt(2)
__device__ __forceinline__ double2 crs_h(const float2* row, const char2* r, int sh, int m) {
  const float2 y = row[6 * m + sh];
  const char2 s = r[m];
  return make_double2(((double)y.x * s.x + (double)y.y * s.y) * M_SQRT1_2, ((double)y.y * s.x - (double)y.x * s.y) * M_SQRT1_2);
}

// Rule 3: hhat of a port at column k from its CRS in grid row `row` (shift sh, signs r).
__device__ double2 chan(const float2* row, const char2* r, int sh, int R, int k) {
  const int d = k - sh, M = 2 * R;
  if (d <= 0) return crs_h(row, r, sh, 0);
  if (d >= 6 * (M - 1)) return crs_h(row, r, sh, M - 1);
  const int m = d / 6;
  const double f = (double)(d - 6 * m) / 6.0;
  const double2 a = crs_h(row, r, sh, m), b = crs_h(row, r, sh, m + 1);
  return make_double2((1 - f) * a.x + f * b.x, (1 - f) * a.y + f * b.y);
}

// Rule 2: the column of PCFICH RE n < 16.
__device__ __forceinline__ int re_col(int n, int R, int n_id) {
  const int i = n >> 2, v = n_id % 3;
  int o = n & 3;
  if (o >= v) o++;
  if (o >= v + 3) o++;
  return (6 * (n_id % (2 * R)) + 6 * ((i * R) / 2)) % (12 * R) + o;
}

// rs_all [cell][20][3][2 MAX_RB] holds the signs of the CRS r = (s.x + j s.y) / sqrt(2); shift_all [cell][20][3][4];
// scr [cell][10] the scrambling bits c_b of each subframe number, bit b of the word.
__global__ void __launch_bounds__(PC_THREADS) pcfich_kernel(const float2* __restrict__ grid, const char2* __restrict__ rs_all,
                                                            const unsigned char* __restrict__ shift_all,
                                                            const PcfichCell* __restrict__ par,
                                                            const uint32_t* __restrict__ scr, lcs_pcfich_meas* out) {
  __shared__ double2 xs[N_SF][2 * PAIRS];        // xhat
  __shared__ unsigned char dec[N_SF];
  const int tid = threadIdx.x, cell = blockIdx.x;
  const PcfichCell cc = par[cell];
  const int R = cc.R, W = 12 * R;
  lcs_pcfich_meas* o = out + cell;
  if (tid < N_SF * PAIRS) {                      // rules 2-4: pair j of subframe s
    const int s = tid / PAIRS, j = tid % PAIRS;
    const float2* G = grid + cc.off + (size_t)s * cc.nw * W;
    const int sl = (2 * s) % N_SLOT_TAB;
    const char2* rs = rs_all + (size_t)cell * N_SLOT_TAB * 3 * 2 * MAX_RB;
    const unsigned char* shift = shift_all + (size_t)cell * N_SLOT_TAB * 3 * 4;
    const int k0 = re_col(2 * j, R, cc.n_id), k1 = re_col(2 * j + 1, R, cc.n_id);
    const double2 y0 = make_double2(G[k0].x, G[k0].y), y1 = make_double2(G[k1].x, G[k1].y);
    const int pa = cc.n_ports == 4 ? (j & 1) : 0, pb = cc.n_ports == 4 ? 2 + (j & 1) : 1;
    auto est = [&](int p, int k) {               // ports 0 and 1 from symbol 0, ports 2 and 3 from symbol 1
      const int s3 = p < 2 ? 0 : 1, tab = sl * 3 + s3;
      return chan(G + (size_t)s3 * W, rs + tab * 2 * MAX_RB, shift[tab * 4 + p], R, k);
    };
    double2 x0, x1;
    if (cc.n_ports == 1) {
      const double2 h0 = est(0, k0), h1 = est(0, k1);
      const double g0 = h0.x * h0.x + h0.y * h0.y, g1 = h1.x * h1.x + h1.y * h1.y;
      const double2 a = cmul_d(y0, conj_d(h0)), b = cmul_d(y1, conj_d(h1));
      x0 = make_double2(a.x / g0, a.y / g0);
      x1 = make_double2(b.x / g1, b.y / g1);
    } else {
      const double2 a0 = est(pa, k0), a1 = est(pa, k1), b0 = est(pb, k0), b1 = est(pb, k1);
      const double2 ha = make_double2((a0.x + a1.x) / 2, (a0.y + a1.y) / 2), hb = make_double2((b0.x + b1.x) / 2, (b0.y + b1.y) / 2);
      const double g = (ha.x * ha.x + ha.y * ha.y) + (hb.x * hb.x + hb.y * hb.y);
      const double2 n0 = cmul_d(conj_d(ha), y0), m0 = cmul_d(hb, conj_d(y1));
      const double2 n1 = cmul_d(conj_d(ha), y1), m1 = cmul_d(hb, conj_d(y0));
      x0 = make_double2(M_SQRT2 * (n0.x + m0.x) / g, M_SQRT2 * (n0.y + m0.y) / g);
      x1 = make_double2(M_SQRT2 * (n1.x - m1.x) / g, M_SQRT2 * (n1.y - m1.y) / g);
    }
    xs[s][2 * j] = x0;
    xs[s][2 * j + 1] = x1;
  }
  __syncthreads();
  if (tid < N_SF) {                              // rule 5: subframe tid
    const int s = tid;
    const uint32_t c = scr[cell * 10 + s % 10];
    double met[3] = {0, 0, 0};
    for (int n = 0; n < 2 * PAIRS; n++) {
      const double2 x = xs[s][n];
#pragma unroll
      for (int h = 0; h < 2; h++) {
        const int b = 2 * n + h;
        const double d = (h ? x.y : x.x) * ((c >> b) & 1 ? -1.0 : 1.0);
#pragma unroll
        for (int k = 0; k < 3; k++) met[k] += b % 3 == k ? d : -d;       // cw_k+1[b] = 0 where b mod 3 = k
      }
    }
    int best = 0;
    double top = 0;
#pragma unroll
    for (int k = 0; k < 3; k++) {
      met[k] *= M_SQRT2 / 32;
      if (k == 0 || met[k] > top) {
        best = k;
        top = met[k];
      }
    }
    double e = 0;
    for (int n = 0; n < 2 * PAIRS; n++) {
      const double2 x = xs[s][n];
      const int b = 2 * n;
      const int e0 = (b % 3 != best) ^ ((c >> b) & 1), e1 = ((b + 1) % 3 != best) ^ ((c >> (b + 1)) & 1);
      const double re = x.x - (e0 ? -M_SQRT1_2 : M_SQRT1_2), im = x.y - (e1 ? -M_SQRT1_2 : M_SQRT1_2);
      e += re * re + im * im;
    }
#pragma unroll
    for (int k = 0; k < 3; k++) o->metric[s][k] = met[k];
    o->sinr[s] = 16.0 / e;
    o->cfi[s] = best + 1;
    dec[s] = (unsigned char)(best + 1);
  }
  __syncthreads();
  if (!tid) {                                    // rule 6
    uint32_t n1 = 0, n2 = 0, n3 = 0;
    for (int s = 0; s < N_SF; s++) {
      n1 += dec[s] == 1;
      n2 += dec[s] == 2;
      n3 += dec[s] == 3;
    }
    const int mode = n3 > n1 && n3 > n2 ? 3 : (n2 > n1 ? 2 : 1);
    o->count[0] = 0;
    o->count[1] = n1;
    o->count[2] = n2;
    o->count[3] = n3;
    o->cfi_mode = mode;
    o->n_ctrl_symbols = mode + (R <= 10);
    o->n_subframes = N_SF;
  }
}

}  // namespace pcfich
}  // namespace lcs

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
      for (int sf = 0; sf < 10; sf++) {          // 36.211 6.7.1
        const uint32_t c_init = (uint32_t)(sf + 1) * (2 * c.n_id_cell + 1) * 512 + c.n_id_cell;
        const std::vector<uint8_t> bits = lte_pn(c_init, 32);
        uint32_t w = 0;
        for (int b = 0; b < 32; b++) w |= (uint32_t)(bits[b] & 1) << b;
        scr[i * 10 + sf] = w;
      }
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
