// xcorr_tc.cu - PSS correlator on the Hopper tensor cores (warpgroup wgmma), exact for 8-bit IQ.
//
// The sliding correlation is a Toeplitz GEMM: D[lag, template] = sum_j z[2*lag + j] * W[template, j],
// j = 0..273 over the interleaved I/Q byte stream z of the capture buffer (rtl-sdr wire format,
// reference src/capbuf.cpp:157-181).  Everything is done in EXACT integer arithmetic:
//
//   * IQ bytes v are used as signed x' = v-128 (a XOR with 0x80; the true sample is (x'+1)/128),
//   * each template component W (double, conj(fshift(pss_td))/137 of searcher.cpp:145-151) is scaled by
//     a power of two S and rounded to a 24-bit integer, split into three balanced base-256 digits
//     W*S = 65536 a0 + 256 a1 + a2, a_j in [-128,127] -> three int8 B operand planes (built on the device, planset.cu),
//   * wgmma.mma_async ... .s32.s8.s8 (s8 x s8 -> s32 accumulators in registers): |sum| <= 274*128*128 < 2^23, no overflow,
//   * real part uses the byte stream as is, the imaginary part a second stream with every (I,Q) pair
//     replaced by (Q, ~I)  (~I = -I'-1): sum a[2m]*Q' + a[2m+1]*(-I'-1) with the same template rows
//     a[2m] = Re W, a[2m+1] = -Im W.
//
// Operand roles: 64 LAGS of a sub-tile are the M dimension (wgmma m64), the templates the N dimension.  A JOB is one
// wgmma N dimension holding all three digit planes of C template columns (tc_layout.hpp); a pass has J jobs and the CTA
// one consumer warpgroup per job.  A warpgroup issues the MMAs of its job and runs the epilogue (digit recombination,
// |xc|^2, fold) on the accumulator registers.  It keeps two accumulator sets and issues the MMAs of the next part before
// the epilogue of the current one, so the tensor core works on its own MMAs as well as on the other warpgroup's while
// it is in an epilogue; setmaxnreg moves the registers the second set needs from the producer warpgroup to the consumers.
//
// The Toeplitz (Hankel) A operand is never materialised per lag: an "expanded" tile P[u][r][16 B] = z[16u+2r ..+15]
// is built once per 256-lag tile in shared memory (8x expansion of ~0.8 KB of raw bytes that a 1-D TMA bulk copy,
// cp.async.bulk + mbarrier complete_tx, stages one tile ahead); block u is exactly the 8-row x 16-byte K-major core
// matrix of (row group g, K chunk c) for every g+c = u, so one wgmma shared-memory descriptor with LBO = SBO = 128 B
// addresses the whole Hankel tile.  The template planes stay resident in shared memory in core-matrix order (loaded by
// TMA bulk copies whenever the CTA moves to another plan / pass).
//
// Work distribution.  The fold positions 0..9599 of a (capture buffer, pass) UNIT are produced by RUNS of consecutive
// 256-lag tiles.  Inside a run the incoherent sums live in a sliding shared-memory window of 256 + 32 positions per
// template: a tile adds |xc|^2 of all n_comb half frames at each template's own k_factor offset (searcher.cpp:298);
// afterwards the 256 oldest positions are final and written out, the 32 youngest carry over to the next tile.  Tiles of a
// run therefore do not overlap (T tiles yield 256 T - 32 positions), and a persistent CTA per SM takes t_cta consecutive
// tiles of the global tile sequence [unit][tile].
// Output: xc_incoherent_single, planar [batch][3][n_f_stride][9600] float.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <cmath>

#include "lcs_ctx.hpp"
#include "wgmma_s8.hpp"

namespace lcs {

struct TcParams {
  const uint8_t* iq;          // [batch][n_cap][2] raw bytes, 16-byte aligned
  unsigned long long iq_bytes;   // size of that allocation
  const uint32_t* buf_plan;   // [batch] plan of each buffer, or NULL (plan 0 for all)
  const uint8_t* b_img;       // [plan][pass][b_bytes] digit planes in core-matrix order
  const float* corr;          // [plan][pass][2][npad] (C_re row, C_im row), MAGIC_VAL already subtracted
  const tc::PassGeo* geo;     // [plan][pass]
  const int16_t* dsh;         // [plan][pass][M_MAX][npad] fold offset of the column minus the pass' staging start smin
  float* single_planar;       // [batch][3][n_f_stride][9600]
  uint32_t n_cap, n_f_stride, n_comb, batch, n_pass;
  uint32_t tu, t_cta;         // tiles per unit / tiles per CTA
  uint32_t n_tiles_total;     // n_units * tu
  float inv2s;                // 1 / (S*128)^2
  float rcp_ncomb;            // RN(1 / n_comb) when the 3-instruction division is exact for n_comb, else 0
};

// ---- small PTX wrappers ----
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
// try_wait parks the warp until the phase completes or the suspend-time hint (ns) expires
#ifndef LCS_TC_WAIT_HINT_NS
#define LCS_TC_WAIT_HINT_NS 2000
#endif
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_LOOP:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1, %2;\n"
      "@p bra DONE;\n"
      "bra WAIT_LOOP;\n"
      "DONE:\n"
      "}\n" ::"r"(bar), "r"(parity), "r"(LCS_TC_WAIT_HINT_NS)
      : "memory");
}
// 1-D TMA bulk copy global -> shared, completion counted in bytes on an mbarrier (UBLKCP in SASS)
__device__ __forceinline__ void bulk_g2s(uint32_t dst_smem, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst_smem), "l"(src),
               "r"(bytes), "r"(bar)
               : "memory");
}
// wgmma matrix descriptor, no swizzle (K-major core matrices of 8 rows x 16 bytes): start>>4 [0,14), LBO>>4 [16,30)
// = distance of core matrices along K, SBO>>4 [32,46) = distance of 8-row groups, base offset 0, layout type 0
__device__ __forceinline__ uint64_t make_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)(lbo_bytes >> 4) << 16) | ((uint64_t)(sbo_bytes >> 4) << 32);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
// wait until at most PENDING committed groups are in flight; d holds the accumulators of a group that has retired then
template <int PENDING, int N>
__device__ __forceinline__ void wgmma_wait(int (&d)[N]) {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(PENDING) : "memory");
#pragma unroll
  for (int i = 0; i < N; i++) asm volatile("" : "+r"(d[i])::"memory");   // the accumulators are read only after the wait
}
// hand registers from the producer warpgroup to the consumer warpgroups (executed by every warp of a warpgroup)
template <uint32_t R>
__device__ __forceinline__ void setmaxnreg_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
template <uint32_t R>
__device__ __forceinline__ void setmaxnreg_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void named_bar(uint32_t id, uint32_t nthreads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory"); }

// ---- work distribution: runs of consecutive tiles (see the header comment) ----
struct TcRun {
  uint32_t b, pp;        // capture buffer, plan-pass index (plan * n_pass + pass)
  int p0, p1;            // fold positions [p0, p1) this run produces
  uint32_t n_tiles;
};
struct TcRunIter {
  uint32_t t, t_end;     // global tile indices [t, t_end) of this CTA
  __device__ __forceinline__ void init(const TcParams& p) {
    t = blockIdx.x * p.t_cta;
    t_end = min(t + p.t_cta, p.n_tiles_total);
  }
  __device__ __forceinline__ bool next(const TcParams& p, TcRun& r) {
    while (t < t_end) {
      const uint32_t u = t / p.tu, base = u * p.tu, a = t - base;
      const uint32_t e = min(t_end, base + p.tu), bb = e - base;
      // runs of this unit that start before tile a: one per CTA boundary (multiple of t_cta) inside (base, base + a]
      const uint32_t nb = (base + a) / p.t_cta - base / p.t_cta;
      t = e;
      const int p0 = 256 * (int)a - tc::HALO * (int)nb;
      if (p0 >= tc::N_FOLD) continue;
      int p1 = 256 * (int)bb - tc::HALO * (int)(nb + 1);
      if (p1 > tc::N_FOLD) p1 = tc::N_FOLD;
      r.p0 = p0;
      r.p1 = p1;
      r.n_tiles = min(bb - a, (uint32_t)(p1 - p0 + tc::HALO + tc::NT - 1) / tc::NT);
      if (p.buf_plan) {          // per-buffer plans: unit = buffer * n_pass + pass
        r.b = u / p.n_pass;
        r.pp = __ldg(p.buf_plan + r.b) * p.n_pass + (u - r.b * p.n_pass);
      } else {                   // one plan: unit = pass * batch + buffer (pass-major, the templates stay resident)
        r.pp = u / p.batch;
        r.b = u - r.pp * p.batch;
      }
      return true;
    }
    return false;
  }
};
struct TcStep {            // (run, tile, half frame) cursor of the producer warp
  TcRunIter it;
  TcRun r;
  uint32_t k, m;
  bool ok;
  __device__ __forceinline__ void init(const TcParams& p) { it.init(p); ok = it.next(p, r); k = 0; m = 0; }
  __device__ __forceinline__ void advance(const TcParams& p) {
    if (++m == p.n_comb) {
      m = 0;
      if (++k == r.n_tiles) { k = 0; ok = it.next(p, r); }
    }
  }
};

// shared-memory map
template <int C, int J>
struct TcSmem {
  static constexpr tc::Layout L{C, J};
  static constexpr int P = 0;                                          // [2 stages][2 variants][P_BYTES]
  static constexpr int B = P + 4 * tc::P_BYTES;                        // [J][njob/8][KCHUNKS][8][16] int8
  static constexpr int WIN = B + L.b_bytes();                          // [npad][WROW] float
  static constexpr int CORR = WIN + L.npad() * tc::WROW * 4;           // [2][npad] float
  static constexpr int DOFF = CORR + 2 * L.npad() * 4;                 // [M_MAX][npad] int32 byte offsets (-4 * dsh)
  static constexpr int RAW = DOFF + tc::M_MAX * L.npad() * 4;          // [2][RAW_BYTES]
  static constexpr int BAR = RAW + 2 * tc::RAW_BYTES;                  // 8 mbarriers
  static constexpr int TOTAL = BAR + 8 * 8;
};

template <int C, int J>
__global__ void __launch_bounds__(128 + 128 * J, 1) xcorr_fold_tc_kernel(const __grid_constant__ TcParams p) {
  using SM = TcSmem<C, J>;
  constexpr tc::Layout LAY{C, J};
  constexpr int NPAD = LAY.npad(), NJOB = LAY.njob();
  constexpr int NACC = NJOB / 2;          // accumulator registers per thread (m64 x NJOB s32 over 128 threads)
  constexpr int CG = C / 8;               // 8-column groups of one digit plane
  constexpr int NV = C / 2;               // results per thread and part: 2 rows x 2 columns per 8-column group
  static_assert(C % 8 == 0, "digit planes must start on an 8-column group of the accumulator fragment");
  static_assert(SM::TOTAL <= 232448, "shared memory");
  // Registers per thread once the producer warpgroup has handed its surplus to the consumers (setmaxnreg).  The pool is
  // what the launch gave the CTA: 65536 / 384 = 168 per thread for J = 2, so 128 * 40 + 256 * 232 = 168 * 384.  J = 1
  // (256 threads) is launched at the consumers' 240 registers, so its increase is already covered by the launch.
  constexpr uint32_t PROD_REGS = 40, CONS_REGS = J == 2 ? 232 : 240;
  static_assert(128 * PROD_REGS + 128 * J * CONS_REGS <= 65536, "register file");
  extern __shared__ __align__(128) uint8_t smem[];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  uint8_t* sP = smem + SM::P;
  float* sWin = reinterpret_cast<float*>(smem + SM::WIN);
  float* sCorr = reinterpret_cast<float*>(smem + SM::CORR);
  int* sDoff = reinterpret_cast<int*>(smem + SM::DOFF);
  const uint32_t bar0 = smem_u32(smem + SM::BAR);
  // barriers (8 B each): 0,1 p_full[stage]; 2,3 p_empty[stage]; 4,5 raw_full[stage]; 6,7 b_full[job]
  const uint32_t BAR_PFULL = bar0, BAR_PEMPTY = bar0 + 16, BAR_RAW = bar0 + 32, BAR_BFULL = bar0 + 48;

  // ---- one-time setup ----
  for (int i = tid; i < NPAD * tc::WROW; i += LAY.threads()) sWin[i] = 0.f;
  if (tid == 0) {
    for (int i = 0; i < 2; i++) {
      mbar_init(BAR_PFULL + 8 * i, 1);
      mbar_init(BAR_PEMPTY + 8 * i, 4 * J);    // every consumer warp, after its warpgroup's MMAs on the stage retired
      mbar_init(BAR_RAW + 8 * i, 1);           // arrive.expect_tx of the producer + TMA bytes
      mbar_init(BAR_BFULL + 8 * i, 1);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();

  if (warp < 4) {
    setmaxnreg_dec<PROD_REGS>();
    if (warp != 0) return;     // warps 1..3 of the producer warpgroup have no work
    // ================= producer: raw bytes by TMA one step ahead, expansion into the Hankel tile =================
    const uint64_t iq_lo = reinterpret_cast<uint64_t>(p.iq), iq_hi = iq_lo + p.iq_bytes;
    const uint32_t raw_addr = smem_u32(smem + SM::RAW);
    auto issue_raw = [&](const TcStep& s, uint32_t rs) -> uint32_t {      // returns the byte offset of the tile inside the staged chunk
      const int smin = __ldg(&p.geo[s.r.pp].smin[s.m]);
      const uint64_t z = iq_lo + 2ull * ((uint64_t)s.r.b * p.n_cap + (uint64_t)(s.r.p0 + (int)(tc::NT * s.k) + smin));
      const uint64_t zal = z & ~15ull;
      // Bytes past the end of the allocation are never needed by a position that is written out (planset.cu checks the
      // fold offsets), so the copy is clamped to the allocation and the rest of the staging buffer keeps its previous
      // contents.  The bulk copy moves whole 16-byte chunks: when the allocation ends inside a chunk, its last (< 16) bytes
      // - the final samples of the last capture buffer, which an extreme k_factor can make necessary - are copied by lanes.
      uint32_t bytes = 0, rem = 0;
      if (zal < iq_hi) {
        const uint64_t avail = iq_hi - zal;
        const uint64_t left = avail & ~15ull;
        if (left < (uint64_t)(tc::RAW_BYTES - 16)) { bytes = (uint32_t)left; rem = (uint32_t)(avail - left); }
        else bytes = (uint32_t)(tc::RAW_BYTES - 16);
      }
      if ((uint32_t)lane < rem) smem[SM::RAW + rs * tc::RAW_BYTES + bytes + lane] = __ldg(reinterpret_cast<const uint8_t*>(zal) + bytes + lane);
      if (lane == 0) {
        if (bytes) {
          mbar_arrive_expect_tx(BAR_RAW + 8 * rs, bytes);
          bulk_g2s(raw_addr + rs * tc::RAW_BYTES, reinterpret_cast<const void*>(zal), bytes, BAR_RAW + 8 * rs);
        } else {
          mbar_arrive(BAR_RAW + 8 * rs);
        }
      }
      return (uint32_t)(z - zal);
    };
    TcStep cur, nxt;
    cur.init(p);
    nxt = cur;
    if (nxt.ok) nxt.advance(p);
    uint32_t zo_cur = 0, zo_nxt = 0;
    if (cur.ok) zo_cur = issue_raw(cur, 0);
    for (uint32_t i = 0; cur.ok; i++) {
      const uint32_t stage = i & 1, use = i >> 1;
      if (nxt.ok) zo_nxt = issue_raw(nxt, stage ^ 1);       // its previous contents were expanded in step i-1
      mbar_wait(BAR_RAW + 8 * stage, use & 1);
      mbar_wait(BAR_PEMPTY + 8 * stage, (use & 1) ^ 1);     // the MMAs that read this P stage retired
      const uint32_t* rw = reinterpret_cast<const uint32_t*>(smem + SM::RAW + stage * tc::RAW_BYTES);
      const int zo = (int)zo_cur;
      uint4* P1 = reinterpret_cast<uint4*>(sP + (stage * 2 + 0) * tc::P_BYTES);
      uint4* P2 = reinterpret_cast<uint4*>(sP + (stage * 2 + 1) * tc::P_BYTES);
#pragma unroll 2
      for (int row = lane; row < tc::NBLK * 8; row += 32) {     // row = u*8 + r  -> 16 bytes at z + 16u + 2r
        const int o = zo + 16 * (row >> 3) + 2 * (row & 7);
        const int ow = o >> 2;
        const bool sh = (o & 3) != 0;
        uint32_t w[5];
#pragma unroll
        for (int e = 0; e < 5; e++) w[e] = rw[ow + e];
        uint32_t x[4], y[4];
#pragma unroll
        for (int e = 0; e < 4; e++) {
          const uint32_t v = sh ? __byte_perm(w[e], w[e + 1], 0x5432) : w[e];
          x[e] = v ^ 0x80808080u;                               // (I', Q') = v - 128
          y[e] = __byte_perm(v, 0, 0x2301) ^ 0x7F807F80u;       // (Q', ~I')
        }
        P1[row] = make_uint4(x[0], x[1], x[2], x[3]);
        P2[row] = make_uint4(y[0], y[1], y[2], y[3]);
      }
      __syncwarp();
      fence_async_smem();      // generic-proxy stores -> visible to the tensor core's async proxy
      __syncwarp();
      if (lane == 0) mbar_arrive(BAR_PFULL + 8 * stage);
      cur = nxt;
      zo_cur = zo_nxt;
      if (nxt.ok) nxt.advance(p);
    }
  } else {
    // ================= consumers: one warpgroup per job - MMAs, then |xc|^2 and the fold on the accumulators =========
    setmaxnreg_inc<CONS_REGS>();
    const int job = (warp >> 2) - 1;
    const int wq = warp & 3;                        // warp of the warpgroup: accumulator rows 16*wq .. +15
    const int wt = tid - 128 * (job + 1);           // thread of the warpgroup
    const int cb = 2 * (lane & 3);                  // first of the two columns this thread holds in each 8-column group
    const uint32_t BAR_ID = 1 + job;                // named barrier of the warpgroup
    const uint32_t sP_addr = smem_u32(sP), sBj_addr = smem_u32(smem + SM::B + job * LAY.b_job_bytes());
    const uint32_t my_bfull = BAR_BFULL + 8 * job;
    // window row of column (job*C + cb) at the fold position of accumulator row (lane>>2) of this warp's 16 rows
    char* myWinB = reinterpret_cast<char*>(sWin + (job * C + cb) * tc::WROW + tc::HALO + 16 * wq + (lane >> 2));
    const float* cre = sCorr + job * C + cb;
    const float* cim = sCorr + NPAD + job * C + cb;
    uint32_t cur_pp = 0xffffffffu, bfull_par = 0, step = 0;
    // One part (re or im) of one 64-lag sub-tile: 9 MMAs over K, committed as one group; its epilogue later computes
    // value = (a0*256 + a1)*256 + a2 + constant for the 2 rows x C/4 columns of this thread.  acc register 4*g + 2*h + e
    // holds row (lane>>2) + 8h, column 8g + cb + e.
    auto mma_part = [&](int (&acc)[NACC], uint32_t a_addr) {
      const uint64_t a_desc = make_desc(a_addr, 128, 128), b_desc = make_desc(sBj_addr, 128, tc::B_SBO);
      wgmma_fence();
#pragma unroll
      for (int s = 0; s < tc::KSTEPS; s++) tc::wgmma_s8<NJOB>(acc, a_desc + (uint64_t)(s * 16), b_desc + (uint64_t)(s * 16), s > 0);
      wgmma_commit();
    };
    // Two accumulator sets: re parts accumulate in acc_re, im parts in acc_im.
    int acc_re[NACC], acc_im[NACC];
    auto recombine = [&](const int (&acc)[NACC], float (&x)[NV], const float* kc) {
#pragma unroll
      for (int g = 0; g < CG; g++) {
        const float2 k2 = *reinterpret_cast<const float2*>(kc + 8 * g);
        const float kk[2] = {k2.x, k2.y};
#pragma unroll
        for (int h = 0; h < 2; h++)
#pragma unroll
          for (int e = 0; e < 2; e++) {
            const int r = 4 * g + 2 * h + e;
            const int t = acc[r] * 256 + acc[r + 4 * CG];
            // float(a2) without an I2F: |a2| < 2^22, so the bit pattern MAGIC_BITS + a2 is the float 1.5*2^23 + a2 (exact);
            // the constant kk already has -1.5*2^23 folded in
            const float f2 = __int_as_float((int)tc::MAGIC_BITS + acc[r + 8 * CG]);
            x[(g * 2 + h) * 2 + e] = __fadd_rn(__fmaf_rn((float)t, 256.f, f2), kk[e]);
          }
      }
    };
    TcRunIter it;
    it.init(p);
    TcRun r;
    while (it.next(p, r)) {
      if (r.pp != cur_pp) {
        // another plan / pass: this job's templates by TMA (every MMA that read the old ones has been waited for), its
        // constants and fold offsets by the warpgroup
        named_bar(BAR_ID, 128);
        if (wt == 0) {
          constexpr uint32_t B_BYTES = (uint32_t)LAY.b_job_bytes(), CHUNK = 27648;     // 12 row groups of 2304 B per copy
          mbar_arrive_expect_tx(my_bfull, B_BYTES);
          const uint8_t* src = p.b_img + (size_t)r.pp * LAY.b_bytes() + (size_t)job * B_BYTES;
          for (uint32_t o = 0; o < B_BYTES; o += CHUNK) bulk_g2s(sBj_addr + o, src + o, min(CHUNK, B_BYTES - o), my_bfull);
        }
        const float* gc = p.corr + (size_t)r.pp * 2 * NPAD;
        const int16_t* gd = p.dsh + (size_t)r.pp * tc::M_MAX * NPAD;
        for (int i = wt; i < 2 * C; i += 128) {
          const int o = (i / C) * NPAD + job * C + i % C;
          sCorr[o] = __ldg(gc + o);
        }
        for (int i = wt; i < (int)p.n_comb * C; i += 128) {
          const int o = (i / C) * NPAD + job * C + i % C;
          sDoff[o] = -4 * (int)__ldg(gd + o);
        }
        named_bar(BAR_ID, 128);
        mbar_wait(my_bfull, bfull_par);
        bfull_par ^= 1;
        cur_pp = r.pp;
      }
      const int f0 = __ldg(&p.geo[r.pp].f0);
      const uint32_t n_templ = 3u * (uint32_t)__ldg(&p.geo[r.pp].n_f);
      for (uint32_t k = 0; k < r.n_tiles; k++) {
        for (uint32_t m = 0; m < p.n_comb; m++, step++) {
          const uint32_t stage = step & 1, use = step >> 1;
          mbar_wait(BAR_PFULL + 8 * stage, use & 1);
          const uint32_t a_stage = sP_addr + stage * 2 * tc::P_BYTES;
          // Software pipeline over the 2 * NSUB parts of the half frame, (re, im) per sub-tile: the MMAs of the next part
          // are issued before the epilogue of the current one, so the tensor core works on them meanwhile.  The sub-tile
          // loop is unrolled: in-flight accumulators then never cross a branch or loop edge, where the compiler would copy
          // them and thereby serialise the MMAs.  The last im epilogue of the half frame follows wait_group 0.
          mma_part(acc_re, a_stage);
#pragma unroll
          for (int q = 0; q < tc::NSUB; q++) {
            float x[NV], rr[NV];
            mma_part(acc_im, a_stage + tc::P_BYTES + q * (tc::NSUBL / 8) * 128);
            wgmma_wait<1>(acc_re);                  // re of sub-tile q retired, im in flight
            recombine(acc_re, x, cre);
#pragma unroll
            for (int v = 0; v < NV; v++) rr[v] = __fmul_rn(x[v], x[v]);
            if (q + 1 < tc::NSUB) {
              mma_part(acc_re, a_stage + (q + 1) * (tc::NSUBL / 8) * 128);
              wgmma_wait<1>(acc_im);
            } else {
              wgmma_wait<0>(acc_im);
              if (lane == 0) mbar_arrive(BAR_PEMPTY + 8 * stage);     // every MMA on the P stage retired
            }
            recombine(acc_im, x, cim);
            // |xc|^2 = re^2 + im^2 (searcher.cpp:300), in the integer scale of the templates; the power-of-two scale
            // factor is applied when the tile is written out
#pragma unroll
            for (int v = 0; v < NV; v++) rr[v] = __fmaf_rn(x[v], x[v], rr[v]);
            // fold into the sliding window: lag q*64 + row of the tile lands at window index lag + HALO - dsh; all loads
            // of the read-modify-write first, then add + store.  d = -4 * (fold offset of the column - staging start),
            // bytes, for the C/4 columns of this thread, read per sub-tile to keep it out of the registers the MMAs overlap.
            int d[CG][2];
#pragma unroll
            for (int g = 0; g < CG; g++) {
              const int2 d2 = *reinterpret_cast<const int2*>(sDoff + m * NPAD + job * C + cb + 8 * g);
              d[g][0] = d2.x;
              d[g][1] = d2.y;
            }
#pragma unroll
            for (int g = 0; g < CG; g++)
#pragma unroll
              for (int h = 0; h < 2; h++)
#pragma unroll
                for (int e = 0; e < 2; e++)
                  x[(g * 2 + h) * 2 + e] =
                      *reinterpret_cast<const float*>(myWinB + d[g][e] + ((8 * g + e) * tc::WROW + q * tc::NSUBL + 8 * h) * 4);
#pragma unroll
            for (int g = 0; g < CG; g++)
#pragma unroll
              for (int h = 0; h < 2; h++)
#pragma unroll
                for (int e = 0; e < 2; e++) {
                  const int v = (g * 2 + h) * 2 + e;
                  *reinterpret_cast<float*>(myWinB + d[g][e] + ((8 * g + e) * tc::WROW + q * tc::NSUBL + 8 * h) * 4) = __fadd_rn(x[v], rr[v]);
                }
          }
          // A lag of one warp at this half frame and a lag of another warp at the next one (different fold offset) can hit
          // the same window index: the warpgroup finishes one half frame's read-modify-writes before the next one starts.
          named_bar(BAR_ID, 128);
        }
        // ---- tile done: the 256 oldest window positions are final -> xc_incoherent_single rows (coalesced); the HALO
        // youngest carry over to the next tile of the run.  A warpgroup owns the window rows of its C columns exclusively,
        // so the jobs write out independently: while one is in its write-out the other keeps the tensor core busy. ----
        const float ncf = (float)p.n_comb, rcp = p.rcp_ncomb;
        const int pb = r.p0 + (int)(tc::NT * k) - tc::HALO;       // fold position of window index 0
        const bool last = k + 1 == r.n_tiles;
        const uint32_t row_end = min(n_templ, (uint32_t)((job + 1) * C));
        for (uint32_t row = job * C + wq; row < row_end; row += 4) {
          const uint32_t rf = row / 3, rt = row - 3 * rf;
          float* dst = p.single_planar + (((size_t)r.b * 3 + rt) * p.n_f_stride + f0 + rf) * tc::N_FOLD;
          float* src = sWin + row * tc::WROW;
#pragma unroll
          for (int j = lane; j < tc::NT; j += 32) {
            const int pos = pb + j;
            const float v = src[j];
            if (pos >= r.p0 && pos < r.p1) {                                                  // searcher.cpp:304: sum / n_comb
              const float x = __fmul_rn(v, p.inv2s);                                          // power-of-two scale: exact
              float qv;
              if (rcp != 0.f) {        // q = RN(x * r), one Newton step: correctly rounded for these divisors (tools/divchk.c)
                qv = __fmul_rn(x, rcp);
                qv = __fmaf_rn(__fmaf_rn(-ncf, qv, x), rcp, qv);
              } else {
                qv = __fdiv_rn(x, ncf);
              }
              dst[pos] = qv;
            }
          }
          const float carry = last ? 0.f : src[tc::NT + lane];
          __syncwarp();
          src[lane] = carry;
#pragma unroll
          for (int j = tc::HALO + lane; j < tc::WSTR; j += 32) src[j] = 0.f;
        }
        named_bar(BAR_ID, 128);
      }
    }
  }
}

// =============================================================================================
// Host side
// =============================================================================================
template <int C, int J>
static cudaError_t tc_set_smem() {
  return cudaFuncSetAttribute(xcorr_fold_tc_kernel<C, J>, cudaFuncAttributeMaxDynamicSharedMemorySize, TcSmem<C, J>::TOTAL);
}
lcs_status tc_init(lcs_ctx* ctx) {
  LCS_CUDA(ctx, (tc_set_smem<16, 1>()));
  LCS_CUDA(ctx, (tc_set_smem<24, 2>()));
  LCS_CUDA(ctx, (tc_set_smem<32, 2>()));
  LCS_CUDA(ctx, (tc_set_smem<48, 2>()));
  return LCS_OK;
}

int launch_xcorr_fold_tc(PlanSet& ps, const void* d_iq_cu8, uint32_t batch, const uint32_t* d_buf_plan, float* d_single_planar,
                         cudaStream_t st) {
  const XcorrGeom& g = ps.geom;
  TcParams q;
  q.iq = reinterpret_cast<const uint8_t*>(d_iq_cu8);
  q.iq_bytes = (unsigned long long)batch * g.n_cap * 2;
  q.buf_plan = d_buf_plan;
  q.b_img = ps.d_b.p;
  q.corr = ps.d_corr.p;
  q.geo = ps.d_geo.p;
  q.dsh = ps.d_dsh.p;
  q.single_planar = d_single_planar;
  q.n_cap = g.n_cap;
  q.n_f_stride = g.n_f_stride;
  q.n_comb = g.n_comb_xc;
  q.batch = batch;
  q.n_pass = ps.n_pass;
  q.inv2s = ps.inv_scale * ps.inv_scale;
  // x / n by  q = RN(x*r); q += RN(x - n*q) * r  (r = RN(1/n)) equals the IEEE quotient for EVERY non-negative float x for
  // these n (exhaustive check, tools/divchk.c); other divisors use the division instruction sequence
  static const bool kExactRcp[25] = {false, true, true, true, true, true, false, true, true, true, false, true, false,
                                     true, false, true, true, true, false, true, false, true, false, true, false};
  q.rcp_ncomb = (g.n_comb_xc <= 24 && kExactRcp[g.n_comb_xc]) ? 1.0f / (float)g.n_comb_xc : 0.f;
  // tiles per unit: T tiles of a run give 256 T - 32 positions, and a unit is cut into at most ceil(tu / t_cta) + 1 runs
  const uint32_t n_units = batch * ps.n_pass, n_sm = (uint32_t)ps.ctx->n_sm;
  uint32_t tu = (tc::N_FOLD + tc::HALO + tc::NT - 1) / tc::NT, t_cta = 1;
  for (;; tu++) {
    t_cta = (uint32_t)(((uint64_t)n_units * tu + n_sm - 1) / n_sm);
    const uint32_t runs = (tu + t_cta - 1) / t_cta + 1;
    if ((int)(tc::NT * tu) - (int)(tc::HALO * runs) >= tc::N_FOLD) break;
  }
  q.tu = tu;
  q.t_cta = t_cta;
  q.n_tiles_total = n_units * tu;
  const uint32_t grid = (q.n_tiles_total + t_cta - 1) / t_cta;
  const tc::Layout& L = ps.lay;
  if (L.cj == 16) xcorr_fold_tc_kernel<16, 1><<<grid, L.threads(), TcSmem<16, 1>::TOTAL, st>>>(q);
  else if (L.cj == 24) xcorr_fold_tc_kernel<24, 2><<<grid, L.threads(), TcSmem<24, 2>::TOTAL, st>>>(q);
  else if (L.cj == 32) xcorr_fold_tc_kernel<32, 2><<<grid, L.threads(), TcSmem<32, 2>::TOTAL, st>>>(q);
  else xcorr_fold_tc_kernel<48, 2><<<grid, L.threads(), TcSmem<48, 2>::TOTAL, st>>>(q);
  return 1;
}

}  // namespace lcs
