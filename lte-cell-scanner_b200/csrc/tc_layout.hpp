// tc_layout.hpp - operand layouts of the tensor-core correlator shared by the plan builder (planset.cu) and the kernel (xcorr_tc.cu).
//
// Templates (3 PSS roots x n_f hypotheses; column = hypothesis*3 + root) are processed in PASSES of at most NPAD = C*J
// columns.  Inside a pass the columns are split into J JOBS of C columns; a job is one wgmma N dimension that carries all
// THREE int8 digit planes of its C columns side by side: B row r of job g = digit plane r / C of column g*C + r % C
// (rows >= 3*C are zero padding up to NJOB, a multiple of 16).  One warpgroup MMA therefore produces a whole 24-bit
// result for C templates, and because C is a multiple of 8 the thread that holds accumulator column c of the wgmma
// fragment also holds columns C + c and 2C + c: the digits of a template recombine in registers.  Each job is owned by
// one consumer warpgroup of the kernel.
#pragma once
#include <stdint.h>

namespace lcs {
namespace tc {

constexpr int NT = 256;            // lags per tile
constexpr int NSUBL = 64;          // lags per MMA (wgmma M)
constexpr int NSUB = NT / NSUBL;   // MMA sub-tiles per tile
constexpr int KB = 288;            // K in bytes: 274 interleaved I/Q taps padded to a multiple of 32
constexpr int KSTEPS = KB / 32;    // wgmma K = 32 bytes
constexpr int KCHUNKS = KB / 16;   // 16-byte K chunks (core-matrix columns)
constexpr int NBLK = NT / 8 + KB / 16 - 1;   // 49 expanded blocks of 128 B per tile
constexpr int P_BYTES = NBLK * 128;          // one variant of one stage
constexpr int B_SBO = KCHUNKS * 128;         // bytes between 8-row groups of the B operand
constexpr int HALO = 32;           // largest fold-offset spread (samples) inside a pass
constexpr int WSTR = NT + HALO;    // fold positions per template row of the sliding fold window
constexpr int WROW = WSTR + 4;     // floats between window rows: rows 2 columns apart fall 8 banks apart
constexpr int M_MAX = 24;          // half frames whose per-template offsets fit the shared-memory table
constexpr int RAW_BYTES = 832;     // raw IQ bytes staged per tile: 2*NT + KB - 2 + 15 (alignment) rounded up to 16, + 16
constexpr int N_FOLD = 9600;
constexpr int MAX_PASS = 8;

// a2 (low digit plane) is converted to float by adding it to the bit pattern of 1.5 * 2^23: exact for |a2| < 2^22.
constexpr uint32_t MAGIC_BITS = 0x4B400000u;
constexpr double MAGIC_VAL = 12582912.0;

struct Layout {
  int cj, j;           // columns per job (a multiple of 8), jobs per pass
  __host__ __device__ constexpr int c() const { return cj; }
  __host__ __device__ constexpr int npad() const { return cj * j; }
  __host__ __device__ constexpr int njob() const { return (3 * cj + 15) / 16 * 16; }
  __host__ __device__ constexpr int b_job_bytes() const { return njob() / 8 * B_SBO; }
  __host__ __device__ constexpr int b_bytes() const { return j * b_job_bytes(); }
  __host__ __device__ constexpr int threads() const { return 128 + 128 * j; }
  __host__ __device__ constexpr int hyp_per_pass() const { return npad() / 3; }
};

// Per-pass geometry built on the host (integer arithmetic only; the templates themselves are built on the device).
struct PassGeo {
  int32_t smin[M_MAX];   // staging start of half frame m: <= every fold offset round_i(m*.005*k_factor*fs) of the pass
                         // (searcher.cpp:298), chosen so that offset - smin is non-decreasing in m (planset_build)
  int32_t f0, n_f;       // first hypothesis of the pass / number of hypotheses in it
  int32_t pad[2];
};

// byte offset of (row r, K byte k) inside a job's B image: K-major 8x16 B core matrices, LBO 128 B, SBO B_SBO
__host__ __device__ constexpr uint32_t b_offset(int r, int k) {
  return (uint32_t)(r / 8) * B_SBO + (uint32_t)(k / 16) * 128 + (uint32_t)(r % 8) * 16 + (uint32_t)(k % 16);
}

}  // namespace tc
}  // namespace lcs
