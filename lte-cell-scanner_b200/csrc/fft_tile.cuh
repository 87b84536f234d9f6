// fft_tile.cuh - the FP32 shared-memory FFT of the Welch spectrum (psd.cu) and the full-carrier measurement (carrier.cu).
//
// Radix-2 decimation in time, in place: a transform is staged in bit-reversed order, and two radix-2 stages run fused in
// registers (a radix-4 step: four loads, two twiddles, four stores and one barrier per pair of stages).  A CTA of THREADS
// threads holds TILE = 4096 points (32 KB) and transforms TILE / N whole transforms of N points at once.  Twiddles are
// computed in double on the host by the caller and kept as float.
#pragma once
#include <cuda_runtime.h>

namespace lcs {
namespace fft {

constexpr int THREADS = 256;
constexpr int LG_TILE = 12;
constexpr int TILE = 1 << LG_TILE;       // points per CTA

__device__ __forceinline__ float2 cmul(float2 a, float2 b) {
  return make_float2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x);
}

// index i of a transform of length 2^lg in bit-reversed order
__device__ __forceinline__ int bitrev(int i, int lg) { return (int)(__brev((unsigned)i) >> (32 - lg)); }

// Where point t of a tile lives in shared memory: bits 5-11 select the same 32-point row, whose 5 low bits are XORed with
// a fold of the row number.  Bit-reversed staging, a column pass's strided columns and a row pass's transposed read then
// hit 32 different banks where the plain layout put every lane of a warp in one; the FFT's own strides are unaffected.
__device__ __forceinline__ int swz(int t) { return t ^ (((t >> 5) ^ (t >> 10)) & 31); }

// TILE / 2^lg transforms of length 2^lg in place, point i of transform b at a[swz(b * 2^lg + i)], each staged in
// bit-reversed order; tw is the table of length 2^lgN (W_n^j = tw[j * 2^lgN / n]).  Ends with a barrier.
__device__ void fft_tile(float2* a, int lg, const float2* __restrict__ tw, int lgN) {
  int s = 0;
  if (lg & 1) {                                      // one radix-2 stage of span 1 (twiddle 1)
    for (int p = threadIdx.x; p < TILE / 2; p += THREADS) {
      const float2 u = a[swz(2 * p)], v = a[swz(2 * p + 1)];
      a[swz(2 * p)] = make_float2(u.x + v.x, u.y + v.y);
      a[swz(2 * p + 1)] = make_float2(u.x - v.x, u.y - v.y);
    }
    s = 1;
    __syncthreads();
  }
  for (; s < lg; s += 2) {                           // stages of span h = 2^s and 2h, fused
    const int h = 1 << s;
    for (int q = threadIdx.x; q < TILE / 4; q += THREADS) {
      const int j = q & (h - 1);
      const int b = ((q >> s) << (s + 2)) + j;
      const int i0 = swz(b), i1 = swz(b + h), i2 = swz(b + 2 * h), i3 = swz(b + 3 * h);
      float2 a0 = a[i0], a1 = a[i1], a2 = a[i2], a3 = a[i3];
      const float2 w1 = __ldg(tw + (j << (lgN - s - 1)));   // W_2h^j
      const float2 w2 = __ldg(tw + (j << (lgN - s - 2)));   // W_4h^j; W_4h^(j+h) = -i W_4h^j
      float2 t = cmul(w1, a1);
      a1 = make_float2(a0.x - t.x, a0.y - t.y);
      a0 = make_float2(a0.x + t.x, a0.y + t.y);
      t = cmul(w1, a3);
      a3 = make_float2(a2.x - t.x, a2.y - t.y);
      a2 = make_float2(a2.x + t.x, a2.y + t.y);
      t = cmul(w2, a2);
      a[i0] = make_float2(a0.x + t.x, a0.y + t.y);
      a[i2] = make_float2(a0.x - t.x, a0.y - t.y);
      t = cmul(w2, a3);
      t = make_float2(t.y, -t.x);
      a[i1] = make_float2(a1.x + t.x, a1.y + t.y);
      a[i3] = make_float2(a1.x - t.x, a1.y - t.y);
    }
    __syncthreads();
  }
}

}  // namespace fft
}  // namespace lcs
