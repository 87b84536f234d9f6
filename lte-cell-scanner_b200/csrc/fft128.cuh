// fft128.cuh - FP64 device helpers shared by the companion kernels (chain_gpu.cu, track.cu): complex multiply and the
// shared-memory 128-point FFT.
#pragma once
#include <cuda_runtime.h>

namespace lcs {

__device__ __forceinline__ double2 cmul(double2 a, double2 b) { return make_double2(a.x * b.x - a.y * b.y, a.x * b.y + a.y * b.x); }

// 128-point forward FFT (e^{-j}), radix-2 DIT, 64 threads, data in shared memory in natural order
// on return.  `buf` must hold the input in BIT-REVERSED order on entry.
__device__ __forceinline__ void fft128_inplace(double2* buf, const double2* tw /*[64] e^{-j2pi k/128}*/, int tid) {
#pragma unroll
  for (int len = 2; len <= 128; len <<= 1) {
    const int half = len >> 1;
    const int k = tid & (half - 1);
    const int i = ((tid / half) * len) + k;
    const double2 w = tw[k * (128 / len)];
    const double2 u = buf[i], v = cmul(buf[i + half], w);
    buf[i] = make_double2(u.x + v.x, u.y + v.y);
    buf[i + half] = make_double2(u.x - v.x, u.y - v.y);
    __syncthreads();
  }
}
__device__ __forceinline__ int bitrev7(int i) { return (int)(__brev((unsigned)i) >> 25); }
__device__ __forceinline__ void make_twiddles(double2* tw, int tid) {
  double s, c;
  sincospi(-(double)tid / 64.0, &s, &c);  // e^{-j 2 pi tid/128}
  tw[tid] = make_double2(c, s);
}

}  // namespace lcs
