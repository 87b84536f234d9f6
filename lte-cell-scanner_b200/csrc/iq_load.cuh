// iq_load.cuh - exact conversion of one raw IQ sample to float, shared by the kernels that read SDR recordings in their
// own format (the channelizer, chan.cu, and the spectrum, psd.cu).
#pragma once
#include "../../include/lcs_b200.h"

namespace lcs {

// sample g of the input, converted exactly to float: ci16 / 32768, cs8 / 128, (cu8 - 127) / 128, cf32 as is
template <int FMT>
__device__ __forceinline__ float2 load_iq(const unsigned char* p, long long g) {
  if constexpr (FMT == LCS_IQ_CI16) {
    const int w = __ldg(reinterpret_cast<const int*>(p) + g);
    return make_float2((float)(short)(w & 0xffff) * (1.f / 32768.f), (float)(short)(w >> 16) * (1.f / 32768.f));
  } else if constexpr (FMT == LCS_IQ_CS8) {
    const unsigned short w = __ldg(reinterpret_cast<const unsigned short*>(p) + g);
    return make_float2((float)(signed char)(w & 0xff) * (1.f / 128.f), (float)(signed char)(w >> 8) * (1.f / 128.f));
  } else if constexpr (FMT == LCS_IQ_CU8) {
    const unsigned short w = __ldg(reinterpret_cast<const unsigned short*>(p) + g);
    return make_float2((float)((int)(w & 0xff) - 127) * (1.f / 128.f), (float)((int)(w >> 8) - 127) * (1.f / 128.f));
  } else {
    return __ldg(reinterpret_cast<const float2*>(p) + g);
  }
}

}  // namespace lcs
