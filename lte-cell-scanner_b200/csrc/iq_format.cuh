// iq_format.cuh - the IQ sample formats of include/lcs_b200.h (LCS_IQ_*): the bytes of a sample, its value as a complex
// number on the device, and which compile-time instance of a kernel serves a runtime format.  No other file knows them.
#pragma once
#include <cuda_runtime.h>

#include <type_traits>

#include "../../include/lcs_b200.h"

namespace lcs {

// Bytes per complex sample of an LCS_IQ_* format; 0 for anything else.
constexpr size_t sample_bytes(int fmt) {
  return fmt == LCS_IQ_CI16 ? 4 : fmt == LCS_IQ_CS8 || fmt == LCS_IQ_CU8 ? 2 : fmt == LCS_IQ_CF32 ? 8 : fmt == LCS_IQ_C128 ? 16 : 0;
}

// The byte that both components of a zero sample are made of.
constexpr unsigned char zero_sample_byte(int fmt) { return fmt == LCS_IQ_CU8 ? 127 : 0; }

// A list of formats: those an entry point takes, and so those its kernels are instantiated for.
template <int... FMTS>
struct IqFormats {
  static constexpr bool has(int fmt) { return ((fmt == FMTS) || ...); }
  // f(std::integral_constant<int, FMT>()) for the FMT of the list that equals fmt; LCS_ERR_ARG, and no call, if none does
  template <class F>
  static lcs_status dispatch(int fmt, F&& f) {
    return ((fmt == FMTS && (f(std::integral_constant<int, FMTS>()), true)) || ...) ? LCS_OK : LCS_ERR_ARG;
  }
  // f for every format of the list
  template <class F>
  static void each(F&& f) { (f(std::integral_constant<int, FMTS>()), ...); }
};
// the correlator, the cell search and the cell measurement
using SearchFormats = IqFormats<LCS_IQ_CF32, LCS_IQ_CU8, LCS_IQ_C128>;
// the channelizer and the spectrum
using StreamFormats = IqFormats<LCS_IQ_CI16, LCS_IQ_CS8, LCS_IQ_CU8, LCS_IQ_CF32>;

// Every load below reads one whole sample (lcs_xcorr_pss_device's alignment rule relies on it).

// cu8 sample i as the integers I - 127 and Q - 127: one 16-bit load, whose mask and shift fold the - 127 into the byte
// extraction (a uchar2 load costs the channelizer's staging loop one more instruction per sample)
__device__ __forceinline__ int2 load_cu8(const void* __restrict__ base, size_t i) {
  const unsigned short w = __ldg(reinterpret_cast<const unsigned short*>(base) + i);
  return make_int2((int)(w & 0xff) - 127, (int)(w >> 8) - 127);
}

// Sample i as float: ci16 / 32768, cs8 / 128, (cu8 - 127) / 128 and cf32 exactly, c128 rounded once.
template <int FMT>
__device__ __forceinline__ float2 load_iq(const void* __restrict__ base, size_t i) {
  if constexpr (FMT == LCS_IQ_CI16) {
    const int w = __ldg(reinterpret_cast<const int*>(base) + i);
    return make_float2((float)(short)(w & 0xffff) * (1.f / 32768.f), (float)(short)(w >> 16) * (1.f / 32768.f));
  } else if constexpr (FMT == LCS_IQ_CS8) {
    const unsigned short w = __ldg(reinterpret_cast<const unsigned short*>(base) + i);
    return make_float2((float)(signed char)(w & 0xff) * (1.f / 128.f), (float)(signed char)(w >> 8) * (1.f / 128.f));
  } else if constexpr (FMT == LCS_IQ_CU8) {
    const int2 v = load_cu8(base, i);
    return make_float2((float)v.x * (1.f / 128.f), (float)v.y * (1.f / 128.f));
  } else if constexpr (FMT == LCS_IQ_CF32) {
    return __ldg(reinterpret_cast<const float2*>(base) + i);
  } else {
    static_assert(FMT == LCS_IQ_C128, "not an LCS_IQ_* format");
    const double2 v = __ldg(reinterpret_cast<const double2*>(base) + i);
    return make_float2((float)v.x, (float)v.y);
  }
}

// Sample i as double, exactly: (cu8 - 127) / 128, cf32 and c128 as stored.
template <int FMT>
__device__ __forceinline__ double2 load_c(const void* __restrict__ base, size_t i) {
  if constexpr (FMT == LCS_IQ_CU8) {
    const int2 v = load_cu8(base, i);
    return make_double2(v.x / 128.0, v.y / 128.0);
  } else if constexpr (FMT == LCS_IQ_CF32) {
    const float2 v = __ldg(reinterpret_cast<const float2*>(base) + i);
    return make_double2((double)v.x, (double)v.y);
  } else {
    static_assert(FMT == LCS_IQ_C128, "load_c takes cu8, cf32 or c128");
    return __ldg(reinterpret_cast<const double2*>(base) + i);
  }
}

}  // namespace lcs
