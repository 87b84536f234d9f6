// dci_fields.hpp - the fields of a decoded common-search-space DCI (rule 13 of include/lcs_pdcch.h) and the RIV of
// 36.213 7.1.6.3, as inline functions that compile under g++ and nvcc: liblcs_pdcch.so parses its records on the host,
// liblcs_sib1.so parses the SI-RNTI DCI of an occasion on the device, from the same code.
#pragma once
#include <cstdint>

#include "../../include/lcs_pdcch.h"

#ifdef __CUDACC__
#define LCS_HD __host__ __device__
#else
#define LCS_HD
#endif

namespace lcs {
namespace pdcch {

LCS_HD inline int ceil_log2(long long x) {
  int b = 0;
  while ((1ll << b) < x) b++;
  return b;
}

LCS_HD inline uint32_t dci_field(uint64_t payload, int n_bits, int first, int width) {
  return (uint32_t)((payload >> (n_bits - first - width)) & ((1ull << width) - 1));
}

// 36.213 7.1.6.3: the RIV of (start, length) on R RBs, and back (false when riv is not one).
LCS_HD inline uint32_t riv_encode(int R, int start, int length) {
  return length - 1 <= R / 2 ? (uint32_t)(R * (length - 1) + start) : (uint32_t)(R * (R - length + 1) + (R - 1 - start));
}

LCS_HD inline bool riv_decode(int R, uint32_t riv, int& start, int& length) {
  const int a = (int)(riv / R), b = (int)(riv % R);
  if (a + b < R) {
    length = a + 1;
    start = b;
  } else {
    length = R - a + 1;
    start = R - 1 - b;
  }
  return a <= R && length >= 1 && start >= 0 && start + length <= R && riv_encode(R, start, length) == riv;
}

// Rule 13's fields of d from its format, n_bits and payload.
LCS_HD inline void parse_dci(lcs_pdcch_dci& d, int R) {
  const uint64_t p = d.payload;
  const int n = (int)d.n_bits;
  d.riv = d.localized = d.mcs = d.harq = d.ndi = d.rv = d.tpc = d.gap = d.tbs_index = 0;
  d.rb_start = d.n_rb = -1;
  if (d.format == LCS_DCI_1A) {                 // flag, localized/distributed, RIV, MCS, HARQ, NDI, RV, TPC (36.212 5.3.3.1.3)
    const int nra = ceil_log2((long long)R * (R + 1) / 2);
    d.localized = dci_field(p, n, 1, 1);
    d.riv = dci_field(p, n, 2, nra);
    d.mcs = dci_field(p, n, 2 + nra, 5);
    d.harq = dci_field(p, n, 7 + nra, 3);
    d.ndi = dci_field(p, n, 10 + nra, 1);
    d.rv = dci_field(p, n, 11 + nra, 2);
    d.tpc = dci_field(p, n, 13 + nra, 2);
    int start, length;
    if (riv_decode(R, d.riv, start, length)) {
      d.rb_start = start;
      d.n_rb = length;
    }
  } else if (d.format == LCS_DCI_1C) {          // gap (R >= 50), RIV, TBS index (36.212 5.3.3.1.4)
    const int g = R >= 50;
    d.gap = g ? dci_field(p, n, 0, 1) : 0;
    d.riv = dci_field(p, n, g, n - g - 5);
    d.tbs_index = dci_field(p, n, n - 5, 5);
  }
}

}  // namespace pdcch
}  // namespace lcs
