// sib1_rules.hpp - the tables and index maps of the SIB1 decoder (contract in include/lcs_sib1.h) as inline functions that
// compile under nvcc and g++: the device kernels of sib1.cu and the host planning of sib1_plan.cpp run the same code, and
// the host copy can be checked on its own under AddressSanitizer.
#pragma once
#include <cstdint>

#include "dci_fields.hpp"

namespace lcs {
namespace sib1 {

constexpr int MAX_K = 2240;                    // the largest code block: TBS 2216 + 24
constexpr int MAX_KW = 3 * 32 * ((MAX_K + 4 + 31) / 32);
constexpr int N_K = 188;                       // code block sizes of 36.212 Table 5.1.3-3
constexpr double KNOWN_ZERO = 1e6;             // the soft value of a filler bit, which is a known 0

// The tables, once for the host and once in device memory: LCS_TAB(x) is the copy the calling side can read.
#define LCS_SIB1_TABLE(type, name, dims, ...) \
  constexpr type name##_h dims = __VA_ARGS__;  \
  LCS_DEV_TABLE(type, name, dims, __VA_ARGS__)
#ifdef __CUDACC__
#define LCS_DEV_TABLE(type, name, dims, ...) __device__ const type name##_d dims = __VA_ARGS__;
#else
#define LCS_DEV_TABLE(type, name, dims, ...)
#endif
#ifdef __CUDA_ARCH__
#define LCS_TAB(name) name##_d
#else
#define LCS_TAB(name) name##_h
#endif
// 36.213 Table 7.1.7.2.1-1, columns N_PRB = 2 and 3, I_TBS 0 .. 26.
LCS_SIB1_TABLE(short, kTbs1a, [27][2], {{32, 56},     {56, 88},     {72, 144},    {104, 176},   {120, 208},   {144, 224},
                          {176, 256},   {224, 328},   {256, 392},   {296, 456},   {328, 504},   {376, 584},
                          {440, 680},   {488, 744},   {552, 840},   {600, 904},   {632, 968},   {696, 1064},
                          {776, 1160},  {840, 1288},  {904, 1384},  {1000, 1480}, {1064, 1608}, {1128, 1736},
                          {1192, 1800}, {1256, 1864}, {1480, 2216}})
// 36.213 Table 7.1.7.2.3-1.
LCS_SIB1_TABLE(short, kTbs1c, [32], {40,  56,  72,  120, 136, 144, 176, 208, 224, 256, 280,  296,  328,  336,  392,  488,
                       552, 600, 632, 696, 776, 840, 904, 1000, 1064, 1128, 1224, 1288, 1384, 1480, 1608, 1736})
// 36.212 Table 5.1.3-3: (f1, f2) of each code block size.
LCS_SIB1_TABLE(short, kQpp, [N_K][2], {
      {3, 10},    {7, 12},    {19, 42},   {7, 16},    {7, 18},    {11, 20},   {5, 22},    {11, 24},   {7, 26},
      {41, 84},   {103, 90},  {15, 32},   {9, 34},    {17, 108},  {9, 38},    {21, 120},  {101, 84},  {21, 44},
      {57, 46},   {23, 48},   {13, 50},   {27, 52},   {11, 36},   {27, 56},   {85, 58},   {29, 60},   {33, 62},
      {15, 32},   {17, 198},  {33, 68},   {103, 210}, {19, 36},   {19, 74},   {37, 76},   {19, 78},   {21, 120},
      {21, 82},   {115, 84},  {193, 86},  {21, 44},   {133, 90},  {81, 46},   {45, 94},   {23, 48},   {243, 98},
      {151, 40},  {155, 102}, {25, 52},   {51, 106},  {47, 72},   {91, 110},  {29, 168},  {29, 114},  {247, 58},
      {29, 118},  {89, 180},  {91, 122},  {157, 62},  {55, 84},   {31, 64},   {17, 66},   {35, 68},   {227, 420},
      {65, 96},   {19, 74},   {37, 76},   {41, 234},  {39, 80},   {185, 82},  {43, 252},  {21, 86},   {155, 44},
      {79, 120},  {139, 92},  {23, 94},   {217, 48},  {25, 98},   {17, 80},   {127, 102}, {25, 52},   {239, 106},
      {17, 48},   {137, 110}, {215, 112}, {29, 114},  {15, 58},   {147, 118}, {29, 60},   {59, 122},  {65, 124},
      {55, 84},   {31, 64},   {17, 66},   {171, 204}, {67, 140},  {35, 72},   {19, 74},   {39, 76},   {19, 78},
      {199, 240}, {21, 82},   {211, 252}, {21, 86},   {43, 88},   {149, 60},  {45, 92},   {49, 846},  {71, 48},
      {13, 28},   {17, 80},   {25, 102},  {183, 104}, {55, 954},  {127, 96},  {27, 110},  {29, 112},  {29, 114},
      {57, 116},  {45, 354},  {31, 120},  {59, 610},  {185, 124}, {113, 420}, {31, 64},   {17, 66},   {171, 136},
      {209, 420}, {253, 216}, {367, 444}, {265, 456}, {181, 468}, {39, 80},   {27, 164},  {127, 504}, {143, 172},
      {43, 88},   {29, 300},  {45, 92},   {157, 188}, {47, 96},   {13, 28},   {111, 240}, {443, 204}, {51, 104},
      {51, 212},  {451, 192}, {257, 220}, {57, 336},  {313, 228}, {271, 232}, {179, 236}, {331, 120}, {363, 244},
      {375, 248}, {127, 168}, {31, 64},   {33, 130},  {43, 264},  {33, 134},  {477, 408}, {35, 138},  {233, 280},
      {357, 142}, {337, 480}, {37, 146},  {71, 444},  {71, 120},  {37, 152},  {39, 462},  {127, 234}, {39, 158},
      {39, 80},   {31, 96},   {113, 902}, {41, 166},  {251, 336}, {43, 170},  {21, 86},   {43, 174},  {45, 176},
      {45, 178},  {161, 120}, {89, 182},  {323, 184}, {47, 186},  {23, 94},   {47, 190},  {263, 480}})
// 36.212 Table 5.1.4-1: the sub-block interleaver's inter-column permutation.
LCS_SIB1_TABLE(unsigned char, kColPerm, [32], {0, 16, 8, 24, 4, 20, 12, 28, 2, 18, 10, 26, 6, 22, 14, 30,
                               1, 17, 9, 25, 5, 21, 13, 29, 3, 19, 11, 27, 7, 23, 15, 31})

// I_TBS, N_PRB^1A -> TBS of format 1A.
LCS_HD inline int tbs_1a(int i_tbs, int n_prb_1a) {
  return i_tbs >= 0 && i_tbs < 27 && (n_prb_1a == 2 || n_prb_1a == 3) ? LCS_TAB(kTbs1a)[i_tbs][n_prb_1a - 2] : 0;
}

// The TBS of a format 1C tbs_index.
LCS_HD inline int tbs_1c(int i_tbs) {
  return i_tbs >= 0 && i_tbs < 32 ? LCS_TAB(kTbs1c)[i_tbs] : 0;
}

// Code block size number i < 188 of 36.212 Table 5.1.3-3: steps of 8 to 512, 16 to 1024, 32 to 2048, 64 to 6144.
LCS_HD inline int k_of(int i) {
  return i < 60 ? 40 + 8 * i : i < 92 ? 512 + 16 * (i - 59) : i < 124 ? 1024 + 32 * (i - 91) : 2048 + 64 * (i - 123);
}

// The smallest code block size >= B (one code block: B <= 6144), or 0.
LCS_HD inline int k_plus(int B) {
  for (int i = 0; i < N_K; i++)
    if (k_of(i) >= B) return k_of(i);
  return 0;
}

// The QPP interleaver parameters (f1, f2) of code block size number i (36.212 Table 5.1.3-3).
LCS_HD inline void qpp_params(int i, int& f1, int& f2) {
  f1 = LCS_TAB(kQpp)[i][0];
  f2 = LCS_TAB(kQpp)[i][1];
}

// The QPP interleaver of K: c'_i = c_pi(i), pi(i) = (f1 i + f2 i^2) mod K.
LCS_HD inline int qpp(int K, int f1, int f2, int i) {
  return (int)(((long long)f1 * i + (long long)f2 * i % K * i) % K);
}

LCS_HD inline int rbg_size(int R) { return R <= 10 ? 1 : R <= 26 ? 2 : R <= 63 ? 3 : 4; }   // 36.213 Table 7.1.6.1-1

// 36.211 Table 6.2.3.2-1: N_gap of gap 1 (2 for gap 2, R >= 50).
LCS_HD inline int n_gap(int R, int gap) {
  if (gap) return R <= 63 ? 9 : 16;
  return R <= 10 ? (R + 1) / 2 : R == 11 ? 4 : R <= 19 ? 8 : R <= 26 ? 12 : R <= 44 ? 18 : R <= 49 ? 27 : R <= 63 ? 27 : R <= 79 ? 32 : 48;
}

// N_VRB,DL of distributed VRBs with gap `gap`.
LCS_HD inline int n_vrb_gap(int R, int gap) {
  const int g = n_gap(R, gap);
  return gap ? (R / (2 * g)) * 2 * g : 2 * (g < R - g ? g : R - g);
}

// 36.211 6.2.3.2: the PRB of distributed VRB n in slot ns (0 even, 1 odd) with gap `gap`.
LCS_HD inline int vrb_to_prb(int R, int gap, int n, int ns) {
  const int g = n_gap(R, gap), P = rbg_size(R);
  const int nt = gap ? 2 * g : n_vrb_gap(R, 0);            // N~_VRB
  const int n_row = (nt + 4 * P - 1) / (4 * P) * P, n_null = 4 * n_row - nt;
  const int v = n % nt, blk = nt * (n / nt);
  const int p1 = 2 * n_row * (v % 2) + v / 2 + blk, p2 = n_row * (v % 4) + v / 4 + blk;
  int p;
  if (n_null && v >= nt - n_null && v % 2 == 1)
    p = p1 - n_row;
  else if (n_null && v >= nt - n_null && v % 2 == 0)
    p = p1 - n_row + n_null / 2;
  else if (n_null && v < nt - n_null && v % 4 >= 2)
    p = p2 - n_null / 2;
  else
    p = p2;
  if (ns) p = (p + nt / 2) % nt + blk;
  return p < nt / 2 ? p : p + g - nt / 2;
}

LCS_HD inline int col_perm(int c) {
  return LCS_TAB(kColPerm)[c];
}

// 36.212 5.1.4.1.1-2: the coded bit at position i < K_w = 96 ceil((K + 4) / 32) of the circular buffer w of a code block
// of size K with F filler bits: stream * (K + 4) + index into d[3][K + 4], or -1 for a NULL (a dummy or a filler bit).
LCS_HD inline int wbuf_pos(int K, int F, int i) {
  const int D = K + 4, rows = (D + 31) / 32, kp = 32 * rows, nd = kp - D;
  int s, y;
  if (i < kp) {
    s = 0;
    y = col_perm(i / rows) + 32 * (i % rows);
  } else {
    const int j = (i - kp) / 2;
    s = (i - kp) % 2 ? 2 : 1;
    y = col_perm(j / rows) + 32 * (j % rows);
    if (s == 2) y = (y + 1) % kp;
  }
  if (y < nd) return -1;
  const int k = y - nd;
  if (s < 2 && k < F) return -1;
  return s * D + k;
}

// The first position of redundancy version rv in the circular buffer (N_cb = K_w).
LCS_HD inline int k0_of(int K, int rv) {
  const int rows = (K + 4 + 31) / 32, kw = 96 * rows;
  return rows * (2 * ((kw + 8 * rows - 1) / (8 * rows)) * rv + 2);
}

// CRC24A (36.212 5.1.1, g = 0x864CFB) of bits[0 .. n): the remainder, 0 when bits ends with its own parity.
LCS_HD inline uint32_t crc24a(const uint8_t* bits, int n) {
  uint32_t r = 0;
  for (int i = 0; i < n; i++) {
    const uint32_t fb = ((r >> 23) & 1u) ^ (bits[i] & 1u);
    r = (r << 1) & 0xffffffu;
    if (fb) r ^= 0x864cfbu;
  }
  return r;
}

// The redundancy version of a SIB1 occasion in a frame with this SFN (36.321 5.3.1).
LCS_HD inline int sib1_rv(int sfn) {
  const int k = (sfn / 2) % 4;
  return ((3 * k + 1) / 2) % 4;
}

}  // namespace sib1
}  // namespace lcs
