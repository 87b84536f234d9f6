// chan.cu - wideband channelizer: one digital down-converter per LTE raster channel (mixer, Kaiser-windowed sinc
// low-pass, decimation by D to 1.92 Msps, 8-bit requantisation), every channel of a push in one launch.  The contract is
// in include/lcs_b200.h and DESIGN.md section 4.6.
//
// The mixer is folded into the taps: exp(-j2pi p[nD-k]/fs) = exp(-j2pi p[nD]/fs) * exp(+j2pi (k*delta mod fs)/fs), so each
// channel convolves the raw input with its own complex taps and rotates once per output.  A CTA stages one ci16 input
// tile in shared memory in polyphase order (phase j mod D, row j / D: the 32 lanes of a warp, 32 consecutive outputs,
// read 32 consecutive words for every tap) and runs 32 channels over it: each warp 4 channels x 128 outputs, each lane 4
// outputs x 4 channels in registers.  The epilogue applies the output rotation (FP64, exact integer phase), the gain, the
// round-to-nearest-even quantisation and the clip count.
//
// rchan_kernel (DESIGN.md section 4.7) generalises this to rational resampling by up / down from any allowed integer-Hz
// rate and to ci16, cs8, cu8 and cf32 input.  Decimation by D is up = 1, down = D, so one host path (create, push, auto
// gain, the chunked launch loop) drives both kernels; chan_kernel runs for ci16 at up = 1 and rchan_kernel for everything
// else, and only the tap table and the launch know which.
#include <climits>
#include <cmath>
#include <complex>
#include <cstring>
#include <new>
#include <numeric>
#include <type_traits>
#include <vector>

#include "iq_format.cuh"
#include "lcs_ctx.hpp"

namespace lcs {
namespace chn {

constexpr int THREADS = 256;
constexpr int WARPS = THREADS / 32;
constexpr int R = 4;                     // outputs per lane (spaced 32 apart)
constexpr int CW = 4;                    // channels per warp
constexpr int TILE = 32 * R;             // outputs per CTA
constexpr int CH_CTA = WARPS * CW;       // channels per CTA
constexpr double kFsCh = 1920000.0;      // output rate
constexpr double kCut = 960000.0;        // prototype cutoff
constexpr double kPass = 700000.0, kStop = 1220000.0;
constexpr double kPassDb = 0.01, kStopDb = 70.0;
constexpr int MAX_TAPS = 4097;
constexpr int RMAX_UP = 128, RMAX_DOWN = 640;
constexpr int RMAX_TAPS = 16385;
// Dynamic shared memory of a launch: the input tile, `down` rows of qlen samples, covering the 32 * RM * down + J inputs
// of a tile's outputs (at up = 1, RM = 4: D rows of TILE + 2M/D + 1).  The kernels' attribute is one value per function
// for the whole process, so a per-channelizer value would cap the launches of channelizers created earlier with a larger
// tile; every create sets the same fixed caps: for chan_kernel the largest tile it can be asked for (D = 64, L = MAX_TAPS),
// for rchan_kernel the opt-in maximum of an H100 CTA.
constexpr int tile_qlen(int down, int J, int RM) { return (32 * RM * down + J + down - 1) / down; }
constexpr size_t tile_smem(int down, int J, int RM) { return (size_t)down * tile_qlen(down, J, RM) * sizeof(float2); }
constexpr int SMEM_CAP = (int)tile_smem(64, MAX_TAPS, R);   // 98 816 bytes
constexpr int RSMEM_CAP = 227 * 1024;
static_assert(SMEM_CAP <= RSMEM_CAP, "input tile exceeds the shared memory of an SM");

// The parameters of a launch.  The two kernels share every field but the tile geometry (run() assigns the shared ones in
// one place); each keeps the layout it was compiled and measured with, which ptxas's register allocation depends on.
struct Params {                // chan_kernel (up = 1: down = D)
  const unsigned char* in;     // packed ci16 (I low, Q high); local sample 0 is the first input of local output 0 (n0*D-M)
  long long n_in;              // valid samples at `in` (later ones read as 0; no valid output uses them)
  int down, L, M, qlen;
  int n_out;                   // outputs of this launch
  long long n0;                // stream index of local output 0
  int n_ch;
  const float2* taps;          // [n_ch][L] complex taps h[t] * exp(+j2pi ((t-M)*delta mod fs)/fs)
  const double2* taps64;       // the same in double (power mode)
  const long long* step;       // [n_ch] (D*delta) mod fs
  long long fs;
  const float* gain;           // [n_ch]
  unsigned char* out;          // [n_ch] rows of out_stride bytes; column 2*i is local output i
  size_t out_stride;
  unsigned long long* clip;    // [n_ch]
  double* pw;                  // power mode: [n_ch][gridDim.x] sum |y|^2 per tile
};

struct RParams {               // rchan_kernel
  const unsigned char* in;     // samples in the input format; local sample 0 is stream sample i_hi(n0) - (J-1)
  long long n_in;              // valid samples at `in` (later ones read as 0; no valid output uses them)
  int up, down, J, RM, qlen;
  long long q0;                // n0*down + M
  int n_out;                   // outputs of this launch
  long long n0;                // stream index of local output 0
  int n_ch;
  const float2* taps;          // [n_ch][up][J] complex branch taps g_phi[j] * exp(+j2pi (j*delta mod fs)/fs)
  const double2* taps64;       // the same in double (power mode)
  const long long* step;       // [n_ch] delta mod fs
  long long fs;
  const float* gain;           // [n_ch]
  unsigned char* out;          // [n_ch] rows of out_stride bytes; column 2*i is local output i
  size_t out_stride;
  unsigned long long* clip;    // [n_ch]
  double* pw;                  // power mode: [n_ch][gridDim.x] sum |y|^2 per tile
};

// a += g * x (complex)
__device__ __forceinline__ void cmac(float2& a, float2 g, float2 x) {
  a.x = fmaf(g.x, x.x, a.x);
  a.x = fmaf(-g.y, x.y, a.x);
  a.y = fmaf(g.x, x.y, a.y);
  a.y = fmaf(g.y, x.x, a.y);
}
__device__ __forceinline__ void cmac(double2& a, double2 g, float2 x) {
  a.x = __fma_rn(g.x, (double)x.x, a.x);
  a.x = __fma_rn(-g.y, (double)x.y, a.x);
  a.y = __fma_rn(g.x, (double)x.y, a.y);
  a.y = __fma_rn(g.y, (double)x.x, a.y);
}

// One output: rotate the accumulator by the exact mixer phase p (cycles * fs) in FP64, scale by gn = 128 * gain, round to
// nearest even about 127 and store the two clamped bytes at o.  Returns how many of the two were clamped.
template <class V>
__device__ __forceinline__ int rotate_quantise(V acc, long long p, long long fs, double gn, unsigned char* o) {
  double sn, cs;
  sincospi(-2.0 * (double)p / (double)fs, &sn, &cs);
  const double yr = (double)acc.x * cs - (double)acc.y * sn;
  const double yi = (double)acc.x * sn + (double)acc.y * cs;
  double vr = rint(127.0 + gn * yr), vi = rint(127.0 + gn * yi);
  const int clipped = (vr < 0 || vr > 255) + (vi < 0 || vi > 255);
  vr = fmin(fmax(vr, 0.0), 255.0);
  vi = fmin(fmax(vi, 0.0), 255.0);
  o[0] = (unsigned char)vr;
  o[1] = (unsigned char)vi;
  return clipped;
}

// the warp's sum of s, in lane 0
__device__ __forceinline__ double warp_sum(double s) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
  return s;
}

template <bool POWER>
__global__ void __launch_bounds__(THREADS) chan_kernel(Params P) {
  extern __shared__ float2 xs[];                     // [D][qlen]
  const int tile = blockIdx.x;
  const int nl0 = tile * TILE;
  const long long j0 = (long long)nl0 * P.down;
  const int span = (TILE - 1) * P.down + 2 * P.M + 1;
  for (int j = threadIdx.x; j < span; j += THREADS) {
    const long long g = j0 + j;
    xs[(j % P.down) * P.qlen + j / P.down] = g < P.n_in ? load_iq<LCS_IQ_CI16>(P.in, g) : make_float2(0.f, 0.f);
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int c0 = blockIdx.y * CH_CTA + warp * CW;
  if (c0 >= P.n_ch) return;
  // the byte path runs in FP32; the power sums of auto gain in FP64 (taps and accumulators), so that the gain does not
  // inherit the FP32 rounding of the taps
  using V = typename std::conditional<POWER, double2, float2>::type;
  const V* tp[CW];
#pragma unroll
  for (int i = 0; i < CW; i++) {
    const size_t off = (size_t)min(c0 + i, P.n_ch - 1) * P.L;
    if constexpr (POWER) tp[i] = P.taps64 + off; else tp[i] = P.taps + off;
  }
  V acc[CW][R];
#pragma unroll
  for (int i = 0; i < CW; i++)
#pragma unroll
    for (int r = 0; r < R; r++) acc[i][r].x = acc[i][r].y = 0;
  // tap t reads local sample (nl0 + o)*D + 2M - t for output o of the tile: phase (2M - t) mod D, row o + (2M - t) / D
  int ph = 0, row = 0;
  for (int u = 0; u < P.L; u++) {
    const int t = 2 * P.M - u;
    const float2* xr = xs + ph * P.qlen + row + lane;
    float2 x[R];
#pragma unroll
    for (int r = 0; r < R; r++) x[r] = xr[32 * r];
#pragma unroll
    for (int i = 0; i < CW; i++) {
      const V g = __ldg(tp[i] + t);
#pragma unroll
      for (int r = 0; r < R; r++) cmac(acc[i][r], g, x[r]);
    }
    if (++ph == P.down) { ph = 0; row++; }
  }
#pragma unroll
  for (int i = 0; i < CW; i++) {
    const int c = c0 + i;
    if (c >= P.n_ch) break;
    if (POWER) {
      double s = 0;
#pragma unroll
      for (int r = 0; r < R; r++)
        if (nl0 + lane + 32 * r < P.n_out) s += (double)acc[i][r].x * acc[i][r].x + (double)acc[i][r].y * acc[i][r].y;
      s = warp_sum(s);
      if (lane == 0) P.pw[(size_t)c * gridDim.x + tile] = s;
    } else {
      const long long st = P.step[c];
      const double gn = 128.0 * (double)P.gain[c];
      unsigned clipped = 0;
#pragma unroll
      for (int r = 0; r < R; r++) {
        const int nl = nl0 + lane + 32 * r;
        if (nl >= P.n_out) continue;
        const long long n = P.n0 + nl;
        const long long p = ((n % P.fs) * st) % P.fs;            // exact phase of output n, in cycles * fs
        clipped += rotate_quantise(acc[i][r], p, P.fs, gn,
                                   P.out + (size_t)c * P.out_stride + 2 * (size_t)nl);
      }
      clipped = __reduce_add_sync(0xffffffffu, clipped);
      if (lane == 0 && clipped) atomicAdd(P.clip + c, (unsigned long long)clipped);
    }
  }
}

// ---- filter design (host, double precision) ---------------------------------------------------------------------------
static double bessel_i0(double x) {
  double s = 1, t = 1;
  for (int k = 1; k < 500; k++) {
    const double q = x / (2.0 * k);
    t *= q * q;
    s += t;
    if (t < 1e-17 * s) break;
  }
  return s;
}

double kaiser_beta() { return 0.1102 * (kStopDb - 8.7); }

// Kaiser-windowed sinc of odd length L, cutoff 0.96 MHz at the rate F, DC gain `gain`, rounded to float.
static void kaiser_sinc(int L, double F, double gain, std::vector<float>& out) {
  const int M = (L - 1) / 2;
  const double beta = kaiser_beta(), i0b = bessel_i0(beta), fcn = 2 * kCut / F;
  std::vector<double> h(L);
  double sum = 0;
  for (int n = 0; n < L; n++) {
    const int m = n - M;
    const double a = L > 1 ? 2.0 * n / (L - 1) - 1.0 : 0.0;
    const double w = bessel_i0(beta * std::sqrt(std::max(0.0, 1 - a * a))) / i0b;
    const double s = m == 0 ? fcn : std::sin(M_PI * fcn * m) / (M_PI * m);
    h[n] = s * w;
    sum += h[n];
  }
  out.resize(L);
  for (int n = 0; n < L; n++) out[n] = (float)(gain * h[n] / sum);
}

// Response of the (symmetric) float taps on the grid of lcs_chan_design_taps: every fs/(64L) from 0 to 0.70 MHz and from
// 1.22 MHz to fs/2, plus the band edges.
static bool meets_spec(const std::vector<float>& h, double fs) {
  const int L = (int)h.size(), M = (L - 1) / 2;
  const double step = fs / (64.0 * L);
  auto resp = [&](double f) {   // h[M] + 2 sum h[M+m] cos(m theta), cosines by the Chebyshev recurrence
    const double th = 2 * M_PI * f / fs, c1 = std::cos(th);
    double cm1 = 1, cm = c1, s = h[M];
    for (int m = 1; m <= M; m++) {
      s += 2.0 * (double)h[M + m] * cm;
      const double nx = 2 * c1 * cm - cm1;
      cm1 = cm;
      cm = nx;
    }
    return s;
  };
  auto pass_ok = [&](double f) { return std::fabs(20 * std::log10(std::fabs(resp(f)))) <= kPassDb; };
  auto stop_ok = [&](double f) { return 20 * std::log10(std::fabs(resp(f)) + 1e-300) <= -kStopDb; };
  for (double f = 0; f < kPass; f += step)
    if (!pass_ok(f)) return false;
  if (!pass_ok(kPass)) return false;
  for (double f = kStop; f < fs / 2; f += step)
    if (!stop_ok(f)) return false;
  return stop_ok(fs / 2);
}

// Shortest odd length from the Kaiser estimate that meets the spec (0 when none up to MAX_TAPS does).
static int design(double fs, std::vector<float>& h) {
  const double dw = 2 * M_PI * (kStop - kPass) / fs;
  int L = (int)std::ceil((kStopDb - 8.0) / (2.285 * dw)) + 1;
  L |= 1;
  kaiser_sinc(L, fs, 1.0, h);
  if (meets_spec(h, fs)) {
    std::vector<float> g;
    while (L >= 5) {
      kaiser_sinc(L - 2, fs, 1.0, g);
      if (!meets_spec(g, fs)) break;
      L -= 2;
      h.swap(g);
    }
    return L;
  }
  while (L < MAX_TAPS) {
    L += 2;
    kaiser_sinc(L, fs, 1.0, h);
    if (meets_spec(h, fs)) return L;
  }
  return 0;
}

static bool decimation(double fs_in, int* D) {
  if (!(fs_in > 0) || !std::isfinite(fs_in)) return false;
  const double d = std::round(fs_in / kFsCh);
  if (d < 2 || d > 64 || std::fabs(fs_in - d * kFsCh) > 1e-6) return false;
  *D = (int)d;
  return true;
}

// ---- rational resampling: any integer-Hz rate, ci16 / cs8 / cu8 / cf32 input (DESIGN.md section 4.7) -----------------
//
// Output n sums h[n*down - i*up + M] x~[i]: with q = n*down + M, its newest input is i_hi = q / up and its taps are branch
// phi = q mod up of the polyphase filter, g_phi[j] = h[phi + j*up] (zero past 2M), applied to x~[i_hi - j], j < J.  The
// mixer folds into the taps as in chan_kernel, referred to the newest input: x~[i_hi - j] = exp(-j2pi p[i_hi]/fs) *
// x[i_hi - j] exp(+j2pi (j*delta mod fs)/fs).  A CTA covers the outputs n0 + up*m + r of 32*RM consecutive m and every
// r < up; a lane's register slot fixes (m / 32, r), so all 32 lanes of a warp use one branch (warp-uniform tap loads) and
// read inputs `down` apart, which the tile staged in polyphase order modulo `down` turns into consecutive words.
template <int FMT, bool POWER>
__global__ void __launch_bounds__(THREADS) rchan_kernel(RParams P) {
  extern __shared__ float2 xs[];                     // [down][qlen]
  const int tile = blockIdx.x;
  const int mt = 32 * P.RM;                          // m values of the tile
  const long long j0 = (long long)tile * mt * P.down;
  const long long c0q = P.q0 / P.up;
  const int c_last = (int)((P.q0 + (long long)(P.up - 1) * P.down) / P.up - c0q);
  const int span = (mt - 1) * P.down + c_last + P.J;
  for (int j = threadIdx.x; j < span; j += THREADS) {
    const long long g = j0 + j;
    xs[(j % P.down) * P.qlen + j / P.down] = g < P.n_in ? load_iq<FMT>(P.in, g) : make_float2(0.f, 0.f);
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int c0 = blockIdx.y * CH_CTA + warp * CW;
  if (c0 >= P.n_ch) return;
  using V = typename std::conditional<POWER, double2, float2>::type;
  const V* tp[CW];
#pragma unroll
  for (int i = 0; i < CW; i++) {
    const size_t off = (size_t)min(c0 + i, P.n_ch - 1) * P.up * P.J;
    if constexpr (POWER) tp[i] = P.taps64 + off; else tp[i] = P.taps + off;
  }
  double pws[CW];
  unsigned clipped[CW];
#pragma unroll
  for (int i = 0; i < CW; i++) { pws[i] = 0; clipped[i] = 0; }
  const int nslot = P.RM * P.up;                     // slot s: m / 32 = s / up, r = s % up
  for (int s0 = 0; s0 < nslot; s0 += R) {
    int ph[R], row[R], toff[R], nl[R];
#pragma unroll
    for (int k = 0; k < R; k++) {
      const int s = min(s0 + k, nslot - 1);
      const int mm = s / P.up, r = s % P.up;
      const long long qr = P.q0 + (long long)r * P.down;
      // tap j = J-1 reads local sample (32 mm + lane) * down + (c_r - c_0): phase e mod down, row lane + e / down
      const int e = 32 * mm * P.down + (int)(qr / P.up - c0q);
      ph[k] = e % P.down;
      row[k] = e / P.down;
      toff[k] = (int)(qr % P.up) * P.J;
      nl[k] = s0 + k < nslot ? P.up * (tile * mt + 32 * mm + lane) + r : INT_MAX;
    }
    V acc[CW][R];
#pragma unroll
    for (int i = 0; i < CW; i++)
#pragma unroll
      for (int k = 0; k < R; k++) acc[i][k].x = acc[i][k].y = 0;
    for (int j = P.J - 1; j >= 0; j--) {             // oldest input first, as chan_kernel
      float2 x[R];
#pragma unroll
      for (int k = 0; k < R; k++) x[k] = xs[ph[k] * P.qlen + row[k] + lane];
#pragma unroll
      for (int i = 0; i < CW; i++)
#pragma unroll
        for (int k = 0; k < R; k++) cmac(acc[i][k], __ldg(tp[i] + toff[k] + j), x[k]);
#pragma unroll
      for (int k = 0; k < R; k++)
        if (++ph[k] == P.down) { ph[k] = 0; row[k]++; }
    }
#pragma unroll
    for (int i = 0; i < CW; i++) {
      const int c = c0 + i;
      if (c >= P.n_ch) break;
#pragma unroll
      for (int k = 0; k < R; k++) {
        if (nl[k] >= P.n_out) continue;
        if (POWER) {
          pws[i] += (double)acc[i][k].x * acc[i][k].x + (double)acc[i][k].y * acc[i][k].y;
          continue;
        }
        const long long ih = (P.q0 + (long long)nl[k] * P.down) / P.up;   // newest input of the output
        const long long p = ((ih % P.fs) * P.step[c]) % P.fs;              // its exact mixer phase, in cycles * fs
        clipped[i] += rotate_quantise(acc[i][k], p, P.fs, 128.0 * (double)P.gain[c],
                                      P.out + (size_t)c * P.out_stride + 2 * (size_t)nl[k]);
      }
    }
  }
#pragma unroll
  for (int i = 0; i < CW; i++) {
    const int c = c0 + i;
    if (c >= P.n_ch) break;
    if (POWER) {
      const double s = warp_sum(pws[i]);
      if (lane == 0) P.pw[(size_t)c * gridDim.x + tile] = s;
    } else {
      const unsigned n = __reduce_add_sync(0xffffffffu, clipped[i]);
      if (lane == 0 && n) atomicAdd(P.clip + c, (unsigned long long)n);
    }
  }
}

// In-place radix-2 FFT of a power-of-two length (forward, unnormalised); w[k] = exp(-j2pi k/(2 * a.size())).
static void fft(std::vector<std::complex<double>>& a, const std::vector<std::complex<double>>& w) {
  const size_t n = a.size();
  for (size_t i = 1, j = 0; i < n; i++) {
    size_t bit = n >> 1;
    for (; j & bit; bit >>= 1) j ^= bit;
    j ^= bit;
    if (i < j) std::swap(a[i], a[j]);
  }
  for (size_t len = 2; len <= n; len <<= 1) {
    const size_t half = len / 2, stride = 2 * n / len;
    for (size_t i = 0; i < n; i += len)
      for (size_t k = 0; k < half; k++) {
        const std::complex<double> t = w[k * stride] * a[i + k + half];
        a[i + k + half] = a[i + k] - t;
        a[i + k] = a[i + k] + t;
      }
  }
}

// |X[k]|, k = 0..N/2, of the N-point DFT of the real taps h zero-padded: one N/2-point complex FFT of the even and odd
// samples packed as real and imaginary parts.
static std::vector<double> dft_magnitude(const std::vector<float>& h, size_t N) {
  const size_t n2 = N / 2;
  std::vector<std::complex<double>> w(n2), z(n2);
  for (size_t k = 0; k < n2; k++) w[k] = std::polar(1.0, -2 * M_PI * (double)k / (double)N);
  for (size_t n = 0; n < h.size(); n++)
    if (n % 2) z[n / 2].imag((double)h[n]); else z[n / 2].real((double)h[n]);
  fft(z, w);
  std::vector<double> m(n2 + 1);
  for (size_t k = 0; k <= n2; k++) {
    const std::complex<double> a = z[k % n2], b = std::conj(z[(n2 - k) % n2]);
    const std::complex<double> e = 0.5 * (a + b), o = std::complex<double>(0, -0.5) * (a - b);
    m[k] = std::abs(e + (k < n2 ? w[k] : std::complex<double>(-1, 0)) * o);
  }
  return m;
}

// The spec of meets_spec for taps of DC gain `gain` at the rate F, on the grid of an FFT of the zero-padded taps (every
// F/N, N the power of two >= 64L) plus the band edges 0.70 and 1.22 MHz.
static bool meets_spec_fft(const std::vector<float>& h, double F, double gain) {
  const int L = (int)h.size(), M = (L - 1) / 2;
  size_t N = 1;
  while (N < 64 * (size_t)L) N <<= 1;
  const std::vector<double> a = dft_magnitude(h, N);
  auto pass_ok = [&](double m) { return std::fabs(20 * std::log10(m / gain)) <= kPassDb; };
  auto stop_ok = [&](double m) { return 20 * std::log10(m / gain + 1e-300) <= -kStopDb; };
  for (size_t k = 0; k <= N / 2; k++) {
    const double f = (double)k * F / (double)N, m = a[k];
    if (f <= kPass && !pass_ok(m)) return false;
    if (f >= kStop && !stop_ok(m)) return false;
  }
  auto resp = [&](double f) {   // h[M] + 2 sum h[M+m] cos(m theta), as meets_spec
    double s = h[M];
    for (int m = 1; m <= M; m++) s += 2.0 * (double)h[M + m] * std::cos(2 * M_PI * f * m / F);
    return std::fabs(s);
  };
  return pass_ok(resp(kPass)) && stop_ok(resp(kStop));
}

// The prototype for fs_in = 1.92 MHz * down / up at F = up * fs_in, DC gain up.  up = 1 is design() itself; otherwise the
// shortest odd length about the Kaiser estimate that meets the spec on the FFT grid and whose length - 2 fails it,
// found by doubling steps and bisection (the spec holds from some length on), so that L ~ 10 000 takes a few FFTs.
static int design_rational(long long fs_in, int up, std::vector<float>& h) {
  if (up == 1) return design((double)fs_in, h);
  const double F = (double)up * (double)fs_in, gain = up;
  auto ok = [&](int L, std::vector<float>& g) {
    kaiser_sinc(L, F, gain, g);
    return meets_spec_fft(g, F, gain);
  };
  const double dw = 2 * M_PI * (kStop - kPass) / F;
  int L = ((int)std::ceil((kStopDb - 8.0) / (2.285 * dw)) + 1) | 1;
  const int first_step = std::max(2, L / 64 / 2 * 2);   // the estimate is within a few per cent
  std::vector<float> g;
  int lo, hi;   // lo fails (or is 1), hi meets and h holds it
  if (ok(L, h)) {
    hi = L;
    for (int step = first_step;; step *= 2) {
      lo = hi - step;
      if (lo < 3) { lo = 1; break; }
      if (!ok(lo, g)) break;
      hi = lo;
      h.swap(g);
    }
  } else {
    lo = L;
    for (int step = first_step;; step *= 2) {
      hi = std::min(lo + step, RMAX_TAPS);
      if (ok(hi, h)) break;
      if (hi == RMAX_TAPS) return 0;
      lo = hi;
    }
  }
  while (hi - lo > 2) {
    const int mid = lo + 2 * std::max(1, (hi - lo) / 4);
    if (ok(mid, g)) { hi = mid; h.swap(g); } else lo = mid;
  }
  return hi;
}

// fs_in an integer number of Hz in (1.92 MHz, 122.88 MHz] with fs_in / 1.92 MHz = down / up in lowest terms,
// up <= 128, down <= 640
static bool rational_rate(double fs_in, long long* fs, int* up, int* down) {
  if (!std::isfinite(fs_in)) return false;
  const double r = std::round(fs_in);
  if (std::fabs(fs_in - r) > 1e-6 || !(r > kFsCh) || r > 64 * kFsCh) return false;
  const long long f = (long long)r, g = std::gcd(f, 1920000LL);
  if (1920000LL / g > RMAX_UP || f / g > RMAX_DOWN) return false;
  *fs = f;
  *up = (int)(1920000LL / g);
  *down = (int)(f / g);
  return true;
}

}  // namespace chn
}  // namespace lcs

using namespace lcs;
using namespace lcs::chn;

struct lcs_chan {
  lcs_ctx* ctx = nullptr;
  // fs / 1.92 MHz = down / up in lowest terms (decimation by D: up = 1, down = D); samples in format fmt;
  // L = 2M + 1 prototype taps, J = 2M / up + 1 of them per output; a tile is 32 * RM * up outputs
  int fmt = LCS_IQ_CI16, up = 1, down = 0, L = 0, M = 0, J = 0, RM = 1;
  long long fs = 0;
  uint32_t n_ch = 0;
  std::vector<float> h;
  std::vector<float> gain;
  std::vector<long long> delta, step;
  DevBuf<float2> d_taps;
  DevBuf<double2> d_taps64;
  DevBuf<long long> d_step;
  DevBuf<float> d_gain;
  DevBuf<unsigned char> d_in;
  DevBuf<unsigned char> d_out;
  DevBuf<unsigned long long> d_clip;
  DevBuf<double> d_pw;
  uint32_t chunk = TILE;                 // outputs per launch (bounds the device scratch)
  SampleCarry carry;                     // stream samples [i_hi(n_out) - (J-1), n_in) (zeros before the stream starts)
  uint64_t n_in = 0, n_out = 0;
  KernelClock clock;                     // one kernel per launch chunk
};

namespace {

lcs_status cfail(const lcs_chan* c, const char* msg) { return fail(c ? c->ctx : nullptr, LCS_ERR_ARG, msg); }

// chan_kernel (the faster one, with its own tap table) serves ci16 at D * 1.92 MHz, rchan_kernel everything else
bool decimating_kernel(const lcs_chan* c) { return c->up == 1 && c->fmt == LCS_IQ_CI16; }

// newest input of output n, and the first input the outputs from n on need
long long newest_input(const lcs_chan* c, uint64_t n) { return (long long)((n * c->down + c->M) / c->up); }
long long first_input(const lcs_chan* c, uint64_t n) { return newest_input(c, n) - (c->J - 1); }
// outputs after n input samples of a stream
uint64_t outputs_after(const lcs_chan* c, uint64_t n) {
  const uint64_t q = n * c->up;
  return q >= (uint64_t)c->M + 1 ? (q - 1 - c->M) / c->down + 1 : 0;
}
// the carry of a fresh stream: the inputs of output 0 before sample 0, of value 0 in the channelizer's format (cu8 127)
SampleCarry fresh_carry(const lcs_chan* c) {
  const size_t esz = sample_bytes(c->fmt);
  return SampleCarry{esz, std::vector<unsigned char>((size_t)-first_input(c, 0) * esz, zero_sample_byte(c->fmt))};
}
int outputs_per_tile(const lcs_chan* c) { return 32 * c->RM * c->up; }

// One launch of the channelizer's kernel: `shared` assigns the fields both kernels read, the rest is the kernel's own.
// LCS_ERR_ARG, and no launch, for a format the channelizer does not take.
template <class F>
lcs_status launch(const lcs_chan* c, bool power, dim3 grid, size_t smem, cudaStream_t st, F shared) {
  if (decimating_kernel(c)) {
    Params P;
    shared(P);
    P.L = c->L;
    P.M = c->M;
    if (power)
      chan_kernel<true><<<grid, THREADS, smem, st>>>(P);
    else
      chan_kernel<false><<<grid, THREADS, smem, st>>>(P);
    return LCS_OK;
  }
  RParams P;
  shared(P);
  P.up = c->up;
  P.J = c->J;
  P.RM = c->RM;
  P.q0 = P.n0 * c->down + c->M;
  return StreamFormats::dispatch(c->fmt, [&](auto FMT) {
    if (power)
      rchan_kernel<FMT, true><<<grid, THREADS, smem, st>>>(P);
    else
      rchan_kernel<FMT, false><<<grid, THREADS, smem, st>>>(P);
  });
}

// The per-channel complex taps (float and double) and epilogue phase step in the format of the channelizer's kernel.
void build_taps(lcs_chan* c, std::vector<float2>& taps, std::vector<double2>& taps64) {
  const long long fs = c->fs;
  const int up = c->up, J = c->J;
  const bool centre = decimating_kernel(c);
  taps.resize((size_t)c->n_ch * (centre ? c->L : up * J));
  taps64.resize(taps.size());
  c->step.resize(c->n_ch);
  for (uint32_t ch = 0; ch < c->n_ch; ch++) {
    const long long delta = c->delta[ch];
    if (centre) {   // referred to the centre tap, [n_ch][L]; the phase advances by D * delta per output
      c->step[ch] = (((long long)c->down * delta) % fs + fs) % fs;
      for (int t = 0; t < c->L; t++) {
        const long long p = (((long long)(t - c->M) * delta) % fs + fs) % fs;
        const double a = 2 * M_PI * (double)p / (double)fs;
        const double2 g = make_double2((double)c->h[t] * std::cos(a), (double)c->h[t] * std::sin(a));
        taps64[(size_t)ch * c->L + t] = g;
        taps[(size_t)ch * c->L + t] = make_float2((float)g.x, (float)g.y);
      }
      continue;
    }
    // referred to the newest input, one branch per output phase, [n_ch][up][J]; the phase advances by delta per input
    c->step[ch] = (delta % fs + fs) % fs;
    for (int j = 0; j < J; j++) {
      const long long p = (((long long)j * delta) % fs + fs) % fs;
      const double a = 2 * M_PI * (double)p / (double)fs, ca = std::cos(a), sa = std::sin(a);
      for (int phi = 0; phi < up; phi++) {
        const int k = phi + j * up;
        const double hk = k <= 2 * c->M ? (double)c->h[k] : 0.0;
        const size_t i = ((size_t)ch * up + phi) * J + j;
        taps64[i] = make_double2(hk * ca, hk * sa);
        taps[i] = make_float2((float)taps64[i].x, (float)taps64[i].y);
      }
    }
  }
}

// Outputs [0, n_out) of the virtual input a ++ b (nb samples) in the channelizer's format, whose sample 0 is the first input
// of output 0 (stream output n_abs0).  power: per-channel sums of |y|^2 are added to pw_sum; otherwise bytes go to out
// (row stride out_stride, on the device or the host) and clip counts to d_clip.
lcs_status run(lcs_chan* c, const SampleCarry& a, const unsigned char* b, size_t nb, uint64_t n_abs0, uint64_t n_out,
               bool power, unsigned char* out, size_t out_stride, bool out_dev, std::vector<double>* pw_sum) {
  lcs_ctx* ctx = c->ctx;
  cudaStream_t st = ctx->streams[0];
  const int T = outputs_per_tile(c);
  const size_t span_max = (size_t)c->chunk * c->down / c->up + c->J + 2;
  LCS_CUDA(ctx, c->d_in.ensure(span_max * a.esz));
  if (!power && !out_dev) LCS_CUDA(ctx, c->d_out.ensure((size_t)c->n_ch * c->chunk * 2));
  if (power) LCS_CUDA(ctx, c->d_pw.ensure((size_t)c->n_ch * ((c->chunk + T - 1) / T)));
  const size_t smem = tile_smem(c->down, c->J, c->RM);
  const long long base = first_input(c, n_abs0);
  std::vector<double> pw;
  for (uint64_t e0 = 0; e0 < n_out; e0 += c->chunk) {
    const uint32_t ne = (uint32_t)std::min<uint64_t>(c->chunk, n_out - e0);
    const uint64_t n0 = n_abs0 + e0;
    // samples [lo, hi) of a ++ b
    const size_t lo = (size_t)(first_input(c, n0) - base);
    const size_t hi = std::min((size_t)(newest_input(c, n0 + ne - 1) + 1 - base), a.size() + nb);
    LCS_CUDA(ctx, a.upload(b, lo, hi, c->d_in.p, st));
    auto shared = [&](auto& P) {
      P.in = c->d_in.p;
      P.n_in = (long long)(hi - lo);
      P.down = c->down;
      P.qlen = tile_qlen(c->down, c->J, c->RM);
      P.n_out = (int)ne;
      P.n0 = (long long)n0;
      P.n_ch = (int)c->n_ch;
      P.taps = c->d_taps.p;
      P.taps64 = c->d_taps64.p;
      P.step = c->d_step.p;
      P.fs = c->fs;
      P.gain = c->d_gain.p;
      P.out = out_dev ? out + 2 * e0 : c->d_out.p;
      P.out_stride = out_dev ? out_stride : (size_t)ne * 2;
      P.clip = c->d_clip.p;
      P.pw = c->d_pw.p;
    };
    const dim3 grid((ne + T - 1) / T, (c->n_ch + CH_CTA - 1) / CH_CTA);
    LCS_CUDA(ctx, c->clock.begin(st));
    if (launch(c, power, grid, smem, st, shared) != LCS_OK) return fail(ctx, LCS_ERR_ARG, "lcs_chan: bad iq_format");
    ctx->launches++;
    LCS_CUDA(ctx, cudaGetLastError());
    LCS_CUDA(ctx, c->clock.end(st, 1));
    if (power) {
      pw.resize((size_t)c->n_ch * grid.x);
      LCS_CUDA(ctx, cudaMemcpyAsync(pw.data(), c->d_pw.p, pw.size() * 8, cudaMemcpyDeviceToHost, st));
    } else if (!out_dev) {
      LCS_CUDA(ctx, cudaMemcpy2DAsync(out + 2 * e0, out_stride, c->d_out.p, (size_t)ne * 2, (size_t)ne * 2, c->n_ch,
                                      cudaMemcpyDeviceToHost, st));
    }
    LCS_CUDA(ctx, cudaStreamSynchronize(st));
    if (power)   // fixed order: tiles of a chunk, chunks in stream order
      for (uint32_t ch = 0; ch < c->n_ch; ch++)
        for (uint32_t t = 0; t < grid.x; t++) (*pw_sum)[ch] += pw[(size_t)ch * grid.x + t];
  }
  return LCS_OK;
}

// What lcs_chan_create and lcs_chan_create_rational share once the rate and format are known to be allowed: `who` is the
// caller's name in the error texts.
lcs_status create(lcs_ctx* ctx, const std::string& who, long long fs, int up, int down, int fmt, double fc_in,
                  uint32_t n_ch, const double* fc_ch, const float* gain, lcs_chan** out) {
  if (n_ch < 1 || n_ch > 1024) return fail(ctx, LCS_ERR_ARG, who + ": n_ch must be in [1, 1024]");
  if (!std::isfinite(fc_in)) return fail(ctx, LCS_ERR_ARG, who + ": fc_in is not finite");
  std::vector<long long> delta(n_ch);
  for (uint32_t c = 0; c < n_ch; c++) {
    const double d = fc_ch[c] - fc_in;
    if (!std::isfinite(d) || std::fabs(d - std::round(d)) > 1e-6)
      return fail(ctx, LCS_ERR_ARG, who + ": channel offset fc_ch - fc_in is not an integer number of Hz");
    delta[c] = (long long)std::llround(d);
    if (2 * std::llabs(delta[c]) > fs - 1920000)
      return fail(ctx, LCS_ERR_ARG, who + ": channel band (+-0.96 MHz) outside the input band");
    if (gain && !(std::isfinite(gain[c]) && gain[c] > 0)) return fail(ctx, LCS_ERR_ARG, who + ": gain must be finite and > 0");
  }
  lcs_chan* c = new (std::nothrow) lcs_chan();
  if (!c) return fail(ctx, LCS_ERR_STATE, who + ": out of memory");
  c->ctx = ctx;
  c->fmt = fmt;
  c->up = up;
  c->down = down;
  c->fs = fs;
  c->n_ch = n_ch;
  c->L = design_rational(fs, up, c->h);
  if (!c->L) {
    delete c;
    return fail(ctx, LCS_ERR_RANGE, who + ": no filter up to the tap limit meets the spec");
  }
  c->M = (c->L - 1) / 2;
  c->J = 2 * c->M / up + 1;
  c->RM = (R + up - 1) / up;                // the lane slots of a tile cover up * RM outputs per m
  c->delta = delta;
  c->gain.assign(n_ch, 1.0f);
  if (gain) c->gain.assign(gain, gain + n_ch);
  c->carry = fresh_carry(c);
  if (tile_smem(down, c->J, c->RM) > (size_t)RSMEM_CAP) {
    delete c;
    return fail(ctx, LCS_ERR_RANGE, who + ": the input tile exceeds shared memory");
  }
  // outputs per launch, whole tiles: device output scratch <= 32 MB, input <= 64 MB
  const uint64_t T = (uint64_t)outputs_per_tile(c);
  const uint64_t by_out = (32ull << 20) / (2ull * n_ch), by_in = (64ull << 20) / c->carry.esz * up / down;
  c->chunk = (uint32_t)std::max<uint64_t>(T, std::min(by_out, by_in) / T * T);
  std::vector<float2> taps;
  std::vector<double2> taps64;
  build_taps(c, taps, taps64);
  cudaError_t e = cudaSetDevice(ctx->device);
  if (e == cudaSuccess) e = c->d_taps.alloc(taps.size());
  if (e == cudaSuccess) e = c->d_taps64.alloc(taps64.size());
  if (e == cudaSuccess) e = c->d_step.alloc(n_ch);
  if (e == cudaSuccess) e = c->d_gain.alloc(n_ch);
  if (e == cudaSuccess) e = c->d_clip.alloc(n_ch);
  if (e == cudaSuccess) e = cudaMemcpy(c->d_taps.p, taps.data(), taps.size() * sizeof(float2), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(c->d_taps64.p, taps64.data(), taps64.size() * sizeof(double2), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(c->d_step.p, c->step.data(), n_ch * 8, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(c->d_gain.p, c->gain.data(), n_ch * 4, cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(chan_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_CAP);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(chan_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_CAP);
  if (e == cudaSuccess)
    StreamFormats::dispatch(fmt, [&](auto FMT) {
      e = cudaFuncSetAttribute(rchan_kernel<FMT, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, RSMEM_CAP);
      if (e == cudaSuccess) e = cudaFuncSetAttribute(rchan_kernel<FMT, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, RSMEM_CAP);
    });
  if (e != cudaSuccess) {
    delete c;
    return fail(ctx, LCS_ERR_CUDA, who + ": " + cudaGetErrorString(e));
  }
  *out = c;
  return LCS_OK;
}

}  // namespace

extern "C" {

lcs_status lcs_chan_design_taps(double fs_in, float* taps, uint32_t* n_taps) {
  int D = 0;
  if (!n_taps || !decimation(fs_in, &D)) return fail(nullptr, LCS_ERR_ARG, "lcs_chan_design_taps: fs_in must be D * 1.92 MHz, D in [2, 64]");
  std::vector<float> h;
  const int L = design(D * kFsCh, h);
  if (!L) return fail(nullptr, LCS_ERR_RANGE, "lcs_chan_design_taps: no filter up to the tap limit meets the spec");
  if (taps) {
    if (*n_taps < (uint32_t)L) return fail(nullptr, LCS_ERR_ARG, "lcs_chan_design_taps: taps array too short");
    std::memcpy(taps, h.data(), L * sizeof(float));
  }
  *n_taps = (uint32_t)L;
  return LCS_OK;
}

lcs_status lcs_chan_design_rational(double fs_in, uint32_t* up, uint32_t* down, float* taps, uint32_t* n_taps) {
  long long fs = 0;
  int u = 0, d = 0;
  if (!up || !down || !n_taps || !rational_rate(fs_in, &fs, &u, &d))
    return fail(nullptr, LCS_ERR_ARG, "lcs_chan_design_rational: fs_in must be an integer number of Hz in (1.92, 122.88] MHz "
                                      "with fs_in / 1.92 MHz = down / up, up <= 128, down <= 640");
  std::vector<float> h;
  const int L = design_rational(fs, u, h);
  if (!L) return fail(nullptr, LCS_ERR_RANGE, "lcs_chan_design_rational: no filter up to the tap limit meets the spec");
  if (taps) {
    if (*n_taps < (uint32_t)L) return fail(nullptr, LCS_ERR_ARG, "lcs_chan_design_rational: taps array too short");
    std::memcpy(taps, h.data(), L * sizeof(float));
  }
  *up = (uint32_t)u;
  *down = (uint32_t)d;
  *n_taps = (uint32_t)L;
  return LCS_OK;
}

lcs_status lcs_chan_create(lcs_ctx* ctx, double fs_in, double fc_in, uint32_t n_ch, const double* fc_ch, const float* gain,
                           lcs_chan** out) {
  if (!ctx || !out || !fc_ch) return fail(ctx, LCS_ERR_ARG, "lcs_chan_create: null argument");
  int D = 0;
  if (!decimation(fs_in, &D)) return fail(ctx, LCS_ERR_ARG, "lcs_chan_create: fs_in must be D * 1.92 MHz, D in [2, 64]");
  return create(ctx, "lcs_chan_create", (long long)D * 1920000LL, 1, D, LCS_IQ_CI16, fc_in, n_ch, fc_ch, gain, out);
}

lcs_status lcs_chan_create_rational(lcs_ctx* ctx, double fs_in, int iq_format, double fc_in, uint32_t n_ch,
                                    const double* fc_ch, const float* gain, lcs_chan** out) {
  if (!ctx || !out || !fc_ch) return fail(ctx, LCS_ERR_ARG, "lcs_chan_create_rational: null argument");
  long long fs = 0;
  int up = 0, down = 0;
  if (!rational_rate(fs_in, &fs, &up, &down))
    return fail(ctx, LCS_ERR_ARG, "lcs_chan_create_rational: fs_in must be an integer number of Hz in (1.92, 122.88] MHz "
                                  "with fs_in / 1.92 MHz = down / up, up <= 128, down <= 640");
  if (!StreamFormats::has(iq_format))
    return fail(ctx, LCS_ERR_ARG, "lcs_chan_create_rational: iq_format must be LCS_IQ_CI16, CS8, CU8 or CF32");
  return create(ctx, "lcs_chan_create_rational", fs, up, down, iq_format, fc_in, n_ch, fc_ch, gain, out);
}

void lcs_chan_destroy(lcs_chan* c) {
  if (!c) return;
  cudaSetDevice(c->ctx->device);             // its buffers and events belong to the context's device
  delete c;
}

lcs_status lcs_chan_auto_gain(lcs_chan* c, const void* iq_host, uint32_t n) {
  if (!c) return LCS_ERR_ARG;
  if (!iq_host) return cfail(c, "lcs_chan_auto_gain: null samples");
  const uint64_t n_out = outputs_after(c, n);             // what a fresh channelizer would produce
  if (n_out == 0) return cfail(c, "lcs_chan_auto_gain: fewer samples than one output needs");
  LCS_CUDA(c->ctx, cudaSetDevice(c->ctx->device));
  std::vector<double> sum(c->n_ch, 0.0);
  lcs_status rc = run(c, fresh_carry(c), static_cast<const unsigned char*>(iq_host), n, 0, n_out, true, nullptr, 0, false, &sum);
  if (rc != LCS_OK) return rc;
  for (uint32_t ch = 0; ch < c->n_ch; ch++) {
    const double ms = sum[ch] / (double)n_out;
    c->gain[ch] = ms > 0 ? (float)(0.25 / std::sqrt(ms)) : 1.0f;
  }
  LCS_CUDA(c->ctx, cudaMemcpy(c->d_gain.p, c->gain.data(), c->n_ch * 4, cudaMemcpyHostToDevice));
  return LCS_OK;
}

lcs_status lcs_chan_auto_gain_ci16(lcs_chan* c, const int16_t* iq_host, uint32_t n) {
  if (!c) return LCS_ERR_ARG;
  if (c->fmt != LCS_IQ_CI16) return cfail(c, "lcs_chan_auto_gain_ci16: the channelizer's input format is not ci16");
  return lcs_chan_auto_gain(c, iq_host, n);
}

lcs_status lcs_chan_gain(const lcs_chan* c, float* gain) {
  if (!c) return LCS_ERR_ARG;
  if (!gain) return cfail(c, "lcs_chan_gain: null pointer");
  std::memcpy(gain, c->gain.data(), c->n_ch * sizeof(float));
  return LCS_OK;
}

lcs_status lcs_chan_n_out(const lcs_chan* c, uint64_t n_in, uint32_t* n_out) {
  if (!c) return LCS_ERR_ARG;
  if (!n_out) return cfail(c, "lcs_chan_n_out: null pointer");
  const uint64_t k = outputs_after(c, c->n_in + n_in) - c->n_out;
  if (k > UINT32_MAX) return cfail(c, "lcs_chan_n_out: push too long");
  *n_out = (uint32_t)k;
  return LCS_OK;
}

lcs_status lcs_chan_push(lcs_chan* c, const void* iq_host, uint32_t n_in, uint8_t* out, uint32_t out_capacity,
                         int out_on_device, uint32_t* n_out, uint64_t* n_clipped) {
  if (!c) return LCS_ERR_ARG;
  if ((!iq_host && n_in) || !n_out) return cfail(c, "lcs_chan_push: null pointer");
  const uint64_t k = outputs_after(c, c->n_in + n_in) - c->n_out;
  if (k > out_capacity) return cfail(c, "lcs_chan_push: out_capacity is smaller than the outputs of this push");
  if (k && !out) return cfail(c, "lcs_chan_push: null output");
  LCS_CUDA(c->ctx, cudaSetDevice(c->ctx->device));
  LCS_CUDA(c->ctx, cudaMemsetAsync(c->d_clip.p, 0, c->n_ch * 8, c->ctx->streams[0]));
  const unsigned char* b = static_cast<const unsigned char*>(iq_host);
  if (k) {
    lcs_status rc = run(c, c->carry, b, n_in, c->n_out, k, false, out, (size_t)out_capacity * 2, out_on_device != 0, nullptr);
    if (rc != LCS_OK) return rc;
  }
  // keep the samples from the first input of the next output on
  c->carry.advance(b, n_in, (size_t)(first_input(c, c->n_out + k) - first_input(c, c->n_out)));
  c->n_in += n_in;
  c->n_out += k;
  *n_out = (uint32_t)k;
  if (n_clipped) {
    if (k)
      LCS_CUDA(c->ctx, cudaMemcpy(n_clipped, c->d_clip.p, c->n_ch * 8, cudaMemcpyDeviceToHost));
    else
      std::memset(n_clipped, 0, c->n_ch * 8);
  }
  return LCS_OK;
}

lcs_status lcs_chan_push_ci16(lcs_chan* c, const int16_t* iq_host, uint32_t n_in, uint8_t* out, uint32_t out_capacity,
                              int out_on_device, uint32_t* n_out, uint64_t* n_clipped) {
  if (!c) return LCS_ERR_ARG;
  if (c->fmt != LCS_IQ_CI16) return cfail(c, "lcs_chan_push_ci16: the channelizer's input format is not ci16");
  return lcs_chan_push(c, iq_host, n_in, out, out_capacity, out_on_device, n_out, n_clipped);
}

lcs_status lcs_chan_timing_read(lcs_chan* c, double* kernel_ms, uint64_t* launches) {
  if (!c) return LCS_ERR_ARG;
  if (!kernel_ms || !launches) return cfail(c, "lcs_chan_timing_read: null pointer");
  LCS_CUDA(c->ctx, c->clock.read(kernel_ms, launches));
  return LCS_OK;
}

}  // extern "C"
