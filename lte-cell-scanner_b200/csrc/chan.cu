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
#include <cmath>
#include <cstring>
#include <new>
#include <type_traits>
#include <vector>

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
// Dynamic shared memory of a launch: the input tile, D rows of TILE + 2M/D + 1 samples.  The largest any channelizer can
// ask for (D = 64, L = MAX_TAPS) is the kernels' attribute, set identically by every lcs_chan_create: the attribute is one
// value per function for the whole process, so a per-channelizer value would cap the launches of channelizers created
// earlier with a larger D.
constexpr int smem_bytes(int D, int M) { return D * (TILE + (2 * M) / D + 1) * (int)sizeof(float2); }
constexpr int SMEM_CAP = smem_bytes(64, (MAX_TAPS - 1) / 2);   // 98 816 bytes
static_assert(SMEM_CAP <= 227 * 1024, "input tile exceeds the shared memory of an SM");

struct Params {
  const int* in;               // packed ci16 (I low, Q high); local sample 0 is the first input of local output 0 (n0*D-M)
  long long n_in;              // valid samples at `in` (later ones read as 0; no valid output uses them)
  int D, L, M, qlen;
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

template <bool POWER>
__global__ void __launch_bounds__(THREADS) chan_kernel(Params P) {
  extern __shared__ float2 xs[];                     // [D][qlen]
  const int tile = blockIdx.x;
  const int nl0 = tile * TILE;
  const long long j0 = (long long)nl0 * P.D;
  const int span = (TILE - 1) * P.D + 2 * P.M + 1;
  for (int j = threadIdx.x; j < span; j += THREADS) {
    const long long g = j0 + j;
    float2 v = make_float2(0.f, 0.f);
    if (g < P.n_in) {
      const int w = __ldg(P.in + g);
      v = make_float2((float)(short)(w & 0xffff) * (1.f / 32768.f), (float)(short)(w >> 16) * (1.f / 32768.f));
    }
    xs[(j % P.D) * P.qlen + j / P.D] = v;
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
    if (++ph == P.D) { ph = 0; row++; }
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
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) s += __shfl_down_sync(0xffffffffu, s, o);
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
        double sn, cs;
        sincospi(-2.0 * (double)p / (double)P.fs, &sn, &cs);
        const double yr = (double)acc[i][r].x * cs - (double)acc[i][r].y * sn;
        const double yi = (double)acc[i][r].x * sn + (double)acc[i][r].y * cs;
        double vr = rint(127.0 + gn * yr), vi = rint(127.0 + gn * yi);
        clipped += (vr < 0 || vr > 255) + (vi < 0 || vi > 255);
        vr = fmin(fmax(vr, 0.0), 255.0);
        vi = fmin(fmax(vi, 0.0), 255.0);
        unsigned char* o = P.out + (size_t)c * P.out_stride + 2 * (size_t)nl;
        o[0] = (unsigned char)vr;
        o[1] = (unsigned char)vi;
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

// Kaiser-windowed sinc of odd length L, cutoff 0.96 MHz at fs, DC gain 1, rounded to float.
static void kaiser_sinc(int L, double fs, std::vector<float>& out) {
  const int M = (L - 1) / 2;
  const double beta = kaiser_beta(), i0b = bessel_i0(beta), fcn = 2 * kCut / fs;
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
  for (int n = 0; n < L; n++) out[n] = (float)(h[n] / sum);
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
  kaiser_sinc(L, fs, h);
  if (meets_spec(h, fs)) {
    std::vector<float> g;
    while (L >= 5) {
      kaiser_sinc(L - 2, fs, g);
      if (!meets_spec(g, fs)) break;
      L -= 2;
      h.swap(g);
    }
    return L;
  }
  while (L < MAX_TAPS) {
    L += 2;
    kaiser_sinc(L, fs, h);
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

}  // namespace chn
}  // namespace lcs

using namespace lcs;
using namespace lcs::chn;

struct lcs_chan {
  lcs_ctx* ctx = nullptr;
  int D = 0, L = 0, M = 0;
  long long fs = 0;
  uint32_t n_ch = 0;
  std::vector<float> h;
  std::vector<float> gain;
  std::vector<long long> delta, step;
  DevBuf<float2> d_taps;
  DevBuf<double2> d_taps64;
  DevBuf<long long> d_step;
  DevBuf<float> d_gain;
  DevBuf<int> d_in;
  DevBuf<unsigned char> d_out;
  DevBuf<unsigned long long> d_clip;
  DevBuf<double> d_pw;
  uint32_t chunk = TILE;                 // outputs per launch (bounds the device scratch)
  std::vector<int> carry;                // stream samples [n_out*D - M, n_in) (zeros before the stream starts)
  uint64_t n_in = 0, n_out = 0;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr;
  double kernel_ms = 0;
  uint64_t kernel_launches = 0;
  ~lcs_chan() {
    if (ev0) cudaEventDestroy(ev0);
    if (ev1) cudaEventDestroy(ev1);
  }
};

namespace {

// outputs after n input samples of a stream
uint64_t outputs_after(int D, int M, uint64_t n) { return n >= (uint64_t)M + 1 ? (n - 1 - M) / D + 1 : 0; }

// Outputs [0, n_out) of the virtual input a (na samples) ++ b (nb samples), whose sample 0 is the first input of output 0
// (stream output n_abs0).  power: per-channel sums of |y|^2 are added to pw_sum; otherwise bytes go to out (row stride
// out_stride, on the device or the host) and clip counts to d_clip.
lcs_status run(lcs_chan* c, const int* a, size_t na, const int* b, size_t nb, uint64_t n_abs0, uint64_t n_out, bool power,
               unsigned char* out, size_t out_stride, bool out_dev, std::vector<double>* pw_sum) {
  lcs_ctx* ctx = c->ctx;
  cudaStream_t st = ctx->streams[0];
  const size_t span_max = (size_t)(c->chunk - 1) * c->D + 2 * c->M + 1;
  LCS_CUDA(ctx, c->d_in.ensure(span_max + (size_t)TILE * c->D));
  if (!power && !out_dev) LCS_CUDA(ctx, c->d_out.ensure((size_t)c->n_ch * c->chunk * 2));
  if (power) LCS_CUDA(ctx, c->d_pw.ensure((size_t)c->n_ch * (c->chunk / TILE)));
  const int qlen = TILE + (2 * c->M) / c->D + 1;
  const size_t smem = (size_t)smem_bytes(c->D, c->M);
  std::vector<double> pw;
  for (uint64_t e0 = 0; e0 < n_out; e0 += c->chunk) {
    const uint32_t ne = (uint32_t)std::min<uint64_t>(c->chunk, n_out - e0);
    const size_t lo = (size_t)e0 * c->D;
    const size_t hi = std::min(lo + (size_t)(ne - 1) * c->D + 2 * c->M + 1, na + nb);
    // samples [lo, hi) of a ++ b
    if (lo < na) LCS_CUDA(ctx, cudaMemcpyAsync(c->d_in.p, a + lo, (std::min(hi, na) - lo) * 4, cudaMemcpyHostToDevice, st));
    if (hi > na) {
      const size_t s = std::max(lo, na);
      LCS_CUDA(ctx, cudaMemcpyAsync(c->d_in.p + (s - lo), b + (s - na), (hi - s) * 4, cudaMemcpyHostToDevice, st));
    }
    Params P;
    P.in = c->d_in.p;
    P.n_in = (long long)(hi - lo);
    P.D = c->D;
    P.L = c->L;
    P.M = c->M;
    P.qlen = qlen;
    P.n_out = (int)ne;
    P.n0 = (long long)(n_abs0 + e0);
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
    const dim3 grid((ne + TILE - 1) / TILE, (c->n_ch + CH_CTA - 1) / CH_CTA);
    LCS_CUDA(ctx, cudaEventRecord(c->ev0, st));
    if (power)
      chan_kernel<true><<<grid, THREADS, smem, st>>>(P);
    else
      chan_kernel<false><<<grid, THREADS, smem, st>>>(P);
    ctx->launches++;
    LCS_CUDA(ctx, cudaGetLastError());
    LCS_CUDA(ctx, cudaEventRecord(c->ev1, st));
    if (power) {
      pw.resize((size_t)c->n_ch * grid.x);
      LCS_CUDA(ctx, cudaMemcpyAsync(pw.data(), c->d_pw.p, pw.size() * 8, cudaMemcpyDeviceToHost, st));
    } else if (!out_dev) {
      LCS_CUDA(ctx, cudaMemcpy2DAsync(out + 2 * e0, out_stride, c->d_out.p, (size_t)ne * 2, (size_t)ne * 2, c->n_ch,
                                      cudaMemcpyDeviceToHost, st));
    }
    LCS_CUDA(ctx, cudaStreamSynchronize(st));
    float ms = 0;
    LCS_CUDA(ctx, cudaEventElapsedTime(&ms, c->ev0, c->ev1));
    c->kernel_ms += ms;
    c->kernel_launches++;
    if (power)   // fixed order: tiles of a chunk, chunks in stream order
      for (uint32_t ch = 0; ch < c->n_ch; ch++)
        for (uint32_t t = 0; t < grid.x; t++) (*pw_sum)[ch] += pw[(size_t)ch * grid.x + t];
  }
  return LCS_OK;
}

lcs_status cfail(const lcs_chan* c, const char* msg) { return fail(c ? c->ctx : nullptr, LCS_ERR_ARG, msg); }

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

lcs_status lcs_chan_create(lcs_ctx* ctx, double fs_in, double fc_in, uint32_t n_ch, const double* fc_ch, const float* gain,
                           lcs_chan** out) {
  if (!ctx || !out || !fc_ch) return fail(ctx, LCS_ERR_ARG, "lcs_chan_create: null argument");
  int D = 0;
  if (!decimation(fs_in, &D)) return fail(ctx, LCS_ERR_ARG, "lcs_chan_create: fs_in must be D * 1.92 MHz, D in [2, 64]");
  if (n_ch < 1 || n_ch > 1024) return fail(ctx, LCS_ERR_ARG, "lcs_chan_create: n_ch must be in [1, 1024]");
  if (!std::isfinite(fc_in)) return fail(ctx, LCS_ERR_ARG, "lcs_chan_create: fc_in is not finite");
  const long long fs = (long long)D * 1920000LL;
  std::vector<long long> delta(n_ch);
  for (uint32_t c = 0; c < n_ch; c++) {
    const double d = fc_ch[c] - fc_in;
    if (!std::isfinite(d) || std::fabs(d - std::round(d)) > 1e-6)
      return fail(ctx, LCS_ERR_ARG, "lcs_chan_create: channel offset fc_ch - fc_in is not an integer number of Hz");
    delta[c] = (long long)std::llround(d);
    if (std::llabs(delta[c]) > fs / 2 - 960000)
      return fail(ctx, LCS_ERR_ARG, "lcs_chan_create: channel band (+-0.96 MHz) outside the input band");
    if (gain && !(std::isfinite(gain[c]) && gain[c] > 0)) return fail(ctx, LCS_ERR_ARG, "lcs_chan_create: gain must be finite and > 0");
  }
  lcs_chan* c = new (std::nothrow) lcs_chan();
  if (!c) return fail(ctx, LCS_ERR_STATE, "lcs_chan_create: out of memory");
  c->ctx = ctx;
  c->D = D;
  c->fs = fs;
  c->n_ch = n_ch;
  c->L = design(D * kFsCh, c->h);
  c->M = (c->L - 1) / 2;
  c->delta = delta;
  c->gain.assign(n_ch, 1.0f);
  if (gain) c->gain.assign(gain, gain + n_ch);
  c->carry.assign(c->M, 0);
  // outputs per launch: device output scratch <= 32 MB, input tile <= 64 MB
  const uint64_t by_out = (32ull << 20) / (2ull * n_ch), by_in = (64ull << 20) / (4ull * D);
  c->chunk = (uint32_t)std::max<uint64_t>(TILE, std::min(by_out, by_in) / TILE * TILE);
  std::vector<float2> taps((size_t)n_ch * c->L);
  std::vector<double2> taps64((size_t)n_ch * c->L);
  c->step.resize(n_ch);
  for (uint32_t ch = 0; ch < n_ch; ch++) {
    c->step[ch] = (((long long)D * delta[ch]) % fs + fs) % fs;
    for (int t = 0; t < c->L; t++) {
      const long long p = (((long long)(t - c->M) * delta[ch]) % fs + fs) % fs;
      const double a = 2 * M_PI * (double)p / (double)fs;
      const double2 g = make_double2((double)c->h[t] * std::cos(a), (double)c->h[t] * std::sin(a));
      taps64[(size_t)ch * c->L + t] = g;
      taps[(size_t)ch * c->L + t] = make_float2((float)g.x, (float)g.y);
    }
  }
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
  if (e == cudaSuccess) e = cudaEventCreate(&c->ev0);
  if (e == cudaSuccess) e = cudaEventCreate(&c->ev1);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(chan_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_CAP);
  if (e == cudaSuccess) e = cudaFuncSetAttribute(chan_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_CAP);
  if (e != cudaSuccess) {
    delete c;
    return fail(ctx, LCS_ERR_CUDA, std::string("lcs_chan_create: ") + cudaGetErrorString(e));
  }
  *out = c;
  return LCS_OK;
}

void lcs_chan_destroy(lcs_chan* c) {
  if (!c) return;
  cudaSetDevice(c->ctx->device);             // its buffers and events belong to the context's device
  delete c;
}

lcs_status lcs_chan_auto_gain_ci16(lcs_chan* c, const int16_t* iq_host, uint32_t n) {
  if (!c) return LCS_ERR_ARG;
  if (!iq_host) return cfail(c, "lcs_chan_auto_gain_ci16: null samples");
  const uint64_t n_out = outputs_after(c->D, c->M, n);      // what a fresh channelizer would produce
  if (n_out == 0) return cfail(c, "lcs_chan_auto_gain_ci16: fewer samples than one output needs");
  LCS_CUDA(c->ctx, cudaSetDevice(c->ctx->device));
  const std::vector<int> zeros(c->M, 0);
  std::vector<double> sum(c->n_ch, 0.0);
  lcs_status rc = run(c, zeros.data(), zeros.size(), reinterpret_cast<const int*>(iq_host), n, 0, n_out, true, nullptr, 0, false, &sum);
  if (rc != LCS_OK) return rc;
  for (uint32_t ch = 0; ch < c->n_ch; ch++) {
    const double ms = sum[ch] / (double)n_out;
    c->gain[ch] = ms > 0 ? (float)(0.25 / std::sqrt(ms)) : 1.0f;
  }
  LCS_CUDA(c->ctx, cudaMemcpy(c->d_gain.p, c->gain.data(), c->n_ch * 4, cudaMemcpyHostToDevice));
  return LCS_OK;
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
  const uint64_t k = outputs_after(c->D, c->M, c->n_in + n_in) - c->n_out;
  if (k > UINT32_MAX) return cfail(c, "lcs_chan_n_out: push too long");
  *n_out = (uint32_t)k;
  return LCS_OK;
}

lcs_status lcs_chan_push_ci16(lcs_chan* c, const int16_t* iq_host, uint32_t n_in, uint8_t* out, uint32_t out_capacity,
                              int out_on_device, uint32_t* n_out, uint64_t* n_clipped) {
  if (!c) return LCS_ERR_ARG;
  if ((!iq_host && n_in) || !n_out) return cfail(c, "lcs_chan_push_ci16: null pointer");
  const uint64_t k = outputs_after(c->D, c->M, c->n_in + n_in) - c->n_out;
  if (k > out_capacity) return cfail(c, "lcs_chan_push_ci16: out_capacity is smaller than the outputs of this push");
  if (k && !out) return cfail(c, "lcs_chan_push_ci16: null output");
  LCS_CUDA(c->ctx, cudaSetDevice(c->ctx->device));
  LCS_CUDA(c->ctx, cudaMemsetAsync(c->d_clip.p, 0, c->n_ch * 8, c->ctx->streams[0]));
  const int* b = reinterpret_cast<const int*>(iq_host);
  if (k) {
    lcs_status rc = run(c, c->carry.data(), c->carry.size(), b, n_in, c->n_out, k, false, out, (size_t)out_capacity * 2,
                        out_on_device != 0, nullptr);
    if (rc != LCS_OK) return rc;
  }
  // keep the samples from the first input of the next output on
  const size_t drop = (size_t)k * c->D, na = c->carry.size();
  std::vector<int> nc;
  nc.reserve(na + n_in - drop);
  if (drop < na) nc.insert(nc.end(), c->carry.begin() + drop, c->carry.end());
  nc.insert(nc.end(), b + (drop > na ? drop - na : 0), b + n_in);
  c->carry.swap(nc);
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

lcs_status lcs_chan_timing_read(lcs_chan* c, double* kernel_ms, uint64_t* launches) {
  if (!c) return LCS_ERR_ARG;
  if (!kernel_ms || !launches) return cfail(c, "lcs_chan_timing_read: null pointer");
  *kernel_ms = c->kernel_ms;
  *launches = c->kernel_launches;
  c->kernel_ms = 0;
  c->kernel_launches = 0;
  return LCS_OK;
}

}  // extern "C"
