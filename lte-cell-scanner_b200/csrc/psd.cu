// psd.cu - Welch power spectral density of a wideband recording (DESIGN.md section 4.8; contract in include/lcs_psd.h).
// Built into liblcs_psd.so, which uses the lcs_ctx of liblcs_b200.so.
//
// Every segment (N samples, hop N/2) is staged from the raw recording with the format conversion of iq_format.cuh, windowed
// by the periodic Hann window and transformed by an FP32 FFT in shared memory; |X|^2 per bin goes to a scratch row per
// segment, and one thread per bin adds the rows of a launch to the FP64 accumulator in segment order.
//
// The FFT is fft_tile (fft_tile.cuh), which carrier.cu shares.  A CTA holds 4096 points (32 KB).  For N <= 4096 one CTA
// transforms 4096/N whole segments.  Larger N is split four-step as
// N = N1 * N2 (N2 = 2^ceil(lg N / 2)): the column pass transforms, for 4096/N1 consecutive n2, the N1 samples
// x[n1*N2 + n2], multiplies by exp(-j2pi n2 k1/N) and writes Y[k1][n2]; the row pass transforms each row Y[k1][.] over
// n2 and gives X[k1 + N1*k2].  Twiddles and window are computed in double on the host and kept as float.
#include <cmath>
#include <cstring>
#include <new>
#include <vector>

#include "../../include/lcs_psd.h"
#include "fft_tile.cuh"
#include "iq_format.cuh"
#include "lcs_ctx.hpp"

namespace lcs {
namespace psd {

using namespace fft;
constexpr int LG_MIN = 6, LG_MAX = 16;   // N = 64 .. 65536

struct Params {
  const unsigned char* in;   // samples in the input format; local sample 0 is the first sample of local segment 0
  int n_seg;                 // segments of this launch
  int lg;                    // log2 N
  int lg1, lg2;              // four-step: log2 N1, log2 N2 (lg1 + lg2 = lg)
  const float* win;          // [N]
  const float2* tw;          // [N] exp(-j2pi m/N)
  float2* y;                 // four-step scratch [n_seg][N1][N2]
  float* pw;                 // [n_seg][N] |X[k]|^2
};

// N <= TILE: CTA b transforms segments [b * TILE/N, (b+1) * TILE/N) whole.
template <int FMT>
__global__ void __launch_bounds__(THREADS) psd_fft_kernel(Params P) {
  __shared__ float2 a[TILE];
  const int lg = P.lg, N = 1 << lg;
  const int seg0 = blockIdx.x << (LG_TILE - lg);
  for (int e = threadIdx.x; e < TILE; e += THREADS) {
    const int b = e >> lg, n = e & (N - 1), s = seg0 + b;
    float2 v = make_float2(0.f, 0.f);
    if (s < P.n_seg) {
      const float w = __ldg(P.win + n);
      v = load_iq<FMT>(P.in, (long long)s * (N / 2) + n);
      v = make_float2(v.x * w, v.y * w);
    }
    a[swz((b << lg) + bitrev(n, lg))] = v;
  }
  __syncthreads();
  fft_tile(a, lg, P.tw, lg);
  for (int e = threadIdx.x; e < TILE; e += THREADS) {
    const int s = seg0 + (e >> lg);
    if (s < P.n_seg) {
      const float2 x = a[swz(e)];
      P.pw[(size_t)s * N + (e & (N - 1))] = x.x * x.x + x.y * x.y;
    }
  }
}

// Four-step column pass: CTA (blockIdx.x, s) transforms columns n2 in [c0, c0 + C), C = TILE/N1, of segment s.
template <int FMT>
__global__ void __launch_bounds__(THREADS) psd_col_kernel(Params P) {
  __shared__ float2 a[TILE];
  const int lg = P.lg, lg1 = P.lg1, lgc = LG_TILE - lg1;
  const int N = 1 << lg, N2 = 1 << P.lg2, C = 1 << lgc;
  const int s = blockIdx.y, c0 = blockIdx.x << lgc;
  const long long m0 = (long long)s * (N / 2);
  for (int e = threadIdx.x; e < TILE; e += THREADS) {
    const int c = e & (C - 1), n1 = e >> lgc;
    const int n = n1 * N2 + c0 + c;
    const float w = __ldg(P.win + n);
    const float2 v = load_iq<FMT>(P.in, m0 + n);
    a[swz((c << lg1) + bitrev(n1, lg1))] = make_float2(v.x * w, v.y * w);
  }
  __syncthreads();
  fft_tile(a, lg1, P.tw, lg);
  float2* y = P.y + (size_t)s * N;
  for (int e = threadIdx.x; e < TILE; e += THREADS) {
    const int c = e & (C - 1), k1 = e >> lgc, n2 = c0 + c;
    y[(size_t)k1 * N2 + n2] = cmul(a[swz((c << lg1) + k1)], __ldg(P.tw + ((n2 * k1) & (N - 1))));
  }
}

// Four-step row pass: CTA (blockIdx.x, s) transforms rows k1 in [r0, r0 + R), R = TILE/N2, of segment s over n2.
__global__ void __launch_bounds__(THREADS) psd_row_kernel(Params P) {
  __shared__ float2 a[TILE];
  const int lg = P.lg, lg2 = P.lg2, lgr = LG_TILE - lg2;
  const int N = 1 << lg, N1 = 1 << P.lg1, N2 = 1 << lg2, R = 1 << lgr;
  const int s = blockIdx.y, r0 = blockIdx.x << lgr;
  const float2* y = P.y + (size_t)s * N + (size_t)r0 * N2;
  for (int e = threadIdx.x; e < TILE; e += THREADS) {
    const int r = e >> lg2, n2 = e & (N2 - 1);
    a[swz((r << lg2) + bitrev(n2, lg2))] = y[e];
  }
  __syncthreads();
  fft_tile(a, lg2, P.tw, lg);
  float* pw = P.pw + (size_t)s * N;
  for (int e = threadIdx.x; e < TILE; e += THREADS) {
    const int r = e & (R - 1), k2 = e >> lgr;
    const float2 x = a[swz((r << lg2) + k2)];
    pw[(r0 + r) + (size_t)N1 * k2] = x.x * x.x + x.y * x.y;
  }
}

// acc[k] += pw[0][k] + pw[1][k] + ... in segment order, one thread per bin.  With only N threads the loads in flight set
// the rate: ACC_UNROLL per thread, and small CTAs so that the threads spread over many SMs.
constexpr int ACC_THREADS = 64, ACC_UNROLL = 32;
__global__ void __launch_bounds__(ACC_THREADS) psd_accum_kernel(const float* __restrict__ pw, int n_seg, int N, double* acc) {
  const int k = blockIdx.x * ACC_THREADS + threadIdx.x;
  if (k >= N) return;
  double s = acc[k];
  int i = 0;
  for (; i + ACC_UNROLL <= n_seg; i += ACC_UNROLL) {
    float v[ACC_UNROLL];
#pragma unroll
    for (int j = 0; j < ACC_UNROLL; j++) v[j] = __ldg(pw + (size_t)(i + j) * N + k);
#pragma unroll
    for (int j = 0; j < ACC_UNROLL; j++) s += (double)v[j];
  }
  for (; i < n_seg; i++) s += (double)__ldg(pw + (size_t)i * N + k);
  acc[k] = s;
}

}  // namespace psd
}  // namespace lcs

using namespace lcs;
using namespace lcs::psd;

struct lcs_psd {
  lcs_ctx* ctx = nullptr;
  int fmt = LCS_IQ_CI16;
  long long fs = 0;
  int lg = 0, lg1 = 0, lg2 = 0;          // lg1 = 0: one pass (N <= TILE)
  uint32_t N = 0;
  double win_ss = 0;                     // sum of w[n]^2 over the double-precision window
  DevBuf<float> d_win;
  DevBuf<float2> d_tw;
  DevBuf<unsigned char> d_in;
  DevBuf<float2> d_y;
  DevBuf<float> d_pw;
  DevBuf<double> d_acc;
  uint32_t chunk = 1;                    // segments per launch (bounds the device scratch)
  SampleCarry carry;                     // stream samples from the first sample of the next segment on (< N of them)
  uint64_t n_seg = 0;                    // segments accumulated since the last read
  KernelClock clock;                     // the kernels of each launch chunk
};

namespace {

lcs_status pfail(const lcs_psd* p, const char* msg) { return fail(p ? p->ctx : nullptr, LCS_ERR_ARG, msg); }

// The transform kernels of a launch chunk; LCS_ERR_ARG, and no launch, for a format the spectrum does not take.
lcs_status launch_fft(const lcs_psd* p, const Params& P, cudaStream_t st) {
  return StreamFormats::dispatch(p->fmt, [&](auto FMT) {
    if (!p->lg1) {
      psd_fft_kernel<FMT><<<(P.n_seg + (TILE >> p->lg) - 1) / (TILE >> p->lg), THREADS, 0, st>>>(P);
    } else {
      psd_col_kernel<FMT><<<dim3((1u << p->lg2) >> (LG_TILE - p->lg1), P.n_seg), THREADS, 0, st>>>(P);
      psd_row_kernel<<<dim3((1u << p->lg1) >> (LG_TILE - p->lg2), P.n_seg), THREADS, 0, st>>>(P);
    }
  });
}

// Segments [0, n) of the virtual input carry ++ b, whose sample 0 is the first sample of segment 0.
lcs_status run(lcs_psd* p, const unsigned char* b, uint64_t n) {
  lcs_ctx* ctx = p->ctx;
  cudaStream_t st = ctx->streams[0];
  const size_t N = p->N, hop = N / 2;
  for (uint64_t c0 = 0; c0 < n; c0 += p->chunk) {
    const uint32_t ns = (uint32_t)std::min<uint64_t>(p->chunk, n - c0);
    LCS_CUDA(ctx, p->carry.upload(b, c0 * hop, (c0 + ns - 1) * hop + N, p->d_in.p, st));
    Params P;
    P.in = p->d_in.p;
    P.n_seg = (int)ns;
    P.lg = p->lg;
    P.lg1 = p->lg1;
    P.lg2 = p->lg2;
    P.win = p->d_win.p;
    P.tw = p->d_tw.p;
    P.y = p->d_y.p;
    P.pw = p->d_pw.p;
    LCS_CUDA(ctx, p->clock.begin(st));
    if (launch_fft(p, P, st) != LCS_OK) return fail(ctx, LCS_ERR_ARG, "lcs_psd: bad iq_format");
    psd_accum_kernel<<<(p->N + ACC_THREADS - 1) / ACC_THREADS, ACC_THREADS, 0, st>>>(p->d_pw.p, (int)ns, (int)p->N, p->d_acc.p);
    const int launches = p->lg1 ? 3 : 2;
    ctx->launches += launches;
    LCS_CUDA(ctx, cudaGetLastError());
    LCS_CUDA(ctx, p->clock.end(st, launches));
    LCS_CUDA(ctx, cudaStreamSynchronize(st));
    p->n_seg += ns;
  }
  return LCS_OK;
}

}  // namespace

extern "C" {

lcs_status lcs_psd_create(lcs_ctx* ctx, double fs_in, int iq_format, uint32_t nfft, lcs_psd** out) {
  if (!ctx || !out) return fail(ctx, LCS_ERR_ARG, "lcs_psd_create: null argument");
  const double r = std::round(fs_in);
  if (!std::isfinite(fs_in) || std::fabs(fs_in - r) > 1e-6 || !(r > 0) || r > 250e6)
    return fail(ctx, LCS_ERR_ARG, "lcs_psd_create: fs_in must be an integer number of Hz in (0, 250] MHz");
  if (!StreamFormats::has(iq_format))
    return fail(ctx, LCS_ERR_ARG, "lcs_psd_create: iq_format must be LCS_IQ_CI16, CS8, CU8 or CF32");
  int lg = 0;
  while (lg <= LG_MAX && (1u << lg) < nfft) lg++;
  if (lg < LG_MIN || lg > LG_MAX || (1u << lg) != nfft)
    return fail(ctx, LCS_ERR_ARG, "lcs_psd_create: nfft must be a power of two in [64, 65536]");
  lcs_psd* p = new (std::nothrow) lcs_psd();
  if (!p) return fail(ctx, LCS_ERR_STATE, "lcs_psd_create: out of memory");
  p->ctx = ctx;
  p->fmt = iq_format;
  p->carry.esz = sample_bytes(iq_format);
  p->fs = (long long)r;
  p->N = nfft;
  p->lg = lg;
  if (lg > LG_TILE) {
    p->lg2 = (lg + 1) / 2;
    p->lg1 = lg - p->lg2;
  }
  std::vector<float> win(nfft);
  std::vector<float2> tw(nfft);
  for (uint32_t n = 0; n < nfft; n++) {
    const double w = 0.5 - 0.5 * std::cos(2 * M_PI * (double)n / (double)nfft);
    win[n] = (float)w;
    p->win_ss += w * w;
    const double ang = -2 * M_PI * (double)n / (double)nfft;
    tw[n] = make_float2((float)std::cos(ang), (float)std::sin(ang));
  }
  // segments per launch: |X|^2 rows (and the four-step rows) within 64 MB
  const size_t per_seg = (size_t)nfft * (sizeof(float) + (p->lg1 ? sizeof(float2) : 0));
  p->chunk = (uint32_t)std::max<size_t>(1, (64ull << 20) / per_seg);
  const size_t in_max = ((size_t)(p->chunk - 1) * (nfft / 2) + nfft) * p->carry.esz;
  cudaError_t e = cudaSetDevice(ctx->device);
  if (e == cudaSuccess) e = p->d_win.alloc(nfft);
  if (e == cudaSuccess) e = p->d_tw.alloc(nfft);
  if (e == cudaSuccess) e = p->d_acc.alloc(nfft);
  if (e == cudaSuccess) e = p->d_pw.alloc((size_t)p->chunk * nfft);
  if (e == cudaSuccess && p->lg1) e = p->d_y.alloc((size_t)p->chunk * nfft);
  if (e == cudaSuccess) e = p->d_in.alloc(in_max);
  if (e == cudaSuccess) e = cudaMemcpy(p->d_win.p, win.data(), nfft * sizeof(float), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(p->d_tw.p, tw.data(), nfft * sizeof(float2), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemset(p->d_acc.p, 0, nfft * sizeof(double));
  if (e != cudaSuccess) {
    delete p;
    return fail(ctx, LCS_ERR_CUDA, std::string("lcs_psd_create: ") + cudaGetErrorString(e));
  }
  *out = p;
  return LCS_OK;
}

void lcs_psd_destroy(lcs_psd* p) {
  if (!p) return;
  cudaSetDevice(p->ctx->device);             // its buffers and events belong to the context's device
  delete p;
}

lcs_status lcs_psd_push(lcs_psd* p, const void* iq_host, uint32_t n_in) {
  if (!p) return LCS_ERR_ARG;
  if (!iq_host && n_in) return pfail(p, "lcs_psd_push: null samples");
  const unsigned char* b = static_cast<const unsigned char*>(iq_host);
  const size_t total = p->carry.size() + n_in, hop = p->N / 2;
  const uint64_t k = total >= p->N ? (total - p->N) / hop + 1 : 0;   // segments this push completes
  if (k) {
    LCS_CUDA(p->ctx, cudaSetDevice(p->ctx->device));
    lcs_status rc = run(p, b, k);
    if (rc != LCS_OK) return rc;
  }
  // keep the samples from the first sample of the next segment on
  p->carry.advance(b, n_in, (size_t)k * hop);
  return LCS_OK;
}

lcs_status lcs_psd_read(lcs_psd* p, double* out, uint64_t* n_segments) {
  if (!p) return LCS_ERR_ARG;
  if (!out || !n_segments) return pfail(p, "lcs_psd_read: null pointer");
  const uint32_t N = p->N;
  std::vector<double> acc(N, 0.0);
  if (p->n_seg) {
    LCS_CUDA(p->ctx, cudaSetDevice(p->ctx->device));
    LCS_CUDA(p->ctx, cudaMemcpy(acc.data(), p->d_acc.p, N * sizeof(double), cudaMemcpyDeviceToHost));
    LCS_CUDA(p->ctx, cudaMemset(p->d_acc.p, 0, N * sizeof(double)));
  }
  const double scale = p->n_seg ? 1.0 / ((double)p->n_seg * (double)p->fs * p->win_ss) : 0.0;
  for (uint32_t i = 0; i < N; i++) out[i] = acc[(i + N / 2) % N] * scale;
  *n_segments = p->n_seg;
  p->n_seg = 0;
  return LCS_OK;
}

lcs_status lcs_psd_timing_read(lcs_psd* p, double* kernel_ms, uint64_t* launches) {
  if (!p) return LCS_ERR_ARG;
  if (!kernel_ms || !launches) return pfail(p, "lcs_psd_timing_read: null pointer");
  LCS_CUDA(p->ctx, p->clock.read(kernel_ms, launches));
  return LCS_OK;
}

}  // extern "C"
