// lcs_ctx.hpp - context / plan objects behind the opaque handles of include/lcs_b200.h.
#pragma once
#include <algorithm>
#include <memory>
#include <string>
#include <vector>

#include "lcs_internal.hpp"
#include "tc_layout.hpp"

namespace lcs {

template <typename T>
struct DevBuf {   // owning device allocation
  T* p = nullptr;
  size_t n = 0;
  DevBuf() {}
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  ~DevBuf() { if (p) cudaFree(p); }
  cudaError_t alloc(size_t count) {
    if (p) { cudaFree(p); p = nullptr; }
    n = count;
    return cudaMalloc((void**)&p, std::max<size_t>(count, 1) * sizeof(T));
  }
  cudaError_t ensure(size_t count) { return (p && n >= count) ? cudaSuccess : alloc(count); }
  void swap(DevBuf& o) { std::swap(p, o.p); std::swap(n, o.n); }
};

template <class T>
struct PinBuf {   // owning page-locked host allocation (asynchronous copies need one)
  T* p = nullptr;
  size_t n = 0;
  PinBuf() {}
  PinBuf(const PinBuf&) = delete;
  PinBuf& operator=(const PinBuf&) = delete;
  ~PinBuf() { if (p) cudaFreeHost(p); }
  cudaError_t ensure(size_t count) {
    if (p && n >= count) return cudaSuccess;
    if (p) { cudaFreeHost(p); p = nullptr; }
    n = count;
    return cudaMallocHost((void**)&p, std::max<size_t>(count, 1) * sizeof(T));
  }
};

// The small host tables of a launch, staged in page-locked memory and uploaded with one asynchronous copy.  reset(bytes)
// makes room for slices of `bytes` in all, counting 16 bytes of alignment per slice; take() and put() hand out host
// slices, upload() copies every slice taken since the reset, and dev() is the device address of a host slice.  A slice
// may be written again once the stream its copy went to has been synchronised.
struct Staging {
  PinBuf<unsigned char> h;
  DevBuf<unsigned char> d;
  size_t off = 0;
  cudaError_t reset(size_t bytes) {
    off = 0;
    cudaError_t e = h.ensure(bytes);
    return e == cudaSuccess ? d.ensure(bytes) : e;
  }
  template <class T> T* take(size_t n) {
    off = (off + 15) & ~(size_t)15;
    T* p = reinterpret_cast<T*>(h.p + off);
    off += n * sizeof(T);
    return p;
  }
  template <class T> T* put(const std::vector<T>& v) {
    T* p = take<T>(v.size());
    std::copy(v.begin(), v.end(), p);
    return p;
  }
  template <class T> T* dev(T* host) const {
    return reinterpret_cast<T*>(d.p + (reinterpret_cast<const unsigned char*>(host) - h.p));
  }
  cudaError_t upload(cudaStream_t st) const { return cudaMemcpyAsync(d.p, h.p, off, cudaMemcpyHostToDevice, st); }
};

// Kernel time of a handle: CUDA event pairs recorded around groups of launches, each committed with the number of kernels
// it covers.  Nothing waits for a pair before read(), so launches that are not synchronised can be timed as well.
class KernelClock {
 public:
  typedef std::pair<cudaEvent_t, cudaEvent_t> Pair;
  KernelClock() = default;
  KernelClock(const KernelClock&) = delete;
  KernelClock& operator=(const KernelClock&) = delete;
  ~KernelClock() {
    for (const Pair& ev : pool_) destroy(ev);
    for (const Used& u : used_) destroy(u.ev);
    destroy(open_);
  }
  // The pair of the next group, for a caller that records it; a group that fails before its commit leaves it open.
  cudaError_t open(const Pair** ev) {
    if (!open_.first && !pool_.empty()) {
      open_ = pool_.back();
      pool_.pop_back();
    }
    cudaError_t e = open_.first ? cudaSuccess : cudaEventCreate(&open_.first);
    if (e == cudaSuccess && !open_.second) e = cudaEventCreate(&open_.second);
    *ev = &open_;
    return e;
  }
  // The open pair has been recorded around `kernels` kernels.
  cudaError_t commit(uint64_t kernels) {
    used_.push_back(Used{open_, kernels});
    open_ = Pair(nullptr, nullptr);
    return used_.size() >= 1024 ? fold(512) : cudaSuccess;   // bound the list: the oldest half into the running sum
  }
  // open and commit for a group whose launches are enqueued between begin and end on one stream.
  cudaError_t begin(cudaStream_t st) {
    const Pair* ev = nullptr;
    cudaError_t e = open(&ev);
    return e == cudaSuccess ? cudaEventRecord(ev->first, st) : e;
  }
  cudaError_t end(cudaStream_t st, uint64_t kernels) {
    cudaError_t e = cudaEventRecord(open_.second, st);
    return e == cudaSuccess ? commit(kernels) : e;
  }
  // Kernel time and kernel count of the groups committed since the last read, summed in record order.
  cudaError_t read(double* ms, uint64_t* kernels) {
    cudaError_t e = fold(used_.size());
    if (e != cudaSuccess) return e;
    *ms = acc_ms_;
    *kernels = acc_n_;
    acc_ms_ = 0;
    acc_n_ = 0;
    return cudaSuccess;
  }

 private:
  struct Used {
    Pair ev;
    uint64_t kernels;
  };
  std::vector<Pair> pool_;
  std::vector<Used> used_;
  Pair open_{nullptr, nullptr};
  double acc_ms_ = 0;        // the pairs already folded out of used_
  uint64_t acc_n_ = 0;
  static void destroy(const Pair& ev) {
    if (ev.first) cudaEventDestroy(ev.first);
    if (ev.second) cudaEventDestroy(ev.second);
  }
  // Wait for the oldest n pairs, add them to the running sums and return them to the pool.
  cudaError_t fold(size_t n) {
    cudaError_t e = cudaSuccess;
    size_t i = 0;
    for (; i < n; i++) {
      float ms = 0;
      e = cudaEventSynchronize(used_[i].ev.second);
      if (e == cudaSuccess) e = cudaEventElapsedTime(&ms, used_[i].ev.first, used_[i].ev.second);
      if (e != cudaSuccess) break;
      acc_ms_ += ms;
      acc_n_ += used_[i].kernels;
      pool_.push_back(used_[i].ev);
    }
    used_.erase(used_.begin(), used_.begin() + i);
    return e;
  }
};

// The raw samples a streaming handle keeps from one push to the next: a push reads carry ++ pushed samples as one input.
struct SampleCarry {
  size_t esz = 0;                    // bytes per sample
  std::vector<unsigned char> bytes;
  size_t size() const { return bytes.size() / esz; }
  // Copy samples [lo, hi) of carry ++ push to dst, asynchronously on st.
  cudaError_t upload(const unsigned char* push, size_t lo, size_t hi, unsigned char* dst, cudaStream_t st) const {
    const size_t na = size();
    cudaError_t e = cudaSuccess;
    if (lo < na) e = cudaMemcpyAsync(dst, bytes.data() + lo * esz, (std::min(hi, na) - lo) * esz, cudaMemcpyHostToDevice, st);
    if (e == cudaSuccess && hi > na) {
      const size_t s = std::max(lo, na);
      e = cudaMemcpyAsync(dst + (s - lo) * esz, push + (s - na) * esz, (hi - s) * esz, cudaMemcpyHostToDevice, st);
    }
    return e;
  }
  // Consume the first `drop` samples of carry ++ push (n_push samples) and carry the rest.
  void advance(const unsigned char* push, size_t n_push, size_t drop) {
    const size_t na = size();
    std::vector<unsigned char> nc;
    nc.reserve((na + n_push - drop) * esz);
    if (drop < na) nc.insert(nc.end(), bytes.begin() + drop * esz, bytes.end());
    if (n_push) nc.insert(nc.end(), push + (drop > na ? drop - na : 0) * esz, push + n_push * esz);
    bytes.swap(nc);
  }
};

// One search configuration: what xcorr_pss is called with besides the capture buffer (searcher.h:22-31).
struct PlanCfg {
  double fc_req = 0, fc_prog = 0, fs_prog = 0;
  std::vector<double> f;      // f_search_set
};

// A set of search configurations that share the capture-buffer shape: the operands of both correlator kernels for every
// plan, resident in HBM.  The integer geometry (fold offsets, pass tables) is computed on the host, the templates
// (conj(fshift(pss_td))/137 of searcher.cpp:145-151, their FP32 roundings and 24-bit digit planes) by one kernel
// (planset.cu) - a frequency sweep builds one plan per centre frequency in a single launch.
struct PlanSet {
  lcs_ctx* ctx = nullptr;
  XcorrGeom geom{};
  uint32_t n_plans = 0;
  std::vector<PlanCfg> cfg;
  std::vector<int> h_nf;
  // builder inputs
  DevBuf<double> d_cfg;            // [n_plans][4 + n_f_stride]: fc_req, fc_prog, fs_prog, n_f, f[]
  DevBuf<int> d_nf;                // [n_plans]
  // FP32 correlator operands
  bool has_fp32 = false;
  DevBuf<float4> d_w01;            // [n_plans][n_f_stride][140] (root0, root1)
  DevBuf<float2> d_w2;             // [n_plans][n_f_stride][140] root2
  DevBuf<int> d_soff;              // [n_plans][n_comb][n_f_stride]
  DevBuf<int> d_smin;              // [n_plans][n_comb][n_fchunk]
  // tensor-core correlator operands
  bool tc_ready = false;
  std::string tc_why;              // why not, when !tc_ready
  tc::Layout lay{48, 2};
  uint32_t n_pass = 1;
  float inv_scale = 0;             // 1 / (S * 128)
  DevBuf<unsigned char> d_b;       // [n_plans][n_pass][lay.b_bytes()] int8 digit planes in wgmma core-matrix order
  DevBuf<float> d_corr;            // [n_plans][n_pass][2][npad]
  DevBuf<tc::PassGeo> d_geo;       // [n_plans][n_pass]
  DevBuf<int16_t> d_dsh;           // [n_plans][n_pass][M_MAX][npad] fold offset of the column minus the pass minimum
  DevBuf<int> d_flag;              // builder diagnostics (non-zero: a digit-plane bound was exceeded)
  PinBuf<unsigned char> h_stage;   // page-locked staging of the host-built tables
  cudaEvent_t staged = nullptr;    // the previous upload out of h_stage has completed
  ~PlanSet() { if (staged) cudaEventDestroy(staged); }
};

// Scratch of the per-peak stages (chain_gpu.cu).  Every stage synchronises its stream before it returns, so the next
// stage, on any stream, may reuse the staging.
struct ChainScratch {
  DevBuf<signed char> d_sss_tab;   // [168][3][2][62] +-1
  DevBuf<double2> d_pss_fd;        // [3][62]
  Staging up;                      // per stage: segment starts and shifts, peak parameters or the cells' grid geometry
  PinBuf<unsigned char> h_down;    // page-locked landing zone of the results
  DevBuf<double2> d_psss;          // [n_seg][62]
  DevBuf<double> d_est;            // [124] np + 4x62 complex
  DevBuf<double> d_ll;             // [4][168]
  DevBuf<double2> d_tfg;           // [cell][TFG_MAX][72]
};

}  // namespace lcs

struct lcs_xcorr_plan;

struct lcs_ctx {
  int device = 0;
  int n_sm = 0;
  static constexpr int N_STREAMS = 3;           // chunks of the host-batch calls rotate over these
  cudaStream_t streams[N_STREAMS] = {nullptr, nullptr, nullptr};
  std::string last_error;
  uint64_t launches = 0;
  std::vector<lcs_xcorr_plan*> cached_plans;   // for the plan-less drop-in calls
  // constants of the plan builder
  lcs::DevBuf<double> d_pss_td;                // [3][137] complex double (lte_lib.cpp:177-188)
  double tc_scale = 0;                         // power of two S: |template component| * S fits 24 bits for every offset
  // scratch of the drop-in host calls
  lcs::DevBuf<double> d_capbuf;                // c128 capture buffer (2 doubles / sample)
  lcs::DevBuf<float> d_ref, d_inc;
  lcs::DevBuf<unsigned char> d_cu8;
  lcs::DevBuf<int> d_flag8;                    // 8-bit exactness probe of lcs_xcorr_pss
  lcs::ChainScratch chain;                     // one thread per context (lcs_b200.h)
};

struct lcs_xcorr_plan {
  lcs_ctx* ctx = nullptr;
  lcs::PlanSet ps;
  uint32_t max_batch = 1;
  int kernel = LCS_KERNEL_AUTO;
  bool timing = false;                         // time the correlator kernel of every launch on `clock`
  lcs::KernelClock clock;
  // per-stream device buffers of the host-input entry points (lcs_xcorr_pss uses stream 0's)
  struct HostBatchBufs {
    lcs::DevBuf<unsigned char> iq;
    lcs::DevBuf<float> single;
    lcs::DevBuf<double> pow, spi;
    lcs::DevBuf<int32_t> frq;
    // device peak search (search_batch.cu)
    lcs::DevBuf<double> work;
    lcs::DevBuf<unsigned char> peaks;
    lcs::DevBuf<int32_t> npeaks;
    lcs::PinBuf<unsigned char> h_peaks;   // page-locked landing zones of the peak lists
    lcs::PinBuf<int32_t> h_npeaks;
    // Room for `chunk` capture buffers of geometry g: the correlator's outputs, the IQ bytes copied from the host
    // (host_iq) and the device peak search's buffers (with_peaks).  Defined in search_batch.cu.
    cudaError_t ensure(const lcs::XcorrGeom& g, uint32_t chunk, size_t samp_bytes, bool host_iq, bool with_peaks);
  } hb[lcs_ctx::N_STREAMS];
};

namespace lcs {

// Capture buffers per chunk of the host-batch calls: large enough that the persistent correlator CTAs get many tiles
// each (64 buffers x 38 tiles = 16.4 tiles per CTA, 3 % rounding loss), small enough that the copies of neighbouring
// chunks overlap the kernels.
constexpr uint32_t BATCH_CHUNK = 64;

// The chunk pipeline of the host-batch calls: issue(b0, s) enqueues chunk k, which starts at buffer b0, on stream
// s = k % N_STREAMS; after issuing chunk k the host calls finish(b0, s) of chunk k - (N_STREAMS - 1).  So N_STREAMS - 1
// chunks are in flight while the oldest one is finished, and the copies of the neighbouring chunks overlap the kernels of
// a chunk (with two streams the upload of chunk i+2 would sit behind the download of chunk i).
template <class Issue, class Finish>
lcs_status rotate_chunks(uint32_t batch, uint32_t chunk, Issue&& issue, Finish&& finish) {
  constexpr uint32_t NS = lcs_ctx::N_STREAMS;
  const uint32_t n_chunks = (batch + chunk - 1) / chunk;
  for (uint32_t k = 0; k < n_chunks + (NS - 1); k++) {
    if (k < n_chunks) {
      lcs_status rc = issue(k * chunk, (int)(k % NS));
      if (rc != LCS_OK) return rc;
    }
    if (k >= NS - 1) {
      const uint32_t kf = k - (NS - 1);
      lcs_status rc = finish(kf * chunk, (int)(kf % NS));
      if (rc != LCS_OK) return rc;
    }
  }
  return LCS_OK;
}

lcs_status fail(lcs_ctx* ctx, lcs_status st, const std::string& msg);
#define LCS_CUDA(ctx, expr)                                                                         \
  do {                                                                                              \
    cudaError_t _e = (expr);                                                                        \
    if (_e != cudaSuccess)                                                                          \
      return ::lcs::fail((ctx), LCS_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e)); \
  } while (0)

// ---- planset.cu ----
// (Re)build the set for `cfgs` (all with the same n_cap / arm).  Asynchronous on `st` apart from the host-side geometry.
// want_fp32: also build the FP32 correlator's templates (skipped for 8-bit-only sweeps).
lcs_status planset_build(lcs_ctx* ctx, PlanSet& ps, uint32_t n_cap, uint8_t arm, const std::vector<PlanCfg>& cfgs,
                         bool want_fp32, cudaStream_t st);
// Wait for the builds queued on `st` (the plans are used from every stream afterwards) and read the builder's
// diagnostics: a digit plane out of range takes the set off the tensor-core correlator.
lcs_status planset_finish(lcs_ctx* ctx, PlanSet& ps, cudaStream_t st);
// Which kernel AUTO resolves to for this set and input format.
int planset_resolve_kernel(const PlanSet& ps, int kernel, int iq_format);
// xcorr_pss for `batch` device-resident capture buffers: correlator + sp_est + delay spread / argmax.  d_buf_plan
// (device, [batch]) names the plan of every buffer (NULL: plan 0).
// ev: optional event pair recorded around the correlator kernel.
lcs_status planset_run(PlanSet& ps, int kernel, const void* d_iq, int iq_format, uint32_t batch, const uint32_t* d_buf_plan,
                       float* d_single, double* d_pow, int32_t* d_frq, double* d_spi, float* d_inc, cudaStream_t st,
                       const std::pair<cudaEvent_t, cudaEvent_t>* ev = nullptr);

lcs_status get_cached_plan(lcs_ctx* ctx, uint32_t n_cap, const double* f_search_set, uint32_t n_f, uint8_t arm,
                           double fc_req, double fc_prog, double fs_prog, lcs_xcorr_plan** out);
// The c128 capture buffer of a drop-in call into ctx->d_capbuf, on the context's device, asynchronously on st.
lcs_status upload_c128(lcs_ctx* ctx, const double* capbuf, uint32_t n_cap, cudaStream_t st);
// ---- xcorr_tc.cu ----
lcs_status tc_init(lcs_ctx* ctx);           // one-time function attributes
int launch_xcorr_fold_tc(PlanSet& ps, const void* d_iq_cu8, uint32_t batch, const uint32_t* d_buf_plan,
                         float* d_single_planar, cudaStream_t st);

}  // namespace lcs
