// Small CUDA helpers for the PDLP solver: error checking, RAII device buffers,
// deterministic block reductions and cache-hinted loads.  sm_90a (Hopper).
#pragma once

#include "lp_problem.hpp"

#include <cuda_runtime.h>

#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <mutex>
#include <string>
#include <vector>

namespace cuopt_b200 {

#define CUOPT_CUDA_TRY(call)                                                                              \
  do {                                                                                                    \
    cudaError_t err__ = (call);                                                                           \
    if (err__ != cudaSuccess) {                                                                           \
      cudaGetLastError();                                                                                 \
      throw ::cuopt_b200::lp_error(                                                                       \
        err__ == cudaErrorMemoryAllocation ? ::cuopt_b200::error_type_t::OutOfMemory                      \
                                           : ::cuopt_b200::error_type_t::RuntimeError,                    \
        std::string("CUDA error: ") + cudaGetErrorString(err__) + " at " + __FILE__ + ":" +               \
          std::to_string(__LINE__));                                                                      \
    }                                                                                                     \
  } while (0)

// CUOPT_B200_TRACE=1: time spent inside cudaMalloc / cudaFree (reported by the solver when it is destroyed)
struct alloc_stats_t {
  bool on = false;
  double malloc_s = 0.0, free_s = 0.0;
  long n_malloc = 0, n_free = 0;
  size_t bytes = 0;
};
inline alloc_stats_t& alloc_stats()
{
  static alloc_stats_t s;
  return s;
}
inline double alloc_clock()
{
  return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

// Freed device blocks are kept (per device, up to a cap) and handed out again to a request of exactly the same size: a solve
// allocates ~100 arrays, and at configs[3] their cudaFree calls alone took 0.5-0.7 s of a 3.5 s end-to-end solve (7 ms each for
// multi-hundred-MB blocks, CUOPT_B200_TRACE=1) — the reference sits on RMM's pool for the same reason.  A block enters the cache
// only after a cudaDeviceSynchronize (the guarantee cudaFree gave: nothing still uses it); over the cap the oldest blocks go back
// to the driver; an out-of-memory cudaMalloc flushes the cache and retries.  CUOPT_B200_DEVICE_CACHE_MB=0 turns it off.
class device_block_cache_t {
 public:
  static device_block_cache_t& get()
  {
    static device_block_cache_t* c = new device_block_cache_t;  // never destroyed: the CUDA context may be gone at exit
    return *c;
  }
  void* take(size_t bytes)
  {
    if (cap_ == 0) return nullptr;
    int dev = 0;
    cudaGetDevice(&dev);
    std::lock_guard<std::mutex> g(mu_);
    for (size_t i = blocks_.size(); i-- > 0;)
      if (blocks_[i].bytes == bytes && blocks_[i].dev == dev) {
        void* p = blocks_[i].p;
        cached_ -= bytes;
        blocks_.erase(blocks_.begin() + (long)i);
        ++hits_;
        return p;
      }
    return nullptr;
  }
  void give(void* p, size_t bytes)
  {
    if (cap_ == 0 || bytes > cap_) {
      cudaFree(p);
      return;
    }
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceSynchronize();
    std::lock_guard<std::mutex> g(mu_);
    blocks_.push_back({p, bytes, dev});
    cached_ += bytes;
    size_t first_kept = 0;
    while (cached_ > cap_ && first_kept < blocks_.size()) {  // oldest first; only blocks of the current device can be freed here
      if (blocks_[first_kept].dev == dev) {
        cudaFree(blocks_[first_kept].p);
        cached_ -= blocks_[first_kept].bytes;
        blocks_.erase(blocks_.begin() + (long)first_kept);
      } else {
        ++first_kept;
      }
    }
  }
  // requests served from the cache so far, all devices (read-only diagnostics)
  long long hits()
  {
    std::lock_guard<std::mutex> g(mu_);
    return hits_;
  }
  void flush()
  {
    int dev = 0;
    cudaGetDevice(&dev);
    std::lock_guard<std::mutex> g(mu_);
    for (size_t i = blocks_.size(); i-- > 0;)
      if (blocks_[i].dev == dev) {
        cudaFree(blocks_[i].p);
        cached_ -= blocks_[i].bytes;
        blocks_.erase(blocks_.begin() + (long)i);
      }
  }

 private:
  struct block_t {
    void* p;
    size_t bytes;
    int dev;
  };
  device_block_cache_t()
  {
    cap_ = size_t(16) << 30;  // a fifth of an 80 GB H100: several configs[3] solves' arrays, room left for the caller
    if (const char* e = std::getenv("CUOPT_B200_DEVICE_CACHE_MB")) cap_ = (size_t)std::strtoull(e, nullptr, 10) << 20;
  }
  std::mutex mu_;
  std::vector<block_t> blocks_;
  size_t cached_ = 0, cap_ = 0;
  long long hits_ = 0;
};

// Device array with value semantics disabled; one allocation per vector, sized once per solve, taken from / returned to the
// block cache above.
template <typename T>
class dvec {
 public:
  dvec() = default;
  explicit dvec(size_t n) { resize(n); }
  dvec(const dvec&)            = delete;
  dvec& operator=(const dvec&) = delete;
  dvec(dvec&& o) noexcept : p_(o.p_), n_(o.n_), slack_(o.slack_) { o.p_ = nullptr; o.n_ = 0; }
  dvec& operator=(dvec&& o) noexcept
  {
    if (this != &o) { release(); p_ = o.p_; n_ = o.n_; slack_ = o.slack_; o.p_ = nullptr; o.n_ = 0; }
    return *this;
  }
  ~dvec() { release(); }
  // `slack` extra elements are allocated (zero-filled) past the logical size: the 16-byte granular bulk
  // copies of the SpMV pipeline may read a few elements beyond the end of idx / val / off.
  void resize(size_t n, size_t slack = 0)
  {
    release();
    n_     = n;
    slack_ = slack;
    if (n + slack) {
      alloc_stats_t& as = alloc_stats();
      const double t0   = as.on ? alloc_clock() : 0.0;
      const size_t bytes = (n + slack) * sizeof(T);
      void* raw          = device_block_cache_t::get().take(bytes);
      if (raw == nullptr) {
        cudaError_t err = cudaMalloc(&raw, bytes);
        if (err == cudaErrorMemoryAllocation) {  // give the cached blocks back and try once more
          cudaGetLastError();
          device_block_cache_t::get().flush();
          err = cudaMalloc(&raw, bytes);
        }
        CUOPT_CUDA_TRY(err);
      }
      p_ = static_cast<T*>(raw);
      if (as.on) {
        as.malloc_s += alloc_clock() - t0;
        as.n_malloc += 1;
        as.bytes += (n + slack) * sizeof(T);
      }
      if (slack) CUOPT_CUDA_TRY(cudaMemset(p_ + n, 0, slack * sizeof(T)));
    }
  }
  void release()
  {
    if (p_) {
      alloc_stats_t& as = alloc_stats();
      const double t0   = as.on ? alloc_clock() : 0.0;
      device_block_cache_t::get().give(p_, (n_ + slack_) * sizeof(T));
      if (as.on) {
        as.free_s += alloc_clock() - t0;
        as.n_free += 1;
      }
    }
    p_ = nullptr;
    n_ = 0;
  }
  void upload(const T* h, size_t n, cudaStream_t s, size_t slack = 0)
  {
    if (n_ != n || slack_ != slack) resize(n, slack);
    if (n) CUOPT_CUDA_TRY(cudaMemcpyAsync(p_, h, n * sizeof(T), cudaMemcpyHostToDevice, s));
  }
  void upload(const std::vector<T>& h, cudaStream_t s, size_t slack = 0) { upload(h.data(), h.size(), s, slack); }
  void download(T* h, cudaStream_t s) const
  {
    if (n_) CUOPT_CUDA_TRY(cudaMemcpyAsync(h, p_, n_ * sizeof(T), cudaMemcpyDeviceToHost, s));
  }
  void zero(cudaStream_t s)
  {
    if (n_) CUOPT_CUDA_TRY(cudaMemsetAsync(p_, 0, n_ * sizeof(T), s));
  }
  void copy_from(const dvec& o, cudaStream_t s)
  {
    if (n_ != o.n_) resize(o.n_, o.slack_);  // same logical size: keep this buffer (it may be padded or peer-mapped)
    if (n_) CUOPT_CUDA_TRY(cudaMemcpyAsync(p_, o.p_, n_ * sizeof(T), cudaMemcpyDeviceToDevice, s));
  }
  T* data() { return p_; }
  const T* data() const { return p_; }
  size_t size() const { return n_; }

 private:
  T* p_         = nullptr;
  size_t n_     = 0;
  size_t slack_ = 0;
};

// ---- device-side helpers ---------------------------------------------------------------------
__device__ __forceinline__ double warp_sum(double v)
{
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
    v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_max(double v)
{
#pragma unroll
  for (int o = 16; o > 0; o >>= 1)
    v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Fixed-shape tree: xor-shuffle inside each warp, then the first warp folds the per-warp values.
// The result is identical run to run for a given blockDim.  `scratch` holds >= 32 doubles.
// All threads receive the result.
template <bool IsMax = false>
__device__ __forceinline__ double block_reduce(double v, double* scratch)
{
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
  v = IsMax ? warp_max(v) : warp_sum(v);
  __syncthreads();  // protect scratch from a previous use
  if (lane == 0) scratch[wid] = v;
  __syncthreads();
  double r = (lane < nw) ? scratch[lane] : 0.0;
  r        = IsMax ? warp_max(r) : warp_sum(r);
  return r;
}

// L2 residency hints (createpolicy + ld/st ...L2::cache_hint).  At configs[3] sizes the vector an SpMV gathers from is
// 80 MB: a large share of it only stays in L2 if the ~2 GB of read-once streams passing by are marked evict-first and
// the vector itself evict-last.  `keep` marks the gathered vector (its producer's stores and the gathers), `stream`
// everything that is touched once per kernel.  Mode 0 (CUOPT_B200_L2_HINTS=0) makes both policies evict-normal.
struct l2_policy_t {
  unsigned long long keep, stream;
};
__device__ __forceinline__ l2_policy_t make_l2_policies(int mode)
{
  l2_policy_t p;
  if (mode) {
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p.keep));
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p.stream));
  } else {
    asm volatile("createpolicy.fractional.L2::evict_normal.b64 %0, 1.0;" : "=l"(p.keep));
    p.stream = p.keep;
  }
  return p;
}
__device__ __forceinline__ double ld_l2(const double* p, unsigned long long policy)
{
  double v;
  asm volatile("ld.global.L1::no_allocate.L2::cache_hint.f64 %0, [%1], %2;" : "=d"(v) : "l"(p), "l"(policy));
  return v;
}
__device__ __forceinline__ void st_l2(double* p, double v, unsigned long long policy)
{
  asm volatile("st.global.L2::cache_hint.f64 [%0], %1, %2;" ::"l"(p), "d"(v), "l"(policy) : "memory");
}

// Streaming (read-once) loads: keep them from displacing the gathered vector in L1/L2.
__device__ __forceinline__ int ld_stream(const int* p) { return __ldcs(p); }
__device__ __forceinline__ double ld_stream(const double* p) { return __ldcs(p); }

}  // namespace cuopt_b200
