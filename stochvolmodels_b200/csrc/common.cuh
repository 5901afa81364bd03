// common.cuh -- error plumbing, launch geometry and block reductions shared by the b200sv kernels.
// sm_90a only (H100 SXM: 132 SMs, 64 fp64 + 128 fp32 lanes / SM / clk, 227 KB smem / CTA, 50 MB L2).
#pragma once
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstring>
#include <string>

namespace b200sv {

// thread-local last error string returned by b200sv_last_error()
inline std::string& last_error() {
  static thread_local std::string s;
  return s;
}
inline int fail(int code, const std::string& msg) {
  last_error() = msg;
  return code;
}

// The stream every HOST-LEVEL entry point of the calling thread works on: b200sv_set_stream (include/b200sv.h).  Defined once in
// mc_kernels.cu; the other translation units reach it through these accessors (one shared library, one thread-local).
cudaStream_t& current_stream_ref();
inline cudaStream_t current_stream() { return current_stream_ref(); }
// Kernel launches of the calling thread since b200sv_reset_launch_count (b200sv_launch_count); defined once in mc_kernels.cu like the stream.
long long& launch_count_ref();

#define B200SV_CUDA(call)                                                                           \
  do {                                                                                              \
    cudaError_t e__ = (call);                                                                       \
    if (e__ != cudaSuccess)                                                                         \
      return ::b200sv::fail(-2, std::string(#call) + ": " + cudaGetErrorString(e__));               \
  } while (0)

#define B200SV_REQUIRE(cond, msg)                                                                   \
  do {                                                                                              \
    if (!(cond)) return ::b200sv::fail(-1, std::string("invalid argument: ") + (msg));              \
  } while (0)

// after every kernel launch: a launch error is reported under `what`, a successful launch is counted.  Launch APIs that return their
// error (cudaLaunchCooperativeKernel) pass it as `e`.
inline int check_launch(const char* what, cudaError_t e = cudaGetLastError()) {
  if (e != cudaSuccess) return fail(-2, std::string(what) + ": " + cudaGetErrorString(e));
  ++launch_count_ref();
  return 0;
}

struct DevBuf {   // RAII for stream-ordered temporaries
  void* p = nullptr;
  cudaStream_t st;
  explicit DevBuf(cudaStream_t s) : st(s) {}
  DevBuf(const DevBuf&) = delete;
  DevBuf& operator=(const DevBuf&) = delete;
  cudaError_t alloc(size_t n) { return cudaMallocAsync(&p, n ? n : 1, st); }
  // allocate n elements of T and queue the copy of host[0, n) into them
  template <typename T>
  cudaError_t upload(const T* host, size_t n) {
    const cudaError_t e = alloc(sizeof(T) * n);
    return e != cudaSuccess ? e : cudaMemcpyAsync(p, host, sizeof(T) * n, cudaMemcpyHostToDevice, st);
  }
  // queue the copy of the first n elements of T back into host; nothing to do for an optional output left null
  template <typename T>
  cudaError_t download(T* host, size_t n) const {
    return host ? cudaMemcpyAsync(host, p, sizeof(T) * n, cudaMemcpyDeviceToHost, st) : cudaSuccess;
  }
  ~DevBuf() {
    if (p) cudaFreeAsync(p, st);
  }
  template <typename T>
  T* as() const {
    return (T*)p;
  }
};

// Every host-level call declares one before its first stream operation and ends with `return sync.done();`, which waits for the
// stream and reports a failed wait (a kernel fault surfaces here).  An early error return waits in the destructor instead, so no
// copy or kernel the call queued still reads or writes the caller's host buffers after it returns.
class StreamSync {
 public:
  explicit StreamSync(cudaStream_t s) : st_(s) {}
  StreamSync(const StreamSync&) = delete;
  StreamSync& operator=(const StreamSync&) = delete;
  ~StreamSync() {
    if (!waited_) cudaStreamSynchronize(st_);
  }
  int done() {
    waited_ = true;
    B200SV_CUDA(cudaStreamSynchronize(st_));
    return 0;
  }

 private:
  cudaStream_t st_;
  bool waited_ = false;
};

inline int device_sm_count() {
  int dev = 0, sms = 132;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  return sms;
}

// persistent-grid geometry: one wave of resident CTAs (multiple of the SM count), capped by the work
struct Grid {
  int blocks;
  int threads;
};
template <typename K>
inline Grid persistent_grid(K kernel, int threads, long long work_items, int items_per_thread = 1) {
  const int sms = device_sm_count();
  int per_sm = 1;
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kernel, threads, 0);
  if (per_sm < 1) per_sm = 1;
  long long need = (work_items + (long long)threads * items_per_thread - 1) / ((long long)threads * items_per_thread);
  long long full = (long long)sms * per_sm;
  Grid g;
  g.threads = threads;
  g.blocks = (int)(need < full ? (need < 1 ? 1 : need) : full);
  return g;
}

// ---- warp / block reductions in fp64 (fixed order => run-to-run deterministic) -------------------
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
  return v;
}

// reduce NV values per thread across the block; result valid in thread 0 (returned in v[])
template <int NV, int THREADS>
__device__ __forceinline__ void block_sum(double (&v)[NV], double* smem /* NV * THREADS/32 doubles */) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  constexpr int NW = THREADS / 32;
#pragma unroll
  for (int k = 0; k < NV; ++k) {
    double s = warp_sum(v[k]);
    if (lane == 0) smem[k * NW + warp] = s;
  }
  __syncthreads();
  if (warp == 0) {
#pragma unroll
    for (int k = 0; k < NV; ++k) {
      double s = lane < NW ? smem[k * NW + lane] : 0.0;
      s = warp_sum(s);
      v[k] = s;
    }
  }
  __syncthreads();
}

// cudaMallocAsync returns freed blocks to the OS at the next synchronisation unless the pool's release threshold is raised;
// the chain entry points allocate GBs of path state per call, so keep it cached (set once per device).
inline void ensure_pool_threshold() {
  static thread_local int done_for = -1;
  int dev = 0;
  if (cudaGetDevice(&dev) != cudaSuccess || dev == done_for) return;
  cudaMemPool_t pool;
  if (cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) {
    unsigned long long thr = ~0ull;
    cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &thr);
  }
  done_for = dev;
}


}  // namespace b200sv
