// Shared host/device helpers for libdirb200 (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_bf16.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <atomic>
#include <vector>
#include "../../include/dirb200.h"

namespace dirb200 {

void set_error(const char* fmt, ...);
extern std::atomic<int64_t> g_launches;

inline cudaStream_t as_stream(void* s) { return reinterpret_cast<cudaStream_t>(s); }

#define DIRB_CHECK_ARG(cond, ...)                \
  do {                                           \
    if (!(cond)) {                               \
      ::dirb200::set_error(__VA_ARGS__);         \
      return DIRB200_ERR_ARG;                    \
    }                                            \
  } while (0)

#define DIRB_CUDA(expr)                                                                  \
  do {                                                                                   \
    cudaError_t _e = (expr);                                                             \
    if (_e != cudaSuccess) {                                                             \
      ::dirb200::set_error("%s:%d %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
      return DIRB200_ERR_CUDA;                                                           \
    }                                                                                    \
  } while (0)

// call after every <<<>>> launch
#define DIRB_LAUNCHED()                           \
  do {                                            \
    ::dirb200::g_launches.fetch_add(1);           \
    DIRB_CUDA(cudaGetLastError());                \
  } while (0)

// SMs the persistent kernels size their grids for.  DIRB200_SMS=<n> caps it (experiments: leaving SMs to a concurrent
// NCCL kernel -- a persistent grid with a static tile walk takes twice as long when even one of its CTAs has to wait
// for an SM).
inline int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    if (cudaGetDevice(&dev) != cudaSuccess) return 132;
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 132;
    if (const char* e = getenv("DIRB200_SMS")) {
      const int cap = atoi(e);
      if (cap > 0 && cap < n) n = cap;
    }
  }
  return n;
}

// An A/B switch such as DIRB200_GRAPH: on unless its value starts with '0'.  Each caller keeps the result in a
// function-local static of its own, so every switch is read once per process.
inline bool env_switch(const char* name) {
  const char* e = getenv(name);
  return !(e != nullptr && e[0] == '0');
}

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// Division by a run-time constant as multiply-high + shift (n < 2^31, d >= 1): a 32-bit `/` by a run-time divisor
// (cpb, kw, hw, wm) compiles to a ~35-instruction SASS sequence, which would dominate the k-loops of the producer warps.
struct FastDiv {
  uint32_t mul, shr, d;
  __device__ __forceinline__ uint32_t div(uint32_t n) const { return d == 1 ? n : (__umulhi(n, mul) >> shr); }
  __device__ __forceinline__ void divmod(uint32_t n, uint32_t& q, uint32_t& r) const {
    q = div(n);
    r = n - q * d;
  }
};
inline FastDiv make_fastdiv(uint32_t d) {
  FastDiv f{0u, 0u, d < 1 ? 1u : d};
  if (f.d == 1) return f;
  uint32_t lg = 0;
  while ((1ull << lg) < f.d) ++lg;
  const uint32_t p = 31 + lg;
  f.mul = static_cast<uint32_t>(((1ull << p) + f.d - 1) / f.d);
  f.shr = p - 32;
  return f;
}

// Test aids over a HOST array of jobs: the descriptors go to a device table that lives in stream order around the
// launch (allocated, copied, launched and freed on st); launch(table) returns the launch's rc.
template <typename Desc, typename Launch>
static int with_device_table(const std::vector<Desc>& descs, cudaStream_t st, Launch&& launch) {
  Desc* dev = nullptr;
  const size_t bytes = sizeof(Desc) * descs.size();
  DIRB_CUDA(cudaMallocAsync(reinterpret_cast<void**>(&dev), bytes, st));
  cudaError_t e = cudaMemcpyAsync(dev, descs.data(), bytes, cudaMemcpyHostToDevice, st);
  int rc = DIRB200_OK;
  if (e != cudaSuccess) {
    set_error("cudaMemcpyAsync of a descriptor table -> %s", cudaGetErrorString(e));
    rc = DIRB200_ERR_CUDA;
  } else {
    rc = launch(dev);
  }
  DIRB_CUDA(cudaFreeAsync(dev, st));
  return rc;
}

// streaming 128-bit global load that does not allocate in L1
__device__ __forceinline__ float4 ldg_stream(const float4* p) {
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
               : "l"(p));
  return r;
}

}  // namespace dirb200
