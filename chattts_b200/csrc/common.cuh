// Shared device/host helpers for the chattts_b200 kernels (sm_90a only).
#pragma once
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <atomic>
#include <map>
#include <mutex>
#include <utility>

#include "../../include/chattts_b200.h"

namespace ctb {

extern thread_local char g_err[512];
extern std::atomic<uint64_t> g_launches;

int set_err(int code, const char* fmt, ...);

#define CTB_CUDA(expr)                                                                      \
  do {                                                                                      \
    cudaError_t _e = (expr);                                                                \
    if (_e != cudaSuccess)                                                                  \
      return ::ctb::set_err(CTB_ERR_CUDA, "%s:%d %s -> %s", __FILE__, __LINE__, #expr,      \
                            cudaGetErrorString(_e));                                        \
  } while (0)

#define CTB_LAUNCH_CHECK()                                                                  \
  do {                                                                                      \
    ::ctb::g_launches.fetch_add(1, std::memory_order_relaxed);                              \
    cudaError_t _e = cudaPeekAtLastError();                                                 \
    if (_e != cudaSuccess)                                                                  \
      return ::ctb::set_err(CTB_ERR_CUDA, "%s:%d launch -> %s", __FILE__, __LINE__,         \
                            cudaGetErrorString(_e));                                        \
  } while (0)

// cudaFuncSetAttribute is per device: remember (function, device) -> largest dynamic shared memory size set so far.
inline int ensure_smem_attr(const void* fn, int bytes) {
  static std::mutex mu;
  static std::map<std::pair<const void*, int>, int> done;
  int dev = 0;
  CTB_CUDA(cudaGetDevice(&dev));
  std::lock_guard<std::mutex> lk(mu);
  int& cur = done[std::make_pair(fn, dev)];
  if (cur >= bytes && cur > 0) return CTB_OK;
  CTB_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  cur = bytes;
  return CTB_OK;
}

constexpr int kPageTokens = 16;

// Programmatic dependent launch (PDL): every kernel of the decode step is launched with
// cudaLaunchAttributeProgrammaticStreamSerialization.  A kernel calls pdl_trigger() first (lets the
// next kernel's CTAs become resident and prefetch their weights) and pdl_wait() before it touches
// anything a previous kernel wrote (griddepcontrol.wait = predecessors complete + memory visible).
__device__ __forceinline__ void pdl_trigger() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }

template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl_cluster(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s,
                                      unsigned cluster_x, Args&&... args) {
  static const int cluster_pdl = getenv("CTB_CLUSTER_PDL") ? atoi(getenv("CTB_CLUSTER_PDL")) : 1;
  cudaLaunchConfig_t cfg{};
  cfg.gridDim = grid; cfg.blockDim = block; cfg.dynamicSmemBytes = smem; cfg.stream = s;
  cudaLaunchAttribute attr[2];
  static const int pdl_on = getenv("CTB_NO_PDL") == nullptr;
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = (cluster_x > 1 && !cluster_pdl) ? 0 : pdl_on;
  cfg.numAttrs = 1;
  if (cluster_x > 1) {
    attr[1].id = cudaLaunchAttributeClusterDimension;
    attr[1].val.clusterDim.x = cluster_x; attr[1].val.clusterDim.y = 1; attr[1].val.clusterDim.z = 1;
    cfg.numAttrs = 2;
  }
  cfg.attrs = attr;
  return cudaLaunchKernelEx(&cfg, kernel, std::forward<Args>(args)...);
}
template <typename... KArgs, typename... Args>
inline cudaError_t launch_pdl(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t s,
                              Args&&... args) {
  return launch_pdl_cluster(kernel, grid, block, smem, s, 1u, std::forward<Args>(args)...);
}  // KV page = 16 tokens (the reference's vLLM fork: velocity/configs.py:567)

// ---------------------------------------------------------------- device helpers
__device__ __forceinline__ float4 ldg_stream(const float4* p) {
  // weights / KV are read exactly once per step: bypass L1, keep L2 for activations
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
               : "l"(p));
  return r;
}

// Activations / loop state / KV written by earlier kernels: L2-coherent loads only.  With PDL a CTA
// can be resident while its predecessors still run, so nothing mutable may be served from L1.
__device__ __forceinline__ float4 ldg_cg(const float4* p) { return __ldcg(p); }
__device__ __forceinline__ float ldg_cg(const float* p) { return __ldcg(p); }
__device__ __forceinline__ int ldg_cg(const int* p) { return __ldcg(p); }
__device__ __forceinline__ int ldg_cg(const uint8_t* p) { return (int)__ldcg(p); }

// 8 consecutive K or V values as fp32: two 16-byte loads from an fp32 cache, one from an fp16 cache
__device__ __forceinline__ void ld_kv8(const float* p, float4& a, float4& b) {
  a = ldg_cg(reinterpret_cast<const float4*>(p));
  b = ldg_cg(reinterpret_cast<const float4*>(p + 4));
}
__device__ __forceinline__ void ld_kv8(const __half* p, float4& a, float4& b) {
  const uint4 u = __ldcg(reinterpret_cast<const uint4*>(p));
  const float2 f0 = __half22float2(*reinterpret_cast<const __half2*>(&u.x));
  const float2 f1 = __half22float2(*reinterpret_cast<const __half2*>(&u.y));
  const float2 f2 = __half22float2(*reinterpret_cast<const __half2*>(&u.z));
  const float2 f3 = __half22float2(*reinterpret_cast<const __half2*>(&u.w));
  a = make_float4(f0.x, f0.y, f1.x, f1.y);
  b = make_float4(f2.x, f2.y, f3.x, f3.y);
}
// a K/V pair appended to the cache (fp16: rounded to nearest even)
__device__ __forceinline__ void st_kv2(float* p, float a, float b) { *reinterpret_cast<float2*>(p) = make_float2(a, b); }
__device__ __forceinline__ void st_kv2(__half* p, float a, float b) { *reinterpret_cast<__half2*>(p) = __floats2half2_rn(a, b); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_sum_d(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Butterfly reduce-scatter: N per-lane partial values (N = power of two <= 32) are summed
// across the 32 lanes; afterwards v[0] of lane l holds the total of value (l >> (5 - log2 N)).
// 31 shuffles for N = 32 instead of 160 for 32 independent all-reduces.
template <int N>
__device__ __forceinline__ void warp_reduce_scatter(float (&v)[N]) {
  const int lane = threadIdx.x & 31;
  int off = 16;
#pragma unroll
  for (int n = N; n > 1; n >>= 1, off >>= 1) {
    const bool hi = (lane & off) != 0;
#pragma unroll
    for (int i = 0; i < n / 2; ++i) {
      float send = hi ? v[i] : v[i + n / 2];
      float keep = hi ? v[i + n / 2] : v[i];
      v[i] = keep + __shfl_xor_sync(0xffffffffu, send, off);
    }
  }
  for (; off > 0; off >>= 1) v[0] += __shfl_xor_sync(0xffffffffu, v[0], off);
}

// Philox4x32-10 (counter-based) Exp(1) noise for the unseeded path (manual_seed=None has no parity target)
__device__ __forceinline__ float philox_exp1(uint64_t seed, uint32_t c0, uint32_t c1, uint32_t c2) {
  uint32_t k0 = (uint32_t)seed, k1 = (uint32_t)(seed >> 32);
  uint32_t x0 = c0, x1 = c1, x2 = c2, x3 = 0x9E3779B9u;
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    const uint32_t h0 = __umulhi(0xD2511F53u, x0), l0 = 0xD2511F53u * x0;
    const uint32_t h1 = __umulhi(0xCD9E8D57u, x2), l1 = 0xCD9E8D57u * x2;
    x0 = h1 ^ x1 ^ k0; x1 = l1; x2 = h0 ^ x3 ^ k1; x3 = l0;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  const float u = ((x0 >> 8) + 1) * (1.0f / 16777216.0f);  // (0, 1]
  return -logf(u);
}

// order-preserving map float -> uint32 (larger float => larger key; -inf smallest).  -0.0 and +0.0 get one key, as
// they compare equal: a -0.0 logit is kept wherever a +0.0 one is (top-k cut, greedy max), like torch's `x < kth`.
__device__ __forceinline__ uint32_t float_key(float f) {
  uint32_t u = __float_as_uint(f);
  if (u == 0x80000000u) u = 0u;
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float key_float(uint32_t k) {
  uint32_t u = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
  return __uint_as_float(u);
}

}  // namespace ctb
