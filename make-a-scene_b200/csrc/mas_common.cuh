// Shared helpers for libmas_b200.so (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <atomic>

#include "mas_b200.h"

namespace mas {

// streaming multiprocessors of the H100 SXM: grid-size heuristics (the persistent kernels query the device instead)
constexpr int NUM_SMS = 132;

extern thread_local char g_err[512];
extern std::atomic<int64_t> g_launches;
extern std::atomic<int64_t> g_tc_launches;

int fail(int code, const char* fmt, ...);
// Checks the launch that was just enqueued (no synchronisation) and counts it.
int launched(const char* what);
// Same, for a kernel that issues tensor-core (wgmma) MMAs (counted separately: mas_tc_launch_count).
int launched_tc(const char* what);

// cudaFuncSetAttribute is per device: true the first time a call site runs on the CURRENT device (bit d of `mask`).
static inline bool first_on_device(std::atomic<uint64_t>& mask) {
  int d = 0;
  cudaGetDevice(&d);
  const uint64_t bit = 1ull << (d & 63);
  return !(mask.load(std::memory_order_relaxed) & bit);
}
static inline void mark_device(std::atomic<uint64_t>& mask) {
  int d = 0;
  cudaGetDevice(&d);
  mask.fetch_or(1ull << (d & 63), std::memory_order_relaxed);
}

static inline cudaStream_t S(void* s) { return reinterpret_cast<cudaStream_t>(s); }
static inline int64_t cdiv(int64_t a, int64_t b) { return (a + b - 1) / b; }

__device__ __forceinline__ float silu_f(float u) { return __fdividef(u, 1.0f + __expf(-u)); }
// d/du [u*sigmoid(u)] = s*(1+u*(1-s))
__device__ __forceinline__ float silu_grad_f(float u) {
  float s = __fdividef(1.0f, 1.0f + __expf(-u));
  return s * (1.0f + u * (1.0f - s));
}
__device__ __forceinline__ float round_tf32(float x) {
  uint32_t r;
  asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
  return __uint_as_float(r);
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

}  // namespace mas

#define MAS_REQUIRE(cond, ...)                                   \
  do {                                                           \
    if (!(cond)) return mas::fail(MAS_ERR_INVALID_ARG, __VA_ARGS__); \
  } while (0)
