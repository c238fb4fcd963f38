// TMA / mbarrier PTX wrappers and operand-conversion helpers shared by the sm_90a contraction kernels
// (contract_tc.cu, conv_tma.cu, gemm_tma.cu); the wgmma wrappers are in wgmma.cuh.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <stdint.h>

namespace mas {
namespace tc {

constexpr int BM = 128;        // pixels per M tile (16 x 8)
constexpr int BN = 128;        // output channels per CTA

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(bar), "r"(parity)
        : "memory");
  } while (!done);
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src),
               "r"(bytes), "r"(bar)
               : "memory");
}
// TMA tiled tensor copies (UTMALDG): one instruction lands a whole box of the tensor in shared memory
__device__ __forceinline__ void tma_load_3d(uint32_t dst, const CUtensorMap* map, int c0, int c1, int c2, uint32_t bar) {
  asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];"
               ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(c2), "r"(bar)
               : "memory");
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap* map, int c0, int c1, int c2, int c3, uint32_t bar) {
  asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];"
               ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(bar)
               : "memory");
}
__device__ __forceinline__ void tma_load_5d(uint32_t dst, const CUtensorMap* map, int c0, int c1, int c2, int c3, int c4, uint32_t bar) {
  asm volatile("cp.async.bulk.tensor.5d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5, %6}], [%7];"
               ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4), "r"(bar)
               : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, int c0, int c1, uint32_t bar) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];"
               ::"r"(dst), "l"(reinterpret_cast<uint64_t>(map)), "r"(c0), "r"(c1), "r"(bar)
               : "memory");
}
// four 8 x 8 fp16 matrices, transposed on the way: lanes 8 i .. 8 i + 7 address the eight 16-byte rows of matrix i, and
// r[i] receives the wgmma / mma A-fragment register of that matrix
__device__ __forceinline__ void ldsm_x4_trans(uint32_t addr, uint32_t* r) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(addr)
               : "memory");
}
// two floats -> packed half2 (lo = a, hi = b), round-to-nearest-even, saturating to +-65504 instead of inf
__device__ __forceinline__ uint32_t pack_h2(float a, float b) {
  uint32_t r;
  asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(r) : "f"(b), "f"(a));
  return r;
}
// power-of-two operand scale for an fp16 operand tensor from its largest magnitude (device scalar; null = 1):
// amax * s lands in [2^14, 2^15), so the whole fp16 normal range (30 binades) sits below the largest element and
// nothing overflows. *inv receives 1/s (exact). Zero / non-finite amax -> s = 1.
// TOP: the binade [2^TOP, 2^(TOP+1)) amax * s lands in: 14 for fp16 and FP8 e5m2 (max 57344), 7 for FP8 e4m3 (max 448).
template <int TOP = 14>
__device__ __forceinline__ float operand_scale(const float* amax, float* inv) {
  float s = 1.f, i = 1.f;
  if (amax) {
    const uint32_t b = __float_as_uint(*amax);
    const int e = (int)((b >> 23) & 0xff);            // biased exponent of amax (0 = zero/denormal, 255 = inf/nan)
    if (e > 0 && e < 255) {
      int se = 127 + TOP - (e - 127);                 // biased exponent of s = 2^(TOP - floor(log2 amax))
      se = se < 1 ? 1 : (se > 254 ? 254 : se);
      s = __uint_as_float((uint32_t)se << 23);
      i = __uint_as_float((uint32_t)(254 - se) << 23);
    }
  }
  *inv = i;
  return s;
}

// read-only 16-byte load that also pulls the surrounding 256 bytes into L2: the K loop walks a pixel's channel vector in
// 32/64-byte steps, so the next chunks of the same pixel hit L2 instead of paying the DRAM latency again
__device__ __forceinline__ float4 ldg_l2pf(const float4* p) {
  float4 v;
  asm volatile("ld.global.nc.L2::256B.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p));
  return v;
}

__device__ __forceinline__ unsigned short to_h(float a) {
  unsigned short r;
  asm("cvt.rn.satfinite.f16.f32 %0, %1;" : "=h"(r) : "f"(a));
  return r;
}
}  // namespace tc
}  // namespace mas
