// Hopper (sm_90a) warpgroup MMA wrappers: wgmma.mma_async m64nNk8 (TF32) / m64nNk16 (fp16), fp32 accumulators in the
// registers of the issuing warpgroup.  Accumulator fragment of m64nN (thread t of the warpgroup, warp w = t / 32, lane l):
//   d[4 j + 2 i + c]  <->  row 16 w + 8 i + l / 4,  column 8 j + 2 (l % 4) + c      (j < N / 8, i, c in {0, 1})
// Shared-memory operand descriptors use the same canonical layouts (8 rows x 16 bytes core matrices; LBO = K-direction
// stride, SBO = 8-row-group stride; swizzle code in bits 62-63) as the producers stage them.
#pragma once
#include <stdint.h>

namespace mas {
namespace wg {

enum { SW_NONE = 0, SW_128 = 1 };

__device__ __forceinline__ uint64_t desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes, uint32_t swizzle = SW_NONE) {
  return (uint64_t)((saddr >> 4) & 0x3FFF) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16) |
         ((uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32) | ((uint64_t)swizzle << 62);
}
__device__ __forceinline__ void fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator reads / writes across an in-flight wgmma
template <int R>
__device__ __forceinline__ void fence_regs(float* d) {
#pragma unroll
  for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// warp-specialised register split (3 warpgroups: one copy-issuing warpgroup gives registers to two MMA warpgroups)
template <int R>
__device__ __forceinline__ void regs_inc() { asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(R)); }
template <int R>
__device__ __forceinline__ void regs_dec() { asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(R)); }
constexpr int MMA_REGS = 232, COPY_REGS = 40;   // 2 x 128 x 232 + 128 x 40 <= 64K registers
// named barrier over a subset of the block's warps (id 0 is __syncthreads)
__device__ __forceinline__ void bar_sync(int id, int nthreads) { asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory"); }

// accumulator operand lists in blocks of 16 registers (%0 .. %R-1 are the accumulators of an asm statement)
#define WG_R0 "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15"
#define WG_R16 "%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31"
#define WG_R32 "%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47"
#define WG_R48 "%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63"
#define WG_R64 "%64,%65,%66,%67,%68,%69,%70,%71,%72,%73,%74,%75,%76,%77,%78,%79"
#define WG_R80 "%80,%81,%82,%83,%84,%85,%86,%87,%88,%89,%90,%91,%92,%93,%94,%95"
#define WG_R96 "%96,%97,%98,%99,%100,%101,%102,%103,%104,%105,%106,%107,%108,%109,%110,%111"
#define WG_R112 "%112,%113,%114,%115,%116,%117,%118,%119,%120,%121,%122,%123,%124,%125,%126,%127"
#define WG_D16(i) "+f"(d[i]), "+f"(d[i + 1]), "+f"(d[i + 2]), "+f"(d[i + 3]), "+f"(d[i + 4]), "+f"(d[i + 5]), "+f"(d[i + 6]), "+f"(d[i + 7]), "+f"(d[i + 8]), "+f"(d[i + 9]), "+f"(d[i + 10]), "+f"(d[i + 11]), "+f"(d[i + 12]), "+f"(d[i + 13]), "+f"(d[i + 14]), "+f"(d[i + 15])
#define WG_D32 WG_D16(0), WG_D16(16)
#define WG_D48 WG_D32, WG_D16(32)
#define WG_D64 WG_D48, WG_D16(48)
#define WG_D128 WG_D64, WG_D16(64), WG_D16(80), WG_D16(96), WG_D16(112)
#define WG_V16 "{" WG_R0 "}"
#define WG_V32 "{" WG_R0 "," WG_R16 "}"
#define WG_V48 "{" WG_R0 "," WG_R16 "," WG_R32 "}"
#define WG_V64 "{" WG_R0 "," WG_R16 "," WG_R32 "," WG_R48 "}"
#define WG_V128 "{" WG_R0 "," WG_R16 "," WG_R32 "," WG_R48 "," WG_R64 "," WG_R80 "," WG_R96 "," WG_R112 "}"
// scale-d predicate from operand %n (0: D = A.B, else D += A.B)
#define WG_PRED(n) "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %" #n ", 0;\n\t"
__device__ __forceinline__ void wgmma_tf32_ss_n32(float* d, uint64_t adesc, uint64_t bdesc, uint32_t acc) {
  asm volatile(WG_PRED(18) "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 " WG_V16 ", %16, %17, p, 1, 1;\n\t}"
               : WG_D16(0) : "l"(adesc), "l"(bdesc), "r"(acc));
}
__device__ __forceinline__ void wgmma_tf32_rs_n32(float* d, const uint32_t* a, uint64_t bdesc, uint32_t acc) {
  asm volatile(WG_PRED(21) "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 " WG_V16 ", {%16,%17,%18,%19}, %20, p, 1, 1;\n\t}"
               : WG_D16(0) : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(acc));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_f16_ss_n16(float* d, uint64_t adesc, uint64_t bdesc, uint32_t acc) {
  asm volatile(WG_PRED(10) "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0,%1,%2,%3,%4,%5,%6,%7}, %8, %9, p, 1, 1, %11, %12;\n\t}"
               : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
               : "l"(adesc), "l"(bdesc), "r"(acc), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_f16_ss_n32(float* d, uint64_t adesc, uint64_t bdesc, uint32_t acc) {
  asm volatile(WG_PRED(18) "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 " WG_V16 ", %16, %17, p, 1, 1, %19, %20;\n\t}"
               : WG_D16(0) : "l"(adesc), "l"(bdesc), "r"(acc), "n"(TA), "n"(TB));
}
__device__ __forceinline__ void wgmma_tf32_ss_n64(float* d, uint64_t adesc, uint64_t bdesc, uint32_t acc) {
  asm volatile(WG_PRED(34) "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 " WG_V32 ", %32, %33, p, 1, 1;\n\t}"
               : WG_D32 : "l"(adesc), "l"(bdesc), "r"(acc));
}
__device__ __forceinline__ void wgmma_tf32_ss_n128(float* d, uint64_t adesc, uint64_t bdesc, uint32_t acc) {
  asm volatile(WG_PRED(66) "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 " WG_V64 ", %64, %65, p, 1, 1;\n\t}"
               : WG_D64 : "l"(adesc), "l"(bdesc), "r"(acc));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_f16_ss_n64(float* d, uint64_t adesc, uint64_t bdesc, uint32_t acc) {
  asm volatile(WG_PRED(34) "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 " WG_V32 ", %32, %33, p, 1, 1, %35, %36;\n\t}"
               : WG_D32 : "l"(adesc), "l"(bdesc), "r"(acc), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_f16_ss_n128(float* d, uint64_t adesc, uint64_t bdesc, uint32_t acc) {
  asm volatile(WG_PRED(66) "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 " WG_V64 ", %64, %65, p, 1, 1, %67, %68;\n\t}"
               : WG_D64 : "l"(adesc), "l"(bdesc), "r"(acc), "n"(TA), "n"(TB));
}
template <int TA, int TB>
__device__ __forceinline__ void wgmma_f16_ss_n256(float* d, uint64_t adesc, uint64_t bdesc, uint32_t acc) {
  asm volatile(WG_PRED(130) "wgmma.mma_async.sync.aligned.m64n256k16.f32.f16.f16 " WG_V128 ", %128, %129, p, 1, 1, %131, %132;\n\t}"
               : WG_D128 : "l"(adesc), "l"(bdesc), "r"(acc), "n"(TA), "n"(TB));
}
template <int TB>
__device__ __forceinline__ void wgmma_f16_rs_n64(float* d, const uint32_t* a, uint64_t bdesc, uint32_t acc) {
  asm volatile(WG_PRED(37) "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 " WG_V32 ", {%32,%33,%34,%35}, %36, p, 1, 1, %38;\n\t}"
               : WG_D32 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(acc), "n"(TB));
}
template <int TB>
__device__ __forceinline__ void wgmma_f16_rs_n128(float* d, const uint32_t* a, uint64_t bdesc, uint32_t acc) {
  asm volatile(WG_PRED(69) "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 " WG_V64 ", {%64,%65,%66,%67}, %68, p, 1, 1, %70;\n\t}"
               : WG_D64 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(acc), "n"(TB));
}
template <int TB>
__device__ __forceinline__ void wgmma_f16_rs_n96(float* d, const uint32_t* a, uint64_t bdesc, uint32_t acc) {
  asm volatile(WG_PRED(53) "wgmma.mma_async.sync.aligned.m64n96k16.f32.f16.f16 " WG_V48 ", {%48,%49,%50,%51}, %52, p, 1, 1, %54;\n\t}"
               : WG_D48 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(acc), "n"(TB));
}
__device__ __forceinline__ void wgmma_tf32_rs_n96(float* d, const uint32_t* a, uint64_t bdesc, uint32_t acc) {
  asm volatile(WG_PRED(53) "wgmma.mma_async.sync.aligned.m64n96k8.f32.tf32.tf32 " WG_V48 ", {%48,%49,%50,%51}, %52, p, 1, 1;\n\t}"
               : WG_D48 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(acc));
}
__device__ __forceinline__ void wgmma_tf32_rs_n128(float* d, const uint32_t* a, uint64_t bdesc, uint32_t acc) {
  asm volatile(WG_PRED(69) "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 " WG_V64 ", {%64,%65,%66,%67}, %68, p, 1, 1;\n\t}"
               : WG_D64 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc), "r"(acc));
}
// FP8 (K = 32 per MMA): A is e4m3, B is e4m3 or (B_E5M2) e5m2.  8-bit operands have no transpose bit: both are K-major.
template <bool B_E5M2>
__device__ __forceinline__ void wgmma_f8_ss_n128(float* d, uint64_t adesc, uint64_t bdesc, uint32_t acc) {
  if constexpr (B_E5M2)
    asm volatile(WG_PRED(66) "wgmma.mma_async.sync.aligned.m64n128k32.f32.e4m3.e5m2 " WG_V64 ", %64, %65, p, 1, 1;\n\t}"
                 : WG_D64 : "l"(adesc), "l"(bdesc), "r"(acc));
  else
    asm volatile(WG_PRED(66) "wgmma.mma_async.sync.aligned.m64n128k32.f32.e4m3.e4m3 " WG_V64 ", %64, %65, p, 1, 1;\n\t}"
                 : WG_D64 : "l"(adesc), "l"(bdesc), "r"(acc));
}

}  // namespace wg
}  // namespace mas
