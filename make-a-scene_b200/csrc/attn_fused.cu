// AttnBlock core, fused (modules.py:175-187): for one image and one tile of 128 queries
//     S = scale * Q K^T  ->  P = softmax_rows(S)  ->  O = P V
// in ONE kernel: S lives in the accumulator registers only, the softmax runs on the accumulator fragment, P goes to shared
// memory as the A operand of the second contraction (and once to global memory, for the backward).  The reference runs both
// contractions in strict fp32 (torch.bmm): operands are split into two fp16 numbers (x*s = h + l, 22 bits; power-of-two
// scales from the tensors' largest magnitude) and every K step issues three fp16 wgmma (hh + lh + hl), accumulated in fp32 -
// the same arithmetic as the VQ filter (vq_tc.cu).
//
//   * grid = (HW / 128 query tiles, N images); two warpgroups, warpgroup g owns query rows 64 g .. 64 g + 63 of the tile and
//     both stage the operands (generic loads, split, st.shared) into a 2-stage ring.
//   * phase 1: Q and K chunks of 32 channels as K-major planes [k/8][row][8 halves] (hi and lo), 6 wgmma.m64nHWk16 per chunk.
//   * softmax on the fragment (a row is spread over the four lanes of a quad): P -> global (fp32) and, split, -> shared
//     memory planes [key/8][row][8 halves] (hi, lo) over the idle phase-1 ring.
//   * phase 2: O = P V in halves of 256 channels: A = P (K-major), B = V chunks of 32 keys staged UNTRANSPOSED as MN-major
//     planes [c/8][key][8 channels], 6 wgmma.m64n256k16 per chunk; each half is stored straight from the fragment.
#include <cuda_fp16.h>

#include "mas_common.cuh"
#include "wgmma.cuh"

namespace mas {
namespace attnf {

constexpr int BM = 128, KC = 32, STAGES = 2;
constexpr int NPROD = 256, NTHREADS = 256;
constexpr int HWMAX = 256;                       // keys (= accumulator columns of S)
constexpr int PITCH_Q = BM * 16 + 32;            // bytes between 8-channel planes of the Q chunk
constexpr int PITCH_K = HWMAX * 16 + 32;         // ... of the K chunk (rows = keys)
constexpr int Q_HALF = (KC / 8) * PITCH_Q, K_HALF = (KC / 8) * PITCH_K;
constexpr int STAGE1 = 2 * Q_HALF + 2 * K_HALF;  // phase-1 stage: Q hi, Q lo, K hi, K lo
constexpr int PITCH_P = BM * 16 + 32;            // bytes between 8-key planes of P
constexpr int P_HALF = (HWMAX / 8) * PITCH_P;
constexpr int REGION1 = (STAGES * STAGE1 > 2 * P_HALF) ? STAGES * STAGE1 : 2 * P_HALF;   // phase-1 ring, then P
constexpr int NV = 256;                          // channels of one O half (N of the phase-2 MMAs)
constexpr int PITCH_V = KC * 16 + 16;            // phase 2, MN-major: plane = 8 channels, rows = the chunk's 32 keys (16 B skew)
constexpr int V_HALF = (NV / 8) * PITCH_V;
constexpr int STAGE2 = 2 * V_HALF;

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ float split_scale(const float* amax, float* inv) {
  float s = 1.f, i = 1.f;
  const uint32_t b = __float_as_uint(*amax);
  const int e = (int)((b >> 23) & 0xff);
  if (e > 0 && e < 255) {
    int se = 127 + 14 - (e - 127);
    se = se < 1 ? 1 : (se > 254 ? 254 : se);
    s = __uint_as_float((uint32_t)se << 23);
    i = __uint_as_float((uint32_t)(254 - se) << 23);
  }
  *inv = i;
  return s;
}
__device__ __forceinline__ void split2(float a, float b, float s, uint32_t* hi, uint32_t* lo) {
  const float as = a * s, bs = b * s;
  const __half2 h = __floats2half2_rn(as, bs);
  const float2 hf = __half22float2(h);
  const __half2 l = __floats2half2_rn(as - hf.x, bs - hf.y);
  *hi = *reinterpret_cast<const uint32_t*>(&h);
  *lo = *reinterpret_cast<const uint32_t*>(&l);
}
__device__ __forceinline__ void split8(const float4& v0, const float4& v1, float s, uint4* h, uint4* l) {
  split2(v0.x, v0.y, s, &h->x, &l->x);
  split2(v0.z, v0.w, s, &h->y, &l->y);
  split2(v1.x, v1.y, s, &h->z, &l->z);
  split2(v1.z, v1.w, s, &h->w, &l->w);
}

struct Params {
  const float* qkv;   // [N*HW, 3C]: q | k | v
  float* P;           // [N, HW, HW] softmax probabilities (saved for the backward)
  float* O;           // [N*HW, C]
  const float* amax;  // device scalar: max |qkv| (one scale for q, k and v)
  int HW, C;
  float scale;
};

template <int HW>
__device__ __forceinline__ void mma_s(float* d, uint64_t a, uint64_t b, uint32_t acc) {
  if (HW == 256) wg::wgmma_f16_ss_n256<0, 0>(d, a, b, acc);
  else wg::wgmma_f16_ss_n128<0, 0>(d, a, b, acc);
}

template <int HW>
__global__ void __launch_bounds__(NTHREADS, 1) attn_core_fwd(const Params p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* vring = smem + REGION1;
  const uint32_t smem_base = smem_u32(smem), v_base = smem_u32(vring);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wgi = warp >> 2, fk = lane & 3;
  const int C = p.C, C3 = 3 * C;
  const int n = blockIdx.y, q0 = blockIdx.x * BM;
  const float* base = p.qkv + (size_t)n * HW * C3;
  const int nchunk1 = C / KC, nchunk2 = HW / KC, nhalf = C / NV;
  const int frow = wgi * 64 + (warp & 3) * 16 + (lane >> 2);   // fragment rows frow, frow + 8 (query within the tile)
  const uint32_t a_rows = (uint32_t)(wgi * 64 * 16);          // this warpgroup's rows inside a K-major plane
  float inv_s;
  const float sc = split_scale(p.amax, &inv_s);
  constexpr float P_SCALE = 16384.0f, P_INV = 1.0f / 16384.0f;    // probabilities in [0, 1] -> [0, 2^14]
  const int pt = tid;

  // ---- phase 1: S = Q K^T over chunks of 32 channels ----
  float acc[HW / 2];
  int stage = 0;
  for (int c = 0; c < nchunk1; ++c) {
    // items: (row, oct) with oct fastest: 4 lanes read one row's 128 contiguous bytes; all loads of a chunk in flight together
    constexpr int NI1 = (BM + HW) * (KC / 8) / NPROD;
    float4 v0[NI1], v1[NI1];
#pragma unroll
    for (int i = 0; i < NI1; ++i) {
      const int it = pt + i * NPROD, oct = it & 3, r = it >> 2;
      const bool isq = r < BM;
      const int rr = isq ? r : r - BM;
      const float4* src = reinterpret_cast<const float4*>(base + (size_t)(isq ? q0 + rr : rr) * C3 + (isq ? 0 : C) + c * KC + oct * 8);
      v0[i] = __ldg(src);
      v1[i] = __ldg(src + 1);
    }
    if (c > 0) __syncthreads();   // both warpgroups have retired the MMAs that last read this stage (wait<1> below)
    uint8_t* st = smem + (size_t)stage * STAGE1;
#pragma unroll
    for (int i = 0; i < NI1; ++i) {
      const int it = pt + i * NPROD, oct = it & 3, r = it >> 2;
      const bool isq = r < BM;
      const int rr = isq ? r : r - BM;
      uint4 h, l;
      split8(v0[i], v1[i], sc, &h, &l);
      uint8_t* dh = isq ? st + oct * PITCH_Q + rr * 16 : st + 2 * Q_HALF + oct * PITCH_K + rr * 16;
      *reinterpret_cast<uint4*>(dh) = h;
      *reinterpret_cast<uint4*>(dh + (isq ? Q_HALF : K_HALF)) = l;
    }
    fence_proxy_async();
    __syncthreads();
    const uint32_t sa = smem_base + (uint32_t)stage * STAGE1;
    wg::fence();
#pragma unroll
    for (int k16 = 0; k16 < KC / 16; ++k16) {
      const uint64_t qh = wg::desc(sa + a_rows + (uint32_t)(k16 * 2 * PITCH_Q), PITCH_Q, 128);
      const uint64_t ql = wg::desc(sa + a_rows + (uint32_t)(Q_HALF + k16 * 2 * PITCH_Q), PITCH_Q, 128);
      const uint64_t kh = wg::desc(sa + (uint32_t)(2 * Q_HALF + k16 * 2 * PITCH_K), PITCH_K, 128);
      const uint64_t kl = wg::desc(sa + (uint32_t)(2 * Q_HALF + K_HALF + k16 * 2 * PITCH_K), PITCH_K, 128);
      mma_s<HW>(acc, qh, kh, (c > 0 || k16 > 0) ? 1u : 0u);
      mma_s<HW>(acc, ql, kh, 1u);
      mma_s<HW>(acc, qh, kl, 1u);
    }
    wg::commit();
    wg::wait<STAGES - 1>();
    if (++stage == STAGES) stage = 0;
  }
  wg::wait<0>();
  wg::fence_regs<HW / 2>(acc);

  // ---- softmax: row frow + 8 i is spread over the four lanes of this quad (keys 8 j + 2 fk + {0, 1}) ----
  const float ss = p.scale * inv_s * inv_s;                   // accumulator -> scale * q.k
  float mx[2] = {-INFINITY, -INFINITY}, sum[2] = {0.f, 0.f};
#pragma unroll
  for (int j = 0; j < HW / 8; ++j)
#pragma unroll
    for (int i = 0; i < 2; ++i) mx[i] = fmaxf(mx[i], fmaxf(acc[4 * j + 2 * i] * ss, acc[4 * j + 2 * i + 1] * ss));
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    mx[i] = fmaxf(mx[i], __shfl_xor_sync(0xffffffffu, mx[i], 1));
    mx[i] = fmaxf(mx[i], __shfl_xor_sync(0xffffffffu, mx[i], 2));
  }
#pragma unroll
  for (int j = 0; j < HW / 8; ++j)
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int cc = 0; cc < 2; ++cc) {
        const float e = expf(acc[4 * j + 2 * i + cc] * ss - mx[i]);
        acc[4 * j + 2 * i + cc] = e;
        sum[i] += e;
      }
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    sum[i] += __shfl_xor_sync(0xffffffffu, sum[i], 1);
    sum[i] += __shfl_xor_sync(0xffffffffu, sum[i], 2);
  }
  __syncthreads();   // every MMA of phase 1 has completed in both warpgroups: the ring becomes the P planes
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const float rs = 1.0f / sum[i];
    const int row = frow + 8 * i;
    float* prow = p.P + ((size_t)n * HW + q0 + row) * HW + 2 * fk;
#pragma unroll
    for (int j = 0; j < HW / 8; ++j) {
      const float a = acc[4 * j + 2 * i] * rs, b = acc[4 * j + 2 * i + 1] * rs;
      *reinterpret_cast<float2*>(prow + 8 * j) = make_float2(a, b);
      uint32_t hi, lo;
      split2(a, b, P_SCALE, &hi, &lo);
      uint8_t* d = smem + (size_t)j * PITCH_P + row * 16 + fk * 4;
      *reinterpret_cast<uint32_t*>(d) = hi;
      *reinterpret_cast<uint32_t*>(d + P_HALF) = lo;
    }
  }
  fence_proxy_async();

  // ---- phase 2: O = P V, 256 channels at a time, 32 keys per chunk ----
  const float oscale = inv_s * P_INV;
  float* oacc = acc;   // HW == 256: the S registers are free again; HW == 128: a separate set
  float oacc_own[HW == 256 ? 1 : NV / 2];
  if (HW != 256) oacc = oacc_own;
  stage = 0;
  int it2 = 0;
  for (int half = 0; half < nhalf; ++half) {
    for (int c = 0; c < nchunk2; ++c, ++it2) {
      constexpr int NI2 = KC * (NV / 8) / NPROD;
      float4 v0[NI2], v1[NI2];
#pragma unroll
      for (int i = 0; i < NI2; ++i) {
        const int it = pt + i * NPROD, oc = it % (NV / 8), key = it / (NV / 8);   // consecutive lanes: consecutive 32 bytes of one key's row
        const float4* src = reinterpret_cast<const float4*>(base + (size_t)(c * KC + key) * C3 + 2 * C + half * NV + oc * 8);
        v0[i] = __ldg(src);
        v1[i] = __ldg(src + 1);
      }
      __syncthreads();   // first chunk: P is complete; later: the MMAs that last read this stage have retired
      uint8_t* st = vring + (size_t)stage * STAGE2;
#pragma unroll
      for (int i = 0; i < NI2; ++i) {
        const int it = pt + i * NPROD, oc = it % (NV / 8), key = it / (NV / 8);
        uint4 h, l;
        split8(v0[i], v1[i], sc, &h, &l);
        uint8_t* dh = st + oc * PITCH_V + key * 16;
        *reinterpret_cast<uint4*>(dh) = h;
        *reinterpret_cast<uint4*>(dh + V_HALF) = l;
      }
      fence_proxy_async();
      __syncthreads();
      const uint32_t sv = v_base + (uint32_t)stage * STAGE2;
      wg::fence();
#pragma unroll
      for (int k16 = 0; k16 < KC / 16; ++k16) {
        const uint32_t poff = (uint32_t)((c * KC / 8 + k16 * 2) * PITCH_P);
        const uint64_t ph = wg::desc(smem_base + a_rows + poff, PITCH_P, 128);
        const uint64_t pl = wg::desc(smem_base + a_rows + (uint32_t)P_HALF + poff, PITCH_P, 128);
        // MN-major B: K groups (8 keys) are 128 bytes apart inside a plane, N groups are the planes
        const uint64_t vh = wg::desc(sv + (uint32_t)(k16 * 256), 128, PITCH_V);
        const uint64_t vl = wg::desc(sv + (uint32_t)(V_HALF + k16 * 256), 128, PITCH_V);
        wg::wgmma_f16_ss_n256<0, 1>(oacc, ph, vh, (c > 0 || k16 > 0) ? 1u : 0u);
        wg::wgmma_f16_ss_n256<0, 1>(oacc, pl, vh, 1u);
        wg::wgmma_f16_ss_n256<0, 1>(oacc, ph, vl, 1u);
      }
      wg::commit();
      wg::wait<STAGES - 1>();
      if (++stage == STAGES) stage = 0;
    }
    wg::wait<0>();
    wg::fence_regs<NV / 2>(oacc);
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      float* orow = p.O + ((size_t)n * HW + q0 + frow + 8 * i) * C + half * NV + 2 * fk;
#pragma unroll
      for (int j = 0; j < NV / 8; ++j)
        *reinterpret_cast<float2*>(orow + 8 * j) = make_float2(oacc[4 * j + 2 * i] * oscale, oacc[4 * j + 2 * i + 1] * oscale);
    }
  }
}

constexpr size_t SMEM_BYTES = (size_t)REGION1 + (size_t)STAGES * STAGE2;

}  // namespace attnf

bool attn_core_fused_ok(int HW, int C) { return (HW == 128 || HW == 256) && C % attnf::NV == 0 && C >= attnf::NV; }

// amax: device scalar holding max |qkv| (mas_amax); P [N,HW,HW] and O [N*HW, C] are written.
int attn_core_fused_launch(const float* qkv, const float* amax, float* P, float* O, int N, int HW, int C, float scale, cudaStream_t st) {
  if (!attn_core_fused_ok(HW, C)) return fail(MAS_ERR_UNSUPPORTED, "fused attention core: HW=%d C=%d not eligible", HW, C);
  static std::atomic<uint64_t> configured{0};
  if (first_on_device(configured)) {
    cudaError_t e = cudaFuncSetAttribute(attnf::attn_core_fwd<256>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)attnf::SMEM_BYTES);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(attnf::attn_core_fwd<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)attnf::SMEM_BYTES);
    if (e != cudaSuccess) return fail(MAS_ERR_LAUNCH, "attn_core_fwd: smem attr: %s", cudaGetErrorString(e));
    mark_device(configured);
  }
  attnf::Params p;
  p.qkv = qkv; p.P = P; p.O = O; p.amax = amax; p.HW = HW; p.C = C; p.scale = scale;
  const dim3 grid((unsigned)(HW / attnf::BM), (unsigned)N);
  if (HW == 256) attnf::attn_core_fwd<256><<<grid, attnf::NTHREADS, attnf::SMEM_BYTES, st>>>(p);
  else attnf::attn_core_fwd<128><<<grid, attnf::NTHREADS, attnf::SMEM_BYTES, st>>>(p);
  return launched_tc("attn_core_fwd");
}

}  // namespace mas
