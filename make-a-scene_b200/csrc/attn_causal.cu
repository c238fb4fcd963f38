// Causal self-attention core of the token transformer, fused (transformer.py:77-103): for one (sequence, head, tile of 128
// queries)
//     S = (q k^T) / sqrt(hd)  ->  P = softmax_rows(S restricted to keys <= query)  ->  ctx = P v
// in ONE kernel over the fused [B, S, 3H] q|k|v activation: the scores live in the accumulator registers only, the softmax
// runs on the accumulator fragment, P goes to shared memory as the A operand of the second contraction (and once to global
// memory, for the backward), ctx is accumulated in registers over the key blocks.  Only the causal key blocks (<= the query
// tile) are visited.  Same arithmetic as the AttnBlock core (attn_fused.cu): the reference runs both contractions in strict
// fp32, so operands are split into two fp16 numbers (x*s = h + l, 22 bits) and every K step issues three fp16 wgmma
// (hh + lh + hl).
//
//   * grid = (S / 128 query tiles - heaviest first, heads, B); two warpgroups, warpgroup g owns query rows 64 g .. 64 g + 63
//     of the tile; both stage the operands (generic loads, split, st.shared).
//   * two passes over the key blocks of 128: pass 0 computes the row maxima and sums online (scores only), pass 1 recomputes the
//     scores, writes the normalised probabilities (global fp32 + split into shared memory) and accumulates ctx += P_blk v_blk.
//     The score contraction is cheap (K = 64), recomputing it is what keeps P exactly normalised without rescaling the
//     accumulator.
//   * shared memory: the Q tile (resident) + a 2-stage ring of K / V tiles (hi and lo images) + the P block, K-major planes
//     [c/8][row][8 halves] for Q, K and P, MN-major planes [c/8][key][8 channels] for V (staged untransposed).
#include <cuda_fp16.h>

#include "mas_common.cuh"
#include "wgmma.cuh"

namespace mas {
namespace attnc {

constexpr int BM = 128, BK = 128, HD = 64, STAGES = 2;
constexpr int NPROD = 256, NTHREADS = 256;
constexpr int PITCH_K = BK * 16 + 32;            // bytes between 8-channel planes of a Q / K tile (rows = queries / keys)
constexpr int K_HALF = (HD / 8) * PITCH_K;       // one image (hi or lo)
constexpr int PITCH_V = BK * 16 + 16;            // MN-major V tile: plane = 8 channels, rows = the block's 128 keys
constexpr int V_HALF = (HD / 8) * PITCH_V;
constexpr int TILE = 2 * K_HALF;                 // hi + lo (the V tile is slightly smaller)
static_assert(2 * V_HALF <= TILE, "V tile must fit a ring stage");
constexpr int PITCH_P = BM * 16 + 32;            // bytes between 8-key planes of the P block (rows = queries)
constexpr int P_HALF = (BK / 8) * PITCH_P;

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
  const float* qkv;   // [B, S, 3H]: q | k | v, head h owns columns h*HD .. of each third
  float* P;           // [B, heads, S, S] softmax probabilities (saved for the backward; zeros above the diagonal)
  float* ctx;         // [B, S, H]
  const float* amax;  // device scalar: max |qkv| (one scale for q, k and v)
  int S, heads;
  float scale;
};

__global__ void __launch_bounds__(NTHREADS, 1) attn_causal_fwd(const Params p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* q_tile = smem;                                   // resident Q tile (hi, lo)
  uint8_t* ring = smem + TILE;                              // STAGES x TILE
  uint8_t* p_blk = ring + (size_t)STAGES * TILE;            // P block (hi, lo)
  const uint32_t q_base = smem_u32(q_tile), ring_base = smem_u32(ring), p_base = smem_u32(p_blk);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wgi = warp >> 2, fk = lane & 3;
  const int S = p.S, heads = p.heads, H = heads * HD, C3 = 3 * H;
  const int qt = (int)gridDim.x - 1 - (int)blockIdx.x;      // heaviest query tiles first
  const int h = blockIdx.y, b = blockIdx.z;
  const int q0 = qt * BM, nkb = qt + 1;                     // causal: key blocks 0 .. qt
  const float* base = p.qkv + (size_t)b * S * C3 + h * HD;
  const int frow = wgi * 64 + (warp & 3) * 16 + (lane >> 2);   // fragment rows frow, frow + 8 (query within the tile)
  const uint32_t a_rows = (uint32_t)(wgi * 64 * 16);          // this warpgroup's rows inside a K-major plane
  float inv_s;
  const float sc = split_scale(p.amax, &inv_s);
  constexpr float P_SCALE = 16384.0f, P_INV = 1.0f / 16384.0f;    // probabilities in [0, 1] -> [0, 2^14]
  const int pt = tid;

  // a [128 rows x 64 channels] fp32 tile of the q / k / v third -> hi / lo images; 1024 items of 8 channels, 4 per thread:
  // item = (row, oct) with oct fastest: 8 lanes read one row's 256 contiguous bytes; all loads of a tile in flight together.
  // The caller has retired every MMA that read dst (wait<0> in both warpgroups, then the barrier below).
  auto fill = [&](uint8_t* dst, int third, int row0, int pitch, int half) {
    float4 v0[4], v1[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int itm = pt + i * NPROD, oct = itm & 7, r = itm >> 3;
      const float4* src = reinterpret_cast<const float4*>(base + (size_t)(row0 + r) * C3 + third * H + oct * 8);
      v0[i] = __ldg(src);
      v1[i] = __ldg(src + 1);
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < 4; ++i) {
      const int itm = pt + i * NPROD, oct = itm & 7, r = itm >> 3;
      uint4 hh, ll;
      split8(v0[i], v1[i], sc, &hh, &ll);
      uint8_t* d = dst + oct * pitch + r * 16;
      *reinterpret_cast<uint4*>(d) = hh;
      *reinterpret_cast<uint4*>(d + half) = ll;
    }
    fence_proxy_async();
    __syncthreads();
  };

  // masked key blocks of the saved probabilities
  {
    float* pt0 = p.P + (((size_t)b * heads + h) * S + q0) * S;
    const int cols = S - nkb * BK;
    for (int i = tid; i < BM * (cols / 4); i += NTHREADS) {
      const int r = i / (cols / 4), c4 = i - r * (cols / 4);
      *reinterpret_cast<float4*>(pt0 + (size_t)r * S + nkb * BK + c4 * 4) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
  fill(q_tile, 0, q0, PITCH_K, K_HALF);

  const float ss = p.scale * inv_s * inv_s;                  // accumulator -> scale * q.k
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f}, rl[2] = {0.f, 0.f};
  float sacc[BK / 2], oacc[HD / 2];
  int stage = 0;
  for (int pass = 0; pass < 2; ++pass) {
    for (int kb = 0; kb < nkb; ++kb) {
      // ---- scores of this key block ----
      uint8_t* st = ring + (size_t)stage * TILE;
      fill(st, 1, kb * BK, PITCH_K, K_HALF);          // K block: K-major planes
      {
        const uint32_t sa = ring_base + (uint32_t)stage * TILE;
        wg::fence();
#pragma unroll
        for (int k16 = 0; k16 < HD / 16; ++k16) {
          const uint64_t qh = wg::desc(q_base + a_rows + (uint32_t)(k16 * 2 * PITCH_K), PITCH_K, 128);
          const uint64_t ql = wg::desc(q_base + a_rows + (uint32_t)(K_HALF + k16 * 2 * PITCH_K), PITCH_K, 128);
          const uint64_t kh = wg::desc(sa + (uint32_t)(k16 * 2 * PITCH_K), PITCH_K, 128);
          const uint64_t kl = wg::desc(sa + (uint32_t)(K_HALF + k16 * 2 * PITCH_K), PITCH_K, 128);
          wg::wgmma_f16_ss_n128<0, 0>(sacc, qh, kh, k16 > 0 ? 1u : 0u);
          wg::wgmma_f16_ss_n128<0, 0>(sacc, ql, kh, 1u);
          wg::wgmma_f16_ss_n128<0, 0>(sacc, qh, kl, 1u);
        }
        wg::commit();
        wg::wait<0>();
        wg::fence_regs<BK / 2>(sacc);
      }
      if (++stage == STAGES) stage = 0;
      const bool diag = kb == qt;                            // the only block with masked entries
      if (pass == 0) {
        // online maximum / sum over this thread's columns of its two rows; the four lanes of a row are combined at the end
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int rit = frow + 8 * i;
          float cm = -INFINITY;
#pragma unroll
          for (int j = 0; j < BK / 8; ++j)
#pragma unroll
            for (int c = 0; c < 2; ++c) {
              const int key = 8 * j + 2 * fk + c;
              const float v = (diag && key > rit) ? -INFINITY : sacc[4 * j + 2 * i + c] * ss;
              sacc[4 * j + 2 * i + c] = v;
              cm = fmaxf(cm, v);
            }
          const float mn = fmaxf(m[i], cm);
          if (mn > -INFINITY) {
            float add = 0.f;
#pragma unroll
            for (int j = 0; j < BK / 8; ++j) add += expf(sacc[4 * j + 2 * i] - mn) + expf(sacc[4 * j + 2 * i + 1] - mn);
            l[i] = l[i] * expf(m[i] - mn) + add;
            m[i] = mn;
          }
        }
        if (kb == nkb - 1) {
#pragma unroll
          for (int i = 0; i < 2; ++i) {
#pragma unroll
            for (int x = 1; x <= 2; x <<= 1) {
              const float om = __shfl_xor_sync(0xffffffffu, m[i], x), ol = __shfl_xor_sync(0xffffffffu, l[i], x);
              const float mn = fmaxf(m[i], om);
              l[i] = (m[i] > -INFINITY ? l[i] * expf(m[i] - mn) : 0.f) + (om > -INFINITY ? ol * expf(om - mn) : 0.f);
              m[i] = mn;
            }
            rl[i] = 1.0f / l[i];
          }
        }
      } else {
        // probabilities: global (fp32) and the split P block in shared memory (the previous block's P V MMAs have retired:
        // the barrier in fill() above)
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int rit = frow + 8 * i;
          float* prow = p.P + (((size_t)b * heads + h) * S + q0 + rit) * S + kb * BK + 2 * fk;
#pragma unroll
          for (int j = 0; j < BK / 8; ++j) {
            const int key = 8 * j + 2 * fk;
            const float a = (diag && key > rit) ? 0.f : expf(sacc[4 * j + 2 * i] * ss - m[i]) * rl[i];
            const float c = (diag && key + 1 > rit) ? 0.f : expf(sacc[4 * j + 2 * i + 1] * ss - m[i]) * rl[i];
            *reinterpret_cast<float2*>(prow + 8 * j) = make_float2(a, c);
            uint32_t hi, lo;
            split2(a, c, P_SCALE, &hi, &lo);
            uint8_t* d = p_blk + (size_t)j * PITCH_P + rit * 16 + fk * 4;
            *reinterpret_cast<uint32_t*>(d) = hi;
            *reinterpret_cast<uint32_t*>(d + P_HALF) = lo;
          }
        }
        // ---- ctx += P_blk V_blk: A = P (K-major), B = the V tile, MN-major ----
        uint8_t* sv = ring + (size_t)stage * TILE;
        fill(sv, 2, kb * BK, PITCH_V, V_HALF);        // V block: MN-major planes [c/8][key][8 channels]; fences the P stores too
        const uint32_t vb = ring_base + (uint32_t)stage * TILE;
        wg::fence();
#pragma unroll
        for (int k16 = 0; k16 < BK / 16; ++k16) {
          const uint64_t ph = wg::desc(p_base + a_rows + (uint32_t)(k16 * 2 * PITCH_P), PITCH_P, 128);
          const uint64_t pl = wg::desc(p_base + a_rows + (uint32_t)(P_HALF + k16 * 2 * PITCH_P), PITCH_P, 128);
          // MN-major B: K groups (8 keys) are 128 bytes apart inside a plane, N groups are the planes
          const uint64_t vh = wg::desc(vb + (uint32_t)(k16 * 256), 128, PITCH_V);
          const uint64_t vl = wg::desc(vb + (uint32_t)(V_HALF + k16 * 256), 128, PITCH_V);
          wg::wgmma_f16_ss_n64<0, 1>(oacc, ph, vh, (kb > 0 || k16 > 0) ? 1u : 0u);
          wg::wgmma_f16_ss_n64<0, 1>(oacc, pl, vh, 1u);
          wg::wgmma_f16_ss_n64<0, 1>(oacc, ph, vl, 1u);
        }
        wg::commit();
        wg::wait<0>();
        wg::fence_regs<HD / 2>(oacc);
        if (++stage == STAGES) stage = 0;
      }
    }
  }
  // ctx tile: straight from the fragment
  const float oscale = inv_s * P_INV;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    float* orow = p.ctx + ((size_t)b * S + q0 + frow + 8 * i) * H + h * HD + 2 * fk;
#pragma unroll
    for (int j = 0; j < HD / 8; ++j)
      *reinterpret_cast<float2*>(orow + 8 * j) = make_float2(oacc[4 * j + 2 * i] * oscale, oacc[4 * j + 2 * i + 1] * oscale);
  }
}

constexpr size_t SMEM_BYTES = (size_t)TILE * (1 + STAGES) + 2 * (size_t)P_HALF;

}  // namespace attnc

bool attn_causal_fused_ok(int S, int heads, int hd) { return hd == attnc::HD && S % attnc::BM == 0 && S >= attnc::BM && heads > 0; }

}  // namespace mas

using namespace mas;

extern "C" int mas_attn_causal_forward(const float* qkv, const float* amax, float* P, float* ctx, int B, int S, int heads, int hd,
                                       float scale, void* stream) {
  MAS_REQUIRE(qkv && amax && P && ctx && B > 0, "attn_causal_forward: bad arguments");
  if (!attn_causal_fused_ok(S, heads, hd))
    return fail(MAS_ERR_UNSUPPORTED, "attn_causal_forward: needs head dim 64 and S %% 128 == 0 (got S=%d, hd=%d)", S, hd);
  if (heads > 65535 || B > 65535) return fail(MAS_ERR_UNSUPPORTED, "attn_causal_forward: heads / batch beyond the grid limits");
  static std::atomic<uint64_t> configured{0};
  if (first_on_device(configured)) {
    cudaError_t e = cudaFuncSetAttribute(attnc::attn_causal_fwd, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)attnc::SMEM_BYTES);
    if (e != cudaSuccess) return fail(MAS_ERR_LAUNCH, "attn_causal_fwd: smem attr: %s", cudaGetErrorString(e));
    mark_device(configured);
  }
  attnc::Params p;
  p.qkv = qkv; p.P = P; p.ctx = ctx; p.amax = amax; p.S = S; p.heads = heads; p.scale = scale;
  const dim3 grid((unsigned)(S / attnc::BM), (unsigned)heads, (unsigned)B);
  attnc::attn_causal_fwd<<<grid, attnc::NTHREADS, attnc::SMEM_BYTES, mas::S(stream)>>>(p);
  return launched_tc("attn_causal_fwd");
}
