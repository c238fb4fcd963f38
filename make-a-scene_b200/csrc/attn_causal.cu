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
//   * head dim 64 or 128 (template parameter HD, tile constants in Cfg<HD>).
//   * two passes over the key blocks of 128 (64 at head dim 128): pass 0 computes the row maxima and sums online (scores only), pass 1 recomputes the
//     scores, writes the normalised probabilities (global fp32 + split into shared memory) and accumulates ctx += P_blk v_blk.
//     The score contraction is cheap (K = 64), recomputing it is what keeps P exactly normalised without rescaling the
//     accumulator.
//   * STATS (mas_attn_causal_forward_stats, the backward recomputes P: attn_causal_bwd.cu): pass 1 stores no probabilities;
//     instead pass 0 writes every row's maximum m and sum l, P = exp(S - m) / l.  The arithmetic is the P-writing kernel's
//     minus the store, so ctx is the same bits.
//   * shared memory: the Q tile (resident) + a 2-stage ring of K / V tiles (hi and lo images) + the P block, K-major planes
//     [c/8][row][8 halves] for Q, K and P, MN-major planes [c/8][key][8 channels] for V (staged untransposed).
//   * DROP (attention dropout, mas_attn_causal_dropout_forward): pass 1 still writes the undropped P (the softmax backward
//     needs it), then zeroes the dropped fragment elements before the split into shared memory.  The factor 1 / (1 - p) is
//     applied to ctx in the epilogue, not to P: the split keeps P * 2^14 within fp16, which P / (1 - p) would leave for large p.
//     The keep bits come from dropout.cuh's Philox groups of four keys: the lane pair (fk, fk ^ 1) covers one group per row,
//     so each lane generates one group per 8-key column block (row frow or frow + 8) and takes the other row's bits from its
//     partner by a shuffle.
//   * PREFIX (mas_attn_causal_prefix_forward, MakeAScene.score(num_samples=n)): the queries are the L suffix positions of
//     row r (qkv [R, L, 3H]), at absolute positions Lp + i, and the keys 0 .. Lp - 1 come from the shared prefix row r / n
//     (qkv_prefix [P, Lp, 3H]).  The tile, the key blocks and their order are those of the query tile at Lp + i of the
//     concatenated sequence; only fill() picks the source row of a block (prefix or suffix).  Nothing but ctx is written, so
//     ctx is the bits mas_attn_causal_forward gives there.
#include <cuda_fp16.h>

#include <type_traits>

#include "dropout.cuh"
#include "mas_common.cuh"
#include "wgmma.cuh"

namespace mas {
namespace attnc {

// Tile constants per head dim.  HD 64: 128-key blocks.  HD 128: 64-key blocks, so that the 128 x 128 Q tile, a 2-stage
// K / V ring and the P block stay within today's ~167 KB of shared memory and the accumulators at 96 fp32 registers a thread
// (scores 64 x 64 + ctx 64 x 128 per warpgroup).  The backward (below) streams 32-row blocks at HD 128 and splits dK / dV's
// output channels over two CTAs.
constexpr int BM = 128, STAGES = 2;
constexpr int NPROD = 256, NTHREADS = 256;
constexpr int PITCH_P = BM * 16 + 32;            // bytes between 8-key planes of the P block (rows = queries)
template <int HD_>
struct Cfg {
  static constexpr int HD = HD_;
  static_assert(HD == 64 || HD == 128, "head dim 64 or 128");
  static constexpr int BK = HD == 64 ? 128 : 64;           // forward key block
  static constexpr int PITCH_Q = BM * 16 + 32;             // bytes between 8-channel planes of a 128-row Q / K tile
  static constexpr int Q_HALF = (HD / 8) * PITCH_Q;        // one image (hi or lo)
  static constexpr int PITCH_K = BK * 16 + 32;             // the same for a K block (rows = its keys)
  static constexpr int K_HALF = (HD / 8) * PITCH_K;
  static constexpr int PITCH_V = BK * 16 + 16;             // MN-major V block: plane = 8 channels, rows = the block's keys
  static constexpr int V_HALF = (HD / 8) * PITCH_V;
  static constexpr int TILE = 2 * K_HALF;                  // a ring stage: hi + lo (the V block is slightly smaller)
  static_assert(2 * V_HALF <= TILE, "V tile must fit a ring stage");
  static constexpr int P_HALF = (BK / 8) * PITCH_P;
  static constexpr size_t SMEM_BYTES = 2 * (size_t)Q_HALF + (size_t)TILE * STAGES + 2 * (size_t)P_HALF;
  // backward (attn_causal_bwd)
  static constexpr int BN = HD == 64 ? 64 : 32;            // streamed rows per block
  static constexpr int NSPLIT = HD == 64 ? 1 : 2;          // DKV: CTAs per key tile, each owning HD / NSPLIT output channels
  static constexpr int PITCH_C = BN * 16 + 32;             // bytes between 8-channel planes of a streamed tile
  static constexpr int C_HALF = (HD / 8) * PITCH_C;
  static constexpr int B_HALF = (BN / 8) * PITCH_P;        // a [128 rows x BN columns] P / dS block, one image
  static constexpr size_t BWD_SMEM_BYTES = 4 * (size_t)Q_HALF + 4 * (size_t)C_HALF + 4 * (size_t)B_HALF;
};
static_assert(Cfg<128>::SMEM_BYTES <= 227 * 1024 && Cfg<128>::BWD_SMEM_BYTES <= 227 * 1024, "shared memory");

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
  float* P;           // [B, heads, S, S] softmax probabilities (saved for the backward; zeros above the diagonal);
                      // STATS: the row statistics instead, m [B, heads, S] followed by l [B, heads, S]
  float* ctx;         // [B, S, H]
  const float* amax;  // device scalar: max |qkv| (one scale for q, k and v)
  int S, heads;
  float scale;
  const float* qkvp;  // PREFIX: the shared prefix [P, Lp, 3H]; S is then the suffix length L, row b reads prefix row b / n
  int Lp, n;
};

// D += A B over one K step of 16, N columns (f16 operands, fp32 accumulators); TB = 1: B is MN-major
template <int N, int TB>
__device__ __forceinline__ void mma(float* d, uint64_t a, uint64_t b, uint32_t acc) {
  if constexpr (N == 32) wg::wgmma_f16_ss_n32<0, TB>(d, a, b, acc);
  else if constexpr (N == 64) wg::wgmma_f16_ss_n64<0, TB>(d, a, b, acc);
  else wg::wgmma_f16_ss_n128<0, TB>(d, a, b, acc);
}

template <int HD, bool DROP, bool STATS = false, bool PREFIX = false>
__global__ void __launch_bounds__(NTHREADS, 1) attn_causal_fwd(const Params p, const DropMask dm) {
  static_assert(!PREFIX || (!DROP && !STATS), "the prefix form writes ctx only");
  using C = Cfg<HD>;
  constexpr int BK = C::BK, PITCH_Q = C::PITCH_Q, Q_HALF = C::Q_HALF, PITCH_K = C::PITCH_K, K_HALF = C::K_HALF;
  constexpr int PITCH_V = C::PITCH_V, V_HALF = C::V_HALF, TILE = C::TILE, P_HALF = C::P_HALF;
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* q_tile = smem;                                   // resident Q tile (hi, lo)
  uint8_t* ring = smem + 2 * Q_HALF;                        // STAGES x TILE
  uint8_t* p_blk = ring + (size_t)STAGES * TILE;            // P block (hi, lo)
  const uint32_t q_base = smem_u32(q_tile), ring_base = smem_u32(ring), p_base = smem_u32(p_blk);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wgi = warp >> 2, fk = lane & 3;
  const int S = p.S, heads = p.heads, H = heads * HD, C3 = 3 * H;
  const int qt = (int)gridDim.x - 1 - (int)blockIdx.x;      // heaviest query tiles first
  const int h = blockIdx.y, b = blockIdx.z;
  const int qa = PREFIX ? qt + p.Lp / BM : qt;              // PREFIX: the tile's absolute position in prefix + suffix
  const int q0 = qa * BM, nkb = (qa + 1) * (BM / BK);       // causal: the key blocks up to the tile's last query
  const float* base = p.qkv + (size_t)b * S * C3 + h * HD;
  const float* pbase = PREFIX ? p.qkvp + (size_t)(b / p.n) * p.Lp * C3 + h * HD : nullptr;
  const int frow = wgi * 64 + (warp & 3) * 16 + (lane >> 2);   // fragment rows frow, frow + 8 (query within the tile)
  const uint32_t a_rows = (uint32_t)(wgi * 64 * 16);          // this warpgroup's rows inside a K-major plane
  float inv_s;
  const float sc = split_scale(p.amax, &inv_s);
  constexpr float P_SCALE = 16384.0f, P_INV = 1.0f / 16384.0f;    // probabilities in [0, 1] -> [0, 2^14]
  const int pt = tid;

  // a [ROWS x HD] fp32 tile of the q / k / v third -> hi / lo images; ROWS * HD / 8 items of 8 channels: item = (row, oct)
  // with oct fastest, so HD / 8 lanes read one row's contiguous bytes; all loads of a tile in flight together.
  // The caller has retired every MMA that read dst (wait<0> in both warpgroups, then the barrier below).
  // row0 is absolute: PREFIX reads rows below Lp from the prefix row, the others from this row's suffix.
  auto fill = [&](auto rows_c, uint8_t* dst, int third, int row0, int pitch, int half) {
    constexpr int N = decltype(rows_c)::value * (HD / 8) / NPROD, OCT_LOG = HD == 64 ? 3 : 4;
    const float* fb = base;
    if constexpr (PREFIX) {
      if (row0 < p.Lp) fb = pbase;
      else row0 -= p.Lp;
    }
    float4 v0[N], v1[N];
#pragma unroll
    for (int i = 0; i < N; ++i) {
      const int itm = pt + i * NPROD, oct = itm & (HD / 8 - 1), r = itm >> OCT_LOG;
      const float4* src = reinterpret_cast<const float4*>(fb + (size_t)(row0 + r) * C3 + third * H + oct * 8);
      v0[i] = __ldg(src);
      v1[i] = __ldg(src + 1);
    }
    __syncthreads();
#pragma unroll
    for (int i = 0; i < N; ++i) {
      const int itm = pt + i * NPROD, oct = itm & (HD / 8 - 1), r = itm >> OCT_LOG;
      uint4 hh, ll;
      split8(v0[i], v1[i], sc, &hh, &ll);
      uint8_t* d = dst + oct * pitch + r * 16;
      *reinterpret_cast<uint4*>(d) = hh;
      *reinterpret_cast<uint4*>(d + half) = ll;
    }
    fence_proxy_async();
    __syncthreads();
  };
  using RQ = std::integral_constant<int, BM>;
  using RK = std::integral_constant<int, BK>;

  // masked key blocks of the saved probabilities
  if constexpr (!STATS && !PREFIX) {
    float* pt0 = p.P + (((size_t)b * heads + h) * S + q0) * S;
    const int cols = S - nkb * BK;
    for (int i = tid; i < BM * (cols / 4); i += NTHREADS) {
      const int r = i / (cols / 4), c4 = i - r * (cols / 4);
      *reinterpret_cast<float4*>(pt0 + (size_t)r * S + nkb * BK + c4 * 4) = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
  fill(RQ{}, q_tile, 0, q0, PITCH_Q, Q_HALF);

  const float ss = p.scale * inv_s * inv_s;                  // accumulator -> scale * q.k
  float m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f}, rl[2] = {0.f, 0.f};
  float sacc[BK / 2], oacc[HD / 2];
  int stage = 0;
  for (int pass = 0; pass < 2; ++pass) {
    for (int kb = 0; kb < nkb; ++kb) {
      // ---- scores of this key block ----
      uint8_t* st = ring + (size_t)stage * TILE;
      fill(RK{}, st, 1, kb * BK, PITCH_K, K_HALF);    // K block: K-major planes
      {
        const uint32_t sa = ring_base + (uint32_t)stage * TILE;
        wg::fence();
#pragma unroll
        for (int k16 = 0; k16 < HD / 16; ++k16) {
          const uint64_t qh = wg::desc(q_base + a_rows + (uint32_t)(k16 * 2 * PITCH_Q), PITCH_Q, 128);
          const uint64_t ql = wg::desc(q_base + a_rows + (uint32_t)(Q_HALF + k16 * 2 * PITCH_Q), PITCH_Q, 128);
          const uint64_t kh = wg::desc(sa + (uint32_t)(k16 * 2 * PITCH_K), PITCH_K, 128);
          const uint64_t kl = wg::desc(sa + (uint32_t)(K_HALF + k16 * 2 * PITCH_K), PITCH_K, 128);
          mma<BK, 0>(sacc, qh, kh, k16 > 0 ? 1u : 0u);
          mma<BK, 0>(sacc, ql, kh, 1u);
          mma<BK, 0>(sacc, qh, kl, 1u);
        }
        wg::commit();
        wg::wait<0>();
        wg::fence_regs<BK / 2>(sacc);
      }
      if (++stage == STAGES) stage = 0;
      // the blocks with masked entries: key kb * BK + key > query q0 + rit for some row of the tile
      const int koff = BK == BM ? 0 : kb * BK - q0;          // the block's first key relative to the tile's first query
      const bool diag = BK == BM ? kb == qa : koff >= 0;
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
              const float v = (diag && key + koff > rit) ? -INFINITY : sacc[4 * j + 2 * i + c] * ss;
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
          if constexpr (STATS) {
            if (fk == 0) {
              float* mrow = p.P + ((size_t)b * heads + h) * S + q0 + frow;
              float* lrow = mrow + (size_t)gridDim.z * heads * S;
#pragma unroll
              for (int i = 0; i < 2; ++i) {
                mrow[8 * i] = m[i];
                lrow[8 * i] = l[i];
              }
            }
          }
        }
      } else {
        // probabilities: global (fp32) and the split P block in shared memory (the previous block's P V MMAs have retired:
        // the barrier in fill() above)
        uint32_t keep[2] = {0u, 0u};                           // DROP: bit 2 j + c <-> key 8 j + 2 fk + c of row frow + 8 i
        if constexpr (DROP) {
          const uint64_t seed = (uint64_t)*dm.seed;
          const uint64_t row0 = (((uint64_t)b * heads + h) * S + q0 + frow + 8 * (fk & 1)) * S + kb * BK + 4 * (fk >> 1);
#pragma unroll
          for (int j = 0; j < BK / 8; ++j) {
            const uint32_t bits = keep_bits4(seed, (row0 + 8 * j) >> 2, dm.t);
            const uint32_t b0 = __shfl_sync(0xffffffffu, bits, lane & ~1), b1 = __shfl_sync(0xffffffffu, bits, lane | 1);
            keep[0] |= ((b0 >> (2 * (fk & 1))) & 3u) << (2 * j);
            keep[1] |= ((b1 >> (2 * (fk & 1))) & 3u) << (2 * j);
          }
        }
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int rit = frow + 8 * i;
          float* prow = p.P + (((size_t)b * heads + h) * S + q0 + rit) * S + kb * BK + 2 * fk;
#pragma unroll
          for (int j = 0; j < BK / 8; ++j) {
            const int key = 8 * j + 2 * fk + koff;
            const float a = (diag && key > rit) ? 0.f : expf(sacc[4 * j + 2 * i] * ss - m[i]) * rl[i];
            const float c = (diag && key + 1 > rit) ? 0.f : expf(sacc[4 * j + 2 * i + 1] * ss - m[i]) * rl[i];
            if constexpr (!STATS && !PREFIX) *reinterpret_cast<float2*>(prow + 8 * j) = make_float2(a, c);
            uint32_t hi, lo;
            if constexpr (DROP)
              split2((keep[i] >> (2 * j)) & 1u ? a : 0.f, (keep[i] >> (2 * j + 1)) & 1u ? c : 0.f, P_SCALE, &hi, &lo);
            else
              split2(a, c, P_SCALE, &hi, &lo);
            uint8_t* d = p_blk + (size_t)j * PITCH_P + rit * 16 + fk * 4;
            *reinterpret_cast<uint32_t*>(d) = hi;
            *reinterpret_cast<uint32_t*>(d + P_HALF) = lo;
          }
        }
        // ---- ctx += P_blk V_blk: A = P (K-major), B = the V tile, MN-major ----
        uint8_t* sv = ring + (size_t)stage * TILE;
        fill(RK{}, sv, 2, kb * BK, PITCH_V, V_HALF);  // V block: MN-major planes [c/8][key][8 channels]; fences the P stores too
        const uint32_t vb = ring_base + (uint32_t)stage * TILE;
        wg::fence();
#pragma unroll
        for (int k16 = 0; k16 < BK / 16; ++k16) {
          const uint64_t ph = wg::desc(p_base + a_rows + (uint32_t)(k16 * 2 * PITCH_P), PITCH_P, 128);
          const uint64_t pl = wg::desc(p_base + a_rows + (uint32_t)(P_HALF + k16 * 2 * PITCH_P), PITCH_P, 128);
          // MN-major B: K groups (8 keys) are 128 bytes apart inside a plane, N groups are the planes
          const uint64_t vh = wg::desc(vb + (uint32_t)(k16 * 256), 128, PITCH_V);
          const uint64_t vl = wg::desc(vb + (uint32_t)(V_HALF + k16 * 256), 128, PITCH_V);
          mma<HD, 1>(oacc, ph, vh, (kb > 0 || k16 > 0) ? 1u : 0u);
          mma<HD, 1>(oacc, pl, vh, 1u);
          mma<HD, 1>(oacc, ph, vl, 1u);
        }
        wg::commit();
        wg::wait<0>();
        wg::fence_regs<HD / 2>(oacc);
        if (++stage == STAGES) stage = 0;
      }
    }
  }
  // ctx tile: straight from the fragment
  float oscale = inv_s * P_INV;
  if constexpr (DROP) oscale *= dm.scale;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    float* orow = p.ctx + ((size_t)b * S + q0 - (PREFIX ? p.Lp : 0) + frow + 8 * i) * H + h * HD + 2 * fk;
#pragma unroll
    for (int j = 0; j < HD / 8; ++j)
      *reinterpret_cast<float2*>(orow + 8 * j) = make_float2(oacc[4 * j + 2 * i] * oscale, oacc[4 * j + 2 * i + 1] * oscale);
  }
}

// ---- backward from the row statistics (mas_attn_causal_backward) --------------------------------------------------------
// P is recomputed from qkv and the forward's m / l, nothing S x S is read.  With dO = dctx, D_q = dO_q . ctx_q (a row
// pre-pass), keep the regenerated dropout mask and s = 1 / (1 - p):
//     dV = (P o keep)^T dO s,  dS = P o (dO v^T o keep s - D),  dQ = dS k * scale,  dK = dS^T q * scale.
// Two kernels of one template, no atomics (deterministic):
//   * DKV, per (sequence, head, 128-key tile): rows = keys; K and V resident, the query blocks of BN at or below the
//     diagonal streamed; S^T = K Q^T and dP^T = V dO^T, then dV += (P^T o keep) dO and dK += dS^T Q, accumulated in registers.
//   * DQ, per (sequence, head, 128-query tile): rows = queries; Q and dO resident, the causal key blocks of BN streamed;
//     S = Q K^T (the forward's operands and MMA order), dP = dO V^T, dQ += dS K.
// Every contraction runs on the 2 x fp16 split with three MMAs per K step.  Power-of-two scales, all derived on the device:
// q / k / v from max|qkv| (the forward's), dO from max|dctx|, P 2^14 (the forward's), dS from its bound
// |dS| <= 2 hd max|dO| max|qkv| / (1 - p).  A streamed [BN rows x HD channels] tile serves both as the K-major operand of the
// first pair of contractions and as the MN-major operand of the second: the planes [c/8][row][8 channels] are both layouts.
// HD 64: BN = 64.  HD 128: the resident tiles double, so BN = 32 keeps the shared memory at 197 KB, and a DKV CTA owns
// the dK / dV channels of one half (NSPLIT = 2, both CTAs of a key tile recompute S and dP) so that dK and dV stay at
// 64 accumulator registers a thread; DQ keeps all 128 channels of dQ (64 registers, no dV).
struct BwdParams {
  const float* qkv;     // [B, S, 3H]
  const float* dctx;    // [B, S, H]
  const float* stats;   // m [B, heads, S] then l [B, heads, S] (mas_attn_causal_forward_stats)
  const float* D;       // [B, heads, S] row dot products dO . ctx
  float* dqkv;          // [B, S, 3H]
  const float* amax;    // device scalar max|qkv|
  const float* amax_do; // device scalar max|dctx|
  int S, heads;
  float scale;
};

template <int HD>
__global__ void __launch_bounds__(256) attn_causal_bwd_rowdot(const float* __restrict__ dctx, const float* __restrict__ ctx,
                                                              float* __restrict__ D, int S, int heads, int64_t rows) {
  const int64_t r = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);      // row (b, q, h) of the [B S heads, HD] view
  if (r >= rows) return;
  const int lane = threadIdx.x & 31;
  float v;
  if constexpr (HD == 64) {
    const float2 a = reinterpret_cast<const float2*>(dctx + r * HD)[lane], c = reinterpret_cast<const float2*>(ctx + r * HD)[lane];
    v = a.x * c.x + a.y * c.y;
  } else {
    const float4 a = reinterpret_cast<const float4*>(dctx + r * HD)[lane], c = reinterpret_cast<const float4*>(ctx + r * HD)[lane];
    v = (a.x * c.x + a.y * c.y) + (a.z * c.z + a.w * c.w);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if (lane == 0) {
    const int64_t b = r / ((int64_t)S * heads), rem = r - b * S * heads;
    const int q = (int)(rem / heads), h = (int)(rem - (int64_t)q * heads);
    D[((size_t)b * heads + h) * S + q] = v;
  }
}

template <int HD, bool DKV, bool DROP>
__global__ void __launch_bounds__(NTHREADS, 1) attn_causal_bwd(const BwdParams p, const DropMask dm) {
  using C = Cfg<HD>;
  constexpr int BN = C::BN, PITCH_Q = C::PITCH_Q, Q_HALF = C::Q_HALF, TILE = 2 * Q_HALF, PITCH_C = C::PITCH_C;
  constexpr int C_HALF = C::C_HALF, B_HALF = C::B_HALF;
  constexpr int NSPLIT = DKV ? C::NSPLIT : 1, NOUT = HD / NSPLIT;   // output channels of this CTA
  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* r1 = smem;                         // resident 128 rows: K (DKV) / Q (DQ), hi + lo
  uint8_t* r2 = r1 + TILE;                    // resident: V / dO
  uint8_t* c1 = r2 + TILE;                    // streamed BN rows: Q / K
  uint8_t* c2 = c1 + 2 * C_HALF;              // streamed: dO / V
  uint8_t* ds_blk = c2 + 2 * C_HALF;          // dS block (A operand of dK / dQ)
  uint8_t* p_blk = ds_blk + 2 * B_HALF;       // DKV: the P o keep block (A operand of dV)
  const uint32_t r1_base = smem_u32(r1), r2_base = smem_u32(r2), c1_base = smem_u32(c1), c2_base = smem_u32(c2);
  const uint32_t ds_base = smem_u32(ds_blk), p_base = smem_u32(p_blk);

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wgi = warp >> 2, fk = lane & 3;
  const int S = p.S, heads = p.heads, H = heads * HD, C3 = 3 * H;
  const int t = DKV ? (int)blockIdx.x / NSPLIT : (int)gridDim.x - 1 - (int)blockIdx.x;   // heaviest tiles first
  const int part = DKV ? (int)blockIdx.x % NSPLIT : 0;                                    // DKV: output channels part * NOUT ..
  const int h = blockIdx.y, b = blockIdx.z;
  const int r0 = t * BM;
  const int cb0 = DKV ? r0 : 0, ncb = DKV ? (S - r0) / BN : (r0 + BM) / BN;    // causal column blocks
  const size_t bh = (size_t)b * heads + h;
  const float* qb = p.qkv + (size_t)b * S * C3 + h * HD;
  const float* ob = p.dctx + (size_t)b * S * H + h * HD;
  const float* mg = p.stats + bh * S;
  const float* lg = mg + (size_t)gridDim.z * heads * S;
  const float* dg = p.D + bh * S;
  const int frow = wgi * 64 + (warp & 3) * 16 + (lane >> 2);
  const uint32_t a_rows = (uint32_t)(wgi * 64 * 16);
  float inv_s, inv_do, inv_ds;
  const float sc = split_scale(p.amax, &inv_s);
  const float sdo = split_scale(p.amax_do, &inv_do);
  const float dsc = DROP ? dm.scale : 1.f;
  const float bound = 2.f * HD * *p.amax_do * *p.amax * dsc;
  const float sds = split_scale(&bound, &inv_ds);
  constexpr float P_SCALE = 16384.0f, P_INV = 1.0f / 16384.0f;
  const float ss = p.scale * inv_s * inv_s;                 // acc1 -> scale * q.k
  const float sdp = inv_s * inv_do;                          // acc2 -> dO . v

  // [ROWS x HD channels] fp32 rows of src (leading dimension ld) -> hi / lo images at dst, scaled by s
  auto fill = [&](auto rows_c, uint8_t* dst, const float* src, int ld, int row0, int pitch, int half, float s) {
    constexpr int N = decltype(rows_c)::value * (HD / 8) / NTHREADS, OCT_LOG = HD == 64 ? 3 : 4;
    float4 v0[N], v1[N];
#pragma unroll
    for (int i = 0; i < N; ++i) {
      const int itm = tid + i * NTHREADS, oct = itm & (HD / 8 - 1), r = itm >> OCT_LOG;
      const float4* g = reinterpret_cast<const float4*>(src + (size_t)(row0 + r) * ld + oct * 8);
      v0[i] = __ldg(g);
      v1[i] = __ldg(g + 1);
    }
#pragma unroll
    for (int i = 0; i < N; ++i) {
      const int itm = tid + i * NTHREADS, oct = itm & (HD / 8 - 1), r = itm >> OCT_LOG;
      uint4 hh, ll;
      split8(v0[i], v1[i], s, &hh, &ll);
      uint8_t* d = dst + oct * pitch + r * 16;
      *reinterpret_cast<uint4*>(d) = hh;
      *reinterpret_cast<uint4*>(d + half) = ll;
    }
  };
  using R128 = std::integral_constant<int, BM>;
  using RN = std::integral_constant<int, BN>;
  if constexpr (DKV) {
    fill(R128{}, r1, qb + H, C3, r0, PITCH_Q, Q_HALF, sc);
    fill(R128{}, r2, qb + 2 * H, C3, r0, PITCH_Q, Q_HALF, sc);
  } else {
    fill(R128{}, r1, qb, C3, r0, PITCH_Q, Q_HALF, sc);
    fill(R128{}, r2, ob, H, r0, PITCH_Q, Q_HALF, sdo);
  }

  // DQ: the statistics of this thread's two query rows
  float qm[2] = {0.f, 0.f}, qrl[2] = {0.f, 0.f}, qd[2] = {0.f, 0.f};
  if constexpr (!DKV) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int q = r0 + frow + 8 * i;
      qm[i] = mg[q];
      qrl[i] = 1.0f / lg[q];
      qd[i] = dg[q];
    }
  }
  float acc1[BN / 2], acc2[BN / 2], g1[NOUT / 2], g2[NOUT / 2];   // g1: dK / dQ, g2: dV
#pragma unroll
  for (int i = 0; i < NOUT / 2; ++i) g1[i] = g2[i] = 0.f;
  const uint64_t seed = DROP ? (uint64_t)*dm.seed : 0ull;
  const uint32_t out_planes = (uint32_t)(part * (NOUT / 8) * PITCH_C);     // this CTA's channels in a streamed tile

  for (int cbi = 0; cbi < ncb; ++cbi) {
    const int cb = cb0 + cbi * BN;
    __syncthreads();                                  // every MMA reading c1 / c2 / the blocks has retired (wait<0> below)
    if constexpr (DKV) {
      fill(RN{}, c1, qb, C3, cb, PITCH_C, C_HALF, sc);
      fill(RN{}, c2, ob, H, cb, PITCH_C, C_HALF, sdo);
    } else {
      fill(RN{}, c1, qb + H, C3, cb, PITCH_C, C_HALF, sc);
      fill(RN{}, c2, qb + 2 * H, C3, cb, PITCH_C, C_HALF, sc);
    }
    fence_proxy_async();
    __syncthreads();
    // ---- acc1 = R1 C1^T (scores), acc2 = R2 C2^T (dP) ----
    wg::fence();
#pragma unroll
    for (int k16 = 0; k16 < HD / 16; ++k16) {
      const uint32_t ao = a_rows + (uint32_t)(k16 * 2 * PITCH_Q), bo = (uint32_t)(k16 * 2 * PITCH_C);
      const uint64_t ah = wg::desc(r1_base + ao, PITCH_Q, 128), al = wg::desc(r1_base + Q_HALF + ao, PITCH_Q, 128);
      const uint64_t bh_ = wg::desc(c1_base + bo, PITCH_C, 128), bl = wg::desc(c1_base + C_HALF + bo, PITCH_C, 128);
      mma<BN, 0>(acc1, ah, bh_, k16 > 0 ? 1u : 0u);
      mma<BN, 0>(acc1, al, bh_, 1u);
      mma<BN, 0>(acc1, ah, bl, 1u);
      const uint64_t dh = wg::desc(r2_base + ao, PITCH_Q, 128), dl = wg::desc(r2_base + Q_HALF + ao, PITCH_Q, 128);
      const uint64_t eh = wg::desc(c2_base + bo, PITCH_C, 128), el = wg::desc(c2_base + C_HALF + bo, PITCH_C, 128);
      mma<BN, 0>(acc2, dh, eh, k16 > 0 ? 1u : 0u);
      mma<BN, 0>(acc2, dl, eh, 1u);
      mma<BN, 0>(acc2, dh, el, 1u);
    }
    wg::commit();
    wg::wait<0>();
    wg::fence_regs<BN / 2>(acc1);
    wg::fence_regs<BN / 2>(acc2);

    // keep bits: bit 2 j + c of keep[i] <-> element (row frow + 8 i, column 8 j + 2 fk + c) of this block
    uint32_t keep[2] = {0u, 0u};
    if constexpr (DROP) {
      if constexpr (DKV) {
        // rows are keys: the four lanes (lane >> 2) & 3 = 0..3 hold the four keys of one Philox group for every column;
        // lane u of the four generates the groups of the combinations 4 n + u of (i, j, c) and hands them round
        constexpr int NC = BN / 2;                      // combinations: 2 rows x BN / 8 column groups x 2
        const int u = (lane >> 2) & 3;
        const uint64_t key4 = (uint64_t)(r0 + (frow & ~3));
        uint32_t gen[NC / 4];
#pragma unroll
        for (int n = 0; n < NC / 4; ++n) {
          const int ic = 4 * n + u, i = ic / (BN / 4), j = (ic >> 1) % (BN / 8), c = ic & 1;
          const uint64_t q = (uint64_t)(cb + 8 * j + 2 * fk + c);
          gen[n] = keep_bits4(seed, ((bh * S + q) * S + key4 + 8 * i) >> 2, dm.t);
        }
#pragma unroll
        for (int ic = 0; ic < NC; ++ic) {
          const uint32_t w = __shfl_sync(0xffffffffu, gen[ic >> 2], (lane & ~12) | ((ic & 3) << 2));
          keep[ic / (BN / 4)] |= ((w >> u) & 1u) << (ic % (BN / 4));
        }
      } else {
        const uint64_t row0 = (bh * S + r0 + frow + 8 * (fk & 1)) * S + cb + 4 * (fk >> 1);
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
          const uint32_t bits = keep_bits4(seed, (row0 + 8 * j) >> 2, dm.t);
          const uint32_t b0 = __shfl_sync(0xffffffffu, bits, lane & ~1), b1 = __shfl_sync(0xffffffffu, bits, lane | 1);
          keep[0] |= ((b0 >> (2 * (fk & 1))) & 3u) << (2 * j);
          keep[1] |= ((b1 >> (2 * (fk & 1))) & 3u) << (2 * j);
        }
      }
    }
    // ---- P (the forward's pass-1 expression), dS; split into the A-operand blocks ----
#pragma unroll
    for (int j = 0; j < BN / 8; ++j) {
      float cm[2], crl[2], cd[2];
      if constexpr (DKV) {                          // columns are queries: their statistics
        const int q = cb + 8 * j + 2 * fk;
        const float2 m2 = *reinterpret_cast<const float2*>(mg + q), l2 = *reinterpret_cast<const float2*>(lg + q);
        const float2 d2 = *reinterpret_cast<const float2*>(dg + q);
        cm[0] = m2.x; cm[1] = m2.y; crl[0] = 1.0f / l2.x; crl[1] = 1.0f / l2.y; cd[0] = d2.x; cd[1] = d2.y;
      }
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int rit = frow + 8 * i;
        float dv[2], pk[2];
#pragma unroll
        for (int c = 0; c < 2; ++c) {
          const int row = r0 + rit, col = cb + 8 * j + 2 * fk + c;
          const int q = DKV ? col : row, key = DKV ? row : col;
          const float m_ = DKV ? cm[c] : qm[i], rl_ = DKV ? crl[c] : qrl[i], d_ = DKV ? cd[c] : qd[i];
          const int e = 4 * j + 2 * i + c;
          const float pr = key > q ? 0.f : expf(acc1[e] * ss - m_) * rl_;
          const bool kept = !DROP || ((keep[i] >> (2 * j + c)) & 1u);
          const float g = kept ? acc2[e] * sdp * dsc : 0.f;
          pk[c] = kept ? pr : 0.f;
          dv[c] = pr * (g - d_);
        }
        uint32_t hi, lo;
        split2(dv[0], dv[1], sds, &hi, &lo);
        uint8_t* d = ds_blk + (size_t)j * PITCH_P + rit * 16 + fk * 4;
        *reinterpret_cast<uint32_t*>(d) = hi;
        *reinterpret_cast<uint32_t*>(d + B_HALF) = lo;
        if constexpr (DKV) {
          split2(pk[0], pk[1], P_SCALE, &hi, &lo);
          uint8_t* e = p_blk + (size_t)j * PITCH_P + rit * 16 + fk * 4;
          *reinterpret_cast<uint32_t*>(e) = hi;
          *reinterpret_cast<uint32_t*>(e + B_HALF) = lo;
        }
      }
    }
    fence_proxy_async();
    __syncthreads();
    // ---- DKV: dK += dS^T Q, dV += (P o keep)^T dO; DQ: dQ += dS K (B operands MN-major from the streamed tiles) ----
    wg::fence();
#pragma unroll
    for (int k16 = 0; k16 < BN / 16; ++k16) {
      const uint32_t ao = a_rows + (uint32_t)(k16 * 2 * PITCH_P), bo = out_planes + (uint32_t)(k16 * 256);
      const uint64_t sh = wg::desc(ds_base + ao, PITCH_P, 128), sl = wg::desc(ds_base + B_HALF + ao, PITCH_P, 128);
      const uint64_t xh = wg::desc(c1_base + bo, 128, PITCH_C), xl = wg::desc(c1_base + C_HALF + bo, 128, PITCH_C);
      mma<NOUT, 1>(g1, sh, xh, 1u);
      mma<NOUT, 1>(g1, sl, xh, 1u);
      mma<NOUT, 1>(g1, sh, xl, 1u);
      if constexpr (DKV) {
        const uint64_t ph = wg::desc(p_base + ao, PITCH_P, 128), pl = wg::desc(p_base + B_HALF + ao, PITCH_P, 128);
        const uint64_t oh = wg::desc(c2_base + bo, 128, PITCH_C), ol = wg::desc(c2_base + C_HALF + bo, 128, PITCH_C);
        mma<NOUT, 1>(g2, ph, oh, 1u);
        mma<NOUT, 1>(g2, pl, oh, 1u);
        mma<NOUT, 1>(g2, ph, ol, 1u);
      }
    }
    wg::commit();
    wg::wait<0>();
    wg::fence_regs<NOUT / 2>(g1);
    if constexpr (DKV) wg::fence_regs<NOUT / 2>(g2);
  }
  // ---- epilogue: straight from the fragments into the fused [B, S, 3H] gradient ----
  const float s1 = inv_ds * inv_s * p.scale, s2 = P_INV * inv_do * dsc;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    float* orow = p.dqkv + ((size_t)b * S + r0 + frow + 8 * i) * C3 + h * HD + part * NOUT + 2 * fk;
#pragma unroll
    for (int j = 0; j < NOUT / 8; ++j) {
      if constexpr (DKV) {
        *reinterpret_cast<float2*>(orow + H + 8 * j) = make_float2(g1[4 * j + 2 * i] * s1, g1[4 * j + 2 * i + 1] * s1);
        *reinterpret_cast<float2*>(orow + 2 * H + 8 * j) = make_float2(g2[4 * j + 2 * i] * s2, g2[4 * j + 2 * i + 1] * s2);
      } else {
        *reinterpret_cast<float2*>(orow + 8 * j) = make_float2(g1[4 * j + 2 * i] * s1, g1[4 * j + 2 * i + 1] * s1);
      }
    }
  }
}

}  // namespace attnc

bool attn_causal_fused_ok(int S, int heads, int hd) { return (hd == 64 || hd == 128) && S % attnc::BM == 0 && S >= attnc::BM && heads > 0; }

}  // namespace mas

using namespace mas;

template <int HD, bool DROP, bool STATS, bool PREFIX = false>
static int attn_causal_launch_hd(const attnc::Params& p, const DropMask& dm, int B, void* stream) {
  static std::atomic<uint64_t> configured{0};
  constexpr size_t smem = attnc::Cfg<HD>::SMEM_BYTES;
  if (first_on_device(configured)) {
    cudaError_t e = cudaFuncSetAttribute(attnc::attn_causal_fwd<HD, DROP, STATS, PREFIX>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return fail(MAS_ERR_LAUNCH, "attn_causal_fwd: smem attr: %s", cudaGetErrorString(e));
    mark_device(configured);
  }
  const dim3 grid((unsigned)(p.S / attnc::BM), (unsigned)p.heads, (unsigned)B);
  attnc::attn_causal_fwd<HD, DROP, STATS, PREFIX><<<grid, attnc::NTHREADS, smem, mas::S(stream)>>>(p, dm);
  if (PREFIX) return launched_tc(HD == 128 ? "attn_causal_prefix_fwd<128>" : "attn_causal_prefix_fwd");
  if (HD == 128)
    return launched_tc(STATS ? (DROP ? "attn_causal_dropout_fwd_stats<128>" : "attn_causal_fwd_stats<128>")
                             : (DROP ? "attn_causal_dropout_fwd<128>" : "attn_causal_fwd<128>"));
  return launched_tc(STATS ? (DROP ? "attn_causal_dropout_fwd_stats" : "attn_causal_fwd_stats")
                           : (DROP ? "attn_causal_dropout_fwd" : "attn_causal_fwd"));
}

template <bool DROP, bool STATS = false>
static int attn_causal_launch(const float* qkv, const float* amax, float* P, float* ctx, int B, int S, int heads, int hd, float scale,
                              const DropMask& dm, void* stream) {
  MAS_REQUIRE(qkv && amax && P && ctx && B > 0, "attn_causal_forward: bad arguments");
  if (!attn_causal_fused_ok(S, heads, hd))
    return fail(MAS_ERR_UNSUPPORTED, "attn_causal_forward: needs head dim 64 or 128 and S %% 128 == 0 (got S=%d, hd=%d)", S, hd);
  if (heads > 65535 || B > 65535) return fail(MAS_ERR_UNSUPPORTED, "attn_causal_forward: heads / batch beyond the grid limits");
  attnc::Params p;
  p.qkv = qkv; p.P = P; p.ctx = ctx; p.amax = amax; p.S = S; p.heads = heads; p.scale = scale;
  p.qkvp = nullptr; p.Lp = 0; p.n = 1;
  return hd == 64 ? attn_causal_launch_hd<64, DROP, STATS>(p, dm, B, stream) : attn_causal_launch_hd<128, DROP, STATS>(p, dm, B, stream);
}

extern "C" int mas_attn_causal_forward(const float* qkv, const float* amax, float* P, float* ctx, int B, int S, int heads, int hd,
                                       float scale, void* stream) {
  return attn_causal_launch<false>(qkv, amax, P, ctx, B, S, heads, hd, scale, DropMask{nullptr, 0, 1.f}, stream);
}

extern "C" int mas_attn_causal_dropout_forward(const float* qkv, const float* amax, float* P, float* ctx, int B, int S, int heads,
                                               int hd, float scale, double p, const int64_t* seed, void* stream) {
  MAS_REQUIRE(seed && p >= 0.0 && p <= 1.0, "attn_causal_dropout_forward: bad dropout arguments");
  return attn_causal_launch<true>(qkv, amax, P, ctx, B, S, heads, hd, scale, DropMask{seed, drop_threshold(p), drop_scale(p)}, stream);
}

extern "C" int mas_attn_causal_forward_stats(const float* qkv, const float* amax, float* stats, float* ctx, int B, int S, int heads,
                                             int hd, float scale, double p, const int64_t* seed, void* stream) {
  MAS_REQUIRE(p >= 0.0 && p <= 1.0 && (p == 0.0 || seed), "attn_causal_forward_stats: bad dropout arguments");
  if (p > 0.0)
    return attn_causal_launch<true, true>(qkv, amax, stats, ctx, B, S, heads, hd, scale,
                                          DropMask{seed, drop_threshold(p), drop_scale(p)}, stream);
  return attn_causal_launch<false, true>(qkv, amax, stats, ctx, B, S, heads, hd, scale, DropMask{nullptr, 0, 1.f}, stream);
}

extern "C" int mas_attn_causal_prefix_forward(const float* qkv_prefix, const float* qkv, const float* amax, float* ctx, int P, int n,
                                              int Lp, int L, int heads, int hd, float scale, void* stream) {
  MAS_REQUIRE(qkv_prefix && qkv && amax && ctx && P > 0 && n > 0, "attn_causal_prefix_forward: bad arguments");
  if (!(hd == 64 || hd == 128) || heads <= 0 || Lp <= 0 || L <= 0 || Lp % attnc::BM || L % attnc::BM)
    return fail(MAS_ERR_UNSUPPORTED, "attn_causal_prefix_forward: needs head dim 64 or 128, Lp %% 128 == 0 and L %% 128 == 0 "
                "(got Lp=%d, L=%d, hd=%d)", Lp, L, hd);
  if (heads > 65535 || (int64_t)P * n > 65535)
    return fail(MAS_ERR_UNSUPPORTED, "attn_causal_prefix_forward: heads / rows beyond the grid limits");
  attnc::Params p;
  p.qkv = qkv; p.P = nullptr; p.ctx = ctx; p.amax = amax; p.S = L; p.heads = heads; p.scale = scale;
  p.qkvp = qkv_prefix; p.Lp = Lp; p.n = n;
  const DropMask dm{nullptr, 0, 1.f};
  return hd == 64 ? attn_causal_launch_hd<64, false, false, true>(p, dm, P * n, stream)
                  : attn_causal_launch_hd<128, false, false, true>(p, dm, P * n, stream);
}

template <int HD, bool DKV, bool DROP>
static int attn_causal_bwd_launch(const attnc::BwdParams& p, const DropMask& dm, int B, void* stream) {
  static std::atomic<uint64_t> configured{0};
  constexpr size_t smem = attnc::Cfg<HD>::BWD_SMEM_BYTES;
  if (first_on_device(configured)) {
    cudaError_t e = cudaFuncSetAttribute(attnc::attn_causal_bwd<HD, DKV, DROP>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return fail(MAS_ERR_LAUNCH, "attn_causal_bwd: smem attr: %s", cudaGetErrorString(e));
    mark_device(configured);
  }
  const dim3 grid((unsigned)(p.S / attnc::BM * (DKV ? attnc::Cfg<HD>::NSPLIT : 1)), (unsigned)p.heads, (unsigned)B);
  attnc::attn_causal_bwd<HD, DKV, DROP><<<grid, attnc::NTHREADS, smem, mas::S(stream)>>>(p, dm);
  if (HD == 128)
    return launched_tc(DKV ? (DROP ? "attn_causal_dropout_bwd_dkv<128>" : "attn_causal_bwd_dkv<128>")
                           : (DROP ? "attn_causal_dropout_bwd_dq<128>" : "attn_causal_bwd_dq<128>"));
  return launched_tc(DKV ? (DROP ? "attn_causal_dropout_bwd_dkv" : "attn_causal_bwd_dkv")
                         : (DROP ? "attn_causal_dropout_bwd_dq" : "attn_causal_bwd_dq"));
}

template <int HD>
static int attn_causal_bwd_hd(const attnc::BwdParams& bp, const float* ctx, double p, const int64_t* seed, int B, void* stream) {
  const int64_t rows = (int64_t)B * bp.S * bp.heads;
  attnc::attn_causal_bwd_rowdot<HD><<<(unsigned)((rows + 7) / 8), 256, 0, mas::S(stream)>>>(bp.dctx, ctx, const_cast<float*>(bp.D),
                                                                                           bp.S, bp.heads, rows);
  int rc = launched_tc(HD == 128 ? "attn_causal_bwd_rowdot<128>" : "attn_causal_bwd_rowdot");
  if (rc != MAS_OK) return rc;
  if (p > 0.0) {
    const DropMask dm{seed, drop_threshold(p), drop_scale(p)};
    rc = attn_causal_bwd_launch<HD, true, true>(bp, dm, B, stream);
    return rc != MAS_OK ? rc : attn_causal_bwd_launch<HD, false, true>(bp, dm, B, stream);
  }
  const DropMask dm{nullptr, 0, 1.f};
  rc = attn_causal_bwd_launch<HD, true, false>(bp, dm, B, stream);
  return rc != MAS_OK ? rc : attn_causal_bwd_launch<HD, false, false>(bp, dm, B, stream);
}

extern "C" int mas_attn_causal_backward(const float* qkv, const float* ctx, const float* dctx, const float* stats, const float* amax,
                                        const float* dctx_amax, float* D, float* dqkv, int B, int S, int heads, int hd, float scale,
                                        double p, const int64_t* seed, void* stream) {
  MAS_REQUIRE(qkv && ctx && dctx && stats && amax && dctx_amax && D && dqkv && B > 0, "attn_causal_backward: bad arguments");
  MAS_REQUIRE(p >= 0.0 && p <= 1.0 && (p == 0.0 || seed), "attn_causal_backward: bad dropout arguments");
  if (!attn_causal_fused_ok(S, heads, hd))
    return fail(MAS_ERR_UNSUPPORTED, "attn_causal_backward: needs head dim 64 or 128 and S %% 128 == 0 (got S=%d, hd=%d)", S, hd);
  if (heads > 65535 || B > 65535) return fail(MAS_ERR_UNSUPPORTED, "attn_causal_backward: heads / batch beyond the grid limits");
  attnc::BwdParams bp;
  bp.qkv = qkv; bp.dctx = dctx; bp.stats = stats; bp.D = D; bp.dqkv = dqkv; bp.amax = amax; bp.amax_do = dctx_amax;
  bp.S = S; bp.heads = heads; bp.scale = scale;
  return hd == 64 ? attn_causal_bwd_hd<64>(bp, ctx, p, seed, B, stream) : attn_causal_bwd_hd<128>(bp, ctx, p, seed, B, stream);
}
