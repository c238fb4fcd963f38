// Hopper tensor-core (wgmma) contraction kernels for sm_90a: fp16 operands (3x3 family; same 11-bit significand as TF32,
// power-of-two operand scales derived on the device) or TF32 operands (1x1 row GEMM, A/B switch), fp32 accumulation in registers.
//
//   conv3x3 family / row GEMM as a "shift-GEMM":
//     D[m, n] = sum_{tap} sum_{k} A[slot(m) + shift(tap), k] * B_tap[n, k]
//   * M tile  = 128 output pixels arranged as 16 rows x 8 columns of the image, so that the eight rows of a
//     UMMA core-matrix group are eight horizontally adjacent pixels (16 B apart in the staged operand) and the
//     group stride (SBO) is the pitch of one staged image row.  The 3x3 taps are then NINE MMAs over the SAME
//     staged halo (18 x 10 pixels): only the descriptor start address moves by (ty*10+tx)*16 B.  The input is
//     staged once per K chunk instead of nine times (no im2col, in memory or in shared memory).
//   * A operand: staged by 256 producer threads (generic loads -> convert -> st.shared, K-major "interleaved" no-swizzle
//     layout [k/8][slot][8 halves] | [k/4][slot][4 floats]) so that upsample (x2 nearest), zero-stuffing (stride-2 data
//     gradient) and the GroupNorm+SiLU prologue are just a different slot->pixel map / register transform.
//   * B operand (weights): pre-packed in global memory in the exact shared-memory image and pulled in with ONE
//     cp.async.bulk (TMA bulk copy, mbarrier complete_tx) per stage.
//   * one CTA per SM, two M tiles (256 pixels) and a 2-stage ring: warps 0-7 (two warpgroups) stage A, then each issues the
//     wgmma of its 64 rows of both tiles and runs the epilogue (registers -> shared-memory image -> bias / residual / GroupNorm
//     statistics -> global); the last warpgroup issues the weight bulk copies; full/empty mbarrier ring.
//   * wgrad_tc: the weight gradient (K = pixels): dy through TMA -> the wgmma A register fragment, the activation halo as an
//     MN-major fp16 operand (untransposed) or a transposed TF32 one.
//
// Reference call sites replaced: nn.Conv2d 3x3 (modules.py:93-104), Upsample/Downsample data paths
// (modules.py:55-59,74-78), nn.Conv2d 1x1 (modules.py:113-117,145-164).
#include <cuda.h>
#include <cudaTypedefs.h>
#include <cuda_fp16.h>
#include <stdlib.h>

#include "mas_common.cuh"
#include "tc_ptx.cuh"
#include "wgmma.cuh"

namespace mas {
namespace tc {

constexpr int NPROD = 256;     // producer threads (warps 0-7)
constexpr int NTHREADS = 384;  // + the bulk-copy warpgroup (one issuing thread; its registers go to the producers)
constexpr int STAGES_CONV = 3;

enum { MAP_S1 = 0, MAP_UP = 2, MAP_ZS = 3, MAP_ROWS = 4 };

struct Params {
  const float* x;    // NHWC input (dense) or row matrix
  const float* wpk;  // packed weights [n_tile][k_chunk][tap][k/4][BN][4]
  const float* bias; // [Cout] or null
  const float* res;  // same layout as y, or null
  float* y;
  int N, Hin, Win, Cin, Hout, Wout, Cout;  // for MAP_ROWS: Hout*Wout*N = rows, Win unused
  int map;
  int64_t ldx, ldy;  // row pitches (elements) of x pixels and y pixels
  int tiles_x, tiles_y;  // tiles per image row / column (image maps)
  int64_t total_tiles;
  float alpha;
  // fused GroupNorm(+SiLU) PROLOGUE on the A operand: a = act(x * sc + sh) with (sc, sh) per (image, input channel) in
  // gn_table [N][Cin][2] (null = plain input).  Padding pixels stay exactly zero (the reference pads the ACTIVATED tensor).
  const float* gn_table;
  int gn_silu;
  // fused GroupNorm-statistics EPILOGUE for the NEXT layer's norm: per (tile, 32-row lane group, channel quad) sum and
  // sum of squares of the stored output, [total_tiles][4][Cout/4][2] floats (null = off); reduced deterministically
  // per (image, group) by mas_gn_finalize_partials.
  float* stats_part;
  // fp16-operand kernels: largest magnitude of x (device scalar) for the power-of-two operand scale, or null (no scaling:
  // activations / weights sit well inside the fp16 range; gradients do not)
  const float* x_amax;
  // output channels actually present in y (pitch ldy): Cout is rounded up to the 128-wide tile, channels >= Cstore are computed
  // from zero weight rows and never stored (the 159-channel VQ-SEG decoder head runs as 2 x 128)
  int Cstore;
};

// One CTA = TILES M-tiles x BN output channels, full K.
// F16 = false: TF32 operands (fp32 words, 4 channels per 16-byte chunk, K = 8 per MMA).
// F16 = true : fp16 operands converted by the producers (8 channels per 16-byte chunk, K = 16 per MMA); KC still counts channels.
template <int TAPS, int KC, int STAGES, int TILES, bool F16>
__global__ void __launch_bounds__(NTHREADS, 1) shift_gemm_tc(const Params p) {
  constexpr int EPC = F16 ? 8 : 4;                      // channels per 16-byte operand chunk
  constexpr int SLOTS = (TAPS == 9) ? 180 : 132;        // staged pixels per tile (18x10 halo | 128 rows + pad)
  constexpr int ROWP = (TAPS == 9) ? 10 : 8;            // staged pixels per image row
  constexpr int LBO_A = SLOTS * 16;                     // bytes between k-chunks of A
  constexpr int SBO_A = ROWP * 16;                      // bytes between 8-pixel groups of A
  constexpr int A_TILE = (KC / EPC) * LBO_A;            // bytes per tile per stage
  constexpr int A_STAGE = TILES * A_TILE;
  constexpr int LBO_B = BN * 16;
  constexpr int B_TAP = (KC / EPC) * LBO_B;
  constexpr int B_STAGE = TAPS * B_TAP;
  constexpr int STAGE = A_STAGE + B_STAGE;
  constexpr int QUADS = KC / EPC;
  constexpr int ITEMS = TILES * SLOTS * QUADS;          // 16-byte operand chunks staged per K chunk
  constexpr int LPI = F16 ? 2 : 1;                      // float4 global loads per staged chunk
  constexpr int PER_THREAD = (ITEMS + NPROD - 1) / NPROD;
  constexpr int ACC_LD = BN + 4;                        // floats per row of the staged accumulator image
  static_assert((SLOTS % 8) == 4, "A plane pitch must be 64 mod 128 bytes for conflict-free producer stores");
  static_assert(BM * ACC_LD * 4 <= STAGES * STAGE, "one tile's accumulators are staged in the idle operand ring");

  extern __shared__ __align__(1024) uint8_t smem[];
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + (size_t)STAGES * STAGE);
  // bars[0..S) full, bars[S..2S) empty
  const uint32_t smem_base = smem_u32(smem);
  const uint32_t bar_base = smem_u32(bars);
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (STAGES + s); };

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int64_t tile0 = (int64_t)blockIdx.x * TILES;
  const int n0 = blockIdx.y * BN;
  const int nchunks = p.Cin / KC;

  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full_bar(s), NPROD + 1);
      mbar_init(empty_bar(s), NPROD);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 8) {
    // ===================== producers: stage A (input pixels) =====================
    wg::regs_inc<wg::MMA_REGS>();
    const float* src[PER_THREAD];
    const float* tab[(TAPS == 9) ? PER_THREAD : 1];   // prologue table pointers (3x3 convolutions only)
    uint32_t dst[PER_THREAD];
#pragma unroll
    for (int i = 0; i < PER_THREAD; ++i) {
      const int item = tid + i * NPROD;
      src[i] = nullptr;
      if (TAPS == 9) tab[i] = nullptr;
      dst[i] = 0xFFFFFFFFu;
      if (item < ITEMS) {
        const int q = item % QUADS, rest = item / QUADS, slot = rest % SLOTS, tl = rest / SLOTS;
        dst[i] = (uint32_t)(tl * A_TILE + q * LBO_A + slot * 16);
        const int64_t tile = tile0 + tl;
        if (tile < p.total_tiles) {
          if (TAPS == 9) {
            const int tx_ = (int)(tile % p.tiles_x), ty_ = (int)((tile / p.tiles_x) % p.tiles_y);
            const int n = (int)(tile / ((int64_t)p.tiles_x * p.tiles_y));
            const int r = slot / 10, c = slot % 10;
            const int vy = ty_ * 16 - 1 + r, vx = tx_ * 8 - 1 + c;  // coordinates in the (virtual) conv input image
            int iy = vy, ix = vx;
            bool ok;
            if (p.map == MAP_S1) {
              ok = (unsigned)vy < (unsigned)p.Hin && (unsigned)vx < (unsigned)p.Win;
            } else if (p.map == MAP_UP) {
              ok = (unsigned)vy < (unsigned)(2 * p.Hin) && (unsigned)vx < (unsigned)(2 * p.Win);
              iy = vy >> 1; ix = vx >> 1;
            } else {  // MAP_ZS
              ok = vy >= 0 && vx >= 0 && (vy & 1) && (vx & 1) && (vy >> 1) < p.Hin && (vx >> 1) < p.Win;
              iy = vy >> 1; ix = vx >> 1;
            }
            if (ok) {
              src[i] = p.x + ((int64_t)(n * p.Hin + iy) * p.Win + ix) * p.ldx + q * EPC;
              if (p.gn_table) tab[i] = p.gn_table + ((size_t)n * p.Cin + q * EPC) * 2;
            }
          } else {
            const int64_t row = tile * BM + slot;
            if (slot >= BM) dst[i] = 0xFFFFFFFFu;  // pad slots are never read by the MMA
            else if (row < (int64_t)p.N * p.Hout * p.Wout) src[i] = p.x + row * p.ldx + q * EPC;
          }
        }
      }
    }
    const int wgi = warp >> 2;             // warpgroup: accumulator rows 64 wgi .. 64 wgi + 63 of each tile
    float acc[TILES][BN / 2];
#pragma unroll
    for (int tl = 0; tl < TILES; ++tl)
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[tl][i] = 0.f;
    int stage = 0, prev = 0;
    uint32_t phase = 0;
    float inv_scale = 1.f;
    const float in_scale = F16 ? operand_scale(p.x_amax, &inv_scale) : 1.f;
    // Two register sets (va, vb) hold the global loads of alternate K chunks: a set is re-issued (for chunk kc + 2) right
    // after it has been converted and stored, so every load has TWO stage times to land instead of one - the kernel was
    // bound by exactly that latency (ncu: long-scoreboard stalls of the producers, tensor pipe 43 % active).
    float4 va[PER_THREAD][LPI], vb[PER_THREAD][LPI];
    auto gload = [&](int kc, float4 (*v)[LPI]) {
#pragma unroll
      for (int i = 0; i < PER_THREAD; ++i) {
#pragma unroll
        for (int h = 0; h < LPI; ++h) {
          v[i][h] = make_float4(0.f, 0.f, 0.f, 0.f);
          if (src[i]) v[i][h] = ldg_l2pf(reinterpret_cast<const float4*>(src[i] + (size_t)kc * KC) + h);
        }
      }
    };
    auto consume = [&](int kc, float4 (*v)[LPI]) {
      if (TAPS == 9) {
        if (p.gn_table) {
          // fused GroupNorm (+SiLU) prologue, applied at CONSUME time so the prefetches stay asynchronous;
          // the (scale, shift) pairs are L1-resident
#pragma unroll
          for (int i = 0; i < PER_THREAD; ++i) {
            if (tab[i]) {
#pragma unroll
              for (int h = 0; h < LPI; ++h) {
                const float4* tp = reinterpret_cast<const float4*>(tab[i] + (size_t)kc * KC * 2) + 2 * h;
                const float4 t0 = __ldg(tp);      // sc0 sh0 sc1 sh1
                const float4 t1 = __ldg(tp + 1);  // sc2 sh2 sc3 sh3
                float a0 = fmaf(v[i][h].x, t0.x, t0.y), a1 = fmaf(v[i][h].y, t0.z, t0.w);
                float a2 = fmaf(v[i][h].z, t1.x, t1.y), a3 = fmaf(v[i][h].w, t1.z, t1.w);
                if (p.gn_silu) { a0 = silu_f(a0); a1 = silu_f(a1); a2 = silu_f(a2); a3 = silu_f(a3); }
                v[i][h] = make_float4(a0, a1, a2, a3);
              }
            }
          }
        }
      }
      mbar_wait(empty_bar(stage), phase ^ 1);
      uint8_t* a_st = smem + (size_t)stage * STAGE;
#pragma unroll
      for (int i = 0; i < PER_THREAD; ++i) {
        if (dst[i] != 0xFFFFFFFFu) {
          if (F16) {
            const float4 lo = v[i][0], hi = v[i][LPI - 1];
            *reinterpret_cast<uint4*>(a_st + dst[i]) =
                make_uint4(pack_h2(lo.x * in_scale, lo.y * in_scale), pack_h2(lo.z * in_scale, lo.w * in_scale),
                           pack_h2(hi.x * in_scale, hi.y * in_scale), pack_h2(hi.z * in_scale, hi.w * in_scale));
          } else {
            *reinterpret_cast<float4*>(a_st + dst[i]) = v[i][0];
          }
        }
      }
      fence_proxy_async();  // make the generic-proxy stores visible to the tensor core (async proxy)
      mbar_arrive(full_bar(stage));
      // every producer's stores and the weight copy have landed: this warpgroup's MMAs over the stage
      mbar_wait(full_bar(stage), phase);
      const uint32_t st = smem_base + (uint32_t)stage * STAGE;
      const uint64_t a_base = wg::desc(st + (uint32_t)(wgi * 8 * SBO_A), LBO_A, SBO_A);
      const uint64_t b_base = wg::desc(st + A_STAGE, LBO_B, 128);
      wg::fence();
#pragma unroll
      for (int tl = 0; tl < TILES; ++tl) {
#pragma unroll
        for (int t = 0; t < TAPS; ++t) {
          const uint32_t tapoff = (TAPS == 9) ? (uint32_t)(((t / 3) * 10 + (t % 3)) * 16) : 0u;
#pragma unroll
          for (int k8 = 0; k8 < KC / (2 * EPC); ++k8) {   // one MMA = two 16-byte chunks of K (8 tf32 | 16 fp16)
            const uint64_t ad = a_base + (uint64_t)((tl * A_TILE + tapoff + k8 * 2 * LBO_A) >> 4);
            const uint64_t bd = b_base + (uint64_t)((t * B_TAP + k8 * 2 * LBO_B) >> 4);
            if (F16) wg::wgmma_f16_ss_n128<0, 0>(acc[tl], ad, bd, 1u);
            else wg::wgmma_tf32_ss_n128(acc[tl], ad, bd, 1u);
          }
        }
      }
      wg::commit();
      // the MMAs of the previous chunk have read their stage: release it to the producers and the weight copy
      wg::wait<1>();
      if (kc > 0) mbar_arrive(empty_bar(prev));
      prev = stage;
      if (++stage == STAGES) { stage = 0; phase ^= 1; }
    };
    gload(0, va);
    if (nchunks > 1) gload(1, vb);
    for (int kc = 0; kc < nchunks; kc += 2) {
      consume(kc, va);
      if (kc + 2 < nchunks) gload(kc + 2, va);
      if (kc + 1 < nchunks) {
        consume(kc + 1, vb);
        if (kc + 3 < nchunks) gload(kc + 3, vb);
      }
    }
    wg::wait<0>();
#pragma unroll
    for (int tl = 0; tl < TILES; ++tl) wg::fence_regs<BN / 2>(acc[tl]);
    const float alpha = p.alpha * inv_scale;

    // ===================== epilogue: registers -> shared-memory accumulator image -> coalesced global stores =====================
    // The fragment of a thread is scattered over 16 rows; the tile is staged as a [128][BN] image in the (now idle) operand
    // ring so that each warp can then read a 32-row x 32-channel block with 8 lanes per pixel row: 4 lines per store
    // instruction, and the residual is read the same way.
    const int lane_grp = warp & 3;           // accumulator rows [32*lane_grp, +32)
    const int chalf = warp >> 2;             // column half of the 128-wide tile
    float* img = reinterpret_cast<float*>(smem);
    const int sub_r = lane >> 3, sub_c = lane & 7;
    const int frow = wgi * 64 + (warp & 3) * 16 + (lane >> 2), fcol = 2 * (lane & 3);
#pragma unroll
    for (int tl = 0; tl < TILES; ++tl) {
      const int64_t tile = tile0 + tl;
      if (tile >= p.total_tiles) break;     // block-uniform
      wg::bar_sync(1, NPROD);               // the previous tile's image has been read (first tile: every MMA has completed)
#pragma unroll
      for (int j = 0; j < BN / 8; ++j)
#pragma unroll
        for (int i = 0; i < 2; ++i)
          *reinterpret_cast<float2*>(img + (frow + 8 * i) * ACC_LD + 8 * j + fcol) =
              make_float2(acc[tl][4 * j + 2 * i] * alpha, acc[tl][4 * j + 2 * i + 1] * alpha);
      wg::bar_sync(1, NPROD);
      int64_t pix_base = 0;                 // pixel index of accumulator row 0 of this tile (image maps: per-row formula)
      int tx_ = 0, ty_ = 0, n_img = 0;
      if (TAPS == 9) {
        tx_ = (int)(tile % p.tiles_x); ty_ = (int)((tile / p.tiles_x) % p.tiles_y);
        n_img = (int)(tile / ((int64_t)p.tiles_x * p.tiles_y));
      } else {
        pix_base = tile * BM;
      }
#pragma unroll 1
      for (int cc = 0; cc < 2; ++cc) {
        const int col = chalf * 64 + cc * 32;
        float4 bq = make_float4(0.f, 0.f, 0.f, 0.f);
        if (p.bias) bq = __ldg(reinterpret_cast<const float4*>(p.bias + n0 + col + sub_c * 4));
        float st_s = 0.f, st_q = 0.f;
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          const int row = i * 4 + sub_r;               // accumulator row within this warp's 32
          const int m = lane_grp * 32 + row;
          int64_t pix;
          if (TAPS == 9) pix = ((int64_t)n_img * p.Hout + ty_ * 16 + (m >> 3)) * p.Wout + tx_ * 8 + (m & 7);
          else pix = pix_base + m;
          if (TAPS == 9 || pix < (int64_t)p.N * p.Hout * p.Wout) {
            float4 o = *reinterpret_cast<const float4*>(img + m * ACC_LD + col + sub_c * 4);
            o.x += bq.x; o.y += bq.y; o.z += bq.z; o.w += bq.w;
            const int64_t off = pix * p.ldy + n0 + col + sub_c * 4;
            if (n0 + col + sub_c * 4 >= p.Cstore) continue;   // padded output channels (4-channel granularity)
            if (p.res) {
              const float4 r4 = __ldg(reinterpret_cast<const float4*>(p.res + off));
              o.x += r4.x; o.y += r4.y; o.z += r4.z; o.w += r4.w;
            }
            *reinterpret_cast<float4*>(p.y + off) = o;
            st_s += (o.x + o.y) + (o.z + o.w);
            st_q = fmaf(o.x, o.x, fmaf(o.y, o.y, fmaf(o.z, o.z, fmaf(o.w, o.w, st_q))));
          }
        }
        if (p.stats_part) {  // fixed-order combine of the four row sub-groups, one (sum, sumsq) per channel quad
          st_s += __shfl_xor_sync(0xffffffffu, st_s, 8);
          st_q += __shfl_xor_sync(0xffffffffu, st_q, 8);
          st_s += __shfl_xor_sync(0xffffffffu, st_s, 16);
          st_q += __shfl_xor_sync(0xffffffffu, st_q, 16);
          if (lane < 8) {
            float* sp = p.stats_part + (((size_t)tile * 4 + lane_grp) * (p.Cout >> 2) + ((n0 + col) >> 2) + sub_c) * 2;
            sp[0] = st_s;
            sp[1] = st_q;
          }
        }
      }
    }
  } else {
    // ===================== weight bulk-copy issuer (one thread) =====================
    wg::regs_dec<wg::COPY_REGS>();
    if (warp == 8 && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      const float* wsrc = p.wpk + (size_t)blockIdx.y * nchunks * (B_STAGE / 4);
      for (int kc = 0; kc < nchunks; ++kc) {
        mbar_wait(empty_bar(stage), phase ^ 1);
        mbar_expect_tx(full_bar(stage), B_STAGE);
        bulk_g2s(smem_base + (uint32_t)stage * STAGE + A_STAGE, wsrc + (size_t)kc * (B_STAGE / 4), B_STAGE, full_bar(stage));
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
    }
    __syncwarp();
  }
}

template <int TAPS, int KC, int STAGES, int TILES, bool F16>
constexpr size_t smem_bytes() {
  constexpr int SLOTS = (TAPS == 9) ? 180 : 132, EPC = F16 ? 8 : 4;
  return (size_t)STAGES * (TILES * (KC / EPC) * SLOTS * 16 + TAPS * (KC / EPC) * BN * 16) + (2 * STAGES + 1) * 8 + 16;
}

// weights [Cout][Cin][TAPS] (reference layout, taps innermost) -> [n_tile][k_chunk][tap][k/4][BN][4], TF32-rounded.
// transpose=1 builds the data-gradient operand: N = Cin, K = Cout, taps flipped.
__global__ void pack_weights_tc(const float* __restrict__ w, float* __restrict__ out, int Cout, int Cin, int taps, int KC, int transpose) {
  const int N = transpose ? Cin : Cout, K = transpose ? Cout : Cin;
  const int64_t total = (int64_t)N * K * taps;
  const int nchunks = K / KC, quads = KC / 4;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t r = i;
    const int e = (int)(r % 4); r /= 4;
    const int nn = (int)(r % BN); r /= BN;
    const int q = (int)(r % quads); r /= quads;
    const int t = (int)(r % taps); r /= taps;
    const int kc = (int)(r % nchunks); r /= nchunks;
    const int nt = (int)r;
    const int n = nt * BN + nn, k = kc * KC + q * 4 + e;
    float v;
    if (!transpose) v = w[((size_t)n * Cin + k) * taps + t];
    else v = w[((size_t)k * Cin + n) * taps + (taps - 1 - t)];
    out[i] = round_tf32(v);
  }
}

// fp16 variant of the packing: [n_tile][k_chunk][tap][k/8][BN][8 halves] (one 16-byte chunk = 8 consecutive K of one n);
// `both` != 0 writes the forward packing to out_f AND the data-gradient packing (N = Cin, K = Cout, taps flipped) to out_d
// in one pass over the weight; otherwise only the one selected by `transpose` goes to out_f.
__global__ void pack_weights_tc16(const float* __restrict__ w, __half* __restrict__ out_f, __half* __restrict__ out_d, int Cout, int Cin,
                                  int taps, int KC, int transpose, int both) {
  const int64_t total = (int64_t)Cout * Cin * taps;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    // i enumerates the SOURCE [co][ci][tap] (coalesced reads); destinations are scattered 2-byte stores into L2
    const int t = (int)(i % taps);
    const int ci = (int)((i / taps) % Cin), co = (int)(i / ((int64_t)taps * Cin));
    const __half v = __float2half_rn(w[i]);
    auto put = [&](__half* out, int n, int k, int tt, int K) {
      const int nchunks = K / KC, octs = KC / 8;
      const int64_t j = (((((int64_t)(n / BN) * nchunks + k / KC) * taps + tt) * octs + (k % KC) / 8) * BN + (n % BN)) * 8 + (k % 8);
      out[j] = v;
    };
    if (both) {
      put(out_f, co, ci, t, Cin);
      put(out_d, ci, co, taps - 1 - t, Cout);
    } else if (!transpose) {
      put(out_f, co, ci, t, Cin);
    } else {
      put(out_f, ci, co, taps - 1 - t, Cout);
    }
  }
}

// forward and data-gradient packings of one 3x3 weight in a single pass over it (both are needed every training step)
__global__ void pack_weights_tc_pair(const float* __restrict__ w, float* __restrict__ out_f, float* __restrict__ out_d, int Cout, int Cin) {
  constexpr int taps = 9, KC = 8, quads = KC / 4;
  const int64_t total = (int64_t)Cout * Cin * taps;
  const int nchunks = Cin / KC, nchunks_d = Cout / KC;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t r = i;
    const int e = (int)(r % 4); r /= 4;
    const int nn = (int)(r % BN); r /= BN;
    const int q = (int)(r % quads); r /= quads;
    const int t = (int)(r % taps); r /= taps;
    const int kc = (int)(r % nchunks); r /= nchunks;
    const int nt = (int)r;
    const int n = nt * BN + nn, k = kc * KC + q * 4 + e;  // n = cout, k = cin
    const float v = round_tf32(w[((size_t)n * Cin + k) * taps + t]);
    out_f[i] = v;
    // data-gradient operand: N = cin, K = cout, taps flipped
    const int td = taps - 1 - t;
    const int64_t j = ((((int64_t)(k / BN) * nchunks_d + n / KC) * taps + td) * quads + (n % KC) / 4) * BN * 4 + (int64_t)(k % BN) * 4 + (n % 4);
    out_d[j] = v;
  }
}


// ------------------------------------------------------------------------------------------------------------
// Weight gradient on the Hopper tensor cores:  dW[tap][co][ci] = sum_pixels dy[p][co] * xa[p + tap][ci]
//   D (registers, 3 | 1 accumulators of 64 co x 3 NT ci per warpgroup)  +=  A (registers: dy^T, rows = co, K = pixels)  x
//   B (smem: xa halo)
//   * The reduction (K) dimension is the PIXEL index.  A is read by each MMA warpgroup straight from the staged dy tile into
//     the wgmma register fragment (rows = co: the transpose is free), so the three kernel rows re-read it at no
//     shared-memory cost; B is the same staged halo the forward kernel uses ([ci/4][slot][4 floats], here a K-major
//     operand whose K stride is one 16-byte pixel chunk), and a tap is a start-address shift of the descriptor.
//   * unit of pipelining = 8x8 output pixels (halo 10x10): 3 kernel rows x 8 image rows = 24 MMAs of 64 x 96 x 8 per warpgroup.
//   * CTA = (128 co) x (NT ci) x (a contiguous range of units); partial results go to the split-K workspace that the
//     SIMT path also uses and are reduced deterministically; the per-channel sums of dy (bias gradient) are taken from the
//     staged dy tile.
constexpr int WG_NT = 32;
constexpr int WG_STAGES = 3;
constexpr int WG_SLOTS = 100;          // 10 x 10 halo
constexpr int WG_THREADS = 12 * 32;    // 8 producer / MMA warps, the dy copy warpgroup
constexpr int WG_DY_STAGE = 64 * 128 * 4;  // staged dy tile: 64 pixels x 128 channels fp32

struct WParams {
  const float* x;   // conv input (activated), NHWC dense [N,Hin,Win,Cin]   | rows [M, Cin] with pitch ldx (TAPS == 1)
  const float* dy;  // output gradient, NHWC dense [N,H,W,Cout]             | rows [M, Cout] with pitch ldy
  float* part;      // [splits][TAPS][Cout][Cin]
  float* bpart;     // [splits][Cout] or null
  int N, Hin, Win, Cin, H, W, Cout, map;
  int units_x, units_y;
  int64_t total_units, units_per_split, rows, ldx, ldy;
  const float* gn_table;  // fused GroupNorm(+SiLU) prologue on x, [N][Cin][2] (sc, sh), or null (3x3 only)
  int gn_silu;
  const float* dy_amax;   // fp16-operand kernel: max|dy| (device scalar) for the power-of-two scale of the A operand, or null
  int Cout_real;          // channels present in dy (Cout = round_up to 128: the TMA copy zero-fills the rest)
  int x_f16;              // fp16-operand kernel: x already holds fp16 (mas_gn_backward's act_out): staged without conversion
  int dy_f16;             // fp16-operand kernel: dy is the fp16 shadow (mas_gn_backward's dx_f16), already scaled by operand_scale(*dy_amax)
};

// TAPS == 9: 3x3 convolution (unit = 8x8 output pixels, halo 10x10).  TAPS == 1: 1x1 convolution / row GEMM
// (unit = 64 consecutive rows, no halo).
// F16 (3x3 only): both operands converted to fp16 on their way to the tensor core (dy scaled by a power of two from
// p.dy_amax); a 16-byte chunk of B then holds 8 pixels = one halo row segment and one MMA (K = 16) covers two image rows
// of the unit.
template <int TAPS, bool PRO, bool F16>
__global__ void __launch_bounds__(WG_THREADS, 1) wgrad_tc(const WParams p, const __grid_constant__ CUtensorMap dy_map) {
  static_assert(!F16 || TAPS == 9, "the fp16-operand weight-gradient kernel is the 3x3 one");
  // B (the shifted operand) must be K-major with K = pixel for TF32 (wgmma transposes 16-bit operands only), so the halo is
  // staged TRANSPOSED ([ci][pixel], 4 pixels per 16-byte chunk) once per horizontal tap offset dx (3 copies); vertical
  // offsets are whole-chunk K advances of the descriptor.
  // Channel ci = 4q + j of the tile sits in operand row n = 8j + q: the 8 lanes of a store phase (q = 0..7) then hit 8
  // different bank groups, and the epilogue undoes the permutation.
  // One MMA covers the three horizontal taps of a kernel row: its N = 3 x NT operand rows are [dx][channel], laid out
  // per 4-pixel chunk as 3*NT/8 consecutive 128-byte core matrices, so a single descriptor (SBO = 128, LBO = chunk
  // pitch) spans all three dx copies.
  constexpr int NT = (TAPS == 9) ? WG_NT : 128, QUADS = NT / 4;
  constexpr int SLOTS = (TAPS == 9) ? WG_SLOTS : 64;
  constexpr int COPIES = (TAPS == 9) ? 3 : 1;
  constexpr int LBO_B = COPIES * NT * 16;                  // TF32: bytes between 16-byte chunks (4 pixels)
  // fp16: the halo is staged UNTRANSPOSED (an MN-major operand: element (n, k) sits at (n%8)*2 + (k%8)*16 + (k/8)*LBO +
  // (n/8)*SBO bytes), as planes [dx copy][ci/8][slot][8 channels]: a pixel's 8 channels are one 16-byte store per dx copy (copy
  // dx holds the halo shifted left by dx pixels) instead of 24 two-byte stores; K groups are image rows (LBO = the 160-byte
  // halo row), N groups are the 12 (dx, ci/8) planes (SBO = plane pitch), a vertical tap is a start-address advance of one
  // halo row.
  constexpr int P16 = SLOTS * 16 + 32;                     // plane pitch (32-byte skew: conflict-free 16-byte stores)
  constexpr int B_STAGE = F16 ? 12 * P16 : ((TAPS == 9) ? 20 : 16) * LBO_B;
  constexpr int ITEMS = SLOTS * QUADS, PER_THREAD = (ITEMS + NPROD - 1) / NPROD;
  constexpr int NMMA = COPIES * NT;                        // N of one MMA (96 | 128)
  constexpr int NACC = (TAPS == 9) ? 3 : 1;                // accumulators: one per kernel row
  constexpr int KSTEPS = F16 ? 4 : 8;                      // MMAs per kernel row and unit (K = 16 | 8 pixels)

  extern __shared__ __align__(1024) uint8_t smem[];
  uint8_t* dy_smem = smem + (size_t)WG_STAGES * B_STAGE;   // [WG_STAGES][64 pixels][128 co] fp32 (or halves), filled by TMA
  uint64_t* bars = reinterpret_cast<uint64_t*>(dy_smem + (size_t)WG_STAGES * WG_DY_STAGE);
  const uint32_t smem_base = smem_u32(smem), bar_base = smem_u32(bars);
  auto fullB = [&](int s) { return bar_base + 8u * s; };
  auto empty = [&](int s) { return bar_base + 8u * (WG_STAGES + s); };
  auto fullD = [&](int s) { return bar_base + 8u * (2 * WG_STAGES + s); };

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int ci0 = blockIdx.x * NT, co0 = blockIdx.y * BM, split = blockIdx.z;
  const int64_t u0 = (int64_t)split * p.units_per_split;
  const int64_t u1 = min(p.total_units, u0 + p.units_per_split);

  if (tid == 0) {
    for (int s = 0; s < WG_STAGES; ++s) {
      mbar_init(fullB(s), NPROD);
      mbar_init(empty(s), NPROD);
      mbar_init(fullD(s), 1);
    }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 8) {
    wg::regs_inc<wg::MMA_REGS>();
    const int wgi = warp >> 2;
    const int frow = wgi * 64 + (warp & 3) * 16 + (lane >> 2), fk = lane & 3;   // fragment row (co) and K quad of this thread
    float acc[NACC][NMMA / 2];
#pragma unroll
    for (int a = 0; a < NACC; ++a)
#pragma unroll
      for (int i = 0; i < NMMA / 2; ++i) acc[a][i] = 0.f;
    float bsum = 0.f;
    const bool want_bias = p.bpart != nullptr && blockIdx.x == 0 && tid < 128;   // thread tid sums channel co0 + tid
    float a_inv = 1.f;
    const float a_scale = F16 ? operand_scale(p.dy_amax, &a_inv) : 1.f;
    // all producers have staged B and the dy tile has landed: this warpgroup's MMAs of unit u
    auto mma_unit = [&](int64_t u, int stage, uint32_t phase) {
      mbar_wait(fullB(stage), phase);
      mbar_wait(fullD(stage), phase);
      const uint8_t* dyt = dy_smem + (size_t)stage * WG_DY_STAGE;
      const bool shadow = F16 && p.dy_f16;
      if (want_bias) {   // the bias gradient falls out of ONE ci-tile's pass over dy (the other ci tiles see the same dy)
        if (shadow) {
          const __half* dh = reinterpret_cast<const __half*>(dyt) + tid;
          for (int j = 0; j < 64; j += 2) bsum += __half2float(dh[j * 128]) + __half2float(dh[(j + 1) * 128]);
        } else {
          const float* df = reinterpret_cast<const float*>(dyt) + tid;
          for (int j = 0; j < 64; ++j) bsum += (TAPS == 9 || u * 64 + j < p.rows) ? df[j * 128] : 0.f;
        }
      }
      // A fragments of the unit: a[ks][0..3] = dy^T rows (frow, frow + 8) x pixels of K step ks
      uint32_t a[KSTEPS][4];
#pragma unroll
      for (int ks = 0; ks < KSTEPS; ++ks) {
#pragma unroll
        for (int h = 0; h < 4; ++h) {
          const int co = frow + 8 * (h & 1);
          if (F16) {
            const int px = ks * 16 + 2 * fk + 8 * (h >> 1);
            if (shadow) {
              const unsigned short* dh = reinterpret_cast<const unsigned short*>(dyt) + co;
              a[ks][h] = (uint32_t)dh[px * 128] | ((uint32_t)dh[(px + 1) * 128] << 16);
            } else {
              const float* df = reinterpret_cast<const float*>(dyt) + co;
              a[ks][h] = pack_h2(df[px * 128] * a_scale, df[(px + 1) * 128] * a_scale);
            }
          } else {
            const int px = ks * 8 + fk + 4 * (h >> 1);
            const float v = reinterpret_cast<const float*>(dyt)[px * 128 + co];
            a[ks][h] = __float_as_uint((TAPS == 9 || u * 64 + px < p.rows) ? v : 0.f);
          }
        }
      }
      const uint32_t b_st = smem_base + (uint32_t)stage * B_STAGE;
      const uint64_t b_base = wg::desc(b_st, LBO_B, 128);
      const uint64_t b16 = wg::desc(b_st, 160, P16);   // MN-major: LBO = K-group (halo row) pitch, SBO = N-group (plane) pitch
      wg::fence();
#pragma unroll
      for (int ks = 0; ks < KSTEPS; ++ks) {
#pragma unroll
        for (int dyy = 0; dyy < NACC; ++dyy) {
          if (F16) {   // K = 16 pixels = image rows (2 ks, 2 ks + 1) of the unit: halo rows 2 ks + dy, 2 ks + dy + 1
            wg::wgmma_f16_rs_n96<1>(acc[dyy], a[ks], b16 + (uint64_t)(((2 * ks + dyy) * 160) >> 4), 1u);
          } else if (TAPS == 9) {   // image row ks + dy starts at chunk 2 (ks + dy); the three dx taps are the N blocks
            wg::wgmma_tf32_rs_n96(acc[dyy], a[ks], b_base + (uint64_t)(((ks + dyy) * 2 * LBO_B) >> 4), 1u);
          } else {
            wg::wgmma_tf32_rs_n128(acc[dyy], a[ks], b_base + (uint64_t)((ks * 2 * LBO_B) >> 4), 1u);
          }
        }
      }
      wg::commit();
      wg::wait<0>();   // the A fragments are reloaded for the next unit
      mbar_arrive(empty(stage));
    };
    if (F16) {
      // ============ producers, fp16: x halo -> shared memory planes [dx][ci/8][slot][8 channels] (no transposition) ============
    constexpr int OCTS = NT / 8, ITEMS16 = SLOTS * OCTS, PT16 = (ITEMS16 + NPROD - 1) / NPROD;   // 400 items, 2 per thread
    int sl_r[PT16], sl_c[PT16], sl_o[PT16];
#pragma unroll
    for (int i = 0; i < PT16; ++i) {
      const int item = tid + i * NPROD, slot = item / OCTS;
      sl_o[i] = item % OCTS;
      sl_r[i] = slot / 10;
      sl_c[i] = item < ITEMS16 ? slot % 10 : -100;
    }
    int pux = (int)(u0 % p.units_x), puy = (int)((u0 / p.units_x) % p.units_y), pn = (int)(u0 / ((int64_t)p.units_x * p.units_y));
    int cux = 0, cuy = 0, cn = 0;   // coordinates of the unit whose data sits in v (for the prologue's padding test)
    auto gload16 = [&](float4 (*v)[2]) {
      const int ux = pux, uy = puy, n = pn;
      if (++pux == p.units_x) { pux = 0; if (++puy == p.units_y) { puy = 0; ++pn; } }
#pragma unroll
      for (int i = 0; i < PT16; ++i) {
        v[i][0] = make_float4(0.f, 0.f, 0.f, 0.f);
        v[i][1] = v[i][0];
        if (sl_c[i] >= 0) {
          const int vy = uy * 8 - 1 + sl_r[i], vx = ux * 8 - 1 + sl_c[i];
          int iy = vy, ix = vx;
          bool ok;
          if (p.map == MAP_S1) {
            ok = (unsigned)vy < (unsigned)p.Hin && (unsigned)vx < (unsigned)p.Win;
          } else {  // MAP_UP
            ok = (unsigned)vy < (unsigned)(2 * p.Hin) && (unsigned)vx < (unsigned)(2 * p.Win);
            iy = vy >> 1; ix = vx >> 1;
          }
          if (ok) {
            const int64_t e = ((int64_t)(n * p.Hin + iy) * p.Win + ix) * p.Cin + ci0 + sl_o[i] * 8;
            if (p.x_f16) {   // eight halves = the 16-byte operand chunk itself (carried in v[i][0])
              v[i][0] = __ldg(reinterpret_cast<const float4*>(reinterpret_cast<const __half*>(p.x) + e));
            } else {
              const float4* src = reinterpret_cast<const float4*>(p.x + e);
              v[i][0] = __ldg(src);
              v[i][1] = __ldg(src + 1);
            }
          }
        }
      }
    };
    int stage = 0;
    uint32_t phase = 0;
    float4 vn[PT16][2];
    if (u0 < u1) gload16(vn);
    for (int64_t u = u0; u < u1; ++u) {
      float4 v[PT16][2];
#pragma unroll
      for (int i = 0; i < PT16; ++i) { v[i][0] = vn[i][0]; v[i][1] = vn[i][1]; }
      if (PRO) {
        cux = (int)(u % p.units_x); cuy = (int)((u / p.units_x) % p.units_y); cn = (int)(u / ((int64_t)p.units_x * p.units_y));
      }
      if (u + 1 < u1) gload16(vn);
      if (PRO && p.gn_table) {
        // the convolution's input is act(GroupNorm(x)): recomputed here instead of stored; padding pixels stay exactly zero
#pragma unroll
        for (int i = 0; i < PT16; ++i) {
          if (sl_c[i] >= 0) {
            const int vy = cuy * 8 - 1 + sl_r[i], vx = cux * 8 - 1 + sl_c[i];
            const bool ok = (p.map == MAP_S1) ? ((unsigned)vy < (unsigned)p.Hin && (unsigned)vx < (unsigned)p.Win)
                                              : ((unsigned)vy < (unsigned)(2 * p.Hin) && (unsigned)vx < (unsigned)(2 * p.Win));
            if (ok) {
#pragma unroll
              for (int h = 0; h < 2; ++h) {
                const float4* tp = reinterpret_cast<const float4*>(p.gn_table + ((size_t)cn * p.Cin + ci0 + sl_o[i] * 8 + h * 4) * 2);
                const float4 t0 = __ldg(tp), t1 = __ldg(tp + 1);
                float a0 = fmaf(v[i][h].x, t0.x, t0.y), a1 = fmaf(v[i][h].y, t0.z, t0.w);
                float a2 = fmaf(v[i][h].z, t1.x, t1.y), a3 = fmaf(v[i][h].w, t1.z, t1.w);
                if (p.gn_silu) { a0 = silu_f(a0); a1 = silu_f(a1); a2 = silu_f(a2); a3 = silu_f(a3); }
                v[i][h] = make_float4(a0, a1, a2, a3);
              }
            }
          }
        }
      }
      mbar_wait(empty(stage), phase ^ 1);
      uint8_t* b_st = smem + (size_t)stage * B_STAGE;
#pragma unroll
      for (int i = 0; i < PT16; ++i) {
        if (sl_c[i] >= 0) {
          const uint4 h = p.x_f16 ? make_uint4(__float_as_uint(v[i][0].x), __float_as_uint(v[i][0].y), __float_as_uint(v[i][0].z),
                                               __float_as_uint(v[i][0].w))
                                  : make_uint4(pack_h2(v[i][0].x, v[i][0].y), pack_h2(v[i][0].z, v[i][0].w), pack_h2(v[i][1].x, v[i][1].y),
                                               pack_h2(v[i][1].z, v[i][1].w));
          const int slot = sl_r[i] * 10 + sl_c[i];
#pragma unroll
          for (int dx = 0; dx < 3; ++dx)
            if (sl_c[i] >= dx) *reinterpret_cast<uint4*>(b_st + (dx * OCTS + sl_o[i]) * P16 + (slot - dx) * 16) = h;
        }
      }
      fence_proxy_async();
      mbar_arrive(fullB(stage));
      mma_unit(u, stage, phase);
      if (++stage == WG_STAGES) { stage = 0; phase ^= 1; }
    }
    } else {
      // ============ producers: x halo / rows -> shared memory, transposed (K = pixel) ============
    int it_r[PER_THREAD], it_c[PER_THREAD], it_q[PER_THREAD];
#pragma unroll
    for (int i = 0; i < PER_THREAD; ++i) {
      const int item = tid + i * NPROD;
      // lanes of a warp = 8 channel quads x 4 consecutive pixel slots (conflict-free transposed stores)
      const int q = (item % 8) + 8 * (item / (8 * SLOTS)), slot = (item / 8) % SLOTS;
      it_q[i] = q;
      if (TAPS == 9) { it_r[i] = slot / 10; it_c[i] = item < ITEMS ? slot % 10 : -100; }
      else { it_r[i] = slot; it_c[i] = item < ITEMS ? 0 : -100; }
    }
    // (n, uy, ux) of the next unit to load, advanced incrementally (no per-unit 64-bit divisions in the hot loop)
    int pux = (int)(u0 % p.units_x), puy = (int)((u0 / p.units_x) % p.units_y), pn = (int)(u0 / ((int64_t)p.units_x * p.units_y));
    auto gload = [&](int64_t u, float4* v) {
      if (TAPS == 9) {
        const int ux = pux, uy = puy, n = pn;
        if (++pux == p.units_x) { pux = 0; if (++puy == p.units_y) { puy = 0; ++pn; } }
#pragma unroll
        for (int i = 0; i < PER_THREAD; ++i) {
          v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
          if (it_c[i] >= 0) {
            const int vy = uy * 8 - 1 + it_r[i], vx = ux * 8 - 1 + it_c[i];
            int iy = vy, ix = vx;
            bool ok;
            if (p.map == MAP_S1) {
              ok = (unsigned)vy < (unsigned)p.Hin && (unsigned)vx < (unsigned)p.Win;
            } else {  // MAP_UP
              ok = (unsigned)vy < (unsigned)(2 * p.Hin) && (unsigned)vx < (unsigned)(2 * p.Win);
              iy = vy >> 1; ix = vx >> 1;
            }
            if (ok) v[i] = __ldg(reinterpret_cast<const float4*>(p.x + ((int64_t)(n * p.Hin + iy) * p.Win + ix) * p.Cin + ci0 + it_q[i] * 4));
          }
        }
      } else {
#pragma unroll
        for (int i = 0; i < PER_THREAD; ++i) {
          v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
          const int64_t row = u * 64 + it_r[i];
          if (it_c[i] >= 0 && row < p.rows) v[i] = __ldg(reinterpret_cast<const float4*>(p.x + row * p.ldx + ci0 + it_q[i] * 4));
        }
      }
    };
    int stage = 0;
    uint32_t phase = 0;
    float4 vn[PER_THREAD];
    if (u0 < u1) gload(u0, vn);
    for (int64_t u = u0; u < u1; ++u) {
      float4 v[PER_THREAD];
#pragma unroll
      for (int i = 0; i < PER_THREAD; ++i) v[i] = vn[i];
      if (u + 1 < u1) gload(u + 1, vn);   // next unit's global loads are in flight while this unit is stored
      if (TAPS == 9 && PRO) {
        if (p.gn_table) {
          // the convolution's input is act(GroupNorm(x)): recomputed here (at consume time) instead of stored.
          // Padding pixels must stay exactly zero, so validity is re-derived from the unit coordinates.
          const int ux = (int)(u % p.units_x), uy = (int)((u / p.units_x) % p.units_y);
          const int n = (int)(u / ((int64_t)p.units_x * p.units_y));
#pragma unroll
          for (int i = 0; i < PER_THREAD; ++i) {
            if (it_c[i] >= 0) {
              const int vy = uy * 8 - 1 + it_r[i], vx = ux * 8 - 1 + it_c[i];
              const bool ok = (p.map == MAP_S1) ? ((unsigned)vy < (unsigned)p.Hin && (unsigned)vx < (unsigned)p.Win)
                                                : ((unsigned)vy < (unsigned)(2 * p.Hin) && (unsigned)vx < (unsigned)(2 * p.Win));
              if (ok) {
                const float4* tp = reinterpret_cast<const float4*>(p.gn_table + ((size_t)n * p.Cin + ci0 + it_q[i] * 4) * 2);
                const float4 t0 = __ldg(tp), t1 = __ldg(tp + 1);
                float a0 = fmaf(v[i].x, t0.x, t0.y), a1 = fmaf(v[i].y, t0.z, t0.w);
                float a2 = fmaf(v[i].z, t1.x, t1.y), a3 = fmaf(v[i].w, t1.z, t1.w);
                if (p.gn_silu) { a0 = silu_f(a0); a1 = silu_f(a1); a2 = silu_f(a2); a3 = silu_f(a3); }
                v[i] = make_float4(a0, a1, a2, a3);
              }
            }
          }
        }
      }
      mbar_wait(empty(stage), phase ^ 1);
      float* b_st = reinterpret_cast<float*>(smem + (size_t)stage * B_STAGE);
#pragma unroll
      for (int i = 0; i < PER_THREAD; ++i) {
        if (it_c[i] >= 0) {
          const float e[4] = {v[i].x, v[i].y, v[i].z, v[i].w};
          if (F16) {
            const unsigned short h[4] = {to_h(e[0]), to_h(e[1]), to_h(e[2]), to_h(e[3])};
#pragma unroll
            for (int dx = 0; dx < COPIES; ++dx) {
              const int c = it_c[i] - dx;
              if ((unsigned)c < 8u) {
                // chunk = halo row it_r; channel 4q+j -> operand row n = (NT/4)*j + q of the dx block; 8 pixels per row
                unsigned short* d = reinterpret_cast<unsigned short*>(b_st) + it_r[i] * (LBO_B / 2) + dx * (NT * 8) + it_q[i] * 8 + c;
#pragma unroll
                for (int j = 0; j < 4; ++j) d[j * NT * 2] = h[j];
              }
            }
            continue;
          }
#pragma unroll
          for (int dx = 0; dx < COPIES; ++dx) {
            const int c = it_c[i] - dx;
            if (TAPS == 1 || (unsigned)c < 8u) {
              const int kk = (TAPS == 9) ? it_r[i] * 8 + c : it_r[i];
              // channel 4q+j -> operand row (within its dx block) n = (NT/4)*j + q; byte offset = n*16
              float* d = b_st + (kk >> 2) * (LBO_B / 4) + dx * (NT * 4) + it_q[i] * 4 + (kk & 3);
#pragma unroll
              for (int j = 0; j < 4; ++j) d[j * NT] = e[j];
            }
          }
        }
      }
      fence_proxy_async();
      mbar_arrive(fullB(stage));
      mma_unit(u, stage, phase);
      if (++stage == WG_STAGES) { stage = 0; phase ^= 1; }
    }
    }
#pragma unroll
    for (int a = 0; a < NACC; ++a) wg::fence_regs<NMMA / 2>(acc[a]);
    if (want_bias) p.bpart[(size_t)split * p.Cout + co0 + tid] = (F16 && p.dy_f16) ? bsum * a_inv : bsum;
    // ============ epilogue: TAPS x [128 co x NT ci] partial sums -> workspace ============
    // acc[dyy][4 j + 2 i + c] = kernel row dyy, co frow + 8 i, operand row n = 8 j + 2 (lane % 4) + c = (dx, channel slot)
    const float inv = F16 ? a_inv : 1.f;
#pragma unroll
    for (int dyy = 0; dyy < NACC; ++dyy) {
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int co = co0 + frow + 8 * i;
#pragma unroll
        for (int j = 0; j < NMMA / 8; ++j) {
#pragma unroll
          for (int c = 0; c < 2; ++c) {
            const int n = 8 * j + 2 * fk + c, dx = n / NT, nn = n % NT;
            const int ci = F16 ? nn : 4 * (nn % QUADS) + nn / QUADS;
            const int t = (TAPS == 9) ? dyy * 3 + dx : 0;
            p.part[(((size_t)split * TAPS + t) * p.Cout + co) * p.Cin + ci0 + ci] = acc[dyy][4 * j + 2 * i + c] * inv;
          }
        }
      }
    }
  } else {
    // ============ dy TMA issuer (one thread): box [8 rows][8 pixels][128 co] (or [64 rows][128 co]) -> shared [64][128] ============
    // a tiled tensor map (cuTensorMapEncodeTiled on the host) lets ONE cp.async.bulk.tensor fetch the whole dy tile of a
    // unit for any Cout; rows beyond the matrix (1x1 tail) are zero-filled by the TMA unit.
    wg::regs_dec<wg::COPY_REGS>();
    if (warp == 8 && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int64_t u = u0; u < u1; ++u) {
        const uint32_t dst = smem_u32(dy_smem) + (uint32_t)stage * WG_DY_STAGE;
        mbar_wait(empty(stage), phase ^ 1);
        mbar_expect_tx(fullD(stage), (F16 && p.dy_f16) ? WG_DY_STAGE / 2 : WG_DY_STAGE);
        if (TAPS == 9) {
          const int ux = (int)(u % p.units_x), uy = (int)((u / p.units_x) % p.units_y);
          const int n = (int)(u / ((int64_t)p.units_x * p.units_y));
          tma_load_4d(dst, &dy_map, co0, ux * 8, uy * 8, n, fullD(stage));
        } else {
          tma_load_2d(dst, &dy_map, co0, (int)(u * 64), fullD(stage));
        }
        if (++stage == WG_STAGES) { stage = 0; phase ^= 1; }
      }
    }
    __syncwarp();
  }
}


// ------------------------------------------------------------------------------------------------------------
// Single-MMA probe (tests/test_gpu_tc_probe.py): D[128 x 32] = A[128 x 8] * B[32 x 8]^T as two wgmma.m64n32k8 (rows 0-63,
// 64-127) with the operand placement / descriptor conventions selected at run time - pins the addressing the production
// kernels rely on.  a_src 1: A from registers (the wgrad_tc form).  b_layout 99: the B descriptor is the host's raw one
// (sm_100 version bits 46-48 dropped; TF32 operands cannot be transposed, so no instruction descriptor applies).
__global__ void __launch_bounds__(128, 1) mma_probe(const float* __restrict__ A, const float* __restrict__ B, float* __restrict__ D,
                                                    int a_src, int b_layout, unsigned long long raw_desc, int raw_off) {
  __shared__ __align__(1024) uint8_t sm[24576];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  float* sa = reinterpret_cast<float*>(sm);           // A: K-major, LBO = 2048 (128 rows * 16 B), SBO = 128
  float* sb = reinterpret_cast<float*>(sm + 8192);    // B region (16 KB: any descriptor of the tests stays inside)
  constexpr int PL = 36 * 16;                         // plane pitch of the MN-major B layout (36 slots)
  for (int i = tid; i < 128 * 8; i += 128) {          // A[m][k] -> (k/4)*2048 + m*16 + (k%4)*4
    int m = i / 8, k = i % 8;
    sa[((k / 4) * 2048 + m * 16 + (k % 4) * 4) / 4] = A[i];
  }
  const int raw = b_layout == 99;      // raw mode: descriptor high bits / start offset come from the host
  const int reveal = b_layout >= 10;   // address-reveal mode: B region holds its own word index
  if (reveal) b_layout = raw ? 0 : b_layout - 10;
  for (int i = tid; i < 4096; i += 128) sb[i] = (reveal && i < 2048) ? (float)i : 0.f;
  __syncthreads();
  if (!reveal) {
    for (int i = tid; i < 32 * 8; i += 128) {
      int n = i / 8, k = i % 8;
      int off = (b_layout == 0) ? ((k / 4) * 512 + n * 16 + (k % 4) * 4) : ((n / 4) * PL + k * 16 + (n % 4) * 4);
      sb[off / 4] = B[i];
    }
  }
  fence_proxy_async();
  __syncthreads();
  uint64_t bd;
  if (b_layout == 0) bd = wg::desc(smem_u32(sb), 512, 128);
  else if (b_layout == 1) bd = wg::desc(smem_u32(sb), 160, PL);   // LBO field = K-group stride, SBO field = MN-quad stride
  else bd = wg::desc(smem_u32(sb), PL, 160);                      // fields swapped
  if (raw) bd = (raw_desc & ~(0x3FFFull | (7ull << 46))) | (uint64_t)(((smem_u32(sb) + (uint32_t)raw_off) >> 4) & 0x3FFF);
  const int r = (warp & 3) * 16 + (lane >> 2), c = lane & 3;      // fragment rows r, r + 8; columns / K quads c, c + 4
  float acc[2][16];
  uint32_t a[2][4];
#pragma unroll
  for (int h = 0; h < 2; ++h)
#pragma unroll
    for (int q = 0; q < 4; ++q) a[h][q] = __float_as_uint(A[(h * 64 + r + 8 * (q & 1)) * 8 + c + 4 * (q >> 1)]);
  wg::fence();
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    if (a_src == 0) wg::wgmma_tf32_ss_n32(acc[h], wg::desc(smem_u32(sa) + h * 1024, 2048, 128), bd, 0u);
    else wg::wgmma_tf32_rs_n32(acc[h], a[h], bd, 0u);
  }
  wg::commit();
  wg::wait<0>();
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    wg::fence_regs<16>(acc[h]);
#pragma unroll
    for (int j = 0; j < 16; ++j) D[(h * 64 + r + 8 * ((j >> 1) & 1)) * 32 + 8 * (j >> 2) + 2 * c + (j & 1)] = acc[h][j];
  }
}

// fp16 address-reveal probe: A (shared memory, K-major) selects k = m % 16 in row m; the B region holds its own half index
// (0 .. 2047); D[k][n] is therefore the index of the half the tensor core reads for element (n, k) of B under the raw shared-
// memory descriptor supplied by the host, read MN-major when b_mn is set (tests/test_gpu_tc_probe.py).
__global__ void __launch_bounds__(128, 1) mma_probe16(float* __restrict__ D, unsigned long long raw_desc, int b_mn, int n, int raw_off) {
  __shared__ __align__(1024) uint8_t sm[16384];
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  __half* sa = reinterpret_cast<__half*>(sm);          // A: 128 x 16 halves, K-major [k/8][m][8]: LBO 2048, SBO 128
  __half* sb = reinterpret_cast<__half*>(sm + 4096);   // B region (12 KB)
  for (int i = tid; i < 128 * 16; i += 128) {
    const int m = i / 16, k = i % 16;
    sa[(k / 8) * 1024 + m * 8 + (k % 8)] = __float2half((k == m % 16) ? 1.f : 0.f);
  }
  for (int i = tid; i < 6144; i += 128) sb[i] = __float2half(i < 2048 ? (float)i : 0.f);
  fence_proxy_async();
  __syncthreads();
  const uint64_t bd = (raw_desc & ~(0x3FFFull | (7ull << 46))) | (uint64_t)(((smem_u32(sb) + (uint32_t)raw_off) >> 4) & 0x3FFF);
  float acc[2][64];   // D = 128 x n (n = 32 or 128)
  wg::fence();
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const uint64_t ad = wg::desc(smem_u32(sa) + h * 1024, 2048, 128);
    if (n == 128) {
      if (b_mn) wg::wgmma_f16_ss_n128<0, 1>(acc[h], ad, bd, 0u);
      else wg::wgmma_f16_ss_n128<0, 0>(acc[h], ad, bd, 0u);
    } else {
      if (b_mn) wg::wgmma_f16_ss_n32<0, 1>(acc[h], ad, bd, 0u);
      else wg::wgmma_f16_ss_n32<0, 0>(acc[h], ad, bd, 0u);
    }
  }
  wg::commit();
  wg::wait<0>();
  const int r = (warp & 3) * 16 + (lane >> 2), c = lane & 3;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    wg::fence_regs<64>(acc[h]);
#pragma unroll
    for (int j = 0; j < 64; ++j)
      if (j < n / 2) D[(h * 64 + r + 8 * ((j >> 1) & 1)) * n + 8 * (j >> 2) + 2 * c + (j & 1)] = acc[h][j];
  }
}

}  // namespace tc

void conv_wgrad_reduce_launch(const float* part, int splits, int ntap, int Cout, int Cin, float* dw, const float* bpart, float* dbias,
                              cudaStream_t st);

static bool dense_nhwc(const mas_tensor4& t) {
  return t.sc == 1 && t.sw == t.c && t.sh == t.w * t.c && t.sn == t.h * t.w * t.c;
}
static inline bool al16p(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

template <typename K>
static int set_smem(K kernel, size_t bytes) {
  cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
  if (e != cudaSuccess) return fail(MAS_ERR_LAUNCH, "cudaFuncSetAttribute(smem=%zu): %s", bytes, cudaGetErrorString(e));
  return MAS_OK;
}

// w_tc must have been produced by mas_pack_conv3x3_tc for the matching direction.
// f16 != 0: w_tc is the fp16 packing (mas_pack_conv3x3_tc16) and x_amax (device scalar or null) scales the A operand.
int conv3x3_fprop_tc_launch(const float* x, mas_tensor4 xs, const float* w_tc, const float* bias, const float* res, float* y,
                            mas_tensor4 ys, int mode, const float* gn_table, int gn_silu, float* stats_part, int f16,
                            const float* x_amax, cudaStream_t st) {
  // ys.c not a multiple of 128 (but of 4): the kernel runs round_up(ys.c, 128) output channels - w_tc / bias must have been
  // packed / padded to that many (zero rows) - and stores only the first ys.c
  const int Cin = (int)xs.c, Cstore = (int)ys.c, Cout = (int)cdiv(ys.c, tc::BN) * tc::BN;
  if (f16 && Cin % 16) return fail(MAS_ERR_UNSUPPORTED, "tc conv (fp16 operands): Cin=%d must be a multiple of 16", Cin);
  if (Cstore % 4) return fail(MAS_ERR_UNSUPPORTED, "tc conv: Cout=%d must be a multiple of 4", Cstore);
  if (Cstore != Cout && (res || stats_part)) return fail(MAS_ERR_UNSUPPORTED, "tc conv: residual / statistics epilogues need Cout %% 128 == 0");
  if (!(mode == MAS_CONV_S1 || mode == MAS_CONV_UP || mode == MAS_CONV_ZS)) return fail(MAS_ERR_UNSUPPORTED, "tc conv: mode %d", mode);
  if (!dense_nhwc(xs) || !dense_nhwc(ys) || Cin % 8 || ys.h % 16 || ys.w % 8 || !al16p(x) || !al16p(y) ||
      (res && !al16p(res)) || (bias && !al16p(bias)) || !al16p(w_tc))
    return fail(MAS_ERR_UNSUPPORTED, "tc conv: shape/layout not eligible (Cin=%d Cout=%d Hout=%lld Wout=%lld)", Cin, Cout,
                (long long)ys.h, (long long)ys.w);
  int64_t eh = (mode == MAS_CONV_S1) ? xs.h : 2 * xs.h, ew = (mode == MAS_CONV_S1) ? xs.w : 2 * xs.w;
  if (ys.h != eh || ys.w != ew || xs.n != ys.n) return fail(MAS_ERR_INVALID_ARG, "tc conv: output extent mismatch");
  tc::Params p;
  p.x = x; p.wpk = w_tc; p.bias = bias; p.res = res; p.y = y;
  p.N = (int)xs.n; p.Hin = (int)xs.h; p.Win = (int)xs.w; p.Cin = Cin; p.Hout = (int)ys.h; p.Wout = (int)ys.w; p.Cout = Cout;
  p.map = (mode == MAS_CONV_S1) ? tc::MAP_S1 : (mode == MAS_CONV_UP ? tc::MAP_UP : tc::MAP_ZS);
  p.ldx = Cin; p.ldy = Cstore; p.Cstore = Cstore;
  p.tiles_x = (int)(ys.w / 8); p.tiles_y = (int)(ys.h / 16);
  p.total_tiles = (int64_t)p.N * p.tiles_x * p.tiles_y;
  p.alpha = 1.0f;
  p.gn_table = gn_table; p.gn_silu = gn_silu; p.stats_part = stats_part;
  p.x_amax = f16 ? x_amax : nullptr;
  if (gn_table && !al16p(gn_table)) return fail(MAS_ERR_INVALID_ARG, "tc conv: gn_table must be 16-byte aligned");
  // one CTA per SM: 2 tiles (2 x 64 accumulator registers per thread and tile half) and a 2-stage ring
  constexpr int T = 2, STG = 2;
  constexpr size_t smem = tc::smem_bytes<9, 8, STG, T, false>();
  static_assert(smem == tc::smem_bytes<9, 16, STG, T, true>(), "both operand formats stage the same bytes per K chunk");
  static std::atomic<uint64_t> configured{0};
  if (first_on_device(configured)) {
    if (int e = set_smem(tc::shift_gemm_tc<9, 8, STG, T, false>, smem)) return e;
    if (int e = set_smem(tc::shift_gemm_tc<9, 16, STG, T, true>, smem)) return e;
    mark_device(configured);
  }
  dim3 grid((unsigned)cdiv(p.total_tiles, T), (unsigned)(Cout / tc::BN));
  if (f16) {
    tc::shift_gemm_tc<9, 16, STG, T, true><<<grid, tc::NTHREADS, smem, st>>>(p);
    return launched_tc("shift_gemm_tc<9,f16>");
  }
  tc::shift_gemm_tc<9, 8, STG, T, false><<<grid, tc::NTHREADS, smem, st>>>(p);
  return launched_tc("shift_gemm_tc<9>");
}

// Row GEMM C[M,N] = alpha * A[M,K] * Wt[N,K]^T + bias + residual with PRE-PACKED weights (mas_pack_gemm_tc).
int gemm_rows_tc_launch(const float* A, int64_t lda, const float* w_tc, float* C, int64_t ldc, int64_t M, int N, int K, float alpha,
                        const float* bias, const float* res, float* stats_part, cudaStream_t st) {
  if (K % 32 || N % tc::BN || lda % 4 || ldc % 4 || !al16p(A) || !al16p(C) || (res && !al16p(res)) || (bias && !al16p(bias)) ||
      !al16p(w_tc))
    return fail(MAS_ERR_UNSUPPORTED, "tc gemm: shape not eligible (M=%lld N=%d K=%d)", (long long)M, N, K);
  tc::Params p;
  p.x = A; p.wpk = w_tc; p.bias = bias; p.res = res; p.y = C;
  p.N = 1; p.Hin = 1; p.Win = 1; p.Cin = K; p.Hout = 1; p.Wout = (int)M; p.Cout = N;
  if (M > 0x7fffffff) return fail(MAS_ERR_UNSUPPORTED, "tc gemm: M too large");
  p.map = tc::MAP_ROWS;
  p.ldx = lda; p.ldy = ldc;
  p.tiles_x = 1; p.tiles_y = 1;
  p.total_tiles = cdiv(M, tc::BM);
  p.alpha = alpha;
  p.gn_table = nullptr; p.gn_silu = 0; p.stats_part = stats_part; p.x_amax = nullptr; p.Cstore = N;
  if (stats_part && (M % tc::BM || ldc != N)) return fail(MAS_ERR_UNSUPPORTED, "tc gemm: fused statistics need M %% 128 == 0 and a dense output");
  constexpr size_t smem = tc::smem_bytes<1, 32, 2, 2, false>();
  static std::atomic<uint64_t> configured{0};
  if (first_on_device(configured)) {
    if (int e = set_smem(tc::shift_gemm_tc<1, 32, 2, 2, false>, smem)) return e;
    mark_device(configured);
  }
  dim3 grid((unsigned)cdiv(p.total_tiles, 2), (unsigned)(N / tc::BN));
  tc::shift_gemm_tc<1, 32, 2, 2, false><<<grid, tc::NTHREADS, smem, st>>>(p);
  return launched_tc("shift_gemm_tc<1>");
}

int gemm_tc_launch(const float*, const float*, float*, int, int, int, int, int64_t, int64_t, int64_t, int64_t, int64_t, int64_t, int, int,
                   float, const float*, const float*, cudaStream_t) {
  return fail(MAS_ERR_UNSUPPORTED, "tc gemm with un-packed B operand: not available (use mas_gemm_rows_packed)");
}
// pad_ok: dys.c may be any multiple of 4 - the caller has sized dw / dbias / workspace for round_up(dys.c, 128) rows
static bool wgrad_tc_ok(const mas_tensor4& xs, const mas_tensor4& dys, int mode, bool pad_ok = false) {
  if (!(mode == MAS_CONV_S1 || mode == MAS_CONV_UP)) return false;
  if (!dense_nhwc(xs) || !dense_nhwc(dys) || xs.c % tc::WG_NT || dys.c % (pad_ok ? 4 : tc::BM) || dys.h % 8 || dys.w % 8) return false;
  int64_t eh = (mode == MAS_CONV_S1) ? xs.h : 2 * xs.h, ew = (mode == MAS_CONV_S1) ? xs.w : 2 * xs.w;
  return dys.h == eh && dys.w == ew && xs.n == dys.n;
}
static int wgrad_tc_splits(int64_t cps, int64_t units) {
  int64_t s = NUM_SMS / cps;
  if (s < 1) s = 1;
  if (s > units) s = units;
  const int64_t ups = cdiv(units, s);
  return (int)cdiv(units, ups);  // every split owns at least one unit
}
size_t conv_wgrad_t16_ws(mas_tensor4 xs, mas_tensor4 dys);   // conv_tma.cu: the shadow-fed kernel splits differently
bool conv_wgrad_t16_ok(mas_tensor4 xs, mas_tensor4 dys);
bool conv3x3_phase_ok(mas_tensor4 xs, mas_tensor4 ys, bool up);   // conv_tma.cu
int conv_wgrad_t16_launch(const void* x16, mas_tensor4 xs, const void* dy16, mas_tensor4 dys, float* dw, float* dbias,
                          const float* dy_amax, void* ws, size_t ws_bytes, cudaStream_t st);
size_t conv_wgrad_tc_ws(mas_tensor4 xs, mas_tensor4 dys, int mode) {
  if (!wgrad_tc_ok(xs, dys, mode, true)) return 0;
  const int64_t coutk = cdiv(dys.c, tc::BM) * tc::BM;
  size_t splits = wgrad_tc_splits((coutk / tc::BM) * (xs.c / tc::WG_NT), dys.n * (dys.h / 8) * (dys.w / 8));
  const size_t a = splits * 9 * (size_t)coutk * xs.c * sizeof(float) + splits * (size_t)coutk * sizeof(float) + 256;
  const size_t b = mode == MAS_CONV_S1 ? conv_wgrad_t16_ws(xs, dys) : 0;
  return a > b ? a : b;
}
PFN_cuTensorMapEncodeTiled tensor_map_encoder() {   // also used by conv_tma.cu
  static PFN_cuTensorMapEncodeTiled fn = nullptr;
  if (!fn) {
    void* ptr = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &ptr, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_cuTensorMapEncodeTiled>(ptr);
  }
  return fn;
}
// dy tile map: 3x3 -> rank 4 (co, x, y, n), box (128, 8, 8, 1); 1x1 -> rank 2 (co, row), box (128, 64)
static int make_dy_map(CUtensorMap* map, const tc::WParams& p, int taps) {
  PFN_cuTensorMapEncodeTiled enc = tensor_map_encoder();
  if (!enc) return fail(MAS_ERR_LAUNCH, "cuTensorMapEncodeTiled entry point not available");
  CUresult r;
  if (taps == 9) {
    const cuuint64_t eb = p.dy_f16 ? 2 : 4;
    cuuint64_t dims[4] = {(cuuint64_t)p.Cout_real, (cuuint64_t)p.W, (cuuint64_t)p.H, (cuuint64_t)p.N};
    cuuint64_t strides[3] = {(cuuint64_t)p.Cout_real * eb, (cuuint64_t)p.W * p.Cout_real * eb, (cuuint64_t)p.H * p.W * p.Cout_real * eb};
    cuuint32_t box[4] = {128, 8, 8, 1}, es[4] = {1, 1, 1, 1};
    r = enc(map, p.dy_f16 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT16 : CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, (void*)p.dy, dims, strides, box, es,
            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  } else {
    cuuint64_t dims[2] = {(cuuint64_t)p.Cout_real, (cuuint64_t)p.rows};
    cuuint64_t strides[1] = {(cuuint64_t)p.ldy * 4};
    cuuint32_t box[2] = {128, 64}, es[2] = {1, 1};
    r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, (void*)p.dy, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
            CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  }
  if (r != CUDA_SUCCESS) return fail(MAS_ERR_LAUNCH, "cuTensorMapEncodeTiled failed (%d)", (int)r);
  return MAS_OK;
}

template <int TAPS, bool PRO, bool F16>
static int wgrad_tc_run(tc::WParams& p, int splits, float* dw, float* dbias, void* ws, cudaStream_t st) {
  p.part = (float*)ws;
  p.bpart = dbias ? (float*)ws + (size_t)splits * TAPS * p.Cout * p.Cin : nullptr;
  p.units_per_split = cdiv(p.total_units, splits);
  constexpr int NT = (TAPS == 9) ? tc::WG_NT : 128;
  constexpr size_t bstage = F16 ? (size_t)12 * (tc::WG_SLOTS * 16 + 32) : (size_t)(TAPS == 9 ? 3 * 20 : 16) * NT * 16;
  constexpr size_t smem = (size_t)tc::WG_STAGES * (bstage + tc::WG_DY_STAGE) + (4 * tc::WG_STAGES + 1) * 8 + 16;
  static std::atomic<uint64_t> configured{0};
  if (first_on_device(configured)) {
    if (int e = set_smem(tc::wgrad_tc<TAPS, PRO, F16>, smem)) return e;
    mark_device(configured);
  }
  CUtensorMap dy_map;
  if (int e = make_dy_map(&dy_map, p, TAPS)) return e;
  dim3 grid((unsigned)(p.Cin / NT), (unsigned)(p.Cout / tc::BM), (unsigned)splits);
  tc::wgrad_tc<TAPS, PRO, F16><<<grid, tc::WG_THREADS, smem, st>>>(p, dy_map);
  if (int e = launched_tc("wgrad_tc")) return e;
  conv_wgrad_reduce_launch((const float*)ws, splits, TAPS, p.Cout, p.Cin, dw, p.bpart, dbias, st);  // + bias partials -> dbias
  return launched("conv_wgrad_reduce");
}
// dbias (may be null) is produced here too when the tensor path runs.
bool conv_wgrad_tc_eligible(mas_tensor4 xs, mas_tensor4 dys, int mode) { return wgrad_tc_ok(xs, dys, mode); }
int conv_wgrad_tc_launch(const float* x, mas_tensor4 xs, const float* dy, mas_tensor4 dys, float* dw, float* dbias, int mode,
                         const float* gn_table, int gn_silu, int f16, const float* dy_amax, int cout_rows, int x_f16, void* ws,
                         size_t ws_bytes, cudaStream_t st) {
  const int dy_f16 = (x_f16 >> 1) & 1;   // operand flags: bit 0 = x holds fp16, bit 1 = dy is the scaled fp16 shadow
  x_f16 &= 1;
  if (x_f16 && (!f16 || gn_table)) return fail(MAS_ERR_INVALID_ARG, "tc wgrad: an fp16 x needs the fp16-operand kernel and no prologue");
  if (dy_f16 && (!f16 || !dy_amax || dys.c % 8)) return fail(MAS_ERR_INVALID_ARG, "tc wgrad: an fp16 dy needs the fp16-operand kernel, its scale source and Cout %% 8 == 0");
  // both operands as fp16 shadows: the pure TMA + MMA kernel (conv_tma.cu); MAS_WGRAD_TMA=0 keeps the register-staged one
  static const bool tma_off = [] { const char* e = getenv("MAS_WGRAD_TMA"); return e && e[0] == '0'; }();
  if (f16 && x_f16 && dy_f16 && mode == MAS_CONV_S1 && !gn_table && !tma_off && conv_wgrad_t16_ok(xs, dys) &&
      cout_rows == (int)(cdiv(dys.c, tc::BM) * tc::BM))
    return conv_wgrad_t16_launch(x, xs, dy, dys, dw, dbias, dy_amax, ws, ws_bytes, st);
  // cout_rows: rows of dw / dbias the caller allocated; padding (dys.c % 128 != 0) only when it equals round_up(dys.c, 128)
  const bool pad_ok = cout_rows == (int)(cdiv(dys.c, tc::BM) * tc::BM);
  if (!wgrad_tc_ok(xs, dys, mode, pad_ok) || !al16p(x) || !al16p(dy)) return fail(MAS_ERR_UNSUPPORTED, "tc wgrad: shape/layout not eligible");
  if (ws_bytes < conv_wgrad_tc_ws(xs, dys, mode)) return fail(MAS_ERR_WORKSPACE, "tc wgrad: workspace too small");
  tc::WParams p;
  p.x = x; p.dy = dy;
  // dys.c not a multiple of 128: dw / dbias must hold round_up(dys.c, 128) output channels (the extra rows come out zero)
  p.N = (int)xs.n; p.Hin = (int)xs.h; p.Win = (int)xs.w; p.Cin = (int)xs.c; p.H = (int)dys.h; p.W = (int)dys.w;
  p.Cout = (int)(cdiv(dys.c, tc::BM) * tc::BM); p.Cout_real = (int)dys.c;
  p.map = (mode == MAS_CONV_S1) ? tc::MAP_S1 : tc::MAP_UP;
  p.units_x = (int)(dys.w / 8); p.units_y = (int)(dys.h / 8);
  p.total_units = (int64_t)p.N * p.units_x * p.units_y;
  p.rows = 0; p.ldx = p.Cin; p.ldy = p.Cout_real;
  p.gn_table = gn_table; p.gn_silu = gn_silu; p.dy_amax = f16 ? dy_amax : nullptr; p.x_f16 = x_f16; p.dy_f16 = dy_f16;
  const int splits = wgrad_tc_splits((p.Cout / tc::BM) * (xs.c / tc::WG_NT), p.total_units);
  if (f16) return gn_table ? wgrad_tc_run<9, true, true>(p, splits, dw, dbias, ws, st) : wgrad_tc_run<9, false, true>(p, splits, dw, dbias, ws, st);
  return gn_table ? wgrad_tc_run<9, true, false>(p, splits, dw, dbias, ws, st) : wgrad_tc_run<9, false, false>(p, splits, dw, dbias, ws, st);
}
static bool wgrad1_tc_ok(const float* x, int64_t ldx, const float* dy, int64_t ldy, int Cin, int Cout) {
  return Cin % 128 == 0 && Cout % tc::BM == 0 && ldx % 4 == 0 && al16p(x) && dy != nullptr && ldy >= Cout && ldy % 4 == 0 && al16p(dy);
}
size_t conv1x1_wgrad_tc_ws(int64_t M, int Cin, int Cout) {
  if (Cin % 128 || Cout % tc::BM) return 0;
  size_t splits = wgrad_tc_splits((int64_t)(Cout / tc::BM) * (Cin / 128), cdiv(M, 64));
  return splits * (size_t)Cout * Cin * sizeof(float) + splits * (size_t)Cout * sizeof(float) + 256;
}
int conv1x1_wgrad_tc_launch(const float* x, int64_t ldx, const float* dy, int64_t ldy, int64_t M, int Cin, int Cout, float* dw,
                            float* dbias, void* ws, size_t ws_bytes, cudaStream_t st) {
  if (!wgrad1_tc_ok(x, ldx, dy, ldy, Cin, Cout)) return fail(MAS_ERR_UNSUPPORTED, "tc wgrad 1x1: shape not eligible");
  if (ws_bytes < conv1x1_wgrad_tc_ws(M, Cin, Cout)) return fail(MAS_ERR_WORKSPACE, "tc wgrad 1x1: workspace too small");
  tc::WParams p;
  p.x = x; p.dy = dy;
  p.N = 1; p.Hin = 1; p.Win = 1; p.Cin = Cin; p.H = 1; p.W = 1; p.Cout = Cout; p.Cout_real = Cout; p.map = tc::MAP_ROWS;
  p.units_x = 1; p.units_y = 1;
  p.total_units = cdiv(M, 64);
  p.rows = M; p.ldx = ldx; p.ldy = ldy;
  p.gn_table = nullptr; p.gn_silu = 0; p.dy_amax = nullptr; p.x_f16 = 0; p.dy_f16 = 0;
  const int splits = wgrad_tc_splits((int64_t)(Cout / tc::BM) * (Cin / 128), p.total_units);
  return wgrad_tc_run<1, false, false>(p, splits, dw, dbias, ws, st);
}

}  // namespace mas

using namespace mas;

extern "C" {

int mas_pack_conv3x3_tc(const float* w_oihw, float* w_tc, int Cout, int Cin, int transpose, void* stream) {
  const int N = transpose ? Cin : Cout, K = transpose ? Cout : Cin;
  if (N % tc::BN || K % 8) return fail(MAS_ERR_UNSUPPORTED, "pack_conv3x3_tc: N=%d must be a multiple of 128 and K=%d of 8", N, K);
  int64_t total = (int64_t)9 * Cout * Cin;
  tc::pack_weights_tc<<<(int)(cdiv(total, 256) < 2368 ? cdiv(total, 256) : 2368), 256, 0, S(stream)>>>(w_oihw, w_tc, Cout, Cin, 9, 8, transpose);
  return launched("pack_weights_tc<9>");
}

int mas_pack_conv3x3_tc_pair(const float* w_oihw, float* w_tc_fwd, float* w_tc_dgrad, int Cout, int Cin, void* stream) {
  if (Cout % tc::BN || Cin % tc::BN) return fail(MAS_ERR_UNSUPPORTED, "pack_conv3x3_tc_pair: Cout=%d and Cin=%d must be multiples of 128", Cout, Cin);
  int64_t total = (int64_t)9 * Cout * Cin;
  tc::pack_weights_tc_pair<<<(int)(cdiv(total, 256) < 2368 ? cdiv(total, 256) : 2368), 256, 0, S(stream)>>>(w_oihw, w_tc_fwd, w_tc_dgrad, Cout, Cin);
  return launched("pack_weights_tc_pair");
}

int mas_pack_conv3x3_tc16(const float* w_oihw, void* w_tc16, void* w_tc16_dgrad, int Cout, int Cin, int transpose, void* stream) {
  // transpose selects the packing written to w_tc16 when w_tc16_dgrad is null; with w_tc16_dgrad both are produced
  const bool both = w_tc16_dgrad != nullptr;
  const int N = (transpose && !both) ? Cin : Cout, K = (transpose && !both) ? Cout : Cin;
  if (N % tc::BN || K % 16 || (both && (Cin % tc::BN || Cout % 16)))
    return fail(MAS_ERR_UNSUPPORTED, "pack_conv3x3_tc16: N must be a multiple of 128 and K of 16 (Cout=%d Cin=%d)", Cout, Cin);
  int64_t total = (int64_t)9 * Cout * Cin;
  tc::pack_weights_tc16<<<(int)(cdiv(total, 256) < 2368 ? cdiv(total, 256) : 2368), 256, 0, S(stream)>>>(
      w_oihw, (__half*)w_tc16, (__half*)w_tc16_dgrad, Cout, Cin, 9, 16, transpose, both ? 1 : 0);
  return launched("pack_weights_tc16<9>");
}

int mas_pack_gemm_tc16(const float* w_nk, void* w_tc16, int N, int K, int transpose, void* stream) {
  // fp16 image for mas_gemm_rows_f16 (gemm_tma.cu): [n_tile][k/16][2][128][8 halves]; w_nk: [N_out][K_in] row-major
  // (nn.Linear / 1x1 convolution weight); transpose=1 packs the data-gradient operand W^T
  if (!w_nk || !w_tc16 || N <= 0 || K <= 0) return fail(MAS_ERR_INVALID_ARG, "pack_gemm_tc16: bad arguments");
  const int Nn = transpose ? K : N, Kk = transpose ? N : K;
  if (Nn % tc::BN || Kk % 64)
    return fail(MAS_ERR_UNSUPPORTED, "pack_gemm_tc16: output features (%d) must be a multiple of 128 and the contraction (%d) of 64", Nn, Kk);
  const int64_t total = (int64_t)N * K;
  tc::pack_weights_tc16<<<(int)(cdiv(total, 256) < 2368 ? cdiv(total, 256) : 2368), 256, 0, S(stream)>>>(w_nk, (__half*)w_tc16, nullptr, N, K, 1, 16,
                                                                                                     transpose, 0);
  return launched("pack_weights_tc16<1>");
}

int mas_pack_gemm_tc(const float* w_nk, float* w_tc, int N, int K, int transpose, void* stream) {
  // w_nk: [N_out][K_in] row-major (a 1x1 convolution weight); transpose=1 packs the [K_in -> N] data-gradient operand
  const int Nn = transpose ? K : N, Kk = transpose ? N : K;
  if (Nn % tc::BN || Kk % 32) return fail(MAS_ERR_UNSUPPORTED, "pack_gemm_tc: N=%d must be a multiple of 128 and K=%d of 32", Nn, Kk);
  int64_t total = (int64_t)N * K;
  tc::pack_weights_tc<<<(int)(cdiv(total, 256) < 2368 ? cdiv(total, 256) : 2368), 256, 0, S(stream)>>>(w_nk, w_tc, N, K, 1, 32, transpose);
  return launched("pack_weights_tc<1>");
}

int mas_gemm_rows_packed(const float* A, int64_t lda, const float* w_tc, float* C, int64_t ldc, int64_t M, int N, int K, float alpha,
                         const float* bias, const float* residual, float* stats_part, void* stream) {
  MAS_REQUIRE(A && w_tc && C && M > 0, "gemm_rows_packed: bad arguments");
  return gemm_rows_tc_launch(A, lda, w_tc, C, ldc, M, N, K, alpha, bias, residual, stats_part, S(stream));
}

int mas_tc_probe(const float* A, const float* B, float* D, int a_src, int b_layout, uint64_t raw_desc, uint32_t raw_idesc,
                 int raw_off, void* stream) {
  (void)raw_idesc;
  tc::mma_probe<<<1, 128, 0, S(stream)>>>(A, B, D, a_src, b_layout, (unsigned long long)raw_desc, raw_off);
  return launched_tc("mma_probe");
}

int mas_tc_probe16(float* D, uint64_t raw_desc, uint32_t raw_idesc, int raw_off, void* stream) {
  // raw_idesc: bit 16 = MN-major B, bits 17-22 = N / 8 (32 or 128; D is 128 x N)
  const int n = (int)((raw_idesc >> 17) & 0x3F) * 8;
  if (n != 32 && n != 128) return fail(MAS_ERR_INVALID_ARG, "tc_probe16: N must be 32 or 128 (got %d)", n);
  tc::mma_probe16<<<1, 128, 0, S(stream)>>>(D, (unsigned long long)raw_desc, (int)((raw_idesc >> 16) & 1), n, raw_off);
  return launched_tc("mma_probe16");
}

int mas_conv3x3_tc_eligible(mas_tensor4 xs, mas_tensor4 ys, int mode) {
  const int Cin = (int)xs.c, Cout = (int)ys.c;
  if (mode == MAS_CONV_UP_PHASE || mode == MAS_CONV_S2_PHASE) return conv3x3_phase_ok(xs, ys, mode == MAS_CONV_UP_PHASE) ? 1 : 0;
  if (!(mode == MAS_CONV_S1 || mode == MAS_CONV_UP || mode == MAS_CONV_ZS)) return 0;
  // (the launch itself also takes Cout % 4 == 0 with weights / bias padded to the next multiple of 128: an explicit path of
  //  the caller, see mas_conv3x3_fprop_tc16; "eligible" means no padding is needed)
  if (!dense_nhwc(xs) || !dense_nhwc(ys) || Cin % 8 || Cout % tc::BN || ys.h % 16 || ys.w % 8) return 0;
  return 1;
}

int mas_conv3x3_fprop_tc(const float* x, mas_tensor4 xs, const float* w_tc, const float* bias, const float* residual, float* y,
                         mas_tensor4 ys, int mode, const float* gn_table, int gn_silu, float* stats_part, void* stream) {
  MAS_REQUIRE(x && w_tc && y, "conv3x3_fprop_tc: null pointer");
  return conv3x3_fprop_tc_launch(x, xs, w_tc, bias, residual, y, ys, mode, gn_table, gn_silu, stats_part, 0, nullptr, S(stream));
}

int mas_conv3x3_fprop_tc16(const float* x, mas_tensor4 xs, const void* w_tc16, const float* bias, const float* residual, float* y,
                           mas_tensor4 ys, int mode, const float* gn_table, int gn_silu, float* stats_part, const float* x_amax,
                           void* stream) {
  MAS_REQUIRE(x && w_tc16 && y, "conv3x3_fprop_tc16: null pointer");
  return conv3x3_fprop_tc_launch(x, xs, (const float*)w_tc16, bias, residual, y, ys, mode, gn_table, gn_silu, stats_part, 1, x_amax,
                                 S(stream));
}

}  // extern "C"
