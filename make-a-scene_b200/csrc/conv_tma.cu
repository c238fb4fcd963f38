// 3x3 stride-1 convolution (fprop / data gradient) as a pure TMA + wgmma kernel: the A operand comes from an fp16 "shadow"
// of the activation (written channels-last by the producing kernel: GroupNorm(+SiLU) apply in the forward pass, GroupNorm
// backward in the backward pass) instead of being converted by producer warps.
//
//   * one persistent CTA per SM walks work items (pair of 128-pixel tiles x 128 output channels);
//   * A: ONE cp.async.bulk.tensor (4-D map over [N][H][W][C] halves, box 1 x 18 x 10 x 64, 128-byte swizzle, out-of-image
//     halo pixels zero-filled by the copy engine) per tile per 64-channel chunk.  The staged halo is [180 pixels][128 B];
//     the nine taps and the four K = 16 steps of the chunk are descriptor start-address shifts ((ty*10+tx)*128 + k*32 bytes)
//     over that one copy: the 8-row core group is eight horizontally adjacent pixels, the group stride (SBO) one staged image
//     row = 1280 B;
//   * B (weights): the same pre-packed no-swizzle stages as shift_gemm_tc (mas_pack_conv3x3_tc16), one bulk copy per
//     16-channel step, ring of three;
//   * operand roles are swapped (D^T = W x X^T: the packed weights are the M-side operand, the pixels the N side of
//     wgmma.m64n256k16 / two m64n128k16): warpgroup g owns output channels 64 g .. 64 g + 63 of the tile, so bias and
//     GroupNorm statistics are per-row scalars of the accumulator fragment;
//   * warps 0-7 MMA + epilogue (two warpgroups), warp 8 copy issuer (its warpgroup hands its registers to the MMA ones): no
//     thread of the CTA touches the operands; the copy issuer fills the rings of the next item while the warpgroups store the current one.
//
// Reference call sites replaced: nn.Conv2d 3x3 stride 1 (modules.py:93-104) forward and its data gradient.
//
// Phase-decomposed form (PH != 0) of the resampling convolutions, on the same kernel with a per-launch tap table:
//   * Upsample (nearest x2, then 3x3): output phase (py, px) is a 2 x 2 convolution of the LOW-resolution input with the taps
//     summed per phase (per dimension, phase 0 reads offsets {-1: w0, 0: w1 + w2}, phase 1 {0: w0 + w1, +1: w2}): 4 taps per
//     output pixel instead of 9;
//   * Downsample ((0,1,0,1) pad, 3x3 stride 2): input phase plane (py, px) = x[2 i + py][2 j + px] holds 4 / 2 / 2 / 1 of the
//     nine taps, each at offset (ty >> 1, tx >> 1): 9 taps per output pixel instead of 36 on a space-to-depth map;
//   * PH 1 "phase-out": one dense source, the item's output phase selects the taps, the epilogue writes that phase plane of
//     the 2x output (Upsample forward, Downsample data gradient); PH 2 "phase-in": the K loop runs over the four phase planes
//     of a 2x source (a 5-D tensor map with doubled pixel / row strides: nothing is materialised; out-of-image zero fill gives
//     the borders and the Downsample pad) and each plane's taps, into a dense output (Downsample forward, Upsample data
//     gradient).
#include <cuda.h>
#include <cudaTypedefs.h>
#include <cuda_fp16.h>
#include <stdlib.h>

#include "mas_common.cuh"
#include "tc_ptx.cuh"
#include "wgmma.cuh"

namespace mas {

PFN_cuTensorMapEncodeTiled tensor_map_encoder();   // contract_tc.cu

namespace tc {

constexpr int T_MMA_WARPS = 8;
constexpr int T_THREADS = (T_MMA_WARPS + 4) * 32;   // + the copy-issuing warpgroup
constexpr int T_ASTAGES = 2, T_BSTAGES = 3;
constexpr int T_ATILE = 23 * 1024;                  // 18 x 10 halo pixels x 128 B = 23040, padded to the 1024-byte swizzle atom
constexpr int T_ASTAGE = 2 * T_ATILE;               // pair of 16 x 8 tiles, or one 32 x 8 tile (34 x 10 halo = 43520 B)
constexpr int T_BSTAGE = 9 * 2 * BN * 16;           // nine taps x 16 channels x 128 output channels (fp16)

struct HParams {
  const void* wpk;    // mas_pack_conv3x3_tc16 packing
  const float* bias;  // [Cout] or null
  const float* res;   // NHWC fp32 like y, or null
  float* y;
  int N, H, W, Cin, Cout, Cstore;
  int64_t ldy;
  int tiles_x, tiles_y;   // 16 x 8 tiles per image row / column
  int64_t units;          // work units of 256 pixels: 32 x 8 tiles (TALL) or pairs of consecutive 16 x 8 tiles
  float* stats_part;   // GroupNorm-statistics epilogue (see shift_gemm_tc), or null
  const float* x_amax; // amax the shadow's power-of-two scale was derived from (null: unscaled shadow)
  int64_t ysn, ysh, ysw;    // element strides of y per image / tile-grid row / tile-grid column
  // phase forms only: per tap group (output phase for PH 1, source plane for PH 2) the staged-halo offsets (ty * 10 + tx)
  // of its four taps and (PH 1) the element offset of its output plane
  int ph_hoff[4][4];
  int64_t ph_yoff[4];
};

// 16 x 8 tile (n, ty, tx) of half `hf` of work unit `u`; false when the unit's second tile does not exist (odd tile count)
template <bool TALL>
__device__ __forceinline__ bool unit_tile(const HParams& p, int64_t u, int hf, int& n, int& ty, int& tx) {
  if (TALL) {
    const int ty2 = p.tiles_y >> 1;
    tx = (int)(u % p.tiles_x);
    ty = (int)((u / p.tiles_x) % ty2) * 2 + hf;
    n = (int)(u / ((int64_t)p.tiles_x * ty2));
    return true;
  }
  const int64_t total = (int64_t)p.N * p.tiles_x * p.tiles_y;
  int64_t t = u * 2 + hf;
  const bool live = t < total;
  if (!live) t = total - 1;
  tx = (int)(t % p.tiles_x);
  ty = (int)((t / p.tiles_x) % p.tiles_y);
  n = (int)(t / ((int64_t)p.tiles_x * p.tiles_y));
  return live;
}

// TALL: the unit is one 32 x 8 tile whose staged halo (34 x 10 pixels, uniform 1280-byte row pitch) is ONE N = 256 operand:
// per K = 16 step and tap a single m64n256 MMA per warpgroup instead of two m64n128 ones over the two halos of a pair.
// PH: 0 the nine taps of a stride-1 3x3 convolution, 1 phase-out, 2 phase-in (see the top of the file).
template <bool TALL, int PH = 0>
__global__ void __launch_bounds__(T_THREADS, 1) shift_gemm_t16(const HParams p, const __grid_constant__ CUtensorMap x_map) {
  constexpr int TAPS = PH == 0 ? 9 : 4;              // phase forms: groups with fewer taps carry zero weights
  constexpr int GOUT = PH == 1 ? 4 : 1;              // output phases per work unit
  constexpr int KPL = PH == 2 ? 4 : 1;               // source planes per K loop
  constexpr int LBO_B = BN * 16, B_TAP = 2 * LBO_B;
  constexpr int A_BYTES = TALL ? 34 * 10 * 128 : 2 * 18 * 10 * 128;

  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_base = smem_u32(smem_raw);
  const uint32_t smem_base = (raw_base + 1023u) & ~1023u;           // swizzle atoms are 1024-byte aligned
  uint8_t* smem = smem_raw + (smem_base - raw_base);
  const uint32_t a_base = smem_base;
  const uint32_t b_base = a_base + T_ASTAGES * T_ASTAGE;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + T_ASTAGES * T_ASTAGE + T_BSTAGES * T_BSTAGE);
  const uint32_t bar_base = smem_u32(bars);
  auto afull = [&](int s) { return bar_base + 8u * s; };
  auto aempty = [&](int s) { return bar_base + 8u * (T_ASTAGES + s); };
  auto bfull = [&](int s) { return bar_base + 8u * (2 * T_ASTAGES + s); };
  auto bempty = [&](int s) { return bar_base + 8u * (2 * T_ASTAGES + T_BSTAGES + s); };

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int achunks = p.Cin / 64;
  const int kiters = KPL * achunks;
  const int n_tiles = p.Cout / BN;
  const int64_t nitems = p.units * n_tiles * GOUT;   // channel tile (then output phase) fastest: a unit's halo is re-read from L2

  if (tid == 0) {
    for (int s = 0; s < T_ASTAGES; ++s) { mbar_init(afull(s), 1); mbar_init(aempty(s), T_MMA_WARPS * 32); }
    for (int s = 0; s < T_BSTAGES; ++s) { mbar_init(bfull(s), 1); mbar_init(bempty(s), T_MMA_WARPS * 32); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < T_MMA_WARPS) {
    wg::regs_inc<wg::MMA_REGS>();
    // ===================== MMA warpgroups, then epilogue =====================
    // acc[64 h + 4 j + 2 i + c] = D^T[channel 64 wgi + 16 (warp % 4) + lane / 4 + 8 i][pixel 128 h + 8 j + 2 (lane % 4) + c]
    float inv_scale = 1.f;
    operand_scale(p.x_amax, &inv_scale);
    const float alpha = inv_scale;
    const int wgi = warp >> 2;
    const int frow = wgi * 64 + (warp & 3) * 16 + (lane >> 2), fcol = 2 * (lane & 3);
    int as = 0, bs = 0, prev_b = 0, prev_a = -1;
    uint32_t aph = 0, bph = 0;
    float acc[128];
    for (int64_t item = blockIdx.x; item < nitems; item += gridDim.x) {
      const int gout = PH == 1 ? (int)((item / n_tiles) % GOUT) : 0;
      for (int kk = 0; kk < kiters; ++kk) {
        const int grp = PH == 2 ? kk / achunks : gout;
        mbar_wait(afull(as), aph);
        const uint64_t xd0 = wg::desc(a_base + (uint32_t)as * T_ASTAGE, 16, 1280, wg::SW_128);
#pragma unroll 1
        for (int sub = 0; sub < 4; ++sub) {
          mbar_wait(bfull(bs), bph);
          const uint64_t wd0 = wg::desc(b_base + (uint32_t)bs * T_BSTAGE + (uint32_t)(wgi * 1024), LBO_B, 128);
          const uint64_t xds = xd0 + (uint64_t)((sub * 32) >> 4);
          const uint32_t acc0 = (kk > 0 || sub > 0) ? 1u : 0u;
          wg::fence();
#pragma unroll
          for (int t = 0; t < TAPS; ++t) {
            const uint32_t tapoff = (uint32_t)((PH == 0 ? (t / 3) * 10 + (t % 3) : p.ph_hoff[grp][t]) * 128);
            const uint64_t wd = wd0 + (uint64_t)((t * B_TAP) >> 4);
            const uint64_t xd = xds + (uint64_t)(tapoff >> 4);
            // D^T = W x X^T: weights on the M side, pixels on the N side
            if (TALL) {
              wg::wgmma_f16_ss_n256<0, 0>(acc, wd, xd, t > 0 ? 1u : acc0);
            } else {
              wg::wgmma_f16_ss_n128<0, 0>(acc, wd, xd, t > 0 ? 1u : acc0);
              wg::wgmma_f16_ss_n128<0, 0>(acc + 64, wd, xd + (uint64_t)(T_ATILE >> 4), t > 0 ? 1u : acc0);
            }
          }
          wg::commit();
          // the previous step's MMAs have read their weight stage (and, after a chunk's last step, its halo stage)
          wg::wait<1>();
          if (kk > 0 || sub > 0) {
            mbar_arrive(bempty(prev_b));
            if (prev_a >= 0) mbar_arrive(aempty(prev_a));
          }
          prev_b = bs;
          prev_a = (sub == 3) ? as : -1;
          if (++bs == T_BSTAGES) { bs = 0; bph ^= 1; }
        }
        if (++as == T_ASTAGES) { as = 0; aph ^= 1; }
      }
      wg::wait<0>();
      wg::fence_regs<128>(acc);
      mbar_arrive(bempty(prev_b));
      mbar_arrive(aempty(prev_a));

      const int ch_tile = (int)(item % n_tiles) * BN;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        int n_img, ty_, tx_;
        const bool live = unit_tile<TALL>(p, item / (n_tiles * GOUT), h, n_img, ty_, tx_);   // block-uniform
        if (!live) continue;
        const int64_t pix0 = ((int64_t)n_img * p.H + ty_ * 16) * p.W + tx_ * 8;
        const int64_t cstep = PH == 0 ? p.ldy : p.ysw;
        const int64_t ybase = PH == 0 ? 0 : n_img * p.ysn + (ty_ * 16) * p.ysh + (tx_ * 8) * p.ysw + (PH == 1 ? p.ph_yoff[gout] : 0);
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const int ch = ch_tile + frow + 8 * i;
          const bool st_ok = ch < p.Cstore;
          const float bv = (p.bias && st_ok) ? __ldg(p.bias + ch) : 0.f;
#pragma unroll
          for (int cb = 0; cb < 4; ++cb) {         // 32-pixel groups = four image rows of the 16 x 8 tile
            float st_s = 0.f, st_q = 0.f;
#pragma unroll
            for (int jj = 0; jj < 4; ++jj) {
              const int j = cb * 4 + jj;           // pixel row j of the tile, columns fcol, fcol + 1
              const int64_t off = PH == 0 ? (pix0 + (int64_t)j * p.W + fcol) * p.ldy + ch : ybase + j * p.ysh + fcol * p.ysw + ch;
#pragma unroll
              for (int cc = 0; cc < 2; ++cc) {
                float o = fmaf(acc[64 * h + 4 * j + 2 * i + cc], alpha, bv);
                if (st_ok) {
                  if (p.res) o += __ldg(p.res + off + cc * cstep);
                  p.y[off + cc * cstep] = o;
                  st_s += o;
                  st_q = fmaf(o, o, st_q);
                }
              }
            }
            if (p.stats_part) {   // same partial layout as shift_gemm_tc: [16 x 8 tile][32-pixel group][channel quad][sum, sumsq]
              st_s += __shfl_xor_sync(0xffffffffu, st_s, 1);   // the four lanes of a channel row: all 32 pixels
              st_q += __shfl_xor_sync(0xffffffffu, st_q, 1);
              st_s += __shfl_xor_sync(0xffffffffu, st_s, 2);
              st_q += __shfl_xor_sync(0xffffffffu, st_q, 2);
              st_s += __shfl_xor_sync(0xffffffffu, st_s, 4);   // four consecutive channel rows: the quad
              st_q += __shfl_xor_sync(0xffffffffu, st_q, 4);
              st_s += __shfl_xor_sync(0xffffffffu, st_s, 8);
              st_q += __shfl_xor_sync(0xffffffffu, st_q, 8);
              if ((lane & 15) == 0) {
                const size_t tile = ((size_t)n_img * p.tiles_y + ty_) * p.tiles_x + tx_;
                float* sp = p.stats_part + ((tile * 4 + cb) * (p.Cout >> 2) + (ch >> 2)) * 2;
                sp[0] = st_s;
                sp[1] = st_q;
              }
            }
          }
        }
      }
    }
  } else {
    // ===================== copy issuer (one thread): halos by tensor map, weight stages by bulk copy =====================
    wg::regs_dec<wg::COPY_REGS>();
    if (warp == T_MMA_WARPS && lane == 0) {
      int as = 0, bs = 0;
      uint32_t aph = 0, bph = 0;
      const int kchunks = p.Cin / 16;
      for (int64_t item = blockIdx.x; item < nitems; item += gridDim.x) {
        const int gout = PH == 1 ? (int)((item / n_tiles) % GOUT) : 0;
        const int64_t unit = item / (n_tiles * GOUT);
        constexpr uint32_t bstage = TAPS * B_TAP;
        const uint8_t* wsrc0 = reinterpret_cast<const uint8_t*>(p.wpk) + (size_t)(item % n_tiles) * kchunks * bstage;
        for (int kk = 0; kk < kiters; ++kk) {
          const int grp = PH == 2 ? kk / achunks : gout, c = kk % achunks;
          // phase forms: one weight image per tap group, [group][n_tile][16-channel K step][4 taps][k / 8][128][8 halves]
          const uint8_t* wsrc = PH == 0 ? wsrc0 : wsrc0 + (size_t)grp * (p.Cout / BN) * kchunks * bstage;
          mbar_wait(aempty(as), aph ^ 1);
          mbar_expect_tx(afull(as), A_BYTES);
#pragma unroll
          for (int hf = 0; hf < (TALL ? 1 : 2); ++hf) {
            int n, ty_, tx_;
            unit_tile<TALL>(p, unit, hf, n, ty_, tx_);   // a missing second tile re-reads the last one (never stored)
            const uint32_t dst = a_base + (uint32_t)(as * T_ASTAGE + hf * T_ATILE);
            if (PH == 2)   // plane (py, px) = grp: channel half px of the pixel pair, row parity py
              tma_load_5d(dst, &x_map, (grp & 1) * p.Cin + c * 64, tx_ * 8 - 1, grp >> 1, ty_ * 16 - 1, n, afull(as));
            else
              tma_load_4d(dst, &x_map, c * 64, tx_ * 8 - 1, ty_ * 16 - 1, n, afull(as));
          }
          if (++as == T_ASTAGES) { as = 0; aph ^= 1; }
          for (int sub = 0; sub < 4; ++sub) {
            mbar_wait(bempty(bs), bph ^ 1);
            mbar_expect_tx(bfull(bs), bstage);
            bulk_g2s(b_base + (uint32_t)bs * T_BSTAGE, wsrc + (size_t)(c * 4 + sub) * bstage, bstage, bfull(bs));
            if (++bs == T_BSTAGES) { bs = 0; bph ^= 1; }
          }
        }
      }
    }
    __syncwarp();
  }
}

constexpr size_t t16_smem_bytes() {
  return 1024 + (size_t)T_ASTAGES * T_ASTAGE + (size_t)T_BSTAGES * T_BSTAGE + (2 * T_ASTAGES + 2 * T_BSTAGES) * 8 + 16;
}

// ------------------------------------------------------------------------------------------------------------
// Weight gradient of the 3x3 stride-1 convolution from the two fp16 shadows (activation x16, output gradient dy16 - already
// scaled), dW[tap][co][ci] = sum_pixels dy[p][co] * x[p + tap][ci]; the reduction runs over PIXELS, so both operands are
// "MN-major" in memory (channels contiguous, pixels strided):
//   * a CTA owns one kernel ROW (3 horizontal taps) of a 128 co x NCI ci block (NCI = 128, or 64 when Cin % 128 != 0) and
//     walks its split's work units (8 x 8 output pixels); warpgroup g multiplies co 64 g .. 64 g + 63 into three m64nNCI
//     accumulators (one per horizontal tap, 3 x 64 fp32 registers per thread at NCI = 128), K = 16 pixels = two image rows;
//   * A = dy^T from REGISTERS: the dy tile of a unit (64 pixels x 128 co) lands as two 64-channel tensor-map boxes under the
//     128-byte swizzle; per K step each warp reads its 16 co x 16 pixel fragment once with ldmatrix.x4.trans and the three
//     tap MMAs use it (RS wgmma), so shared memory feeds the tensor cores the B operand only;
//   * B = the activation halo exactly as the copy engine lands it: NCI / 64 boxes of [8 rows][10 pixels][64 ci] with 128-byte
//     pixel rows, read as ONE MN-major operand (K groups = image rows of 8 pixels, SBO = the 1280-byte halo row; the 64-channel
//     swizzle atoms are the boxes, LBO = the box stride). A tap is a descriptor start shift (dx * 128 B);
//   * one commit group per K step, two register sets for A: a step's fragment is reloaded only after the group that read it
//     has retired, while the next group keeps the tensor cores busy;
//   * split-K over the units; partial sums go to the caller's workspace in the layout conv_wgrad_reduce expects. The bias
//     gradient comes from the same A fragments (fp32 sums per thread, reduced over the four lanes of a row) in the CTAs of
//     kernel row 0 / ci block 0, so the bias adds no shared-memory pass and no CTA does more than the others.
constexpr int WT_STAGES = 5;
constexpr int WT_XATOM = 8 * 10 * 128;      // one 64-channel halo box: 8 halo rows x 10 pixels x 128 B
constexpr int WT_DYATOM = 64 * 128;         // 64 pixels x 64 co halves
constexpr int WT_DY = 2 * WT_DYATOM;        // 64 pixels x 128 co halves
constexpr int WT_THREADS = 12 * 32;
template <int NCI>
__host__ __device__ constexpr int wt_stage() { return (NCI / 64) * WT_XATOM + WT_DY; }
static_assert(wt_stage<64>() % 1024 == 0 && wt_stage<128>() % 1024 == 0 && WT_XATOM % 1024 == 0,
              "stages must keep the swizzle atoms 1024-byte aligned");
template <int NCI>
constexpr size_t wt_smem_bytes() { return 1024 + (size_t)WT_STAGES * wt_stage<NCI>() + 2 * WT_STAGES * 8 + 16; }
static inline int wt_nci(int64_t cin) { return cin % 128 == 0 ? 128 : 64; }

struct WTParams {
  float* part;      // [splits][9][Cout][Cin]
  float* bpart;     // [splits][Cout] or null
  int N, H, W, Cin, Cout;
  int units_x, units_y;
  int64_t total_units, units_per_split;
  const float* dy_amax;   // the magnitude dy16's power-of-two scale was derived from
};

template <int NCI>
__device__ __forceinline__ void wgmma_rs(float* d, const uint32_t* a, uint64_t bdesc) {
  if (NCI == 128) wg::wgmma_f16_rs_n128<1>(d, a, bdesc, 1u);
  else wg::wgmma_f16_rs_n64<1>(d, a, bdesc, 1u);
}

template <int NCI>
__global__ void __launch_bounds__(WT_THREADS, 1) wgrad_t16(const WTParams p, const __grid_constant__ CUtensorMap x_map,
                                                          const __grid_constant__ CUtensorMap dy_map) {
  constexpr int XBOX = NCI / 64;               // 64-channel halo boxes per stage
  constexpr int STAGE = wt_stage<NCI>();
  constexpr int NR = NCI / 2;                  // accumulator registers per tap
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_base = smem_u32(smem_raw);
  const uint32_t smem_base = (raw_base + 1023u) & ~1023u;
  uint8_t* smem = smem_raw + (smem_base - raw_base);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + (size_t)WT_STAGES * STAGE);
  const uint32_t bar_base = smem_u32(bars);
  auto fullD = [&](int s) { return bar_base + 8u * s; };                      // copies of the stage have landed
  auto empty = [&](int s) { return bar_base + 8u * (WT_STAGES + s); };        // the MMAs of the stage have completed

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int dyy = blockIdx.x % 3, ci0 = (blockIdx.x / 3) * NCI, co0 = blockIdx.y * BM, split = blockIdx.z;
  const int64_t u0 = (int64_t)split * p.units_per_split;
  const int64_t u1 = min(p.total_units, u0 + p.units_per_split);

  if (tid == 0) {
    for (int s = 0; s < WT_STAGES; ++s) { mbar_init(fullD(s), 1); mbar_init(empty(s), 256); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 8) {
    // ============ MMA warpgroups, then epilogue ============
    wg::regs_inc<wg::MMA_REGS>();
    const int wgi = warp >> 2;
    float a_inv;
    operand_scale(p.dy_amax, &a_inv);
    const bool want_bias = p.bpart != nullptr && blockIdx.x == 0;
    float bsum[2] = {0.f, 0.f};                // co rows lane / 4 and lane / 4 + 8 of the warp
    float acc[3][NR];
#pragma unroll
    for (int dx = 0; dx < 3; ++dx)
#pragma unroll
      for (int i = 0; i < NR; ++i) acc[dx][i] = 0.f;
    // ldmatrix.x4.trans: lane l addresses pixel 8 (l / 16) + l % 8 of the K step, co chunk 2 (warp % 4) + (l / 8) % 2 of the
    // warpgroup's 64; matrices (co +0 / +8) x (pixels +0 / +8) give the wgmma A fragment registers 0..3 in order. The
    // 128-byte swizzle XORs the 16-byte chunk with the pixel's row in the atom, which is l % 8 for every K step.
    const int lpix = ((lane >> 4) << 3) + (lane & 7);
    const uint32_t a_lane = (uint32_t)(lpix * 128 + (((((warp & 3) << 1) | ((lane >> 3) & 1)) ^ (lane & 7)) << 4));
    uint32_t a[2][4] = {{0u, 0u, 0u, 0u}, {0u, 0u, 0u, 0u}};
    int stage = 0, prev = -1;
    uint32_t phase = 0;
    for (int64_t u = u0; u < u1; ++u) {
      mbar_wait(fullD(stage), phase);
      const uint32_t xs = smem_base + (uint32_t)stage * STAGE;
      const uint64_t xd0 = wg::desc(xs, WT_XATOM, 1280, wg::SW_128);
      const uint32_t arow = xs + XBOX * WT_XATOM + (uint32_t)(wgi * WT_DYATOM) + a_lane;
#pragma unroll
      for (int s = 0; s < 4; ++s) {             // K step s: image rows 2 s, 2 s + 1 of the unit
        uint32_t* af = a[s & 1];
        wg::wait<1>();                          // the group that last read af (two steps back) has retired
#pragma unroll
        for (int i = 0; i < 4; ++i) asm volatile("" : "+r"(af[i]));   // ... so af stays untouched until here
        if (s == 1 && prev >= 0) mbar_arrive(empty(prev));             // the previous unit's last group has retired too
        ldsm_x4_trans(arow + (uint32_t)(s * 16 * 128), af);
        if (want_bias) {
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&af[i]));
            bsum[i & 1] += f.x + f.y;
          }
        }
        wg::fence();
#pragma unroll
        for (int dx = 0; dx < 3; ++dx) wgmma_rs<NCI>(acc[dx], af, xd0 + (uint64_t)((s * 2 * 1280 + dx * 128) >> 4));
        wg::commit();
      }
      prev = stage;
      if (++stage == WT_STAGES) { stage = 0; phase ^= 1; }
    }
    wg::wait<0>();
#pragma unroll
    for (int dx = 0; dx < 3; ++dx) wg::fence_regs<NR>(acc[dx]);
    const int frow = wgi * 64 + (warp & 3) * 16 + (lane >> 2), fcol = 2 * (lane & 3);
    if (want_bias) {
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        bsum[i] += __shfl_xor_sync(0xffffffffu, bsum[i], 1);
        bsum[i] += __shfl_xor_sync(0xffffffffu, bsum[i], 2);
        if ((lane & 3) == 0) p.bpart[(size_t)split * p.Cout + co0 + frow + 8 * i] = bsum[i] * a_inv;
      }
    }
#pragma unroll
    for (int dx = 0; dx < 3; ++dx) {
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        float* o = p.part + (((size_t)split * 9 + dyy * 3 + dx) * p.Cout + co0 + frow + 8 * i) * p.Cin + ci0 + fcol;
#pragma unroll
        for (int j = 0; j < NCI / 8; ++j)
          *reinterpret_cast<float2*>(o + 8 * j) = make_float2(acc[dx][4 * j + 2 * i] * a_inv, acc[dx][4 * j + 2 * i + 1] * a_inv);
      }
    }
  } else {
    // ============ copy issuer (one thread): dy tile + activation halo rows of this kernel row ============
    wg::regs_dec<wg::COPY_REGS>();
    if (warp == 8 && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int64_t u = u0; u < u1; ++u) {
        const int ux = (int)(u % p.units_x), uy = (int)((u / p.units_x) % p.units_y);
        const int n = (int)(u / ((int64_t)p.units_x * p.units_y));
        const uint32_t dst = smem_base + (uint32_t)stage * STAGE;
        mbar_wait(empty(stage), phase ^ 1);
        mbar_expect_tx(fullD(stage), STAGE);
#pragma unroll
        for (int b = 0; b < XBOX; ++b)
          tma_load_4d(dst + (uint32_t)(b * WT_XATOM), &x_map, ci0 + b * 64, ux * 8 - 1, uy * 8 + dyy - 1, n, fullD(stage));
#pragma unroll
        for (int hf = 0; hf < 2; ++hf)
          tma_load_4d(dst + (uint32_t)(XBOX * WT_XATOM + hf * WT_DYATOM), &dy_map, co0 + hf * 64, ux * 8, uy * 8, n, fullD(stage));
        if (++stage == WT_STAGES) { stage = 0; phase ^= 1; }
      }
    }
    __syncwarp();
  }
}

// fp32 -> fp16 shadow (optionally scaled by the power-of-two operand scale of *amax): plain vectorised copy
__global__ void to_half_kernel(const float4* __restrict__ x, uint2* __restrict__ y, int64_t n4, const float* __restrict__ amax) {
  float inv;
  const float s = operand_scale(amax, &inv);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    const float4 v = __ldg(x + i);
    y[i] = make_uint2(pack_h2(v.x * s, v.y * s), pack_h2(v.z * s, v.w * s));
  }
}

// Tap table of a phase-decomposed resampling convolution: per tap group (output phase / source plane, index 2 py + px) the
// staged-halo offset of each of its four taps and the set of the nine weight taps (bit ty * 3 + tx) summed into it. The
// Downsample's groups hold 4 / 2 / 2 / 1 taps; the others are padded with empty sets (zero weights), so that every group
// runs the same four MMAs per K step: a tap count that varies inside the kernel would serialise the asynchronous MMAs.
struct PhaseTable {
  int hoff[4][4];
  int mask[4][4];
};

// fp16 weight images of the four tap groups, [group][n_tile][K / 16][4 taps][k / 8][128][8 halves] (each group like
// pack_weights_tc16); a combined tap is summed in fp32 and rounded once. transpose: N = Cin, K = Cout (data gradient; the
// table already holds the mirrored geometry, so taps are not flipped here).
__global__ void pack_phase16(const float* __restrict__ w, __half* __restrict__ out, int Cout, int Cin, int transpose, PhaseTable tb,
                             int64_t total) {
  const int N = transpose ? Cin : Cout, K = transpose ? Cout : Cin;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t r = i;
    const int k8 = (int)(r % 8); r /= 8;
    const int nn = (int)(r % BN); r /= BN;
    const int oct = (int)(r % 2); r /= 2;
    const int j = (int)(r % 4); r /= 4;
    const int kc = (int)(r % (K / 16)); r /= K / 16;
    const int nt_ = (int)(r % (N / BN)), g = (int)(r / (N / BN));
    const int n = nt_ * BN + nn, k = kc * 16 + oct * 8 + k8;
    const int co = transpose ? k : n, ci = transpose ? n : k;
    const float* src = w + ((size_t)co * Cin + ci) * 9;
    float s = 0.f;
    for (int t = 0; t < 9; ++t)
      if ((tb.mask[g][j] >> t) & 1) s += src[t];
    out[i] = __float2half_rn(s);
  }
}

}  // namespace tc

// up: Upsample (else Downsample); transpose: the data gradient. Staged halos start one pixel up / left of the tile, so a
// tap at source offset (oy, ox) sits at halo offset (oy + 1) * 10 + ox + 1.
static tc::PhaseTable phase_table(bool up, bool transpose) {
  tc::PhaseTable tb{};
  for (int g = 0; g < 4; ++g) {
    const int py = g >> 1, px = g & 1;
    if (up) {
      // phase p, tap a of a dimension: offset p - 1 + a, original taps {0} / {1, 2} (p = 0) or {0, 1} / {2} (p = 1)
      auto set = [](int ph, int a) { return ph == 0 ? (a == 0 ? 1 : 6) : (a == 0 ? 3 : 4); };
      for (int a = 0; a < 2; ++a)
        for (int b = 0; b < 2; ++b) {
          const int oy = py - 1 + a, ox = px - 1 + b, j = a * 2 + b;
          // forward: output phase g reads x[i + o]; data gradient: source plane g of dy contributes to dx[i] from dy[i - o]
          tb.hoff[g][j] = transpose ? (1 - oy) * 10 + (1 - ox) : (oy + 1) * 10 + (ox + 1);
          int m = 0;
          for (int ty = 0; ty < 3; ++ty)
            for (int tx = 0; tx < 3; ++tx)
              if (((set(py, a) >> ty) & 1) && ((set(px, b) >> tx) & 1)) m |= 1 << (ty * 3 + tx);
          tb.mask[g][j] = m;
        }
    } else {
      // plane (py, px) holds the taps with ty % 2 == py, tx % 2 == px, at plane offset (ty / 2, tx / 2)
      int j = 0;
      for (int ty = py; ty < 3; ty += 2)
        for (int tx = px; tx < 3; tx += 2, ++j) {
          const int oy = ty >> 1, ox = tx >> 1;
          tb.hoff[g][j] = transpose ? (1 - oy) * 10 + (1 - ox) : (oy + 1) * 10 + (ox + 1);
          tb.mask[g][j] = 1 << (ty * 3 + tx);
        }
      for (; j < 4; ++j) {   // padding taps: empty weight set, any in-halo offset
        tb.hoff[g][j] = 11;
        tb.mask[g][j] = 0;
      }
    }
  }
  return tb;
}

static bool dense_nhwc4(const mas_tensor4& t) {
  return t.sc == 1 && t.sw == t.c && t.sh == t.w * t.c && t.sn == t.h * t.w * t.c;
}

bool conv3x3_tma16_ok(mas_tensor4 xs, mas_tensor4 ys) {
  return dense_nhwc4(xs) && dense_nhwc4(ys) && xs.c % 64 == 0 && xs.c >= 64 && ys.c % 4 == 0 && ys.h % 16 == 0 && ys.w % 8 == 0 &&
         xs.h == ys.h && xs.w == ys.w && xs.n == ys.n;
}

// x16: fp16 NHWC shadow of the (activated) input, scaled by operand_scale(*x_amax) when x_amax is given.
int conv3x3_fprop_tma16_launch(const void* x16, mas_tensor4 xs, const void* w_tc16, const float* bias, const float* res, float* y,
                               mas_tensor4 ys, float* stats_part, const float* x_amax, cudaStream_t st) {
  if (!conv3x3_tma16_ok(xs, ys)) return fail(MAS_ERR_UNSUPPORTED, "tma conv: shape/layout not eligible (Cin=%lld Cout=%lld H=%lld W=%lld)",
                                              (long long)xs.c, (long long)ys.c, (long long)ys.h, (long long)ys.w);
  const int Cstore = (int)ys.c, Cout = (int)cdiv(ys.c, tc::BN) * tc::BN;
  if (Cstore != Cout && (res || stats_part)) return fail(MAS_ERR_UNSUPPORTED, "tma conv: residual / statistics epilogues need Cout %% 128 == 0");
  auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  if (!al16(x16) || !al16(y) || !al16(w_tc16) || (res && !al16(res)) || (bias && !al16(bias)))
    return fail(MAS_ERR_INVALID_ARG, "tma conv: pointers must be 16-byte aligned");
  tc::HParams p;
  p.wpk = w_tc16; p.bias = bias; p.res = res; p.y = y;
  p.N = (int)xs.n; p.H = (int)xs.h; p.W = (int)xs.w; p.Cin = (int)xs.c; p.Cout = Cout; p.Cstore = Cstore; p.ldy = Cstore;
  p.tiles_x = (int)(ys.w / 8); p.tiles_y = (int)(ys.h / 16);
  p.stats_part = stats_part; p.x_amax = x_amax;
  const bool tall = ys.h % 32 == 0;
  const int64_t tiles = (int64_t)p.N * p.tiles_x * p.tiles_y;
  p.units = tall ? tiles / 2 : cdiv(tiles, 2);

  PFN_cuTensorMapEncodeTiled enc = tensor_map_encoder();
  if (!enc) return fail(MAS_ERR_LAUNCH, "cuTensorMapEncodeTiled entry point not available");
  CUtensorMap map;
  cuuint64_t dims[4] = {(cuuint64_t)xs.c, (cuuint64_t)xs.w, (cuuint64_t)xs.h, (cuuint64_t)xs.n};
  cuuint64_t strides[3] = {(cuuint64_t)xs.c * 2, (cuuint64_t)xs.w * xs.c * 2, (cuuint64_t)xs.h * xs.w * xs.c * 2};
  cuuint32_t box[4] = {64, 10, tall ? 34u : 18u, 1}, es[4] = {1, 1, 1, 1};
  CUresult r = enc(&map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(x16), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(MAS_ERR_LAUNCH, "cuTensorMapEncodeTiled (conv halo map) failed (%d)", (int)r);

  constexpr size_t smem = tc::t16_smem_bytes();
  static std::atomic<uint64_t> configured{0};
  static int sm_count = 132;
  if (first_on_device(configured)) {
    cudaError_t e = cudaFuncSetAttribute(tc::shift_gemm_t16<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(tc::shift_gemm_t16<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return fail(MAS_ERR_LAUNCH, "cudaFuncSetAttribute(smem=%zu): %s", smem, cudaGetErrorString(e));
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, dev);
    mark_device(configured);
  }
  const int64_t nitems = p.units * (Cout / tc::BN);
  const unsigned g = (unsigned)(nitems < sm_count ? nitems : sm_count);
  if (tall) tc::shift_gemm_t16<true><<<g, tc::T_THREADS, smem, st>>>(p, map);
  else tc::shift_gemm_t16<false><<<g, tc::T_THREADS, smem, st>>>(p, map);
  return launched_tc(tall ? "shift_gemm_t16<tall>" : "shift_gemm_t16<pair>");
}

// Phase-decomposed Upsample / Downsample convolution, xs / ys the shapes of the layer's input and output (forward).
bool conv3x3_phase_ok(mas_tensor4 xs, mas_tensor4 ys, bool up) {
  const mas_tensor4& lo = up ? xs : ys;   // the low-resolution side: the phase planes' extent
  const mas_tensor4& hi = up ? ys : xs;
  return dense_nhwc4(xs) && dense_nhwc4(ys) && xs.c % 128 == 0 && ys.c % 128 == 0 && xs.n == ys.n && hi.h == 2 * lo.h &&
         hi.w == 2 * lo.w && lo.h % 16 == 0 && lo.w % 8 == 0;
}

int pack_phase16_launch(const float* w, void* out, int Cout, int Cin, bool up, bool transpose, cudaStream_t st) {
  if (Cout % tc::BN || Cin % tc::BN) return fail(MAS_ERR_UNSUPPORTED, "pack_conv3x3_phase16: Cout=%d and Cin=%d must be multiples of 128", Cout, Cin);
  const tc::PhaseTable tb = phase_table(up, transpose);
  const int64_t total = (int64_t)16 * Cout * Cin;
  tc::pack_phase16<<<(unsigned)(cdiv(total, 256) < 2368 ? cdiv(total, 256) : 2368), 256, 0, st>>>(w, (__half*)out, Cout, Cin, transpose ? 1 : 0,
                                                                                              tb, total);
  return launched("pack_phase16");
}

// x16: fp16 NHWC shadow of the convolution's source (the layer input, or for the data gradient the output gradient, scaled
// by operand_scale(*x_amax) when x_amax is given); xs / ys: source and destination of THIS pass; w_ph16: pack_phase16 image
// of the same (up, transpose).
int conv3x3_phase_tma16_launch(const void* x16, mas_tensor4 xs, const void* wpk, const float* bias, float* y, mas_tensor4 ys, bool up,
                               bool transpose, const float* x_amax, cudaStream_t st) {
  const bool phase_out = up != transpose;   // Upsample forward / Downsample data gradient: the destination is the 2x side
  if (!conv3x3_phase_ok(phase_out ? xs : ys, phase_out ? ys : xs, true))
    return fail(MAS_ERR_UNSUPPORTED, "phase conv: shape/layout not eligible (Cin=%lld Cout=%lld H=%lld W=%lld)", (long long)xs.c,
                (long long)ys.c, (long long)xs.h, (long long)xs.w);
  auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  if (!al16(x16) || !al16(y) || !al16(wpk) || (bias && !al16(bias))) return fail(MAS_ERR_INVALID_ARG, "phase conv: pointers must be 16-byte aligned");
  const tc::PhaseTable tb = phase_table(up, transpose);
  const mas_tensor4& lo = phase_out ? xs : ys;
  tc::HParams p{};
  p.wpk = wpk; p.bias = bias; p.res = nullptr; p.y = y;
  p.N = (int)xs.n; p.H = (int)lo.h; p.W = (int)lo.w; p.Cin = (int)xs.c; p.Cout = (int)ys.c; p.Cstore = (int)ys.c; p.ldy = ys.c;
  p.tiles_x = (int)(lo.w / 8); p.tiles_y = (int)(lo.h / 16);
  p.stats_part = nullptr; p.x_amax = x_amax;
  const bool tall = lo.h % 32 == 0;
  const int64_t tiles = (int64_t)p.N * p.tiles_x * p.tiles_y;
  p.units = tall ? tiles / 2 : cdiv(tiles, 2);
  p.ysn = ys.sn;
  p.ysh = phase_out ? 2 * ys.sh : ys.sh;
  p.ysw = phase_out ? 2 * ys.sw : ys.sw;
  for (int g = 0; g < 4; ++g) {
    for (int j = 0; j < 4; ++j) p.ph_hoff[g][j] = tb.hoff[g][j];
    p.ph_yoff[g] = phase_out ? (g >> 1) * ys.sh + (g & 1) * ys.sw : 0;
  }

  PFN_cuTensorMapEncodeTiled enc = tensor_map_encoder();
  if (!enc) return fail(MAS_ERR_LAUNCH, "cuTensorMapEncodeTiled entry point not available");
  CUtensorMap map;
  CUresult r;
  const cuuint32_t hbox = tall ? 34u : 18u;
  if (phase_out) {
    cuuint64_t dims[4] = {(cuuint64_t)xs.c, (cuuint64_t)xs.w, (cuuint64_t)xs.h, (cuuint64_t)xs.n};
    cuuint64_t strides[3] = {(cuuint64_t)xs.c * 2, (cuuint64_t)xs.w * xs.c * 2, (cuuint64_t)xs.h * xs.w * xs.c * 2};
    cuuint32_t box[4] = {64, 10, hbox, 1}, es[4] = {1, 1, 1, 1};
    r = enc(&map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(x16), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  } else {
    // the four phase planes of the 2x source: [n][row pair][row parity py][pixel pair][px * C + c]
    cuuint64_t dims[5] = {(cuuint64_t)xs.c * 2, (cuuint64_t)xs.w / 2, 2, (cuuint64_t)xs.h / 2, (cuuint64_t)xs.n};
    cuuint64_t strides[4] = {(cuuint64_t)xs.c * 4, (cuuint64_t)xs.w * xs.c * 2, (cuuint64_t)xs.w * xs.c * 4, (cuuint64_t)xs.h * xs.w * xs.c * 2};
    cuuint32_t box[5] = {64, 10, 1, hbox, 1}, es[5] = {1, 1, 1, 1, 1};
    r = enc(&map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 5, const_cast<void*>(x16), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  }
  if (r != CUDA_SUCCESS) return fail(MAS_ERR_LAUNCH, "cuTensorMapEncodeTiled (phase conv map) failed (%d)", (int)r);

  constexpr size_t smem = tc::t16_smem_bytes();
  static std::atomic<uint64_t> configured{0};
  static int sm_count = 132;
  if (first_on_device(configured)) {
    cudaError_t e = cudaFuncSetAttribute(tc::shift_gemm_t16<true, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(tc::shift_gemm_t16<false, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(tc::shift_gemm_t16<true, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(tc::shift_gemm_t16<false, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return fail(MAS_ERR_LAUNCH, "cudaFuncSetAttribute(smem=%zu): %s", smem, cudaGetErrorString(e));
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, dev);
    mark_device(configured);
  }
  const int64_t nitems = p.units * (p.Cout / tc::BN) * (phase_out ? 4 : 1);
  const unsigned g = (unsigned)(nitems < sm_count ? nitems : sm_count);
  if (phase_out) {
    if (tall) tc::shift_gemm_t16<true, 1><<<g, tc::T_THREADS, smem, st>>>(p, map);
    else tc::shift_gemm_t16<false, 1><<<g, tc::T_THREADS, smem, st>>>(p, map);
    return launched_tc(tall ? "shift_gemm_t16<tall, phase-out>" : "shift_gemm_t16<pair, phase-out>");
  }
  if (tall) tc::shift_gemm_t16<true, 2><<<g, tc::T_THREADS, smem, st>>>(p, map);
  else tc::shift_gemm_t16<false, 2><<<g, tc::T_THREADS, smem, st>>>(p, map);
  return launched_tc(tall ? "shift_gemm_t16<tall, phase-in>" : "shift_gemm_t16<pair, phase-in>");
}

void conv_wgrad_reduce_launch(const float* part, int splits, int ntap, int Cout, int Cin, float* dw, const float* bpart, float* dbias,
                              cudaStream_t st);   // contract_simt.cu

// splits of the pixel reduction: as many as keep all CTAs (cps per split) in one wave of the 132 SMs - more waves would add
// partial-sum traffic for the reduction and, for the small deep layers, leave CTAs with too few units to hide the epilogue
static int wt_splits(int64_t cps, int64_t units) {
  int64_t s = 132 / cps;
  if (s < 1) s = 1;
  if (s > units) s = units;
  const int64_t ups = cdiv(units, s);
  return (int)cdiv(units, ups);
}
bool conv_wgrad_t16_ok(mas_tensor4 xs, mas_tensor4 dys) {
  return dense_nhwc4(xs) && dense_nhwc4(dys) && xs.c % 64 == 0 && dys.c % 8 == 0 && dys.h % 8 == 0 && dys.w % 8 == 0 && xs.h == dys.h &&
         xs.w == dys.w && xs.n == dys.n;
}
size_t conv_wgrad_t16_ws(mas_tensor4 xs, mas_tensor4 dys) {
  if (!conv_wgrad_t16_ok(xs, dys)) return 0;
  const int64_t coutk = cdiv(dys.c, tc::BM) * tc::BM;
  const size_t splits = wt_splits((coutk / tc::BM) * (xs.c / tc::wt_nci(xs.c)) * 3, dys.n * (dys.h / 8) * (dys.w / 8));
  return splits * 9 * (size_t)coutk * xs.c * sizeof(float) + splits * (size_t)coutk * sizeof(float) + 256;
}
// x16: fp16 activation shadow; dy16: fp16 output-gradient shadow scaled by operand_scale(*dy_amax); dw/dbias sized for
// round_up(dys.c, 128) output channels (the copy engine zero-fills the channels dy does not have).
int conv_wgrad_t16_launch(const void* x16, mas_tensor4 xs, const void* dy16, mas_tensor4 dys, float* dw, float* dbias,
                          const float* dy_amax, void* ws, size_t ws_bytes, cudaStream_t st) {
  if (!conv_wgrad_t16_ok(xs, dys) || !dy_amax) return fail(MAS_ERR_UNSUPPORTED, "tma wgrad: shape/layout not eligible");
  if (ws_bytes < conv_wgrad_t16_ws(xs, dys)) return fail(MAS_ERR_WORKSPACE, "tma wgrad: workspace too small");
  tc::WTParams p;
  p.N = (int)xs.n; p.H = (int)xs.h; p.W = (int)xs.w; p.Cin = (int)xs.c; p.Cout = (int)(cdiv(dys.c, tc::BM) * tc::BM);
  p.units_x = (int)(dys.w / 8); p.units_y = (int)(dys.h / 8);
  p.total_units = (int64_t)p.N * p.units_x * p.units_y;
  p.dy_amax = dy_amax;
  const int nci = tc::wt_nci(p.Cin);
  const int splits = wt_splits((int64_t)(p.Cout / tc::BM) * (p.Cin / nci) * 3, p.total_units);
  p.units_per_split = cdiv(p.total_units, splits);
  p.part = (float*)ws;
  p.bpart = dbias ? (float*)ws + (size_t)splits * 9 * p.Cout * p.Cin : nullptr;

  PFN_cuTensorMapEncodeTiled enc = tensor_map_encoder();
  if (!enc) return fail(MAS_ERR_LAUNCH, "cuTensorMapEncodeTiled entry point not available");
  CUtensorMap xmap, dmap;
  {
    cuuint64_t dims[4] = {(cuuint64_t)xs.c, (cuuint64_t)xs.w, (cuuint64_t)xs.h, (cuuint64_t)xs.n};
    cuuint64_t strides[3] = {(cuuint64_t)xs.c * 2, (cuuint64_t)xs.w * xs.c * 2, (cuuint64_t)xs.h * xs.w * xs.c * 2};
    cuuint32_t box[4] = {64, 10, 8, 1}, es[4] = {1, 1, 1, 1};
    CUresult r = enc(&xmap, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(x16), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(MAS_ERR_LAUNCH, "cuTensorMapEncodeTiled (wgrad halo map) failed (%d)", (int)r);
  }
  {
    cuuint64_t dims[4] = {(cuuint64_t)dys.c, (cuuint64_t)dys.w, (cuuint64_t)dys.h, (cuuint64_t)dys.n};
    cuuint64_t strides[3] = {(cuuint64_t)dys.c * 2, (cuuint64_t)dys.w * dys.c * 2, (cuuint64_t)dys.h * dys.w * dys.c * 2};
    cuuint32_t box[4] = {64, 8, 8, 1}, es[4] = {1, 1, 1, 1};
    CUresult r = enc(&dmap, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void*>(dy16), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(MAS_ERR_LAUNCH, "cuTensorMapEncodeTiled (wgrad dy map) failed (%d)", (int)r);
  }
  static std::atomic<uint64_t> configured{0};
  if (first_on_device(configured)) {
    cudaError_t e = cudaFuncSetAttribute(tc::wgrad_t16<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tc::wt_smem_bytes<128>());
    if (e == cudaSuccess)
      e = cudaFuncSetAttribute(tc::wgrad_t16<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tc::wt_smem_bytes<64>());
    if (e != cudaSuccess) return fail(MAS_ERR_LAUNCH, "cudaFuncSetAttribute(wgrad_t16): %s", cudaGetErrorString(e));
    mark_device(configured);
  }
  dim3 grid((unsigned)((p.Cin / nci) * 3), (unsigned)(p.Cout / tc::BM), (unsigned)splits);
  if (nci == 128) tc::wgrad_t16<128><<<grid, tc::WT_THREADS, tc::wt_smem_bytes<128>(), st>>>(p, xmap, dmap);
  else tc::wgrad_t16<64><<<grid, tc::WT_THREADS, tc::wt_smem_bytes<64>(), st>>>(p, xmap, dmap);
  if (int e = launched_tc(nci == 128 ? "wgrad_t16<128>" : "wgrad_t16<64>")) return e;
  conv_wgrad_reduce_launch((const float*)ws, splits, 9, p.Cout, p.Cin, dw, p.bpart, dbias, st);
  return launched("conv_wgrad_reduce");
}

int to_half_launch(const float* x, void* y, int64_t n, const float* amax, cudaStream_t st) {
  if (n % 4 || (reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(y) & 7))
    return fail(MAS_ERR_INVALID_ARG, "to_half: n %% 4 == 0 and aligned pointers required");
  const int64_t n4 = n / 4;
  const int64_t blocks = cdiv(n4, 256);
  tc::to_half_kernel<<<(unsigned)(blocks < 132 * 16 ? blocks : 132 * 16), 256, 0, st>>>(reinterpret_cast<const float4*>(x),
                                                                                       reinterpret_cast<uint2*>(y), n4, amax);
  return launched("to_half");
}

}  // namespace mas

extern "C" {

int mas_conv3x3_tc16h_eligible(mas_tensor4 xs, mas_tensor4 ys) { return mas::conv3x3_tma16_ok(xs, ys) ? 1 : 0; }

int mas_conv3x3_fprop_tc16h(const void* x_f16, mas_tensor4 xs, const void* w_tc16, const float* bias, const float* residual, float* y,
                            mas_tensor4 ys, float* stats_part, const float* x_amax, void* stream) {
  MAS_REQUIRE(x_f16 && w_tc16 && y, "conv3x3_fprop_tc16h: null pointer");
  return mas::conv3x3_fprop_tma16_launch(x_f16, xs, w_tc16, bias, residual, y, ys, stats_part, x_amax, mas::S(stream));
}

int mas_to_half(const float* x, void* y_f16, int64_t n, const float* amax, void* stream) {
  MAS_REQUIRE(x && y_f16 && n > 0, "to_half: bad arguments");
  return mas::to_half_launch(x, y_f16, n, amax, mas::S(stream));
}

int mas_pack_conv3x3_phase16(const float* w_oihw, void* w_ph16, int Cout, int Cin, int mode, int transpose, void* stream) {
  MAS_REQUIRE(w_oihw && w_ph16, "pack_conv3x3_phase16: null pointer");
  MAS_REQUIRE(mode == MAS_CONV_UP_PHASE || mode == MAS_CONV_S2_PHASE, "pack_conv3x3_phase16: mode %d", mode);
  return mas::pack_phase16_launch(w_oihw, w_ph16, Cout, Cin, mode == MAS_CONV_UP_PHASE, transpose != 0, mas::S(stream));
}

int mas_conv3x3_phase_tc16h(const void* x_f16, mas_tensor4 xs, const void* w_ph16, const float* bias, float* y, mas_tensor4 ys,
                            int mode, int transpose, const float* x_amax, void* stream) {
  MAS_REQUIRE(x_f16 && w_ph16 && y, "conv3x3_phase_tc16h: null pointer");
  MAS_REQUIRE(mode == MAS_CONV_UP_PHASE || mode == MAS_CONV_S2_PHASE, "conv3x3_phase_tc16h: mode %d", mode);
  return mas::conv3x3_phase_tma16_launch(x_f16, xs, w_ph16, bias, y, ys, mode == MAS_CONV_UP_PHASE, transpose != 0, x_amax,
                                         mas::S(stream));
}

}  // extern "C"
