// Row GEMM  y[M, N] = alpha * x[M, K] . W[N, K]^T (+ bias, + residual)  as a pure TMA + wgmma kernel on fp16 operands: the
// Linear layers of the token transformer (transformer.py:17-56, forward and data gradient) and, in general, any 1x1
// convolution whose input exists as a dense fp16 [M, K] matrix.  It is shift_gemm_t16 (conv_tma.cu) with one tap:
//   * A side of the problem (activations): ONE 2-D tensor-map copy per 64-channel chunk, box 64 halves x 256 rows under the
//     128-byte swizzle = the K-major SW128 operand image (rows at a 128-byte pitch, 8-row groups 1024 bytes apart); rows past
//     M are zero-filled by the copy engine;
//   * weights: mas_pack_gemm_tc16 image [n_tile][k/16][k/8 % 2][128][8 halves] (no swizzle): the four K = 16 steps of a chunk are
//     16 KB contiguous -> one cp.async.bulk per chunk, into the same ring stage as the activation tile (one barrier pair);
//   * operand roles swapped (D^T = W x X^T: weights on the M side, 256 rows on the N side of wgmma.m64n256k16): warpgroup g
//     owns output features 64 g .. 64 g + 63 of the 128-feature tile, bias is a per-row scalar of the fragment;
//   * one persistent CTA per SM over (256-row tile x 128-feature tile) items, feature tile fastest (the row tile is re-read
//     from L2), 4-stage ring of 48 KB that keeps running across items while the warpgroups store the previous item;
//   * warps 0-7 MMA + epilogue (two warpgroups), warp 8 copy issuer (its warpgroup hands its registers to the MMA ones):
//     no thread touches an operand.
// The rows per work item are a template parameter: 256 for training, 16 .. 256 with split-K for the sampler's decode steps
// (mas_linear_rows_f16).
#include <cuda.h>
#include <cudaTypedefs.h>
#include <cuda_fp16.h>

#include "mas_common.cuh"
#include "tc_ptx.cuh"
#include "wgmma.cuh"

namespace mas {

PFN_cuTensorMapEncodeTiled tensor_map_encoder();   // contract_tc.cu

namespace tc {

constexpr int G_MMA_WARPS = 8;
constexpr int G_THREADS = (G_MMA_WARPS + 4) * 32;   // + the copy-issuing warpgroup
constexpr int G_ROWS = 256;                        // rows of x per work item of the training GEMM (N of the MMA)
constexpr int G_BSUB = 2 * BN * 16;                // one K = 16 step of the packed weights: [2][128][8 halves] = 4 KB
constexpr int G_B = 4 * G_BSUB;                    // the chunk's four steps

// ROWS rows of x per work item (the MMA's N: 16 .. 256).  256 is the training GEMM's shape (4 stages of 48 KB); the narrow
// decode shapes keep more stages of their smaller tiles in flight, since every stage is mostly weight bytes.
template <int ROWS>
struct GTile {
  static constexpr int A = ROWS * 128;             // ROWS rows x 64 halves
  static constexpr int STAGE = A + G_B;
  static constexpr int STAGES = ROWS == G_ROWS ? 4 : (200 * 1024 / STAGE < 8 ? 200 * 1024 / STAGE : 8);
  static constexpr size_t SMEM = 1024 + (size_t)STAGES * STAGE + 2 * STAGES * 8 + 16;
  static_assert(STAGE % 1024 == 0, "stages must keep the swizzle atoms 1024-byte aligned");
};

struct GParams {
  const void* wpk;     // mas_pack_gemm_tc16 image
  const float* bias;   // [N] or null
  const float* res;    // [M, ldy] like y, or null
  float* y;            // split s writes y + s * split_stride
  int64_t M, ldy;
  int K, N, Nstore;    // N: padded to 128 (rows of the packed image), Nstore: columns actually stored
  int64_t units;       // ROWS-row tiles
  const float* x_amax; // amax the fp16 copy of x was scaled from (null: unscaled)
  float alpha;
  // decode form only
  int splits, cps;     // split-K: splits slices of cps 64-wide chunks each
  int act;             // 1: tanh-GELU after the bias
  int64_t split_stride;
};

__device__ __forceinline__ float gelu_tanh(float v) {   // OpenAI tanh-GELU, transformer.py:11-14 (as mas_linear_small)
  const float u = 0.7978845608028654f * v * (1.f + 0.044715f * v * v);
  return 0.5f * v * (1.f + tanhf(u));
}

template <int ROWS>
__device__ __forceinline__ void wgmma_rows(float* acc, uint64_t wd, uint64_t xd, uint32_t scale_d) {
  if constexpr (ROWS == 256) wg::wgmma_f16_ss_n256<0, 0>(acc, wd, xd, scale_d);
  else if constexpr (ROWS == 128) wg::wgmma_f16_ss_n128<0, 0>(acc, wd, xd, scale_d);
  else if constexpr (ROWS == 64) wg::wgmma_f16_ss_n64<0, 0>(acc, wd, xd, scale_d);
  else if constexpr (ROWS == 32) wg::wgmma_f16_ss_n32<0, 0>(acc, wd, xd, scale_d);
  else wg::wgmma_f16_ss_n16<0, 0>(acc, wd, xd, scale_d);
}

// DECODE: the decode-step form (split-K slices, fused GELU); the training GEMM is <256, false>.
template <int ROWS, bool DECODE>
__global__ void __launch_bounds__(G_THREADS, 1) rows_gemm_t16(const GParams p, const __grid_constant__ CUtensorMap x_map) {
  using T = GTile<ROWS>;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_base = smem_u32(smem_raw);
  const uint32_t smem_base = (raw_base + 1023u) & ~1023u;           // swizzle atoms are 1024-byte aligned
  uint8_t* smem = smem_raw + (smem_base - raw_base);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + (size_t)T::STAGES * T::STAGE);
  const uint32_t bar_base = smem_u32(bars);
  auto full = [&](int s) { return bar_base + 8u * s; };
  auto empty = [&](int s) { return bar_base + 8u * (T::STAGES + s); };

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int chunks = p.K / 64;
  const int n_tiles = p.N / BN;
  const int splits = DECODE ? p.splits : 1, cps = DECODE ? p.cps : chunks;
  const int64_t nitems = p.units * splits * n_tiles;   // feature tile fastest, then the K slice, then the row tile

  if (tid == 0) {
    for (int s = 0; s < T::STAGES; ++s) { mbar_init(full(s), 1); mbar_init(empty(s), G_MMA_WARPS * 32); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < G_MMA_WARPS) {
    // ===================== MMA warpgroups: fragment row = output feature, column = row of x =====================
    wg::regs_inc<wg::MMA_REGS>();
    float inv_scale = 1.f;
    operand_scale(p.x_amax, &inv_scale);
    const float alpha = inv_scale * p.alpha;
    const int wgi = warp >> 2;
    const int frow = wgi * 64 + (warp & 3) * 16 + (lane >> 2), fcol = 2 * (lane & 3);
    int s = 0, prev = 0;
    uint32_t sph = 0;
    float acc[ROWS / 2];
    for (int64_t item = blockIdx.x; item < nitems; item += gridDim.x) {
      int split = 0, c0 = 0, c1 = chunks;
      if constexpr (DECODE) {
        split = (int)(item / n_tiles % splits);
        c0 = split * cps;
        c1 = min(chunks, c0 + cps);
      }
      for (int c = c0; c < c1; ++c) {
        mbar_wait(full(s), sph);
        const uint32_t st = smem_base + (uint32_t)s * T::STAGE;
        const uint64_t xd0 = wg::desc(st, 16, 1024, wg::SW_128);
        const uint64_t wd0 = wg::desc(st + T::A + (uint32_t)(wgi * 1024), BN * 16, 128);
        wg::fence();
#pragma unroll
        for (int sub = 0; sub < 4; ++sub)   // D^T = W x X^T: weights on the M side, the ROWS rows on the N side
          wgmma_rows<ROWS>(acc, wd0 + (uint64_t)((sub * G_BSUB) >> 4), xd0 + (uint64_t)((sub * 32) >> 4), (c > c0 || sub > 0) ? 1u : 0u);
        wg::commit();
        wg::wait<1>();
        if (c > c0) mbar_arrive(empty(prev));   // the previous chunk's MMAs have read their stage
        prev = s;
        if (++s == T::STAGES) { s = 0; sph ^= 1; }
      }
      wg::wait<0>();
      wg::fence_regs<ROWS / 2>(acc);
      mbar_arrive(empty(prev));
      const int64_t unit = DECODE ? item / n_tiles / splits : item / n_tiles;
      const int64_t row0 = unit * ROWS + fcol;
      float* y = DECODE ? p.y + split * p.split_stride : p.y;
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int ch = (int)(item % n_tiles) * BN + frow + 8 * i;
        if (ch < p.Nstore) {
          const float bv = p.bias ? __ldg(p.bias + ch) : 0.f;
#pragma unroll
          for (int j = 0; j < ROWS / 8; ++j) {
#pragma unroll
            for (int cc = 0; cc < 2; ++cc) {
              const int64_t r = row0 + 8 * j + cc;
              if (r < p.M) {
                float o = fmaf(acc[4 * j + 2 * i + cc], alpha, bv);
                if (p.res) o += __ldg(p.res + r * p.ldy + ch);
                if (DECODE && p.act) o = gelu_tanh(o);
                y[r * p.ldy + ch] = o;
              }
            }
          }
        }
      }
    }
  } else {
    // ===================== copy issuer (one thread) =====================
    wg::regs_dec<wg::COPY_REGS>();
    if (warp == G_MMA_WARPS && lane == 0) {
      int s = 0;
      uint32_t sph = 0;
      const int ksteps = p.K / 16;
      for (int64_t item = blockIdx.x; item < nitems; item += gridDim.x) {
        const int64_t unit = DECODE ? item / n_tiles / splits : item / n_tiles;
        const int c0 = DECODE ? (int)(item / n_tiles % splits) * cps : 0, c1 = DECODE ? min(chunks, c0 + cps) : chunks;
        const uint8_t* wsrc = reinterpret_cast<const uint8_t*>(p.wpk) + (size_t)(item % n_tiles) * ksteps * G_BSUB;
        for (int c = c0; c < c1; ++c) {
          mbar_wait(empty(s), sph ^ 1);
          const uint32_t st = smem_base + (uint32_t)s * T::STAGE;
          mbar_expect_tx(full(s), T::STAGE);
          tma_load_2d(st, &x_map, c * 64, (int)(unit * ROWS), full(s));
          bulk_g2s(st + T::A, wsrc + (size_t)c * G_B, G_B, full(s));
          if (++s == T::STAGES) { s = 0; sph ^= 1; }
        }
      }
    }
    __syncwarp();
  }
}

// y[r, n] = act(sum over the splits in order of part[s][r][n] + bias[n])
__global__ void rows_split_reduce(const float* __restrict__ part, int splits, int64_t stride, int64_t M, int N,
                                  const float* __restrict__ bias, int act, float* __restrict__ y, int64_t ldy) {
  const int64_t total = M * N;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / N;
    const int n = (int)(i % N);
    float v = part[i];
    for (int s = 1; s < splits; ++s) v += part[s * stride + i];
    if (bias) v += __ldg(bias + n);
    if (act) v = gelu_tanh(v);
    y[r * ldy + n] = v;
  }
}

// ------------------------------------------------------------------------------------------------------------
// Weight gradient of a Linear layer from the two fp16 copies (activation x16 [M,K], output gradient dy16 [M,N], both scaled by
// their power-of-two operand scales): dW[n][k] = sum_m dy[m][n] * x[m][k].  The reduction runs over ROWS, so both operands are
// "MN-major" in memory (features contiguous, rows strided) - a one-tap relative of wgrad_t16 (conv_tma.cu), both operands in shared memory:
//   * A = dy^T: the dy tile of a unit (64 rows x 128 features) lands as two 64-feature tensor-map boxes under the 128-byte
//     swizzle, an MN-major operand; warpgroup g multiplies features 64 g .. 64 g + 63;
//   * B = x tiles exactly as the copy engine lands them under the 128-byte swizzle: [64 rows][64 features] atoms read as an
//     MN-major operand (K groups = 8 rows, SBO = 1024 B), N = 64 MMAs, K = 16 rows per MMA;
//   * a CTA owns a 128 x NCI block of dW (NCI / 64 accumulator fragments per warpgroup); split-K over the 64-row units; partial
//     sums (and the bias gradient, summed from the staged dy tile) go to the caller's workspace in the layout conv_wgrad_reduce
//     expects (one tap).
constexpr int RW_STAGES = 4;
constexpr int RW_XATOM = 64 * 128;          // 64 rows x 64 features (halves)
constexpr int RW_DY = 2 * RW_XATOM;         // 64 rows x 128 features (halves), two swizzle atoms
constexpr int RW_THREADS = 12 * 32;

struct RWParams {
  float* part;      // [splits][N][K]
  float* bpart;     // [splits][N] or null
  int N, K;         // dW is [N][K]
  int64_t total_units, units_per_split;
  const float* dy_amax;   // magnitudes the two fp16 copies were scaled from (null: unscaled)
  const float* x_amax;
};

template <int NCI>
__global__ void __launch_bounds__(RW_THREADS, 1) rows_wgrad_t16(const RWParams p, const __grid_constant__ CUtensorMap x_map,
                                                               const __grid_constant__ CUtensorMap dy_map) {
  constexpr int XB = (NCI / 64) * RW_XATOM, STAGE = XB + RW_DY;
  static_assert(STAGE % 1024 == 0, "stages must keep the swizzle atoms 1024-byte aligned");

  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_base = smem_u32(smem_raw);
  const uint32_t smem_base = (raw_base + 1023u) & ~1023u;
  uint8_t* smem = smem_raw + (smem_base - raw_base);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + (size_t)RW_STAGES * STAGE);
  const uint32_t bar_base = smem_u32(bars);
  auto fullD = [&](int s) { return bar_base + 8u * s; };                      // copies of the stage have landed
  auto empty = [&](int s) { return bar_base + 8u * (RW_STAGES + s); };        // the MMAs of the stage have completed

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int ci0 = blockIdx.x * NCI, co0 = blockIdx.y * BM, split = blockIdx.z;
  const int64_t u0 = (int64_t)split * p.units_per_split;
  const int64_t u1 = min(p.total_units, u0 + p.units_per_split);

  if (tid == 0) {
    for (int s = 0; s < RW_STAGES; ++s) { mbar_init(fullD(s), 1); mbar_init(empty(s), 256); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 8) {
    // ============ MMA warpgroups (bias-gradient sums by warpgroup 0), then epilogue ============
    wg::regs_inc<wg::MMA_REGS>();
    const int wgi = warp >> 2;
    float dy_inv, x_inv;
    operand_scale(p.dy_amax, &dy_inv);
    operand_scale(p.x_amax, &x_inv);
    float bsum = 0.f;
    const bool want_bias = p.bpart != nullptr && blockIdx.x == 0 && tid < 128;
    float acc[NCI / 64][32];
#pragma unroll
    for (int h = 0; h < NCI / 64; ++h)
#pragma unroll
      for (int i = 0; i < 32; ++i) acc[h][i] = 0.f;
    int stage = 0, prev = 0;
    uint32_t phase = 0;
    for (int64_t u = u0; u < u1; ++u) {
      mbar_wait(fullD(stage), phase);
      const uint32_t xs = smem_base + (uint32_t)stage * STAGE;
      // MN-major, 128-byte swizzle: K groups (8 rows of 128 bytes) are SBO = 1024 B apart
      const uint64_t xd0 = wg::desc(xs, 16, 1024, wg::SW_128);
      const uint64_t ad0 = wg::desc(xs + XB + (uint32_t)(wgi * RW_XATOM), 16, 1024, wg::SW_128);
      wg::fence();
#pragma unroll
      for (int r = 0; r < 4; ++r) {             // K = 16 rows per MMA: rows 16 r .. 16 r + 15 of the unit
#pragma unroll
        for (int hf = 0; hf < NCI / 64; ++hf)
          wg::wgmma_f16_ss_n64<1, 1>(acc[hf], ad0 + (uint64_t)((r * 2048) >> 4), xd0 + (uint64_t)((hf * RW_XATOM + r * 2048) >> 4), 1u);
      }
      wg::commit();
      if (want_bias) {
        // column tid of the staged dy tile (swizzled: 16-byte chunk index XOR row % 8), rows in pairs
        const uint8_t* dyt = smem + (size_t)stage * STAGE + XB + (tid >> 6) * RW_XATOM;
        const int ch = (tid & 63) >> 3, e = tid & 7;
#pragma unroll 4
        for (int m = 0; m < 64; m += 2) {
          const __half lo = *reinterpret_cast<const __half*>(dyt + m * 128 + ((ch ^ (m & 7)) << 4) + e * 2);
          const __half hi = *reinterpret_cast<const __half*>(dyt + (m + 1) * 128 + ((ch ^ ((m + 1) & 7)) << 4) + e * 2);
          bsum += __half2float(lo) + __half2float(hi);
        }
      }
      wg::wait<1>();
      if (u > u0) mbar_arrive(empty(prev));
      prev = stage;
      if (++stage == RW_STAGES) { stage = 0; phase ^= 1; }
    }
    wg::wait<0>();
#pragma unroll
    for (int h = 0; h < NCI / 64; ++h) wg::fence_regs<32>(acc[h]);
    if (want_bias) p.bpart[(size_t)split * p.N + co0 + tid] = bsum * dy_inv;
    const float a_inv = dy_inv * x_inv;
    const int frow = wgi * 64 + (warp & 3) * 16 + (lane >> 2), fcol = 2 * (lane & 3);
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      float* o = p.part + ((size_t)split * p.N + co0 + frow + 8 * i) * p.K + ci0 + fcol;
#pragma unroll
      for (int hf = 0; hf < NCI / 64; ++hf)
#pragma unroll
        for (int j = 0; j < 8; ++j)
          *reinterpret_cast<float2*>(o + hf * 64 + 8 * j) = make_float2(acc[hf][4 * j + 2 * i] * a_inv, acc[hf][4 * j + 2 * i + 1] * a_inv);
    }
  } else {
    // ============ copy issuer (one thread): dy tile + x tiles of the unit ============
    wg::regs_dec<wg::COPY_REGS>();
    if (warp == 8 && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      for (int64_t u = u0; u < u1; ++u) {
        const uint32_t dst = smem_base + (uint32_t)stage * STAGE;
        mbar_wait(empty(stage), phase ^ 1);
        mbar_expect_tx(fullD(stage), STAGE);
#pragma unroll
        for (int hf = 0; hf < NCI / 64; ++hf) tma_load_2d(dst + (uint32_t)(hf * RW_XATOM), &x_map, ci0 + hf * 64, (int)(u * 64), fullD(stage));
#pragma unroll
        for (int hf = 0; hf < 2; ++hf) tma_load_2d(dst + XB + (uint32_t)(hf * RW_XATOM), &dy_map, co0 + hf * 64, (int)(u * 64), fullD(stage));
        if (++stage == RW_STAGES) { stage = 0; phase ^= 1; }
      }
    }
    __syncwarp();
  }
}

template <int NCI>
constexpr size_t rw_smem_bytes() {
  return 1024 + (size_t)RW_STAGES * ((NCI / 64) * RW_XATOM + RW_DY) + 2 * RW_STAGES * 8 + 16;
}

}  // namespace tc

bool gemm_rows_f16_ok(int64_t M, int N, int K) { return M > 0 && N > 0 && K >= 64 && K % 64 == 0 && M < (1ll << 31) - 256; }

template <int ROWS, bool DECODE>
static int rows_gemm_run(tc::GParams p, const void* x16, cudaStream_t st) {
  using T = tc::GTile<ROWS>;
  PFN_cuTensorMapEncodeTiled enc = tensor_map_encoder();
  if (!enc) return fail(MAS_ERR_LAUNCH, "cuTensorMapEncodeTiled entry point not available");
  CUtensorMap map;
  cuuint64_t dims[2] = {(cuuint64_t)p.K, (cuuint64_t)p.M};
  cuuint64_t strides[1] = {(cuuint64_t)p.K * 2};
  cuuint32_t box[2] = {64, (cuuint32_t)ROWS}, es[2] = {1, 1};
  CUresult r = enc(&map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(x16), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(MAS_ERR_LAUNCH, "cuTensorMapEncodeTiled (row GEMM map) failed (%d)", (int)r);

  static std::atomic<uint64_t> configured{0};
  static int sm_count = 132;
  if (first_on_device(configured)) {
    cudaError_t e = cudaFuncSetAttribute(tc::rows_gemm_t16<ROWS, DECODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)T::SMEM);
    if (e != cudaSuccess) return fail(MAS_ERR_LAUNCH, "cudaFuncSetAttribute(smem=%zu): %s", T::SMEM, cudaGetErrorString(e));
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, dev);
    mark_device(configured);
  }
  p.units = cdiv(p.M, ROWS);
  const int64_t nitems = p.units * (DECODE ? p.splits : 1) * (p.N / tc::BN);
  const unsigned g = (unsigned)(nitems < sm_count ? nitems : sm_count);
  tc::rows_gemm_t16<ROWS, DECODE><<<g, tc::G_THREADS, T::SMEM, st>>>(p, map);
  return launched_tc("rows_gemm_t16");
}

int gemm_rows_f16_launch(const void* x16, int64_t M, int K, const void* w_tc16, float* y, int64_t ldy, int N, const float* bias,
                         const float* res, const float* x_amax, float alpha, cudaStream_t st) {
  if (!gemm_rows_f16_ok(M, N, K)) return fail(MAS_ERR_UNSUPPORTED, "gemm_rows_f16: needs K %% 64 == 0 (M=%lld N=%d K=%d)", (long long)M, N, K);
  auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  if (!al16(x16) || !al16(w_tc16)) return fail(MAS_ERR_INVALID_ARG, "gemm_rows_f16: x16 / packed weights must be 16-byte aligned");
  tc::GParams p;
  p.wpk = w_tc16; p.bias = bias; p.res = res; p.y = y; p.M = M; p.ldy = ldy; p.split_stride = 0; p.K = K;
  p.N = (int)cdiv(N, tc::BN) * tc::BN; p.Nstore = N;
  p.splits = 1; p.cps = K / 64; p.act = 0;
  p.x_amax = x_amax; p.alpha = alpha;
  return rows_gemm_run<tc::G_ROWS, false>(p, x16, st);
}

// ---- decode-step Linear layers (a few to a few hundred rows): the same kernel with the rows on a narrower MMA N side and the
// contraction split so that one wave covers the SMs.  The split factor depends on (N, K) only, never on the row count, so a
// row's result does not depend on how many rows share the call.  ops.linear_small decides per shape and row count whether this
// form or the training GEMM serves a decode step.
static int linear_rows_splits(int N, int K) {
  const int64_t tiles = cdiv(N, tc::BN);
  const int chunks = K / 64;
  int best = 1;
  double best_score = -1.0;
  for (int s = 1; s <= 16 && s <= chunks; ++s) {
    const int cps = (int)cdiv(chunks, s), se = (int)cdiv(chunks, cps);
    const int64_t g = tiles * se;
    const double eff = (double)g / (double)(cdiv(g, 132) * 132) - 0.02 * se;   // partial sums cost bytes: fewer splits win ties
    if (eff > best_score + 1e-9) { best_score = eff; best = se; }
  }
  return best;
}
static size_t linear_rows_ws(int64_t R, int N, int K) {
  const int s = linear_rows_splits(N, K);
  return s > 1 ? (size_t)s * R * N * sizeof(float) : 0;
}

int linear_rows_f16_launch(const void* x16, int64_t R, int K, const void* w_tc16, float* y, int64_t ldy, int N, const float* bias,
                           const float* x_amax, int act, void* ws, size_t ws_bytes, cudaStream_t st) {
  if (!gemm_rows_f16_ok(R, N, K)) return fail(MAS_ERR_UNSUPPORTED, "linear_rows_f16: needs K %% 64 == 0 (R=%lld N=%d K=%d)", (long long)R, N, K);
  auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  if (!al16(x16) || !al16(w_tc16) || !al16(ws)) return fail(MAS_ERR_INVALID_ARG, "linear_rows_f16: x16 / packed weights / workspace must be 16-byte aligned");
  if (act != 0 && act != 1) return fail(MAS_ERR_INVALID_ARG, "linear_rows_f16: act must be 0 (none) or 1 (tanh-GELU)");
  if (ws_bytes < linear_rows_ws(R, N, K)) return fail(MAS_ERR_WORKSPACE, "linear_rows_f16: workspace too small");
  tc::GParams p;
  const int splits = linear_rows_splits(N, K);
  p.wpk = w_tc16; p.res = nullptr; p.M = R; p.K = K;
  p.N = (int)cdiv(N, tc::BN) * tc::BN; p.Nstore = N;
  p.splits = splits; p.cps = (int)cdiv(K / 64, splits);
  p.x_amax = x_amax; p.alpha = 1.f;
  if (splits > 1) {   // partial sums to the workspace, bias and activation after the ordered sum
    p.bias = nullptr; p.act = 0; p.y = (float*)ws; p.ldy = N; p.split_stride = R * N;
  } else {
    p.bias = bias; p.act = act; p.y = y; p.ldy = ldy; p.split_stride = 0;
  }
  int e;
  if (R <= 16) e = rows_gemm_run<16, true>(p, x16, st);
  else if (R <= 32) e = rows_gemm_run<32, true>(p, x16, st);
  else if (R <= 64) e = rows_gemm_run<64, true>(p, x16, st);
  else if (R <= 128) e = rows_gemm_run<128, true>(p, x16, st);
  else e = rows_gemm_run<256, true>(p, x16, st);
  if (e || splits == 1) return e;
  const int64_t total = R * N;
  tc::rows_split_reduce<<<(unsigned)(cdiv(total, 256) < 2368 ? cdiv(total, 256) : 2368), 256, 0, st>>>((const float*)ws, splits, R * N, R, N,
                                                                                                      bias, act, y, ldy);
  return launched("rows_split_reduce");
}

void conv_wgrad_reduce_launch(const float* part, int splits, int ntap, int Cout, int Cin, float* dw, const float* bpart, float* dbias,
                              cudaStream_t st);   // contract_simt.cu

bool wgrad_rows_f16_ok(int64_t M, int N, int K) { return M > 0 && N % 128 == 0 && K % 128 == 0 && N > 0 && K > 0 && M < (1ll << 31) - 64; }
static int rw_nci(int K) { return K % 256 == 0 ? 256 : 128; }
static int rw_splits(int64_t M, int N, int K) {
  // split-K factor: fill whole waves of the 132 SMs (the partial sums cost a reduction pass, so fewer splits win ties)
  const int64_t ctas = (int64_t)(N / 128) * (K / rw_nci(K)), units = cdiv(M, 64);
  int best = 1;
  double best_score = -1.0;
  for (int s = 1; s <= 16 && s <= units; ++s) {
    const int64_t g = ctas * s;
    const double eff = (double)g / (double)(cdiv(g, 132) * 132) - 0.02 * s;
    if (eff > best_score + 1e-9) { best_score = eff; best = s; }
  }
  const int64_t ups = cdiv(units, best);
  return (int)cdiv(units, ups);
}
size_t wgrad_rows_f16_ws(int64_t M, int N, int K) {
  if (!wgrad_rows_f16_ok(M, N, K)) return 0;
  const size_t splits = (size_t)rw_splits(M, N, K);
  return splits * ((size_t)N * K + N) * sizeof(float) + 256;
}
// dw [N][K] = dy16^T . x16, dbias [N] = column sums of dy (may be null)
int wgrad_rows_f16_launch(const void* x16, const void* dy16, int64_t M, int N, int K, float* dw, float* dbias, const float* x_amax,
                          const float* dy_amax, void* ws, size_t ws_bytes, cudaStream_t st) {
  if (!wgrad_rows_f16_ok(M, N, K)) return fail(MAS_ERR_UNSUPPORTED, "wgrad_rows_f16: needs N %% 128 == 0 and K %% 128 == 0 (N=%d K=%d)", N, K);
  if (ws_bytes < wgrad_rows_f16_ws(M, N, K)) return fail(MAS_ERR_WORKSPACE, "wgrad_rows_f16: workspace too small");
  auto al16 = [](const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; };
  if (!al16(x16) || !al16(dy16) || !al16(ws)) return fail(MAS_ERR_INVALID_ARG, "wgrad_rows_f16: pointers must be 16-byte aligned");
  tc::RWParams p;
  const int nci = rw_nci(K), splits = rw_splits(M, N, K);
  p.N = N; p.K = K; p.total_units = cdiv(M, 64); p.units_per_split = cdiv(p.total_units, splits);
  p.dy_amax = dy_amax; p.x_amax = x_amax;
  p.part = (float*)ws;
  p.bpart = dbias ? (float*)ws + (size_t)splits * N * K : nullptr;
  PFN_cuTensorMapEncodeTiled enc = tensor_map_encoder();
  if (!enc) return fail(MAS_ERR_LAUNCH, "cuTensorMapEncodeTiled entry point not available");
  CUtensorMap xmap, dmap;
  {
    cuuint64_t dims[2] = {(cuuint64_t)K, (cuuint64_t)M};
    cuuint64_t strides[1] = {(cuuint64_t)K * 2};
    cuuint32_t box[2] = {64, 64}, es[2] = {1, 1};
    CUresult r = enc(&xmap, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(x16), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(MAS_ERR_LAUNCH, "cuTensorMapEncodeTiled (row wgrad x map) failed (%d)", (int)r);
  }
  {
    cuuint64_t dims[2] = {(cuuint64_t)N, (cuuint64_t)M};
    cuuint64_t strides[1] = {(cuuint64_t)N * 2};
    cuuint32_t box[2] = {64, 64}, es[2] = {1, 1};
    CUresult r = enc(&dmap, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(dy16), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail(MAS_ERR_LAUNCH, "cuTensorMapEncodeTiled (row wgrad dy map) failed (%d)", (int)r);
  }
  static std::atomic<uint64_t> configured{0};
  if (first_on_device(configured)) {
    cudaError_t e = cudaFuncSetAttribute(tc::rows_wgrad_t16<256>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tc::rw_smem_bytes<256>());
    if (e == cudaSuccess) e = cudaFuncSetAttribute(tc::rows_wgrad_t16<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tc::rw_smem_bytes<128>());
    if (e != cudaSuccess) return fail(MAS_ERR_LAUNCH, "cudaFuncSetAttribute(rows_wgrad_t16): %s", cudaGetErrorString(e));
    mark_device(configured);
  }
  dim3 grid((unsigned)(K / nci), (unsigned)(N / 128), (unsigned)splits);
  if (nci == 256) tc::rows_wgrad_t16<256><<<grid, tc::RW_THREADS, tc::rw_smem_bytes<256>(), st>>>(p, xmap, dmap);
  else tc::rows_wgrad_t16<128><<<grid, tc::RW_THREADS, tc::rw_smem_bytes<128>(), st>>>(p, xmap, dmap);
  if (int e = launched_tc("rows_wgrad_t16")) return e;
  conv_wgrad_reduce_launch((const float*)ws, splits, 1, N, K, dw, p.bpart, dbias, st);
  return launched("conv_wgrad_reduce");
}

}  // namespace mas

extern "C" {

int mas_gemm_rows_f16(const void* x_f16, int64_t M, int K, const void* w_tc16, float* y, int64_t ldy, int N, const float* bias,
                      const float* residual, const float* x_amax, float alpha, void* stream) {
  MAS_REQUIRE(x_f16 && w_tc16 && y && ldy >= N, "gemm_rows_f16: bad arguments");
  return mas::gemm_rows_f16_launch(x_f16, M, K, w_tc16, y, ldy, N, bias, residual, x_amax, alpha, mas::S(stream));
}

size_t mas_linear_rows_f16_ws_bytes(int64_t R, int N, int K) { return mas::gemm_rows_f16_ok(R, N, K) ? mas::linear_rows_ws(R, N, K) : 0; }

int mas_linear_rows_f16(const void* x_f16, int64_t R, int K, const void* w_tc16, float* y, int64_t ldy, int N, const float* bias,
                        const float* x_amax, int act, void* ws, size_t ws_bytes, void* stream) {
  MAS_REQUIRE(x_f16 && w_tc16 && y && ldy >= N, "linear_rows_f16: bad arguments");
  return mas::linear_rows_f16_launch(x_f16, R, K, w_tc16, y, ldy, N, bias, x_amax, act, ws, ws_bytes, mas::S(stream));
}

size_t mas_wgrad_rows_f16_ws_bytes(int64_t M, int N, int K) { return mas::wgrad_rows_f16_ws(M, N, K); }

int mas_wgrad_rows_f16(const void* x_f16, const void* dy_f16, int64_t M, int N, int K, float* dw, float* dbias, const float* x_amax,
                       const float* dy_amax, void* ws, size_t ws_bytes, void* stream) {
  MAS_REQUIRE(x_f16 && dy_f16 && dw && ws, "wgrad_rows_f16: bad arguments");
  return mas::wgrad_rows_f16_launch(x_f16, dy_f16, M, N, K, dw, dbias, x_amax, dy_amax, ws, ws_bytes, mas::S(stream));
}

}  // extern "C"
