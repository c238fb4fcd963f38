// FP8 Linear layers of the token transformer (opt-in: MakeAScene(fp8_linear=True)): forward, data gradient and weight
// gradient on sm_90a's e4m3 / e5m2 wgmma, with per-tensor power-of-two scales derived on the device (current scaling).
//   * Formats: activations x and weights W are e4m3 (max 448), the output gradient dy is e5m2 (max 57344).  The scale puts
//     max|.| in the top full binade below the format's maximum ([2^7, 2^8) for e4m3, [2^14, 2^15) for e5m2), so nothing
//     saturates; conversion is cvt.rn.satfinite (round to nearest even).  Zero / non-finite amax -> scale 1; NaN stays NaN.
//   * Layouts: fp8 wgmma reads only K-major shared-memory operands (no transpose bit for 8-bit types).  The forward
//     y = x.W^T and the data gradient dx = dy.W contract over the feature dimension and read row-major copies; the weight
//     gradient dW = dy^T.x contracts over the M rows and reads transposed copies x^T [K, M'] and dy^T [N, M'] (M' = M rounded
//     up to 16 for the copy engine's 16-byte stride rule, zero padded).  One cast pass (to_fp8) writes either or both.
//   * One GEMM kernel serves all three products: D[r][f] = sum_k B[r][k] A[f][k], A = the "features" operand (W, W^T or x^T,
//     always e4m3), B = the "rows" operand (x: e4m3; dy or dy^T: e5m2), both landed by 2-D tensor-map copies of 128 rows x
//     128 bytes under the 128-byte swizzle.  Warpgroup g multiplies features 64 g .. 64 g + 63 (wgmma M side) with the
//     item's 128 rows (N side): m64n128k32.
//   * Accumulation: the FP8 MMA does not keep a full fp32 sum while it accumulates (DeepSeek-V3 report, §3.3.2; measured
//     here: DESIGN §3.5).  Each stage holds 128 K elements = four k32 MMAs that start from zero, and their sum is promoted
//     into fp32 registers after every stage.  The second accumulator is why the tile is m64n128 per warpgroup instead of
//     rows_gemm_t16's m64n256 (2 x 128 registers would not fit in 255).
//   * Split-K (weight gradient only): partial products in the caller's workspace, added in a fixed order by
//     conv_wgrad_reduce, so every call gives the same bits.
#include <cuda.h>
#include <cudaTypedefs.h>

#include "mas_common.cuh"
#include "tc_ptx.cuh"
#include "wgmma.cuh"

namespace mas {

PFN_cuTensorMapEncodeTiled tensor_map_encoder();   // contract_tc.cu
void conv_wgrad_reduce_launch(const float* part, int splits, int ntap, int Cout, int Cin, float* dw, const float* bpart, float* dbias,
                              cudaStream_t st);   // contract_simt.cu

namespace tc {

constexpr int E4M3_TOP = 7, E5M2_TOP = 14;   // operand_scale binades of the two formats

// ------------------------------------------------------------------------------------------------------------
// Cast pass: fp32 [M, K] -> fp8 row-major [M, K] and / or transposed [K, M'] (zero rows M .. M'-1), optionally the fp32 column
// sums of the unscaled input (per 64-row tile into colpart, then added over the tiles in order by colsum_finish).
// A CTA owns a 64 x 64 tile: coalesced float4 loads, the row-major bytes straight from registers, the transposed ones
// through a shared-memory copy of the tile (16 rows of one column per thread = one 16-byte store).
__device__ __forceinline__ uint32_t f8x4(float a, float b, float c, float d, bool e5m2) {
  uint16_t lo, hi;   // cvt packs its first source into the upper byte
  if (e5m2) {
    asm("cvt.rn.satfinite.e5m2x2.f32 %0, %1, %2;" : "=h"(lo) : "f"(b), "f"(a));
    asm("cvt.rn.satfinite.e5m2x2.f32 %0, %1, %2;" : "=h"(hi) : "f"(d), "f"(c));
  } else {
    asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(lo) : "f"(b), "f"(a));
    asm("cvt.rn.satfinite.e4m3x2.f32 %0, %1, %2;" : "=h"(hi) : "f"(d), "f"(c));
  }
  return (uint32_t)lo | ((uint32_t)hi << 16);
}

template <bool E5M2>
__global__ void __launch_bounds__(256) to_fp8(const float* __restrict__ x, int64_t M, int K, const float* __restrict__ amax,
                                              uint8_t* __restrict__ rows, uint8_t* __restrict__ cols, int64_t Mp,
                                              float* __restrict__ colpart) {
  __shared__ float t[64][65];
  const int tid = threadIdx.x;
  const int64_t r0 = (int64_t)blockIdx.x * 64;
  const int c0 = blockIdx.y * 64;
  float inv;
  const float s = operand_scale<E5M2 ? E5M2_TOP : E4M3_TOP>(amax, &inv);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int idx = tid + 256 * i, r = idx >> 4, q = idx & 15;
    const int64_t gr = r0 + r;
    const int gc = c0 + 4 * q;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (gr < M && gc < K) {
      v = __ldg(reinterpret_cast<const float4*>(x + gr * K + gc));
      if (rows) *reinterpret_cast<uint32_t*>(rows + gr * K + gc) = f8x4(v.x * s, v.y * s, v.z * s, v.w * s, E5M2);
    }
    t[r][4 * q] = v.x; t[r][4 * q + 1] = v.y; t[r][4 * q + 2] = v.z; t[r][4 * q + 3] = v.w;
  }
  if (!cols && !colpart) return;
  __syncthreads();
  const int c = tid >> 2, q = tid & 3;   // column c of the tile, rows 16 q .. 16 q + 15
  float sum = 0.f;
  uint32_t w[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const float a = t[16 * q + 4 * j][c], b = t[16 * q + 4 * j + 1][c], cc = t[16 * q + 4 * j + 2][c], d = t[16 * q + 4 * j + 3][c];
    sum += a; sum += b; sum += cc; sum += d;
    w[j] = f8x4(a * s, b * s, cc * s, d * s, E5M2);
  }
  const int64_t gr0 = r0 + 16 * q;
  if (cols && c0 + c < K && gr0 < Mp)
    *reinterpret_cast<uint4*>(cols + (int64_t)(c0 + c) * Mp + gr0) = make_uint4(w[0], w[1], w[2], w[3]);
  if (colpart) {
    sum += __shfl_xor_sync(0xffffffffu, sum, 1);
    sum += __shfl_xor_sync(0xffffffffu, sum, 2);
    if (q == 0 && c0 + c < K) colpart[(int64_t)blockIdx.x * K + c0 + c] = sum;
  }
}

// colsum[c] = sum over the 64-row tiles, in order, of colpart[tile][c]
__global__ void colsum_finish(const float* __restrict__ colpart, int tiles, int K, float* __restrict__ colsum) {
  for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < K; c += gridDim.x * blockDim.x) {
    float v = 0.f;
    for (int i = 0; i < tiles; ++i) v += colpart[(int64_t)i * K + c];
    colsum[c] = v;
  }
}

// ------------------------------------------------------------------------------------------------------------
// GEMM: y[r][f] (+ split * split_stride) = alpha * sum_k B[r][k] A[f][k] (+ bias[f]), alpha = the two inverse operand scales.
constexpr int F8_TILE = 128 * 128;            // 128 rows x 128 bytes of one operand
constexpr int F8_STAGE = 2 * F8_TILE;         // features tile, then rows tile
constexpr int F8_STAGES = 6;
constexpr size_t F8_SMEM = 1024 + (size_t)F8_STAGES * F8_STAGE + 2 * F8_STAGES * 8 + 16;
constexpr int F8_THREADS = 12 * 32;           // two MMA warpgroups + the copy-issuing warpgroup

struct F8Params {
  float* y;
  int64_t ldy, split_stride;
  const float* bias;     // [N] or null
  const float* a_amax;   // the features operand's scale source (e4m3)
  const float* b_amax;   // the rows operand's (e4m3, or e5m2 with B_E5M2)
  int64_t M;             // rows
  int N, K;              // features, contraction length
  int splits, cps;       // split-K: splits slices of cps 128-wide chunks
};

template <bool B_E5M2>
__global__ void __launch_bounds__(F8_THREADS, 1) rows_gemm_f8(const F8Params p, const __grid_constant__ CUtensorMap a_map,
                                                              const __grid_constant__ CUtensorMap b_map) {
  extern __shared__ uint8_t smem_raw[];
  const uint32_t raw_base = smem_u32(smem_raw);
  const uint32_t smem_base = (raw_base + 1023u) & ~1023u;
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem_raw + (smem_base - raw_base) + (size_t)F8_STAGES * F8_STAGE);
  const uint32_t bar_base = smem_u32(bars);
  auto full = [&](int s) { return bar_base + 8u * s; };
  auto empty = [&](int s) { return bar_base + 8u * (F8_STAGES + s); };

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int chunks = (p.K + 127) / 128;
  const int n_tiles = (p.N + 127) / 128;
  const int64_t nitems = (p.M + 127) / 128 * p.splits * n_tiles;   // feature tile fastest, then the K slice, then the row tile

  if (tid == 0) {
    for (int s = 0; s < F8_STAGES; ++s) { mbar_init(full(s), 1); mbar_init(empty(s), 256); }
    fence_barrier_init();
  }
  __syncthreads();

  if (warp < 8) {
    // ===================== MMA warpgroups: fragment row = feature, column = row =====================
    wg::regs_inc<wg::MMA_REGS>();
    float a_inv, b_inv;
    operand_scale<E4M3_TOP>(p.a_amax, &a_inv);
    operand_scale<B_E5M2 ? E5M2_TOP : E4M3_TOP>(p.b_amax, &b_inv);
    const float alpha = a_inv * b_inv;
    const int wgi = warp >> 2;
    const int frow = wgi * 64 + (warp & 3) * 16 + (lane >> 2), fcol = 2 * (lane & 3);
    int s = 0;
    uint32_t sph = 0;
    float acc[64], tot[64];
    for (int64_t item = blockIdx.x; item < nitems; item += gridDim.x) {
      const int split = (int)(item / n_tiles % p.splits);
      const int c0 = split * p.cps, c1 = min(chunks, c0 + p.cps);
#pragma unroll
      for (int i = 0; i < 64; ++i) tot[i] = 0.f;
      for (int c = c0; c < c1; ++c) {
        mbar_wait(full(s), sph);
        const uint32_t st = smem_base + (uint32_t)s * F8_STAGE;
        const uint64_t ad0 = wg::desc(st + (uint32_t)(wgi * 64 * 128), 16, 1024, wg::SW_128);
        const uint64_t bd0 = wg::desc(st + F8_TILE, 16, 1024, wg::SW_128);
        wg::fence();
#pragma unroll
        for (int sub = 0; sub < 4; ++sub)   // K = 32 bytes per MMA inside the 128-byte swizzled rows
          wg::wgmma_f8_ss_n128<B_E5M2>(acc, ad0 + (uint64_t)((sub * 32) >> 4), bd0 + (uint64_t)((sub * 32) >> 4), sub > 0 ? 1u : 0u);
        wg::commit();
        wg::wait<0>();
        wg::fence_regs<64>(acc);
        mbar_arrive(empty(s));
#pragma unroll
        for (int i = 0; i < 64; ++i) tot[i] += acc[i];   // promotion into fp32 every 128 K elements
        if (++s == F8_STAGES) { s = 0; sph ^= 1; }
      }
      const int64_t row0 = item / n_tiles / p.splits * 128 + fcol;
      float* y = p.y + split * p.split_stride;
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int ch = (int)(item % n_tiles) * 128 + frow + 8 * i;
        if (ch < p.N) {
          const float bv = p.bias ? __ldg(p.bias + ch) : 0.f;
#pragma unroll
          for (int j = 0; j < 16; ++j) {
#pragma unroll
            for (int cc = 0; cc < 2; ++cc) {
              const int64_t r = row0 + 8 * j + cc;
              if (r < p.M) y[r * p.ldy + ch] = fmaf(tot[4 * j + 2 * i + cc], alpha, bv);
            }
          }
        }
      }
    }
  } else {
    // ===================== copy issuer (one thread) =====================
    wg::regs_dec<wg::COPY_REGS>();
    if (warp == 8 && lane == 0) {
      int s = 0;
      uint32_t sph = 0;
      for (int64_t item = blockIdx.x; item < nitems; item += gridDim.x) {
        const int64_t unit = item / n_tiles / p.splits;
        const int c0 = (int)(item / n_tiles % p.splits) * p.cps, c1 = min(chunks, c0 + p.cps);
        const int ft = (int)(item % n_tiles);
        for (int c = c0; c < c1; ++c) {
          mbar_wait(empty(s), sph ^ 1);
          const uint32_t st = smem_base + (uint32_t)s * F8_STAGE;
          mbar_expect_tx(full(s), F8_STAGE);
          tma_load_2d(st, &a_map, c * 128, ft * 128, full(s));
          tma_load_2d(st + F8_TILE, &b_map, c * 128, (int)(unit * 128), full(s));
          if (++s == F8_STAGES) { s = 0; sph ^= 1; }
        }
      }
    }
    __syncwarp();
  }
}

}  // namespace tc

static bool al16(const void* q) { return (reinterpret_cast<uintptr_t>(q) & 15) == 0; }
static int64_t pad16(int64_t m) { return (m + 15) / 16 * 16; }

static size_t to_fp8_ws(int64_t M, int K) { return (size_t)cdiv(M, 64) * K * sizeof(float); }

static int to_fp8_launch(const float* x, int64_t M, int K, int fmt, const float* amax, void* y_rows, void* y_cols, float* colsum,
                         void* ws, size_t ws_bytes, cudaStream_t st) {
  if (M <= 0 || M >= (1ll << 31) || K <= 0 || K % 16 || K / 64 >= 65535)
    return fail(MAS_ERR_UNSUPPORTED, "to_fp8: needs 0 < M < 2^31 and K %% 16 == 0 (M=%lld K=%d)", (long long)M, K);
  if (fmt != MAS_FP8_E4M3 && fmt != MAS_FP8_E5M2) return fail(MAS_ERR_INVALID_ARG, "to_fp8: fmt must be MAS_FP8_E4M3 or MAS_FP8_E5M2");
  if (!al16(x) || !al16(y_rows) || !al16(y_cols)) return fail(MAS_ERR_INVALID_ARG, "to_fp8: x and the outputs must be 16-byte aligned");
  if (colsum && (!ws || ws_bytes < to_fp8_ws(M, K))) return fail(MAS_ERR_WORKSPACE, "to_fp8: workspace too small for the column sums");
  const dim3 grid((unsigned)cdiv(M, 64), (unsigned)cdiv(K, 64));
  float* part = colsum ? (float*)ws : nullptr;
  uint8_t *r = (uint8_t*)y_rows, *c = (uint8_t*)y_cols;
  if (fmt == MAS_FP8_E5M2) tc::to_fp8<true><<<grid, 256, 0, st>>>(x, M, K, amax, r, c, pad16(M), part);
  else tc::to_fp8<false><<<grid, 256, 0, st>>>(x, M, K, amax, r, c, pad16(M), part);
  if (int e = launched(fmt == MAS_FP8_E5M2 ? "to_fp8<e5m2>" : "to_fp8<e4m3>")) return e;
  if (!colsum) return MAS_OK;
  tc::colsum_finish<<<(unsigned)cdiv(K, 256), 256, 0, st>>>(part, (int)grid.x, K, colsum);
  return launched("fp8_colsum_finish");
}

// [rows, cols] fp8 bytes, row pitch cols: 128 x 128-byte boxes under the 128-byte swizzle (zero fill past the extents)
static int encode_f8(CUtensorMap* map, const void* base, int64_t rows, int64_t cols, const char* what) {
  PFN_cuTensorMapEncodeTiled enc = tensor_map_encoder();
  if (!enc) return fail(MAS_ERR_LAUNCH, "cuTensorMapEncodeTiled entry point not available");
  cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
  cuuint64_t strides[1] = {(cuuint64_t)cols};
  cuuint32_t box[2] = {128, 128}, es[2] = {1, 1};
  CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_UINT8, 2, const_cast<void*>(base), dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                   CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) return fail(MAS_ERR_LAUNCH, "cuTensorMapEncodeTiled (%s) failed (%d)", what, (int)r);
  return MAS_OK;
}

// features operand a [N, K] (e4m3), rows operand b [M, K] (e4m3, or e5m2 with b_e5m2), K the row pitch in bytes of both
static int gemm_f8_run(bool b_e5m2, tc::F8Params p, const void* a, const void* b, cudaStream_t st) {
  CUtensorMap amap, bmap;
  if (int e = encode_f8(&amap, a, p.N, p.K, "fp8 features operand")) return e;
  if (int e = encode_f8(&bmap, b, p.M, p.K, "fp8 rows operand")) return e;
  static std::atomic<uint64_t> configured{0};
  static int sm_count = NUM_SMS;
  if (first_on_device(configured)) {
    cudaError_t e = cudaFuncSetAttribute(tc::rows_gemm_f8<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tc::F8_SMEM);
    if (e == cudaSuccess) e = cudaFuncSetAttribute(tc::rows_gemm_f8<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tc::F8_SMEM);
    if (e != cudaSuccess) return fail(MAS_ERR_LAUNCH, "cudaFuncSetAttribute(rows_gemm_f8, smem=%zu): %s", tc::F8_SMEM, cudaGetErrorString(e));
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&sm_count, cudaDevAttrMultiProcessorCount, dev);
    mark_device(configured);
  }
  const int64_t nitems = cdiv(p.M, 128) * p.splits * cdiv(p.N, 128);
  const unsigned g = (unsigned)(nitems < sm_count ? nitems : sm_count);
  if (b_e5m2) tc::rows_gemm_f8<true><<<g, tc::F8_THREADS, tc::F8_SMEM, st>>>(p, amap, bmap);
  else tc::rows_gemm_f8<false><<<g, tc::F8_THREADS, tc::F8_SMEM, st>>>(p, amap, bmap);
  return launched_tc(b_e5m2 ? "rows_gemm_f8<e4m3.e5m2>" : "rows_gemm_f8<e4m3.e4m3>");
}

static bool gemm_f8_ok(int64_t M, int N, int K) { return M > 0 && M < (1ll << 31) && N > 0 && K > 0 && K % 16 == 0; }

// weight gradient: rows = N (dy^T), features = K (x^T), contraction over M' = pad16(M).  Split-K over the 128-wide chunks of M'
// so that the (N/128 x K/128) tiles fill whole waves of the 132 SMs; the partial sums cost a reduction pass, so fewer splits
// win ties.  The split depends on the shape only.
static int wgrad_f8_splits(int64_t M, int N, int K) {
  const int64_t tiles = cdiv(N, 128) * cdiv(K, 128), chunks = cdiv(pad16(M), 128);
  int best = 1;
  double best_score = -1.0;
  for (int s = 1; s <= 16 && s <= chunks; ++s) {
    const int64_t g = tiles * s;
    const double eff = (double)g / (double)(cdiv(g, NUM_SMS) * NUM_SMS) - 0.02 * s;
    if (eff > best_score + 1e-9) { best_score = eff; best = s; }
  }
  const int64_t cps = cdiv(chunks, best);
  return (int)cdiv(chunks, cps);
}
static size_t wgrad_f8_ws(int64_t M, int N, int K) {
  if (!gemm_f8_ok(pad16(M), N, K)) return 0;
  const int s = wgrad_f8_splits(M, N, K);
  return s > 1 ? (size_t)s * N * K * sizeof(float) : 0;
}

}  // namespace mas

extern "C" {

size_t mas_to_fp8_ws_bytes(int64_t M, int K) { return (M > 0 && K > 0) ? mas::to_fp8_ws(M, K) : 0; }

int mas_to_fp8(const float* x, int64_t M, int K, int fmt, const float* amax, void* y_rows, void* y_cols, float* colsum, void* ws,
               size_t ws_bytes, void* stream) {
  MAS_REQUIRE(x && (y_rows || y_cols || colsum), "to_fp8: bad arguments");
  return mas::to_fp8_launch(x, M, K, fmt, amax, y_rows, y_cols, colsum, ws, ws_bytes, mas::S(stream));
}

int mas_pack_gemm_f8(const float* w_nk, int N, int K, void* w_f8, void* wt_f8, float* amax, void* stream) {
  MAS_REQUIRE(w_nk && w_f8 && wt_f8 && amax, "pack_gemm_f8: bad arguments");
  if (N <= 0 || K <= 0 || N % 16 || K % 16) return mas::fail(MAS_ERR_UNSUPPORTED, "pack_gemm_f8: needs N %% 16 == 0 and K %% 16 == 0 (N=%d K=%d)", N, K);
  if (int e = mas_amax(w_nk, (int64_t)N * K, amax, stream)) return e;
  return mas::to_fp8_launch(w_nk, N, K, MAS_FP8_E4M3, amax, w_f8, wt_f8, nullptr, nullptr, 0, mas::S(stream));
}

int mas_gemm_rows_f8(const void* x_f8, int64_t M, int K, int x_fmt, const float* x_amax, const void* w_f8, int N, const float* w_amax,
                     const float* bias, float* y, int64_t ldy, void* stream) {
  MAS_REQUIRE(x_f8 && w_f8 && x_amax && w_amax && y && ldy >= N, "gemm_rows_f8: bad arguments");
  if (!mas::gemm_f8_ok(M, N, K)) return mas::fail(MAS_ERR_UNSUPPORTED, "gemm_rows_f8: needs M, N > 0 and K %% 16 == 0 (M=%lld N=%d K=%d)", (long long)M, N, K);
  if (x_fmt != MAS_FP8_E4M3 && x_fmt != MAS_FP8_E5M2) return mas::fail(MAS_ERR_INVALID_ARG, "gemm_rows_f8: x_fmt must be MAS_FP8_E4M3 or MAS_FP8_E5M2");
  if (!mas::al16(x_f8) || !mas::al16(w_f8)) return mas::fail(MAS_ERR_INVALID_ARG, "gemm_rows_f8: operands must be 16-byte aligned");
  mas::tc::F8Params p;
  p.y = y; p.ldy = ldy; p.split_stride = 0; p.bias = bias; p.a_amax = w_amax; p.b_amax = x_amax;
  p.M = M; p.N = N; p.K = K; p.splits = 1; p.cps = (int)mas::cdiv(K, 128);
  return mas::gemm_f8_run(x_fmt == MAS_FP8_E5M2, p, w_f8, x_f8, mas::S(stream));
}

size_t mas_wgrad_rows_f8_ws_bytes(int64_t M, int N, int K) { return mas::wgrad_f8_ws(M, N, K); }

int mas_wgrad_rows_f8(const void* xt_f8, const void* dyt_f8, int64_t M, int N, int K, const float* x_amax, const float* dy_amax, float* dw,
                      void* ws, size_t ws_bytes, void* stream) {
  MAS_REQUIRE(xt_f8 && dyt_f8 && x_amax && dy_amax && dw, "wgrad_rows_f8: bad arguments");
  const int64_t Mp = mas::pad16(M);
  if (M <= 0 || Mp >= (1 << 30) || N <= 0 || K <= 0)
    return mas::fail(MAS_ERR_UNSUPPORTED, "wgrad_rows_f8: needs 0 < M < 2^30 and N, K > 0 (M=%lld N=%d K=%d)", (long long)M, N, K);
  if (ws_bytes < mas::wgrad_f8_ws(M, N, K) || (mas::wgrad_f8_ws(M, N, K) && !ws)) return mas::fail(MAS_ERR_WORKSPACE, "wgrad_rows_f8: workspace too small");
  if (!mas::al16(xt_f8) || !mas::al16(dyt_f8) || !mas::al16(ws)) return mas::fail(MAS_ERR_INVALID_ARG, "wgrad_rows_f8: operands and workspace must be 16-byte aligned");
  const int splits = mas::wgrad_f8_splits(M, N, K);
  mas::tc::F8Params p;
  p.bias = nullptr; p.a_amax = x_amax; p.b_amax = dy_amax;
  p.M = N; p.N = K; p.K = (int)Mp; p.splits = splits; p.cps = (int)mas::cdiv(mas::cdiv(Mp, 128), splits);
  p.ldy = K;
  p.y = splits > 1 ? (float*)ws : dw;
  p.split_stride = (int64_t)N * K;
  if (int e = mas::gemm_f8_run(true, p, xt_f8, dyt_f8, mas::S(stream))) return e;
  if (splits == 1) return MAS_OK;
  mas::conv_wgrad_reduce_launch((const float*)ws, splits, 1, N, K, dw, nullptr, nullptr, mas::S(stream));
  return mas::launched("conv_wgrad_reduce");
}

}  // extern "C"
