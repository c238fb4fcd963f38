// Codebook (vector quantiser) kernels — replaces modules.py:501-517 (distance matrix, argmin, gather,
// loss, straight-through) with one fused kernel; the [R,K] distance matrix is never written.
//
// Arithmetic contract (SURVEY.md 7.3 #1): d[r,k] = fl( fl(|z_r|^2 + |e_k|^2) - 2*dot(z_r,e_k) ) with the
// dot product accumulated in fp32 FMA over k ascending, strict '<' scan over codes ascending =>
// first-index tie-break, i.e. the reference's formula, association and argmin semantics.  Pure fp32 FFMA:
// no TF32/BF16 on this contraction, so indices agree with a strict-fp32 oracle except on rows whose two best
// distances are within a few ulp (classified by the tests with an fp64 gap).
#include <stdlib.h>

#include "mas_common.cuh"

namespace mas {

// tensor-core filter stage (vq_tc.cu)
bool vq_filter_tc_ok(int64_t R, int K, int D);
int vq_filter_splits(int64_t R, int K);
size_t vq_filter_pack_bytes(int K, int D);
int vq_filter_tc_launch(const float* z, const float* E, const float* ee, const float* z_amax, const float* e_amax, int64_t R, int K,
                        int D, float* cand, int splits, void* pack_buf, cudaStream_t st);

constexpr int VQ_BM = 64;    // latent rows per CTA
constexpr int VQ_BN = 128;   // codes per tile
constexpr int VQ_BK = 32;    // dims per smem stage
constexpr int VQ_LDE = VQ_BK + 4;
constexpr int VQ_THREADS = 256;  // 16 (codes) x 16 (row groups); each thread owns a 4 x 8 register tile
constexpr int VQ_TM = 4;       // (8 x 8 tiles with 128 threads measured slower: 168 registers, 12 warps/SM)

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem) {
  uint32_t s = (uint32_t)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(s), "l"(gmem));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;"); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;" ::"n"(N)); }

// |e_k|^2 per code: one warp per code, lanes stride the row, xor-tree combine (deterministic)
__global__ void vq_code_norms(const float* __restrict__ E, int K, int D, float* __restrict__ ee,
                              unsigned int* __restrict__ ee_max /*or null: max_k |e_k|^2 (float bits, zeroed by the caller)*/) {
  int k = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (k >= K) return;
  int lane = threadIdx.x & 31;
  float s = 0.f;
  for (int d = lane; d < D; d += 32) {
    float v = E[(size_t)k * D + d];
    s = fmaf(v, v, s);
  }
  s = warp_sum(s);
  if (lane == 0) {
    ee[k] = s;
    if (ee_max) atomicMax(ee_max, __float_as_uint(s));
  }
}

__global__ void __launch_bounds__(VQ_THREADS, 2)
vq_forward_kernel(const float* __restrict__ z, const float* __restrict__ E, const float* __restrict__ ee, int64_t R, int K, int D,
                  float* __restrict__ best_val /*[R][splits]*/, int* __restrict__ best_idx /*[R][splits]*/,
                  const int* __restrict__ row_list /*or null: the rows to evaluate, in this order*/,
                  const int* __restrict__ row_count /*with row_list: how many (device scalar)*/, int blk_off) {
  if (row_list) {   // fallback pass of the tensor-core filter: only the listed rows, results indexed by list position
    R = *row_count;
    if (((int64_t)blockIdx.x + blk_off) * VQ_BM >= R) return;
  }
  extern __shared__ __align__(16) float smem[];
  const int LDZ = D + 4;
  float* Zs = smem;                             // [VQ_BM][LDZ]
  float* Es = Zs + VQ_BM * LDZ;                 // [2][VQ_BN][VQ_LDE]
  float* zz_s = Es + 2 * VQ_BN * VQ_LDE;        // [VQ_BM]
  int* idx_s = reinterpret_cast<int*>(zz_s + VQ_BM);  // [VQ_BM]
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const int tx = t & 15, ty = t >> 4;
  const int64_t row0 = ((int64_t)blockIdx.x + blk_off) * VQ_BM;
  // blockIdx.y selects a contiguous slice of the code tiles: two CTAs per SM (one per slice) double the resident
  // warps of this FFMA-bound kernel; the slices are merged (smaller distance, then smaller index) by vq_merge_kernel
  const int nkc = D / VQ_BK, ntile_all = (K + VQ_BN - 1) / VQ_BN;
  const int tiles_per = (ntile_all + gridDim.y - 1) / gridDim.y;
  const int tile_lo = blockIdx.y * tiles_per, tile_hi = min(ntile_all, tile_lo + tiles_per);
  const int ntile = max(0, tile_hi - tile_lo), nstage = nkc * ntile;

  auto load_stage = [&](int s) {
    const int ct = tile_lo + s / nkc, kc = s % nkc;
    float* dst = Es + (s & 1) * VQ_BN * VQ_LDE;
#pragma unroll
    for (int i = 0; i < (VQ_BN * VQ_BK / 4) / VQ_THREADS; ++i) {
      int f = t + i * VQ_THREADS, code = f >> 3, kq = f & 7;
      int gcode = min(ct * VQ_BN + code, K - 1);
      cp_async16(dst + code * VQ_LDE + kq * 4, E + (size_t)gcode * D + kc * VQ_BK + kq * 4);
    }
    cp_async_commit();
  };
  if (nstage > 0) load_stage(0);

  // z tile -> shared (zero rows beyond R), and |z|^2 per row
  for (int f = t; f < VQ_BM * (D / 4); f += VQ_THREADS) {
    int r = f / (D / 4), q = f % (D / 4);
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (row0 + r < R) {
      const int64_t src = row_list ? (int64_t)row_list[row0 + r] : row0 + r;
      v = __ldg(reinterpret_cast<const float4*>(z + (size_t)src * D) + q);
    }
    *reinterpret_cast<float4*>(Zs + r * LDZ + q * 4) = v;
  }
  __syncthreads();
  for (int r = warp * (VQ_BM / (VQ_THREADS / 32)); r < (warp + 1) * (VQ_BM / (VQ_THREADS / 32)); ++r) {
    float s = 0.f;
    for (int d = lane; d < D; d += 32) {
      float v = Zs[r * LDZ + d];
      s = fmaf(v, v, s);
    }
    s = warp_sum(s);
    if (lane == 0) zz_s[r] = s;
  }

  float acc[VQ_TM][8];
  float best[VQ_TM];
  int bidx[VQ_TM];
#pragma unroll
  for (int i = 0; i < VQ_TM; ++i) {
    best[i] = INFINITY;
    bidx[i] = 0;
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
  }

  for (int s = 0; s < nstage; ++s) {
    if (s + 1 < nstage) {
      load_stage(s + 1);
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();
    const int ct = tile_lo + s / nkc, kc = s % nkc;
    const float* es = Es + (s & 1) * VQ_BN * VQ_LDE;
    const float* zs = Zs + kc * VQ_BK;
#pragma unroll
    for (int k4 = 0; k4 < VQ_BK / 4; ++k4) {
      float4 a[VQ_TM], b[8];
#pragma unroll
      for (int i = 0; i < VQ_TM; ++i) a[i] = *reinterpret_cast<const float4*>(zs + (ty * VQ_TM + i) * LDZ + k4 * 4);
#pragma unroll
      for (int j = 0; j < 8; ++j) b[j] = *reinterpret_cast<const float4*>(es + (j * 16 + tx) * VQ_LDE + k4 * 4);
#pragma unroll
      for (int i = 0; i < VQ_TM; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          acc[i][j] = fmaf(a[i].x, b[j].x, acc[i][j]);
          acc[i][j] = fmaf(a[i].y, b[j].y, acc[i][j]);
          acc[i][j] = fmaf(a[i].z, b[j].z, acc[i][j]);
          acc[i][j] = fmaf(a[i].w, b[j].w, acc[i][j]);
        }
    }
    if (kc == nkc - 1) {  // tile finished: distances + running argmin (codes ascending inside a thread)
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        int code = ct * VQ_BN + j * 16 + tx;
        if (code < K) {
          float e2 = __ldg(ee + code);
#pragma unroll
          for (int i = 0; i < VQ_TM; ++i) {
            float d = (zz_s[ty * VQ_TM + i] + e2) - 2.0f * acc[i][j];
            if (d < best[i]) {
              best[i] = d;
              bidx[i] = code;
            }
          }
        }
#pragma unroll
        for (int i = 0; i < VQ_TM; ++i) acc[i][j] = 0.f;
      }
    }
    __syncthreads();  // stage buffer (s&1) is refilled by the prefetch issued in iteration s+1
  }

  // combine the 16 tx-lanes of each row: smaller distance wins, ties -> smaller index (first occurrence)
#pragma unroll
  for (int i = 0; i < VQ_TM; ++i) {
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) {
      float ov = __shfl_xor_sync(0xffffffffu, best[i], o);
      int oi = __shfl_xor_sync(0xffffffffu, bidx[i], o);
      if (ov < best[i] || (ov == best[i] && oi < bidx[i])) {
        best[i] = ov;
        bidx[i] = oi;
      }
    }
    if (tx == 0 && row0 + ty * VQ_TM + i < R) {
      best_val[(row0 + ty * VQ_TM + i) * gridDim.y + blockIdx.y] = best[i];
      best_idx[(row0 + ty * VQ_TM + i) * gridDim.y + blockIdx.y] = bidx[i];
    }
  }
}

// merge the code slices (first index wins ties), gather + straight-through value + loss partial (modules.py:505-512)
__global__ void __launch_bounds__(256) vq_merge_kernel(const float* __restrict__ z, const float* __restrict__ E,
                                                       const float* __restrict__ best_val, const int* __restrict__ best_idx,
                                                       int splits, int64_t R, int D, int64_t* __restrict__ idx_out,
                                                       float* __restrict__ zq_out, double* __restrict__ loss_part) {
  __shared__ double red_s[8];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * 8 + warp;
  float ls = 0.f;
  if (row < R) {
    float bv = best_val[row * splits];
    int bi = best_idx[row * splits];
    for (int s = 1; s < splits; ++s) {
      float v = best_val[row * splits + s];
      int i = best_idx[row * splits + s];
      if (v < bv || (v == bv && i < bi)) { bv = v; bi = i; }
    }
    if (lane == 0 && idx_out) idx_out[row] = (int64_t)bi;
    for (int q = lane; q < (D >> 2); q += 32) {
      const float4 e = __ldg(reinterpret_cast<const float4*>(E + (size_t)bi * D) + q);
      const float4 zv = __ldg(reinterpret_cast<const float4*>(z + (size_t)row * D) + q);
      const float4 df = make_float4(e.x - zv.x, e.y - zv.y, e.z - zv.z, e.w - zv.w);
      ls += df.x * df.x + df.y * df.y + df.z * df.z + df.w * df.w;
      // z + (z_q - z).detach(): the forward VALUE carries these two roundings in the reference too
      reinterpret_cast<float4*>(zq_out + (size_t)row * D)[q] = make_float4(zv.x + df.x, zv.y + df.y, zv.z + df.z, zv.w + df.w);
    }
  }
  ls = warp_sum(ls);
  if (lane == 0) red_s[warp] = (double)ls;
  __syncthreads();
  if (threadIdx.x == 0) {
    double a = 0;
    for (int k = 0; k < 8; ++k) a += red_s[k];
    loss_part[blockIdx.x] = a;
  }
}

// ---- tensor-core filter, resolve stage (see vq_tc.cu) ----------------------------------------------------------------
// Error model behind the margin.  For a pair (row r, code k) let P = |z_r| * max_k |e_k| >= sum_i |z_i e_i|.
//   * operand split: each operand keeps >= 22 significant bits and the product of the two low parts is dropped:
//       |error| <= (2^-21 + 2^-22) P;
//   * fp32 accumulation in the tensor cores: at most 3 * D/16 + 16 * 3 additions per dot product in whatever order and
//     rounding mode (truncation assumed): <= (3*D/16 + 48) * 2^-23 * 3 P   (the factor 3: three partial products of size <= P);
//   * the exact path itself (the FFMA kernel, and equally the reference's sgemm in any summation order):
//       <= (D + 2) * 2^-24 * P  for the dot product, + 3 * 2^-24 * (|z|^2 + |e|^2) for the two roundings of the formula.
// d = |z|^2 + |e|^2 - 2 dot, so a distance is known to  err_d = 2 * (sum of the dot bounds) + the formula term, and two
// codes whose approximate distances differ by more than 2 * err_d cannot swap order in ANY of these evaluations.
constexpr int VQ_REC = 12, VQ_NCAND = 4, VQ_FB_SPLITS = 16;

__device__ __forceinline__ float vq_margin(float zz, float ee_max, int D) {
  const float P = sqrtf(zz) * sqrtf(ee_max);
  const float c_split = 7.2e-7f;                                        // 2^-21 + 2^-22, rounded up
  const float c_acc = (float)(3 * (D / 16) + 48) * 3.0f * 1.1920929e-7f;  // 2^-23 per addition
  const float c_exact = (float)(D + 2) * 5.9604645e-8f;                 // 2^-24 per FMA
  const float err_d = 2.0f * (c_split + c_acc + c_exact) * P + 3.0f * 5.9604645e-8f * (zz + ee_max) * 2.0f;
  return 2.0f * err_d * 1.25f;                                           // 25 % slack on top of the bound
}

// warp per row: merge the code splits' candidate lists, decide, re-evaluate exactly where needed
__global__ void __launch_bounds__(256) vq_resolve_kernel(const float* __restrict__ z, const float* __restrict__ E, const float* __restrict__ ee,
                                                         const float* __restrict__ cand, int splits, int64_t R, int K, int D,
                                                         const unsigned int* __restrict__ ee_max_bits, int* __restrict__ final_idx,
                                                         int* __restrict__ list, int* __restrict__ count) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * 8 + warp;
  if (row >= R) return;
  // |z|^2 exactly as the FFMA kernel computes it (lane-strided fp32 FMA partials, xor-tree combine)
  float zz = 0.f;
  for (int d = lane; d < D; d += 32) {
    const float v = __ldg(z + (size_t)row * D + d);
    zz = fmaf(v, v, zz);
  }
  zz = warp_sum(zz);
  // merged candidate list (every lane computes the same thing from broadcast loads: splits <= 4, 4 entries each)
  float b[VQ_NCAND + 1];
  int ci[VQ_NCAND];
#pragma unroll
  for (int j = 0; j <= VQ_NCAND; ++j) b[j] = INFINITY;
#pragma unroll
  for (int j = 0; j < VQ_NCAND; ++j) ci[j] = 0x7fffffff;
  for (int s = 0; s < splits; ++s) {
    const float* rec = cand + ((size_t)row * splits + s) * VQ_REC;
#pragma unroll
    for (int j = 0; j <= VQ_NCAND; ++j) {
      const float d = rec[j];
      const int code = j < VQ_NCAND ? __float_as_int(rec[5 + j]) : 0x7fffffff;
      // insertion keeping (value, then code) ascending; the fifth value of a split only matters as a value
      if (d < b[VQ_NCAND]) {
        int pos = VQ_NCAND;
        while (pos > 0 && (d < b[pos - 1] || (d == b[pos - 1] && pos - 1 < VQ_NCAND && code < ci[pos - 1]))) --pos;
        for (int q = VQ_NCAND; q > pos; --q) {
          b[q] = b[q - 1];
          if (q < VQ_NCAND) ci[q] = ci[q - 1];
        }
        b[pos] = d;
        if (pos < VQ_NCAND) ci[pos] = code;
      }
    }
  }
  const float margin = vq_margin(zz, __uint_as_float(*ee_max_bits), D);
  const float lim = b[0] + margin;
  int n_in = 1;
#pragma unroll
  for (int j = 1; j < VQ_NCAND; ++j) n_in += (b[j] <= lim) ? 1 : 0;
  const bool multi = b[VQ_NCAND] <= lim || !(b[0] < INFINITY);
  // a candidate slot may hold a value without a code (the fifth value of one split promoted by the merge): treat as "too many"
  bool unknown = false;
#pragma unroll
  for (int j = 0; j < VQ_NCAND; ++j) unknown = unknown || (j < n_in && ci[j] == 0x7fffffff);
  if (multi || unknown) {
    if (lane == 0) {
      const int pos = atomicAdd(count, 1);
      list[pos] = (int)row;
      final_idx[row] = -1;
    }
    return;
  }
  if (n_in == 1) {
    if (lane == 0) final_idx[row] = ci[0];
    return;
  }
  // exact re-evaluation of the candidates: fl(fl(|z|^2 + |e|^2) - 2 dot), dot in fp32 FMA over k ascending (vq_forward_kernel)
  float dv = INFINITY;
  int dc = 0x7fffffff;
  if (lane < n_in) {
    int code = ci[0];
#pragma unroll
    for (int j = 1; j < VQ_NCAND; ++j) code = (lane == j) ? ci[j] : code;
    const float* zr = z + (size_t)row * D;
    const float* er = E + (size_t)code * D;
    float acc = 0.f;
    for (int k = 0; k < D; k += 4) {
      const float4 a = __ldg(reinterpret_cast<const float4*>(zr + k)), e4 = __ldg(reinterpret_cast<const float4*>(er + k));
      acc = fmaf(a.x, e4.x, acc);
      acc = fmaf(a.y, e4.y, acc);
      acc = fmaf(a.z, e4.z, acc);
      acc = fmaf(a.w, e4.w, acc);
    }
    dv = (zz + __ldg(ee + code)) - 2.0f * acc;
    dc = code;
  }
#pragma unroll
  for (int o = 2; o > 0; o >>= 1) {   // lanes 0..3: smaller distance wins, ties -> smaller code (first occurrence)
    const float ov = __shfl_xor_sync(0xffffffffu, dv, o);
    const int oc = __shfl_xor_sync(0xffffffffu, dc, o);
    if (ov < dv || (ov == dv && oc < dc)) { dv = ov; dc = oc; }
  }
  if (lane == 0) final_idx[row] = dc;
}

// rows the filter could not decide: merge the exact kernel's per-split results (indexed by list position)
__global__ void vq_fallback_merge_kernel(const float* __restrict__ fb_val, const int* __restrict__ fb_idx, int splits,
                                         const int* __restrict__ list, const int* __restrict__ count, int* __restrict__ final_idx) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= *count) return;
  float bv = fb_val[(size_t)j * splits];
  int bi = fb_idx[(size_t)j * splits];
  for (int s = 1; s < splits; ++s) {
    const float v = fb_val[(size_t)j * splits + s];
    const int i = fb_idx[(size_t)j * splits + s];
    if (v < bv || (v == bv && i < bi)) { bv = v; bi = i; }
  }
  final_idx[list[j]] = bi;
}

// ---- k-means update step of the codebook re-initialisation (modules.py:487-499; the assignment step is the VQ kernel) ----
__global__ void kmeans_accumulate_kernel(const float* __restrict__ x, const int64_t* __restrict__ idx, int64_t n, int D,
                                         double* __restrict__ sums, int* __restrict__ cnt) {
  const int D4 = D >> 2;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n * D4; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t r = i / D4;
    const int q = (int)(i % D4);
    const int64_t k = idx[r];
    const float4 v = __ldg(reinterpret_cast<const float4*>(x) + i);
    double* s = sums + (size_t)k * D + q * 4;   // fp64 accumulation: the order of the atomics is invisible after rounding to fp32
    atomicAdd(s + 0, (double)v.x);
    atomicAdd(s + 1, (double)v.y);
    atomicAdd(s + 2, (double)v.z);
    atomicAdd(s + 3, (double)v.w);
    if (q == 0) atomicAdd(cnt + k, 1);
  }
}
// new centre = mean of its members (an empty cluster keeps its old centre); shift2 += |new - old|^2
__global__ void kmeans_finalize_kernel(const double* __restrict__ sums, const int* __restrict__ cnt, const float* __restrict__ old_c,
                                       float* __restrict__ new_c, int K, int D, double* __restrict__ shift2) {
  double acc = 0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < (int64_t)K * D; i += (int64_t)gridDim.x * blockDim.x) {
    const int k = (int)(i / D);
    const int c = cnt[k];
    const float o = old_c[i];
    const float v = c > 0 ? (float)(sums[i] / (double)c) : o;
    new_c[i] = v;
    acc += ((double)v - o) * ((double)v - o);
  }
  for (int off = 16; off > 0; off >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, off);
  if ((threadIdx.x & 31) == 0 && acc != 0) atomicAdd(shift2, acc);
}

__global__ void kmeans_shift_kernel(const double* __restrict__ shift2, float* __restrict__ out) { out[0] = (float)sqrt(shift2[0]); }

// caller-supplied code indices (int64, clamped) -> the (value, index) slot layout vq_merge_kernel reads with splits = 1
__global__ void vq_given_indices_kernel(const int64_t* __restrict__ idx_in, int64_t R, int K, float* __restrict__ best_val,
                                        int* __restrict__ best_idx) {
  int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  int64_t k = idx_in[r];
  best_idx[r] = (int)(k < 0 ? 0 : (k >= K ? K - 1 : k));
  best_val[r] = 0.f;
}

__global__ void vq_loss_final(const double* __restrict__ part, int n, double inv_count, float beta, float* __restrict__ out) {
  __shared__ double sh[256];
  double a = 0;
  for (int i = threadIdx.x; i < n; i += 256) a += part[i];
  sh[threadIdx.x] = a;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    float m = (float)(sh[0] * inv_count);
    out[0] = m + beta * m;  // mean((zq.detach()-z)^2) + beta*mean((zq-z.detach())^2), modules.py:509
  }
}

__global__ void vq_backward_kernel(const float* __restrict__ g_zq, const float* __restrict__ g_loss, const float* __restrict__ z,
                                   const float* __restrict__ E, const int64_t* __restrict__ idx, int64_t R, int D, float beta,
                                   float* __restrict__ grad_z, float* __restrict__ grad_E) {
  const int D4 = D >> 2;
  const float gl = g_loss ? g_loss[0] : 0.f;
  const float cz = gl * 2.0f / (float)((double)R * D), ce = cz * beta;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < R * D4; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t r = i / D4;
    int q = (int)(i % D4);
    int64_t k = idx[r];
    float4 zv = __ldg(reinterpret_cast<const float4*>(z) + i);
    float4 e = __ldg(reinterpret_cast<const float4*>(E + (size_t)k * D) + q);
    float4 g = g_zq ? __ldg(reinterpret_cast<const float4*>(g_zq) + i) : make_float4(0.f, 0.f, 0.f, 0.f);
    float4 df = make_float4(zv.x - e.x, zv.y - e.y, zv.z - e.z, zv.w - e.w);
    if (grad_z) reinterpret_cast<float4*>(grad_z)[i] = make_float4(g.x + cz * df.x, g.y + cz * df.y, g.z + cz * df.z, g.w + cz * df.w);
    if (grad_E && gl != 0.f) {
      float* ge = grad_E + (size_t)k * D + q * 4;
      atomicAdd(ge + 0, -ce * df.x);
      atomicAdd(ge + 1, -ce * df.y);
      atomicAdd(ge + 2, -ce * df.z);
      atomicAdd(ge + 3, -ce * df.w);
    }
  }
}

__global__ void vq_gather_kernel(const float* __restrict__ E, const int64_t* __restrict__ idx, int64_t R, int K, int D,
                                 float* __restrict__ out) {
  const int D4 = D >> 2;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < R * D4; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t r = i / D4, k = idx[r];
    k = k < 0 ? 0 : (k >= K ? K - 1 : k);
    reinterpret_cast<float4*>(out)[i] = __ldg(reinterpret_cast<const float4*>(E + (size_t)k * D) + (i % D4));
  }
}

}  // namespace mas

using namespace mas;

extern "C" {

static int vq_splits(int64_t R) { return cdiv(R, VQ_BM) < NUM_SMS * 2 ? 2 : 1; }
static size_t a256(size_t v) { return (v + 255) / 256 * 256; }
static std::atomic<int> g_vq_tc{-1};   // -1: unset (MAS_VQ_TC=0 in the environment disables), 0 / 1: mas_vq_select_path
static bool vq_use_tc(int64_t R, int K, int D) {
  int v = g_vq_tc.load(std::memory_order_relaxed);
  if (v < 0) {
    const char* e = getenv("MAS_VQ_TC");
    v = (e && e[0] == '0') ? 0 : 1;
  }
  return v != 0 && vq_filter_tc_ok(R, K, D) && R <= 0x7fffffff / 16;
}

int mas_vq_select_path(int use_tensor_core_filter) {
  g_vq_tc.store(use_tensor_core_filter ? 1 : 0);
  return MAS_OK;
}

size_t mas_vq_ws_bytes(int64_t R, int K, int D) {
  size_t base = a256((size_t)K * sizeof(float)) + a256((size_t)R * 4 * sizeof(float)) + a256((size_t)R * 4 * sizeof(int)) +
                a256((size_t)cdiv(R, 8) * sizeof(double)) + 256;
  if (vq_use_tc(R, K, D))   // candidate records, final indices, undecided-row list, fallback results, scalars
    base += a256((size_t)R * 4 * VQ_REC * sizeof(float)) + 2 * a256((size_t)R * sizeof(int)) +
            2 * a256((size_t)R * VQ_FB_SPLITS * sizeof(float)) + a256(vq_filter_pack_bytes(K, D)) + 256;
  return base;
}

static int vq_config_exact() {
  static std::atomic<uint64_t> configured{0};   // per-device: the opt-in ceiling (227 KB), whatever D asks for later
  if (first_on_device(configured)) {
    cudaError_t e = cudaFuncSetAttribute(vq_forward_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 232448);
    if (e != cudaSuccess) return fail(MAS_ERR_LAUNCH, "vq_forward: smem attr: %s", cudaGetErrorString(e));
    mark_device(configured);
  }
  return MAS_OK;
}

int mas_vq_forward(const float* z, const float* E, int64_t R, int K, int D, float beta, int64_t* idx_out, float* zq_out,
                   float* loss_out, void* ws, size_t ws_bytes, void* stream) {
  MAS_REQUIRE(R > 0 && K > 0 && D > 0, "vq_forward: bad shape R=%lld K=%d D=%d", (long long)R, K, D);
  if (D % VQ_BK != 0) return fail(MAS_ERR_UNSUPPORTED, "vq_forward: D=%d must be a multiple of %d", D, VQ_BK);
  if (ws_bytes < mas_vq_ws_bytes(R, K, D)) return fail(MAS_ERR_WORKSPACE, "vq_forward: workspace too small");
  char* w = (char*)ws;
  float* ee = (float*)w; w += a256((size_t)K * sizeof(float));
  float* bval = (float*)w; w += a256((size_t)R * 4 * sizeof(float));
  int* bidx = (int*)w; w += a256((size_t)R * 4 * sizeof(int));
  double* part = (double*)w; w += a256((size_t)cdiv(R, 8) * sizeof(double));
  size_t smem = ((size_t)VQ_BM * (D + 4) + 2 * VQ_BN * VQ_LDE + VQ_BM) * sizeof(float) + VQ_BM * sizeof(int);
  if (smem > 232448) return fail(MAS_ERR_UNSUPPORTED, "vq_forward: D=%d needs %zu bytes of shared memory", D, smem);
  if (int e = vq_config_exact()) return e;
  const int mblocks = (int)cdiv(R, 8);
  if (vq_use_tc(R, K, D)) {
    // tensor-core filter -> resolve (exact re-evaluation of near ties) -> FFMA kernel on the undecided rows only
    float* cand = (float*)w; w += a256((size_t)R * 4 * VQ_REC * sizeof(float));
    int* final_idx = (int*)w; w += a256((size_t)R * sizeof(int));
    int* list = (int*)w; w += a256((size_t)R * sizeof(int));
    float* fb_val = (float*)w; w += a256((size_t)R * VQ_FB_SPLITS * sizeof(float));
    int* fb_idx = (int*)w; w += a256((size_t)R * VQ_FB_SPLITS * sizeof(float));
    void* pack_buf = w; w += a256(vq_filter_pack_bytes(K, D));
    float* scal = (float*)w;   // [0] max|z|  [1] max|E|  [2] max |e|^2 (bits)  [3] undecided-row count
    cudaError_t ce = cudaMemsetAsync(scal, 0, 4 * sizeof(float), S(stream));
    if (ce != cudaSuccess) return fail(MAS_ERR_LAUNCH, "vq_forward: memset: %s", cudaGetErrorString(ce));
    if (int e = mas_amax(z, R * D, scal + 0, stream)) return e;
    if (int e = mas_amax(E, (int64_t)K * D, scal + 1, stream)) return e;
    vq_code_norms<<<(int)cdiv(K, 8), 256, 0, S(stream)>>>(E, K, D, ee, reinterpret_cast<unsigned int*>(scal + 2));
    if (int e = launched("vq_code_norms")) return e;
    const int fsplits = vq_filter_splits(R, K);
    if (int e = vq_filter_tc_launch(z, E, ee, scal + 0, scal + 1, R, K, D, cand, fsplits, pack_buf, S(stream))) return e;
    vq_resolve_kernel<<<mblocks, 256, 0, S(stream)>>>(z, E, ee, cand, fsplits, R, K, D, reinterpret_cast<const unsigned int*>(scal + 2),
                                                     final_idx, list, reinterpret_cast<int*>(scal + 3));
    if (int e = launched("vq_resolve")) return e;
    // every CTA beyond the undecided-row count returns at once: with ordinary data this launch is a few microseconds
    const int64_t fb_blocks = cdiv(R, VQ_BM);
    for (int64_t off = 0; off < fb_blocks; off += 1024) {
      const unsigned nb = (unsigned)(fb_blocks - off < 1024 ? fb_blocks - off : 1024);
      vq_forward_kernel<<<dim3(nb, VQ_FB_SPLITS), VQ_THREADS, smem, S(stream)>>>(z, E, ee, R, K, D, fb_val, fb_idx, list,
                                                                                  reinterpret_cast<const int*>(scal + 3), (int)off);
      if (int e = launched("vq_forward(undecided rows)")) return e;
    }
    vq_fallback_merge_kernel<<<(int)cdiv(R, 256), 256, 0, S(stream)>>>(fb_val, fb_idx, VQ_FB_SPLITS, list,
                                                                        reinterpret_cast<const int*>(scal + 3), final_idx);
    if (int e = launched("vq_fallback_merge")) return e;
    vq_merge_kernel<<<mblocks, 256, 0, S(stream)>>>(z, E, bval, final_idx, 1, R, D, idx_out, zq_out, part);
    if (int e = launched("vq_merge")) return e;
  } else {
    const int blocks = (int)cdiv(R, VQ_BM), splits = vq_splits(R);
    vq_code_norms<<<(int)cdiv(K, 8), 256, 0, S(stream)>>>(E, K, D, ee, nullptr);
    if (int e = launched("vq_code_norms")) return e;
    vq_forward_kernel<<<dim3(blocks, splits), VQ_THREADS, smem, S(stream)>>>(z, E, ee, R, K, D, bval, bidx, nullptr, nullptr, 0);
    if (int e = launched("vq_forward")) return e;
    vq_merge_kernel<<<mblocks, 256, 0, S(stream)>>>(z, E, bval, bidx, splits, R, D, idx_out, zq_out, part);
    if (int e = launched("vq_merge")) return e;
  }
  vq_loss_final<<<1, 256, 0, S(stream)>>>(part, mblocks, 1.0 / ((double)R * D), beta, loss_out);
  return launched("vq_loss_final");
}

int mas_vq_forward_given(const float* z, const float* E, const int64_t* idx_in, int64_t R, int K, int D, float beta,
                         float* zq_out, float* loss_out, void* ws, size_t ws_bytes, void* stream) {
  MAS_REQUIRE(R > 0 && K > 0 && D > 0 && D % 4 == 0, "vq_forward_given: bad shape R=%lld K=%d D=%d", (long long)R, K, D);
  if (ws_bytes < mas_vq_ws_bytes(R, K, D)) return fail(MAS_ERR_WORKSPACE, "vq_forward_given: workspace too small");
  char* w = (char*)ws;
  w += a256((size_t)K * sizeof(float));
  float* bval = (float*)w; w += a256((size_t)R * 4 * sizeof(float));
  int* bidx = (int*)w; w += a256((size_t)R * 4 * sizeof(int));
  double* part = (double*)w;
  vq_given_indices_kernel<<<(int)cdiv(R, 256), 256, 0, S(stream)>>>(idx_in, R, K, bval, bidx);
  if (int e = launched("vq_given_indices")) return e;
  const int mblocks = (int)cdiv(R, 8);
  vq_merge_kernel<<<mblocks, 256, 0, S(stream)>>>(z, E, bval, bidx, 1, R, D, nullptr, zq_out, part);
  if (int e = launched("vq_merge")) return e;
  vq_loss_final<<<1, 256, 0, S(stream)>>>(part, mblocks, 1.0 / ((double)R * D), beta, loss_out);
  return launched("vq_loss_final");
}

size_t mas_kmeans_ws_bytes(int K, int D) { return a256((size_t)K * D * sizeof(double)) + a256((size_t)K * sizeof(int)) + 256; }

int mas_kmeans_update(const float* x, const int64_t* idx, int64_t n, int K, int D, const float* centres_old, float* centres_new,
                      float* shift_out, void* ws, size_t ws_bytes, void* stream) {
  MAS_REQUIRE(x && idx && centres_old && centres_new && n > 0 && K > 0 && D > 0 && D % 4 == 0, "kmeans_update: bad arguments");
  if (ws_bytes < mas_kmeans_ws_bytes(K, D)) return fail(MAS_ERR_WORKSPACE, "kmeans_update: workspace too small");
  char* w = (char*)ws;
  double* sums = (double*)w; w += a256((size_t)K * D * sizeof(double));
  int* cnt = (int*)w; w += a256((size_t)K * sizeof(int));
  double* shift2 = (double*)w;
  cudaError_t e = cudaMemsetAsync(ws, 0, mas_kmeans_ws_bytes(K, D), S(stream));
  if (e != cudaSuccess) return fail(MAS_ERR_LAUNCH, "kmeans_update: memset: %s", cudaGetErrorString(e));
  const int64_t items = n * (D / 4);
  kmeans_accumulate_kernel<<<(int)(cdiv(items, 256) < NUM_SMS * 16 ? cdiv(items, 256) : NUM_SMS * 16), 256, 0, S(stream)>>>(x, idx, n, D, sums, cnt);
  if (int er = launched("kmeans_accumulate")) return er;
  const int64_t tot = (int64_t)K * D;
  kmeans_finalize_kernel<<<(int)(cdiv(tot, 256) < NUM_SMS * 8 ? cdiv(tot, 256) : NUM_SMS * 8), 256, 0, S(stream)>>>(sums, cnt, centres_old, centres_new,
                                                                                                       K, D, shift2);
  if (int er = launched("kmeans_finalize")) return er;
  if (shift_out) {
    kmeans_shift_kernel<<<1, 1, 0, S(stream)>>>(shift2, shift_out);
    return launched("kmeans_shift");
  }
  return MAS_OK;
}

int mas_vq_backward(const float* g_zq, const float* g_loss, const float* z, const float* E, const int64_t* idx, int64_t R, int K,
                    int D, float beta, float* grad_z, float* grad_E, void* stream) {
  (void)K;
  MAS_REQUIRE(R > 0 && D > 0 && D % 4 == 0, "vq_backward: bad shape");
  int64_t n = R * (D / 4);
  int grid = (int)(cdiv(n, 256) < NUM_SMS * 16 ? cdiv(n, 256) : NUM_SMS * 16);
  vq_backward_kernel<<<grid, 256, 0, S(stream)>>>(g_zq, g_loss, z, E, idx, R, D, beta, grad_z, grad_E);
  return launched("vq_backward");
}

int mas_vq_gather(const float* E, const int64_t* idx, int64_t R, int K, int D, float* out, void* stream) {
  MAS_REQUIRE(R > 0 && D > 0 && D % 4 == 0, "vq_gather: bad shape");
  int64_t n = R * (D / 4);
  int grid = (int)(cdiv(n, 256) < NUM_SMS * 16 ? cdiv(n, 256) : NUM_SMS * 16);
  vq_gather_kernel<<<grid, 256, 0, S(stream)>>>(E, idx, R, K, D, out);
  return launched("vq_gather");
}

}  // extern "C"
