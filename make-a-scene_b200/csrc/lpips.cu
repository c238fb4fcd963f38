// LPIPS perceptual loss (losses/lpips.py): everything around the thirteen VGG16 3x3 convolutions, which run on the 3x3
// family (shift_gemm_tc fp16 operands where the shape is tensor-eligible, the exact-fp32 SIMT kernel elsewhere).
//
//   * prep: ScalingLayer (x - shift) / scale of real and fake into ONE channels-last [2B, H, W, 3] batch, real first;
//   * ReLU in place with its max (the power-of-two operand scale of the next convolution), 2x2 floor max-pool with its max;
//   * head forward per tap: n = f / (sqrt(sum_c f^2) + 1e-10), sum_c w_c (n_real - n_fake)^2, per-image partial sums in a
//     fixed order (deterministic), then the five spatial means added in layer order;
//   * tap backward: the head gradient for a unit seed per image, plus the max-pool gradient routed to the FIRST maximum of
//     its window (row-major, as max_pool2d), then the ReLU mask as a select, so a zero-norm pixel (NaN in the reference's
//     sqrt backward, replaced by the ReLU backward's select) writes 0;
//   * ReLU mask select between the data-gradient convolutions, the ScalingLayer backward (division by scale) into the
//     NCHW per-image Jacobian, and the per-image scaling g_b * J_b of every traversal of the graph.
// Every kernel that feeds a convolution also publishes max|output| (atomicMax on the bit pattern of a non-negative float).
#include <cuda_runtime.h>

#include "mas_common.cuh"

namespace mas {

constexpr int LP_HEAD_BLOCKS = 128;   // per-image partial sums of the head (one per block: a fixed reduction order)
constexpr int LP_MAXC = 512;          // widest tap (relu4_3, relu5_3)

__device__ __forceinline__ void block_amax(float m, float* amax) {
  __shared__ float sh[32];
  m = warp_max(m);
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int k = 1; k < (int)(blockDim.x >> 5); ++k) m = fmaxf(m, sh[k]);
    atomicMax(reinterpret_cast<unsigned int*>(amax), __float_as_uint(m));
  }
}

static int grid_of(int64_t work, int threads) {
  const int64_t b = cdiv(work > 0 ? work : 1, threads);
  return (int)(b < NUM_SMS * 16 ? b : NUM_SMS * 16);
}

static int zero_amax(float* amax, cudaStream_t st) {
  if (!amax) return MAS_OK;
  cudaError_t e = cudaMemsetAsync(amax, 0, sizeof(float), st);
  return e == cudaSuccess ? MAS_OK : fail(MAS_ERR_LAUNCH, "lpips: memset: %s", cudaGetErrorString(e));
}

__global__ void lpips_prep_kernel(const float* __restrict__ real, const float* __restrict__ fake, const float* __restrict__ shift,
                                  const float* __restrict__ scale, float* __restrict__ out, int B, int64_t HW) {
  const int64_t total = 2 * (int64_t)B * HW * 3;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % 3);
    const int64_t p = (i / 3) % HW;
    const int64_t n = i / (3 * HW);
    const float* src = n < B ? real + (n * 3 + c) * HW : fake + ((n - B) * 3 + c) * HW;
    out[i] = (__ldg(src + p) - __ldg(shift + c)) / __ldg(scale + c);
  }
}

__global__ void lpips_relu_kernel(float4* __restrict__ y, int64_t n4, float* __restrict__ amax) {
  float m = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    float4 v = y[i];
    v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f);
    y[i] = v;
    m = fmaxf(m, fmaxf(fmaxf(v.x, v.y), fmaxf(v.z, v.w)));
  }
  if (amax) block_amax(m, amax);
}

// x [N, H, W, C] -> y [N, H / 2, W / 2, C] (floor), four channels per thread
__global__ void lpips_maxpool_kernel(const float4* __restrict__ x, float4* __restrict__ y, int N, int H, int W, int C4,
                                     float* __restrict__ amax) {
  const int Ho = H / 2, Wo = W / 2;
  const int64_t total = (int64_t)N * Ho * Wo * C4;
  float m = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C4);
    const int64_t q = i / C4;
    const int j = (int)(q % Wo), r = (int)((q / Wo) % Ho);
    const int64_t n = q / ((int64_t)Wo * Ho);
    const float4* s = x + ((n * H + 2 * r) * W + 2 * j) * C4 + c;
    const float4 a = __ldg(s), b = __ldg(s + C4), d = __ldg(s + (int64_t)W * C4), e = __ldg(s + (int64_t)W * C4 + C4);
    float4 o;
    o.x = fmaxf(fmaxf(a.x, b.x), fmaxf(d.x, e.x));
    o.y = fmaxf(fmaxf(a.y, b.y), fmaxf(d.y, e.y));
    o.z = fmaxf(fmaxf(a.z, b.z), fmaxf(d.z, e.z));
    o.w = fmaxf(fmaxf(a.w, b.w), fmaxf(d.w, e.w));
    y[i] = o;
    m = fmaxf(m, fmaxf(fmaxf(fabsf(o.x), fabsf(o.y)), fmaxf(fabsf(o.z), fabsf(o.w))));
  }
  if (amax) block_amax(m, amax);
}

// grid (LP_HEAD_BLOCKS, B), one warp per pixel: part[b][block] = sum over the block's pixels of sum_c w_c (n_r - n_f)^2
__global__ void __launch_bounds__(256) lpips_head_fwd_kernel(const float* __restrict__ tap, const float* __restrict__ wl, int B,
                                                             int64_t HW, int C, double* __restrict__ part) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, b = blockIdx.y;
  const int kc = C / 32;
  double acc = 0.0;
  for (int64_t p = (int64_t)blockIdx.x * 8 + warp; p < HW; p += (int64_t)LP_HEAD_BLOCKS * 8) {
    const float* r = tap + ((int64_t)b * HW + p) * C;
    const float* f = tap + ((int64_t)(B + b) * HW + p) * C;
    float rv[LP_MAXC / 32], fv[LP_MAXC / 32];
    float sr = 0.f, sf = 0.f;
#pragma unroll
    for (int k = 0; k < LP_MAXC / 32; ++k) {
      if (k < kc) {
        rv[k] = __ldg(r + k * 32 + lane);
        fv[k] = __ldg(f + k * 32 + lane);
        sr = fmaf(rv[k], rv[k], sr);
        sf = fmaf(fv[k], fv[k], sf);
      }
    }
    const float nr = sqrtf(warp_sum(sr)) + 1e-10f, nf = sqrtf(warp_sum(sf)) + 1e-10f;
    float v = 0.f;
#pragma unroll
    for (int k = 0; k < LP_MAXC / 32; ++k) {
      if (k < kc) {
        const float d = rv[k] / nr - fv[k] / nf;
        v = fmaf(__ldg(wl + k * 32 + lane), d * d, v);
      }
    }
    v = warp_sum(v);
    acc += (double)v;
  }
  __shared__ double sh[8];
  if (lane == 0) sh[warp] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int k = 0; k < 8; ++k) s += sh[k];
    part[(int64_t)b * LP_HEAD_BLOCKS + blockIdx.x] = s;
  }
}

struct HW5 { int64_t v[5]; };

// out[b] = mean_0 + mean_1 + ... + mean_4 (fp32, in the reference's order); part [5][B][LP_HEAD_BLOCKS]
__global__ void lpips_head_finalize_kernel(const double* __restrict__ part, int B, HW5 hw, float* __restrict__ out) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= B) return;
  float o = 0.f;
  for (int l = 0; l < 5; ++l) {
    const double* q = part + ((int64_t)l * B + b) * LP_HEAD_BLOCKS;
    double s = 0.0;
    for (int k = 0; k < LP_HEAD_BLOCKS; ++k) s += q[k];
    o += (float)(s / (double)hw.v[l]);
  }
  out[b] = o;
}

// Gradient images gi = 0 .. G-1 are tap images g0 + gi; the partner of tap image t is (t + B) mod 2B.  For a unit seed on
// p_b: a_c = 2 w_c (n_c - n'_c) / HW, d p / d x_c = a_c / D - x_c (sum_k a_k x_k) / (u D^2), u = |x|, D = u + 1e-10.
// dpool [G, H / 2, W / 2, C] (or null) is added at the first maximum of its window; then the ReLU mask (x > 0) selects.
__global__ void __launch_bounds__(256) lpips_tap_bwd_kernel(const float* __restrict__ tap, const float* __restrict__ wl, int B, int H,
                                                            int W, int C, int g0, int G, const float* __restrict__ dpool,
                                                            float* __restrict__ dz, float* __restrict__ amax) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int kc = C / 32;
  const int64_t HW = (int64_t)H * W;
  const int Hp = H / 2, Wp = W / 2;
  const float inv_hw = 1.0f / (float)HW;
  float m = 0.f;
  for (int64_t q = (int64_t)blockIdx.x * 8 + warp; q < (int64_t)G * HW; q += (int64_t)gridDim.x * 8) {
    const int gi = (int)(q / HW);
    const int64_t p = q % HW;
    const int t = g0 + gi, o = t < B ? t + B : t - B;
    const float* xs = tap + ((int64_t)t * HW + p) * C;
    const float* os = tap + ((int64_t)o * HW + p) * C;
    float xv[LP_MAXC / 32], ov[LP_MAXC / 32];
    float sx = 0.f, so = 0.f;
#pragma unroll
    for (int k = 0; k < LP_MAXC / 32; ++k) {
      if (k < kc) {
        xv[k] = __ldg(xs + k * 32 + lane);
        ov[k] = __ldg(os + k * 32 + lane);
        sx = fmaf(xv[k], xv[k], sx);
        so = fmaf(ov[k], ov[k], so);
      }
    }
    const float u = sqrtf(warp_sum(sx));
    const float D = u + 1e-10f, Do = sqrtf(warp_sum(so)) + 1e-10f;
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < LP_MAXC / 32; ++k) {
      if (k < kc) {
        ov[k] = 2.f * __ldg(wl + k * 32 + lane) * (xv[k] / D - ov[k] / Do) * inv_hw;   // a_c
        s = fmaf(ov[k], xv[k], s);
      }
    }
    s = warp_sum(s);
    const float corr = u > 0.f ? s / (u * D * D) : 0.f;
    const int y = (int)(p / W), x = (int)(p % W);
    const bool pooled = dpool != nullptr && y < 2 * Hp && x < 2 * Wp;
    const int y0 = y & ~1, x0 = x & ~1, own = (y - y0) * 2 + (x - x0);
    const float* win = tap + ((int64_t)t * HW + (int64_t)y0 * W + x0) * C;
    float* out = dz + q * C;
#pragma unroll
    for (int k = 0; k < LP_MAXC / 32; ++k) {
      if (k < kc) {
        const int c = k * 32 + lane;
        float g = u > 0.f ? ov[k] / D - xv[k] * corr : 0.f;
        if (pooled) {
          const float v0 = __ldg(win + c), v1 = __ldg(win + C + c), v2 = __ldg(win + (int64_t)W * C + c),
                      v3 = __ldg(win + (int64_t)W * C + C + c);
          int am = 0;
          float best = v0;
          if (v1 > best) { best = v1; am = 1; }
          if (v2 > best) { best = v2; am = 2; }
          if (v3 > best) { am = 3; }
          if (am == own) g += __ldg(dpool + (((int64_t)gi * Hp + (y >> 1)) * Wp + (x >> 1)) * C + c);
        }
        g = xv[k] > 0.f ? g : 0.f;
        out[c] = g;
        m = fmaxf(m, fabsf(g));
      }
    }
  }
  if (amax) block_amax(m, amax);
}

__global__ void lpips_relu_bwd_kernel(const float4* __restrict__ dy, const float4* __restrict__ y, float4* __restrict__ dx, int64_t n4,
                                      float* __restrict__ amax) {
  float m = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    const float4 g = dy[i], a = __ldg(y + i);
    float4 o;
    o.x = a.x > 0.f ? g.x : 0.f;
    o.y = a.y > 0.f ? g.y : 0.f;
    o.z = a.z > 0.f ? g.z : 0.f;
    o.w = a.w > 0.f ? g.w : 0.f;
    dx[i] = o;
    m = fmaxf(m, fmaxf(fmaxf(fabsf(o.x), fabsf(o.y)), fmaxf(fabsf(o.z), fabsf(o.w))));
  }
  if (amax) block_amax(m, amax);
}

// dxp [G, H, W, 3] (gradient of the ScalingLayer output) -> J [G, 3, H, W] = dxp / scale
__global__ void lpips_prep_bwd_kernel(const float* __restrict__ dxp, const float* __restrict__ scale, float* __restrict__ J, int G,
                                      int64_t HW) {
  const int64_t total = (int64_t)G * 3 * HW;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t p = i % HW;
    const int c = (int)((i / HW) % 3);
    const int64_t n = i / (3 * HW);
    J[i] = __ldg(dxp + (n * HW + p) * 3 + c) / __ldg(scale + c);
  }
}

__global__ void lpips_scale_kernel(const float* __restrict__ J, const float* __restrict__ g, int64_t gstride, float* __restrict__ out,
                                   int B, int64_t per) {
  const int64_t total = (int64_t)B * per;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x)
    out[i] = __ldg(g + (i / per) * gstride) * __ldg(J + i);
}

static bool al16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// ---- object-aware loss: LPIPS over box crops on canvases (losses/object_loss.py) ---------------------------------------------
// One size class = 2K canvases [2K, Hc, Wc, C] (crops 0 .. K-1 of img, then the same K of rec), each crop at the canvas origin.
// tab: OBJ_ROW ints per crop (image b, y0, x0, h, w, global box index k), then the per-image row ranges [B+1].  At pooling
// level l the valid region of crop r is (h >> l) x (w >> l); everything outside it is held at zero, which makes every 3x3
// convolution, 2x2 floor pool and head mean on the canvas equal to the same step on the crop alone.
constexpr int OBJ_ROW = 6;

__device__ __forceinline__ void obj_extent(const int* __restrict__ tab, int r, int level, int& h, int& w) {
  h = __ldg(tab + OBJ_ROW * r + 3) >> level;
  w = __ldg(tab + OBJ_ROW * r + 4) >> level;
}

// out [2K, Hc, Wc, 3]: ScalingLayer of the crop inside its extent (pixels outside the image read 0), 0 outside the extent
__global__ void obj_gather_kernel(const int* __restrict__ tab, int K, const float* __restrict__ img, const float* __restrict__ rec,
                                  const float* __restrict__ shift, const float* __restrict__ scale, float* __restrict__ out, int H,
                                  int W, int Hc, int Wc) {
  const int64_t total = 2 * (int64_t)K * Hc * Wc * 3;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % 3);
    const int64_t q = i / 3;
    const int x = (int)(q % Wc), y = (int)((q / Wc) % Hc);
    const int n = (int)(q / ((int64_t)Wc * Hc));
    const int r = n < K ? n : n - K;
    const int* row = tab + OBJ_ROW * r;
    float v = 0.f;
    if (y < __ldg(row + 3) && x < __ldg(row + 4)) {
      const int iy = __ldg(row + 1) + y, ix = __ldg(row + 2) + x;
      const float* src = n < K ? img : rec;
      const float p = (iy >= 0 && iy < H && ix >= 0 && ix < W) ? __ldg(src + (((int64_t)__ldg(row) * 3 + c) * H + iy) * W + ix) : 0.f;
      v = (p - __ldg(shift + c)) / __ldg(scale + c);
    }
    out[i] = v;
  }
}

// y [2K, H, W, C] in place: ReLU inside the level's extent, 0 outside
__global__ void obj_relu_kernel(float4* __restrict__ y, const int* __restrict__ tab, int K, int H, int W, int C4, int level,
                                float* __restrict__ amax) {
  const int64_t n4 = 2 * (int64_t)K * H * W * C4;
  float m = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    const int64_t q = i / C4;
    const int x = (int)(q % W), yy = (int)((q / W) % H);
    const int n = (int)(q / ((int64_t)W * H));
    int h, w;
    obj_extent(tab, n < K ? n : n - K, level, h, w);
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (yy < h && x < w) {
      v = y[i];
      v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f);
      m = fmaxf(m, fmaxf(fmaxf(v.x, v.y), fmaxf(v.z, v.w)));
    }
    y[i] = v;
  }
  if (amax) block_amax(m, amax);
}

// x [2K, H, W, C] at level l -> y [2K, H / 2, W / 2, C]: 2x2 max inside the extent of level l + 1, 0 outside
__global__ void obj_maxpool_kernel(const float4* __restrict__ x, float4* __restrict__ y, const int* __restrict__ tab, int K, int H,
                                   int W, int C4, int level, float* __restrict__ amax) {
  const int Ho = H / 2, Wo = W / 2;
  const int64_t total = 2 * (int64_t)K * Ho * Wo * C4;
  float m = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C4);
    const int64_t q = i / C4;
    const int j = (int)(q % Wo), r = (int)((q / Wo) % Ho);
    const int n = (int)(q / ((int64_t)Wo * Ho));
    int h, w;
    obj_extent(tab, n < K ? n : n - K, level + 1, h, w);
    float4 o = make_float4(0.f, 0.f, 0.f, 0.f);
    if (r < h && j < w) {
      const float4* s = x + (((int64_t)n * H + 2 * r) * W + 2 * j) * C4 + c;
      const float4 a = __ldg(s), b = __ldg(s + C4), d = __ldg(s + (int64_t)W * C4), e = __ldg(s + (int64_t)W * C4 + C4);
      o.x = fmaxf(fmaxf(a.x, b.x), fmaxf(d.x, e.x));
      o.y = fmaxf(fmaxf(a.y, b.y), fmaxf(d.y, e.y));
      o.z = fmaxf(fmaxf(a.z, b.z), fmaxf(d.z, e.z));
      o.w = fmaxf(fmaxf(a.w, b.w), fmaxf(d.w, e.w));
      m = fmaxf(m, fmaxf(fmaxf(fabsf(o.x), fabsf(o.y)), fmaxf(fabsf(o.z), fabsf(o.w))));
    }
    y[i] = o;
  }
  if (amax) block_amax(m, amax);
}

// grid (LP_HEAD_BLOCKS, K), one warp per pixel of crop r's extent: part[r][block], the head sum of lpips_head_fwd_kernel
__global__ void __launch_bounds__(256) obj_head_fwd_kernel(const float* __restrict__ tap, const float* __restrict__ wl,
                                                           const int* __restrict__ tab, int K, int H, int W, int C, int level,
                                                           double* __restrict__ part) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, b = blockIdx.y;
  const int kc = C / 32;
  int h, w;
  obj_extent(tab, b, level, h, w);
  const int64_t area = (int64_t)h * w, HW = (int64_t)H * W;
  double acc = 0.0;
  for (int64_t p = (int64_t)blockIdx.x * 8 + warp; p < area; p += (int64_t)LP_HEAD_BLOCKS * 8) {
    const int64_t pix = (p / w) * W + p % w;
    const float* r = tap + ((int64_t)b * HW + pix) * C;
    const float* f = tap + ((int64_t)(K + b) * HW + pix) * C;
    float rv[LP_MAXC / 32], fv[LP_MAXC / 32];
    float sr = 0.f, sf = 0.f;
#pragma unroll
    for (int k = 0; k < LP_MAXC / 32; ++k) {
      if (k < kc) {
        rv[k] = __ldg(r + k * 32 + lane);
        fv[k] = __ldg(f + k * 32 + lane);
        sr = fmaf(rv[k], rv[k], sr);
        sf = fmaf(fv[k], fv[k], sf);
      }
    }
    const float nr = sqrtf(warp_sum(sr)) + 1e-10f, nf = sqrtf(warp_sum(sf)) + 1e-10f;
    float v = 0.f;
#pragma unroll
    for (int k = 0; k < LP_MAXC / 32; ++k) {
      if (k < kc) {
        const float d = rv[k] / nr - fv[k] / nf;
        v = fmaf(__ldg(wl + k * 32 + lane), d * d, v);
      }
    }
    v = warp_sum(v);
    acc += (double)v;
  }
  __shared__ double sh[8];
  if (lane == 0) sh[warp] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0.0;
    for (int k = 0; k < 8; ++k) s += sh[k];
    part[(int64_t)b * LP_HEAD_BLOCKS + blockIdx.x] = s;
  }
}

// p[k of crop r] = sum over the five levels, in order, of (fp32) part[l][r] / valid area of level l; part [5][K][LP_HEAD_BLOCKS]
__global__ void obj_head_finalize_kernel(const double* __restrict__ part, const int* __restrict__ tab, int K, float* __restrict__ p) {
  const int r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= K) return;
  float o = 0.f;
  for (int l = 0; l < 5; ++l) {
    const double* q = part + ((int64_t)l * K + r) * LP_HEAD_BLOCKS;
    double s = 0.0;
    for (int k = 0; k < LP_HEAD_BLOCKS; ++k) s += q[k];
    int h, w;
    obj_extent(tab, r, l, h, w);
    o += (float)(s / (double)((int64_t)h * w));
  }
  p[tab[OBJ_ROW * r + 5]] = o;
}

// lpips_tap_bwd_kernel per canvas: canvases g0 .. g0+G-1 of the 2K, partner (t + K) mod 2K, the crop's own valid area as the
// mean's divisor, the pooled gradient only inside the extent of level l + 1, and 0 written outside the extent of level l.
__global__ void __launch_bounds__(256) obj_tap_bwd_kernel(const float* __restrict__ tap, const float* __restrict__ wl,
                                                          const int* __restrict__ tab, int K, int H, int W, int C, int level, int g0,
                                                          int G, const float* __restrict__ dpool, float* __restrict__ dz,
                                                          float* __restrict__ amax) {
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int kc = C / 32;
  const int64_t HW = (int64_t)H * W;
  const int Hp = H / 2, Wp = W / 2;
  float m = 0.f;
  for (int64_t q = (int64_t)blockIdx.x * 8 + warp; q < (int64_t)G * HW; q += (int64_t)gridDim.x * 8) {
    const int gi = (int)(q / HW);
    const int64_t p = q % HW;
    const int t = g0 + gi, o = t < K ? t + K : t - K;
    const int y = (int)(p / W), x = (int)(p % W);
    int h, w;
    obj_extent(tab, t < K ? t : t - K, level, h, w);
    float* out = dz + q * C;
    if (y >= h || x >= w) {
#pragma unroll
      for (int k = 0; k < LP_MAXC / 32; ++k)
        if (k < kc) out[k * 32 + lane] = 0.f;
      continue;
    }
    const float inv_hw = 1.0f / (float)((int64_t)h * w);
    const float* xs = tap + ((int64_t)t * HW + p) * C;
    const float* os = tap + ((int64_t)o * HW + p) * C;
    float xv[LP_MAXC / 32], ov[LP_MAXC / 32];
    float sx = 0.f, so = 0.f;
#pragma unroll
    for (int k = 0; k < LP_MAXC / 32; ++k) {
      if (k < kc) {
        xv[k] = __ldg(xs + k * 32 + lane);
        ov[k] = __ldg(os + k * 32 + lane);
        sx = fmaf(xv[k], xv[k], sx);
        so = fmaf(ov[k], ov[k], so);
      }
    }
    const float u = sqrtf(warp_sum(sx));
    const float D = u + 1e-10f, Do = sqrtf(warp_sum(so)) + 1e-10f;
    float s = 0.f;
#pragma unroll
    for (int k = 0; k < LP_MAXC / 32; ++k) {
      if (k < kc) {
        ov[k] = 2.f * __ldg(wl + k * 32 + lane) * (xv[k] / D - ov[k] / Do) * inv_hw;   // a_c
        s = fmaf(ov[k], xv[k], s);
      }
    }
    s = warp_sum(s);
    const float corr = u > 0.f ? s / (u * D * D) : 0.f;
    const bool pooled = dpool != nullptr && y < 2 * (h / 2) && x < 2 * (w / 2);
    const int y0 = y & ~1, x0 = x & ~1, own = (y - y0) * 2 + (x - x0);
    const float* win = tap + ((int64_t)t * HW + (int64_t)y0 * W + x0) * C;
#pragma unroll
    for (int k = 0; k < LP_MAXC / 32; ++k) {
      if (k < kc) {
        const int c = k * 32 + lane;
        float g = u > 0.f ? ov[k] / D - xv[k] * corr : 0.f;
        if (pooled) {
          const float v0 = __ldg(win + c), v1 = __ldg(win + C + c), v2 = __ldg(win + (int64_t)W * C + c),
                      v3 = __ldg(win + (int64_t)W * C + C + c);
          int am = 0;
          float best = v0;
          if (v1 > best) { best = v1; am = 1; }
          if (v2 > best) { best = v2; am = 2; }
          if (v3 > best) { am = 3; }
          if (am == own) g += __ldg(dpool + (((int64_t)gi * Hp + (y >> 1)) * Wp + (x >> 1)) * C + c);
        }
        g = xv[k] > 0.f ? g : 0.f;
        out[c] = g;
        m = fmaxf(m, fabsf(g));
      }
    }
  }
  if (amax) block_amax(m, amax);
}

// J [B,3,H,W] (+)= sum, in row order, over the crops of image b on `side` that cover the pixel of w_k * dxp[crop] / scale
__global__ void obj_scatter_kernel(const float* __restrict__ dxp, const float* __restrict__ scale, const int* __restrict__ tab,
                                   const float* __restrict__ wts, int K, int g0, int side, int Hc, int Wc, float* __restrict__ J,
                                   int B, int H, int W, int accumulate) {
  const int64_t HW = (int64_t)H * W, total = (int64_t)B * 3 * HW;
  const int* offs = tab + OBJ_ROW * K;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int x = (int)(i % W), y = (int)((i / W) % H);
    const int c = (int)((i / HW) % 3), b = (int)(i / (3 * HW));
    const int r1 = __ldg(offs + b + 1);
    const float inv = 1.0f / __ldg(scale + c);
    float s = 0.f;
    for (int r = __ldg(offs + b); r < r1; ++r) {
      const int* row = tab + OBJ_ROW * r;
      const int yy = y - __ldg(row + 1), xx = x - __ldg(row + 2);
      if (yy >= 0 && yy < __ldg(row + 3) && xx >= 0 && xx < __ldg(row + 4)) {
        const int64_t n = (int64_t)side * K + r - g0;
        s = fmaf(__ldg(wts + __ldg(row + 5)), __ldg(dxp + ((n * Hc + yy) * Wc + xx) * 3 + c) * inv, s);
      }
    }
    J[i] = accumulate ? J[i] + s : s;
  }
}

// out = sum_k w_k p_k, fp64 in index order (one thread: K is the number of boxes of a batch)
__global__ void obj_loss_kernel(const float* __restrict__ p, const float* __restrict__ wts, int K, float* __restrict__ out) {
  double s = 0.0;
  for (int k = 0; k < K; ++k) s += (double)wts[k] * (double)p[k];
  *out = (float)s;
}

static bool obj_tab_ok(const int* tab, int K) { return tab != nullptr && K > 0; }

}  // namespace mas

using namespace mas;

extern "C" {

int mas_lpips_prep(const float* real, const float* fake, const float* shift, const float* scale, float* out, int B, int H, int W,
                   void* stream) {
  MAS_REQUIRE(real && fake && shift && scale && out && B > 0 && H > 0 && W > 0, "lpips_prep: bad arguments");
  const int64_t HW = (int64_t)H * W;
  lpips_prep_kernel<<<grid_of(2 * B * HW * 3, 256), 256, 0, S(stream)>>>(real, fake, shift, scale, out, B, HW);
  return launched("lpips_prep");
}

int mas_lpips_relu(float* y, int64_t n, float* amax, void* stream) {
  MAS_REQUIRE(y && n > 0 && n % 4 == 0 && al16(y), "lpips_relu: y must be 16-byte aligned with n %% 4 == 0");
  if (int e = zero_amax(amax, S(stream))) return e;
  lpips_relu_kernel<<<grid_of(n / 4, 256), 256, 0, S(stream)>>>(reinterpret_cast<float4*>(y), n / 4, amax);
  return launched("lpips_relu");
}

int mas_lpips_maxpool(const float* x, float* y, int N, int H, int W, int C, float* amax, void* stream) {
  MAS_REQUIRE(x && y && N > 0 && H >= 2 && W >= 2 && C % 4 == 0 && al16(x) && al16(y), "lpips_maxpool: bad arguments");
  if (int e = zero_amax(amax, S(stream))) return e;
  const int64_t total = (int64_t)N * (H / 2) * (W / 2) * (C / 4);
  lpips_maxpool_kernel<<<grid_of(total, 256), 256, 0, S(stream)>>>(reinterpret_cast<const float4*>(x), reinterpret_cast<float4*>(y),
                                                                  N, H, W, C / 4, amax);
  return launched("lpips_maxpool");
}

int mas_lpips_head_blocks(void) { return LP_HEAD_BLOCKS; }

int mas_lpips_head_forward(const float* tap, const float* w_lin, int B, int H, int W, int C, double* part, void* stream) {
  MAS_REQUIRE(tap && w_lin && part && B > 0 && H > 0 && W > 0 && C % 32 == 0 && C > 0 && C <= LP_MAXC,
              "lpips_head_forward: bad arguments (C=%d must be a multiple of 32, at most %d)", C, LP_MAXC);
  lpips_head_fwd_kernel<<<dim3(LP_HEAD_BLOCKS, B), 256, 0, S(stream)>>>(tap, w_lin, B, (int64_t)H * W, C, part);
  return launched("lpips_head_fwd");
}

int mas_lpips_head_finalize(const double* part, int B, int64_t hw0, int64_t hw1, int64_t hw2, int64_t hw3, int64_t hw4, float* out,
                            void* stream) {
  MAS_REQUIRE(part && out && B > 0, "lpips_head_finalize: bad arguments");
  HW5 hw{{hw0, hw1, hw2, hw3, hw4}};
  lpips_head_finalize_kernel<<<(int)cdiv(B, 128), 128, 0, S(stream)>>>(part, B, hw, out);
  return launched("lpips_head_finalize");
}

int mas_lpips_tap_backward(const float* tap, const float* w_lin, int B, int H, int W, int C, int g0, int G, const float* dpool,
                           float* dz, float* amax, void* stream) {
  MAS_REQUIRE(tap && w_lin && dz && B > 0 && H > 0 && W > 0 && C % 32 == 0 && C > 0 && C <= LP_MAXC && G > 0 && g0 >= 0 &&
                  g0 + G <= 2 * B && (!dpool || (H >= 2 && W >= 2)),
              "lpips_tap_backward: bad arguments");
  if (int e = zero_amax(amax, S(stream))) return e;
  const int64_t warps = (int64_t)G * H * W;
  lpips_tap_bwd_kernel<<<grid_of(warps * 32, 256), 256, 0, S(stream)>>>(tap, w_lin, B, H, W, C, g0, G, dpool, dz, amax);
  return launched("lpips_tap_bwd");
}

int mas_lpips_relu_backward(const float* dy, const float* y, float* dx, int64_t n, float* amax, void* stream) {
  MAS_REQUIRE(dy && y && dx && n > 0 && n % 4 == 0 && al16(dy) && al16(y) && al16(dx), "lpips_relu_backward: bad arguments");
  if (int e = zero_amax(amax, S(stream))) return e;
  lpips_relu_bwd_kernel<<<grid_of(n / 4, 256), 256, 0, S(stream)>>>(reinterpret_cast<const float4*>(dy), reinterpret_cast<const float4*>(y),
                                                                   reinterpret_cast<float4*>(dx), n / 4, amax);
  return launched("lpips_relu_bwd");
}

int mas_lpips_prep_backward(const float* dxp, const float* scale, float* J, int G, int H, int W, void* stream) {
  MAS_REQUIRE(dxp && scale && J && G > 0 && H > 0 && W > 0, "lpips_prep_backward: bad arguments");
  const int64_t HW = (int64_t)H * W;
  lpips_prep_bwd_kernel<<<grid_of(G * 3 * HW, 256), 256, 0, S(stream)>>>(dxp, scale, J, G, HW);
  return launched("lpips_prep_bwd");
}

int mas_lpips_scale_jacobian(const float* J, const float* g, int64_t g_stride, float* out, int B, int64_t per, void* stream) {
  MAS_REQUIRE(J && g && out && B > 0 && per > 0, "lpips_scale_jacobian: bad arguments");
  lpips_scale_kernel<<<grid_of(B * per, 256), 256, 0, S(stream)>>>(J, g, g_stride, out, B, per);
  return launched("lpips_scale");
}

int mas_object_gather(const int* tab, int K, const float* img, const float* rec, const float* shift, const float* scale, float* out,
                      int H, int W, int Hc, int Wc, void* stream) {
  MAS_REQUIRE(obj_tab_ok(tab, K) && img && rec && shift && scale && out && H > 0 && W > 0 && Hc > 0 && Wc > 0,
              "object_gather: bad arguments");
  obj_gather_kernel<<<grid_of(2 * (int64_t)K * Hc * Wc * 3, 256), 256, 0, S(stream)>>>(tab, K, img, rec, shift, scale, out, H, W, Hc, Wc);
  return launched("object_gather");
}

int mas_object_relu(float* y, const int* tab, int K, int H, int W, int C, int level, float* amax, void* stream) {
  MAS_REQUIRE(y && obj_tab_ok(tab, K) && H > 0 && W > 0 && C > 0 && C % 4 == 0 && level >= 0 && al16(y),
              "object_relu: bad arguments (C=%d must be a multiple of 4, y 16-byte aligned)", C);
  if (int e = zero_amax(amax, S(stream))) return e;
  obj_relu_kernel<<<grid_of(2 * (int64_t)K * H * W * (C / 4), 256), 256, 0, S(stream)>>>(reinterpret_cast<float4*>(y), tab, K, H, W,
                                                                                       C / 4, level, amax);
  return launched("object_relu");
}

int mas_object_maxpool(const float* x, float* y, const int* tab, int K, int H, int W, int C, int level, float* amax, void* stream) {
  MAS_REQUIRE(x && y && obj_tab_ok(tab, K) && H >= 2 && W >= 2 && C > 0 && C % 4 == 0 && level >= 0 && al16(x) && al16(y),
              "object_maxpool: bad arguments");
  if (int e = zero_amax(amax, S(stream))) return e;
  const int64_t total = 2 * (int64_t)K * (H / 2) * (W / 2) * (C / 4);
  obj_maxpool_kernel<<<grid_of(total, 256), 256, 0, S(stream)>>>(reinterpret_cast<const float4*>(x), reinterpret_cast<float4*>(y), tab,
                                                                K, H, W, C / 4, level, amax);
  return launched("object_maxpool");
}

int mas_object_head_forward(const float* tap, const float* w_lin, const int* tab, int K, int H, int W, int C, int level, double* part,
                            void* stream) {
  MAS_REQUIRE(tap && w_lin && part && obj_tab_ok(tab, K) && H > 0 && W > 0 && C % 32 == 0 && C > 0 && C <= LP_MAXC && level >= 0,
              "object_head_forward: bad arguments (C=%d must be a multiple of 32, at most %d)", C, LP_MAXC);
  obj_head_fwd_kernel<<<dim3(LP_HEAD_BLOCKS, K), 256, 0, S(stream)>>>(tap, w_lin, tab, K, H, W, C, level, part);
  return launched("object_head_fwd");
}

int mas_object_head_finalize(const double* part, const int* tab, int K, float* p, void* stream) {
  MAS_REQUIRE(part && p && obj_tab_ok(tab, K), "object_head_finalize: bad arguments");
  obj_head_finalize_kernel<<<(int)cdiv(K, 128), 128, 0, S(stream)>>>(part, tab, K, p);
  return launched("object_head_finalize");
}

int mas_object_tap_backward(const float* tap, const float* w_lin, const int* tab, int K, int H, int W, int C, int level, int g0, int G,
                            const float* dpool, float* dz, float* amax, void* stream) {
  MAS_REQUIRE(tap && w_lin && dz && obj_tab_ok(tab, K) && H > 0 && W > 0 && C % 32 == 0 && C > 0 && C <= LP_MAXC && level >= 0 &&
                  G > 0 && g0 >= 0 && g0 + G <= 2 * K && (!dpool || (H >= 2 && W >= 2)),
              "object_tap_backward: bad arguments");
  if (int e = zero_amax(amax, S(stream))) return e;
  obj_tap_bwd_kernel<<<grid_of((int64_t)G * H * W * 32, 256), 256, 0, S(stream)>>>(tap, w_lin, tab, K, H, W, C, level, g0, G, dpool,
                                                                                  dz, amax);
  return launched("object_tap_bwd");
}

int mas_object_scatter(const float* dxp, const float* scale, const int* tab, const float* wts, int K, int g0, int G, int side, int Hc,
                       int Wc, float* J, int B, int H, int W, int accumulate, void* stream) {
  MAS_REQUIRE(dxp && scale && wts && J && obj_tab_ok(tab, K) && (side == 0 || side == 1) && g0 >= 0 && G > 0 && g0 + G <= 2 * K &&
                  side * K >= g0 && side * K + K <= g0 + G && Hc > 0 && Wc > 0 && B > 0 && H > 0 && W > 0,
              "object_scatter: bad arguments (the canvases g0 .. g0+G-1 must hold every crop of side %d)", side);
  obj_scatter_kernel<<<grid_of((int64_t)B * 3 * H * W, 256), 256, 0, S(stream)>>>(dxp, scale, tab, wts, K, g0, side, Hc, Wc, J, B, H, W,
                                                                                 accumulate);
  return launched("object_scatter");
}

int mas_object_loss(const float* p, const float* wts, int K, float* out, void* stream) {
  MAS_REQUIRE(p && wts && out && K > 0, "object_loss: bad arguments");
  obj_loss_kernel<<<1, 1, 0, S(stream)>>>(p, wts, K, out);
  return launched("object_loss");
}

}  // extern "C"
