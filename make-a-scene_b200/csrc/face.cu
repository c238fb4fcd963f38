// VGGFace2 face loss (losses/face_loss.py): everything around the ResNet-50's 1x1 convolutions (row GEMMs on fp16 operands)
// and 3x3 convolutions (the 3x3 family), forward and data gradient.
//
//   * prepare: crop (zeros outside the image) + antialiased bilinear Resize(256) + CenterCrop(254) of every used face from
//     the NCHW (any-stride) img / rec into ONE channels-last batch [F, 254, 254, 3], from a per-face table built on the host
//     (separable tap weights); its adjoint gathers per image pixel over the faces in a fixed order (deterministic, boxes
//     may overlap);
//   * stem: the 7x7/2 3 -> 64 convolution (feature 0, fp32) and its data gradient, direct kernels with the weights in
//     shared memory (Cin = 3 does not fit the tensor tiles);
//   * bn1 + ReLU + 3x3/2 max-pool in one pass (window argmax kept for the backward), and its backward: the pooled gradient
//     at the FIRST maximum of each window (row-major, as max_pool2d), the ReLU select, the bn1 scale, plus feature 0's seed;
//   * the L1 taps: per level sum |a - b| over the pairs (a: face p, b: face p + P) in per-block fp64 partials reduced in a
//     fixed order, and sign(a - b) as int8 for the backward seeds alpha_l * sign / (C H W);
//   * Bottleneck glue: stride-2 subsample into the scaled fp16 operand of the 1x1 GEMMs, and the block output's ReLU backward
//     with the seed of a tap and the (possibly stride-2 zero-stuffed) gradient of the next block added in.
// Every kernel that feeds a convolution publishes max|output| (atomicMax on the bit pattern of a non-negative float).
#include <cuda_fp16.h>
#include <cuda_runtime.h>

#include "mas_common.cuh"
#include "tc_ptx.cuh"

namespace mas {
namespace face {

constexpr int CROP = 254;        // CenterCrop(254)
constexpr int META = 14;         // ints per face in the table (see mas_face_prepare in mas_b200.h)
constexpr int L1_BLOCKS = 128;   // partial sums per level (one per block: a fixed reduction order)
constexpr int STEM_C = 64;

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
  return e == cudaSuccess ? MAS_OK : fail(MAS_ERR_LAUNCH, "face: memset: %s", cudaGetErrorString(e));
}

static bool al16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// meta row: src image, side (0 img, 1 rec), top, left, crop h, crop w, taps y, taps x, then absolute offsets into tab of the
// row / column start indices (254 each) and of the row / column adjoint ranges (2 per crop row / column: [lo, hi) of the
// output rows / columns that read it), and into wts of the row / column weights (254 x taps each).
struct Meta {
  int src, side, top, left, ch, cw, ky, kx, o_sy, o_sx, o_ay, o_ax, o_wy, o_wx;
};

__device__ __forceinline__ Meta meta_of(const int* __restrict__ tab, int f) {
  const int* m = tab + f * META;
  return Meta{m[0], m[1], m[2], m[3], m[4], m[5], m[6], m[7], m[8], m[9], m[10], m[11], m[12], m[13]};
}

__global__ void prepare_kernel(const int* __restrict__ tab, const float* __restrict__ wts, int F, const float* __restrict__ img,
                               mas_tensor4 is, const float* __restrict__ rec, mas_tensor4 rs, float* __restrict__ out) {
  const int64_t total = (int64_t)F * CROP * CROP;
  for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < total; q += (int64_t)gridDim.x * blockDim.x) {
    const int x = (int)(q % CROP), y = (int)((q / CROP) % CROP), f = (int)(q / (CROP * CROP));
    const Meta m = meta_of(tab, f);
    const float* src = m.side ? rec : img;
    const mas_tensor4 t = m.side ? rs : is;
    const float* base = src + (int64_t)m.src * t.sn;
    const int sy = __ldg(tab + m.o_sy + y), sx = __ldg(tab + m.o_sx + x);
    float a0 = 0.f, a1 = 0.f, a2 = 0.f;
    for (int i = 0; i < m.ky; ++i) {
      const float wy = __ldg(wts + m.o_wy + y * m.ky + i);
      const int cy = sy + i, r = m.top + cy;
      if (wy == 0.f || cy >= m.ch || r < 0 || r >= t.h) continue;
      float b0 = 0.f, b1 = 0.f, b2 = 0.f;
      for (int j = 0; j < m.kx; ++j) {
        const float wx = __ldg(wts + m.o_wx + x * m.kx + j);
        const int cx = sx + j, c = m.left + cx;
        if (wx == 0.f || cx >= m.cw || c < 0 || c >= t.w) continue;
        const float* p = base + (int64_t)r * t.sh + (int64_t)c * t.sw;
        b0 = fmaf(wx, __ldg(p), b0);
        b1 = fmaf(wx, __ldg(p + t.sc), b1);
        b2 = fmaf(wx, __ldg(p + 2 * t.sc), b2);
      }
      a0 = fmaf(wy, b0, a0);
      a1 = fmaf(wy, b1, a1);
      a2 = fmaf(wy, b2, a2);
    }
    float* o = out + q * 3;
    o[0] = a0; o[1] = a1; o[2] = a2;
  }
}

// d [G, 254, 254, 3] is the gradient of faces f0 .. f0+G-1; J [B, 3, H, W] (dense NCHW) receives, for every pixel of the
// side's images, the sum over those faces (in face order) that crop it from this side.
__global__ void prepare_bwd_kernel(const int* __restrict__ tab, const float* __restrict__ wts, int f0, int G, int side,
                                   const float* __restrict__ d, float* __restrict__ J, int B, int H, int W) {
  const int64_t HW = (int64_t)H * W, total = (int64_t)B * HW;
  for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < total; q += (int64_t)gridDim.x * blockDim.x) {
    const int b = (int)(q / HW);
    const int r = (int)((q % HW) / W), c = (int)(q % W);
    float a0 = 0.f, a1 = 0.f, a2 = 0.f;
    for (int g = 0; g < G; ++g) {
      const Meta m = meta_of(tab, f0 + g);
      if (m.side != side || m.src != b) continue;
      const int cy = r - m.top, cx = c - m.left;
      if (cy < 0 || cy >= m.ch || cx < 0 || cx >= m.cw) continue;
      const int ylo = __ldg(tab + m.o_ay + 2 * cy), yhi = __ldg(tab + m.o_ay + 2 * cy + 1);
      const int xlo = __ldg(tab + m.o_ax + 2 * cx), xhi = __ldg(tab + m.o_ax + 2 * cx + 1);
      const float* dg = d + (int64_t)g * CROP * CROP * 3;
      for (int y = ylo; y < yhi; ++y) {
        const int i = cy - __ldg(tab + m.o_sy + y);
        if (i < 0 || i >= m.ky) continue;
        const float wy = __ldg(wts + m.o_wy + y * m.ky + i);
        float b0 = 0.f, b1 = 0.f, b2 = 0.f;
        for (int x = xlo; x < xhi; ++x) {
          const int j = cx - __ldg(tab + m.o_sx + x);
          if (j < 0 || j >= m.kx) continue;
          const float wx = __ldg(wts + m.o_wx + x * m.kx + j);
          const float* p = dg + ((int64_t)y * CROP + x) * 3;
          b0 = fmaf(wx, __ldg(p), b0);
          b1 = fmaf(wx, __ldg(p + 1), b1);
          b2 = fmaf(wx, __ldg(p + 2), b2);
        }
        a0 = fmaf(wy, b0, a0);
        a1 = fmaf(wy, b1, a1);
        a2 = fmaf(wy, b2, a2);
      }
    }
    float* o = J + (int64_t)b * 3 * HW + (q % HW);
    o[0] = a0; o[HW] = a1; o[2 * HW] = a2;
  }
}

// x [N, H, W, 3] -> y [N, Ho, Wo, 64], y = conv7x7/2 pad 3 (no bias). One output pixel (all 64 channels) per thread; the
// weights sit in shared memory as [tap][ci][co] and every warp reads them by broadcast.
__global__ void __launch_bounds__(128) stem_fwd_kernel(const float* __restrict__ x, const float* __restrict__ w_oihw,
                                                       float* __restrict__ y, int N, int H, int W, int Ho, int Wo) {
  __shared__ __align__(16) float ws[49 * 3 * STEM_C];
  for (int i = threadIdx.x; i < 49 * 3 * STEM_C; i += blockDim.x) {
    const int co = i % STEM_C, ci = (i / STEM_C) % 3, t = i / (3 * STEM_C);
    ws[i] = __ldg(w_oihw + (co * 3 + ci) * 49 + t);
  }
  __syncthreads();
  const int64_t total = (int64_t)N * Ho * Wo;
  const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= total) return;
  const int ox = (int)(q % Wo), oy = (int)((q / Wo) % Ho);
  const int64_t n = q / ((int64_t)Wo * Ho);
  float acc[STEM_C];
#pragma unroll
  for (int k = 0; k < STEM_C; ++k) acc[k] = 0.f;
  for (int ky = 0; ky < 7; ++ky) {
    const int iy = 2 * oy - 3 + ky;
    if (iy < 0 || iy >= H) continue;
    for (int kx = 0; kx < 7; ++kx) {
      const int ix = 2 * ox - 3 + kx;
      if (ix < 0 || ix >= W) continue;
      const float* px = x + ((n * H + iy) * W + ix) * 3;
      const float4* wt = reinterpret_cast<const float4*>(ws + (ky * 7 + kx) * 3 * STEM_C);
#pragma unroll
      for (int ci = 0; ci < 3; ++ci) {
        const float v = __ldg(px + ci);
#pragma unroll
        for (int k = 0; k < STEM_C / 4; ++k) {
          const float4 w4 = wt[ci * (STEM_C / 4) + k];
          acc[4 * k] = fmaf(v, w4.x, acc[4 * k]);
          acc[4 * k + 1] = fmaf(v, w4.y, acc[4 * k + 1]);
          acc[4 * k + 2] = fmaf(v, w4.z, acc[4 * k + 2]);
          acc[4 * k + 3] = fmaf(v, w4.w, acc[4 * k + 3]);
        }
      }
    }
  }
  float4* o = reinterpret_cast<float4*>(y + q * STEM_C);
#pragma unroll
  for (int k = 0; k < STEM_C / 4; ++k) o[k] = make_float4(acc[4 * k], acc[4 * k + 1], acc[4 * k + 2], acc[4 * k + 3]);
}

// dy [N, Ho, Wo, 64] -> dx [N, H, W, 3]: dx(iy, ix, ci) = sum over the taps with iy = 2 oy - 3 + ky (and likewise x) of
// dy(oy, ox, :) . w(:, ci, ky, kx). Threads are ordered (n, iy, ix parity, ix / 2) so a warp shares its tap set.
__global__ void __launch_bounds__(128) stem_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ w_oihw,
                                                       float* __restrict__ dx, int N, int H, int W, int Ho, int Wo) {
  __shared__ float ws[49 * STEM_C * 3];   // [tap][co][ci]
  for (int i = threadIdx.x; i < 49 * STEM_C * 3; i += blockDim.x) {
    const int ci = i % 3, co = (i / 3) % STEM_C, t = i / (3 * STEM_C);
    ws[i] = __ldg(w_oihw + (co * 3 + ci) * 49 + t);
  }
  __syncthreads();
  const int Wh = (W + 1) / 2;
  const int64_t total = (int64_t)N * H * 2 * Wh;
  const int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (q >= total) return;
  const int jx = (int)(q % Wh), px = (int)((q / Wh) & 1);
  const int iy = (int)((q / (2 * Wh)) % H);
  const int64_t n = q / (2 * (int64_t)Wh * H);
  const int ix = 2 * jx + px;
  if (ix >= W) return;
  float a0 = 0.f, a1 = 0.f, a2 = 0.f;
  for (int ky = (iy + 3) & 1; ky < 7; ky += 2) {
    const int oy = (iy + 3 - ky) >> 1;
    if (oy < 0 || oy >= Ho) continue;
    for (int kx = (ix + 3) & 1; kx < 7; kx += 2) {
      const int ox = (ix + 3 - kx) >> 1;
      if (ox < 0 || ox >= Wo) continue;
      const float4* g = reinterpret_cast<const float4*>(dy + ((n * Ho + oy) * Wo + ox) * STEM_C);
      const float* wt = ws + (ky * 7 + kx) * STEM_C * 3;
#pragma unroll 4
      for (int k = 0; k < STEM_C / 4; ++k) {
        const float4 gv = __ldg(g + k);
        const float gg[4] = {gv.x, gv.y, gv.z, gv.w};
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float* w3 = wt + (4 * k + e) * 3;
          a0 = fmaf(gg[e], w3[0], a0);
          a1 = fmaf(gg[e], w3[1], a1);
          a2 = fmaf(gg[e], w3[2], a2);
        }
      }
    }
  }
  float* o = dx + ((n * H + iy) * W + ix) * 3;
  o[0] = a0; o[1] = a1; o[2] = a2;
}

// x [N, H, W, C] (the stem output), bn [2][C] = (scale, shift) of the eval BatchNorm: y [N, Ho, Wo, C] = max over the 3x3/2
// window of relu(x * scale + shift); arg [N, Ho, Wo, C] = row-major index (0..8) of the window's first maximum.
__global__ void pool_fwd_kernel(const float* __restrict__ x, const float* __restrict__ bn, float* __restrict__ y,
                                uint8_t* __restrict__ arg, int N, int H, int W, int C, int Ho, int Wo, float* __restrict__ amax) {
  const int64_t total = (int64_t)N * Ho * Wo * C;
  float m = 0.f;
  for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < total; q += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(q % C);
    const int64_t p = q / C;
    const int ox = (int)(p % Wo), oy = (int)((p / Wo) % Ho);
    const int64_t n = p / ((int64_t)Wo * Ho);
    const float s = __ldg(bn + c), t = __ldg(bn + C + c);
    float best = 0.f;
    int bi = 0;
#pragma unroll
    for (int k = 0; k < 9; ++k) {
      const int iy = 2 * oy + k / 3, ix = 2 * ox + k % 3;
      const float v = fmaxf(fmaf(__ldg(x + ((n * H + iy) * W + ix) * C + c), s, t), 0.f);
      if (k == 0 || v > best) { best = v; bi = k; }
    }
    y[q] = best;
    arg[q] = (uint8_t)bi;
    m = fmaxf(m, best);
  }
  if (amax) block_amax(m, amax);
}

// Seed of tap level l for face f0 + g: coef * sign(a - b) with + for the first half of the pairs (a), - for the second (b).
__device__ __forceinline__ float seed_of(const int8_t* __restrict__ sgn, float coef, int f, int P, int64_t per, int64_t e) {
  const int p = f < P ? f : f - P;
  const float v = coef * (float)__ldg(sgn + (int64_t)p * per + e);
  return f < P ? v : -v;
}

// dx [G, H, W, C] = scale_c * [relu'(z)] * (sum of dp over the windows whose first maximum is this element) + seed,
// z = x * scale + shift; x, arg, dp are the images f0 .. f0+G-1 (x, arg: [G, ...] slices given by the caller).
__global__ void pool_bwd_kernel(const float* __restrict__ x, const float* __restrict__ bn, const uint8_t* __restrict__ arg,
                                const float* __restrict__ dp, const int8_t* __restrict__ sgn, float coef, int f0, int P, int G,
                                int H, int W, int C, int Ho, int Wo, float* __restrict__ dx) {
  const int64_t per = (int64_t)H * W * C;
  const int64_t total = (int64_t)G * per;
  for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < total; q += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(q % C);
    const int64_t p = q / C;
    const int ix = (int)(p % W), iy = (int)((p / W) % H);
    const int g = (int)(p / ((int64_t)W * H));
    float acc = 0.f;
    if (dp) {
      const int oy1 = min(iy / 2, Ho - 1), ox1 = min(ix / 2, Wo - 1);
      for (int oy = max((iy - 1) / 2, 0); oy <= oy1; ++oy) {
        if (iy - 2 * oy > 2 || iy < 2 * oy) continue;
        for (int ox = max((ix - 1) / 2, 0); ox <= ox1; ++ox) {
          if (ix - 2 * ox > 2 || ix < 2 * ox) continue;
          const int64_t o = (((int64_t)g * Ho + oy) * Wo + ox) * C + c;
          if ((int)__ldg(arg + o) == (iy - 2 * oy) * 3 + (ix - 2 * ox)) acc += __ldg(dp + o);
        }
      }
      const float s = __ldg(bn + c);
      const float z = fmaf(__ldg(x + q), s, __ldg(bn + C + c));
      acc = z > 0.f ? acc * s : 0.f;
    }
    if (sgn) acc += seed_of(sgn, coef, f0 + g, P, per, q % per);
    dx[q] = acc;
  }
}

// grid (L1_BLOCKS): part[block] = sum over the block's elements of |a - b|, a = feature of pair p, b = of pair p + P;
// sgn = sign(a - b).
__global__ void __launch_bounds__(256) l1_fwd_kernel(const float* __restrict__ f, int64_t n, int8_t* __restrict__ sgn,
                                                     double* __restrict__ part) {
  double acc = 0.0;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float a = __ldg(f + i), b = __ldg(f + n + i);
    acc += (double)fabsf(a - b);
    if (sgn) sgn[i] = (int8_t)((a > b) - (a < b));
  }
  __shared__ double sh[256];
  sh[threadIdx.x] = acc;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) part[blockIdx.x] = sh[0];
}

struct Coef5 { double v[5]; };

// terms[l] = coef_l * sum_k part[l][k] (coef_l = alpha_l / (C H W)), loss = terms summed in level order (fp32)
__global__ void l1_finalize_kernel(const double* __restrict__ part, Coef5 coef, float* __restrict__ terms, float* __restrict__ loss) {
  if (threadIdx.x != 0) return;
  float o = 0.f;
  for (int l = 0; l < 5; ++l) {
    double s = 0.0;
    for (int k = 0; k < L1_BLOCKS; ++k) s += part[l * L1_BLOCKS + k];
    const float t = (float)(coef.v[l] * s);
    terms[l] = t;
    o += t;
  }
  *loss = o;
}

// x [N, H, W, C] -> y16 [N, ceil(H/2), ceil(W/2), C] = fp16(x[2i, 2j] * s), s the power-of-two operand scale of *amax
__global__ void subsample_half_kernel(const float4* __restrict__ x, uint2* __restrict__ y, int N, int H, int W, int C4,
                                      const float* __restrict__ amax) {
  float inv;
  const float s = tc::operand_scale(amax, &inv);
  const int Ho = (H + 1) / 2, Wo = (W + 1) / 2;
  const int64_t total = (int64_t)N * Ho * Wo * C4;
  for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < total; q += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(q % C4);
    const int64_t p = q / C4;
    const int j = (int)(p % Wo), i = (int)((p / Wo) % Ho);
    const int64_t n = p / ((int64_t)Wo * Ho);
    const float4 v = __ldg(x + ((n * H + 2 * i) * W + 2 * j) * C4 + c);
    const __half2 lo = __floats2half2_rn(v.x * s, v.y * s), hi = __floats2half2_rn(v.z * s, v.w * s);
    uint2 o;
    o.x = *reinterpret_cast<const uint32_t*>(&lo);
    o.y = *reinterpret_cast<const uint32_t*>(&hi);
    y[q] = o;
  }
}

// dz [G, H, W, C] = out > 0 ? (dout + seed) : 0 for the block output `out` (images f0 .. f0+G-1). dout: [G, H, W, C], or with
// half != 0 the gradient [G, ceil(H/2), ceil(W/2), C] of a stride-2 consumer (it reaches the even positions only), or null.
__global__ void relu_seed_bwd_kernel(const float* __restrict__ out, const float* __restrict__ dout, int half,
                                     const int8_t* __restrict__ sgn, float coef, int f0, int P, int G, int H, int W, int C,
                                     float* __restrict__ dz, float* __restrict__ amax) {
  const int64_t per = (int64_t)H * W * C;
  const int64_t total = (int64_t)G * per;
  const int Hh = (H + 1) / 2, Wh = (W + 1) / 2;
  float m = 0.f;
  for (int64_t q = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; q < total; q += (int64_t)gridDim.x * blockDim.x) {
    float g = 0.f;
    if (__ldg(out + q) > 0.f) {
      if (dout) {
        if (half) {
          const int c = (int)(q % C);
          const int64_t p = q / C;
          const int x = (int)(p % W), y = (int)((p / W) % H);
          const int64_t n = p / ((int64_t)W * H);
          if (!(x & 1) && !(y & 1)) g = __ldg(dout + ((n * Hh + (y >> 1)) * Wh + (x >> 1)) * C + c);
        } else {
          g = __ldg(dout + q);
        }
      }
      if (sgn) g += seed_of(sgn, coef, f0 + (int)(q / per), P, per, q % per);
    }
    dz[q] = g;
    m = fmaxf(m, fabsf(g));
  }
  if (amax) block_amax(m, amax);
}

}  // namespace face
}  // namespace mas

using namespace mas;
using namespace mas::face;

extern "C" {

int mas_face_prepare(const int* tab, const float* wts, int F, const float* img, mas_tensor4 is, const float* rec, mas_tensor4 rs,
                     float* out, void* stream) {
  MAS_REQUIRE(tab && wts && img && rec && out && F > 0 && is.c == 3 && rs.c == 3, "face_prepare: bad arguments");
  prepare_kernel<<<grid_of((int64_t)F * CROP * CROP, 256), 256, 0, S(stream)>>>(tab, wts, F, img, is, rec, rs, out);
  return launched("face_prepare");
}

int mas_face_prepare_backward(const int* tab, const float* wts, int f0, int G, int side, const float* d, float* J, int B, int H,
                              int W, void* stream) {
  MAS_REQUIRE(tab && wts && d && J && f0 >= 0 && G > 0 && (side == 0 || side == 1) && B > 0 && H > 0 && W > 0,
              "face_prepare_backward: bad arguments");
  prepare_bwd_kernel<<<grid_of((int64_t)B * H * W, 256), 256, 0, S(stream)>>>(tab, wts, f0, G, side, d, J, B, H, W);
  return launched("face_prepare_bwd");
}

int mas_face_stem_forward(const float* x, const float* w, float* y, int N, int H, int W, void* stream) {
  MAS_REQUIRE(x && w && y && N > 0 && H > 0 && W > 0 && al16(y), "face_stem_forward: bad arguments");
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
  stem_fwd_kernel<<<(int)cdiv((int64_t)N * Ho * Wo, 128), 128, 0, S(stream)>>>(x, w, y, N, H, W, Ho, Wo);
  return launched("face_stem_fwd");
}

int mas_face_stem_backward(const float* dy, const float* w, float* dx, int N, int H, int W, void* stream) {
  MAS_REQUIRE(dy && w && dx && N > 0 && H > 0 && W > 0 && al16(dy), "face_stem_backward: bad arguments");
  const int Ho = (H - 1) / 2 + 1, Wo = (W - 1) / 2 + 1;
  stem_bwd_kernel<<<(int)cdiv((int64_t)N * H * 2 * ((W + 1) / 2), 128), 128, 0, S(stream)>>>(dy, w, dx, N, H, W, Ho, Wo);
  return launched("face_stem_bwd");
}

int mas_face_pool_forward(const float* x, const float* bn, float* y, uint8_t* arg, int N, int H, int W, int C, float* amax,
                          void* stream) {
  MAS_REQUIRE(x && bn && y && arg && N > 0 && H >= 3 && W >= 3 && C > 0 && (H - 3) % 2 == 0 && (W - 3) % 2 == 0,
              "face_pool_forward: bad arguments (every 3x3/2 window must be full: H, W odd and >= 3)");
  if (int e = zero_amax(amax, S(stream))) return e;
  const int Ho = (H - 3) / 2 + 1, Wo = (W - 3) / 2 + 1;
  pool_fwd_kernel<<<grid_of((int64_t)N * Ho * Wo * C, 256), 256, 0, S(stream)>>>(x, bn, y, arg, N, H, W, C, Ho, Wo, amax);
  return launched("face_pool_fwd");
}

int mas_face_pool_backward(const float* x, const float* bn, const uint8_t* arg, const float* dp, const int8_t* sgn, float coef,
                           int f0, int P, int G, int H, int W, int C, float* dx, void* stream) {
  MAS_REQUIRE(x && bn && dx && G > 0 && H >= 3 && W >= 3 && C > 0 && (H - 3) % 2 == 0 && (W - 3) % 2 == 0 && (!dp || arg) &&
                  (!sgn || (P > 0 && f0 >= 0 && f0 + G <= 2 * P)),
              "face_pool_backward: bad arguments");
  const int Ho = (H - 3) / 2 + 1, Wo = (W - 3) / 2 + 1;
  pool_bwd_kernel<<<grid_of((int64_t)G * H * W * C, 256), 256, 0, S(stream)>>>(x, bn, arg, dp, sgn, coef, f0, P, G, H, W, C, Ho,
                                                                              Wo, dx);
  return launched("face_pool_bwd");
}

int mas_face_l1_blocks(void) { return L1_BLOCKS; }

int mas_face_l1_forward(const float* f, int64_t n, int8_t* sgn, double* part, void* stream) {
  MAS_REQUIRE(f && part && n > 0, "face_l1_forward: bad arguments");
  l1_fwd_kernel<<<L1_BLOCKS, 256, 0, S(stream)>>>(f, n, sgn, part);
  return launched("face_l1_fwd");
}

int mas_face_l1_finalize(const double* part, double c0, double c1, double c2, double c3, double c4, float* terms, float* loss,
                         void* stream) {
  MAS_REQUIRE(part && terms && loss, "face_l1_finalize: bad arguments");
  Coef5 c{{c0, c1, c2, c3, c4}};
  l1_finalize_kernel<<<1, 32, 0, S(stream)>>>(part, c, terms, loss);
  return launched("face_l1_finalize");
}

int mas_face_subsample_half(const float* x, void* y16, int N, int H, int W, int C, const float* amax, void* stream) {
  MAS_REQUIRE(x && y16 && N > 0 && H > 0 && W > 0 && C % 4 == 0 && al16(x) && (reinterpret_cast<uintptr_t>(y16) & 7) == 0,
              "face_subsample_half: bad arguments");
  const int64_t total = (int64_t)N * ((H + 1) / 2) * ((W + 1) / 2) * (C / 4);
  subsample_half_kernel<<<grid_of(total, 256), 256, 0, S(stream)>>>(reinterpret_cast<const float4*>(x), reinterpret_cast<uint2*>(y16),
                                                                    N, H, W, C / 4, amax);
  return launched("face_subsample_half");
}

int mas_face_relu_seed_backward(const float* out, const float* dout, int half, const int8_t* sgn, float coef, int f0, int P, int G,
                                int H, int W, int C, float* dz, float* amax, void* stream) {
  MAS_REQUIRE(out && dz && G > 0 && H > 0 && W > 0 && C > 0 && (!sgn || (P > 0 && f0 >= 0 && f0 + G <= 2 * P)),
              "face_relu_seed_backward: bad arguments");
  if (int e = zero_amax(amax, S(stream))) return e;
  relu_seed_bwd_kernel<<<grid_of((int64_t)G * H * W * C, 256), 256, 0, S(stream)>>>(out, dout, half, sgn, coef, f0, P, G, H, W, C,
                                                                                   dz, amax);
  return launched("face_relu_seed_bwd");
}

}  // extern "C"
