// GroupNorm(+SiLU), Swish, softmax, BatchNorm statistics, column sums, strided copy, 2x2 sum-pool,
// weighted BCE — the HBM-bound kernels of the VQ-IMG path.  All fp32 I/O, NHWC rows.
// Reference call sites: modules.py:35-41 (Normalize/nonlinearity), :180-181 (softmax), vqvae.py:16 (BN).
#include <stdarg.h>

#include <cuda_fp16.h>
#include <stdlib.h>

#include "mas_common.cuh"
#include "tc_ptx.cuh"

namespace mas {

thread_local char g_err[512] = {0};
std::atomic<int64_t> g_launches{0};
std::atomic<int64_t> g_tc_launches{0};

int fail(int code, const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
  return code;
}

int launched(const char* what) {
  g_launches.fetch_add(1, std::memory_order_relaxed);
  cudaError_t e = cudaGetLastError();
  if (e != cudaSuccess) return fail(MAS_ERR_LAUNCH, "%s: %s", what, cudaGetErrorString(e));
  return MAS_OK;
}

int launched_tc(const char* what) {
  g_tc_launches.fetch_add(1, std::memory_order_relaxed);
  return launched(what);
}

// ------------------------------------------------------------------------------------------------
// GroupNorm.  x [N, HW, C]; a block owns GN_PIX consecutive pixels of one image; thread t owns the
// channel quad (t % U), U = C/4, and walks pixels t/U, t/U + 256/U, ...  Sums are kept in fp64
// (cheap in an HBM-bound kernel) so that var = E[x^2]-E[x]^2 has no fp32 cancellation problem.
// ------------------------------------------------------------------------------------------------
constexpr int GN_THREADS = 256;
constexpr int GN_PIX = 1024;  // pixels per block for large images; small ones get smaller chunks (gn_chunks) so the grid fills the GPU

__global__ void __launch_bounds__(GN_THREADS) gn_stats_partial(const float* __restrict__ x, int HW, int C, int G,
                                                               double* __restrict__ part /*[N][chunks][G][2]*/) {
  extern __shared__ double sm[];  // [C][2] then reused
  const int U = C >> 2, n = blockIdx.y, chunk = blockIdx.x, nchunks = gridDim.x;
  const int t = threadIdx.x, u = t % U, lanes = GN_THREADS / U, pl = t / U;
  const int PIX = (HW + gridDim.x - 1) / gridDim.x;
  const int p0 = chunk * PIX, p1 = min(HW, p0 + PIX);
  double s[4] = {0, 0, 0, 0}, q[4] = {0, 0, 0, 0};
  const float4* xp = reinterpret_cast<const float4*>(x + (size_t)n * HW * C) + u;
  // four independent 16-byte loads in flight per thread; per-quad fp32 partial sums over 4 pixels feed the fp64 totals
  int p = p0 + pl;
  for (; p + 3 * lanes < p1; p += 4 * lanes) {
    float4 v[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) v[k] = __ldg(xp + (size_t)(p + k * lanes) * U);
    float fs[4] = {0.f, 0.f, 0.f, 0.f}, fq[4] = {0.f, 0.f, 0.f, 0.f};  // fp32 over 4 pixels, fp64 across batches
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      fs[0] += v[k].x; fq[0] = fmaf(v[k].x, v[k].x, fq[0]);
      fs[1] += v[k].y; fq[1] = fmaf(v[k].y, v[k].y, fq[1]);
      fs[2] += v[k].z; fq[2] = fmaf(v[k].z, v[k].z, fq[2]);
      fs[3] += v[k].w; fq[3] = fmaf(v[k].w, v[k].w, fq[3]);
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) { s[k] += fs[k]; q[k] += fq[k]; }
  }
  for (; p < p1; p += lanes) {
    float4 v = __ldg(xp + (size_t)p * U);
    s[0] += v.x; q[0] += (double)v.x * v.x;
    s[1] += v.y; q[1] += (double)v.y * v.y;
    s[2] += v.z; q[2] += (double)v.z * v.z;
    s[3] += v.w; q[3] += (double)v.w * v.w;
  }
  // deterministic block reduction: [lanes][C][2] in shared memory, then fixed-order sums
  double* buf = sm;  // lanes*C*2 doubles
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    buf[((size_t)pl * C + u * 4 + i) * 2 + 0] = s[i];
    buf[((size_t)pl * C + u * 4 + i) * 2 + 1] = q[i];
  }
  __syncthreads();
  const int cpg = C / G;
  if (t < G) {
    double a = 0, b = 0;
    for (int c = t * cpg; c < (t + 1) * cpg; ++c)
      for (int l = 0; l < lanes; ++l) {
        a += buf[((size_t)l * C + c) * 2 + 0];
        b += buf[((size_t)l * C + c) * 2 + 1];
      }
    double* o = part + (((size_t)n * nchunks + chunk) * G + t) * 2;
    o[0] = a;
    o[1] = b;
  }
}

__global__ void gn_stats_final(const double* __restrict__ part, int nchunks, int G, double count, float eps,
                               float* __restrict__ mean, float* __restrict__ rstd, int NG) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= NG) return;
  int n = i / G, g = i % G;
  double a = 0, b = 0;
  for (int c = 0; c < nchunks; ++c) {
    const double* o = part + (((size_t)n * nchunks + c) * G + g) * 2;
    a += o[0];
    b += o[1];
  }
  double m = a / count, var = b / count - m * m;
  if (var < 0) var = 0;
  mean[i] = (float)m;
  rstd[i] = (float)(1.0 / sqrt(var + (double)eps));
}

// apply: same block/thread mapping as the statistics kernel (block = GN_PIX pixels of one image, thread = one channel
// quad), so the per-channel scale/shift are loop invariants and four independent 16-byte loads are in flight per thread.
__global__ void __launch_bounds__(GN_THREADS) gn_apply_kernel(const float* __restrict__ x, const float* __restrict__ mean,
                                                              const float* __restrict__ rstd, const float* __restrict__ gamma,
                                                              const float* __restrict__ beta, float* __restrict__ y, int HW, int C,
                                                              int G, int silu, int rtf32) {
  const int U = C >> 2, n = blockIdx.y, cpg = C / G;
  const int t = threadIdx.x, u = t % U, lanes = GN_THREADS / U, pl = t / U;
  const int PIX = (HW + gridDim.x - 1) / gridDim.x;
  const int p0 = blockIdx.x * PIX, p1 = min(HW, p0 + PIX);
  float sc[4], sh[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int c = u * 4 + k, g = c / cpg;
    const float a = rstd[n * G + g] * gamma[c];
    sc[k] = a;
    sh[k] = beta[c] - mean[n * G + g] * a;
  }
  const float4* xp = reinterpret_cast<const float4*>(x + (size_t)n * HW * C) + u;
  float4* yp = reinterpret_cast<float4*>(y + (size_t)n * HW * C) + u;
  auto f = [&](float v, int k) {
    float o = fmaf(v, sc[k], sh[k]);
    if (silu) o = silu_f(o);
    if (rtf32) o = round_tf32(o);
    return o;
  };
  int p = p0 + pl;
  if (rtf32 == 2) {
    // fp16 output: the channels-last "shadow" the TMA-fed convolution kernel reads (conv_tma.cu); 8 bytes per channel quad
    uint2* hp = reinterpret_cast<uint2*>(reinterpret_cast<__half*>(y) + (size_t)n * HW * C) + u;
    rtf32 = 0;
    auto h4 = [&](const float4& v) {
      uint2 h;
      const float a0 = f(v.x, 0), a1 = f(v.y, 1), a2 = f(v.z, 2), a3 = f(v.w, 3);
      asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(h.x) : "f"(a1), "f"(a0));
      asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(h.y) : "f"(a3), "f"(a2));
      return h;
    };
    for (; p + 3 * lanes < p1; p += 4 * lanes) {
      float4 v[4];
#pragma unroll
      for (int k = 0; k < 4; ++k) v[k] = __ldg(xp + (size_t)(p + k * lanes) * U);
#pragma unroll
      for (int k = 0; k < 4; ++k) hp[(size_t)(p + k * lanes) * U] = h4(v[k]);
    }
    for (; p < p1; p += lanes) hp[(size_t)p * U] = h4(__ldg(xp + (size_t)p * U));
    return;
  }
  for (; p + 3 * lanes < p1; p += 4 * lanes) {
    float4 v[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) v[k] = __ldg(xp + (size_t)(p + k * lanes) * U);
#pragma unroll
    for (int k = 0; k < 4; ++k) yp[(size_t)(p + k * lanes) * U] = make_float4(f(v[k].x, 0), f(v[k].y, 1), f(v[k].z, 2), f(v[k].w, 3));
  }
  for (; p < p1; p += lanes) {
    float4 v = __ldg(xp + (size_t)p * U);
    yp[(size_t)p * U] = make_float4(f(v.x, 0), f(v.y, 1), f(v.z, 2), f(v.w, 3));
  }
}

// backward pass 1: per (n, chunk, channel): s1 = sum dyu*xhat, s2 = sum dyu, with dyu = dy*silu'(u)
__global__ void __launch_bounds__(GN_THREADS) gn_bwd_partial(const float* __restrict__ dy, const float* __restrict__ x,
                                                             const float* __restrict__ mean, const float* __restrict__ rstd,
                                                             const float* __restrict__ gamma, const float* __restrict__ beta,
                                                             int HW, int C, int G, int silu,
                                                             double* __restrict__ part /*[N][chunks][C][2]*/,
                                                             float* __restrict__ act_out /*or null: also write act(GN(x))*/,
                                                             int act_f16 /*act_out holds fp16 (the fp16-operand weight gradient's input)*/,
                                                             unsigned int* __restrict__ mx /*or null: [0] max|dy*silu'*gamma|, [1] max|xhat| (float bits)*/) {
  extern __shared__ double sm[];
  const int U = C >> 2, n = blockIdx.y, chunk = blockIdx.x, nchunks = gridDim.x, cpg = C / G;
  const int t = threadIdx.x, u = t % U, lanes = GN_THREADS / U, pl = t / U;
  const int PIX = (HW + gridDim.x - 1) / gridDim.x;
  const int p0 = chunk * PIX, p1 = min(HW, p0 + PIX);
  float m[4], r[4], ga[4], be[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    int c = u * 4 + k, g = c / cpg;
    m[k] = mean[n * G + g];
    r[k] = rstd[n * G + g];
    ga[k] = gamma[c];
    be[k] = beta[c];
  }
  double s1[4] = {0, 0, 0, 0}, s2[4] = {0, 0, 0, 0};
  const float4* xp = reinterpret_cast<const float4*>(x + (size_t)n * HW * C) + u;
  const float4* dp = reinterpret_cast<const float4*>(dy + (size_t)n * HW * C) + u;
  float f1[4], f2[4];
  float4* ap = (act_out && !act_f16) ? reinterpret_cast<float4*>(act_out + (size_t)n * HW * C) + u : nullptr;
  uint2* ap16 = (act_out && act_f16) ? reinterpret_cast<uint2*>(reinterpret_cast<__half*>(act_out) + (size_t)n * HW * C) + u : nullptr;
  // the activation act(GN(x)) (needed by the weight-gradient kernel, never stored in the forward) is re-materialised here
  // as a by-product: x is being read anyway, so this replaces a separate read+write pass by one extra write
  float tmd = 0.f, tmx = 0.f;   // running max|d*gamma| and max|xhat|: the inputs of the rigorous bound on |dx| (gn_bwd_final)
  auto accum = [&](const float4& xv, const float4& dv, size_t idx) {
    float xi[4] = {xv.x, xv.y, xv.z, xv.w}, di[4] = {dv.x, dv.y, dv.z, dv.w}, ao[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      float xh = (xi[k] - m[k]) * r[k];
      float d = di[k];
      const float uu = xh * ga[k] + be[k];
      if (silu) d *= silu_grad_f(uu);
      ao[k] = silu ? silu_f(uu) : uu;
      f1[k] = fmaf(d, xh, f1[k]);
      f2[k] += d;
      tmd = fmaxf(tmd, fabsf(d * ga[k]));
      tmx = fmaxf(tmx, fabsf(xh));
    }
    if (ap) ap[idx] = make_float4(ao[0], ao[1], ao[2], ao[3]);
    if (ap16) {   // round-to-nearest, saturating: the conversion the weight-gradient producers would apply anyway
      uint2 h;
      asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(h.x) : "f"(ao[1]), "f"(ao[0]));
      asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(h.y) : "f"(ao[3]), "f"(ao[2]));
      ap16[idx] = h;
    }
  };
  auto flush = [&]() {
#pragma unroll
    for (int k = 0; k < 4; ++k) { s1[k] += f1[k]; s2[k] += f2[k]; f1[k] = 0.f; f2[k] = 0.f; }
  };
#pragma unroll
  for (int k = 0; k < 4; ++k) { f1[k] = 0.f; f2[k] = 0.f; }
  int p = p0 + pl;
  for (; p + 3 * lanes < p1; p += 4 * lanes) {
    float4 xv[4], dv[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      xv[k] = __ldg(xp + (size_t)(p + k * lanes) * U);
      dv[k] = __ldg(dp + (size_t)(p + k * lanes) * U);
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) accum(xv[k], dv[k], (size_t)(p + k * lanes) * U);
    flush();  // fp32 over 4 pixels, fp64 across batches
  }
  for (; p < p1; p += lanes) accum(__ldg(xp + (size_t)p * U), __ldg(dp + (size_t)p * U), (size_t)p * U);
  flush();
  double* buf = sm;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    buf[((size_t)pl * C + u * 4 + k) * 2 + 0] = s1[k];
    buf[((size_t)pl * C + u * 4 + k) * 2 + 1] = s2[k];
  }
  __syncthreads();
  for (int c = t; c < C; c += GN_THREADS) {
    double a = 0, b = 0;
    for (int l = 0; l < lanes; ++l) {
      a += buf[((size_t)l * C + c) * 2 + 0];
      b += buf[((size_t)l * C + c) * 2 + 1];
    }
    double* o = part + (((size_t)n * nchunks + chunk) * C + c) * 2;
    o[0] = a;
    o[1] = b;
  }
  if (mx) {
    tmd = warp_max(tmd);
    tmx = warp_max(tmx);
    if ((t & 31) == 0) {   // non-negative floats order like their bit patterns; order-independent: deterministic
      atomicMax(mx, __float_as_uint(tmd));
      atomicMax(mx + 1, __float_as_uint(tmx));
    }
  }
}

// backward finalize, stage 1: per (n,c) sums over chunks
__global__ void gn_bwd_nc(const double* __restrict__ part, int N, int nchunks, int C, double* __restrict__ nc /*[N][C][2]*/) {
  int i = threadIdx.x + blockIdx.x * blockDim.x;
  if (i >= N * C) return;
  int n = i / C, c = i % C;
  double a = 0, b = 0;
  const double2* o = reinterpret_cast<const double2*>(part) + (size_t)n * nchunks * C + c;
  int k = 0;
  for (; k + 7 < nchunks; k += 8) {   // eight chunks in flight (fixed order of additions)
    double2 v[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) v[j] = o[(size_t)(k + j) * C];
#pragma unroll
    for (int j = 0; j < 8; ++j) { a += v[j].x; b += v[j].y; }
  }
  for (; k < nchunks; ++k) { const double2 v = o[(size_t)k * C]; a += v.x; b += v.y; }
  nc[(size_t)i * 2 + 0] = a;
  nc[(size_t)i * 2 + 1] = b;
}
// stage 2: dgamma/dbeta (blocks [0, cblocks): one thread per channel, sum over images) and the per-(n,g) coefficients
// A,B of the apply pass (remaining blocks: one thread per (image, group)).  Both read only nc, so they share a launch.
__global__ void __launch_bounds__(128) gn_bwd_final(int N, int C, int G, const float* __restrict__ gamma, const double* __restrict__ nc,
                                                    float* __restrict__ dgamma, float* __restrict__ dbeta,
                                                    float* __restrict__ AB /*[N][G][2]*/, double inv_m, int cblocks,
                                                    const float* __restrict__ rstd, unsigned int* __restrict__ mx /*or null*/) {
  const int cpg = C / G;
  if ((int)blockIdx.x < cblocks) {
    const int c = blockIdx.x * 128 + threadIdx.x;
    if (c >= C) return;
    double a = 0, b = 0;
    const double2* p = reinterpret_cast<const double2*>(nc) + c;
    int n = 0;
    for (; n + 7 < N; n += 8) {   // eight images in flight (fixed order of additions)
      double2 v[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) v[k] = p[(size_t)(n + k) * C];
#pragma unroll
      for (int k = 0; k < 8; ++k) { a += v[k].x; b += v[k].y; }
    }
    for (; n < N; ++n) { const double2 v = p[(size_t)n * C]; a += v.x; b += v.y; }
    dgamma[c] = (float)a;
    dbeta[c] = (float)b;
  } else {
    const int i = (blockIdx.x - cblocks) * 128 + threadIdx.x;
    if (i >= N * G) return;
    const int n = i / G, g = i % G;
    double a = 0, b = 0;
    for (int c = g * cpg; c < (g + 1) * cpg; ++c) {
      a += (double)gamma[c] * nc[((size_t)n * C + c) * 2 + 0];
      b += (double)gamma[c] * nc[((size_t)n * C + c) * 2 + 1];
    }
    AB[i * 2 + 0] = (float)(a * inv_m);
    AB[i * 2 + 1] = (float)(b * inv_m);
    if (mx) {
      // dx = rstd*(d*gamma - B - xhat*A) (+ dx_add): |dx - dx_add| <= rstd*(max|d*gamma| + |B| + max|xhat|*|A|) for every
      // element of this (image, group); the maximum over (image, group) lands in mx[2]
      const float bnd = rstd[i] * (__uint_as_float(mx[0]) + fabsf((float)(b * inv_m)) + __uint_as_float(mx[1]) * fabsf((float)(a * inv_m)));
      atomicMax(mx + 2, __float_as_uint(bnd));
    }
  }
}

__global__ void __launch_bounds__(GN_THREADS) gn_bwd_apply(const float* __restrict__ dy, const float* __restrict__ x,
                                                           const float* __restrict__ mean, const float* __restrict__ rstd,
                                                           const float* __restrict__ gamma, const float* __restrict__ beta,
                                                           const float* __restrict__ AB, const float* __restrict__ dx_add,
                                                           float* __restrict__ dx, int HW, int C, int G, int silu,
                                                           unsigned int* __restrict__ dx_amax /*or null: max|dx| (float bits)*/,
                                                           __half* __restrict__ dx16 /*or null: fp16 shadow of dx, scaled*/,
                                                           const unsigned int* __restrict__ mx, const float* __restrict__ add_amax,
                                                           float* __restrict__ dx_bound /*the magnitude the shadow's scale derives from*/) {
  const int U = C >> 2, n = blockIdx.y, cpg = C / G;
  // shadow scale: a power of two from a rigorous bound on max|dx| (known BEFORE this pass, unlike max|dx| itself); every
  // block derives the same value, block (0, 0) publishes it for the convolution that reads the shadow
  __shared__ float sh_bound;
  float sscale = 1.f;
  if (dx16) {
    if (threadIdx.x == 0) {
      const float bnd = __uint_as_float(mx[2]) * 1.01f + (add_amax ? *add_amax : 0.f);
      sh_bound = bnd;
      if (blockIdx.x == 0 && blockIdx.y == 0) *dx_bound = bnd;
    }
    __syncthreads();
    float inv_unused;
    sscale = tc::operand_scale(&sh_bound, &inv_unused);
  }
  const int t = threadIdx.x, u = t % U, lanes = GN_THREADS / U, pl = t / U;
  const int PIX = (HW + gridDim.x - 1) / gridDim.x;
  const int p0 = blockIdx.x * PIX, p1 = min(HW, p0 + PIX);
  float m[4], r[4], ga[4], be[4], A[4], B[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int c = u * 4 + k, g = c / cpg;
    m[k] = mean[n * G + g]; r[k] = rstd[n * G + g]; ga[k] = gamma[c]; be[k] = beta[c];
    A[k] = AB[(n * G + g) * 2]; B[k] = AB[(n * G + g) * 2 + 1];
  }
  const size_t base = (size_t)n * HW * C;
  const float4* xp = reinterpret_cast<const float4*>(x + base) + u;
  const float4* dp = reinterpret_cast<const float4*>(dy + base) + u;
  const float4* ap = dx_add ? reinterpret_cast<const float4*>(dx_add + base) + u : nullptr;
  float4* op = dx ? reinterpret_cast<float4*>(dx + base) + u : nullptr;   // null: only the fp16 shadow is wanted
  uint2* hp = dx16 ? reinterpret_cast<uint2*>(dx16 + base) + u : nullptr;
  auto h4 = [&](const float4& v) {
    uint2 h;
    asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(h.x) : "f"(v.y * sscale), "f"(v.x * sscale));
    asm("cvt.rn.satfinite.f16x2.f32 %0, %1, %2;" : "=r"(h.y) : "f"(v.w * sscale), "f"(v.z * sscale));
    return h;
  };
  float amx = 0.f;   // the consumers of dx are fp16-operand tensor-core kernels: their operand scale comes from max|dx|
  auto one = [&](const float4& xv, const float4& dv, const float4& av) {
    float xi[4] = {xv.x, xv.y, xv.z, xv.w}, di[4] = {dv.x, dv.y, dv.z, dv.w}, ad[4] = {av.x, av.y, av.z, av.w}, o[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      float xh = (xi[k] - m[k]) * r[k];
      float d = di[k];
      if (silu) d *= silu_grad_f(xh * ga[k] + be[k]);
      o[k] = r[k] * (d * ga[k] - B[k] - xh * A[k]) + ad[k];
    }
    if (dx_amax) amx = fmaxf(amx, fmaxf(fmaxf(fabsf(o[0]), fabsf(o[1])), fmaxf(fabsf(o[2]), fabsf(o[3]))));
    return make_float4(o[0], o[1], o[2], o[3]);
  };
  const float4 z4 = make_float4(0.f, 0.f, 0.f, 0.f);
  int p = p0 + pl;
  for (; p + lanes < p1; p += 2 * lanes) {
    const size_t i0 = (size_t)p * U, i1 = (size_t)(p + lanes) * U;
    float4 x0 = __ldg(xp + i0), x1 = __ldg(xp + i1), d0 = __ldg(dp + i0), d1 = __ldg(dp + i1);
    float4 a0 = ap ? __ldg(ap + i0) : z4, a1 = ap ? __ldg(ap + i1) : z4;
    const float4 o0 = one(x0, d0, a0), o1 = one(x1, d1, a1);
    if (op) { op[i0] = o0; op[i1] = o1; }
    if (hp) { hp[i0] = h4(o0); hp[i1] = h4(o1); }
  }
  for (; p < p1; p += lanes) {
    const size_t i0 = (size_t)p * U;
    const float4 o0 = one(__ldg(xp + i0), __ldg(dp + i0), ap ? __ldg(ap + i0) : z4);
    if (op) op[i0] = o0;
    if (hp) hp[i0] = h4(o0);
  }
  if (dx_amax) {
    amx = warp_max(amx);
    if ((t & 31) == 0 && amx > 0.f) atomicMax(dx_amax, __float_as_uint(amx));   // order-independent: deterministic
  }
}

// statistics emitted by the convolution epilogues: part[tile][4][C/4][2] -> mean/rstd per (image, group); warp per (n,g)
__global__ void gn_finalize_partials_kernel(const float* __restrict__ part, int tiles_per_image, int C, int G, double count, float eps,
                                            float* __restrict__ mean, float* __restrict__ rstd, int NG) {
  const int wid = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (wid >= NG) return;
  const int n = wid / G, g = wid % G, Q = C >> 2, qpg = Q / G;  // channel quads per group (C/G >= 4)
  double a = 0, b = 0;
  const int rows = tiles_per_image * 4;
  const float2* pb = reinterpret_cast<const float2*>(part) + (size_t)n * rows * Q + (size_t)g * qpg;
  int r = lane;
  for (; r + 7 * 32 < rows; r += 8 * 32) {  // eight rows in flight per lane: the loop is latency-bound (L2 hits, 8 of 256 bytes per row)
    for (int q = 0; q < qpg; ++q) {
      float2 v[8];
#pragma unroll
      for (int k = 0; k < 8; ++k) v[k] = __ldg(pb + (size_t)(r + k * 32) * Q + q);
#pragma unroll
      for (int k = 0; k < 8; ++k) { a += v[k].x; b += v[k].y; }
    }
  }
  for (; r < rows; r += 32)
    for (int q = 0; q < qpg; ++q) {
      const float2 v = __ldg(pb + (size_t)r * Q + q);
      a += v.x; b += v.y;
    }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    a += __shfl_xor_sync(0xffffffffu, a, o);
    b += __shfl_xor_sync(0xffffffffu, b, o);
  }
  if (lane == 0) {
    double m = a / count, var = b / count - m * m;
    if (var < 0) var = 0;
    mean[wid] = (float)m;
    rstd[wid] = (float)(1.0 / sqrt(var + (double)eps));
  }
}
// (sc, sh) per (image, channel): act(GroupNorm(x)) = act(x*sc + sh)
__global__ void gn_table_kernel(const float* __restrict__ mean, const float* __restrict__ rstd, const float* __restrict__ gamma,
                                const float* __restrict__ beta, int N, int C, int G, float* __restrict__ table) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= N * C) return;
  int n = i / C, c = i % C, g = c / (C / G);
  float a = rstd[n * G + g] * gamma[c];
  table[(size_t)i * 2] = a;
  table[(size_t)i * 2 + 1] = beta[c] - mean[n * G + g] * a;
}

__global__ void add_kernel(const float* __restrict__ a, const float* __restrict__ b, float* __restrict__ o, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) o[i] = a[i] + b[i];
}
__global__ void silu_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    y[i] = silu_f(x[i]);
}
__global__ void silu_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ x, float* __restrict__ dx, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    dx[i] = dy[i] * silu_grad_f(x[i]);
}

// ------------------------------------------------------------------------------------------------ softmax (warp per row)
__global__ void softmax_fwd_kernel(const float* __restrict__ s, float* __restrict__ p, int64_t rows, int cols) {
  int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  int lane = threadIdx.x & 31;
  const float* sr = s + row * cols;
  float* pr = p + row * cols;
  float mx = -INFINITY;
  for (int c = lane; c < cols; c += 32) mx = fmaxf(mx, sr[c]);
  mx = warp_max(mx);
  float sum = 0.f;
  for (int c = lane; c < cols; c += 32) sum += expf(sr[c] - mx);
  sum = warp_sum(sum);
  float inv = 1.0f / sum;
  for (int c = lane; c < cols; c += 32) pr[c] = expf(sr[c] - mx) * inv;
}
__global__ void softmax_bwd_kernel(const float* __restrict__ p, const float* __restrict__ dp, float* __restrict__ ds,
                                   int64_t rows, int cols, float scale) {
  int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  int lane = threadIdx.x & 31;
  const float* pr = p + row * cols;
  const float* dr = dp + row * cols;
  float dot = 0.f;
  for (int c = lane; c < cols; c += 32) dot += pr[c] * dr[c];
  dot = warp_sum(dot);
  for (int c = lane; c < cols; c += 32) ds[row * cols + c] = pr[c] * (dr[c] - dot) * scale;
}

// ------------------------------------------------------------------------------------------------ BatchNorm pieces
// one block per 32-channel tile; blockDim (32, 8); deterministic; R*C is small (8192 x 256) on this path
__global__ void bn_stats_kernel(const float* __restrict__ x, int64_t R, int C, double* __restrict__ out /*[2C]*/) {
  __shared__ double sh[8][32][2];
  int c = blockIdx.x * 32 + threadIdx.x;
  double a = 0, b = 0;
  if (c < C)
    for (int64_t r = threadIdx.y; r < R; r += 8) {
      float v = x[r * C + c];
      a += v;
      b += (double)v * v;
    }
  sh[threadIdx.y][threadIdx.x][0] = a;
  sh[threadIdx.y][threadIdx.x][1] = b;
  __syncthreads();
  if (threadIdx.y == 0 && c < C) {
    for (int k = 1; k < 8; ++k) {
      a += sh[k][threadIdx.x][0];
      b += sh[k][threadIdx.x][1];
    }
    out[c] = a;
    out[C + c] = b;
    if (c == 0) out[2 * C] = (double)R;   // local element count per channel: reduced across ranks with the sums
  }
}
__global__ void bn_finalize_kernel(const double* __restrict__ stats, double count, int C, float eps, float momentum,
                                   float* __restrict__ mean, float* __restrict__ invstd, float* __restrict__ run_mean,
                                   float* __restrict__ run_var) {
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  if (count <= 0) count = stats[2 * C];   // the (all-reduced) element count travels with the sums
  double m = stats[c] / count, var = stats[C + c] / count - m * m;
  if (var < 0) var = 0;
  mean[c] = (float)m;
  invstd[c] = (float)(1.0 / sqrt(var + (double)eps));
  if (run_mean) {
    double unb = count > 1 ? var * count / (count - 1) : var;
    run_mean[c] = (float)((1.0 - momentum) * run_mean[c] + momentum * m);
    run_var[c] = (float)((1.0 - momentum) * run_var[c] + momentum * unb);
  }
}
// largest |x| of a tensor (bit pattern of a non-negative float orders like the unsigned integer): the power-of-two operand
// scale of the fp16 tensor-core kernels is derived from it on the device. NaNs are ignored, +-inf saturates the result.
__global__ void __launch_bounds__(256) amax_kernel(const float4* __restrict__ x, int64_t n4, const float* __restrict__ tail, int ntail,
                                                   unsigned int* __restrict__ out) {
  float m = 0.f;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n4; i += (int64_t)gridDim.x * blockDim.x) {
    const float4 v = __ldg(x + i);
    m = fmaxf(m, fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w))));
  }
  if (blockIdx.x == 0 && (int)threadIdx.x < ntail) m = fmaxf(m, fabsf(tail[threadIdx.x]));
  m = warp_max(m);
  __shared__ float sh[8];
  if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int k = 1; k < 8; ++k) m = fmaxf(m, sh[k]);
    atomicMax(out, __float_as_uint(m));
  }
}
__global__ void bn_invstd_kernel(const float* __restrict__ var, float eps, float* __restrict__ out, int C) {
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < C) out[c] = (float)(1.0 / sqrt((double)var[c] + (double)eps));
}
__global__ void bn_apply_kernel(const float* __restrict__ x, const float* __restrict__ mean, const float* __restrict__ invstd,
                                const float* __restrict__ gamma, const float* __restrict__ beta, float* __restrict__ y,
                                int64_t total, int C, float slope) {
  // slope: LeakyReLU on the output (1 = none: v * 1 is exact)
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int c = (int)(i % C);
    float v = (x[i] - mean[c]) * invstd[c] * gamma[c] + beta[c];
    y[i] = v > 0.f ? v : v * slope;
  }
}
__global__ void bn_bwd_reduce_kernel(const float* __restrict__ dy, const float* __restrict__ x, const float* __restrict__ mean,
                                     const float* __restrict__ invstd, int64_t R, int C, double* __restrict__ out /*[2C]*/) {
  __shared__ double sh[8][32][2];
  int c = blockIdx.x * 32 + threadIdx.x;
  double a = 0, b = 0;
  if (c < C) {
    float m = mean[c], is = invstd[c];
    for (int64_t r = threadIdx.y; r < R; r += 8) {
      float d = dy[r * C + c];
      a += d;
      b += (double)d * ((x[r * C + c] - m) * is);
    }
  }
  sh[threadIdx.y][threadIdx.x][0] = a;
  sh[threadIdx.y][threadIdx.x][1] = b;
  __syncthreads();
  if (threadIdx.y == 0 && c < C) {
    for (int k = 1; k < 8; ++k) {
      a += sh[k][threadIdx.x][0];
      b += sh[k][threadIdx.x][1];
    }
    out[c] = a;
    out[C + c] = b;
    if (c == 0) out[2 * C] = (double)R;
  }
}
// BatchNorm+LeakyReLU backward sums over row chunks of BN_RB rows (grid: C/32 x chunks), then an ordered sum of the chunks:
// deterministic, and enough blocks to fill the GPU at the discriminator's R = N*H*W of 10^4..10^5 rows
constexpr int BN_RB = 1024;
__global__ void bn_bwd_reduce_lrelu_part(const float* __restrict__ dy, const float* __restrict__ act_y, float slope,
                                         const float* __restrict__ x, const float* __restrict__ mean, const float* __restrict__ invstd,
                                         int64_t R, int C, double* __restrict__ part /*[chunks][2C]*/) {
  __shared__ double sh[8][32][2];
  const int c = blockIdx.x * 32 + threadIdx.x;
  const int64_t r0 = (int64_t)blockIdx.y * BN_RB, r1 = min(R, r0 + BN_RB);
  double a = 0, b = 0;
  if (c < C) {
    const float m = mean[c], is = invstd[c];
    for (int64_t r = r0 + threadIdx.y; r < r1; r += 8) {
      float d = dy[r * C + c];
      if (!(act_y[r * C + c] > 0.f)) d *= slope;
      a += d;
      b += (double)d * ((x[r * C + c] - m) * is);
    }
  }
  sh[threadIdx.y][threadIdx.x][0] = a;
  sh[threadIdx.y][threadIdx.x][1] = b;
  __syncthreads();
  if (threadIdx.y == 0 && c < C) {
    for (int k = 1; k < 8; ++k) {
      a += sh[k][threadIdx.x][0];
      b += sh[k][threadIdx.x][1];
    }
    part[(int64_t)blockIdx.y * 2 * C + c] = a;
    part[(int64_t)blockIdx.y * 2 * C + C + c] = b;
  }
}
__global__ void bn_bwd_reduce_lrelu_final(const double* __restrict__ part, int chunks, int64_t R, int C, double* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < 2 * C) {
    double s = 0;
    for (int k = 0; k < chunks; ++k) s += part[(int64_t)k * 2 * C + i];
    out[i] = s;
  }
  if (i == 0) out[2 * C] = (double)R;
}
__global__ void bn_bwd_apply_kernel(const float* __restrict__ dy, const float* __restrict__ x, const float* __restrict__ mean,
                                    const float* __restrict__ invstd, const float* __restrict__ gamma,
                                    const double* __restrict__ sums /*[2C] global sums*/, double inv_count,
                                    float* __restrict__ dx, float* __restrict__ dgamma, float* __restrict__ dbeta,
                                    const double* __restrict__ local_sums, int64_t total, int C,
                                    const float* __restrict__ act_y, float slope) {
  if (inv_count <= 0) inv_count = 1.0 / sums[2 * C];
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int c = (int)(i % C);
    float xh = (x[i] - mean[c]) * invstd[c];
    float sd = (float)(sums[c] * inv_count), sdx = (float)(sums[C + c] * inv_count);
    float d = dy[i];
    if (act_y && !(act_y[i] > 0.f)) d *= slope;
    dx[i] = gamma[c] * invstd[c] * (d - sd - xh * sdx);
    if (i < C && dgamma) {  // parameter grads are LOCAL sums (DDP all-reduces them like any other grad)
      dbeta[c] = (float)local_sums[c];
      dgamma[c] = (float)local_sums[C + c];
    }
  }
}

// ------------------------------------------------------------------------------------------------ column sums (bias grads)
// out[c] = sum over (n,h,w) of x[n,h,w,c] for a strided view; two-stage deterministic.
constexpr int CS_ROWS = 2048;
__global__ void colsum_partial(const float* __restrict__ x, mas_tensor4 t, double* __restrict__ part /*[chunks][C]*/) {
  __shared__ double sh[8][32];
  int c = blockIdx.x * 32 + threadIdx.x;
  int64_t rows = t.n * t.h * t.w, r0 = (int64_t)blockIdx.y * CS_ROWS, r1 = min(rows, r0 + CS_ROWS);
  double a = 0;
  if (c < t.c)
    for (int64_t r = r0 + threadIdx.y; r < r1; r += 8) {
      int64_t w = r % t.w, h = (r / t.w) % t.h, n = r / (t.w * t.h);
      a += x[n * t.sn + h * t.sh + w * t.sw + c * t.sc];
    }
  sh[threadIdx.y][threadIdx.x] = a;
  __syncthreads();
  if (threadIdx.y == 0 && c < t.c) {
    for (int k = 1; k < 8; ++k) a += sh[k][threadIdx.x];
    part[(size_t)blockIdx.y * t.c + c] = a;
  }
}
__global__ void colsum_final(const double* __restrict__ part, int chunks, int C, float* __restrict__ out) {
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  double a = 0;
  for (int k = 0; k < chunks; ++k) a += part[(size_t)k * C + c];
  out[c] = (float)a;
}

__global__ void copy_strided_kernel(const float* __restrict__ x, mas_tensor4 xs, float* __restrict__ y, mas_tensor4 ys,
                                    int64_t total) {
  // iterate in y's fastest order when y is channel-innermost, else in x's; simple generic version
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t c, w, h, n;
    if (ys.sc == 1) { c = i % xs.c; w = (i / xs.c) % xs.w; h = (i / (xs.c * xs.w)) % xs.h; n = i / (xs.c * xs.w * xs.h); }
    else { w = i % xs.w; h = (i / xs.w) % xs.h; c = (i / (xs.w * xs.h)) % xs.c; n = i / (xs.w * xs.h * xs.c); }
    y[n * ys.sn + h * ys.sh + w * ys.sw + c * ys.sc] = x[n * xs.sn + h * xs.sh + w * xs.sw + c * xs.sc];
  }
}

// NCHW (contiguous) -> channels-last with CP >= C channels (the extra ones zero): block = 32 pixels of one image row, planes read
// as 128-byte rows, transposed through shared memory, written as one contiguous 32 x CP block.  The padded copy is what lets a
// 159-channel input run on the 16-channel K steps of the tensor-core convolution.
__global__ void __launch_bounds__(256) nchw_to_nhwc_pad_kernel(const float* __restrict__ x, float* __restrict__ y, int C, int CP, int H, int W) {
  extern __shared__ float tile[];   // [C][33]
  const int w0 = blockIdx.x * 32, h = blockIdx.y, n = blockIdx.z;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int c = ty; c < C; c += 8) tile[c * 33 + tx] = (w0 + tx < W) ? __ldg(x + (((size_t)n * C + c) * H + h) * W + w0 + tx) : 0.f;
  __syncthreads();
  const size_t base = (((size_t)n * H + h) * W + w0) * CP;
  const int npx = min(32, W - w0);
  for (int i = threadIdx.x; i < npx * CP; i += 256) {
    const int px = i / CP, c = i - px * CP;
    y[base + i] = c < C ? tile[c * 33 + px] : 0.f;
  }
}
__global__ void scale_by_kernel(const float* __restrict__ x, const float* __restrict__ g, float* __restrict__ y, int64_t n) {
  const float s = g[0];
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) y[i] = x[i] * s;
}

__global__ void sumpool2x2_kernel(const float* __restrict__ x, float* __restrict__ y, int H, int W, int C4, int64_t total4) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total4; i += (int64_t)gridDim.x * blockDim.x) {
    int c = (int)(i % C4);
    int64_t p = i / C4;
    int w = (int)(p % W), h = (int)((p / W) % H);
    int64_t n = p / ((int64_t)W * H);
    const float4* b = reinterpret_cast<const float4*>(x) + ((n * 2 * H + 2 * h) * 2 * W + 2 * w) * C4 + c;
    float4 a0 = __ldg(b), a1 = __ldg(b + C4), a2 = __ldg(b + (int64_t)2 * W * C4), a3 = __ldg(b + (int64_t)2 * W * C4 + C4);
    reinterpret_cast<float4*>(y)[i] = make_float4((a0.x + a1.x) + (a2.x + a3.x), (a0.y + a1.y) + (a2.y + a3.y),
                                                  (a0.z + a1.z) + (a2.z + a3.z), (a0.w + a1.w) + (a2.w + a3.w));
  }
}

// weighted BCE-with-logits (loss_seg.py:15-19): l = -[pw*t*log(sig(x)) + (1-t)*log(1-sig(x))]
//   = (1-t)*x + (1+(pw-1)*t) * softplus(-x);  dl/dx = (1-t) - (1+(pw-1)*t)*sigmoid(-x)
constexpr int BCE_CHUNK = 256 * 8;
__global__ void __launch_bounds__(256) bce_kernel(const float* __restrict__ lg, mas_tensor4 ls, const float* __restrict__ tg,
                                                  mas_tensor4 ts, const float* __restrict__ pw, float* __restrict__ grad,
                                                  mas_tensor4 gs, float gscale, double* __restrict__ part, int64_t total) {
  double acc = 0;
  int64_t base = (int64_t)blockIdx.x * BCE_CHUNK;
  for (int k = 0; k < 8; ++k) {
    int64_t i = base + k * 256 + threadIdx.x;
    if (i < total) {
      // i enumerates (n,h,w,c) with w innermost when the logits are NCHW, else c innermost
      int64_t c, w, h, n;
      if (ls.sc == 1) { c = i % ls.c; w = (i / ls.c) % ls.w; h = (i / (ls.c * ls.w)) % ls.h; n = i / (ls.c * ls.w * ls.h); }
      else { w = i % ls.w; h = (i / ls.w) % ls.h; c = (i / (ls.w * ls.h)) % ls.c; n = i / (ls.w * ls.h * ls.c); }
      float x = lg[n * ls.sn + h * ls.sh + w * ls.sw + c * ls.sc];
      float t = tg[n * ts.sn + h * ts.sh + w * ts.sw + c * ts.sc];
      float coef = 1.0f + (pw[c] - 1.0f) * t;
      float sp = fmaxf(-x, 0.f) + log1pf(expf(-fabsf(x)));  // softplus(-x)
      acc += (double)((1.0f - t) * x + coef * sp);
      if (grad) {
        float sg = 1.0f / (1.0f + expf(x));  // sigmoid(-x)
        grad[n * gs.sn + h * gs.sh + w * gs.sw + c * gs.sc] = gscale * ((1.0f - t) - coef * sg);
      }
    }
  }
  __shared__ double red[256];
  red[threadIdx.x] = acc;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) part[blockIdx.x] = red[0];
}
// Same loss for the layouts the VQ-SEG step actually has: logits channels-last with pitch CP >= C (the padded output of
// the decoder's last convolution), target NCHW (the data loader's one-hot maps).  Block = 32 consecutive pixels of one image
// row: the target tile is read plane by plane (128-byte rows) and transposed through shared memory, the logits / gradient
// tile is one contiguous 32 x CP block.  MODE 0: loss partials.  MODE 1: gradient g * gscale * dl/dx (pad channels get 0).
template <int MODE>
__global__ void __launch_bounds__(256) bce_cl_kernel(const float* __restrict__ lg, const float* __restrict__ tg, const float* __restrict__ pw,
                                                     int C, int CP, int H, int W, const float* __restrict__ g, float gscale,
                                                     float* __restrict__ grad, double* __restrict__ part) {
  extern __shared__ float tile[];   // [C][33]
  const int w0 = blockIdx.x * 32, h = blockIdx.y, n = blockIdx.z;
  const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
  for (int c = ty; c < C; c += 8) tile[c * 33 + tx] = __ldg(tg + (((size_t)n * C + c) * H + h) * W + w0 + tx);
  __syncthreads();
  const size_t base = (((size_t)n * H + h) * W + w0) * CP;
  const float gs = MODE == 1 ? gscale * (g ? g[0] : 1.f) : 0.f;
  double acc = 0;
  for (int i = threadIdx.x; i < 32 * CP; i += 256) {
    const int px = i / CP, c = i - px * CP;
    if (c < C) {
      const float x = __ldg(lg + base + i), t = tile[c * 33 + px];
      const float coef = 1.0f + (__ldg(pw + c) - 1.0f) * t;
      if (MODE == 0) {
        const float sp = fmaxf(-x, 0.f) + log1pf(expf(-fabsf(x)));
        acc += (double)((1.0f - t) * x + coef * sp);
      } else {
        const float sg = 1.0f / (1.0f + expf(x));
        grad[base + i] = gs * ((1.0f - t) - coef * sg);
      }
    } else if (MODE == 1) {
      grad[base + i] = 0.f;
    }
  }
  if (MODE == 0) {
    __shared__ double red[256];
    red[threadIdx.x] = acc;
    __syncthreads();
    for (int s = 128; s > 0; s >>= 1) {
      if (threadIdx.x < s) red[threadIdx.x] += red[threadIdx.x + s];
      __syncthreads();
    }
    if (threadIdx.x == 0) part[((size_t)n * H + h) * gridDim.x + blockIdx.x] = red[0];
  }
}
__global__ void sum_final_kernel(const double* __restrict__ part, int n, double scale, float* __restrict__ out) {
  __shared__ double sh[256];
  double a = 0;
  for (int i = threadIdx.x; i < n; i += 256) a += part[i];
  sh[threadIdx.x] = a;
  __syncthreads();
  for (int s = 128; s > 0; s >>= 1) {
    if (threadIdx.x < s) sh[threadIdx.x] += sh[threadIdx.x + s];
    __syncthreads();
  }
  if (threadIdx.x == 0) out[0] = (float)(sh[0] * scale);
}

static inline int ew_grid(int64_t n, int threads = 256) {
  int64_t b = cdiv(n, threads);
  return (int)(b < NUM_SMS * 16 ? (b < 1 ? 1 : b) : NUM_SMS * 16);
}

}  // namespace mas

using namespace mas;

extern "C" {

int mas_version(void) { return 100; }
const char* mas_last_error(void) { return g_err; }
int64_t mas_launch_count(void) { return g_launches.load(); }
int64_t mas_tc_launch_count(void) { return g_tc_launches.load(); }

static int gn_check(int N, int HW, int C, int G) {
  if (N <= 0 || HW <= 0 || C <= 0 || G <= 0 || C % G != 0) return fail(MAS_ERR_INVALID_ARG, "groupnorm: bad shape N=%d HW=%d C=%d G=%d", N, HW, C, G);
  if (C % 4 != 0 || GN_THREADS % (C / 4) != 0) return fail(MAS_ERR_UNSUPPORTED, "groupnorm: C=%d must be 4*{1,2,4,...,256}", C);
  return MAS_OK;
}
// chunks per image: GN_PIX pixels per block, halved until the grid has ~4 blocks per SM (the 16x16 and 32x32 levels would
// otherwise run on 32 blocks) but never below four pixels per thread-lane
static int gn_chunks(int N, int HW, int C) {
  const int lanes = GN_THREADS / (C / 4);
  int pix = GN_PIX;
  while (pix > 4 * lanes && pix > 8 && (int64_t)N * cdiv(HW, pix) < 4 * NUM_SMS) pix >>= 1;
  return (int)cdiv(HW, pix);
}

size_t mas_gn_ws_bytes(int N, int HW, int C, int G) {
  size_t part = (size_t)N * gn_chunks(N, HW, C) * C * 2 * sizeof(double);  // backward partials are the larger use
  size_t nc = (size_t)N * C * 2 * sizeof(double);
  size_t ab = (size_t)N * G * 2 * sizeof(float);
  return part + nc + ab + 256;
}

int mas_gn_stats(const float* x, int N, int HW, int C, int G, float eps, float* mean, float* rstd, void* ws, size_t ws_bytes,
                 void* stream) {
  if (int e = gn_check(N, HW, C, G)) return e;
  int chunks = gn_chunks(N, HW, C);
  size_t need = (size_t)N * chunks * G * 2 * sizeof(double);
  if (ws_bytes < need) return fail(MAS_ERR_WORKSPACE, "gn_stats: workspace %zu < %zu", ws_bytes, need);
  int lanes = GN_THREADS / (C / 4);
  size_t smem = (size_t)lanes * C * 2 * sizeof(double);
  gn_stats_partial<<<dim3(chunks, N), GN_THREADS, smem, S(stream)>>>(x, HW, C, G, (double*)ws);
  if (int e = launched("gn_stats_partial")) return e;
  gn_stats_final<<<(int)cdiv(N * G, 128), 128, 0, S(stream)>>>((const double*)ws, chunks, G, (double)HW * (C / G), eps, mean, rstd, N * G);
  return launched("gn_stats_final");
}

int mas_gn_apply(const float* x, const float* mean, const float* rstd, const float* gamma, const float* beta, float* y, int N,
                 int HW, int C, int G, int silu, int round_tf32, void* stream) {
  if (int e = gn_check(N, HW, C, G)) return e;
  gn_apply_kernel<<<dim3(gn_chunks(N, HW, C), N), GN_THREADS, 0, S(stream)>>>(x, mean, rstd, gamma, beta, y, HW, C, G, silu, round_tf32);
  return launched("gn_apply");
}

int mas_gn_backward(const float* dy, const float* x, const float* mean, const float* rstd, const float* gamma, const float* beta,
                    const float* dx_add, float* dx, float* dgamma, float* dbeta, void* act_out, int act_f16, float* dx_amax,
                    const float* add_amax, void* dx_f16, float* dx_bound, int N, int HW, int C, int G, int silu, void* ws,
                    size_t ws_bytes, void* stream) {
  if (int e = gn_check(N, HW, C, G)) return e;
  if (!dx && !dx_f16) return fail(MAS_ERR_INVALID_ARG, "gn_backward: dx may only be NULL when dx_f16 is given");
  if (dx_f16 && (!dx_bound || (dx_add && !add_amax)))
    return fail(MAS_ERR_INVALID_ARG, "gn_backward: the fp16 shadow of dx needs dx_bound (and add_amax with dx_add)");
  if (ws_bytes < mas_gn_ws_bytes(N, HW, C, G)) return fail(MAS_ERR_WORKSPACE, "gn_backward: workspace too small");
  int chunks = gn_chunks(N, HW, C);
  double* part = (double*)ws;
  double* nc = part + (size_t)N * chunks * C * 2;
  float* AB = (float*)(nc + (size_t)N * C * 2);
  unsigned int* mx = dx_f16 ? reinterpret_cast<unsigned int*>(AB + (size_t)N * G * 2) : nullptr;   // 3 words (inside the +256 slack)
  if (mx) {
    cudaError_t e = cudaMemsetAsync(mx, 0, 3 * sizeof(unsigned int), S(stream));
    if (e != cudaSuccess) return fail(MAS_ERR_LAUNCH, "gn_backward: memset: %s", cudaGetErrorString(e));
  }
  int lanes = GN_THREADS / (C / 4);
  size_t smem = (size_t)lanes * C * 2 * sizeof(double);
  // (A single-kernel form - pass 1, per-image hand-over through an arrival counter, pass 2 on the same chunk hoping for L2 hits -
  //  was built and measured: 22.0 vs 18.2 ms per step for all GroupNorm backwards, and its spin-wait hung on small shapes; removed.)
  gn_bwd_partial<<<dim3(chunks, N), GN_THREADS, smem, S(stream)>>>(dy, x, mean, rstd, gamma, beta, HW, C, G, silu, part, (float*)act_out,
                                                                   act_f16, mx);
  if (int e = launched("gn_bwd_partial")) return e;
  gn_bwd_nc<<<(int)cdiv((int64_t)N * C, 128), 128, 0, S(stream)>>>(part, N, chunks, C, nc);
  if (int e = launched("gn_bwd_nc")) return e;
  const int cblocks = (int)cdiv(C, 128);
  gn_bwd_final<<<cblocks + (int)cdiv((int64_t)N * G, 128), 128, 0, S(stream)>>>(N, C, G, gamma, nc, dgamma, dbeta, AB,
                                                                                1.0 / ((double)HW * (C / G)), cblocks, rstd, mx);
  if (int e = launched("gn_bwd_final")) return e;
  if (dx_amax) {
    cudaError_t e = cudaMemsetAsync(dx_amax, 0, sizeof(float), S(stream));
    if (e != cudaSuccess) return fail(MAS_ERR_LAUNCH, "gn_backward: memset: %s", cudaGetErrorString(e));
  }
  gn_bwd_apply<<<dim3(chunks, N), GN_THREADS, 0, S(stream)>>>(dy, x, mean, rstd, gamma, beta, AB, dx_add, dx, HW, C, G, silu,
                                                              reinterpret_cast<unsigned int*>(dx_amax), reinterpret_cast<__half*>(dx_f16), mx,
                                                              add_amax, dx_bound);
  return launched("gn_bwd_apply");
}

int mas_gn_finalize_partials(const float* part, int tiles_per_image, int N, int C, int G, int64_t hw, float eps, float* mean,
                             float* rstd, void* stream) {
  if (C % 4 || (C / 4) % G) return fail(MAS_ERR_UNSUPPORTED, "gn_finalize_partials: need C/G >= 4");
  gn_finalize_partials_kernel<<<(int)cdiv((int64_t)N * G, 8), 256, 0, S(stream)>>>(part, tiles_per_image, C, G, (double)hw * (C / G), eps,
                                                                                  mean, rstd, N * G);
  return launched("gn_finalize_partials");
}
int mas_gn_table(const float* mean, const float* rstd, const float* gamma, const float* beta, int N, int C, int G, float* table,
                 void* stream) {
  gn_table_kernel<<<(int)cdiv((int64_t)N * C, 256), 256, 0, S(stream)>>>(mean, rstd, gamma, beta, N, C, G, table);
  return launched("gn_table");
}
int mas_add(const float* a, const float* b, float* out, int64_t n, void* stream) {
  add_kernel<<<ew_grid(n), 256, 0, S(stream)>>>(a, b, out, n);
  return launched("add");
}
int mas_silu_forward(const float* x, float* y, int64_t n, void* stream) {
  silu_fwd_kernel<<<ew_grid(n), 256, 0, S(stream)>>>(x, y, n);
  return launched("silu_fwd");
}
int mas_silu_backward(const float* dy, const float* x, float* dx, int64_t n, void* stream) {
  silu_bwd_kernel<<<ew_grid(n), 256, 0, S(stream)>>>(dy, x, dx, n);
  return launched("silu_bwd");
}

int mas_softmax_forward(const float* s, float* p, int64_t rows, int cols, void* stream) {
  MAS_REQUIRE(rows > 0 && cols > 0, "softmax: bad shape");
  softmax_fwd_kernel<<<(unsigned)cdiv(rows, 8), 256, 0, S(stream)>>>(s, p, rows, cols);
  return launched("softmax_fwd");
}
int mas_softmax_backward(const float* p, const float* dp, float* ds, int64_t rows, int cols, float scale, void* stream) {
  MAS_REQUIRE(rows > 0 && cols > 0, "softmax: bad shape");
  softmax_bwd_kernel<<<(unsigned)cdiv(rows, 8), 256, 0, S(stream)>>>(p, dp, ds, rows, cols, scale);
  return launched("softmax_bwd");
}

int mas_bn_stats(const float* x, int64_t R, int C, double* stats_out, void* stream) {
  MAS_REQUIRE(R > 0 && C > 0, "bn_stats: bad shape");
  bn_stats_kernel<<<(int)cdiv(C, 32), dim3(32, 8), 0, S(stream)>>>(x, R, C, stats_out);
  return launched("bn_stats");
}
int mas_bn_finalize(const double* stats, double count, int C, float eps, float momentum, float* mean, float* invstd,
                    float* running_mean, float* running_var, void* stream) {
  bn_finalize_kernel<<<(int)cdiv(C, 128), 128, 0, S(stream)>>>(stats, count, C, eps, momentum, mean, invstd, running_mean, running_var);
  return launched("bn_finalize");
}
int mas_amax(const float* x, int64_t n, float* out, void* stream) {
  MAS_REQUIRE(x && out && n > 0, "amax: bad arguments");
  if (reinterpret_cast<uintptr_t>(x) & 15) return fail(MAS_ERR_UNSUPPORTED, "amax: x must be 16-byte aligned");
  cudaError_t e = cudaMemsetAsync(out, 0, sizeof(float), S(stream));
  if (e != cudaSuccess) return fail(MAS_ERR_LAUNCH, "amax: memset: %s", cudaGetErrorString(e));
  const int64_t n4 = n / 4;
  const int64_t blocks = cdiv(n4 > 0 ? n4 : 1, 256 * 8);
  amax_kernel<<<(int)(blocks < NUM_SMS * 8 ? blocks : NUM_SMS * 8), 256, 0, S(stream)>>>(reinterpret_cast<const float4*>(x), n4, x + n4 * 4,
                                                                                 (int)(n - n4 * 4), reinterpret_cast<unsigned int*>(out));
  return launched("amax");
}
int mas_bn_invstd(const float* running_var, float eps, float* invstd, int C, void* stream) {
  bn_invstd_kernel<<<(int)cdiv(C, 128), 128, 0, S(stream)>>>(running_var, eps, invstd, C);
  return launched("bn_invstd");
}
int mas_bn_apply(const float* x, const float* mean, const float* invstd, const float* gamma, const float* beta, float* y,
                 int64_t R, int C, void* stream) {
  bn_apply_kernel<<<ew_grid(R * C), 256, 0, S(stream)>>>(x, mean, invstd, gamma, beta, y, R * C, C, 1.0f);
  return launched("bn_apply");
}
int mas_bn_apply_lrelu(const float* x, const float* mean, const float* invstd, const float* gamma, const float* beta, float slope,
                       float* y, int64_t R, int C, void* stream) {
  MAS_REQUIRE(R > 0 && C > 0, "bn_apply_lrelu: bad shape");
  bn_apply_kernel<<<ew_grid(R * C), 256, 0, S(stream)>>>(x, mean, invstd, gamma, beta, y, R * C, C, slope);
  return launched("bn_apply_lrelu");
}
int mas_bn_backward_reduce(const float* dy, const float* x, const float* mean, const float* invstd, int64_t R, int C,
                           double* sums_out, void* stream) {
  bn_bwd_reduce_kernel<<<(int)cdiv(C, 32), dim3(32, 8), 0, S(stream)>>>(dy, x, mean, invstd, R, C, sums_out);
  return launched("bn_bwd_reduce");
}
size_t mas_bn_backward_reduce_lrelu_ws_bytes(int64_t R, int C) { return (size_t)cdiv(R, BN_RB) * 2 * C * sizeof(double) + 64; }
int mas_bn_backward_reduce_lrelu(const float* dy, const float* y, float slope, const float* x, const float* mean, const float* invstd,
                                 int64_t R, int C, double* sums_out, void* ws, size_t ws_bytes, void* stream) {
  MAS_REQUIRE(R > 0 && C > 0 && y, "bn_backward_reduce_lrelu: bad arguments");
  if (!ws || ws_bytes < mas_bn_backward_reduce_lrelu_ws_bytes(R, C)) return fail(MAS_ERR_WORKSPACE, "bn_backward_reduce_lrelu: workspace too small");
  const int chunks = (int)cdiv(R, BN_RB);
  bn_bwd_reduce_lrelu_part<<<dim3((unsigned)cdiv(C, 32), (unsigned)chunks), dim3(32, 8), 0, S(stream)>>>(dy, y, slope, x, mean, invstd,
                                                                                                           R, C, (double*)ws);
  if (int e = launched("bn_bwd_reduce_lrelu_part")) return e;
  bn_bwd_reduce_lrelu_final<<<(int)cdiv(2 * C, 128), 128, 0, S(stream)>>>((const double*)ws, chunks, R, C, sums_out);
  return launched("bn_bwd_reduce_lrelu_final");
}
int mas_bn_backward_apply(const float* dy, const float* x, const float* mean, const float* invstd, const float* gamma,
                          const double* sums_global, const double* sums_local, double inv_count, float* dx, float* dgamma,
                          float* dbeta, int64_t R, int C, void* stream) {
  bn_bwd_apply_kernel<<<ew_grid(R * C), 256, 0, S(stream)>>>(dy, x, mean, invstd, gamma, sums_global, inv_count, dx, dgamma, dbeta,
                                                             sums_local, R * C, C, nullptr, 1.0f);
  return launched("bn_bwd_apply");
}
int mas_bn_backward_apply_lrelu(const float* dy, const float* y, float slope, const float* x, const float* mean, const float* invstd,
                                const float* gamma, const double* sums, float* dx, float* dgamma, float* dbeta, int64_t R, int C,
                                void* stream) {
  MAS_REQUIRE(R > 0 && C > 0 && y, "bn_backward_apply_lrelu: bad arguments");
  bn_bwd_apply_kernel<<<ew_grid(R * C), 256, 0, S(stream)>>>(dy, x, mean, invstd, gamma, sums, 0.0, dx, dgamma, dbeta, sums, R * C, C,
                                                             y, slope);
  return launched("bn_bwd_apply_lrelu");
}

size_t mas_colsum_ws_bytes(mas_tensor4 t) { return (size_t)cdiv(t.n * t.h * t.w, CS_ROWS) * t.c * sizeof(double) + 64; }
int mas_colsum(const float* x, mas_tensor4 t, float* out, void* ws, size_t ws_bytes, void* stream) {
  if (ws_bytes < mas_colsum_ws_bytes(t)) return fail(MAS_ERR_WORKSPACE, "colsum: workspace too small");
  int chunks = (int)cdiv(t.n * t.h * t.w, CS_ROWS);
  colsum_partial<<<dim3((unsigned)cdiv(t.c, 32), chunks), dim3(32, 8), 0, S(stream)>>>(x, t, (double*)ws);
  if (int e = launched("colsum_partial")) return e;
  colsum_final<<<(int)cdiv(t.c, 128), 128, 0, S(stream)>>>((const double*)ws, chunks, (int)t.c, out);
  return launched("colsum_final");
}

int mas_copy_strided(const float* x, mas_tensor4 xs, float* y, mas_tensor4 ys, void* stream) {
  MAS_REQUIRE(xs.n == ys.n && xs.h == ys.h && xs.w == ys.w && xs.c == ys.c, "copy_strided: shape mismatch");
  int64_t total = xs.n * xs.h * xs.w * xs.c;
  copy_strided_kernel<<<ew_grid(total), 256, 0, S(stream)>>>(x, xs, y, ys, total);
  return launched("copy_strided");
}

int mas_nchw_to_nhwc_pad(const float* x_nchw, float* y_nhwc, int N, int C, int CP, int H, int W, void* stream) {
  MAS_REQUIRE(x_nchw && y_nhwc && N > 0 && C > 0 && CP >= C && H > 0 && W > 0, "nchw_to_nhwc_pad: bad arguments");
  if ((size_t)C * 33 * sizeof(float) > 48 * 1024) return fail(MAS_ERR_UNSUPPORTED, "nchw_to_nhwc_pad: C=%d too large", C);
  nchw_to_nhwc_pad_kernel<<<dim3((unsigned)cdiv(W, 32), H, N), 256, (size_t)C * 33 * sizeof(float), S(stream)>>>(x_nchw, y_nhwc, C, CP, H, W);
  return launched("nchw_to_nhwc_pad");
}
int mas_scale_by(const float* x, const float* g, float* y, int64_t n, void* stream) {
  scale_by_kernel<<<ew_grid(n), 256, 0, S(stream)>>>(x, g, y, n);
  return launched("scale_by");
}

int mas_sumpool2x2(const float* x, float* y, int N, int H, int W, int C, void* stream) {
  MAS_REQUIRE(C % 4 == 0, "sumpool2x2: C %% 4 != 0");
  int64_t total4 = (int64_t)N * H * W * (C / 4);
  sumpool2x2_kernel<<<ew_grid(total4), 256, 0, S(stream)>>>(x, y, H, W, C / 4, total4);
  return launched("sumpool2x2");
}

// channels-last logits (pitch CP) x NCHW target: loss (mean over N*C*H*W) and, separately, the gradient scaled by the
// upstream gradient g (device scalar or NULL = 1) - nothing of the loss's backward runs in the host framework
size_t mas_bce_cl_ws_bytes(int N, int H, int W) { return (size_t)N * H * cdiv(W, 32) * sizeof(double) + 64; }
int mas_bce_cl_forward(const float* logits, const float* target_nchw, const float* pos_weight, int N, int C, int CP, int H, int W,
                       float* loss_out, void* ws, size_t ws_bytes, void* stream) {
  MAS_REQUIRE(logits && target_nchw && pos_weight && loss_out && N > 0 && C > 0 && CP >= C && W % 32 == 0, "bce_cl_forward: bad arguments");
  if (ws_bytes < mas_bce_cl_ws_bytes(N, H, W)) return fail(MAS_ERR_WORKSPACE, "bce_cl_forward: workspace too small");
  const int nb = N * H * (W / 32);
  bce_cl_kernel<0><<<dim3(W / 32, H, N), 256, (size_t)C * 33 * sizeof(float), S(stream)>>>(logits, target_nchw, pos_weight, C, CP, H, W, nullptr,
                                                                                          0.f, nullptr, (double*)ws);
  if (int e = launched("bce_cl_loss")) return e;
  sum_final_kernel<<<1, 256, 0, S(stream)>>>((const double*)ws, nb, 1.0 / ((double)N * C * H * W), loss_out);
  return launched("bce_final");
}
int mas_bce_cl_backward(const float* logits, const float* target_nchw, const float* pos_weight, const float* g, int N, int C, int CP,
                        int H, int W, float* grad, void* stream) {
  MAS_REQUIRE(logits && target_nchw && pos_weight && grad && N > 0 && C > 0 && CP >= C && W % 32 == 0, "bce_cl_backward: bad arguments");
  bce_cl_kernel<1><<<dim3(W / 32, H, N), 256, (size_t)C * 33 * sizeof(float), S(stream)>>>(
      logits, target_nchw, pos_weight, C, CP, H, W, g, (float)(1.0 / ((double)N * C * H * W)), grad, nullptr);
  return launched("bce_cl_grad");
}

size_t mas_bce_ws_bytes(mas_tensor4 ls) { return (size_t)cdiv(ls.n * ls.h * ls.w * ls.c, BCE_CHUNK) * sizeof(double) + 64; }
int mas_bce_logits(const float* logits, mas_tensor4 ls, const float* target, mas_tensor4 ts, const float* pos_weight,
                   float* loss_out, float* grad, mas_tensor4 gs, float grad_scale, void* ws, size_t ws_bytes, void* stream) {
  int64_t total = ls.n * ls.h * ls.w * ls.c;
  if (ws_bytes < mas_bce_ws_bytes(ls)) return fail(MAS_ERR_WORKSPACE, "bce: workspace too small");
  int blocks = (int)cdiv(total, BCE_CHUNK);
  bce_kernel<<<blocks, 256, 0, S(stream)>>>(logits, ls, target, ts, pos_weight, grad, gs, grad_scale, (double*)ws, total);
  if (int e = launched("bce")) return e;
  sum_final_kernel<<<1, 256, 0, S(stream)>>>((const double*)ws, blocks, 1.0 / (double)total, loss_out);
  return launched("bce_final");
}

}  // extern "C"
