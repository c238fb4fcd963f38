// fp32 FFMA (SIMT) contraction kernels: 3x3 convolution family (fprop / data-grad via packed weights /
// weight-grad), batched GEMM (1x1 convolutions, attention bmm).  Exact fp32: these are both the
// general-shape path (edge layers: Cin=3, Cout=3, NCHW views, odd sizes) and the on-GPU checker for the
// wgmma path (contract_tc.cu).  Reference call sites: modules.py:44-81,93-117,145-164,179,186.
#include "mas_common.cuh"

namespace mas {

struct ConvGeom {
  int N, Hin, Win, Cin, Hout, Wout, Cout, mode, ks;
  int64_t xsn, xsh, xsw, xsc, ysn, ysh, ysw, ysc;
};

// input coordinate of output (oy,ox) under tap (ty,tx); returns false if the tap reads padding
__device__ __forceinline__ bool conv_coord(const ConvGeom& g, int oy, int ox, int ty, int tx, int& iy, int& ix) {
  if (g.ks == 1) { iy = oy; ix = ox; return true; }
  switch (g.mode) {
    case MAS_CONV_S1:
      iy = oy + ty - 1; ix = ox + tx - 1;
      return (unsigned)iy < (unsigned)g.Hin && (unsigned)ix < (unsigned)g.Win;
    case MAS_CONV_S2:
      iy = 2 * oy + ty; ix = 2 * ox + tx;
      return iy < g.Hin && ix < g.Win;
    case MAS_CONV_UP: {
      int uy = oy + ty - 1, ux = ox + tx - 1;
      iy = uy >> 1; ix = ux >> 1;
      return (unsigned)uy < (unsigned)(2 * g.Hin) && (unsigned)ux < (unsigned)(2 * g.Win);
    }
    default: {  // MAS_CONV_ZS: value sits at odd (uy,ux) of the x2 grid
      int uy = oy + ty - 1, ux = ox + tx - 1;
      iy = uy >> 1; ix = ux >> 1;
      return uy >= 0 && ux >= 0 && (uy & 1) && (ux & 1) && iy < g.Hin && ix < g.Win;
    }
  }
}

__device__ __forceinline__ void ld4c(const float* p, int64_t sc, int c, int C, bool vec, float e[4]) {
  if (vec) {
    float4 v = __ldg(reinterpret_cast<const float4*>(p + c));
    e[0] = v.x; e[1] = v.y; e[2] = v.z; e[3] = v.w;
  } else {
#pragma unroll
    for (int i = 0; i < 4; ++i) e[i] = (c + i < C) ? __ldg(p + (int64_t)(c + i) * sc) : 0.f;
  }
}

// ------------------------------------------------------------------------------------------------ conv fprop
// y[m, co] = sum_{tap,ci} x[coord(m,tap), ci] * w[(tap*Cin+ci), co] + bias[co] + res[m, co]
// tile 128 pixels x BN couts, 256 threads as 16(tx: couts) x 16(ty: pixels), 8 x TN per thread, K step 8.
constexpr int CF_BM = 128, CF_BK = 8, CF_LDA = 132;

template <int BN, int TN>
__global__ void __launch_bounds__(256) conv_fprop_simt(const float* __restrict__ x, const float* __restrict__ w,
                                                       const float* __restrict__ bias, const float* __restrict__ res,
                                                       float* __restrict__ y, ConvGeom g, int vecA, int vecB, int vecY) {
  __shared__ __align__(16) float As[CF_BK][CF_LDA];
  __shared__ __align__(16) float Bs[CF_BK][BN];
  const int t = threadIdx.x, tx = t & 15, ty = t >> 4;
  const int64_t M = (int64_t)g.N * g.Hout * g.Wout;
  const int64_t m0 = (int64_t)blockIdx.x * CF_BM;
  const int co0 = blockIdx.y * BN;
  // A-load role: pixel pm, channel quad
  const int pm = t >> 1, cqa = (t & 1) * 4;
  const int64_t ma = m0 + pm;
  const bool mval = ma < M;
  int an = 0, aoy = 0, aox = 0;
  if (mval) {
    aox = (int)(ma % g.Wout);
    aoy = (int)((ma / g.Wout) % g.Hout);
    an = (int)(ma / ((int64_t)g.Wout * g.Hout));
  }
  const int ntap = g.ks * g.ks, nck = (g.Cin + CF_BK - 1) / CF_BK, nk = ntap * nck;

  float acc[8][TN];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < TN; ++j) acc[i][j] = 0.f;

  float ra[4], rb[4];
  auto gload = [&](int kt) {
    const int tap = kt / nck, ci0 = (kt % nck) * CF_BK;
    const int tyy = tap / g.ks, txx = tap % g.ks;
    int iy, ix;
    ra[0] = ra[1] = ra[2] = ra[3] = 0.f;
    if (mval && conv_coord(g, aoy, aox, tyy, txx, iy, ix) && ci0 + cqa < g.Cin)
      ld4c(x + an * g.xsn + iy * g.xsh + ix * g.xsw, g.xsc, ci0 + cqa, g.Cin, vecA, ra);
    rb[0] = rb[1] = rb[2] = rb[3] = 0.f;
    if constexpr (BN == 128) {
      const int kk = t >> 5, cq = (t & 31) * 4;
      if (ci0 + kk < g.Cin && co0 + cq < g.Cout)
        ld4c(w + (int64_t)(tap * g.Cin + ci0 + kk) * g.Cout, 1, co0 + cq, g.Cout, vecB, rb);
    } else {
      const int kk = t >> 4, c = t & 15;
      if (t < 128 && ci0 + kk < g.Cin && co0 + c < g.Cout) rb[0] = __ldg(w + (int64_t)(tap * g.Cin + ci0 + kk) * g.Cout + co0 + c);
    }
  };
  auto sstore = [&]() {
#pragma unroll
    for (int i = 0; i < 4; ++i) As[cqa + i][pm] = ra[i];
    if constexpr (BN == 128) {
      const int kk = t >> 5, cq = (t & 31) * 4;
      *reinterpret_cast<float4*>(&Bs[kk][cq]) = make_float4(rb[0], rb[1], rb[2], rb[3]);
    } else if (t < 128) {
      Bs[t >> 4][t & 15] = rb[0];
    }
  };

  gload(0);
  for (int kt = 0; kt < nk; ++kt) {
    sstore();
    __syncthreads();
    if (kt + 1 < nk) gload(kt + 1);
#pragma unroll
    for (int kk = 0; kk < CF_BK; ++kk) {
      float a[8], b[TN];
      float4 a0 = *reinterpret_cast<const float4*>(&As[kk][ty * 8]);
      float4 a1 = *reinterpret_cast<const float4*>(&As[kk][ty * 8 + 4]);
      a[0] = a0.x; a[1] = a0.y; a[2] = a0.z; a[3] = a0.w; a[4] = a1.x; a[5] = a1.y; a[6] = a1.z; a[7] = a1.w;
      if constexpr (TN == 8) {
        float4 b0 = *reinterpret_cast<const float4*>(&Bs[kk][tx * 4]);
        float4 b1 = *reinterpret_cast<const float4*>(&Bs[kk][(BN / 2) + tx * 4]);
        b[0] = b0.x; b[1] = b0.y; b[2] = b0.z; b[3] = b0.w; b[4] = b1.x; b[5] = b1.y; b[6] = b1.z; b[7] = b1.w;
      } else {
        b[0] = Bs[kk][tx];
      }
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
    }
    __syncthreads();
  }

  // epilogue
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int64_t m = m0 + ty * 8 + i;
    if (m >= M) continue;
    const int ox = (int)(m % g.Wout), oy = (int)((m / g.Wout) % g.Hout), n = (int)(m / ((int64_t)g.Wout * g.Hout));
    const int64_t base = n * g.ysn + oy * g.ysh + ox * g.ysw;
    if constexpr (TN == 8) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int c = co0 + h * (BN / 2) + tx * 4;
        if (c >= g.Cout) continue;
        float v[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) v[j] = acc[i][h * 4 + j];
        if (vecY) {
          if (bias) { float4 bb = __ldg(reinterpret_cast<const float4*>(bias + c)); v[0] += bb.x; v[1] += bb.y; v[2] += bb.z; v[3] += bb.w; }
          if (res) { float4 rr = __ldg(reinterpret_cast<const float4*>(res + base + c)); v[0] += rr.x; v[1] += rr.y; v[2] += rr.z; v[3] += rr.w; }
          *reinterpret_cast<float4*>(y + base + c) = make_float4(v[0], v[1], v[2], v[3]);
        } else {
#pragma unroll
          for (int j = 0; j < 4; ++j)
            if (c + j < g.Cout) {
              float o = v[j] + (bias ? __ldg(bias + c + j) : 0.f);
              if (res) o += __ldg(res + base + (int64_t)(c + j) * g.ysc);
              y[base + (int64_t)(c + j) * g.ysc] = o;
            }
        }
      }
    } else {
      const int c = co0 + tx;
      if (c < g.Cout) {
        float o = acc[i][0] + (bias ? __ldg(bias + c) : 0.f);
        if (res) o += __ldg(res + base + (int64_t)c * g.ysc);
        y[base + (int64_t)c * g.ysc] = o;
      }
    }
  }
}

// ------------------------------------------------------------------------------------------------ conv wgrad
// part[split][tap][co][ci] = sum_{m in split} dy[m, co] * x[coord(m,tap), ci]; 64x64 tile, 16 pixels per stage
constexpr int WG_BP = 16;
__global__ void __launch_bounds__(256) conv_wgrad_simt(const float* __restrict__ x, const float* __restrict__ dy,
                                                       float* __restrict__ part, ConvGeom g, int64_t chunk, int ci_tiles, int vecX,
                                                       int vecD) {
  __shared__ __align__(16) float As[WG_BP][64];  // dy  [pixel][co]
  __shared__ __align__(16) float Bs[WG_BP][64];  // x   [pixel][ci]
  const int t = threadIdx.x, tx = t & 15, ty = t >> 4;
  const int co0 = (blockIdx.x / ci_tiles) * 64, ci0 = (blockIdx.x % ci_tiles) * 64;
  const int tap = blockIdx.y, tyy = tap / g.ks, txx = tap % g.ks;
  const int64_t M = (int64_t)g.N * g.Hout * g.Wout;
  const int64_t p0 = (int64_t)blockIdx.z * chunk, p1 = min(M, p0 + chunk);
  const int lp = t >> 4, cq = (t & 15) * 4;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  float ra[4], rb[4];
  auto gload = [&](int64_t pb) {
    const int64_t m = pb + lp;
    ra[0] = ra[1] = ra[2] = ra[3] = 0.f;
    rb[0] = rb[1] = rb[2] = rb[3] = 0.f;
    if (m < p1) {
      const int ox = (int)(m % g.Wout), oy = (int)((m / g.Wout) % g.Hout), n = (int)(m / ((int64_t)g.Wout * g.Hout));
      if (co0 + cq < g.Cout) ld4c(dy + n * g.ysn + oy * g.ysh + ox * g.ysw, g.ysc, co0 + cq, g.Cout, vecD, ra);
      int iy, ix;
      if (ci0 + cq < g.Cin && conv_coord(g, oy, ox, tyy, txx, iy, ix))
        ld4c(x + n * g.xsn + iy * g.xsh + ix * g.xsw, g.xsc, ci0 + cq, g.Cin, vecX, rb);
    }
  };
  gload(p0);
  for (int64_t pb = p0; pb < p1; pb += WG_BP) {
    *reinterpret_cast<float4*>(&As[lp][cq]) = make_float4(ra[0], ra[1], ra[2], ra[3]);
    *reinterpret_cast<float4*>(&Bs[lp][cq]) = make_float4(rb[0], rb[1], rb[2], rb[3]);
    __syncthreads();
    if (pb + WG_BP < p1) gload(pb + WG_BP);
#pragma unroll
    for (int k = 0; k < WG_BP; ++k) {
      float4 a = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
      float4 b = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
      float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
  float* o = part + ((size_t)blockIdx.z * gridDim.y + tap) * g.Cout * g.Cin;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int co = co0 + ty * 4 + i, ci = ci0 + tx * 4 + j;
      if (co < g.Cout && ci < g.Cin) o[(size_t)co * g.Cin + ci] = acc[i][j];
    }
}
// dw[co][ci][tap] = sum_split part[split][tap][co][ci]
// optionally also dbias[c] = sum_split bpart[split][c] (the tensor-path kernel emits bias partials next to the weight partials)
__global__ void conv_wgrad_reduce(const float* __restrict__ part, int splits, int ntap, int Cout, int Cin, float* __restrict__ dw,
                                  const float* __restrict__ bpart = nullptr, float* __restrict__ dbias = nullptr) {
  if (bpart)
    for (int c = blockIdx.x * blockDim.x + threadIdx.x; c < Cout; c += gridDim.x * blockDim.x) {
      float a = 0.f;
      for (int s = 0; s < splits; ++s) a += bpart[(size_t)s * Cout + c];
      dbias[c] = a;
    }
  int64_t total = (int64_t)Cout * Cin * ntap;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int tap = (int)(i / ((int64_t)Cout * Cin));
    int64_t r = i % ((int64_t)Cout * Cin);
    int co = (int)(r / Cin), ci = (int)(r % Cin);
    float a = 0.f;
    for (int s = 0; s < splits; ++s) a += part[((size_t)s * ntap + tap) * Cout * Cin + r];
    dw[((size_t)co * Cin + ci) * ntap + tap] = a;
  }
}

// [Cout][Cin][3][3] -> fprop form [(tap*Cin+ci)][co] or data-grad form [(tap*Cout+co)][ci] with flipped taps
__global__ void pack_conv3x3_kernel(const float* __restrict__ w, float* __restrict__ out, int Cout, int Cin, int flipT, int rtf32) {
  int64_t total = (int64_t)9 * Cout * Cin;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    float v;
    if (!flipT) {
      int co = (int)(i % Cout);
      int64_t r = i / Cout;
      int ci = (int)(r % Cin), tap = (int)(r / Cin);
      v = w[((size_t)co * Cin + ci) * 9 + tap];
    } else {
      int ci = (int)(i % Cin);
      int64_t r = i / Cin;
      int co = (int)(r % Cout), tap = (int)(r / Cout);
      v = w[((size_t)co * Cin + ci) * 9 + (8 - tap)];
    }
    out[i] = rtf32 ? round_tf32(v) : v;
  }
}

// ------------------------------------------------------------------------------------------------ batched GEMM
// C[b] = alpha*op(A[b])*op(B[b]) + bias[n] + residual; 64x64 tile, K step 16, 4x4 per thread.
constexpr int GM_BK = 16, GM_LD = 68;
__device__ __forceinline__ void ld4_gemm(const float* p, int64_t ld, int r, int R, int c, int Cn, bool vec, float e[4]) {
  // four consecutive elements p[r*ld + c .. c+3], zero outside [0,R) x [0,Cn)
  e[0] = e[1] = e[2] = e[3] = 0.f;
  if (r >= R || c >= Cn) return;
  if (vec && c + 3 < Cn) {
    float4 v = __ldg(reinterpret_cast<const float4*>(p + (int64_t)r * ld + c));
    e[0] = v.x; e[1] = v.y; e[2] = v.z; e[3] = v.w;
  } else {
#pragma unroll
    for (int i = 0; i < 4; ++i)
      if (c + i < Cn) e[i] = __ldg(p + (int64_t)r * ld + c + i);
  }
}
__global__ void __launch_bounds__(256) gemm_simt(const float* __restrict__ A, const float* __restrict__ B, float* __restrict__ C, int M,
                                                 int N, int K, int64_t lda, int64_t ldb, int64_t ldc, int64_t sa, int64_t sb,
                                                 int64_t sc, int ta, int tb, float alpha, const float* __restrict__ bias,
                                                 const float* __restrict__ res, int vecA, int vecB, int vecC) {
  __shared__ __align__(16) float As[GM_BK][GM_LD];
  __shared__ __align__(16) float Bs[GM_BK][GM_LD];
  const int t = threadIdx.x, tx = t & 15, ty = t >> 4;
  const int m0 = blockIdx.y * 64, n0 = blockIdx.x * 64;
  A += (int64_t)blockIdx.z * sa;
  B += (int64_t)blockIdx.z * sb;
  C += (int64_t)blockIdx.z * sc;
  if (res) res += (int64_t)blockIdx.z * sc;
  float acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;
  float ra[4], rb[4];
  auto gload = [&](int k0) {
    if (ta) ld4_gemm(A, lda, k0 + (t >> 4), K, m0 + (t & 15) * 4, M, vecA, ra);  // stored K x M
    else ld4_gemm(A, lda, m0 + (t >> 2), M, k0 + (t & 3) * 4, K, vecA, ra);       // stored M x K
    if (tb) ld4_gemm(B, ldb, n0 + (t >> 2), N, k0 + (t & 3) * 4, K, vecB, rb);    // stored N x K
    else ld4_gemm(B, ldb, k0 + (t >> 4), K, n0 + (t & 15) * 4, N, vecB, rb);      // stored K x N
  };
  auto sstore = [&]() {
    if (ta) *reinterpret_cast<float4*>(&As[t >> 4][(t & 15) * 4]) = make_float4(ra[0], ra[1], ra[2], ra[3]);
    else {
#pragma unroll
      for (int i = 0; i < 4; ++i) As[(t & 3) * 4 + i][t >> 2] = ra[i];
    }
    if (!tb) *reinterpret_cast<float4*>(&Bs[t >> 4][(t & 15) * 4]) = make_float4(rb[0], rb[1], rb[2], rb[3]);
    else {
#pragma unroll
      for (int i = 0; i < 4; ++i) Bs[(t & 3) * 4 + i][t >> 2] = rb[i];
    }
  };
  gload(0);
  for (int k0 = 0; k0 < K; k0 += GM_BK) {
    sstore();
    __syncthreads();
    if (k0 + GM_BK < K) gload(k0 + GM_BK);
#pragma unroll
    for (int k = 0; k < GM_BK; ++k) {
      float4 a = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
      float4 b = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
      float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    __syncthreads();
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= M) continue;
    const int n = n0 + tx * 4;
    if (n >= N) continue;
    float v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) v[j] = alpha * acc[i][j] + ((bias && n + j < N) ? __ldg(bias + n + j) : 0.f);
    float* cp = C + (int64_t)m * ldc + n;
    if (vecC && n + 3 < N) {
      if (res) { float4 r = __ldg(reinterpret_cast<const float4*>(res + (int64_t)m * ldc + n)); v[0] += r.x; v[1] += r.y; v[2] += r.z; v[3] += r.w; }
      *reinterpret_cast<float4*>(cp) = make_float4(v[0], v[1], v[2], v[3]);
    } else {
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (n + j < N) cp[j] = v[j] + (res ? __ldg(res + (int64_t)m * ldc + n + j) : 0.f);
    }
  }
}

// Large aligned case (the AttnBlock token contractions: M, N multiples of 128, K of 16, 16-byte aligned operands):
// 128x128 tile, 8x8 accumulators per thread as 2x2 blocks of 4x4 (so every shared-memory read is a conflict-free LDS.128
// and four of them feed 64 FMAs), K step 16, register-prefetched global loads into a double-buffered tile: one barrier
// per K step.  Strict fp32 like torch.bmm (modules.py:180,186).
constexpr int G2_BK = 16, G2_LD = 132;
__global__ void __launch_bounds__(256, 2) gemm_simt128(const float* __restrict__ A, const float* __restrict__ B, float* __restrict__ C, int K,
                                                    int64_t lda, int64_t ldb, int64_t ldc, int64_t sa, int64_t sb, int64_t sc, int ta, int tb,
                                                    float alpha, const float* __restrict__ bias, const float* __restrict__ res) {
  __shared__ __align__(16) float As[2][G2_BK][G2_LD];
  __shared__ __align__(16) float Bs[2][G2_BK][G2_LD];
  const int t = threadIdx.x, tx = t & 15, ty = t >> 4;
  const int m0 = blockIdx.y * 128, n0 = blockIdx.x * 128;
  A += (int64_t)blockIdx.z * sa;
  B += (int64_t)blockIdx.z * sb;
  C += (int64_t)blockIdx.z * sc;
  if (res) res += (int64_t)blockIdx.z * sc;
  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
  float4 ra[2], rb[2];
  // operand stored [rows = M or N][K] (K contiguous): thread reads 4 consecutive k of row (t>>2)+64*i -> transposed scalar stores
  // operand stored [K][rows]          (rows contiguous): thread reads 4 consecutive rows of k = (t>>5)+8*i -> one 16-byte store
  auto gload = [&](int k0) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      ra[i] = ta ? __ldg(reinterpret_cast<const float4*>(A + (int64_t)(k0 + (t >> 5) + 8 * i) * lda + m0 + (t & 31) * 4))
                 : __ldg(reinterpret_cast<const float4*>(A + (int64_t)(m0 + (t >> 2) + 64 * i) * lda + k0 + (t & 3) * 4));
      rb[i] = tb ? __ldg(reinterpret_cast<const float4*>(B + (int64_t)(n0 + (t >> 2) + 64 * i) * ldb + k0 + (t & 3) * 4))
                 : __ldg(reinterpret_cast<const float4*>(B + (int64_t)(k0 + (t >> 5) + 8 * i) * ldb + n0 + (t & 31) * 4));
    }
  };
  auto sstore = [&](int buf) {
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      if (ta) *reinterpret_cast<float4*>(&As[buf][(t >> 5) + 8 * i][(t & 31) * 4]) = ra[i];
      else {
        const int r = (t >> 2) + 64 * i, k = (t & 3) * 4;
        As[buf][k + 0][r] = ra[i].x; As[buf][k + 1][r] = ra[i].y; As[buf][k + 2][r] = ra[i].z; As[buf][k + 3][r] = ra[i].w;
      }
      if (!tb) *reinterpret_cast<float4*>(&Bs[buf][(t >> 5) + 8 * i][(t & 31) * 4]) = rb[i];
      else {
        const int r = (t >> 2) + 64 * i, k = (t & 3) * 4;
        Bs[buf][k + 0][r] = rb[i].x; Bs[buf][k + 1][r] = rb[i].y; Bs[buf][k + 2][r] = rb[i].z; Bs[buf][k + 3][r] = rb[i].w;
      }
    }
  };
  gload(0);
  sstore(0);
  __syncthreads();
  int buf = 0;
  for (int k0 = 0; k0 < K; k0 += G2_BK) {
    const bool more = k0 + G2_BK < K;
    if (more) gload(k0 + G2_BK);
#pragma unroll
    for (int k = 0; k < G2_BK; ++k) {
      const float4 a0 = *reinterpret_cast<const float4*>(&As[buf][k][ty * 4]);
      const float4 a1 = *reinterpret_cast<const float4*>(&As[buf][k][64 + ty * 4]);
      const float4 b0 = *reinterpret_cast<const float4*>(&Bs[buf][k][tx * 4]);
      const float4 b1 = *reinterpret_cast<const float4*>(&Bs[buf][k][64 + tx * 4]);
      const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w}, bv[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
      for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
    }
    if (more) {
      sstore(buf ^ 1);   // the other buffer was last read before the previous barrier
      __syncthreads();
      buf ^= 1;
    }
  }
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const int m = m0 + (i < 4 ? ty * 4 + i : 64 + ty * 4 + i - 4);
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int n = n0 + h * 64 + tx * 4;
      float4 v = make_float4(alpha * acc[i][h * 4 + 0], alpha * acc[i][h * 4 + 1], alpha * acc[i][h * 4 + 2], alpha * acc[i][h * 4 + 3]);
      if (bias) {
        const float4 bb = __ldg(reinterpret_cast<const float4*>(bias + n));
        v.x += bb.x; v.y += bb.y; v.z += bb.z; v.w += bb.w;
      }
      if (res) {
        const float4 r = __ldg(reinterpret_cast<const float4*>(res + (int64_t)m * ldc + n));
        v.x += r.x; v.y += r.y; v.z += r.z; v.w += r.w;
      }
      *reinterpret_cast<float4*>(C + (int64_t)m * ldc + n) = v;
    }
  }
}

static inline bool al16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

int conv_geom(ConvGeom& g, mas_tensor4 xs, mas_tensor4 ys, int Cin, int Cout, int mode, int ks) {
  g.N = (int)xs.n; g.Hin = (int)xs.h; g.Win = (int)xs.w; g.Cin = Cin;
  g.Hout = (int)ys.h; g.Wout = (int)ys.w; g.Cout = Cout; g.mode = mode; g.ks = ks;
  g.xsn = xs.sn; g.xsh = xs.sh; g.xsw = xs.sw; g.xsc = xs.sc;
  g.ysn = ys.sn; g.ysh = ys.sh; g.ysw = ys.sw; g.ysc = ys.sc;
  if (xs.n != ys.n) return fail(MAS_ERR_INVALID_ARG, "conv: batch mismatch");
  int64_t eh, ew;
  if (ks == 1) { eh = xs.h; ew = xs.w; }
  else if (mode == MAS_CONV_S1) { eh = xs.h; ew = xs.w; }
  else if (mode == MAS_CONV_S2) { eh = xs.h / 2; ew = xs.w / 2; }
  else if (mode == MAS_CONV_UP || mode == MAS_CONV_ZS) { eh = xs.h * 2; ew = xs.w * 2; }
  else return fail(MAS_ERR_INVALID_ARG, "conv: unknown mode %d", mode);
  if (ys.h != eh || ys.w != ew) return fail(MAS_ERR_INVALID_ARG, "conv: output %lldx%lld, expected %lldx%lld (mode %d)", (long long)ys.h, (long long)ys.w, (long long)eh, (long long)ew, mode);
  return MAS_OK;
}

static bool vec_ok(const float* p, int C, int64_t sn, int64_t sh, int64_t sw, int64_t sc) {
  return sc == 1 && C % 4 == 0 && sn % 4 == 0 && sh % 4 == 0 && sw % 4 == 0 && al16(p);
}

int conv3x3_fprop_simt_launch(const float* x, mas_tensor4 xs, const float* w, const float* bias, const float* res, float* y,
                              mas_tensor4 ys, int mode, int ks, cudaStream_t st) {
  ConvGeom g;
  if (int e = conv_geom(g, xs, ys, (int)xs.c, (int)ys.c, mode, ks)) return e;
  int64_t M = (int64_t)g.N * g.Hout * g.Wout;
  int vecA = vec_ok(x, g.Cin, g.xsn, g.xsh, g.xsw, g.xsc);
  int vecB = g.Cout % 4 == 0 && al16(w);
  int vecY = vec_ok(y, g.Cout, g.ysn, g.ysh, g.ysw, g.ysc) && (!res || al16(res)) && (!bias || al16(bias));
  if (g.Cout > 16) {
    dim3 grid((unsigned)cdiv(M, CF_BM), (unsigned)cdiv(g.Cout, 128));
    conv_fprop_simt<128, 8><<<grid, 256, 0, st>>>(x, w, bias, res, y, g, vecA, vecB, vecY);
  } else {
    dim3 grid((unsigned)cdiv(M, CF_BM), 1);
    conv_fprop_simt<16, 1><<<grid, 256, 0, st>>>(x, w, bias, res, y, g, vecA, vecB, vecY);
  }
  return launched("conv_fprop_simt");
}

static int wgrad_splits(int64_t M, int tiles, int ntap) {
  int64_t want = cdiv(NUM_SMS * 4, (int64_t)tiles * ntap);
  int64_t maxs = cdiv(M, 256);
  int64_t s = want < 1 ? 1 : want;
  if (s > maxs) s = maxs;
  if (s > 128) s = 128;
  return (int)(s < 1 ? 1 : s);
}

size_t conv_wgrad_simt_ws(mas_tensor4 xs, mas_tensor4 dys, int ks) {
  int Cin = (int)xs.c, Cout = (int)dys.c, ntap = ks * ks;
  int tiles = (int)(cdiv(Cout, 64) * cdiv(Cin, 64));
  int64_t M = dys.n * dys.h * dys.w;
  return (size_t)wgrad_splits(M, tiles, ntap) * ntap * Cout * Cin * sizeof(float) + 256;
}

int conv_wgrad_simt_launch(const float* x, mas_tensor4 xs, const float* dy, mas_tensor4 dys, float* dw, int mode, int ks, void* ws,
                           size_t ws_bytes, cudaStream_t st) {
  ConvGeom g;
  if (int e = conv_geom(g, xs, dys, (int)xs.c, (int)dys.c, mode, ks)) return e;
  if (ws_bytes < conv_wgrad_simt_ws(xs, dys, ks)) return fail(MAS_ERR_WORKSPACE, "conv_wgrad: workspace too small");
  int ntap = ks * ks, ci_tiles = (int)cdiv(g.Cin, 64), tiles = (int)cdiv(g.Cout, 64) * ci_tiles;
  int64_t M = (int64_t)g.N * g.Hout * g.Wout;
  int splits = wgrad_splits(M, tiles, ntap);
  int64_t chunk = cdiv(cdiv(M, splits), WG_BP) * WG_BP;
  int vecX = vec_ok(x, g.Cin, g.xsn, g.xsh, g.xsw, g.xsc), vecD = vec_ok(dy, g.Cout, g.ysn, g.ysh, g.ysw, g.ysc);
  conv_wgrad_simt<<<dim3(tiles, ntap, splits), 256, 0, st>>>(x, dy, (float*)ws, g, chunk, ci_tiles, vecX, vecD);
  if (int e = launched("conv_wgrad_simt")) return e;
  int64_t total = (int64_t)ntap * g.Cout * g.Cin;
  conv_wgrad_reduce<<<(int)(cdiv(total, 256) < 1184 ? cdiv(total, 256) : 1184), 256, 0, st>>>((const float*)ws, splits, ntap, g.Cout, g.Cin, dw);
  return launched("conv_wgrad_reduce");
}

void conv_wgrad_reduce_launch(const float* part, int splits, int ntap, int Cout, int Cin, float* dw, const float* bpart, float* dbias,
                              cudaStream_t st) {
  int64_t total = (int64_t)ntap * Cout * Cin;
  conv_wgrad_reduce<<<(int)(cdiv(total, 256) < 1184 ? cdiv(total, 256) : 1184), 256, 0, st>>>(part, splits, ntap, Cout, Cin, dw,
                                                                                             dbias ? bpart : nullptr, dbias);
}

int gemm_simt_launch(const float* A, const float* B, float* C, int M, int N, int K, int batch, int64_t lda, int64_t ldb, int64_t ldc,
                     int64_t sa, int64_t sb, int64_t sc, int ta, int tb, float alpha, const float* bias, const float* res,
                     cudaStream_t st) {
  int vecA = al16(A) && lda % 4 == 0 && sa % 4 == 0, vecB = al16(B) && ldb % 4 == 0 && sb % 4 == 0;
  int vecC = al16(C) && ldc % 4 == 0 && sc % 4 == 0 && (!res || al16(res));
  if (M % 128 == 0 && N % 128 == 0 && K % G2_BK == 0 && vecA && vecB && vecC && (!bias || al16(bias))) {
    gemm_simt128<<<dim3(N / 128, M / 128, batch), 256, 0, st>>>(A, B, C, K, lda, ldb, ldc, sa, sb, sc, ta, tb, alpha, bias, res);
    return launched("gemm_simt128");
  }
  dim3 grid((unsigned)cdiv(N, 64), (unsigned)cdiv(M, 64), batch);
  gemm_simt<<<grid, 256, 0, st>>>(A, B, C, M, N, K, lda, ldb, ldc, sa, sb, sc, ta, tb, alpha, bias, res, vecA, vecB, vecC);
  return launched("gemm_simt");
}

}  // namespace mas

using namespace mas;

extern "C" {

int mas_pack_conv3x3(const float* w_oihw, float* w_packed, int Cout, int Cin, int flip_transpose, int round_tf32, void* stream) {
  MAS_REQUIRE(Cout > 0 && Cin > 0, "pack_conv3x3: bad shape");
  int64_t total = (int64_t)9 * Cout * Cin;
  pack_conv3x3_kernel<<<(int)(cdiv(total, 256) < 2368 ? cdiv(total, 256) : 2368), 256, 0, S(stream)>>>(w_oihw, w_packed, Cout, Cin,
                                                                                                       flip_transpose, round_tf32);
  return launched("pack_conv3x3");
}

}  // extern "C"
