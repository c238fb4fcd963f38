// 4x4 pad-1 convolution family of the PatchGAN discriminator (losses/discriminator.py:21-35): forward, data gradient and
// weight gradient for stride 1 and 2, as exact-fp32 SIMT implicit GEMMs over explicit mas_tensor4 strides.
//
//   forward  y [m=(n,oh,ow)][co]  = sum_{k=(t,ci)} x (n, s*oh-1+kh, s*ow-1+kw, ci) * wf[k][co]
//   dgrad    dx[m=(n,ih,iw)][ci]  = sum_{k=(t,co)} dy(n, (ih+1-kh)/s, (iw+1-kw)/s, co) * wd[k][ci]
//                                   (only taps whose quotient is exact and inside dy contribute)
//   wgrad    dw[co][j=(t,ci)]     = sum_{p=(n,oh,ow)} dy(p, co) * x(n, s*oh-1+kh, s*ow-1+kw, ci)
//
// The large layers (model.2 / 5 / 8) instead run as 3x3 convolutions of a shift map on the fp16 wgmma kernels: see the
// shift-map kernels below and include/mas_b200.h.
//
// with t = 4*kh + kw.  k runs tap-major (k = t*C + c) so that consecutive k are consecutive channels: coalesced loads from a
// channels-last tensor.  wf / wd are the packed weights of mas_pack_conv4x4 (transpose 0 / 1).
#include "mas_common.cuh"

namespace mas {
namespace {

constexpr int BM = 64, BN = 64, BK = 16, NT = 256;

// One BK slice of the 64x64 tile: thread (ty, tx) owns rows 4ty..4ty+3 and columns 4tx..4tx+3.
__device__ __forceinline__ void tile_fma(const float (*As)[BM + 4], const float (*Bs)[BN + 4], float acc[4][4], int tx, int ty) {
#pragma unroll
  for (int k = 0; k < BK; ++k) {
    const float4 a = *reinterpret_cast<const float4*>(&As[k][ty * 4]);
    const float4 b = *reinterpret_cast<const float4*>(&Bs[k][tx * 4]);
    const float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
  }
}

// Forward (DGRAD = false: a = x, o = y) or data gradient (DGRAD = true: a = dy, o = dx).  Ca = channels of a, K = 16*Ca.
template <bool DGRAD>
__global__ void __launch_bounds__(NT) conv4x4_kernel(const float* __restrict__ a, mas_tensor4 as, const float* __restrict__ wp,
                                                      const float* __restrict__ bias, float* __restrict__ out, mas_tensor4 os,
                                                      int stride, float slope, int act) {
  __shared__ __align__(16) float As[BK][BM + 4];
  __shared__ __align__(16) float Bs[BK][BN + 4];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int64_t ohw = os.h * os.w, M = os.n * ohw;
  const int Nc = (int)os.c, Ca = (int)as.c, K = 16 * Ca;
  const int64_t m0 = (int64_t)blockIdx.x * BM;
  const int n0 = blockIdx.y * BN;

  // A rows of this thread: (tid >> 4) + 16 j, at k column tid & 15
  const int ka = tid & 15;
  int64_t abase[4];
  int ar[4], ac[4];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int64_t m = m0 + (tid >> 4) + 16 * j;
    if (m < M) {
      const int64_t n = m / ohw, r = m - n * ohw;
      abase[j] = n * as.sn;
      ar[j] = (int)(r / os.w);
      ac[j] = (int)(r - (int64_t)ar[j] * os.w);
    } else {
      abase[j] = 0;
      ar[j] = -(1 << 28);   // every tap falls outside a
      ac[j] = 0;
    }
  }
  const int nb = n0 + (tid & 63);

  float ra[4], rb[4];
  auto load = [&](int k0) {
    const int k = k0 + ka;
    const int t = k < K ? k / Ca : 0, c = k - t * Ca, kh = t >> 2, kw = t & 3;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      int ih, iw;
      bool ok = k < K;
      if (!DGRAD) {
        ih = ar[j] * stride - 1 + kh;
        iw = ac[j] * stride - 1 + kw;
      } else {
        const int u = ar[j] + 1 - kh, v = ac[j] + 1 - kw;
        if (stride == 2) {
          ok = ok && !(u & 1) && !(v & 1);
          ih = u >> 1;
          iw = v >> 1;
        } else {
          ih = u;
          iw = v;
        }
      }
      ok = ok && ih >= 0 && iw >= 0 && ih < as.h && iw < as.w;
      ra[j] = ok ? __ldg(a + abase[j] + ih * as.sh + iw * as.sw + c * as.sc) : 0.f;
    }
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int kk = k0 + (tid >> 6) + 4 * j;
      rb[j] = (kk < K && nb < Nc) ? __ldg(wp + (int64_t)kk * Nc + nb) : 0.f;
    }
  };

  float acc[4][4] = {};
  load(0);
  for (int k0 = 0; k0 < K; k0 += BK) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      As[ka][(tid >> 4) + 16 * j] = ra[j];
      Bs[(tid >> 6) + 4 * j][tid & 63] = rb[j];
    }
    __syncthreads();
    if (k0 + BK < K) load(k0 + BK);
    tile_fma(As, Bs, acc, tx, ty);
    __syncthreads();
  }

#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int64_t m = m0 + ty * 4 + i;
    if (m >= M) continue;
    const int64_t n = m / ohw, r = m - n * ohw, h = r / os.w, w = r - h * os.w;
    float* o = out + n * os.sn + h * os.sh + w * os.sw;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int co = n0 + tx * 4 + j;
      if (co >= Nc) continue;
      float v = acc[i][j] + (bias ? bias[co] : 0.f);
      if (act && !(v > 0.f)) v *= slope;
      o[co * os.sc] = v;
    }
  }
}

// Weight gradient, split over the pixels: part[split][co][j] for the pixel range of blockIdx.z.
__global__ void __launch_bounds__(NT) conv4x4_wgrad_kernel(const float* __restrict__ x, mas_tensor4 xs, const float* __restrict__ dy,
                                                            mas_tensor4 dys, int stride, int64_t chunk, float* __restrict__ part) {
  __shared__ __align__(16) float As[BK][BM + 4];
  __shared__ __align__(16) float Bs[BK][BN + 4];
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
  const int Cout = (int)dys.c, Cin = (int)xs.c, J = 16 * Cin;
  const int64_t ohw = dys.h * dys.w, P = dys.n * ohw;
  const int m0 = blockIdx.x * BM, n0 = blockIdx.y * BN;
  const int64_t p0 = (int64_t)blockIdx.z * chunk, p1 = min(P, p0 + chunk);

  const int col = tid & 63;                   // A: co = m0 + col;  B: j = n0 + col
  const int co = m0 + col, jj = n0 + col;
  const int t = jj < J ? jj / Cin : 0, ci = jj - t * Cin, kh = t >> 2, kw = t & 3;

  float ra[4], rb[4];
  auto load = [&](int64_t pk) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int64_t p = pk + (tid >> 6) + 4 * j;
      float va = 0.f, vb = 0.f;
      if (p < p1) {
        const int64_t n = p / ohw, r = p - n * ohw;
        const int oh = (int)(r / dys.w), ow = (int)(r - (int64_t)oh * dys.w);
        if (co < Cout) va = __ldg(dy + n * dys.sn + oh * dys.sh + ow * dys.sw + co * dys.sc);
        const int ih = oh * stride - 1 + kh, iw = ow * stride - 1 + kw;
        if (jj < J && ih >= 0 && iw >= 0 && ih < xs.h && iw < xs.w) vb = __ldg(x + n * xs.sn + ih * xs.sh + iw * xs.sw + ci * xs.sc);
      }
      ra[j] = va;
      rb[j] = vb;
    }
  };

  float acc[4][4] = {};
  load(p0);
  for (int64_t pk = p0; pk < p1; pk += BK) {
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      As[(tid >> 6) + 4 * j][col] = ra[j];
      Bs[(tid >> 6) + 4 * j][col] = rb[j];
    }
    __syncthreads();
    if (pk + BK < p1) load(pk + BK);
    tile_fma(As, Bs, acc, tx, ty);
    __syncthreads();
  }

  float* dst = part + (int64_t)blockIdx.z * Cout * J;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int m = m0 + ty * 4 + i;
    if (m >= Cout) continue;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int n = n0 + tx * 4 + j;
      if (n < J) dst[(int64_t)m * J + n] = acc[i][j];
    }
  }
}

// dw[co][ci][t] = sum over splits (in order: deterministic) of part[s][co][t*Cin + ci]
__global__ void conv4x4_wgrad_reduce(const float* __restrict__ part, int splits, int Cout, int Cin, float* __restrict__ dw) {
  const int64_t total = (int64_t)Cout * Cin * 16;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int t = (int)(i & 15);
    const int64_t oc = i >> 4;
    const int ci = (int)(oc % Cin), co = (int)(oc / Cin);
    const int64_t src = (int64_t)co * 16 * Cin + t * Cin + ci, stride = (int64_t)Cout * 16 * Cin;
    float s = 0.f;
    for (int k = 0; k < splits; ++k) s += part[k * stride + src];
    dw[i] = s;
  }
}

// transpose = 0: wf[(t*Cin + ci)][co];  transpose = 1: wd[(t*Cout + co)][ci]
__global__ void pack_conv4x4_kernel(const float* __restrict__ w, float* __restrict__ wp, int Cout, int Cin, int transpose) {
  const int64_t total = (int64_t)Cout * Cin * 16;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int t = (int)(i & 15);
    const int64_t oc = i >> 4;
    const int ci = (int)(oc % Cin), co = (int)(oc / Cin);
    const int64_t dst = transpose ? ((int64_t)t * Cout + co) * Cin + ci : ((int64_t)t * Cin + ci) * Cout + co;
    wp[dst] = w[i];
  }
}

__global__ void lrelu_backward_kernel(const float* __restrict__ dy, const float* __restrict__ y, float slope, float* __restrict__ dx,
                                      int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x)
    dx[i] = y[i] > 0.f ? dy[i] : dy[i] * slope;
}

// ---- tensor-core route: the 4x4 convolution as a 3x3 stride-1 pad-1 convolution of a 4*Cin-channel map
// X'(i, j, (2p + q)*Cin + c) = x(s*i + p, s*j + q, c) (0 outside x).  The 4x4 tap kh reads x row s*o + kh - 1 =
// s*(o + a - 1) + p, so it is the 3x3 tap a of plane p: stride 2: kh = 2a - 1 + p (16 of 36 taps); stride 1: kh = a for
// kh < 3 (p = 0) and kh = 3 -> (a = 2, p = 1) (one representative per 4x4 tap).
__host__ __device__ __forceinline__ int tap4_of(int a, int p, int stride) {
  if (stride == 2) {
    const int kh = 2 * a - 1 + p;
    return (kh >= 0 && kh < 4) ? kh : -1;
  }
  if (p == 0) return a;
  return a == 2 ? 3 : -1;
}

__global__ void shift_map_kernel(const float* __restrict__ x, mas_tensor4 xs, float* __restrict__ y, int Hs, int Ws, int stride) {
  const int C = (int)xs.c, C4 = 4 * C;
  const int64_t total = xs.n * Hs * Ws * C4;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int ch = (int)(i % C4);
    const int64_t pix = i / C4;
    const int j = (int)(pix % Ws), r = (int)((pix / Ws) % Hs);
    const int64_t n = pix / ((int64_t)Ws * Hs);
    const int pq = ch / C, c = ch - pq * C;
    const int ih = stride * r + (pq >> 1), iw = stride * j + (pq & 1);
    y[i] = (ih < xs.h && iw < xs.w) ? x[n * xs.sn + ih * xs.sh + iw * xs.sw + c * xs.sc] : 0.f;
  }
}

// adjoint of shift_map: dx(n, h, w, c) = sum over (p, q) with h = s*i + p, w = s*j + q inside X' of dX'(i, j, (2p + q)*C + c)
__global__ void shift_map_adjoint_kernel(const float* __restrict__ dxs_, int Hs, int Ws, float* __restrict__ dx, mas_tensor4 dxs,
                                         int stride) {
  const int C = (int)dxs.c, C4 = 4 * C;
  const int64_t total = dxs.n * dxs.h * dxs.w * C;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int c = (int)(i % C);
    const int64_t pix = i / C;
    const int w = (int)(pix % dxs.w), h = (int)((pix / dxs.w) % dxs.h);
    const int64_t n = pix / (dxs.w * dxs.h);
    float s = 0.f;
#pragma unroll
    for (int pq = 0; pq < 4; ++pq) {
      const int u = h - (pq >> 1), v = w - (pq & 1);
      if (u < 0 || v < 0 || u % stride || v % stride) continue;
      const int r = u / stride, j = v / stride;
      if (r < Hs && j < Ws) s += dxs_[((n * Hs + r) * Ws + j) * C4 + pq * C + c];
    }
    dx[n * dxs.sn + h * dxs.sh + w * dxs.sw + c * dxs.sc] = s;
  }
}

// to3x3 = 1: w3[co][(2p+q)*Cin + c][a][b] = w4[co][c][tap4(a,p)][tap4(b,q)] (0 where no 4x4 tap maps);
// to3x3 = 0: the adjoint for the weight gradient, dw4[co][c][kh][kw] = dw3 at the representative of (kh, kw).
__global__ void remap_weight_kernel(const float* __restrict__ src, float* __restrict__ dst, int Cout, int Cin, int stride, int to3x3) {
  const int64_t total = (int64_t)Cout * 4 * Cin * 9;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int b = (int)(i % 3), a = (int)((i / 3) % 3);
    const int ch = (int)((i / 9) % (4 * Cin));
    const int64_t co = i / (9 * 4 * (int64_t)Cin);
    const int pq = ch / Cin, c = ch - pq * Cin;
    const int kh = tap4_of(a, pq >> 1, stride), kw = tap4_of(b, pq & 1, stride);
    const int64_t i4 = ((co * Cin + c) * 4 + (kh < 0 ? 0 : kh)) * 4 + (kw < 0 ? 0 : kw);
    if (to3x3)
      dst[i] = (kh >= 0 && kw >= 0) ? src[i4] : 0.f;
    else if (kh >= 0 && kw >= 0)
      dst[i4] = src[i];
  }
}

inline int ew_blocks(int64_t n) { return (int)std::min<int64_t>(cdiv(n, 256), NUM_SMS * 16); }

inline int64_t out_extent(int64_t in, int stride) { return (in + 2 - 4) / stride + 1; }

bool geometry_ok(const mas_tensor4& in, const mas_tensor4& out, int stride) {
  return (stride == 1 || stride == 2) && in.n == out.n && in.h >= 2 && in.w >= 2 && out.h == out_extent(in.h, stride) &&
         out.w == out_extent(in.w, stride) && in.c > 0 && out.c > 0;
}

int wgrad_splits(const mas_tensor4& xs, const mas_tensor4& dys) {
  const int64_t tiles = cdiv(dys.c, BM) * cdiv(16 * xs.c, BN), P = dys.n * dys.h * dys.w;
  const int64_t want = cdiv(4 * NUM_SMS, tiles), most = cdiv(P, 4 * BK);
  return (int)std::max<int64_t>(1, std::min(want, most));
}

}  // namespace
}  // namespace mas

using namespace mas;

extern "C" {

int mas_pack_conv4x4(const float* w_oihw, float* w_packed, int Cout, int Cin, int transpose, void* stream) {
  MAS_REQUIRE(w_oihw && w_packed && Cout > 0 && Cin > 0, "pack_conv4x4: bad arguments");
  pack_conv4x4_kernel<<<ew_blocks((int64_t)Cout * Cin * 16), 256, 0, S(stream)>>>(w_oihw, w_packed, Cout, Cin, transpose != 0);
  return launched("pack_conv4x4");
}

int mas_conv4x4(const float* x, mas_tensor4 xs, const float* w_packed, const float* bias, float* y, mas_tensor4 ys, int stride,
                float act_slope, int act, void* stream) {
  MAS_REQUIRE(x && w_packed && y && geometry_ok(xs, ys, stride), "conv4x4: bad arguments or shapes");
  const int64_t M = ys.n * ys.h * ys.w;
  dim3 grid((unsigned)cdiv(M, BM), (unsigned)cdiv(ys.c, BN));
  conv4x4_kernel<false><<<grid, NT, 0, S(stream)>>>(x, xs, w_packed, bias, y, ys, stride, act_slope, act);
  return launched("conv4x4_fprop");
}

int mas_conv4x4_dgrad(const float* dy, mas_tensor4 dys, const float* w_packed_t, float* dx, mas_tensor4 dxs, int stride,
                      void* stream) {
  MAS_REQUIRE(dy && w_packed_t && dx && geometry_ok(dxs, dys, stride), "conv4x4_dgrad: bad arguments or shapes");
  const int64_t M = dxs.n * dxs.h * dxs.w;
  dim3 grid((unsigned)cdiv(M, BM), (unsigned)cdiv(dxs.c, BN));
  conv4x4_kernel<true><<<grid, NT, 0, S(stream)>>>(dy, dys, w_packed_t, nullptr, dx, dxs, stride, 0.f, 0);
  return launched("conv4x4_dgrad");
}

size_t mas_conv4x4_wgrad_ws_bytes(mas_tensor4 xs, mas_tensor4 dys) {
  return (size_t)wgrad_splits(xs, dys) * dys.c * 16 * xs.c * sizeof(float) + 64;
}

int mas_conv4x4_wgrad(const float* x, mas_tensor4 xs, const float* dy, mas_tensor4 dys, float* dw_oihw, int stride, void* ws,
                      size_t ws_bytes, void* stream) {
  MAS_REQUIRE(x && dy && dw_oihw && geometry_ok(xs, dys, stride), "conv4x4_wgrad: bad arguments or shapes");
  if (!ws || ws_bytes < mas_conv4x4_wgrad_ws_bytes(xs, dys)) return fail(MAS_ERR_WORKSPACE, "conv4x4_wgrad: workspace too small");
  const int splits = wgrad_splits(xs, dys);
  const int64_t P = dys.n * dys.h * dys.w, chunk = cdiv(cdiv(P, splits), BK) * BK;
  const int used = (int)cdiv(P, chunk);
  dim3 grid((unsigned)cdiv(dys.c, BM), (unsigned)cdiv(16 * xs.c, BN), (unsigned)used);
  conv4x4_wgrad_kernel<<<grid, NT, 0, S(stream)>>>(x, xs, dy, dys, stride, chunk, (float*)ws);
  if (int e = launched("conv4x4_wgrad")) return e;
  conv4x4_wgrad_reduce<<<ew_blocks(dys.c * xs.c * 16), 256, 0, S(stream)>>>((const float*)ws, used, (int)dys.c, (int)xs.c, dw_oihw);
  return launched("conv4x4_wgrad_reduce");
}

int mas_conv4x4_shift_map(const float* x, mas_tensor4 xs, float* y, int stride, void* stream) {
  MAS_REQUIRE(x && y && (stride == 1 || stride == 2) && xs.h >= 2 && xs.w >= 2, "conv4x4_shift_map: bad arguments");
  MAS_REQUIRE(stride == 1 || (xs.h % 2 == 0 && xs.w % 2 == 0), "conv4x4_shift_map: stride 2 needs even extents");
  const int Hs = (int)(xs.h / stride), Ws = (int)(xs.w / stride);
  shift_map_kernel<<<ew_blocks(xs.n * Hs * Ws * 4 * xs.c), 256, 0, S(stream)>>>(x, xs, y, Hs, Ws, stride);
  return launched("conv4x4_shift_map");
}

int mas_conv4x4_shift_map_adjoint(const float* dmap, float* dx, mas_tensor4 dxs, int stride, void* stream) {
  MAS_REQUIRE(dmap && dx && (stride == 1 || stride == 2) && dxs.h >= 2 && dxs.w >= 2, "conv4x4_shift_map_adjoint: bad arguments");
  MAS_REQUIRE(stride == 1 || (dxs.h % 2 == 0 && dxs.w % 2 == 0), "conv4x4_shift_map_adjoint: stride 2 needs even extents");
  shift_map_adjoint_kernel<<<ew_blocks(dxs.n * dxs.h * dxs.w * dxs.c), 256, 0, S(stream)>>>(dmap, (int)(dxs.h / stride),
                                                                                           (int)(dxs.w / stride), dx, dxs, stride);
  return launched("conv4x4_shift_map_adjoint");
}

int mas_conv4x4_remap_weight(const float* src, float* dst, int Cout, int Cin, int stride, int to3x3, void* stream) {
  MAS_REQUIRE(src && dst && Cout > 0 && Cin > 0 && (stride == 1 || stride == 2), "conv4x4_remap_weight: bad arguments");
  remap_weight_kernel<<<ew_blocks((int64_t)Cout * Cin * 36), 256, 0, S(stream)>>>(src, dst, Cout, Cin, stride, to3x3 != 0);
  return launched("conv4x4_remap_weight");
}

int mas_lrelu_backward(const float* dy, const float* y, float slope, float* dx, int64_t n, void* stream) {
  MAS_REQUIRE(dy && y && dx && n > 0, "lrelu_backward: bad arguments");
  lrelu_backward_kernel<<<ew_blocks(n), 256, 0, S(stream)>>>(dy, y, slope, dx, n);
  return launched("lrelu_backward");
}

}  // extern "C"
