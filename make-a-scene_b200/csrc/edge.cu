// Edge convolutions of the VQ-IMG path: conv_in (3 -> 128, reads the caller's NCHW image) and conv_out
// (128 -> 3, writes the NCHW reconstruction) — modules.py:219 and :364.  K = 27 / N = 3 do not map onto
// 128-wide MMA tiles (SURVEY.md 7.3 #7); these layers are HBM-bound (one 128-channel fp32 tensor read or
// written), so they get direct fp32 kernels: thread = output (or input) channel, image tile broadcast from
// shared memory.  All four directions (fprop, data gradient, weight/bias gradient) are covered.
#include "mas_common.cuh"
#include "edge.cuh"

namespace mas {

constexpr int ET_H = 8, ET_W = 32;  // pixels per block tile

// ---------------------------------------------------------------------------------------------------- small Cin -> big Cout
// y[n,oy,ox,co] = bias[co] + sum_{ci<3,tap} xs[n,ci,oy+ty-1,ox+tx-1] * W(co,ci,tap)
//   flipT = 0: W = w[(co*3+ci)*9+tap]            (conv_in forward,  w is [Cbig][3][3][3])
//   flipT = 1: W = w[(ci*Cbig+co)*9+(8-tap)]     (conv_out data gradient, w is [3][Cbig][3][3])
__global__ void __launch_bounds__(256) small_cin_fprop(const float* __restrict__ xs, const float* __restrict__ w,
                                                       const float* __restrict__ bias, float* __restrict__ y, EdgeGeom g, int flipT) {
  __shared__ float xt[SC][ET_H + 2][ET_W + 2];
  const int t = threadIdx.x, col = t & 127, half = t >> 7;
  const int co = blockIdx.z % ((g.Cbig + 127) / 128) * 128 + col, n = blockIdx.z / ((g.Cbig + 127) / 128);
  const int y0 = blockIdx.y * ET_H, x0 = blockIdx.x * ET_W;
  for (int i = t; i < SC * (ET_H + 2) * (ET_W + 2); i += 256) {
    int ci = i / ((ET_H + 2) * (ET_W + 2)), r = (i / (ET_W + 2)) % (ET_H + 2), c = i % (ET_W + 2);
    int iy = y0 - 1 + r, ix = x0 - 1 + c;
    float v = 0.f;
    if ((unsigned)iy < (unsigned)g.H && (unsigned)ix < (unsigned)g.W) v = __ldg(xs + n * g.sn + ci * g.sc + iy * g.sh + ix * g.sw);
    xt[ci][r][c] = v;
  }
  float wr[SC * 9];
  const bool cov = co < g.Cbig;
#pragma unroll
  for (int ci = 0; ci < SC; ++ci)
#pragma unroll
    for (int tap = 0; tap < 9; ++tap)
      wr[ci * 9 + tap] = !cov ? 0.f : (flipT ? __ldg(w + ((size_t)ci * g.Cbig + co) * 9 + (8 - tap)) : __ldg(w + ((size_t)co * SC + ci) * 9 + tap));
  const float b = (bias && cov) ? __ldg(bias + co) : 0.f;
  __syncthreads();
  for (int r = half * (ET_H / 2); r < (half + 1) * (ET_H / 2); ++r) {
    const int oy = y0 + r;
    if (oy >= g.H) break;
#pragma unroll 4
    for (int c = 0; c < ET_W; ++c) {
      const int ox = x0 + c;
      if (ox >= g.W) break;
      float acc = b;
#pragma unroll
      for (int ci = 0; ci < SC; ++ci)
#pragma unroll
        for (int ty = 0; ty < 3; ++ty)
#pragma unroll
          for (int tx = 0; tx < 3; ++tx) acc = fmaf(xt[ci][r + ty][c + tx], wr[ci * 9 + ty * 3 + tx], acc);
      if (cov) y[((size_t)(n * g.H + oy) * g.W + ox) * g.Cbig + co] = acc;
    }
  }
}

// dW[co][ci][tap] = sum_p dy[p][co] * xs[p+tap][ci], db[co] = sum_p dy[p][co]; persistent blocks, partial[block][half][28][Cbig]
__global__ void __launch_bounds__(256) small_cin_wgrad(const float* __restrict__ xs, const float* __restrict__ dy,
                                                       float* __restrict__ part, EdgeGeom g, int tiles_x, int tiles_y, int cblk) {
  __shared__ float xt[SC][ET_H + 2][ET_W + 2];
  const int t = threadIdx.x, col = t & 127, half = t >> 7;
  const int co = cblk * 128 + col;
  const bool cov = co < g.Cbig;
  float acc[SC * 9 + 1];
#pragma unroll
  for (int i = 0; i < SC * 9 + 1; ++i) acc[i] = 0.f;
  const int64_t ntiles = (int64_t)g.N * tiles_x * tiles_y;
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int tx_ = (int)(tile % tiles_x), ty_ = (int)((tile / tiles_x) % tiles_y), n = (int)(tile / ((int64_t)tiles_x * tiles_y));
    const int y0 = ty_ * ET_H, x0 = tx_ * ET_W;
    __syncthreads();
    for (int i = t; i < SC * (ET_H + 2) * (ET_W + 2); i += 256) {
      int ci = i / ((ET_H + 2) * (ET_W + 2)), r = (i / (ET_W + 2)) % (ET_H + 2), c = i % (ET_W + 2);
      int iy = y0 - 1 + r, ix = x0 - 1 + c;
      float v = 0.f;
      if ((unsigned)iy < (unsigned)g.H && (unsigned)ix < (unsigned)g.W) v = __ldg(xs + n * g.sn + ci * g.sc + iy * g.sh + ix * g.sw);
      xt[ci][r][c] = v;
    }
    __syncthreads();
    for (int r = half * (ET_H / 2); r < (half + 1) * (ET_H / 2); ++r) {
      const int oy = y0 + r;
      if (oy >= g.H) break;
#pragma unroll 4
      for (int c = 0; c < ET_W; ++c) {
        const int ox = x0 + c;
        if (ox >= g.W) break;
        const float d = cov ? __ldg(dy + ((size_t)(n * g.H + oy) * g.W + ox) * g.Cbig + co) : 0.f;
        acc[SC * 9] += d;
#pragma unroll
        for (int ci = 0; ci < SC; ++ci)
#pragma unroll
          for (int ty = 0; ty < 3; ++ty)
#pragma unroll
            for (int tx = 0; tx < 3; ++tx) acc[ci * 9 + ty * 3 + tx] = fmaf(d, xt[ci][r + ty][c + tx], acc[ci * 9 + ty * 3 + tx]);
      }
    }
  }
  if (cov) {
    float* o = part + ((size_t)(blockIdx.x * 2 + half) * (SC * 9 + 1)) * g.Cbig + co;
#pragma unroll
    for (int i = 0; i < SC * 9 + 1; ++i) o[(size_t)i * g.Cbig] = acc[i];
  }
}
// part[P][28][Cbig] -> dw[co][ci][tap] (i = ci*9+tap), db[co]
__global__ void small_cin_wgrad_reduce(const float* __restrict__ part, int P, int Cbig, float* __restrict__ dw, float* __restrict__ db) {
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (SC * 9 + 1) * Cbig) return;
  int i = idx / Cbig, co = idx % Cbig;
  float a = 0.f;
  for (int p = 0; p < P; ++p) a += part[((size_t)p * (SC * 9 + 1) + i) * Cbig + co];
  if (i < SC * 9) dw[(size_t)co * SC * 9 + i] = a;
  else if (db) db[co] = a;
}

// ---------------------------------------------------------------------------------------------------- big Cin -> small Cout
// ys[n,co,oy,ox] = bias[co] + sum_{ci,tap} a[n,oy+ty-1,ox+tx-1,ci] * w[(co*Cbig+ci)*9+tap]; warp per pixel, lane = channel quad
__global__ void __launch_bounds__(256) small_cout_fprop(const float* __restrict__ a, const float* __restrict__ w,
                                                        const float* __restrict__ bias, float* __restrict__ ys, EdgeGeom g) {
  extern __shared__ __align__(16) float wsm[];  // [SC][9][Cbig]
  const int t = threadIdx.x, warp = t >> 5, lane = t & 31;
  for (int i = t; i < SC * 9 * g.Cbig; i += 256) {
    int co = i / (9 * g.Cbig), tap = (i / g.Cbig) % 9, ci = i % g.Cbig;
    wsm[i] = __ldg(w + ((size_t)co * g.Cbig + ci) * 9 + tap);
  }
  __syncthreads();
  const int n = blockIdx.z, oy = blockIdx.y * ET_H + warp, x0 = blockIdx.x * ET_W;
  if (oy >= g.H) return;
  const int Q = g.Cbig >> 2;
  for (int c = 0; c < ET_W; ++c) {
    const int ox = x0 + c;
    if (ox >= g.W) break;
    float s0 = 0.f, s1 = 0.f, s2 = 0.f;
    for (int q = lane; q < Q; q += 32) {
#pragma unroll
      for (int tap = 0; tap < 9; ++tap) {
        const int iy = oy + tap / 3 - 1, ix = ox + tap % 3 - 1;
        if ((unsigned)iy < (unsigned)g.H && (unsigned)ix < (unsigned)g.W) {
          const float4 v = __ldg(reinterpret_cast<const float4*>(a + ((size_t)(n * g.H + iy) * g.W + ix) * g.Cbig) + q);
          const float4 w0 = *reinterpret_cast<const float4*>(wsm + (0 * 9 + tap) * g.Cbig + q * 4);
          const float4 w1 = *reinterpret_cast<const float4*>(wsm + (1 * 9 + tap) * g.Cbig + q * 4);
          const float4 w2 = *reinterpret_cast<const float4*>(wsm + (2 * 9 + tap) * g.Cbig + q * 4);
          s0 += v.x * w0.x + v.y * w0.y + v.z * w0.z + v.w * w0.w;
          s1 += v.x * w1.x + v.y * w1.y + v.z * w1.z + v.w * w1.w;
          s2 += v.x * w2.x + v.y * w2.y + v.z * w2.z + v.w * w2.w;
        }
      }
    }
    s0 = warp_sum(s0); s1 = warp_sum(s1); s2 = warp_sum(s2);
    if (lane < SC) {
      float v = lane == 0 ? s0 : (lane == 1 ? s1 : s2);
      ys[n * g.sn + lane * g.sc + oy * g.sh + ox * g.sw] = v + (bias ? __ldg(bias + lane) : 0.f);
    }
  }
}

// dW[co][ci][tap] = sum_p dys[n,co,p] * a[p+tap][ci]; db[co] = sum dys; thread = ci, persistent; part[block][half][27+3][Cbig]
__global__ void __launch_bounds__(256) small_cout_wgrad(const float* __restrict__ a, const float* __restrict__ dys,
                                                        float* __restrict__ part, EdgeGeom g, int tiles_x, int tiles_y, int cblk) {
  const int t = threadIdx.x, col = t & 127, half = t >> 7;
  const int ci = cblk * 128 + col;
  const bool cov = ci < g.Cbig;
  float acc[SC * 9], bs[SC];
#pragma unroll
  for (int i = 0; i < SC * 9; ++i) acc[i] = 0.f;
#pragma unroll
  for (int i = 0; i < SC; ++i) bs[i] = 0.f;
  const int64_t ntiles = (int64_t)g.N * tiles_x * tiles_y;
  for (int64_t tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
    const int tx_ = (int)(tile % tiles_x), ty_ = (int)((tile / tiles_x) % tiles_y), n = (int)(tile / ((int64_t)tiles_x * tiles_y));
    const int y0 = ty_ * ET_H, x0 = tx_ * ET_W;
    for (int r = half * (ET_H / 2); r < (half + 1) * (ET_H / 2); ++r) {
      const int oy = y0 + r;
      if (oy >= g.H) break;
      for (int c = 0; c < ET_W; ++c) {
        const int ox = x0 + c;
        if (ox >= g.W) break;
        float d[SC];
#pragma unroll
        for (int co = 0; co < SC; ++co) {
          d[co] = __ldg(dys + n * g.sn + co * g.sc + oy * g.sh + ox * g.sw);
          bs[co] += d[co];
        }
#pragma unroll
        for (int tap = 0; tap < 9; ++tap) {
          const int iy = oy + tap / 3 - 1, ix = ox + tap % 3 - 1;
          float v = 0.f;
          if (cov && (unsigned)iy < (unsigned)g.H && (unsigned)ix < (unsigned)g.W) v = __ldg(a + ((size_t)(n * g.H + iy) * g.W + ix) * g.Cbig + ci);
#pragma unroll
          for (int co = 0; co < SC; ++co) acc[co * 9 + tap] = fmaf(d[co], v, acc[co * 9 + tap]);
        }
      }
    }
  }
  if (cov) {
    float* o = part + ((size_t)(blockIdx.x * 2 + half) * (SC * 9 + SC)) * g.Cbig + ci;
#pragma unroll
    for (int i = 0; i < SC * 9; ++i) o[(size_t)i * g.Cbig] = acc[i];
#pragma unroll
    for (int i = 0; i < SC; ++i) o[(size_t)(SC * 9 + i) * g.Cbig] = bs[i];
  }
}
// part[P][30][Cbig] -> dw[co][ci][tap] (i = co*9+tap), db[co] (every channel column carries the same bias sums; take column 0's)
__global__ void small_cout_wgrad_reduce(const float* __restrict__ part, int P, int Cbig, float* __restrict__ dw, float* __restrict__ db) {
  int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= (SC * 9 + SC) * Cbig) return;
  int i = idx / Cbig, ci = idx % Cbig;
  float a = 0.f;
  for (int p = 0; p < P; ++p) a += part[((size_t)p * (SC * 9 + SC) + i) * Cbig + ci];
  if (i < SC * 9) dw[((size_t)(i / 9) * Cbig + ci) * 9 + (i % 9)] = a;
  else if (db && ci == 0) db[i - SC * 9] = a;
}

static int edge_geom(EdgeGeom& g, mas_tensor4 small, mas_tensor4 big, const char* what) {
  if (small.c != SC) return fail(MAS_ERR_UNSUPPORTED, "%s: small side must have exactly %d channels", what, SC);
  if (small.n != big.n || small.h != big.h || small.w != big.w) return fail(MAS_ERR_INVALID_ARG, "%s: extent mismatch", what);
  if (!(big.sc == 1 && big.sw == big.c && big.sh == big.w * big.c && big.sn == big.h * big.w * big.c))
    return fail(MAS_ERR_UNSUPPORTED, "%s: the wide tensor must be dense NHWC", what);
  g.N = (int)big.n; g.H = (int)big.h; g.W = (int)big.w; g.Cbig = (int)big.c;
  g.sn = small.sn; g.sh = small.sh; g.sw = small.sw; g.sc = small.sc;
  return MAS_OK;
}
constexpr int EDGE_PBLOCKS = NUM_SMS * 4;

}  // namespace mas

using namespace mas;

extern "C" {

int mas_edge_small_cin_fprop(const float* xs, mas_tensor4 xst, const float* w, const float* bias, float* y, mas_tensor4 yst,
                             int flip_transpose, void* stream) {
  EdgeGeom g;
  if (int e = edge_geom(g, xst, yst, "edge_small_cin_fprop")) return e;
  if (g.Cbig % 128 == 0) return small_cin_fprop_q_launch(xs, w, bias, y, g, flip_transpose, S(stream));
  dim3 grid((unsigned)cdiv(g.W, ET_W), (unsigned)cdiv(g.H, ET_H), (unsigned)(g.N * cdiv(g.Cbig, 128)));
  small_cin_fprop<<<grid, 256, 0, S(stream)>>>(xs, w, bias, y, g, flip_transpose);
  return launched("small_cin_fprop");
}

size_t mas_edge_wgrad_ws_bytes(int Cbig) { return (size_t)EDGE_PBLOCKS * 2 * (SC * 9 + SC) * Cbig * sizeof(float) + 256; }

int mas_edge_small_cin_wgrad(const float* xs, mas_tensor4 xst, const float* dy, mas_tensor4 dyt, float* dw, float* dbias, void* ws,
                             size_t ws_bytes, void* stream) {
  EdgeGeom g;
  if (int e = edge_geom(g, xst, dyt, "edge_small_cin_wgrad")) return e;
  if (ws_bytes < mas_edge_wgrad_ws_bytes(g.Cbig)) return fail(MAS_ERR_WORKSPACE, "edge wgrad: workspace too small");
  if (g.Cbig % 128 == 0) {
    if (int e = small_cin_wgrad_q_launch(xs, dy, (float*)ws, g, S(stream))) return e;
    small_cin_wgrad_reduce<<<(int)cdiv((SC * 9 + 1) * g.Cbig, 128), 128, 0, S(stream)>>>((const float*)ws, EDGE_Q_BLOCKS, g.Cbig, dw, dbias);
    return launched("small_cin_wgrad_reduce");
  }
  const int tx = (int)cdiv(g.W, ET_W), ty = (int)cdiv(g.H, ET_H);
  const int64_t ntiles = (int64_t)g.N * tx * ty;
  const int blocks = (int)(ntiles < EDGE_PBLOCKS ? ntiles : EDGE_PBLOCKS);
  for (int cb = 0; cb < (int)cdiv(g.Cbig, 128); ++cb) {
    small_cin_wgrad<<<blocks, 256, 0, S(stream)>>>(xs, dy, (float*)ws, g, tx, ty, cb);
    if (int e = launched("small_cin_wgrad")) return e;
  }
  small_cin_wgrad_reduce<<<(int)cdiv((SC * 9 + 1) * g.Cbig, 128), 128, 0, S(stream)>>>((const float*)ws, blocks * 2, g.Cbig, dw, dbias);
  return launched("small_cin_wgrad_reduce");
}

int mas_edge_small_cout_fprop(const float* a, mas_tensor4 at, const float* w, const float* bias, float* ys, mas_tensor4 yst,
                              void* stream) {
  EdgeGeom g;
  if (int e = edge_geom(g, yst, at, "edge_small_cout_fprop")) return e;
  if (g.Cbig == 128) return small_cout_fprop_q_launch(a, w, bias, ys, g, S(stream));
  if (g.Cbig % 4) return fail(MAS_ERR_UNSUPPORTED, "edge_small_cout_fprop: Cin %% 4 != 0");
  size_t smem = (size_t)SC * 9 * g.Cbig * sizeof(float);
  if (smem > 48 * 1024) return fail(MAS_ERR_UNSUPPORTED, "edge_small_cout_fprop: Cin=%d too wide", g.Cbig);
  dim3 grid((unsigned)cdiv(g.W, ET_W), (unsigned)cdiv(g.H, ET_H), (unsigned)g.N);
  small_cout_fprop<<<grid, 256, smem, S(stream)>>>(a, w, bias, ys, g);
  return launched("small_cout_fprop");
}

int mas_edge_small_cout_wgrad(const float* a, mas_tensor4 at, const float* dys, mas_tensor4 dyt, float* dw, float* dbias, void* ws,
                              size_t ws_bytes, void* stream) {
  EdgeGeom g;
  if (int e = edge_geom(g, dyt, at, "edge_small_cout_wgrad")) return e;
  if (ws_bytes < mas_edge_wgrad_ws_bytes(g.Cbig)) return fail(MAS_ERR_WORKSPACE, "edge wgrad: workspace too small");
  if (g.Cbig % 128 == 0) {
    if (int e = small_cout_wgrad_q_launch(a, dys, (float*)ws, g, S(stream))) return e;
    small_cout_wgrad_reduce<<<(int)cdiv((SC * 9 + SC) * g.Cbig, 128), 128, 0, S(stream)>>>((const float*)ws, EDGE_Q_BLOCKS, g.Cbig, dw, dbias);
    return launched("small_cout_wgrad_reduce");
  }
  const int tx = (int)cdiv(g.W, ET_W), ty = (int)cdiv(g.H, ET_H);
  const int64_t ntiles = (int64_t)g.N * tx * ty;
  const int blocks = (int)(ntiles < EDGE_PBLOCKS ? ntiles : EDGE_PBLOCKS);
  for (int cb = 0; cb < (int)cdiv(g.Cbig, 128); ++cb) {
    small_cout_wgrad<<<blocks, 256, 0, S(stream)>>>(a, dys, (float*)ws, g, tx, ty, cb);
    if (int e = launched("small_cout_wgrad")) return e;
  }
  small_cout_wgrad_reduce<<<(int)cdiv((SC * 9 + SC) * g.Cbig, 128), 128, 0, S(stream)>>>((const float*)ws, blocks * 2, g.Cbig, dw, dbias);
  return launched("small_cout_wgrad_reduce");
}

}  // extern "C"

// ---------------------------------------------------------------------------------------------------- stride-2 conv via space-to-depth
// Downsample (modules.py:74-78) = pad(0,1,0,1) + conv3x3 stride 2.  With X4[n,i,j,(py,px,c)] = x[n,2i+py,2j+px,c] the
// stride-2 gather becomes a unit-stride 2x2-tap convolution over 4C channels, which the wgmma stride-1 kernels run as a
// 3x3 convolution whose other five taps are zero:  y[o] = sum_{a,b in {0,1}} X4[o+(a,b)] . W9[(a+1,b+1)],
// W9[(a+1,b+1)][(py,px,c)] = W[2a+py][2b+px][c] (0 where 2a+py or 2b+px exceeds 2).  Zero padding beyond the last X4
// row/column is exactly the reference's bottom/right pad.
namespace mas {
__global__ void space_to_depth_kernel(const float* __restrict__ x, float* __restrict__ y, int H, int W, int C4, int64_t total4) {
  // x [N,H,W,C] -> y [N,H/2,W/2,4C], channel block (py*2+px)
  const int Ho = H >> 1, Wo = W >> 1;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total4; i += (int64_t)gridDim.x * blockDim.x) {
    int c = (int)(i % C4);
    int64_t r = i / C4;
    int ph = (int)(r % 4); r /= 4;
    int j = (int)(r % Wo); r /= Wo;
    int ii = (int)(r % Ho);
    int64_t n = r / Ho;
    const float4 v = __ldg(reinterpret_cast<const float4*>(x) + (((n * H + 2 * ii + (ph >> 1)) * W + 2 * j + (ph & 1)) * C4 + c));
    reinterpret_cast<float4*>(y)[i] = v;
  }
}
// W [Cout][C][3][3] -> W9 [Cout][4C][3][3]
__global__ void s2d_pack_weights(const float* __restrict__ w, float* __restrict__ w9, int Cout, int C) {
  int64_t total = (int64_t)Cout * 4 * C * 9;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int tap = (int)(i % 9);
    int64_t r = i / 9;
    int cc = (int)(r % (4 * C));
    int co = (int)(r / (4 * C));
    int ph = cc / C, c = cc % C, py = ph >> 1, px = ph & 1;
    int a = tap / 3 - 1, b = tap % 3 - 1;  // offsets of the 3x3 tap; only a,b in {0,1} carry weight
    float v = 0.f;
    if (a >= 0 && b >= 0) {
      int ty = 2 * a + py, tx = 2 * b + px;
      if (ty <= 2 && tx <= 2) v = w[((size_t)co * C + c) * 9 + ty * 3 + tx];
    }
    w9[i] = v;
  }
}
// dW9 [Cout][4C][3][3] -> dW [Cout][C][3][3]
__global__ void s2d_unpack_wgrad(const float* __restrict__ dw9, float* __restrict__ dw, int Cout, int C) {
  int64_t total = (int64_t)Cout * C * 9;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int t = (int)(i % 9);
    int64_t r = i / 9;
    int c = (int)(r % C), co = (int)(r / C);
    int ty = t / 3, tx = t % 3, a = ty >> 1, py = ty & 1, b = tx >> 1, px = tx & 1;
    dw[i] = dw9[((size_t)co * 4 * C + (py * 2 + px) * C + c) * 9 + (a + 1) * 3 + (b + 1)];
  }
}
}  // namespace mas

extern "C" {
int mas_space_to_depth(const float* x, float* y, int N, int H, int W, int C, void* stream) {
  if (C % 4 || H % 2 || W % 2) return fail(MAS_ERR_UNSUPPORTED, "space_to_depth: needs C %% 4 == 0 and even H, W");
  int64_t total4 = (int64_t)N * H * W * (C / 4);
  int grid = (int)(cdiv(total4, 256) < NUM_SMS * 16 ? cdiv(total4, 256) : NUM_SMS * 16);
  space_to_depth_kernel<<<grid, 256, 0, S(stream)>>>(x, y, H, W, C / 4, total4);
  return launched("space_to_depth");
}
int mas_s2d_pack_weights(const float* w, float* w9, int Cout, int C, void* stream) {
  int64_t total = (int64_t)Cout * 4 * C * 9;
  s2d_pack_weights<<<(int)(cdiv(total, 256) < 2368 ? cdiv(total, 256) : 2368), 256, 0, S(stream)>>>(w, w9, Cout, C);
  return launched("s2d_pack_weights");
}
int mas_s2d_unpack_wgrad(const float* dw9, float* dw, int Cout, int C, void* stream) {
  int64_t total = (int64_t)Cout * C * 9;
  s2d_unpack_wgrad<<<(int)(cdiv(total, 256) < 2368 ? cdiv(total, 256) : 2368), 256, 0, S(stream)>>>(dw9, dw, Cout, C);
  return launched("s2d_unpack_wgrad");
}
}
