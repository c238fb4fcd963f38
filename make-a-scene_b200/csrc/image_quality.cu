// Reconstruction quality of images on the device: per-image PSNR and SSIM of rec against ref (mas_image_quality).  The
// definition is stated in include/mas_b200.h and DESIGN §3.9.2.
//
// One CTA owns a TH x TW tile of output pixels of one (image, channel).  It loads the tile and its 5-pixel halo of both images
// through the strides into shared memory once (clamped to [-1, 1] and mapped to [0, 1]), runs the 11-tap Gaussian along rows
// over the five products x, y, x^2, y^2, xy, then along columns, and evaluates the SSIM map at the tile's pixels whose 11 x 11
// window lies inside the image.  The squared error is summed over the tile's own pixels (no halo) in the load loop.  Each CTA
// reduces its two sums in a fixed order into one fp64 pair of the workspace; a second kernel adds each image's pairs in a fixed
// order.  No floating-point atomics: the result depends only on the values, not on the strides or the schedule.
//
// The second moments are taken about the tile's mean (a per-tile shift s, the fp32 mean of the tile's own mapped pixels):
// sigma^2 = G*(x-s)^2 - (G*(x-s))^2.  Raw fp32 moments G*x^2 - mu^2 cancel on flat regions down to ~1e-7, which C2 = 9e-4
// turns into SSIM errors of ~1e-4; about the tile mean a constant tile has exactly zero moments.
#include <cuda_runtime.h>

#include <math.h>

#include "mas_common.cuh"

namespace mas {
namespace iq {

constexpr int R = 5, K = 2 * R + 1;           // window radius and taps
constexpr int TW = 32, TH = 32;               // output tile: one column per lane, 4 rows per warp
constexpr int PW = TW + 2 * R, PH = TH + 2 * R;
constexpr int THREADS = 256, WARPS = THREADS / 32, RPT = TH / WARPS;   // rows per thread in the vertical pass
constexpr float C1 = 0.01f * 0.01f, C2 = 0.03f * 0.03f;
static_assert(RPT * WARPS == TH && TW == 32, "tile layout");

struct Taps {
  float w[K];
};

// Clamp to [-1, 1] without fminf / fmaxf, which would turn a NaN into a bound: a NaN fails both comparisons and stays NaN.
__device__ __forceinline__ float clamp1(float v) { return v < -1.f ? -1.f : (v > 1.f ? 1.f : v); }

__device__ __forceinline__ double block_sum(double v, double* red) {
  // fixed order: xor butterfly within each warp, then warp 0 adds the warps' sums in warp order
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  double t = 0.0;
  for (int i = 0; i < WARPS; ++i) t += red[i];
  return t;
}

__global__ void __launch_bounds__(THREADS) tile_kernel(const float* __restrict__ rec, mas_tensor4 rs, const float* __restrict__ ref,
                                                       mas_tensor4 fs, Taps taps, int tiles_x, double* __restrict__ part) {
  __shared__ float sx[PH][PW], sy[PH][PW];
  __shared__ float hb[5][PH][TW];   // row-filtered x, y, x^2, y^2, xy (about the tile's shifts)
  __shared__ double red[WARPS];
  __shared__ float shift[2];
  const int tile = blockIdx.x, c = blockIdx.y, b = blockIdx.z;
  const int64_t H = rs.h, W = rs.w;
  const int64_t y0 = (int64_t)(tile / tiles_x) * TH, x0 = (int64_t)(tile % tiles_x) * TW;
  const float* pr = rec + b * rs.sn + c * rs.sc;
  const float* pf = ref + b * fs.sn + c * fs.sc;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;

  // load tile + halo (0 outside the image: those values only reach windows that are not evaluated), the squared error and
  // the sums of the tile's own pixels
  double sq = 0.0;
  float ox = 0.f, oy = 0.f;
  for (int i = threadIdx.x; i < PH * PW; i += THREADS) {
    const int r = i / PW, q = i - r * PW;
    const int64_t gy = y0 - R + r, gx = x0 - R + q;
    float vx = 0.f, vy = 0.f;
    if (gy >= 0 && gy < H && gx >= 0 && gx < W) {
      const float a = clamp1(__ldg(pr + gy * rs.sh + gx * rs.sw)), e = clamp1(__ldg(pf + gy * fs.sh + gx * fs.sw));
      vx = __fmul_rn(__fadd_rn(a, 1.f), 0.5f);
      vy = __fmul_rn(__fadd_rn(e, 1.f), 0.5f);
      if (r >= R && r < R + TH && q >= R && q < R + TW) {
        const double d = 0.5 * (double)__fsub_rn(a, e);   // (a + 1) / 2 - (e + 1) / 2 with one rounding
        sq += d * d;
        ox += vx;
        oy += vy;
      }
    }
    sx[r][q] = vx;
    sy[r][q] = vy;
  }
  const int64_t own_h = min((int64_t)TH, H - y0), own_w = min((int64_t)TW, W - x0);
  {
    const float tx = warp_sum(ox), ty = warp_sum(oy);
    __shared__ float wsum[2][WARPS];
    if (lane == 0) wsum[0][warp] = tx, wsum[1][warp] = ty;
    __syncthreads();
    if (threadIdx.x < 2) {
      float t = 0.f;
      for (int k = 0; k < WARPS; ++k) t += wsum[threadIdx.x][k];
      shift[threadIdx.x] = t / (float)(own_h * own_w);
    }
    __syncthreads();
  }
  // valid centres of this tile: 5 <= gy <= H - 6, 5 <= gx <= W - 6
  const int64_t vy0 = max(y0, (int64_t)R), vy1 = min(y0 + TH, H - R), vx0 = max(x0, (int64_t)R), vx1 = min(x0 + TW, W - R);
  double ss = 0.0;
  if (vy0 < vy1 && vx0 < vx1) {   // uniform across the block
    const float hx = shift[0], hy = shift[1];
    for (int i = threadIdx.x; i < PH * PW; i += THREADS) {
      float* px = &sx[0][0] + i;
      float* py = &sy[0][0] + i;
      *px = __fsub_rn(*px, hx);
      *py = __fsub_rn(*py, hy);
    }
    __syncthreads();
    for (int r = warp; r < PH; r += WARPS) {
      float a[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
#pragma unroll
      for (int k = 0; k < K; ++k) {
        const float x = sx[r][lane + k], y = sy[r][lane + k], w = taps.w[k];
        a[0] = __fmaf_rn(w, x, a[0]);
        a[1] = __fmaf_rn(w, y, a[1]);
        a[2] = __fmaf_rn(w, __fmul_rn(x, x), a[2]);
        a[3] = __fmaf_rn(w, __fmul_rn(y, y), a[3]);
        a[4] = __fmaf_rn(w, __fmul_rn(x, y), a[4]);
      }
#pragma unroll
      for (int p = 0; p < 5; ++p) hb[p][r][lane] = a[p];
    }
    __syncthreads();
    float m[5][RPT];
#pragma unroll
    for (int p = 0; p < 5; ++p) {
#pragma unroll
      for (int i = 0; i < RPT; ++i) m[p][i] = 0.f;
#pragma unroll
      for (int t = 0; t < RPT + K - 1; ++t) {
        const float v = hb[p][warp * RPT + t][lane];
#pragma unroll
        for (int i = 0; i < RPT; ++i)
          if (t - i >= 0 && t - i < K) m[p][i] = __fmaf_rn(taps.w[t - i], v, m[p][i]);
      }
    }
    const int64_t gx = x0 + lane;
#pragma unroll
    for (int i = 0; i < RPT; ++i) {
      const int64_t gy = y0 + warp * RPT + i;
      if (gy >= vy0 && gy < vy1 && gx >= vx0 && gx < vx1) {
        // explicit roundings: with rec == ref every pair of terms below is bitwise equal, so the map is exactly 1
        const float a = m[0][i], e = m[1][i];
        const float mx = __fadd_rn(hx, a), my = __fadd_rn(hy, e);
        const float vx = __fsub_rn(m[2][i], __fmul_rn(a, a)), vy = __fsub_rn(m[3][i], __fmul_rn(e, e));
        const float cxy = __fsub_rn(m[4][i], __fmul_rn(a, e));
        const float ln = __fadd_rn(__fmul_rn(2.f, __fmul_rn(mx, my)), C1);
        const float ld = __fadd_rn(__fadd_rn(__fmul_rn(mx, mx), __fmul_rn(my, my)), C1);
        const float cn = __fadd_rn(__fmul_rn(2.f, cxy), C2);
        const float cd = __fadd_rn(__fadd_rn(vx, vy), C2);
        ss += (double)__fdiv_rn(__fmul_rn(ln, cn), __fmul_rn(ld, cd));
      }
    }
  }
  sq = block_sum(sq, red);
  ss = block_sum(ss, red);
  if (threadIdx.x == 0) {
    double* o = part + 2 * (((int64_t)b * gridDim.y + c) * gridDim.x + tile);
    o[0] = sq;
    o[1] = ss;
  }
}

// One block per image: its C * tiles pairs, strided over the threads and then reduced in a fixed tree.
__global__ void __launch_bounds__(THREADS) finalize_kernel(const double* __restrict__ part, int64_t per_image, double n_all,
                                                           double n_valid, float* __restrict__ psnr, float* __restrict__ ssim) {
  __shared__ double red[WARPS];
  const int b = blockIdx.x;
  const double* p = part + 2 * (int64_t)b * per_image;
  double sq = 0.0, ss = 0.0;
  for (int64_t i = threadIdx.x; i < per_image; i += THREADS) {
    sq += p[2 * i];
    ss += p[2 * i + 1];
  }
  sq = block_sum(sq, red);
  ss = block_sum(ss, red);
  if (threadIdx.x == 0) {
    psnr[b] = (float)(-10.0 * log10(sq / n_all));   // mse = 0 -> +inf, NaN stays NaN
    ssim[b] = (float)(ss / n_valid);
  }
}

static inline int64_t tiles_of(int64_t H, int64_t W) { return cdiv(H, TH) * cdiv(W, TW); }

}  // namespace iq
}  // namespace mas

using namespace mas;
using namespace mas::iq;

extern "C" {

size_t mas_image_quality_ws_bytes(int B, int C, int64_t H, int64_t W) {
  if (B < 1 || C < 1 || H < K || W < K) return 0;
  return (size_t)B * (size_t)C * (size_t)tiles_of(H, W) * 2 * sizeof(double);
}

int mas_image_quality(const float* rec, mas_tensor4 rs, const float* ref, mas_tensor4 fs, float* psnr, float* ssim, void* ws,
                      size_t ws_bytes, void* stream) {
  MAS_REQUIRE(rec && ref && psnr && ssim && ws, "image_quality: null pointer");
  MAS_REQUIRE(rs.n >= 1 && rs.c >= 1 && rs.h >= K && rs.w >= K,
              "image_quality: need B, C >= 1 and H, W >= 11, got [%lld, %lld, %lld, %lld]", (long long)rs.n, (long long)rs.c,
              (long long)rs.h, (long long)rs.w);
  MAS_REQUIRE(fs.n == rs.n && fs.c == rs.c && fs.h == rs.h && fs.w == rs.w, "image_quality: rec and ref differ in shape");
  MAS_REQUIRE(rs.n <= 65535 && rs.c <= 65535 && tiles_of(rs.h, rs.w) <= INT32_MAX, "image_quality: extents over the grid limits");
  const int B = (int)rs.n, C = (int)rs.c;
  MAS_REQUIRE(ws_bytes >= mas_image_quality_ws_bytes(B, C, rs.h, rs.w), "image_quality: workspace too small");
  // the Gaussian window: sigma 1.5, normalised in fp64, rounded once to fp32
  Taps taps;
  double g[K], sum = 0.0;
  for (int k = 0; k < K; ++k) sum += (g[k] = exp(-(double)((k - R) * (k - R)) / (2.0 * 1.5 * 1.5)));
  for (int k = 0; k < K; ++k) taps.w[k] = (float)(g[k] / sum);
  const int tiles_x = (int)cdiv(rs.w, TW);
  const int64_t tiles = tiles_of(rs.h, rs.w);
  double* part = static_cast<double*>(ws);
  tile_kernel<<<dim3((unsigned)tiles, (unsigned)C, (unsigned)B), THREADS, 0, S(stream)>>>(rec, rs, ref, fs, taps, tiles_x, part);
  if (const int e = launched("image_quality_tiles")) return e;
  finalize_kernel<<<B, THREADS, 0, S(stream)>>>(part, C * tiles, (double)C * rs.h * rs.w, (double)C * (rs.h - 2 * R) * (rs.w - 2 * R),
                                                psnr, ssim);
  return launched("image_quality_finalize");
}

}  // extern "C"
