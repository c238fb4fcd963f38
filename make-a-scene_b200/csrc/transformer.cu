// Tier-2 token transformer (reference models/transformer.py): LayerNorm (+fused residual add, the sandwich-LN
// pattern of transformer.py:176-210), tanh-GELU (transformer.py:11-14), causal softmax (transformer.py:57-71,90 — the
// PB-relax shift is softmax-invariant and the -10000 fill underflows to exactly 0 in fp32, so this is plain causal
// softmax), fused token + row/column position embedding gather (transformer.py:329-364).  Linear layers and the
// attention contractions reuse the GEMM kernels (contract_tc.cu / contract_simt.cu).  fp32 throughout.
#include "mas_common.cuh"

namespace mas {

// ---------------------------------------------------------------------------------------------------- LayerNorm, few rows
// Decode steps normalise 2-8 rows: a warp per row walks H = 1024 in 32 dependent trips per pass (13 us measured). Here a
// 256-thread block owns one row, keeps it in registers (up to four 16-byte quads per thread: H <= 4096), and needs two
// block reductions; same two-pass statistics (mean, then centred sum of squares) as the warp-per-row kernel.
__global__ void __launch_bounds__(256) layernorm_fwd_block_kernel(const float* __restrict__ x, const float* __restrict__ gamma,
                                                                  const float* __restrict__ beta, const float* __restrict__ res,
                                                                  float* __restrict__ y, float* __restrict__ mean,
                                                                  float* __restrict__ rstd, int H, float eps) {
  __shared__ float red[2][8];
  const int64_t row = blockIdx.x;
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5, Q = H >> 2;
  const float4* xr = reinterpret_cast<const float4*>(x + row * H);
  float4 v[4];
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int q = t + 256 * i;
    v[i] = q < Q ? __ldg(xr + q) : make_float4(0.f, 0.f, 0.f, 0.f);
    s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
  }
  s = warp_sum(s);
  if (lane == 0) red[0][warp] = s;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) tot += red[0][w];
  const float m = tot / (float)H;
  float qd = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i)
    if (t + 256 * i < Q) {
      const float a = v[i].x - m, b = v[i].y - m, c = v[i].z - m, d = v[i].w - m;
      qd = fmaf(a, a, qd); qd = fmaf(b, b, qd); qd = fmaf(c, c, qd); qd = fmaf(d, d, qd);
    }
  qd = warp_sum(qd);
  if (lane == 0) red[1][warp] = qd;
  __syncthreads();
  float tq = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) tq += red[1][w];
  const float rs = rsqrtf(tq / (float)H + eps);
  const float4* g4 = reinterpret_cast<const float4*>(gamma);
  const float4* b4 = reinterpret_cast<const float4*>(beta);
  const float4* r4 = res ? reinterpret_cast<const float4*>(res + row * H) : nullptr;
  float4* y4 = reinterpret_cast<float4*>(y + row * H);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int q = t + 256 * i;
    if (q < Q) {
      const float4 g = __ldg(g4 + q), b = __ldg(b4 + q);
      float4 o = make_float4((v[i].x - m) * rs * g.x + b.x, (v[i].y - m) * rs * g.y + b.y, (v[i].z - m) * rs * g.z + b.z,
                             (v[i].w - m) * rs * g.w + b.w);
      if (r4) {
        const float4 r = __ldg(r4 + q);
        o.x += r.x; o.y += r.y; o.z += r.z; o.w += r.w;
      }
      y4[q] = o;
    }
  }
  if (t == 0) {
    mean[row] = m;
    rstd[row] = rs;
  }
}

// Two chained LayerNorms of a decode step in one launch (inference): y1 = res + LN1(x) (the sandwich LayerNorm with its
// residual, transformer.py:183-208; res may be null) and y2 = LN2(y1) (the next sub-layer's input norm / final_ln).  Same
// row-in-registers scheme and the same two-pass statistics as layernorm_fwd_block_kernel, applied twice.
__device__ __forceinline__ void ln_row_stats_256(const float4 (&v)[4], int Q, int H, float eps, float (*red)[8], float* m_out, float* rs_out) {
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) s += (v[i].x + v[i].y) + (v[i].z + v[i].w);
  s = warp_sum(s);
  if (lane == 0) red[0][warp] = s;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) tot += red[0][w];
  const float m = tot / (float)H;
  float qd = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i)
    if (t + 256 * i < Q) {
      const float a = v[i].x - m, b = v[i].y - m, c = v[i].z - m, d = v[i].w - m;
      qd = fmaf(a, a, qd); qd = fmaf(b, b, qd); qd = fmaf(c, c, qd); qd = fmaf(d, d, qd);
    }
  qd = warp_sum(qd);
  if (lane == 0) red[1][warp] = qd;
  __syncthreads();
  float tq = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) tq += red[1][w];
  *m_out = m;
  *rs_out = rsqrtf(tq / (float)H + eps);
  __syncthreads();      // red[] is reused by the second normalisation
}
__global__ void __launch_bounds__(256) layernorm2_fwd_block_kernel(const float* __restrict__ x, const float* __restrict__ g1,
                                                                   const float* __restrict__ b1, const float* __restrict__ res,
                                                                   float* __restrict__ y1, const float* __restrict__ g2,
                                                                   const float* __restrict__ b2, float* __restrict__ y2, int H, float eps1,
                                                                   float eps2) {
  __shared__ float red[2][8];
  const int64_t row = blockIdx.x;
  const int t = threadIdx.x, Q = H >> 2;
  const float4* xr = reinterpret_cast<const float4*>(x + row * H);
  float4 v[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int q = t + 256 * i;
    v[i] = q < Q ? __ldg(xr + q) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  float m, rs;
  ln_row_stats_256(v, Q, H, eps1, red, &m, &rs);
  const float4* r4 = res ? reinterpret_cast<const float4*>(res + row * H) : nullptr;
  float4* o1 = reinterpret_cast<float4*>(y1 + row * H);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int q = t + 256 * i;
    if (q < Q) {
      const float4 g = __ldg(reinterpret_cast<const float4*>(g1) + q), b = __ldg(reinterpret_cast<const float4*>(b1) + q);
      float4 o = make_float4((v[i].x - m) * rs * g.x + b.x, (v[i].y - m) * rs * g.y + b.y, (v[i].z - m) * rs * g.z + b.z,
                             (v[i].w - m) * rs * g.w + b.w);
      if (r4) {
        const float4 r = __ldg(r4 + q);
        o.x += r.x; o.y += r.y; o.z += r.z; o.w += r.w;
      }
      o1[q] = o;
      v[i] = o;
    } else {
      v[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
  ln_row_stats_256(v, Q, H, eps2, red, &m, &rs);
  float4* o2 = reinterpret_cast<float4*>(y2 + row * H);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int q = t + 256 * i;
    if (q < Q) {
      const float4 g = __ldg(reinterpret_cast<const float4*>(g2) + q), b = __ldg(reinterpret_cast<const float4*>(b2) + q);
      o2[q] = make_float4((v[i].x - m) * rs * g.x + b.x, (v[i].y - m) * rs * g.y + b.y, (v[i].z - m) * rs * g.z + b.z,
                          (v[i].w - m) * rs * g.w + b.w);
    }
  }
}

// ---------------------------------------------------------------------------------------------------- LayerNorm (warp per row)
__global__ void layernorm_fwd_kernel(const float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
                                     const float* __restrict__ res, float* __restrict__ y, float* __restrict__ mean,
                                     float* __restrict__ rstd, int64_t R, int H, float eps) {
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= R) return;
  const int lane = threadIdx.x & 31;
  const float* xr = x + row * H;
  float s = 0.f;
  for (int c = lane; c < H; c += 32) s += xr[c];
  const float m = warp_sum(s) / (float)H;
  float q = 0.f;
  for (int c = lane; c < H; c += 32) {
    float d = xr[c] - m;
    q = fmaf(d, d, q);
  }
  const float rs = rsqrtf(warp_sum(q) / (float)H + eps);
  for (int c = lane; c < H; c += 32) {
    float o = (xr[c] - m) * rs * gamma[c] + beta[c];
    if (res) o += res[row * H + c];
    y[row * H + c] = o;
  }
  if (lane == 0) {
    mean[row] = m;
    rstd[row] = rs;
  }
}

__global__ void layernorm_bwd_dx_kernel(const float* __restrict__ dy, const float* __restrict__ x, const float* __restrict__ mean,
                                        const float* __restrict__ rstd, const float* __restrict__ gamma, float* __restrict__ dx,
                                        int64_t R, int H) {
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= R) return;
  const int lane = threadIdx.x & 31;
  const float m = mean[row], rs = rstd[row];
  const float* xr = x + row * H;
  const float* dr = dy + row * H;
  float a = 0.f, b = 0.f;
  for (int c = lane; c < H; c += 32) {
    float g = dr[c] * gamma[c], xh = (xr[c] - m) * rs;
    a = fmaf(g, xh, a);
    b += g;
  }
  a = warp_sum(a) / (float)H;
  b = warp_sum(b) / (float)H;
  for (int c = lane; c < H; c += 32) {
    float g = dr[c] * gamma[c], xh = (xr[c] - m) * rs;
    dx[row * H + c] = rs * (g - b - xh * a);
  }
}

// Block-per-row form for H <= 4096 (the row's dy and x stay in registers: one pass over global memory instead of three
// dependent warp-strided passes; the warp-per-row kernel above walked H = 1024 in 32 trips per pass).
__global__ void __launch_bounds__(256) layernorm_bwd_dx_block_kernel(const float* __restrict__ dy, const float* __restrict__ x,
                                                                     const float* __restrict__ mean, const float* __restrict__ rstd,
                                                                     const float* __restrict__ gamma, float* __restrict__ dx, int H) {
  __shared__ float red[2][8];
  const int64_t row = blockIdx.x;
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5, Q = H >> 2;
  const float m = mean[row], rs = rstd[row];
  const float4* dr = reinterpret_cast<const float4*>(dy + row * H);
  const float4* xr = reinterpret_cast<const float4*>(x + row * H);
  const float4* g4 = reinterpret_cast<const float4*>(gamma);
  float4 g[4], xh[4];
  float a = 0.f, b = 0.f;
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int q = t + 256 * i;
    if (q < Q) {
      const float4 d = __ldg(dr + q), xv = __ldg(xr + q), gm = __ldg(g4 + q);
      g[i] = make_float4(d.x * gm.x, d.y * gm.y, d.z * gm.z, d.w * gm.w);
      xh[i] = make_float4((xv.x - m) * rs, (xv.y - m) * rs, (xv.z - m) * rs, (xv.w - m) * rs);
      a = fmaf(g[i].x, xh[i].x, a); a = fmaf(g[i].y, xh[i].y, a); a = fmaf(g[i].z, xh[i].z, a); a = fmaf(g[i].w, xh[i].w, a);
      b += (g[i].x + g[i].y) + (g[i].z + g[i].w);
    } else {
      g[i] = xh[i] = make_float4(0.f, 0.f, 0.f, 0.f);
    }
  }
  a = warp_sum(a);
  b = warp_sum(b);
  if (lane == 0) { red[0][warp] = a; red[1][warp] = b; }
  __syncthreads();
  float ta = 0.f, tb = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) { ta += red[0][w]; tb += red[1][w]; }
  ta /= (float)H;
  tb /= (float)H;
  float4* o4 = reinterpret_cast<float4*>(dx + row * H);
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int q = t + 256 * i;
    if (q < Q)
      o4[q] = make_float4(rs * (g[i].x - tb - xh[i].x * ta), rs * (g[i].y - tb - xh[i].y * ta), rs * (g[i].z - tb - xh[i].z * ta),
                          rs * (g[i].w - tb - xh[i].w * ta));
  }
}

// column sums for dgamma / dbeta: block (32,8) per 32-column tile and row chunk; deterministic two-stage
constexpr int LN_ROWS = 128;    // rows per partial block: 5120 rows x 1024 columns -> 32 x 40 blocks (1024 rows per block left 160 blocks for 132 SMs)
__global__ void layernorm_bwd_param_partial(const float* __restrict__ dy, const float* __restrict__ x, const float* __restrict__ mean,
                                            const float* __restrict__ rstd, int64_t R, int H, double* __restrict__ part) {
  __shared__ double sh[8][32][2];
  const int c = blockIdx.x * 32 + threadIdx.x;
  const int64_t r0 = (int64_t)blockIdx.y * LN_ROWS, r1 = min(R, r0 + LN_ROWS);
  double a = 0, b = 0;
  if (c < H)
    for (int64_t r = r0 + threadIdx.y; r < r1; r += 8) {
      float d = dy[r * H + c];
      a += (double)d * ((x[r * H + c] - mean[r]) * rstd[r]);
      b += d;
    }
  sh[threadIdx.y][threadIdx.x][0] = a;
  sh[threadIdx.y][threadIdx.x][1] = b;
  __syncthreads();
  if (threadIdx.y == 0 && c < H) {
    for (int k = 1; k < 8; ++k) {
      a += sh[k][threadIdx.x][0];
      b += sh[k][threadIdx.x][1];
    }
    part[((size_t)blockIdx.y * H + c) * 2] = a;
    part[((size_t)blockIdx.y * H + c) * 2 + 1] = b;
  }
}
__global__ void layernorm_bwd_param_final(const double* __restrict__ part, int chunks, int H, float* __restrict__ dgamma,
                                          float* __restrict__ dbeta) {
  int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= H) return;
  double a = 0, b = 0;
  for (int k = 0; k < chunks; ++k) {
    a += part[((size_t)k * H + c) * 2];
    b += part[((size_t)k * H + c) * 2 + 1];
  }
  dgamma[c] = (float)a;
  dbeta[c] = (float)b;
}

// ---------------------------------------------------------------------------------------------------- GELU (tanh form)
__device__ __forceinline__ float gelu_f(float x) { return 0.5f * x * (1.0f + tanhf(0.7978845608028654f * x * (1.0f + 0.044715f * x * x))); }
__global__ void gelu_fwd_kernel(const float* __restrict__ x, float* __restrict__ y, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) y[i] = gelu_f(x[i]);
}
__global__ void gelu_bwd_kernel(const float* __restrict__ dy, const float* __restrict__ x, float* __restrict__ dx, int64_t n) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    float v = x[i];
    float u = 0.7978845608028654f * v * (1.0f + 0.044715f * v * v);
    float t = tanhf(u);
    float du = 0.7978845608028654f * (1.0f + 3.0f * 0.044715f * v * v);
    dx[i] = dy[i] * (0.5f * (1.0f + t) + 0.5f * v * (1.0f - t * t) * du);
  }
}

// ---------------------------------------------------------------------------------------------------- causal softmax (warp per row)
__global__ void softmax_causal_kernel(const float* __restrict__ s, float* __restrict__ p, int64_t total_rows, int rows, int cols) {
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= total_rows) return;
  const int lane = threadIdx.x & 31;
  const int i = (int)(row % rows), lim = i + (cols - rows);  // columns 0..lim are visible
  const float* sr = s + row * cols;
  float* pr = p + row * cols;
  float mx = -INFINITY;
  for (int c = lane; c <= lim; c += 32) mx = fmaxf(mx, sr[c]);
  mx = warp_max(mx);
  float sum = 0.f;
  for (int c = lane; c <= lim; c += 32) sum += expf(sr[c] - mx);
  const float inv = 1.0f / warp_sum(sum);
  for (int c = lane; c < cols; c += 32) pr[c] = c <= lim ? expf(sr[c] - mx) * inv : 0.f;
}

__global__ void softmax_causal_bwd_kernel(const float* __restrict__ p, const float* __restrict__ dp, float* __restrict__ ds,
                                          int64_t total_rows, int rows, int cols, float scale) {
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= total_rows) return;
  const int lane = threadIdx.x & 31;
  const int i = (int)(row % rows), lim = i + (cols - rows);  // columns 0..lim are visible
  const float* pr = p + row * cols;
  const float* dr = dp + row * cols;
  float dot = 0.f;
  for (int c = lane; c <= lim; c += 32) dot += pr[c] * dr[c];
  dot = warp_sum(dot);
  for (int c = lane; c < cols; c += 32) ds[row * cols + c] = c <= lim ? pr[c] * (dr[c] - dot) * scale : 0.f;
}

// ---------------------------------------------------------------------------------------------------- embeddings
// out[(r/seg)*total + off + r%seg][:] = T0[id0[r]] + T1[id1[r % seg or r]] + T2[...]; ids are int64; a table pointer may be null
__global__ void embed3_fwd_kernel(const float* __restrict__ t0, const int64_t* __restrict__ id0, const float* __restrict__ t1,
                                  const int64_t* __restrict__ id1, const float* __restrict__ t2, const int64_t* __restrict__ id2,
                                  float* __restrict__ out, int64_t R, int H, int seg, int total, int off) {
  const int64_t r = blockIdx.x;
  if (r >= R) return;
  const int64_t orow = (r / seg) * total + off + r % seg;
  const float* a = t0 + id0[r] * H;
  const float* b = t1 ? t1 + id1[r % seg] * H : nullptr;
  const float* c = t2 ? t2 + id2[r % seg] * H : nullptr;
  for (int h = threadIdx.x; h < H; h += blockDim.x) {
    float v = a[h];
    if (b) v += b[h];
    if (c) v += c[h];
    out[orow * H + h] = v;
  }
}
__global__ void embed3_bwd_kernel(const float* __restrict__ dout, const int64_t* __restrict__ id0, float* __restrict__ d0,
                                  const int64_t* __restrict__ id1, float* __restrict__ d1, const int64_t* __restrict__ id2,
                                  float* __restrict__ d2, int64_t R, int H, int seg, int total, int off) {
  const int64_t r = blockIdx.x;
  if (r >= R) return;
  const int64_t orow = (r / seg) * total + off + r % seg;
  for (int h = threadIdx.x; h < H; h += blockDim.x) {
    const float g = dout[orow * H + h];
    atomicAdd(d0 + id0[r] * H + h, g);
    if (d1) atomicAdd(d1 + id1[r % seg] * H + h, g);
    if (d2) atomicAdd(d2 + id2[r % seg] * H + h, g);
  }
}

// ---------------------------------------------------------------------------------------------------- cross-entropy
// train.py:150-153: F.cross_entropy(logits.view(-1, V), img_token.view(-1)) (mean over rows).  Block per row: max, then
// sum of exp, loss_r = logsumexp - x[target]; the row's logsumexp is kept for the backward.  A target outside [0, V) marks
// an ignored row (F.cross_entropy's ignore_index = -100): zero loss, zero gradient, not counted in the mean.
__device__ __forceinline__ float block_max_256(float v, float* red) {
  v = warp_max(v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = red[0];
#pragma unroll
  for (int w = 1; w < 8; ++w) r = fmaxf(r, red[w]);
  __syncthreads();
  return r;
}
__device__ __forceinline__ float block_sum_256(float v, float* red) {
  v = warp_sum(v);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) r += red[w];
  __syncthreads();
  return r;
}
__global__ void __launch_bounds__(256) ce_fwd_kernel(const float* __restrict__ logits, int64_t ld, const int64_t* __restrict__ target,
                                                     float* __restrict__ loss_rows, float* __restrict__ lse, int V) {
  __shared__ float red[8];
  const int64_t row = blockIdx.x;
  const float* x = logits + row * ld;
  float mx = -INFINITY;
  for (int c = threadIdx.x; c < V; c += 256) mx = fmaxf(mx, x[c]);
  mx = block_max_256(mx, red);
  float s = 0.f;
  for (int c = threadIdx.x; c < V; c += 256) s += expf(x[c] - mx);
  s = block_sum_256(s, red);
  if (threadIdx.x == 0) {
    const float l = mx + logf(s);
    const int64_t t = target[row];
    lse[row] = l;
    loss_rows[row] = (t >= 0 && t < V) ? l - x[t] : 0.f;
  }
}
// out[0] = mean of the counted rows' losses (fp64 totals, fixed order), out[1] = number of counted rows
__global__ void __launch_bounds__(256) ce_reduce_kernel(const float* __restrict__ loss_rows, const int64_t* __restrict__ target, int64_t R,
                                                        int V, float* __restrict__ out) {
  __shared__ double sd[256];
  __shared__ int sn[256];
  double a = 0.0;
  int n = 0;
  for (int64_t r = threadIdx.x; r < R; r += 256) {
    const int64_t t = target[r];
    if (t >= 0 && t < V) { a += (double)loss_rows[r]; ++n; }
  }
  sd[threadIdx.x] = a;
  sn[threadIdx.x] = n;
  __syncthreads();
  for (int o = 128; o > 0; o >>= 1) {
    if ((int)threadIdx.x < o) { sd[threadIdx.x] += sd[threadIdx.x + o]; sn[threadIdx.x] += sn[threadIdx.x + o]; }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    out[0] = sn[0] > 0 ? (float)(sd[0] / (double)sn[0]) : 0.f;
    out[1] = (float)sn[0];
  }
}
// dlogits[r, c] = (softmax(x_r)[c] - [c == t_r]) * dloss / count   (zero rows for ignored targets)
__global__ void __launch_bounds__(256) ce_bwd_kernel(const float* __restrict__ logits, int64_t ld, const int64_t* __restrict__ target,
                                                     const float* __restrict__ lse, const float* __restrict__ stat,
                                                     const float* __restrict__ dloss, float* __restrict__ dlogits, int64_t ldd, int V) {
  const int64_t row = blockIdx.x;
  const int64_t t = target[row];
  const bool on = t >= 0 && t < V;
  const float cnt = stat[1];
  const float g = on && cnt > 0.f ? dloss[0] / cnt : 0.f;
  const float l = lse[row];
  const float* x = logits + row * ld;
  float* d = dlogits + row * ldd;
  for (int c = threadIdx.x; c < V; c += 256) d[c] = on ? (expf(x[c] - l) - (c == (int)t ? 1.f : 0.f)) * g : 0.f;
}

static inline int ew_grid2(int64_t n) {
  int64_t b = cdiv(n, 256);
  return (int)(b < NUM_SMS * 16 ? (b < 1 ? 1 : b) : NUM_SMS * 16);
}

}  // namespace mas

using namespace mas;

extern "C" {

int mas_layernorm_forward(const float* x, const float* gamma, const float* beta, const float* residual, float* y, float* mean,
                          float* rstd, int64_t R, int H, float eps, void* stream) {
  MAS_REQUIRE(x && gamma && beta && y && mean && rstd && R > 0 && H > 0, "layernorm_forward: bad arguments");
  auto al16 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  if (R <= 64 && H % 4 == 0 && H <= 4096 && al16(x) && al16(y) && al16(gamma) && al16(beta) && (!residual || al16(residual))) {
    layernorm_fwd_block_kernel<<<(unsigned)R, 256, 0, S(stream)>>>(x, gamma, beta, residual, y, mean, rstd, H, eps);
    return launched("layernorm_fwd_block");
  }
  layernorm_fwd_kernel<<<(unsigned)cdiv(R, 8), 256, 0, S(stream)>>>(x, gamma, beta, residual, y, mean, rstd, R, H, eps);
  return launched("layernorm_fwd");
}
int mas_layernorm2_forward(const float* x, const float* gamma1, const float* beta1, const float* residual, float* y1,
                           const float* gamma2, const float* beta2, float* y2, int64_t R, int H, float eps1, float eps2, void* stream) {
  MAS_REQUIRE(x && gamma1 && beta1 && y1 && gamma2 && beta2 && y2 && R > 0 && H > 0, "layernorm2_forward: bad arguments");
  auto al16 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  if (!(R <= 64 && H % 4 == 0 && H <= 4096 && al16(x) && al16(y1) && al16(y2) && al16(gamma1) && al16(beta1) && al16(gamma2) &&
        al16(beta2) && (!residual || al16(residual))))
    return fail(MAS_ERR_UNSUPPORTED, "layernorm2_forward: needs R <= 64, H %% 4 == 0, H <= 4096 and 16-byte aligned operands");
  layernorm2_fwd_block_kernel<<<(unsigned)R, 256, 0, S(stream)>>>(x, gamma1, beta1, residual, y1, gamma2, beta2, y2, H, eps1, eps2);
  return launched("layernorm2_fwd_block");
}
size_t mas_layernorm_ws_bytes(int64_t R, int H) { return (size_t)cdiv(R, LN_ROWS) * H * 2 * sizeof(double) + 64; }
int mas_layernorm_backward(const float* dy, const float* x, const float* mean, const float* rstd, const float* gamma, float* dx,
                           float* dgamma, float* dbeta, int64_t R, int H, void* ws, size_t ws_bytes, void* stream) {
  MAS_REQUIRE(dy && x && mean && rstd && gamma && dx && R > 0 && H > 0, "layernorm_backward: bad arguments");
  if (ws_bytes < mas_layernorm_ws_bytes(R, H)) return fail(MAS_ERR_WORKSPACE, "layernorm_backward: workspace too small");
  auto al16 = [](const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
  if (H % 4 == 0 && H <= 4096 && H >= 256 && al16(dy) && al16(x) && al16(gamma) && al16(dx)) {
    layernorm_bwd_dx_block_kernel<<<(unsigned)R, 256, 0, S(stream)>>>(dy, x, mean, rstd, gamma, dx, H);
    if (int e = launched("layernorm_bwd_dx_block")) return e;
  } else {
    layernorm_bwd_dx_kernel<<<(unsigned)cdiv(R, 8), 256, 0, S(stream)>>>(dy, x, mean, rstd, gamma, dx, R, H);
    if (int e = launched("layernorm_bwd_dx")) return e;
  }
  if (dgamma && dbeta) {
    const int chunks = (int)cdiv(R, LN_ROWS);
    layernorm_bwd_param_partial<<<dim3((unsigned)cdiv(H, 32), chunks), dim3(32, 8), 0, S(stream)>>>(dy, x, mean, rstd, R, H, (double*)ws);
    if (int e = launched("layernorm_bwd_param_partial")) return e;
    layernorm_bwd_param_final<<<(int)cdiv(H, 128), 128, 0, S(stream)>>>((const double*)ws, chunks, H, dgamma, dbeta);
    return launched("layernorm_bwd_param_final");
  }
  return MAS_OK;
}
int mas_gelu_forward(const float* x, float* y, int64_t n, void* stream) {
  gelu_fwd_kernel<<<ew_grid2(n), 256, 0, S(stream)>>>(x, y, n);
  return launched("gelu_fwd");
}
int mas_gelu_backward(const float* dy, const float* x, float* dx, int64_t n, void* stream) {
  gelu_bwd_kernel<<<ew_grid2(n), 256, 0, S(stream)>>>(dy, x, dx, n);
  return launched("gelu_bwd");
}
int mas_softmax_causal_forward(const float* s, float* p, int64_t mats, int rows, int cols, void* stream) {
  MAS_REQUIRE(mats > 0 && rows > 0 && cols >= rows, "softmax_causal: bad shape");
  softmax_causal_kernel<<<(unsigned)cdiv(mats * rows, 8), 256, 0, S(stream)>>>(s, p, mats * rows, rows, cols);
  return launched("softmax_causal");
}
int mas_softmax_causal_backward(const float* p, const float* dp, float* ds, int64_t mats, int rows, int cols, float scale, void* stream) {
  MAS_REQUIRE(p && dp && ds && mats > 0 && rows > 0 && cols >= rows, "softmax_causal_backward: bad arguments");
  softmax_causal_bwd_kernel<<<(unsigned)cdiv(mats * rows, 8), 256, 0, S(stream)>>>(p, dp, ds, mats * rows, rows, cols, scale);
  return launched("softmax_causal_bwd");
}
int mas_embed3_forward(const float* t0, const int64_t* id0, const float* t1, const int64_t* id1, const float* t2, const int64_t* id2,
                       float* out, int64_t R, int H, int seg, int total, int off, void* stream) {
  MAS_REQUIRE(t0 && id0 && out && R > 0 && H > 0 && seg > 0, "embed3_forward: bad arguments");
  embed3_fwd_kernel<<<(unsigned)R, 128, 0, S(stream)>>>(t0, id0, t1, id1, t2, id2, out, R, H, seg, total, off);
  return launched("embed3_fwd");
}
int mas_embed3_backward(const float* dout, const int64_t* id0, float* d0, const int64_t* id1, float* d1, const int64_t* id2, float* d2,
                        int64_t R, int H, int seg, int total, int off, void* stream) {
  MAS_REQUIRE(dout && id0 && d0 && R > 0 && H > 0 && seg > 0, "embed3_backward: bad arguments");
  embed3_bwd_kernel<<<(unsigned)R, 128, 0, S(stream)>>>(dout, id0, d0, id1, d1, id2, d2, R, H, seg, total, off);
  return launched("embed3_bwd");
}

int mas_ce_forward(const float* logits, int64_t ld, const int64_t* target, float* loss_rows, float* lse, float* out, int64_t R, int V,
                   void* stream) {
  MAS_REQUIRE(logits && target && loss_rows && lse && out && R > 0 && V > 0 && ld >= V, "ce_forward: bad arguments");
  ce_fwd_kernel<<<(unsigned)R, 256, 0, S(stream)>>>(logits, ld, target, loss_rows, lse, V);
  if (int e = launched("ce_fwd")) return e;
  ce_reduce_kernel<<<1, 256, 0, S(stream)>>>(loss_rows, target, R, V, out);
  return launched("ce_reduce");
}
int mas_ce_backward(const float* logits, int64_t ld, const int64_t* target, const float* lse, const float* stat, const float* dloss,
                    float* dlogits, int64_t ldd, int64_t R, int V, void* stream) {
  MAS_REQUIRE(logits && target && lse && stat && dloss && dlogits && R > 0 && V > 0 && ld >= V && ldd >= V, "ce_backward: bad arguments");
  ce_bwd_kernel<<<(unsigned)R, 256, 0, S(stream)>>>(logits, ld, target, lse, stat, dloss, dlogits, ldd, V);
  return launched("ce_bwd");
}

}  // extern "C"
