// Autoregressive sampling of the token transformer (SURVEY.md 8f-3): KV cache + single-token decode kernels.
// The reference has no working implementation of this path (models/transformer.py:73-115 vs :176-210 disagree on the
// cache layout and train.py never samples); the specification is the non-cached forward (transformer.py:77-103,
// 216-244): a decode step must reproduce the logits the full causal forward gives at that position.
//   * mas_linear_small : y[r,n] = act(sum_k x[r,k] W[n,k] + b[n]) for a handful of rows (cond + uncond streams): a
//     weight-streaming kernel — every weight is read exactly once per token, so it is HBM-bound by construction
//     (371 M parameters = 1.48 GB per token for the 24-layer / 1024-wide model); strict fp32, up to 8 rows. More rows run
//     mas_linear_rows_f16 (gemm_tma.cu).
//   * mas_kv_append    : scatters the k / v thirds of a fused qkv activation into the [R, heads, Tmax, hd] caches.
//   * mas_attn_decode  : one query per (row, head) against the cache: scores, softmax, weighted sum of v.
//     The _f16 variants of both keep the caches in fp16 (decoding more than 8 rows).
//   * mas_attn_decode_shared(_append) : mas_attn_decode(_append) for groups of rows that share a prompt's prefix cache
//     (generate(num_samples = n)); a block reads the group's prefix once for up to 4 of its rows.
//   * mas_cfg_mix      : classifier-free guidance, out = uncond + scale * (cond - uncond); mas_cfg_mix_rows: one scale per row.
//   * mas_sample_topk / _filtered / _filtered_logp / _rows : the token draw (mas_sample_rows: per-row controls and seeds).
#include <cuda_fp16.h>

#include "dropout.cuh"
#include "mas_common.cuh"

using namespace mas;

namespace {

constexpr int LS_MAXR = 8;

// one warp per output column n; lanes stride over k in float4 steps (W row n is contiguous: 512-byte warp transactions)
template <int R>
__global__ void __launch_bounds__(256) linear_small_kernel(const float* __restrict__ x, int64_t ldx, const float* __restrict__ W,
                                                           const float* __restrict__ bias, float* __restrict__ y, int64_t ldy, int N,
                                                           int K, int act) {
  const int lane = threadIdx.x & 31, n = blockIdx.x * 8 + (threadIdx.x >> 5);
  if (n >= N) return;
  const float4* w4 = reinterpret_cast<const float4*>(W + (size_t)n * K);
  float acc[R];
#pragma unroll
  for (int r = 0; r < R; ++r) acc[r] = 0.f;
  const int K4 = K >> 2;
  int k = lane;
  for (; k + 224 < K4; k += 256) {  // eight weight quads (128 B per lane, 4 KB per warp) in flight: the stream is latency-bound
    float4 wv[8];
#pragma unroll
    for (int u = 0; u < 8; ++u) wv[u] = __ldg(w4 + k + 32 * u);
#pragma unroll
    for (int u = 0; u < 8; ++u)
#pragma unroll
      for (int r = 0; r < R; ++r) {
        const float4 xv = __ldg(reinterpret_cast<const float4*>(x + (size_t)r * ldx) + k + 32 * u);
        acc[r] = fmaf(wv[u].x, xv.x, acc[r]); acc[r] = fmaf(wv[u].y, xv.y, acc[r]);
        acc[r] = fmaf(wv[u].z, xv.z, acc[r]); acc[r] = fmaf(wv[u].w, xv.w, acc[r]);
      }
  }
  for (; k < K4; k += 32) {
    const float4 wv = __ldg(w4 + k);
#pragma unroll
    for (int r = 0; r < R; ++r) {
      const float4 xv = __ldg(reinterpret_cast<const float4*>(x + (size_t)r * ldx) + k);
      acc[r] = fmaf(wv.x, xv.x, acc[r]); acc[r] = fmaf(wv.y, xv.y, acc[r]);
      acc[r] = fmaf(wv.z, xv.z, acc[r]); acc[r] = fmaf(wv.w, xv.w, acc[r]);
    }
  }
#pragma unroll
  for (int r = 0; r < R; ++r) acc[r] = warp_sum(acc[r]);
  if (lane == 0) {
    const float b = bias ? __ldg(bias + n) : 0.f;
#pragma unroll
    for (int r = 0; r < R; ++r) {
      float v = acc[r] + b;
      if (act == 1) {  // OpenAI tanh-GELU, transformer.py:11-14
        const float u = 0.7978845608028654f * v * (1.f + 0.044715f * v * v);
        v = 0.5f * v * (1.f + tanhf(u));
      }
      y[(size_t)r * ldy + n] = v;
    }
  }
}

// Cache elements: fp32 (up to 8 rows: strict fp32 decoding) or fp16 (more rows: half the cache bytes, which dominate a decode
// step at a few hundred rows).  k / v are rounded once, to nearest, as mas_to_half rounds; everything downstream is fp32.
__device__ __forceinline__ float to_elem(float v, float*) { return v; }
__device__ __forceinline__ __half to_elem(float v, __half*) { return __float2half_rn(v); }
__device__ __forceinline__ float elem_f(float v) { return v; }
__device__ __forceinline__ float elem_f(__half v) { return __half2float(v); }
__device__ __forceinline__ void store4(float* p, float4 v) { *reinterpret_cast<float4*>(p) = v; }
__device__ __forceinline__ void store4(__half* p, float4 v) {
  const __half2 a = __floats2half2_rn(v.x, v.y), b = __floats2half2_rn(v.z, v.w);
  uint2 u;
  u.x = *reinterpret_cast<const uint32_t*>(&a);
  u.y = *reinterpret_cast<const uint32_t*>(&b);
  *reinterpret_cast<uint2*>(p) = u;
}
// one 16-byte load: 4 fp32 or 8 fp16 elements, widened to fp32
template <typename T> struct Vec16 { static constexpr int E = 16 / sizeof(T); };
__device__ __forceinline__ void load16(const float* p, float* o) {
  const float4 v = __ldg(reinterpret_cast<const float4*>(p));
  o[0] = v.x; o[1] = v.y; o[2] = v.z; o[3] = v.w;
}
__device__ __forceinline__ void load16(const __half* p, float* o) {
  const uint4 u = __ldg(reinterpret_cast<const uint4*>(p));
  const uint32_t w[4] = {u.x, u.y, u.z, u.w};
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const float2 f = __half22float2(*reinterpret_cast<const __half2*>(&w[i]));
    o[2 * i] = f.x; o[2 * i + 1] = f.y;
  }
}

// qkv [R, T, 3H] -> kcache / vcache [R, heads, Tmax, hd] at positions pos0 .. pos0+T-1
template <typename T>
__global__ void kv_append_kernel(const float* __restrict__ qkv, int R, int T_, int heads, int hd, T* __restrict__ kc,
                                 T* __restrict__ vc, int Tmax, int pos0) {
  const int H = heads * hd, Q = hd >> 2;
  const int64_t total = (int64_t)R * T_ * heads * Q;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    int64_t r_ = i;
    const int q = (int)(r_ % Q); r_ /= Q;
    const int h = (int)(r_ % heads); r_ /= heads;
    const int t = (int)(r_ % T_);
    const int r = (int)(r_ / T_);
    const float* src = qkv + ((size_t)r * T_ + t) * 3 * H + h * hd + q * 4;
    const size_t dst = (((size_t)r * heads + h) * Tmax + pos0 + t) * hd + q * 4;
    store4(kc + dst, __ldg(reinterpret_cast<const float4*>(src + H)));
    store4(vc + dst, __ldg(reinterpret_cast<const float4*>(src + 2 * H)));
  }
}

// block per (row, head), 256 threads; q = this token's query (row r of qkv [R, 3H]); len cached positions (incl. this one).
// Everything is latency-bound here (a few hundred KB per block), so both passes keep many independent 16-byte loads in
// flight: HD is a template parameter (fully unrolled dot products), the v pass is unrolled eight positions deep.
// APPEND: the token's own k / v (the k and v thirds of its qkv row) are written to the caches at position len-1 by this
// kernel (no separate mas_kv_append launch) and enter the attention from shared memory - the freshly written cache lines are
// never read back here (the cache loads use the read-only path).  With an fp16 cache they enter as the rounded values stored.
template <int HD, bool APPEND, typename T>
__global__ void __launch_bounds__(256) attn_decode_kernel(const float* __restrict__ qkv, T* __restrict__ kc, T* __restrict__ vc,
                                                          float* __restrict__ ctx, int heads, int Tmax, int len) {
  // [HD] q, [len] scores, [32] scratch, [256/(HD/E)][HD] partial outputs, [2 HD] own k, v
  extern __shared__ __align__(16) float sm[];
  constexpr int E = Vec16<T>::E;                 // cache elements per 16-byte load
  constexpr int Q = HD / 4, VQ = HD / E, GROUPS = 256 / VQ;
  float* qs = sm;
  float* sc = sm + HD;
  float* red = sc + ((len + 3) & ~3);
  float* po = red + 32;
  float* ks = po + GROUPS * HD;
  float* vs = ks + HD;
  const int r = blockIdx.x / heads, h = blockIdx.x % heads, H = heads * HD, t0 = threadIdx.x, lane = t0 & 31, warp = t0 >> 5;
  const int lenc = APPEND ? len - 1 : len;     // positions read from the cache
  if (t0 < HD) {
    const float* tokrow = qkv + (size_t)r * 3 * H + h * HD + t0;
    qs[t0] = tokrow[0];
    if (APPEND) {
      const T kv = to_elem(tokrow[H], (T*)nullptr), vv = to_elem(tokrow[2 * H], (T*)nullptr);
      ks[t0] = elem_f(kv);
      vs[t0] = elem_f(vv);
      const size_t dst = (((size_t)r * heads + h) * Tmax + (len - 1)) * HD + t0;
      kc[dst] = kv;
      vc[dst] = vv;
    }
  }
  __syncthreads();
  const float alpha = rsqrtf((float)HD);
  const T* kb = kc + ((size_t)r * heads + h) * Tmax * HD;
  const T* vb = vc + ((size_t)r * heads + h) * Tmax * HD;
  float4 q4[Q];
#pragma unroll
  for (int i = 0; i < Q; ++i) q4[i] = *reinterpret_cast<const float4*>(qs + 4 * i);
  float mx = -INFINITY;
  for (int t = t0; t < lenc; t += 256) {
    float kv[HD];
#pragma unroll
    for (int i = 0; i < VQ; ++i) load16(kb + (size_t)t * HD + i * E, kv + i * E);
    float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
#pragma unroll
    for (int i = 0; i < Q; ++i) {
      s0 = fmaf(q4[i].x, kv[4 * i], s0); s1 = fmaf(q4[i].y, kv[4 * i + 1], s1);
      s2 = fmaf(q4[i].z, kv[4 * i + 2], s2); s3 = fmaf(q4[i].w, kv[4 * i + 3], s3);
    }
    const float s = ((s0 + s1) + (s2 + s3)) * alpha;
    sc[t] = s;
    mx = fmaxf(mx, s);
  }
  if (APPEND && t0 == 255) {   // the token itself: k from shared memory, same summation order as above
    float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
#pragma unroll
    for (int i = 0; i < Q; ++i) {
      const float4 kv = *reinterpret_cast<const float4*>(ks + 4 * i);
      s0 = fmaf(q4[i].x, kv.x, s0); s1 = fmaf(q4[i].y, kv.y, s1);
      s2 = fmaf(q4[i].z, kv.z, s2); s3 = fmaf(q4[i].w, kv.w, s3);
    }
    const float s = ((s0 + s1) + (s2 + s3)) * alpha;
    sc[len - 1] = s;
    mx = fmaxf(mx, s);
  }
  mx = warp_max(mx);
  if (lane == 0) red[warp] = mx;
  __syncthreads();
  mx = red[0];
#pragma unroll
  for (int w = 1; w < 8; ++w) mx = fmaxf(mx, red[w]);
  __syncthreads();
  float sum = 0.f;
  for (int t = t0; t < len; t += 256) {
    const float e = expf(sc[t] - mx);
    sc[t] = e;
    sum += e;
  }
  sum = warp_sum(sum);
  if (lane == 0) red[8 + warp] = sum;
  __syncthreads();
  float tot = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) tot += red[8 + w];
  const float inv = 1.f / tot;
  // ctx[d] = sum_t p_t v[t][d]: thread = (E-wide slice of d, one of GROUPS interleaved t ranges); 16-byte loads coalesced over d.
  // GROUPS doubles for fp16 (E = 8), so the fp16 cache's partial sums are grouped and added differently from the fp32 cache's.
  const int dq = t0 % VQ, g = t0 / VQ;
  float o[E];
#pragma unroll
  for (int e = 0; e < E; ++e) o[e] = 0.f;
  int t = g;
  for (; t + 7 * GROUPS < lenc; t += 8 * GROUPS) {
    float vv[8][E];
#pragma unroll
    for (int u = 0; u < 8; ++u) load16(vb + (size_t)(t + u * GROUPS) * HD + dq * E, vv[u]);
#pragma unroll
    for (int u = 0; u < 8; ++u) {
      const float p = sc[t + u * GROUPS];
#pragma unroll
      for (int e = 0; e < E; ++e) o[e] = fmaf(p, vv[u][e], o[e]);
    }
  }
  for (; t < lenc; t += GROUPS) {
    float vv[E];
    load16(vb + (size_t)t * HD + dq * E, vv);
    const float p = sc[t];
#pragma unroll
    for (int e = 0; e < E; ++e) o[e] = fmaf(p, vv[e], o[e]);
  }
  if (APPEND && g == 0) {
    const float p = sc[len - 1];
#pragma unroll
    for (int e = 0; e < E; ++e) o[e] = fmaf(p, vs[E * dq + e], o[e]);
  }
#pragma unroll
  for (int e = 0; e < E; e += 4)
    *reinterpret_cast<float4*>(po + (size_t)g * HD + E * dq + e) = make_float4(o[e], o[e + 1], o[e + 2], o[e + 3]);
  __syncthreads();
  if (t0 < HD) {
    float v = 0.f;
#pragma unroll 4
    for (int g2 = 0; g2 < GROUPS; ++g2) v += po[g2 * HD + t0];
    ctx[(size_t)r * H + h * HD + t0] = v * inv;
  }
}

// q . k over HD in attn_decode_kernel's order: four interleaved fmaf chains, added pairwise, then scaled.
template <int HD>
__device__ __forceinline__ float decode_score(const float* q, const float* kv, float alpha) {
  float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
#pragma unroll
  for (int i = 0; i < HD / 4; ++i) {
    const float4 qv = *reinterpret_cast<const float4*>(q + 4 * i);
    s0 = fmaf(qv.x, kv[4 * i], s0); s1 = fmaf(qv.y, kv[4 * i + 1], s1);
    s2 = fmaf(qv.z, kv[4 * i + 2], s2); s3 = fmaf(qv.w, kv[4 * i + 3], s3);
  }
  return ((s0 + s1) + (s2 + s3)) * alpha;
}

// Shared-prefix decode attention (generate(num_samples = n)): the R sample rows form groups of n consecutive rows that share a
// prompt. Row r attends over positions 0..P-1 of prompt row r / n's prefix cache (kp / vp [R/n, heads, P, HD]), then over
// positions P..len-1 of its own suffix cache (ks / vs [R, heads, Tsuf, HD], slot = position - P).  A block serves g <= G rows of
// one group for one head, so each 16-byte prefix load feeds g rows' scores and v partials; blocks of the same (group, head) are
// adjacent in the grid, so the slices of one group also meet its prefix in L2.  Per row the arithmetic is
// attn_decode_kernel<HD, APPEND, T>'s: the same thread owns the same positions in the same order in every pass (scores, max,
// exp / sum, v pass, the GROUPS-partial reduction), so ctx is bit-identical to the unshared kernel run on the concatenated cache.
// APPEND: this token's k / v are stored at slot len-1-P and enter from shared memory, its p v term last in partial group 0 (as
// mas_attn_decode_append adds it).  Without APPEND, position len-1 is read from the suffix cache like every other one, so its
// term lands in group (len-1) % GROUPS (as mas_attn_decode adds it after mas_kv_append).
template <int HD, int G, bool APPEND, typename T>
__global__ void __launch_bounds__(256) attn_decode_shared_kernel(const float* __restrict__ qkv, const T* __restrict__ kp,
                                                                 const T* __restrict__ vp, T* __restrict__ ks, T* __restrict__ vs,
                                                                 float* __restrict__ ctx, int n, int heads, int P, int Tsuf, int len) {
  // [G][HD] q, own k, own v; [G][16] scratch; [G][len] scores; [G][GROUPS][HD] partial outputs
  extern __shared__ __align__(16) float sm[];
  constexpr int E = Vec16<T>::E;
  constexpr int VQ = HD / E, GROUPS = 256 / VQ;
  const int lenc = APPEND ? len - 1 : len, scl = (len + 3) & ~3;     // positions read from the caches
  float* qs = sm;
  float* kself = qs + G * HD;
  float* vself = kself + G * HD;
  float* red = vself + G * HD;
  float* sc = red + G * 16;
  float* po = sc + G * scl;
  const int slices = (n + G - 1) / G, s = blockIdx.x % slices, h = (blockIdx.x / slices) % heads, grp = blockIdx.x / slices / heads;
  const int r0 = grp * n + s * G, g = min(G, n - s * G), H = heads * HD, t0 = threadIdx.x, lane = t0 & 31, warp = t0 >> 5;
  for (int i = t0; i < G * HD; i += 256) {
    const int j = i / HD, d = i % HD;
    float q = 0.f, kf = 0.f, vf = 0.f;
    if (j < g) {
      const float* tokrow = qkv + (size_t)(r0 + j) * 3 * H + h * HD + d;
      q = tokrow[0];
      if (APPEND) {
        const T kv = to_elem(tokrow[H], (T*)nullptr), vv = to_elem(tokrow[2 * H], (T*)nullptr);
        kf = elem_f(kv);
        vf = elem_f(vv);
        const size_t dst = (((size_t)(r0 + j) * heads + h) * Tsuf + (len - 1 - P)) * HD + d;
        ks[dst] = kv;
        vs[dst] = vv;
      }
    }
    qs[i] = q;
    kself[i] = kf;
    vself[i] = vf;
  }
  __syncthreads();
  const float alpha = rsqrtf((float)HD);
  const T* kpb = kp + ((size_t)grp * heads + h) * P * HD;
  const T* vpb = vp + ((size_t)grp * heads + h) * P * HD;
  const size_t suf0 = ((size_t)r0 * heads + h) * Tsuf * HD, sufj = (size_t)heads * Tsuf * HD;   // row r0 + j's suffix: suf0 + j * sufj
  float mx[G];
#pragma unroll
  for (int j = 0; j < G; ++j) mx[j] = -INFINITY;
  int t = t0;
  for (; t < P; t += 256) {                      // prefix: one load, g rows
    float kv[HD];
#pragma unroll
    for (int i = 0; i < VQ; ++i) load16(kpb + (size_t)t * HD + i * E, kv + i * E);
#pragma unroll
    for (int j = 0; j < G; ++j)
      if (j < g) {
        const float sj = decode_score<HD>(qs + j * HD, kv, alpha);
        sc[j * scl + t] = sj;
        mx[j] = fmaxf(mx[j], sj);
      }
  }
  for (; t < lenc; t += 256) {                   // suffix: each row its own
#pragma unroll
    for (int j = 0; j < G; ++j)
      if (j < g) {
        float kv[HD];
#pragma unroll
        for (int i = 0; i < VQ; ++i) load16(ks + suf0 + j * sufj + (size_t)(t - P) * HD + i * E, kv + i * E);
        const float sj = decode_score<HD>(qs + j * HD, kv, alpha);
        sc[j * scl + t] = sj;
        mx[j] = fmaxf(mx[j], sj);
      }
  }
  if (APPEND && t0 == 255) {
#pragma unroll
    for (int j = 0; j < G; ++j)
      if (j < g) {
        const float sj = decode_score<HD>(qs + j * HD, kself + j * HD, alpha);
        sc[j * scl + len - 1] = sj;
        mx[j] = fmaxf(mx[j], sj);
      }
  }
#pragma unroll
  for (int j = 0; j < G; ++j) {
    const float m = warp_max(mx[j]);
    if (lane == 0) red[j * 16 + warp] = m;
  }
  __syncthreads();
#pragma unroll
  for (int j = 0; j < G; ++j) {
    float m = red[j * 16];
#pragma unroll
    for (int w = 1; w < 8; ++w) m = fmaxf(m, red[j * 16 + w]);
    mx[j] = m;
  }
  __syncthreads();
#pragma unroll
  for (int j = 0; j < G; ++j) {
    float sum = 0.f;
    if (j < g)
      for (int tt = t0; tt < len; tt += 256) {
        const float e = expf(sc[j * scl + tt] - mx[j]);
        sc[j * scl + tt] = e;
        sum += e;
      }
    sum = warp_sum(sum);
    if (lane == 0) red[j * 16 + 8 + warp] = sum;
  }
  __syncthreads();
  float inv[G];
#pragma unroll
  for (int j = 0; j < G; ++j) {
    float tot = 0.f;
#pragma unroll
    for (int w = 0; w < 8; ++w) tot += red[j * 16 + 8 + w];
    inv[j] = 1.f / tot;
  }
  const int dq = t0 % VQ, gg = t0 / VQ;
  float o[G][E];
#pragma unroll
  for (int j = 0; j < G; ++j)
#pragma unroll
    for (int e = 0; e < E; ++e) o[j][e] = 0.f;
  t = gg;
  for (; t + 7 * GROUPS < P; t += 8 * GROUPS) {
    float vv[8][E];
#pragma unroll
    for (int u = 0; u < 8; ++u) load16(vpb + (size_t)(t + u * GROUPS) * HD + dq * E, vv[u]);
#pragma unroll
    for (int u = 0; u < 8; ++u)
#pragma unroll
      for (int j = 0; j < G; ++j)
        if (j < g) {
          const float p = sc[j * scl + t + u * GROUPS];
#pragma unroll
          for (int e = 0; e < E; ++e) o[j][e] = fmaf(p, vv[u][e], o[j][e]);
        }
  }
  for (; t < P; t += GROUPS) {
    float vv[E];
    load16(vpb + (size_t)t * HD + dq * E, vv);
#pragma unroll
    for (int j = 0; j < G; ++j)
      if (j < g) {
        const float p = sc[j * scl + t];
#pragma unroll
        for (int e = 0; e < E; ++e) o[j][e] = fmaf(p, vv[e], o[j][e]);
      }
  }
  for (; t < lenc; t += GROUPS) {
#pragma unroll
    for (int j = 0; j < G; ++j)
      if (j < g) {
        float vv[E];
        load16(vs + suf0 + j * sufj + (size_t)(t - P) * HD + dq * E, vv);
        const float p = sc[j * scl + t];
#pragma unroll
        for (int e = 0; e < E; ++e) o[j][e] = fmaf(p, vv[e], o[j][e]);
      }
  }
#pragma unroll
  for (int j = 0; j < G; ++j)
    if (j < g) {
      if (APPEND && gg == 0) {
        const float p = sc[j * scl + len - 1];
#pragma unroll
        for (int e = 0; e < E; ++e) o[j][e] = fmaf(p, vself[j * HD + E * dq + e], o[j][e]);
      }
#pragma unroll
      for (int e = 0; e < E; e += 4)
        *reinterpret_cast<float4*>(po + ((size_t)j * GROUPS + gg) * HD + E * dq + e) = make_float4(o[j][e], o[j][e + 1], o[j][e + 2], o[j][e + 3]);
    }
  __syncthreads();
#pragma unroll
  for (int j = 0; j < G; ++j)
    if (j < g && t0 < HD) {
      float v = 0.f;
#pragma unroll 4
      for (int g2 = 0; g2 < GROUPS; ++g2) v += po[((size_t)j * GROUPS + g2) * HD + t0];
      ctx[(size_t)(r0 + j) * H + h * HD + t0] = v * inv[j];
    }
}

__global__ void cfg_mix_kernel(const float* __restrict__ cond, const float* __restrict__ uncond, float* __restrict__ out, int64_t n,
                               float scale) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float u = uncond[i];
    out[i] = fmaf(scale, cond[i] - u, u);
  }
}

// cfg_mix_kernel with one scale per row of V elements: row r is cfg_mix_kernel's expression at scale[r], bit for bit.
__global__ void cfg_mix_rows_kernel(const float* __restrict__ cond, const float* __restrict__ uncond, float* __restrict__ out, int R,
                                    int64_t V, const float* __restrict__ scale) {
  for (int r = blockIdx.y; r < R; r += gridDim.y) {
    const float s = scale[r];
    const size_t o = (size_t)r * V;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < V; i += (int64_t)gridDim.x * blockDim.x) {
      const float u = uncond[o + i];
      out[o + i] = fmaf(s, cond[o + i] - u, u);
    }
  }
}

// Token draw (Make-A-Scene paper 3.4 / generate()), block per row:
//   1. z = logits / temperature;
//   2. top-k: keep the top_k largest (all values equal to the k-th largest are kept, like `z < kth -> -inf`);
//   3. top-p (top_p < 1): of the entries top-k kept, keep those whose softmax mass of kept entries with a STRICTLY larger z is
//      <= top_p (top_k_top_p_filtering's rule, with ties decided by value: equal z are kept or dropped together; the largest
//      entry is always kept);
//   4. token = inverse CDF of softmax(z) over the kept set at u, in index order (first index whose running sum exceeds
//      u * total).
// Both filters are thresholds on order-preserving keys of z, found by 4-pass radix selects (8 bits per pass): top-k on counts,
// top-p on masses.  The masses are exp(z - max) in 2^-40 fixed point, added with 64-bit integer atomics: associative, so the
// threshold (and the token) is the same on every launch whatever the block's scheduling.  Quantisation moves a mass by less
// than V * 2^-40 of the largest entry's, so only an entry whose mass above lies that close to top_p can be decided otherwise
// than in exact arithmetic.
// temperature == 0: greedy, the first index of the largest logit (torch.argmax's rule); u is not read.
// Prompt (pmask != NULL): rows with pmask[r * pld] != 0 take tok = ptok[r * pld] and draw nothing.
// logp != NULL: logp[r * lpld] = log of the probability the token was drawn with, (z_tok - mx) - log(total) with total the
// kept-set sum the draw itself used (one store per row, no further pass over V); 0 for prompt and greedy rows (certain).
// ROWS (mas_sample_rows): the row reads its temperature, top_k and top_p from rc's arrays instead of the scalar arguments, and
// with rc.seeds its uniform from seeded_uniform instead of u; everything after those reads is the scalar kernel's code, so a row
// gets the bits the scalar entries give it at its own values.  ROWS = false compiles to the kernel of the scalar entries.
__device__ __forceinline__ uint32_t order_key(float f) {
  const uint32_t b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
constexpr float MASS_ONE = 1099511627776.f;          // 2^40: the largest entry's mass exp(0)

struct RowControls {
  const float* temperature;   // [R]
  const int* top_k;           // [R]
  const float* top_p;         // [R], >= 1: off
  const int64_t* seeds;       // [R] or NULL (then u)
  int64_t position;
};

// The uniform of a row with this seed at this position (include/mas_b200.h, mas_sample_rows): the top 24 bits of word 0 of
// Philox4x32-10(counter = (lo32(position), hi32(position), 0, 0), key = (lo32(seed), hi32(seed))), times 2^-24: in [0, 1).
__device__ __forceinline__ float seeded_uniform(int64_t seed, int64_t position) {
  const uint64_t s = (uint64_t)seed, p = (uint64_t)position;
  const uint4 w = philox4x32_10(make_uint4((uint32_t)p, (uint32_t)(p >> 32), 0u, 0u), (uint32_t)s, (uint32_t)(s >> 32));
  return (float)(w.x >> 8) * 5.9604644775390625e-8f;
}

template <bool ROWS>
__global__ void __launch_bounds__(256) sample_topk_kernel(const float* __restrict__ logits, int64_t ld, int V, float temperature, int top_k,
                                                          float top_p, const float* __restrict__ u, const int64_t* __restrict__ ptok,
                                                          const uint8_t* __restrict__ pmask, int64_t pld, int64_t* __restrict__ tok,
                                                          float* __restrict__ logp, int64_t lpld, RowControls rc) {
  __shared__ int hist[256];
  __shared__ unsigned long long mhist[256];
  __shared__ uint32_t s_prefix;
  __shared__ int s_remaining;
  __shared__ unsigned long long s_above, s_budget;
  __shared__ float red[8];
  __shared__ int redi[8];
  __shared__ float csum[256];
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const float* x = logits + (int64_t)blockIdx.x * ld;
  if (pmask && pmask[(int64_t)blockIdx.x * pld]) {   // uniform over the block
    if (t == 0) {
      tok[blockIdx.x] = ptok[(int64_t)blockIdx.x * pld];
      if (logp) logp[(int64_t)blockIdx.x * lpld] = 0.f;
    }
    return;
  }
  if (ROWS) {
    temperature = rc.temperature[blockIdx.x];
    top_k = rc.top_k[blockIdx.x];
    top_p = rc.top_p[blockIdx.x];
  }
  if (temperature == 0.f) {                           // greedy: (value, index) maximum, ties to the lower index
    float best = -INFINITY;
    int bi = -1;
    for (int c = t; c < V; c += 256) {
      const float v = x[c];
      if (bi < 0 || v > best) { best = v; bi = c; }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      const float ov = __shfl_down_sync(0xffffffffu, best, o);
      const int oi = __shfl_down_sync(0xffffffffu, bi, o);
      if (oi >= 0 && (bi < 0 || ov > best || (ov == best && oi < bi))) { best = ov; bi = oi; }
    }
    if (lane == 0) { red[warp] = best; redi[warp] = bi; }
    __syncthreads();
    if (t == 0) {
      for (int w = 1; w < 8; ++w)
        if (redi[w] >= 0 && (bi < 0 || red[w] > best || (red[w] == best && redi[w] < bi))) { best = red[w]; bi = redi[w]; }
      tok[blockIdx.x] = (int64_t)bi;
      if (logp) logp[(int64_t)blockIdx.x * lpld] = 0.f;
    }
    return;
  }
  uint32_t thr = 0;                                   // keys >= thr are kept
  if (top_k > 0 && top_k < V) {
    uint32_t prefix = 0, mask = 0;
    int remaining = top_k;
    for (int pass = 3; pass >= 0; --pass) {
      const int shift = pass * 8;
      hist[t] = 0;
      __syncthreads();
      for (int c = t; c < V; c += 256) {
        const uint32_t key = order_key(x[c] / temperature);
        if ((key & mask) == prefix) atomicAdd(&hist[(key >> shift) & 255u], 1);
      }
      __syncthreads();
      if (t == 0) {
        int rem = remaining, b = 255;
        for (; b > 0; --b) {
          const int cnt = hist[b];
          if (cnt >= rem) break;
          rem -= cnt;
        }
        s_prefix = prefix | ((uint32_t)b << shift);
        s_remaining = rem;
      }
      __syncthreads();
      prefix = s_prefix;
      remaining = s_remaining;
      mask |= 0xFFu << shift;
      __syncthreads();
    }
    thr = prefix;
  }
  float mx = -INFINITY;
  for (int c = t; c < V; c += 256) mx = fmaxf(mx, x[c] / temperature);
  mx = warp_max(mx);
  if (lane == 0) red[warp] = mx;
  __syncthreads();
  mx = red[0];
#pragma unroll
  for (int w = 1; w < 8; ++w) mx = fmaxf(mx, red[w]);
  if (top_p < 1.f) {
    // keys >= thr stay kept when the mass above them is <= budget = top_p * (kept mass).  Each pass picks the lowest bucket
    // whose mass above (s_above + the buckets higher in this pass) is within the budget: the threshold key lies in it,
    // since every key of a lower bucket has at least that bucket's mass above it.  Zero-mass buckets are skipped: exp is
    // monotone, so they lie below every positive mass and have the whole kept mass above them.
    uint32_t prefix = 0, mask = 0;
    unsigned long long above = 0;
    for (int pass = 3; pass >= 0; --pass) {
      const int shift = pass * 8;
      mhist[t] = 0ull;
      __syncthreads();
      for (int c = t; c < V; c += 256) {
        const float z = x[c] / temperature;
        const uint32_t key = order_key(z);
        if (key >= thr && (key & mask) == prefix) {
          const unsigned long long q = __float2ull_rz(expf(z - mx) * MASS_ONE);
          if (q) atomicAdd(&mhist[(key >> shift) & 255u], q);
        }
      }
      __syncthreads();
      if (warp == 0) {                                // lane l owns buckets 8l .. 8l+7; integer sums: any order gives the same bits
        unsigned long long m[8], loc = 0;
#pragma unroll
        for (int j = 0; j < 8; ++j) loc += (m[j] = mhist[8 * lane + j]);
        if (pass == 3) {
          unsigned long long total = loc;
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) total += __shfl_xor_sync(0xffffffffu, total, o);
          if (lane == 0) s_budget = (unsigned long long)((double)total * (double)top_p);
          __syncwarp();
        }
        unsigned long long suf = loc;                 // mass of lanes >= l, then of the buckets above 8l+7
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const unsigned long long v = __shfl_down_sync(0xffffffffu, suf, o);
          if (lane + o < 32) suf += v;
        }
        const unsigned long long budget = s_budget;
        unsigned long long run = above + (suf - loc), pick_above = 0;
        int pick = 256;
#pragma unroll
        for (int j = 7; j >= 0; --j) {               // the mass above a bucket only grows downwards: the last fit is the lowest
          if (m[j] && run <= budget) { pick = 8 * lane + j; pick_above = run; }
          run += m[j];
        }
        const int low = (int)__reduce_min_sync(0xffffffffu, (unsigned)pick);
        if (pick == low) {                            // exactly one lane; one always fits (the top bucket's mass above is <= budget)
          s_prefix = prefix | ((uint32_t)pick << shift);
          s_above = pick_above;
        }
      }
      __syncthreads();
      prefix = s_prefix;
      above = s_above;
      mask |= 0xFFu << shift;
      __syncthreads();
    }
    thr = prefix;
  }
  // contiguous chunks per thread so that the running sum follows the index order
  const int per = (V + 255) / 256, c0 = t * per, c1 = min(V, c0 + per);
  float loc = 0.f;
  for (int c = c0; c < c1; ++c) {
    const float z = x[c] / temperature;
    if (order_key(z) >= thr) loc += expf(z - mx);
  }
  csum[t] = loc;
  __syncthreads();
  if (t == 0) {
    float total = 0.f;
    for (int j = 0; j < 256; ++j) total += csum[j];
    const float ur = (ROWS && rc.seeds) ? seeded_uniform(rc.seeds[blockIdx.x], rc.position) : u[blockIdx.x];
    const float target = ur * total;
    float run = 0.f;
    int j = 0, last_chunk = 0;
    for (; j < 256; ++j) {
      if (csum[j] > 0.f) last_chunk = j;
      if (run + csum[j] > target) break;
      run += csum[j];
    }
    if (j == 256) {              // rounding pushed the target to the total: the last kept entry
      j = last_chunk;
      run = -INFINITY;
    }
    int pick = -1, last_kept = -1;
    const int a0 = j * per, a1 = min(V, a0 + per);
    for (int c = a0; c < a1; ++c) {
      const float z = x[c] / temperature;
      if (order_key(z) >= thr) {
        last_kept = c;
        run += expf(z - mx);
        if (run > target) { pick = c; break; }
      }
    }
    const int drawn = pick >= 0 ? pick : last_kept;
    tok[blockIdx.x] = (int64_t)drawn;
    if (logp) logp[(int64_t)blockIdx.x * lpld] = (x[drawn] / temperature - mx) - logf(total);
  }
}

// K-split variant for long rows and few outputs (MLP.lin2: N = 1024, K = 4096 gives only 128 blocks of the kernel above
// and a 16 KB latency-bound stream per warp): a block owns two outputs, four warps each split one row of W, partials are
// folded in a fixed order (deterministic).
template <int R>
__global__ void __launch_bounds__(256) linear_small_ks_kernel(const float* __restrict__ x, int64_t ldx, const float* __restrict__ W,
                                                              const float* __restrict__ bias, float* __restrict__ y, int64_t ldy, int N,
                                                              int K, int act) {
  __shared__ float part[8][R];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n = blockIdx.x * 2 + (warp >> 2), slice = warp & 3;
  const int K4 = K >> 2, per = (K4 + 3) / 4, k0 = slice * per, k1 = min(K4, k0 + per);
  float acc[R];
#pragma unroll
  for (int r = 0; r < R; ++r) acc[r] = 0.f;
  if (n < N) {
    const float4* w4 = reinterpret_cast<const float4*>(W + (size_t)n * K);
    int k = k0 + lane;
    for (; k + 224 < k1; k += 256) {
      float4 wv[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) wv[u] = __ldg(w4 + k + 32 * u);
#pragma unroll
      for (int u = 0; u < 8; ++u)
#pragma unroll
        for (int r = 0; r < R; ++r) {
          const float4 xv = __ldg(reinterpret_cast<const float4*>(x + (size_t)r * ldx) + k + 32 * u);
          acc[r] = fmaf(wv[u].x, xv.x, acc[r]); acc[r] = fmaf(wv[u].y, xv.y, acc[r]);
          acc[r] = fmaf(wv[u].z, xv.z, acc[r]); acc[r] = fmaf(wv[u].w, xv.w, acc[r]);
        }
    }
    for (; k < k1; k += 32) {
      const float4 wv = __ldg(w4 + k);
#pragma unroll
      for (int r = 0; r < R; ++r) {
        const float4 xv = __ldg(reinterpret_cast<const float4*>(x + (size_t)r * ldx) + k);
        acc[r] = fmaf(wv.x, xv.x, acc[r]); acc[r] = fmaf(wv.y, xv.y, acc[r]);
        acc[r] = fmaf(wv.z, xv.z, acc[r]); acc[r] = fmaf(wv.w, xv.w, acc[r]);
      }
    }
  }
#pragma unroll
  for (int r = 0; r < R; ++r) acc[r] = warp_sum(acc[r]);
  if (lane == 0)
#pragma unroll
    for (int r = 0; r < R; ++r) part[warp][r] = acc[r];
  __syncthreads();
  if (threadIdx.x < 2 * R) {
    const int o = threadIdx.x / R, r = threadIdx.x % R, nn = blockIdx.x * 2 + o;
    if (nn < N) {
      float v = ((part[o * 4 + 0][r] + part[o * 4 + 1][r]) + (part[o * 4 + 2][r] + part[o * 4 + 3][r])) + (bias ? __ldg(bias + nn) : 0.f);
      if (act == 1) {
        const float u = 0.7978845608028654f * v * (1.f + 0.044715f * v * v);
        v = 0.5f * v * (1.f + tanhf(u));
      }
      y[(size_t)r * ldy + nn] = v;
    }
  }
}

template <int R>
int linear_small_run(const float* x, int64_t ldx, const float* W, const float* bias, float* y, int64_t ldy, int N, int K, int act,
                     cudaStream_t st) {
  if (K >= 2048 && N <= 2048) {
    linear_small_ks_kernel<R><<<(int)cdiv(N, 2), 256, 0, st>>>(x, ldx, W, bias, y, ldy, N, K, act);
    return launched("linear_small_ks");
  }
  linear_small_kernel<R><<<(int)cdiv(N, 8), 256, 0, st>>>(x, ldx, W, bias, y, ldy, N, K, act);
  return launched("linear_small");
}

}  // namespace

extern "C" {

int mas_linear_small(const float* x, int64_t ldx, const float* W, const float* bias, float* y, int64_t ldy, int R, int N, int K, int act,
                     void* stream) {
  MAS_REQUIRE(x && W && y && R > 0 && N > 0 && K > 0, "linear_small: bad arguments");
  if (R > LS_MAXR) return fail(MAS_ERR_UNSUPPORTED, "linear_small: at most %d rows (got %d); use mas_gemm_rows_packed", LS_MAXR, R);
  if (K % 4 || ldx % 4 || (reinterpret_cast<uintptr_t>(x) & 15) || (reinterpret_cast<uintptr_t>(W) & 15))
    return fail(MAS_ERR_UNSUPPORTED, "linear_small: K and ldx must be multiples of 4 and x / W 16-byte aligned");
  if (act != 0 && act != 1) return fail(MAS_ERR_INVALID_ARG, "linear_small: act must be 0 (none) or 1 (tanh-GELU)");
  cudaStream_t st = S(stream);
  switch (R) {
    case 1: return linear_small_run<1>(x, ldx, W, bias, y, ldy, N, K, act, st);
    case 2: return linear_small_run<2>(x, ldx, W, bias, y, ldy, N, K, act, st);
    case 3: return linear_small_run<3>(x, ldx, W, bias, y, ldy, N, K, act, st);
    case 4: return linear_small_run<4>(x, ldx, W, bias, y, ldy, N, K, act, st);
    case 5: return linear_small_run<5>(x, ldx, W, bias, y, ldy, N, K, act, st);
    case 6: return linear_small_run<6>(x, ldx, W, bias, y, ldy, N, K, act, st);
    case 7: return linear_small_run<7>(x, ldx, W, bias, y, ldy, N, K, act, st);
    default: return linear_small_run<8>(x, ldx, W, bias, y, ldy, N, K, act, st);
  }
}

}  // extern "C"

template <typename T>
static int kv_append_run(const float* qkv, int R, int T_, int heads, int hd, T* kcache, T* vcache, int Tmax, int pos0, void* stream) {
  MAS_REQUIRE(qkv && kcache && vcache && R > 0 && T_ > 0 && heads > 0 && hd > 0, "kv_append: bad arguments");
  if (hd % 4) return fail(MAS_ERR_UNSUPPORTED, "kv_append: head dim %% 4 != 0");
  if (pos0 < 0 || pos0 + T_ > Tmax) return fail(MAS_ERR_INVALID_ARG, "kv_append: positions %d..%d outside the cache (%d)", pos0, pos0 + T_, Tmax);
  const int64_t total = (int64_t)R * T_ * heads * (hd / 4);
  kv_append_kernel<T><<<(int)(cdiv(total, 256) < 2368 ? cdiv(total, 256) : 2368), 256, 0, S(stream)>>>(qkv, R, T_, heads, hd, kcache,
                                                                                                    vcache, Tmax, pos0);
  return launched("kv_append");
}

template <typename T>
static int attn_decode_run(const float* qkv, T* kcache, T* vcache, float* ctx, int R, int heads, int hd, int Tmax, int len,
                           bool append, void* stream) {
  MAS_REQUIRE(qkv && kcache && vcache && ctx && R > 0 && heads > 0, "attn_decode: bad arguments");
  if (len <= 0 || len > Tmax) return fail(MAS_ERR_INVALID_ARG, "attn_decode: cache length %d outside (0, %d]", len, Tmax);
  const size_t smem = (size_t)(hd + ((len + 3) & ~3) + 32 + 256 * Vec16<T>::E + 2 * hd) * sizeof(float);
  if (smem > 48 * 1024) return fail(MAS_ERR_UNSUPPORTED, "attn_decode: sequence too long for the single-pass kernel (%d)", len);
  const int grid = R * heads;
#define MAS_AD(HD_)                                                                                                           \
  if (append) attn_decode_kernel<HD_, true, T><<<grid, 256, smem, S(stream)>>>(qkv, kcache, vcache, ctx, heads, Tmax, len); \
  else attn_decode_kernel<HD_, false, T><<<grid, 256, smem, S(stream)>>>(qkv, kcache, vcache, ctx, heads, Tmax, len)
  switch (hd) {
    case 16: MAS_AD(16); break;
    case 32: MAS_AD(32); break;
    case 64: MAS_AD(64); break;
    case 128: MAS_AD(128); break;
    default: return fail(MAS_ERR_UNSUPPORTED, "attn_decode: head dim %d (supported: 16, 32, 64, 128)", hd);
  }
#undef MAS_AD
  return launched(append ? "attn_decode_append" : "attn_decode");
}

template <typename T>
static size_t shared_decode_smem(int G, int hd, int len) {
  return (size_t)G * (3 * hd + 16 + ((len + 3) & ~3) + 256 * Vec16<T>::E) * sizeof(float);
}

template <int HD, int G, bool APPEND, typename T>
static int attn_decode_shared_launch(const float* qkv, const T* kp, const T* vp, T* ks, T* vs, float* ctx, int R, int n, int heads, int P,
                                     int Tsuf, int len, int optin, size_t smem, cudaStream_t st) {
  static std::atomic<uint64_t> configured{0};    // per instantiation and device: allow the device's largest dynamic shared memory
  if (first_on_device(configured)) {
    const cudaError_t e = cudaFuncSetAttribute(attn_decode_shared_kernel<HD, G, APPEND, T>, cudaFuncAttributeMaxDynamicSharedMemorySize, optin);
    if (e != cudaSuccess) return fail(MAS_ERR_LAUNCH, "attn_decode_shared: smem attr (%d): %s", optin, cudaGetErrorString(e));
    mark_device(configured);
  }
  const int grid = (R / n) * heads * ((n + G - 1) / G);
  attn_decode_shared_kernel<HD, G, APPEND, T><<<grid, 256, smem, st>>>(qkv, kp, vp, ks, vs, ctx, n, heads, P, Tsuf, len);
  return launched(APPEND ? "attn_decode_shared_append" : "attn_decode_shared");
}

// Rows per block: a block of G rows reads its group's prefix once for G rows, but a group of n rows then fills only
// ceil(n / G) blocks per head. Auto (rows_per_block = 0): the smallest power of two >= n, capped at 4, halved while the grid
// would be under two blocks per SM or the block's shared memory would exceed the device's opt-in limit.  The cap is measured
// (tools/bench_decode.py, H100 SXM 80 GB, 700 W, 256 rows, n = 8, 16 x 64 heads, length 512): 8 rows per block took 155 us
// against 121 us for one row, its 4 KB of v partials per row costing occupancy; 4 rows per block beat one row at every n.
// len: positions attended (the last one is this token's, at suffix slot len-1-P: stored here when append, else already cached).
template <typename T>
static int attn_decode_shared_run(const float* qkv, const T* kp, const T* vp, T* ks, T* vs, float* ctx, int R, int n, int heads, int hd,
                                  int P, int Tsuf, int len, bool append, int rows_per_block, void* stream) {
  MAS_REQUIRE(qkv && kp && vp && ks && vs && ctx && R > 0 && heads > 0, "attn_decode_shared: bad arguments");
  if (n < 1 || R % n) return fail(MAS_ERR_INVALID_ARG, "attn_decode_shared: %d rows are not groups of %d", R, n);
  if (P < 1 || Tsuf < 1 || len <= P || len > P + Tsuf)
    return fail(MAS_ERR_INVALID_ARG, "attn_decode_shared: position %d outside the suffix cache (%d..%d)", len - 1, P, P + Tsuf - 1);
  if (rows_per_block != 0 && rows_per_block != 1 && rows_per_block != 2 && rows_per_block != 4)
    return fail(MAS_ERR_INVALID_ARG, "attn_decode_shared: rows_per_block must be 0 (auto), 1, 2 or 4 (got %d)", rows_per_block);
  int dev = 0, sms = 0, optin = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev);
  int G = rows_per_block;
  if (G == 0) {
    G = 4;
    while (G > 1 && G / 2 >= n) G /= 2;
    while (G > 1 && ((size_t)(R / n) * heads * ((n + G - 1) / G) < (size_t)2 * sms || shared_decode_smem<T>(G, hd, len) > (size_t)optin)) G /= 2;
  }
  const size_t smem = shared_decode_smem<T>(G, hd, len);
  if (smem > (size_t)optin)
    return fail(MAS_ERR_UNSUPPORTED, "attn_decode_shared: %d rows per block over %d positions need %zu bytes of shared memory", G, len,
                smem);
  cudaStream_t st = S(stream);
#define MAS_ADS_G(HD_, G_)                                                                                                   \
  return append ? attn_decode_shared_launch<HD_, G_, true, T>(qkv, kp, vp, ks, vs, ctx, R, n, heads, P, Tsuf, len, optin, smem, st) \
                : attn_decode_shared_launch<HD_, G_, false, T>(qkv, kp, vp, ks, vs, ctx, R, n, heads, P, Tsuf, len, optin, smem, st);
#define MAS_ADS(HD_)              \
  switch (G) {                    \
    case 1: MAS_ADS_G(HD_, 1)     \
    case 2: MAS_ADS_G(HD_, 2)     \
    default: MAS_ADS_G(HD_, 4)    \
  }
  switch (hd) {
    case 16: MAS_ADS(16)
    case 32: MAS_ADS(32)
    case 64: MAS_ADS(64)
    case 128: MAS_ADS(128)
    default: return fail(MAS_ERR_UNSUPPORTED, "attn_decode_shared: head dim %d (supported: 16, 32, 64, 128)", hd);
  }
#undef MAS_ADS
#undef MAS_ADS_G
}

extern "C" {

int mas_attn_decode_shared_append(const float* qkv, const float* kprefix, const float* vprefix, float* ksuffix, float* vsuffix, float* ctx,
                                  int R, int n, int heads, int hd, int prefix_len, int Tsuf, int pos, int rows_per_block, void* stream) {
  return attn_decode_shared_run(qkv, kprefix, vprefix, ksuffix, vsuffix, ctx, R, n, heads, hd, prefix_len, Tsuf, pos + 1, true,
                                rows_per_block, stream);
}

int mas_attn_decode_shared_append_f16(const float* qkv, const void* kprefix, const void* vprefix, void* ksuffix, void* vsuffix, float* ctx,
                                      int R, int n, int heads, int hd, int prefix_len, int Tsuf, int pos, int rows_per_block,
                                      void* stream) {
  return attn_decode_shared_run(qkv, (const __half*)kprefix, (const __half*)vprefix, (__half*)ksuffix, (__half*)vsuffix, ctx, R, n, heads,
                                hd, prefix_len, Tsuf, pos + 1, true, rows_per_block, stream);
}

int mas_attn_decode_shared(const float* qkv, const float* kprefix, const float* vprefix, const float* ksuffix, const float* vsuffix,
                           float* ctx, int R, int n, int heads, int hd, int prefix_len, int Tsuf, int len, int rows_per_block, void* stream) {
  return attn_decode_shared_run(qkv, kprefix, vprefix, const_cast<float*>(ksuffix), const_cast<float*>(vsuffix), ctx, R, n, heads, hd,
                                prefix_len, Tsuf, len, false, rows_per_block, stream);
}

int mas_attn_decode_shared_f16(const float* qkv, const void* kprefix, const void* vprefix, const void* ksuffix, const void* vsuffix,
                               float* ctx, int R, int n, int heads, int hd, int prefix_len, int Tsuf, int len, int rows_per_block,
                               void* stream) {
  return attn_decode_shared_run(qkv, (const __half*)kprefix, (const __half*)vprefix, (__half*)const_cast<void*>(ksuffix),
                                (__half*)const_cast<void*>(vsuffix), ctx, R, n, heads, hd, prefix_len, Tsuf, len, false, rows_per_block,
                                stream);
}

int mas_kv_append(const float* qkv, int R, int T, int heads, int hd, float* kcache, float* vcache, int Tmax, int pos0, void* stream) {
  return kv_append_run(qkv, R, T, heads, hd, kcache, vcache, Tmax, pos0, stream);
}

int mas_kv_append_f16(const float* qkv, int R, int T, int heads, int hd, void* kcache, void* vcache, int Tmax, int pos0, void* stream) {
  return kv_append_run(qkv, R, T, heads, hd, (__half*)kcache, (__half*)vcache, Tmax, pos0, stream);
}

int mas_attn_decode(const float* qkv, const float* kcache, const float* vcache, float* ctx, int R, int heads, int hd, int Tmax, int len,
                    void* stream) {
  return attn_decode_run(qkv, const_cast<float*>(kcache), const_cast<float*>(vcache), ctx, R, heads, hd, Tmax, len, false, stream);
}

int mas_attn_decode_f16(const float* qkv, const void* kcache, const void* vcache, float* ctx, int R, int heads, int hd, int Tmax, int len,
                        void* stream) {
  return attn_decode_run(qkv, (__half*)const_cast<void*>(kcache), (__half*)const_cast<void*>(vcache), ctx, R, heads, hd, Tmax, len, false,
                         stream);
}

int mas_attn_decode_append(const float* qkv, float* kcache, float* vcache, float* ctx, int R, int heads, int hd, int Tmax, int pos,
                           void* stream) {
  if (pos < 0 || pos >= Tmax) return fail(MAS_ERR_INVALID_ARG, "attn_decode_append: position %d outside the cache (%d)", pos, Tmax);
  return attn_decode_run(qkv, kcache, vcache, ctx, R, heads, hd, Tmax, pos + 1, true, stream);
}

int mas_attn_decode_append_f16(const float* qkv, void* kcache, void* vcache, float* ctx, int R, int heads, int hd, int Tmax, int pos,
                               void* stream) {
  if (pos < 0 || pos >= Tmax) return fail(MAS_ERR_INVALID_ARG, "attn_decode_append: position %d outside the cache (%d)", pos, Tmax);
  return attn_decode_run(qkv, (__half*)kcache, (__half*)vcache, ctx, R, heads, hd, Tmax, pos + 1, true, stream);
}

int mas_cfg_mix(const float* cond, const float* uncond, float* out, int64_t n, float scale, void* stream) {
  MAS_REQUIRE(cond && uncond && out && n > 0, "cfg_mix: bad arguments");
  cfg_mix_kernel<<<(int)(cdiv(n, 256) < 1184 ? cdiv(n, 256) : 1184), 256, 0, S(stream)>>>(cond, uncond, out, n, scale);
  return launched("cfg_mix");
}

int mas_cfg_mix_rows(const float* cond, const float* uncond, float* out, int R, int64_t V, const float* scale, void* stream) {
  MAS_REQUIRE(cond && uncond && out && scale && R > 0 && V > 0, "cfg_mix_rows: bad arguments");
  const int gy = R < 65535 ? R : 65535;
  const int64_t gx_max = 1184 / gy > 0 ? 1184 / gy : 1;
  const int gx = (int)(cdiv(V, 256) < gx_max ? cdiv(V, 256) : gx_max);
  cfg_mix_rows_kernel<<<dim3(gx, gy), 256, 0, S(stream)>>>(cond, uncond, out, R, V, scale);
  return launched("cfg_mix_rows");
}

int mas_sample_topk(const float* logits, int64_t ld, int R, int V, float temperature, int top_k, const float* u, int64_t* tokens,
                    void* stream) {
  MAS_REQUIRE(logits && u && tokens && R > 0 && V > 0 && ld >= V, "sample_topk: bad arguments");
  if (!(temperature > 0.f)) return fail(MAS_ERR_INVALID_ARG, "sample_topk: temperature must be > 0 (greedy decoding: top_k = 1)");
  sample_topk_kernel<false><<<R, 256, 0, S(stream)>>>(logits, ld, V, temperature, top_k, 1.f, u, nullptr, nullptr, 0, tokens, nullptr, 0,
                                                      RowControls{});
  return launched("sample_topk");
}

static int sample_filtered_run(const char* name, const float* logits, int64_t ld, int R, int V, float temperature, int top_k,
                               float top_p, const float* u, const int64_t* prompt_tokens, const uint8_t* prompt_mask,
                               int64_t prompt_ld, int64_t* tokens, float* logp, int64_t logp_ld, void* stream) {
  if (!(logits && tokens && R > 0 && V > 0 && ld >= V)) return fail(MAS_ERR_INVALID_ARG, "%s: bad arguments", name);
  if (!(temperature >= 0.f)) return fail(MAS_ERR_INVALID_ARG, "%s: temperature must be >= 0 (0: greedy)", name);
  if (temperature > 0.f && !u) return fail(MAS_ERR_INVALID_ARG, "%s: sampling (temperature > 0) needs the uniforms u", name);
  if (!(top_p > 0.f)) return fail(MAS_ERR_INVALID_ARG, "%s: top_p must be > 0 (>= 1: no nucleus filter)", name);
  if (!prompt_tokens != !prompt_mask) return fail(MAS_ERR_INVALID_ARG, "%s: prompt tokens and prompt mask go together", name);
  if (prompt_mask && prompt_ld < 0) return fail(MAS_ERR_INVALID_ARG, "%s: negative prompt row stride", name);
  if (logp && logp_ld < 0) return fail(MAS_ERR_INVALID_ARG, "%s: negative log-probability row stride", name);
  sample_topk_kernel<false><<<R, 256, 0, S(stream)>>>(logits, ld, V, temperature, top_k, top_p, u, prompt_tokens, prompt_mask,
                                                      prompt_ld, tokens, logp, logp_ld, RowControls{});
  return launched(name);
}

int mas_sample_filtered(const float* logits, int64_t ld, int R, int V, float temperature, int top_k, float top_p, const float* u,
                        const int64_t* prompt_tokens, const uint8_t* prompt_mask, int64_t prompt_ld, int64_t* tokens, void* stream) {
  return sample_filtered_run("sample_filtered", logits, ld, R, V, temperature, top_k, top_p, u, prompt_tokens, prompt_mask,
                             prompt_ld, tokens, nullptr, 0, stream);
}

int mas_sample_filtered_logp(const float* logits, int64_t ld, int R, int V, float temperature, int top_k, float top_p,
                             const float* u, const int64_t* prompt_tokens, const uint8_t* prompt_mask, int64_t prompt_ld,
                             int64_t* tokens, float* logp, int64_t logp_ld, void* stream) {
  if (!logp) return fail(MAS_ERR_INVALID_ARG, "sample_filtered_logp: logp is NULL (mas_sample_filtered draws without it)");
  return sample_filtered_run("sample_filtered_logp", logits, ld, R, V, temperature, top_k, top_p, u, prompt_tokens, prompt_mask,
                             prompt_ld, tokens, logp, logp_ld, stream);
}

int mas_sample_rows(const float* logits, int64_t ld, int R, int V, const float* temperature, const int* top_k, const float* top_p,
                    const float* u, const int64_t* seeds, int64_t position, const int64_t* prompt_tokens, const uint8_t* prompt_mask,
                    int64_t prompt_ld, int64_t* tokens, float* logp, int64_t logp_ld, void* stream) {
  if (!(logits && tokens && R > 0 && V > 0 && ld >= V)) return fail(MAS_ERR_INVALID_ARG, "sample_rows: bad arguments");
  if (!(temperature && top_k && top_p)) return fail(MAS_ERR_INVALID_ARG, "sample_rows: temperature, top_k and top_p are [R] arrays");
  if (!u == !seeds) return fail(MAS_ERR_INVALID_ARG, "sample_rows: give exactly one source of uniforms, u or seeds");
  if (!prompt_tokens != !prompt_mask) return fail(MAS_ERR_INVALID_ARG, "sample_rows: prompt tokens and prompt mask go together");
  if (prompt_mask && prompt_ld < 0) return fail(MAS_ERR_INVALID_ARG, "sample_rows: negative prompt row stride");
  if (logp && logp_ld < 0) return fail(MAS_ERR_INVALID_ARG, "sample_rows: negative log-probability row stride");
  sample_topk_kernel<true><<<R, 256, 0, S(stream)>>>(logits, ld, V, 0.f, 0, 1.f, u, prompt_tokens, prompt_mask, prompt_ld, tokens, logp,
                                                     logp_ld, RowControls{temperature, top_k, top_p, seeds, position});
  return launched("sample_rows");
}

}  // extern "C"
