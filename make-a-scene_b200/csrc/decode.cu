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
//   * mas_cfg_mix      : classifier-free guidance, out = uncond + scale * (cond - uncond).
#include <cuda_fp16.h>

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

__global__ void cfg_mix_kernel(const float* __restrict__ cond, const float* __restrict__ uncond, float* __restrict__ out, int64_t n,
                               float scale) {
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) {
    const float u = uncond[i];
    out[i] = fmaf(scale, cond[i] - u, u);
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
__device__ __forceinline__ uint32_t order_key(float f) {
  const uint32_t b = __float_as_uint(f);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
constexpr float MASS_ONE = 1099511627776.f;          // 2^40: the largest entry's mass exp(0)
__global__ void __launch_bounds__(256) sample_topk_kernel(const float* __restrict__ logits, int64_t ld, int V, float temperature, int top_k,
                                                          float top_p, const float* __restrict__ u, const int64_t* __restrict__ ptok,
                                                          const uint8_t* __restrict__ pmask, int64_t pld, int64_t* __restrict__ tok) {
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
    if (t == 0) tok[blockIdx.x] = ptok[(int64_t)blockIdx.x * pld];
    return;
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
    const float target = u[blockIdx.x] * total;
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
    tok[blockIdx.x] = (int64_t)(pick >= 0 ? pick : last_kept);
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

extern "C" {

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

int mas_sample_topk(const float* logits, int64_t ld, int R, int V, float temperature, int top_k, const float* u, int64_t* tokens,
                    void* stream) {
  MAS_REQUIRE(logits && u && tokens && R > 0 && V > 0 && ld >= V, "sample_topk: bad arguments");
  if (!(temperature > 0.f)) return fail(MAS_ERR_INVALID_ARG, "sample_topk: temperature must be > 0 (greedy decoding: top_k = 1)");
  sample_topk_kernel<<<R, 256, 0, S(stream)>>>(logits, ld, V, temperature, top_k, 1.f, u, nullptr, nullptr, 0, tokens);
  return launched("sample_topk");
}

int mas_sample_filtered(const float* logits, int64_t ld, int R, int V, float temperature, int top_k, float top_p, const float* u,
                        const int64_t* prompt_tokens, const uint8_t* prompt_mask, int64_t prompt_ld, int64_t* tokens, void* stream) {
  MAS_REQUIRE(logits && tokens && R > 0 && V > 0 && ld >= V, "sample_filtered: bad arguments");
  if (!(temperature >= 0.f)) return fail(MAS_ERR_INVALID_ARG, "sample_filtered: temperature must be >= 0 (0: greedy)");
  if (temperature > 0.f && !u) return fail(MAS_ERR_INVALID_ARG, "sample_filtered: sampling (temperature > 0) needs the uniforms u");
  if (!(top_p > 0.f)) return fail(MAS_ERR_INVALID_ARG, "sample_filtered: top_p must be > 0 (>= 1: no nucleus filter)");
  if (!prompt_tokens != !prompt_mask) return fail(MAS_ERR_INVALID_ARG, "sample_filtered: prompt tokens and prompt mask go together");
  if (prompt_mask && prompt_ld < 0) return fail(MAS_ERR_INVALID_ARG, "sample_filtered: negative prompt row stride");
  sample_topk_kernel<<<R, 256, 0, S(stream)>>>(logits, ld, V, temperature, top_k, top_p, u, prompt_tokens, prompt_mask, prompt_ld,
                                               tokens);
  return launched("sample_filtered");
}

}  // extern "C"
