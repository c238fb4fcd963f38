// Compact scene maps on the output side of VQ-SEG: the 159 logits of a pixel decoded into the four label planes mas_scene_expand
// reads (mas_scene_decode), and the per-plane confusion matrices of a decoded map against a target map (mas_scene_confusion),
// from which per-class IoU follows.  Both are HBM-bound.
//
// The rule (include/mas_b200.h): a channel is "on" when its logit is > 0, the BCE decision boundary sigma(x) = 0.5.  Each
// one-hot plane is 1 + the argmax of its channel group when that maximum is > 0, else 0; edges are 1 when x[158] > 0.  The
// argmax compares order keys: the float's bits mapped monotonically onto unsigned ints, -0 folded onto +0 (so the two zeros
// tie, as in torch.argmax) and NaN mapped to 0, below every number, so that a NaN never wins and is never > 0.  Ties go to the
// lowest channel.
#include <cuda_runtime.h>

#include <algorithm>

#include "mas_common.cuh"

namespace mas {
namespace scene {

constexpr int C = 159;
constexpr unsigned KEY_ZERO = 0x80000000u;   // key(+0) = key(-0); key(x) > KEY_ZERO  <=>  x > 0
constexpr unsigned NO_INDEX = 0xffffffffu;

__device__ __forceinline__ unsigned order_key(float x) {
  if (x != x) return 0u;
  if (x == 0.f) return KEY_ZERO;
  const unsigned u = __float_as_uint(x);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ unsigned code_of(unsigned key, unsigned idx) { return key > KEY_ZERO ? idx + 1u : 0u; }

// Padded channels-last logits (sc == 1; one pixel = C contiguous floats): a block covers up to 32 consecutive pixels of one
// image row, each warp 4 of them.  Lane l holds channels l + 32k (k = 0..4; lane 31 never reads channel 159, the pad): all 20
// loads of a warp are issued before any reduction.  Per plane the warp reduces the lanes' best keys with one redux.sync max and
// the lowest channel holding that key with one redux.sync min.  The codes are staged in shared memory and written as 32-byte
// rows of the four output planes.
__global__ void __launch_bounds__(256) decode_cl_kernel(const float* __restrict__ x, mas_tensor4 xs, uint8_t* __restrict__ out) {
  __shared__ uint8_t s[4][32];
  const int w0 = blockIdx.x * 32, h = blockIdx.y, n = blockIdx.z;
  const int W = (int)xs.w, npx = min(32, W - w0);
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned full = 0xffffffffu;
  float v[4][5];
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int px = warp * 4 + j;
    const float* p = x + n * xs.sn + (int64_t)h * xs.sh + (int64_t)(w0 + px) * xs.sw + lane;
#pragma unroll
    for (int k = 0; k < 5; ++k) v[j][k] = (px < npx && (k < 4 || lane < 31)) ? __ldcs(p + 32 * k) : 0.f;
  }
#pragma unroll
  for (int j = 0; j < 4; ++j) {
    const int px = warp * 4 + j;
    if (px >= npx) break;   // uniform across the warp
    // panoptic: channels lane + 32k for k < 4, and 128 + lane for lane < 5; ascending channel per lane, so > keeps the lowest
    unsigned best = order_key(v[j][0]), bi = lane;
#pragma unroll
    for (int k = 1; k < 5; ++k) {
      const unsigned key = (k < 4 || lane < 5) ? order_key(v[j][k]) : 0u;
      if (key > best) best = key, bi = lane + 32 * k;
    }
    const unsigned k4 = order_key(v[j][4]);
    const unsigned hk = (lane >= 5 && lane < 25) ? k4 : 0u, fk = (lane >= 25 && lane < 30) ? k4 : 0u;
    const unsigned pm = __reduce_max_sync(full, best), hm = __reduce_max_sync(full, hk), fm = __reduce_max_sync(full, fk);
    const unsigned pi = __reduce_min_sync(full, best == pm ? bi : NO_INDEX);
    const unsigned hi = __reduce_min_sync(full, hk == hm ? (unsigned)lane - 5u : NO_INDEX);
    const unsigned fi = __reduce_min_sync(full, fk == fm ? (unsigned)lane - 25u : NO_INDEX);
    const bool edge = __ballot_sync(full, lane == 30 && k4 > KEY_ZERO) != 0u;
    if (lane == 0) {
      s[0][px] = (uint8_t)code_of(pm, pi);
      s[1][px] = (uint8_t)code_of(hm, hi);
      s[2][px] = (uint8_t)code_of(fm, fi);
      s[3][px] = edge ? 1 : 0;
    }
  }
  __syncthreads();
  if (threadIdx.x < 128) {
    const int p = threadIdx.x >> 5, px = threadIdx.x & 31;
    const int64_t H = xs.h;
    if (px < npx) out[(((int64_t)n * 4 + p) * H + h) * W + w0 + px] = s[p][px];
  }
}

// Any other strides: one thread per pixel walks its 159 channels (lanes on consecutive w, so NCHW planes are read as
// 128-byte rows).  The same keys and comparisons, so the same codes bit for bit.
__device__ __forceinline__ unsigned group_code(const float* __restrict__ p, int64_t sc, int c0, int c1) {
  unsigned best = 0u, bi = 0u;
  for (int c = c0; c < c1; ++c) {
    const unsigned key = order_key(__ldg(p + c * sc));
    if (key > best) best = key, bi = (unsigned)(c - c0);
  }
  return code_of(best, bi);
}
__global__ void __launch_bounds__(128) decode_strided_kernel(const float* __restrict__ x, mas_tensor4 xs, uint8_t* __restrict__ out) {
  const int w = blockIdx.x * 32 + threadIdx.x, h = blockIdx.y * 4 + threadIdx.y, n = blockIdx.z;
  const int64_t H = xs.h, W = xs.w;
  if (w >= W || h >= H) return;
  const float* p = x + n * xs.sn + h * xs.sh + w * xs.sw;
  uint8_t* o = out + ((int64_t)n * 4 * H + h) * W + w;
  o[0] = (uint8_t)group_code(p, xs.sc, 0, 133);
  o[H * W] = (uint8_t)group_code(p, xs.sc, 133, 153);
  o[2 * H * W] = (uint8_t)group_code(p, xs.sc, 153, 158);
  o[3 * H * W] = __ldg(p + 158 * xs.sc) > 0.f ? 1 : 0;
}

// Confusion matrices, target row x prediction column, in one int64 buffer:
//   [0, 17956) panoptic 134 x 134 | [17956, 18397) human 21 x 21 | [18397, 18433) face 6 x 6 | [18433, 18437) edges 2 x 2 |
//   [18437] pixels with a plane counted nowhere (its target or prediction byte out of the plane's range; at most 1 a pixel).
// A block accumulates u32 counts in shared memory (73.8 KB), then adds its non-zero counts into conf with 64-bit integer
// atomics: integer sums are exact, so the result does not depend on the order.  The dominant "none -> none" cell of every plane,
// the edge cells and the out-of-range count are counted per warp with a ballot; the other cells take shared-memory atomics.
// Every count of a block is at most its number of pixels, kept <= 2^30 by the launch, so no u32 count can overflow.
constexpr int PAN = 134, HUM = 21, FACE = 6;
constexpr int OFF_HUM = PAN * PAN, OFF_FACE = OFF_HUM + HUM * HUM, OFF_EDGE = OFF_FACE + FACE * FACE, OFF_BAD = OFF_EDGE + 4;
constexpr int CONF_LEN = OFF_BAD + 1;
constexpr int CF_THREADS = 512;
static_assert(CONF_LEN == 18438, "confusion layout");

__global__ void __launch_bounds__(CF_THREADS) confusion_kernel(const uint8_t* __restrict__ pred, const uint8_t* __restrict__ target,
                                                              int64_t P, int64_t total, int64_t per_block, unsigned long long* __restrict__ conf) {
  extern __shared__ unsigned hist[];
  for (int i = threadIdx.x; i < CONF_LEN; i += CF_THREADS) hist[i] = 0u;
  __syncthreads();
  const unsigned full = 0xffffffffu;
  const int lane = threadIdx.x & 31;
  const int64_t q0 = (int64_t)blockIdx.x * per_block, q1 = min(total, q0 + per_block);
  for (int64_t base = q0; base < q1; base += CF_THREADS) {   // base uniform across the block: every lane takes part in the ballots
    const int64_t q = base + threadIdx.x;
    const bool in = q < q1;
    unsigned t[4] = {0, 0, 0, 0}, y[4] = {0, 0, 0, 0};
    if (in) {
      const int64_t n = q / P, i = q - n * P;
      const int64_t o = n * 4 * P + i;
#pragma unroll
      for (int p = 0; p < 4; ++p) t[p] = __ldcs(target + o + p * P), y[p] = __ldcs(pred + o + p * P);
    }
    bool bad = false;
    // the three one-hot planes: cell t * K + y of the plane's matrix
#pragma unroll
    for (int p = 0; p < 3; ++p) {
      const unsigned K = p == 0 ? PAN : p == 1 ? HUM : FACE, off = p == 0 ? 0 : p == 1 ? OFF_HUM : OFF_FACE;
      const bool ok = in && t[p] < K && y[p] < K;
      bad |= in && !ok;
      const unsigned zero = __ballot_sync(full, ok && t[p] == 0 && y[p] == 0);
      if (ok && (t[p] | y[p])) atomicAdd(hist + off + t[p] * K + y[p], 1u);
      if (lane == 0 && zero) atomicAdd(hist + off, (unsigned)__popc(zero));
    }
    // edges: a count of 1 or 2 is an edge
    const bool eok = in && t[3] <= 2u && y[3] <= 2u;
    bad |= in && !eok;
    const unsigned te = t[3] != 0u, ye = y[3] != 0u;
    unsigned e[4];
#pragma unroll
    for (int k = 0; k < 4; ++k) e[k] = __ballot_sync(full, eok && te * 2 + ye == (unsigned)k);
    const unsigned nb = __popc(__ballot_sync(full, bad));
    if (lane == 0) {
#pragma unroll
      for (int k = 0; k < 4; ++k)
        if (e[k]) atomicAdd(hist + OFF_EDGE + k, (unsigned)__popc(e[k]));
      if (nb) atomicAdd(hist + OFF_BAD, nb);
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < CONF_LEN; i += CF_THREADS)
    if (const unsigned c = hist[i]) atomicAdd(conf + i, (unsigned long long)c);
}

}  // namespace scene
}  // namespace mas

using namespace mas;
using namespace mas::scene;

extern "C" {

int mas_scene_decode(const float* x, mas_tensor4 xs, uint8_t* planes, void* stream) {
  MAS_REQUIRE(x && planes && xs.n > 0 && xs.h > 0 && xs.w > 0 && xs.c == C && xs.n <= 65535 && xs.h <= 65535 && xs.w <= INT32_MAX,
              "scene_decode: bad arguments (need a [B, 159, H, W] tensor, B and H <= 65535)");
  if (xs.sc == 1) {
    decode_cl_kernel<<<dim3((unsigned)cdiv(xs.w, 32), (unsigned)xs.h, (unsigned)xs.n), 256, 0, S(stream)>>>(x, xs, planes);
    return launched("scene_decode_cl");
  }
  decode_strided_kernel<<<dim3((unsigned)cdiv(xs.w, 32), (unsigned)cdiv(xs.h, 4), (unsigned)xs.n), dim3(32, 4), 0, S(stream)>>>(x, xs, planes);
  return launched("scene_decode_strided");
}

size_t mas_scene_confusion_ws_bytes(int64_t pixels_per_image, int B) {
  (void)pixels_per_image;
  (void)B;
  return 0;
}

int mas_scene_confusion(const uint8_t* pred, const uint8_t* target, int64_t pixels_per_image, int B, int64_t* conf, void* ws,
                        size_t ws_bytes, void* stream) {
  MAS_REQUIRE(pred && target && conf && pixels_per_image > 0 && B > 0, "scene_confusion: bad arguments");
  (void)ws;
  (void)ws_bytes;
  static std::atomic<uint64_t> configured{0};
  if (first_on_device(configured)) {
    const cudaError_t a = cudaFuncSetAttribute(confusion_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                               CONF_LEN * (int)sizeof(unsigned));
    if (a != cudaSuccess) return fail(MAS_ERR_LAUNCH, "scene_confusion: cudaFuncSetAttribute: %s", cudaGetErrorString(a));
    mark_device(configured);
  }
  int dev = 0, sms = 0;
  cudaGetDevice(&dev);
  if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) sms = NUM_SMS;
  cudaError_t e = cudaMemsetAsync(conf, 0, CONF_LEN * sizeof(int64_t), S(stream));
  if (e != cudaSuccess) return fail(MAS_ERR_LAUNCH, "scene_confusion: %s", cudaGetErrorString(e));
  // at most one block per SM of this device keeps the flush of the 18438 block counts small; a block's share stays at most
  // 2^30 pixels (a multiple of CF_THREADS), so that no u32 count can overflow
  const int64_t total = pixels_per_image * B;
  const int64_t blocks = std::max<int64_t>(std::min<int64_t>(sms, cdiv(total, CF_THREADS * 16)), cdiv(total, (int64_t)1 << 30));
  const int64_t per_block = cdiv(cdiv(total, blocks), CF_THREADS) * CF_THREADS;
  confusion_kernel<<<(unsigned)cdiv(total, per_block), CF_THREADS, CONF_LEN * sizeof(unsigned), S(stream)>>>(
      pred, target, pixels_per_image, total, per_block, reinterpret_cast<unsigned long long*>(conf));
  return launched("scene_confusion");
}

}  // extern "C"
