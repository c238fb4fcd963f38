// Codebook argmin, tensor-core FILTER stage (modules.py:501-505; SURVEY.md 7.3 #1).
//
// The reference's index is the arg-min over fp32 distances d[r,k] = fl(fl(|z_r|^2 + |e_k|^2) - 2 z_r.e_k).  The exact-fp32
// FFMA kernel (vq.cu) reproduces that arithmetic but is bound by the FMA pipe (4.2 MFLOP per latent row).  This kernel
// computes the R x K dot products on the tensor cores instead, to a KNOWN accuracy, and keeps per row the few smallest
// approximate distances; vq_resolve (vq.cu) then
//   * accepts the best code outright when the runner-up is farther than a rigorous error margin (nothing any fp32
//     evaluation order could reorder),
//   * re-evaluates the (at most four) candidates inside the margin with the EXACT arithmetic of the FFMA kernel, or
//   * (more candidates than that: tie-heavy codebooks) hands the row to the FFMA kernel.
// The indices are therefore those of the exact kernel, bit for bit, at tensor-core speed for ordinary data.
//
// Arithmetic: operand splitting into two fp16 numbers, x*s = h + l (h = fp16(x*s), l = fp16(x*s - h): 22 significant
// bits; s a power of two from the tensor's largest magnitude), and three fp16 wgmma per K step,
//   z.e ~= (zh.eh + zl.eh + zh.el) / (s_z s_e),   dropped term zl.el ~ 2^-22 relative,
// accumulated in fp32.
//
// Structure (one CTA = 128 latent rows x a contiguous range of 128-code tiles):
//   * A (the 128 x D latent tile, both halves) is converted once and stays in SHARED MEMORY for the whole sweep (K-major
//     no-swizzle planes [hi|lo][d/8][row][8 halves], 130 KB for D = 256), the rest of shared memory is a 5-stage ring of
//     code stages;
//   * B (codes): split ONCE per launch by vq_pack_codes into the exact shared-memory image of a pipeline stage
//     ([tile][32-dim chunk][hi|lo][k/8][code][8 halves], K-major no-swizzle layout), so one thread feeds the ring with
//     a single cp.async.bulk (16.6 KB, mbarrier complete_tx) per stage;
//   * two warpgroups issue the wgmma.m64n128k16 of latent rows 64 g .. 64 g + 63 (3 per K step) and keep, per fragment row,
//     the five smallest values (four of them with their code index) in a sorted insertion list; the four lanes that share
//     a row merge their lists at the end.
#include <cuda_fp16.h>

#include "mas_common.cuh"
#include "wgmma.cuh"

namespace mas {
namespace vqtc {

constexpr int BM = 128, BN = 128, KC = 32, STAGES = 5;
constexpr int NMMA = 256, NTHREADS = NMMA + 128;   // warps 0-7: A staging, MMA and candidate lists; warp 8: code-stage feeder
constexpr int PITCH_B = BN * 16 + 32;   // bytes between 8-dimension planes of a B stage half
constexpr int B_HALF = (KC / 8) * PITCH_B;
constexpr int B_STAGE = 2 * B_HALF;     // hi planes then lo planes (16.6 KB)
constexpr int NCAND = 4;                // candidates kept with their index (+ one more value)
constexpr int REC = 12;                 // floats per (row, split) record: b[5], i[4] (as int bits), pad
constexpr int D_MAX = 256;              // latent dimensions the shared-memory A tile holds
constexpr int PITCH_A = BM * 16 + 32;   // bytes between 8-dimension planes of the A tile

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done)
        : "r"(bar), "r"(parity)
        : "memory");
  } while (!done);
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(dst), "l"(src),
               "r"(bytes), "r"(bar)
               : "memory");
}
__device__ __forceinline__ void fence_barrier_init() { asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory"); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// power-of-two scale putting the tensor's largest magnitude into [2^14, 2^15) (fp16 tops out at 65504); *inv = 1/s, exact
__device__ __forceinline__ float split_scale(const float* amax, float* inv) {
  float s = 1.f, i = 1.f;
  const uint32_t b = __float_as_uint(*amax);
  const int e = (int)((b >> 23) & 0xff);
  if (e > 0 && e < 255) {
    int se = 127 + 14 - (e - 127);
    se = se < 1 ? 1 : (se > 254 ? 254 : se);
    s = __uint_as_float((uint32_t)se << 23);
    i = __uint_as_float((uint32_t)(254 - se) << 23);
  }
  *inv = i;
  return s;
}
// (a, b) * s -> packed fp16 pairs (hi, lo): x*s = hi + lo up to 2^-22 relative
__device__ __forceinline__ void split2(float a, float b, float s, uint32_t* hi, uint32_t* lo) {
  const float as = a * s, bs = b * s;
  const __half2 h = __floats2half2_rn(as, bs);
  const float2 hf = __half22float2(h);
  const __half2 l = __floats2half2_rn(as - hf.x, bs - hf.y);
  *hi = *reinterpret_cast<const uint32_t*>(&h);
  *lo = *reinterpret_cast<const uint32_t*>(&l);
}

// sorted insertion (ascending by value, then by code) into a five-entry list
__device__ __forceinline__ void cand_insert(float* b, int* ci, float d, int code) {
  auto lt = [&](int k) { return d < b[k] || (d == b[k] && code < ci[k]); };
  if (d == INFINITY || !lt(4)) return;   // +inf: a code beyond K (or an empty slot of another list) is never a candidate
  if (lt(3)) {
    b[4] = b[3]; ci[4] = ci[3];
    if (lt(2)) {
      b[3] = b[2]; ci[3] = ci[2];
      if (lt(1)) {
        b[2] = b[1]; ci[2] = ci[1];
        if (lt(0)) { b[1] = b[0]; ci[1] = ci[0]; b[0] = d; ci[0] = code; }
        else { b[1] = d; ci[1] = code; }
      } else { b[2] = d; ci[2] = code; }
    } else { b[3] = d; ci[3] = code; }
  } else {
    b[4] = d; ci[4] = code;
  }
}

struct Params {
  const float* z;      // [R, D]
  const uint8_t* Epk;  // packed split codes: [ntile][D/32][B_STAGE bytes] (vq_pack_codes)
  const float* ee;     // [K] |e_k|^2 (vq_code_norms: the exact kernel's values)
  const float* z_amax; // device scalars
  const float* e_amax;
  float* cand;         // [R][splits][REC]
  int64_t R;
  int K, D, tiles_per_split;
};

__global__ void __launch_bounds__(NTHREADS, 1) vq_filter_tc(const Params p) {
  extern __shared__ __align__(1024) uint8_t smem[];
  const int a_half = (p.D / 8) * PITCH_A;
  uint8_t* a_smem = smem;                                  // [hi|lo][d/8][row][8 halves]
  uint8_t* b_smem = smem + 2 * a_half;
  uint64_t* bars = reinterpret_cast<uint64_t*>(b_smem + (size_t)STAGES * B_STAGE);
  const uint32_t a_base = smem_u32(a_smem), b_base = smem_u32(b_smem), bar_base = smem_u32(bars);
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (STAGES + s); };

  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
  const int64_t row0 = (int64_t)blockIdx.x * BM;
  const int ntile_all = (p.K + BN - 1) / BN;
  const int tile_lo = blockIdx.y * p.tiles_per_split, tile_hi = min(ntile_all, tile_lo + p.tiles_per_split);
  const int nchunk = p.D / KC;

  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(full_bar(s), 1);
      mbar_init(empty_bar(s), NMMA);
    }
    fence_barrier_init();
  }

  float inv_z, inv_e;
  const float s_z = split_scale(p.z_amax, &inv_z);
  split_scale(p.e_amax, &inv_e);

  // ---- A: thread = (latent row, half of the dimensions); 8 dimensions at a time -> one 16-byte hi and one lo store ----
  if (warp < 8) {
    const int r = tid & (BM - 1);
    const int64_t row = row0 + r;
    const float4* src = reinterpret_cast<const float4*>(p.z + (size_t)(row < p.R ? row : 0) * p.D);
    const int octs = p.D / 8;
    for (int oc = (tid >> 7) * (octs / 2); oc < ((tid >> 7) + 1) * (octs / 2); ++oc) {
      float4 v0 = make_float4(0.f, 0.f, 0.f, 0.f), v1 = v0;
      if (row < p.R) { v0 = __ldg(src + 2 * oc); v1 = __ldg(src + 2 * oc + 1); }
      uint4 h, l;
      split2(v0.x, v0.y, s_z, &h.x, &l.x);
      split2(v0.z, v0.w, s_z, &h.y, &l.y);
      split2(v1.x, v1.y, s_z, &h.z, &l.z);
      split2(v1.z, v1.w, s_z, &h.w, &l.w);
      uint8_t* dst = a_smem + (size_t)oc * PITCH_A + r * 16;
      *reinterpret_cast<uint4*>(dst) = h;
      *reinterpret_cast<uint4*>(dst + a_half) = l;
    }
    fence_proxy_async();
  }
  __syncthreads();

  if (warp < 8) {
    // ===================== MMA warpgroups: running five smallest approximate distances per fragment row =====================
    wg::regs_inc<wg::MMA_REGS>();
    const int wgi = warp >> 2, fk = lane & 3;
    float b[2][NCAND + 1];
    int ci[2][NCAND + 1];
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int j = 0; j <= NCAND; ++j) { b[i][j] = INFINITY; ci[i][j] = 0; }
    const float m2 = -2.0f * inv_z * inv_e;          // dot (scaled) -> -2 z.e
    int stage = 0, prev = 0;
    uint32_t phase = 0;
    float acc[BN / 2];
    const uint32_t a_rows = a_base + (uint32_t)(wgi * 64 * 16);
    for (int t = tile_lo; t < tile_hi; ++t) {
      for (int c = 0; c < nchunk; ++c) {
        mbar_wait(full_bar(stage), phase);
        const uint32_t bst = b_base + (uint32_t)stage * B_STAGE;
        wg::fence();
#pragma unroll
        for (int k16 = 0; k16 < KC / 16; ++k16) {
          const uint32_t aoff = (uint32_t)((c * KC / 8 + k16 * 2) * PITCH_A);
          const uint64_t ah = wg::desc(a_rows + aoff, PITCH_A, 128), al = wg::desc(a_rows + (uint32_t)a_half + aoff, PITCH_A, 128);
          const uint64_t bh = wg::desc(bst + (uint32_t)(k16 * 2 * PITCH_B), PITCH_B, 128);
          const uint64_t bl = wg::desc(bst + (uint32_t)(B_HALF + k16 * 2 * PITCH_B), PITCH_B, 128);
          wg::wgmma_f16_ss_n128<0, 0>(acc, ah, bh, (c > 0 || k16 > 0) ? 1u : 0u);   // zh . eh
          wg::wgmma_f16_ss_n128<0, 0>(acc, al, bh, 1u);                           // zl . eh
          wg::wgmma_f16_ss_n128<0, 0>(acc, ah, bl, 1u);                           // zh . el
        }
        wg::commit();
        wg::wait<1>();
        if (t > tile_lo || c > 0) mbar_arrive(empty_bar(prev));
        prev = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
      wg::wait<0>();
      wg::fence_regs<BN / 2>(acc);
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
        for (int cc = 0; cc < 2; ++cc) {
          const int code = t * BN + 8 * j + 2 * fk + cc;
          const float e2 = code < p.K ? __ldg(p.ee + code) : INFINITY;     // INFINITY for codes beyond K: never inserted
#pragma unroll
          for (int i = 0; i < 2; ++i) cand_insert(b[i], ci[i], fmaf(acc[4 * j + 2 * i + cc], m2, e2), code);
        }
      }
    }
    if (tile_hi > tile_lo) mbar_arrive(empty_bar(prev));
    // the four lanes of a fragment row hold disjoint code subsets: merge their lists
#pragma unroll
    for (int x = 1; x <= 2; x <<= 1) {
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        float ob[NCAND + 1];
        int oc[NCAND + 1];
#pragma unroll
        for (int j = 0; j <= NCAND; ++j) {
          ob[j] = __shfl_xor_sync(0xffffffffu, b[i][j], x);
          oc[j] = __shfl_xor_sync(0xffffffffu, ci[i][j], x);
        }
#pragma unroll
        for (int j = 0; j <= NCAND; ++j) cand_insert(b[i], ci[i], ob[j], oc[j]);
      }
    }
    if (fk == 0) {
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const int64_t row = row0 + wgi * 64 + (warp & 3) * 16 + (lane >> 2) + 8 * i;
        if (row < p.R) {
          float* o = p.cand + ((size_t)row * gridDim.y + blockIdx.y) * REC;
#pragma unroll
          for (int j = 0; j <= NCAND; ++j) o[j] = b[i][j];
#pragma unroll
          for (int j = 0; j < NCAND; ++j) o[5 + j] = __int_as_float(ci[i][j]);
        }
      }
    }
  } else {
    // ===================== code-stage feeder (one thread): one bulk copy per stage =====================
    wg::regs_dec<wg::COPY_REGS>();
    if (warp == 8 && lane == 0) {
      int stage = 0;
      uint32_t phase = 0;
      const int nsteps = (tile_hi - tile_lo) * nchunk;
      const uint8_t* src = p.Epk + (size_t)tile_lo * nchunk * B_STAGE;
      for (int step = 0; step < nsteps; ++step) {
        mbar_wait(empty_bar(stage), phase ^ 1);
        mbar_expect_tx(full_bar(stage), B_STAGE);
        bulk_g2s(b_base + (uint32_t)stage * B_STAGE, src + (size_t)step * B_STAGE, B_STAGE, full_bar(stage));
        if (++stage == STAGES) { stage = 0; phase ^= 1; }
      }
    }
    __syncwarp();
  }
}

size_t filter_smem_bytes(int D) { return (size_t)2 * (D / 8) * PITCH_A + (size_t)STAGES * B_STAGE + 2 * STAGES * 8; }

}  // namespace vqtc

// Codes -> the packed, split stage images the filter streams (one pass over E per launch; the codebook changes once per
// optimizer step).  Thread = (code, 8-dimension group); codes beyond K are zero rows (masked by their +inf |e|^2).
__global__ void vq_pack_codes(const float* __restrict__ E, const float* __restrict__ e_amax, int K, int D, uint8_t* __restrict__ out) {
  using namespace vqtc;
  const int octs = D >> 3, nchunk = D / KC, ntile = (K + BN - 1) / BN;
  const int64_t total = (int64_t)ntile * BN * octs;
  float inv;
  const float s_e = split_scale(e_amax, &inv);
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int oc = (int)(i % octs);
    const int64_t code = i / octs;
    uint4 h = make_uint4(0u, 0u, 0u, 0u), l = h;
    if (code < K) {
      const float4* src = reinterpret_cast<const float4*>(E + (size_t)code * D + oc * 8);
      const float4 v0 = __ldg(src), v1 = __ldg(src + 1);
      split2(v0.x, v0.y, s_e, &h.x, &l.x);
      split2(v0.z, v0.w, s_e, &h.y, &l.y);
      split2(v1.x, v1.y, s_e, &h.z, &l.z);
      split2(v1.z, v1.w, s_e, &h.w, &l.w);
    }
    const int t = (int)(code / BN), cl = (int)(code % BN), c = oc / (KC / 8), o = oc % (KC / 8);
    uint8_t* dst = out + ((size_t)t * nchunk + c) * B_STAGE + (size_t)o * PITCH_B + (size_t)cl * 16;
    *reinterpret_cast<uint4*>(dst) = h;
    *reinterpret_cast<uint4*>(dst + B_HALF) = l;
  }
}

// Host side: eligibility and launch (called from mas_vq_forward in vq.cu).
bool vq_filter_tc_ok(int64_t R, int K, int D) {
  return D % 64 == 0 && D >= 64 && D <= vqtc::D_MAX && K >= 8 && R > 0;   // latent tile: two fp16 halves in shared memory
}
int vq_filter_splits(int64_t R, int K) {
  const int64_t row_blocks = cdiv(R, vqtc::BM);
  const int ntile = (int)cdiv(K, vqtc::BN);
  int s = (int)(132 / row_blocks);
  if (s < 1) s = 1;
  if (s > ntile) s = ntile;
  if (s > 4) s = 4;
  return s;
}
size_t vq_filter_pack_bytes(int K, int D) { return (size_t)cdiv(K, vqtc::BN) * (D / vqtc::KC) * vqtc::B_STAGE; }
int vq_filter_tc_launch(const float* z, const float* E, const float* ee, const float* z_amax, const float* e_amax, int64_t R, int K,
                        int D, float* cand, int splits, void* pack_buf, cudaStream_t st) {
  const int64_t pk_items = cdiv(K, vqtc::BN) * vqtc::BN * (D / 8);
  vq_pack_codes<<<(int)(cdiv(pk_items, 256) < 1184 ? cdiv(pk_items, 256) : 1184), 256, 0, st>>>(E, e_amax, K, D, (uint8_t*)pack_buf);
  if (int e = launched("vq_pack_codes")) return e;
  vqtc::Params p;
  p.z = z; p.Epk = (const uint8_t*)pack_buf; p.ee = ee; p.z_amax = z_amax; p.e_amax = e_amax; p.cand = cand;
  p.R = R; p.K = K; p.D = D;
  const int ntile = (int)cdiv(K, vqtc::BN);
  p.tiles_per_split = (int)cdiv(ntile, splits);
  const size_t smem = vqtc::filter_smem_bytes(D);
  static std::atomic<uint64_t> configured{0};
  if (first_on_device(configured)) {
    cudaError_t e = cudaFuncSetAttribute(vqtc::vq_filter_tc, cudaFuncAttributeMaxDynamicSharedMemorySize, 232448);
    if (e != cudaSuccess) return fail(MAS_ERR_LAUNCH, "vq_filter_tc: smem attr: %s", cudaGetErrorString(e));
    mark_device(configured);
  }
  dim3 grid((unsigned)cdiv(R, vqtc::BM), (unsigned)splits);
  vqtc::vq_filter_tc<<<grid, vqtc::NTHREADS, smem, st>>>(p);
  return launched_tc("vq_filter_tc");
}

}  // namespace mas
