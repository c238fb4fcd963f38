// Batched fp32-accurate GEMM on the Hopper tensor cores by operand splitting ("3xTF32"): for the contractions the reference
// runs in strict fp32 (torch.bmm in AttnBlock, modules.py:180,186; the transformer's QK^T / PV, transformer.py:77-103) a
// single TF32 pass (10-bit mantissa) is not acceptable, but
//     a = a_hi + a_lo,  b = b_hi + b_lo   (a_hi = tf32(a), a_lo = tf32(a - a_hi), same for b)
//     a.b ~= a_hi.b_hi + a_lo.b_hi + a_hi.b_lo          (dropped term a_lo.b_lo ~ 2^-22 relative)
// accumulated in fp32 recovers fp32-level accuracy at three MMAs per K step - still several times the FFMA rate.
//
//   C[b][m,n] = alpha * sum_k opA(A[b])[m,k] * opB(B[b])[n,k]
//   * CTA = one 128 x BN output tile (BN = 128, or 64 for 64-channel attention heads), full K, K chunks of 32
//   * BOTH operands are staged by the two warpgroups straight from the activation tensors (no pack pass): generic loads,
//     split into hi / lo in registers, st.shared into the K-major no-swizzle wgmma layout [k/4][row][4] (the layout the
//     convolution kernels use for their weight operand).  Either source orientation works: [row][k] (16-byte loads along
//     k, one 16-byte store) or [k][row] (16-byte loads along rows, four 4-byte stores) - so Q.K^T, P.V and all four of
//     their gradients run without a transposing copy.
//   * warpgroup g issues the wgmma.m64nBNk8 of rows 64 g .. 64 g + 63 (12 per chunk) and keeps that half of the tile in
//     registers; the loads of chunk k+1 and, with two stages, the stores of chunk k+1 overlap the MMAs of chunk k.
//
// Selected by impl = MAS_IMPL_TC3 of mas_gemm / mas_gemm_batched2: the AttnBlock backward and the token transformer's attention
// contractions run on it (tests/test_gpu_gemm3.py, tests/test_gpu_transformer.py).
#include <stdlib.h>

#include "mas_common.cuh"
#include "wgmma.cuh"

namespace mas {
namespace tc3 {

constexpr int BM = 128, KC = 32;   // the N tile (128 or 64: attention heads of 64) and the ring depth are template parameters
constexpr int NPROD = 256, NTHREADS = 256;   // two warpgroups: producers, MMA issuers and epilogue
constexpr int SLOTS = 132;                   // row pitch of an operand plane in 16-byte units (132 % 8 == 4: conflict-free stores)
constexpr int LBO = SLOTS * 16;              // bytes between k-quads
constexpr int PLANE = (KC / 4) * LBO;        // one operand image (hi or lo) per stage: 16 896 B
constexpr int STAGE = 4 * PLANE;             // A_hi, A_lo, B_hi, B_lo

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

template <int BN>
__device__ __forceinline__ void mma_tf32(float* d, uint64_t a, uint64_t b) {
  if (BN == 128) wg::wgmma_tf32_ss_n128(d, a, b, 1u);
  else wg::wgmma_tf32_ss_n64(d, a, b, 1u);
}

struct P3 {
  const float* A;
  const float* B;
  float* C;
  int M, N, K;
  int64_t lda, ldb, ldc, sa, sb, sc;
  int ta, tb;   // 0: operand stored [row][k] (k contiguous); 1: stored [k][row] (rows contiguous)
  float alpha;
  // two-level batch: blockIdx.z = outer * inner + i -> offsets outer * s?2 + i * s? (attention heads inside a fused
  // [B, S, 3H] activation: outer = batch element, inner = head).  inner = batch, s?2 = 0 for the plain batched form.
  int inner;
  int64_t sa2, sb2, sc2;
  // causal structure of the token transformer's attention matrices (queries x keys, key <= query): whole K chunks / output
  // tiles that are identically zero are skipped.  1: A[m][k] = 0 for k > m (dQ = dS K, ctx = P V): chunks beyond the row tile;
  // 2: A stored [K][M] with A[k][m] = 0 for k < m (dV = P^T dO, dK = dS^T Q): chunks before the row tile; 3: only output
  // entries n <= m are consumed (S = Q K^T, dP = dO V^T): tiles above the diagonal are written as zeros.
  int causal;
};

// One operand of one K chunk: 128 rows x 32 k = 1024 quads, four per producer thread; returns them split into hi / lo.
struct Quad4 {
  float4 v[4];
};

// STAGES = 2: one CTA per SM, the stores of chunk k+1 overlap the MMAs of chunk k.  STAGES = 1 (short reductions, K <= 64:
// the attention heads' 64-wide contractions are two chunks): half the shared memory so that two or three CTAs share an SM
// and overlap each other's load / MMA / epilogue phases instead.
template <int BN, int STAGES>
__global__ void __launch_bounds__(NTHREADS, STAGES == 1 ? 2 : 1) gemm3_tc(const P3 p) {
  constexpr int B_ITEMS = BN * (KC / 4) / NPROD;    // 16-byte items of the B operand per producer thread (4 or 2)
  extern __shared__ __align__(1024) uint8_t smem[];
  const uint32_t smem_base = smem_u32(smem);
  const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, wgi = warp >> 2;
  const int n0 = blockIdx.x * BN, m0 = blockIdx.y * BM;
  const int zo = (int)blockIdx.z / p.inner, zi = (int)blockIdx.z - zo * p.inner;
  const float* Ab = p.A + (int64_t)zo * p.sa2 + (int64_t)zi * p.sa;
  const float* Bb = p.B + (int64_t)zo * p.sb2 + (int64_t)zi * p.sb;
  float* Cb = p.C + (int64_t)zo * p.sc2 + (int64_t)zi * p.sc;
  const int nchunks = p.K / KC;
  int kc0 = 0, kc1 = nchunks;
  if (p.causal == 1) kc1 = min(nchunks, (m0 + BM) / KC);
  else if (p.causal == 2) kc0 = min(nchunks, m0 / KC);
  else if (p.causal == 3 && n0 >= m0 + BM) kc1 = 0;
  const bool empty = kc0 >= kc1;          // block-uniform: nothing to contract, the tile is zero

  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;

    auto load_op = [&](const float* base, int64_t ld, int trans, int row0, int rows_total, int kc, Quad4& out, int nitems) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        if (i >= nitems) break;
        const int item = tid + i * NPROD;
        float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
        if (!trans) {
          const int q = item & 7, row = item >> 3;
          if (row0 + row < rows_total) v = __ldg(reinterpret_cast<const float4*>(base + (int64_t)(row0 + row) * ld + kc * KC + q * 4));
        } else {
          const int k = item & 31, rq = item >> 5;
          const int r = row0 + rq * 4;
          const float* src = base + (int64_t)(kc * KC + k) * ld + r;
          if (r + 3 < rows_total) v = __ldg(reinterpret_cast<const float4*>(src));
          else {
            if (r < rows_total) v.x = __ldg(src);
            if (r + 1 < rows_total) v.y = __ldg(src + 1);
            if (r + 2 < rows_total) v.z = __ldg(src + 2);
          }
        }
        out.v[i] = v;
      }
    };
    auto store_op = [&](uint8_t* hi_plane, uint8_t* lo_plane, int trans, const Quad4& in, int nitems) {
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        if (i >= nitems) break;
        const int item = tid + i * NPROD;
        const float4 v = in.v[i];
        float4 h = make_float4(round_tf32(v.x), round_tf32(v.y), round_tf32(v.z), round_tf32(v.w));
        float4 l = make_float4(round_tf32(v.x - h.x), round_tf32(v.y - h.y), round_tf32(v.z - h.z), round_tf32(v.w - h.w));
        if (!trans) {
          const int q = item & 7, row = item >> 3;
          const int off = q * LBO + row * 16;
          *reinterpret_cast<float4*>(hi_plane + off) = h;
          *reinterpret_cast<float4*>(lo_plane + off) = l;
        } else {
          const int k = item & 31, rq = item >> 5;
          const int off = (k >> 2) * LBO + rq * 64 + (k & 3) * 4;
          float* hp = reinterpret_cast<float*>(hi_plane + off);
          float* lp = reinterpret_cast<float*>(lo_plane + off);
          hp[0] = h.x; hp[4] = h.y; hp[8] = h.z; hp[12] = h.w;     // consecutive rows are 16 bytes apart
          lp[0] = l.x; lp[4] = l.y; lp[8] = l.z; lp[12] = l.w;
        }
      }
    };
    int stage = 0;
    Quad4 an, bn;
    if (!empty) {
      load_op(Ab, p.lda, p.ta, m0, p.M, kc0, an, 4);
      load_op(Bb, p.ldb, p.tb, n0, p.N, kc0, bn, B_ITEMS);
    }
    for (int kc = kc0; kc < kc1; ++kc) {
      const Quad4 a = an, b = bn;
      if (kc + 1 < kc1) {   // next chunk's loads fly while this one is split, stored and multiplied
        load_op(Ab, p.lda, p.ta, m0, p.M, kc + 1, an, 4);
        load_op(Bb, p.ldb, p.tb, n0, p.N, kc + 1, bn, B_ITEMS);
      }
      // the stage about to be overwritten was last read by the MMAs of chunk kc - STAGES: both warpgroups have waited for
      // those (wait<STAGES - 1> below) before arriving here
      if (kc > kc0) __syncthreads();
      uint8_t* st = smem + (size_t)stage * STAGE;
      store_op(st, st + PLANE, p.ta, a, 4);
      store_op(st + 2 * PLANE, st + 3 * PLANE, p.tb, b, B_ITEMS);
      fence_proxy_async();  // make the generic-proxy stores visible to the tensor core (async proxy)
      __syncthreads();
      const uint32_t sa = smem_base + (uint32_t)stage * STAGE;
      // rows 64 g .. 64 g + 63 of A start 64 * 16 bytes into each k-quad plane
      const uint64_t a_hi = wg::desc(sa + wgi * 1024, LBO, 128), a_lo = wg::desc(sa + PLANE + wgi * 1024, LBO, 128);
      const uint64_t b_hi = wg::desc(sa + 2 * PLANE, LBO, 128), b_lo = wg::desc(sa + 3 * PLANE, LBO, 128);
      wg::fence();
#pragma unroll
      for (int k8 = 0; k8 < KC / 8; ++k8) {
        const uint64_t ko = (uint64_t)((k8 * 2 * LBO) >> 4);
        mma_tf32<BN>(acc, a_hi + ko, b_hi + ko);
        mma_tf32<BN>(acc, a_lo + ko, b_hi + ko);
        mma_tf32<BN>(acc, a_hi + ko, b_lo + ko);
      }
      wg::commit();
      wg::wait<STAGES - 1>();
      if (++stage == STAGES) stage = 0;
    }
    wg::wait<0>();
    wg::fence_regs<BN / 2>(acc);

    // ---------------- epilogue: straight from the accumulator fragment ----------------
    const int rbase = m0 + wgi * 64 + (warp & 3) * 16 + (lane >> 2);
    float* cp = Cb + n0 + 2 * (lane & 3);
#pragma unroll
    for (int i = 0; i < 2; ++i) {
      const int m = rbase + 8 * i;
      if (m < p.M) {
#pragma unroll
        for (int j = 0; j < BN / 8; ++j)
          *reinterpret_cast<float2*>(cp + (int64_t)m * p.ldc + 8 * j) = make_float2(acc[4 * j + 2 * i] * p.alpha, acc[4 * j + 2 * i + 1] * p.alpha);
      }
    }
}

template <int STAGES>
constexpr size_t smem_bytes() { return (size_t)STAGES * STAGE; }

}  // namespace tc3

static inline bool al16q(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

// C[b] = alpha * opA(A[b]) . opB(B[b])^T, fp32-accurate on the tensor cores.  ta / tb as in mas_gemm: trans_a = 1 means A is
// stored [K][M]; trans_b = 1 means B is stored [N][K] (k contiguous), trans_b = 0 means B is stored [K][N].
int gemm_tc3_launch2(const float* A, const float* B, float* C, int M, int N, int K, int outer, int batch, int64_t lda, int64_t ldb,
                     int64_t ldc, int64_t sa2, int64_t sb2, int64_t sc2, int64_t sa, int64_t sb, int64_t sc, int ta, int tb, float alpha,
                     const float* bias, const float* res, int causal, cudaStream_t st);
int gemm_tc3_launch(const float* A, const float* B, float* C, int M, int N, int K, int batch, int64_t lda, int64_t ldb, int64_t ldc,
                    int64_t sa, int64_t sb, int64_t sc, int ta, int tb, float alpha, const float* bias, const float* res,
                    cudaStream_t st) {
  return gemm_tc3_launch2(A, B, C, M, N, K, 1, batch, lda, ldb, ldc, 0, 0, 0, sa, sb, sc, ta, tb, alpha, bias, res, 0, st);
}
// outer x batch matrices: matrix (o, i) lives at o * s?2 + i * s?
int gemm_tc3_launch2(const float* A, const float* B, float* C, int M, int N, int K, int outer, int batch, int64_t lda, int64_t ldb,
                     int64_t ldc, int64_t sa2, int64_t sb2, int64_t sc2, int64_t sa, int64_t sb, int64_t sc, int ta, int tb, float alpha,
                     const float* bias, const float* res, int causal, cudaStream_t st) {
  if (causal < 0 || causal > 3 || (causal == 2 && !ta) || (causal == 1 && ta))
    return fail(MAS_ERR_INVALID_ARG, "tc3 gemm: causal mode %d does not fit the operand orientation", causal);
  if (outer < 1 || batch < 1 || (int64_t)outer * batch > 65535) return fail(MAS_ERR_UNSUPPORTED, "tc3 gemm: outer * batch must be in [1, 65535]");
  if (sa2 % 4 || sb2 % 4 || sc2 % 4) return fail(MAS_ERR_UNSUPPORTED, "tc3 gemm: outer strides must be multiples of 4 elements");
  if (bias || res) return fail(MAS_ERR_UNSUPPORTED, "tc3 gemm: bias / residual epilogue not available");
  if (N % 64 || K % tc3::KC || lda % 4 || ldb % 4 || ldc % 4 || sa % 4 || sb % 4 || sc % 4 || !al16q(A) || !al16q(B) || !al16q(C))
    return fail(MAS_ERR_UNSUPPORTED, "tc3 gemm: need N %% 64 == 0, K %% 32 == 0, pitches %% 4 == 0 and 16-byte aligned operands");
  if (ta && M % 4) return fail(MAS_ERR_UNSUPPORTED, "tc3 gemm: a [K][M] stored A operand needs M %% 4 == 0");
  tc3::P3 p;
  p.A = A; p.B = B; p.C = C; p.M = M; p.N = N; p.K = K;
  p.lda = lda; p.ldb = ldb; p.ldc = ldc; p.sa = sa; p.sb = sb; p.sc = sc;
  p.ta = ta ? 1 : 0;        // A stored [K][M]  -> rows (m) contiguous
  p.tb = tb ? 0 : 1;        // B stored [N][K] (tb = 1) is the k-contiguous orientation; [K][N] (tb = 0) is row-contiguous
  p.alpha = alpha;
  p.inner = batch; p.sa2 = sa2; p.sb2 = sb2; p.sc2 = sc2; p.causal = causal;
  const int zdim = outer * batch;
  static std::atomic<uint64_t> configured{0};
  if (first_on_device(configured)) {
    cudaError_t e = cudaFuncSetAttribute(tc3::gemm3_tc<128, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tc3::smem_bytes<2>());
    if (e == cudaSuccess) e = cudaFuncSetAttribute(tc3::gemm3_tc<64, 2>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tc3::smem_bytes<2>());
    if (e == cudaSuccess) e = cudaFuncSetAttribute(tc3::gemm3_tc<128, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tc3::smem_bytes<1>());
    if (e == cudaSuccess) e = cudaFuncSetAttribute(tc3::gemm3_tc<64, 1>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tc3::smem_bytes<1>());
    if (e != cudaSuccess) return fail(MAS_ERR_LAUNCH, "cudaFuncSetAttribute(smem=%zu): %s", tc3::smem_bytes<2>(), cudaGetErrorString(e));
    mark_device(configured);
  }
  static const bool shallow_on = [] { const char* e = getenv("MAS_TC3_SHALLOW"); return !(e && e[0] == '0'); }();
  const bool shallow = shallow_on && K <= 64;     // two chunks at most: co-resident CTAs instead of a 2-stage ring
  if (N % 128 == 0) {
    dim3 grid((unsigned)(N / 128), (unsigned)cdiv(M, tc3::BM), (unsigned)zdim);
    if (shallow) tc3::gemm3_tc<128, 1><<<grid, tc3::NTHREADS, tc3::smem_bytes<1>(), st>>>(p);
    else tc3::gemm3_tc<128, 2><<<grid, tc3::NTHREADS, tc3::smem_bytes<2>(), st>>>(p);
  } else {   // attention heads of 64 channels: P.V and the q / k / v gradients of the token transformer
    dim3 grid((unsigned)(N / 64), (unsigned)cdiv(M, tc3::BM), (unsigned)zdim);
    if (shallow) tc3::gemm3_tc<64, 1><<<grid, tc3::NTHREADS, tc3::smem_bytes<1>(), st>>>(p);
    else tc3::gemm3_tc<64, 2><<<grid, tc3::NTHREADS, tc3::smem_bytes<2>(), st>>>(p);
  }
  return launched_tc("gemm3_tc");
}

}  // namespace mas
