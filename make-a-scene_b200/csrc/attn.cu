// AttnBlock (modules.py:139-191) as two C-ABI calls: the whole forward and the whole backward of
//   GN -> q,k,v 1x1 -> softmax(q^T k / sqrt(C)) over keys -> v.P^T -> proj_out 1x1 -> + x
// enqueued on the caller's stream from caller-provided buffers. The q/k/v projections run as ONE row GEMM against the
// concatenated [3C, C] weight (forward: N = 3C; data gradient: K = 3C; weight gradient: Cout = 3C), the 1x1 convolutions
// go to the wgmma row-GEMM / weight-gradient kernels when the shape is eligible, and the two batched token contractions
// (QK^T and PV, plus their four gradients) keep fp32-level accuracy like the reference's torch.bmm (modules.py:180,186):
// 3xTF32 operand splitting on the tensor cores (contract_tc3.cu), or the FFMA kernel for extents off its tiles.
#include <stdlib.h>

#include "mas_common.cuh"

using namespace mas;

namespace mas {
bool attn_core_fused_ok(int HW, int C);
int attn_core_fused_launch(const float* qkv, const float* amax, float* P, float* O, int N, int HW, int C, float scale, cudaStream_t st);
}

namespace {
__global__ void cat3_kernel(const float* __restrict__ a, const float* __restrict__ b, const float* __restrict__ c, float* __restrict__ out,
                            int64_t n, const float* __restrict__ ba, const float* __restrict__ bb, const float* __restrict__ bc,
                            float* __restrict__ bout, int nb) {
  const int64_t total = 3 * n;
  for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (int64_t)gridDim.x * blockDim.x) {
    const int which = (int)(i / n);
    const int64_t j = i - which * n;
    out[i] = which == 0 ? a[j] : which == 1 ? b[j] : c[j];
  }
  if (bout && blockIdx.x == 0)
    for (int i = threadIdx.x; i < 3 * nb; i += blockDim.x) {
      const int which = i / nb, j = i - which * nb;
      const float* s = which == 0 ? ba : which == 1 ? bb : bc;
      bout[i] = s ? s[j] : 0.f;
    }
}
size_t al(size_t v) { return (v + 255) / 256 * 256; }
bool rows_on_tc(int impl, int N, int K) { return impl != MAS_IMPL_SIMT && N % 128 == 0 && K % 32 == 0; }
// implementation of the token contractions (QK^T, PV and their four gradients): the operand-split 3xTF32 wgmma GEMM
// (contract_tc3.cu: fp32-level accuracy like the reference's strict-fp32 torch.bmm, validated against fp64) when the
// extents fit its tiles, else the strict-fp32 FFMA kernel. MAS_ATTN_TC3=0 forces the FFMA kernel (A/B measurements).
int bmm_impl(int impl, int HW, int C) {
  static const bool off = [] { const char* e = getenv("MAS_ATTN_TC3"); return e && e[0] == '0'; }();
  return (!off && impl != MAS_IMPL_SIMT && HW % 128 == 0 && C % 128 == 0) ? MAS_IMPL_TC3 : impl;
}

struct Carver {
  char* p;
  size_t left;
  bool ok = true;
  float* take(size_t floats) {
    size_t b = al(floats * sizeof(float));
    if (b > left) { ok = false; return nullptr; }
    float* r = reinterpret_cast<float*>(p);
    p += b;
    left -= b;
    return r;
  }
};
}  // namespace

extern "C" {

size_t mas_attnblock_ws_bytes(int N, int HW, int C, int G) {
  const size_t M = (size_t)N * HW, c = (size_t)C;
  size_t fwd = al(3 * c * c * 4) * 2 + al(3 * c * 4);
  size_t w1 = mas_conv1x1_wgrad_ws_bytes((int64_t)M, C, C), w3 = mas_conv1x1_wgrad_ws_bytes((int64_t)M, C, 3 * C);
  size_t g = mas_gn_ws_bytes(N, HW, C, G);
  size_t scratch = al(w1 > w3 ? w1 : w3);
  if (al(g) > scratch) scratch = al(g);
  size_t bwd = al(M * c * 4) * 2 + al(M * 3 * c * 4) + al((size_t)N * HW * HW * 4) + al(3 * c * c * 4) * 2 + scratch;
  return (fwd > bwd ? fwd : bwd) + 256;
}

int mas_attnblock_forward(const float* x, int N, int HW, int C, int G, const float* mean, const float* rstd, const float* norm_w,
                          const float* norm_b, const float* q_w, const float* q_b, const float* k_w, const float* k_b,
                          const float* v_w, const float* v_b, const float* proj_w, const float* proj_b, float* hn, float* qkv, float* P,
                          float* O, float* out, float* stats_part, int impl, void* ws, size_t ws_bytes, void* stream) {
  MAS_REQUIRE(x && mean && rstd && norm_w && norm_b && q_w && k_w && v_w && proj_w && hn && qkv && P && O && out,
              "attnblock_forward: null pointer");
  MAS_REQUIRE(N > 0 && HW > 0 && C > 0 && G > 0 && C % G == 0, "attnblock_forward: bad shape");
  if (ws_bytes < mas_attnblock_ws_bytes(N, HW, C, G)) return fail(MAS_ERR_WORKSPACE, "attnblock_forward: workspace too small");
  const int64_t M = (int64_t)N * HW, c = C;
  const float scale = (float)pow((double)C, -0.5);  // int(c) ** (-0.5), modules.py:181
  const bool tc = rows_on_tc(impl, C, C);
  if (stats_part && !(tc && HW % 128 == 0)) return fail(MAS_ERR_UNSUPPORTED, "attnblock_forward: statistics epilogue needs the tensor path and HW %% 128 == 0");
  Carver cv{(char*)ws, ws_bytes};
  float* wcat = cv.take(3 * c * c);
  float* wpk = cv.take(3 * c * c);
  float* bcat = cv.take(3 * c);
  if (!cv.ok) return fail(MAS_ERR_WORKSPACE, "attnblock_forward: workspace too small");
  if (int e = mas_gn_apply(x, mean, rstd, norm_w, norm_b, hn, N, HW, C, G, 0, 0, stream)) return e;
  if (tc) {
    cat3_kernel<<<296, 256, 0, S(stream)>>>(q_w, k_w, v_w, wcat, c * c, q_b, k_b, v_b, bcat, C);
    if (int e = launched("attn_cat3")) return e;
    if (int e = mas_pack_gemm_tc(wcat, wpk, 3 * C, C, 0, stream)) return e;
    if (int e = mas_gemm_rows_packed(hn, c, wpk, qkv, 3 * c, M, 3 * C, C, 1.f, bcat, nullptr, nullptr, stream)) return e;
  } else {
    const float* ws_[3] = {q_w, k_w, v_w};
    const float* bs_[3] = {q_b, k_b, v_b};
    for (int i = 0; i < 3; ++i)
      if (int e = mas_gemm(hn, ws_[i], qkv + i * c, (int)M, C, C, 1, c, c, 3 * c, 0, 0, 0, 0, 1, 1.f, bs_[i], nullptr, impl, stream)) return e;
  }
  // fused core (attn_fused.cu): S = scale q k^T in registers -> softmax on the fragment -> P (shared memory) -> O = P v
  static const bool fused_off = [] { const char* e = getenv("MAS_ATTN_FUSED"); return e && e[0] == '0'; }();
  if (!fused_off && impl != MAS_IMPL_SIMT && attn_core_fused_ok(HW, C)) {
    float* amax = wpk;   // scratch: the packed QKV weight is dead once the QKV GEMM is enqueued (stream order), proj re-packs later
    if (int e = mas_amax(qkv, M * 3 * c, amax, stream)) return e;
    if (int e = attn_core_fused_launch(qkv, amax, P, O, N, HW, C, scale, S(stream))) return e;
  } else {
  // S[i,j] = scale * sum_c q[i,c] k[j,c]   (w_ = bmm(q^T, k) * c^-0.5)
  if (int e = mas_gemm(qkv, qkv + c, P, HW, HW, C, N, 3 * c, 3 * c, HW, (int64_t)HW * 3 * c, (int64_t)HW * 3 * c, (int64_t)HW * HW, 0, 1,
                       scale, nullptr, nullptr, bmm_impl(impl, HW, C), stream))
    return e;
  if (int e = mas_softmax_forward(P, P, (int64_t)N * HW, HW, stream)) return e;
  // O[i,c] = sum_j P[i,j] v[j,c]
  if (int e = mas_gemm(P, qkv + 2 * c, O, HW, C, HW, N, HW, 3 * c, c, (int64_t)HW * HW, (int64_t)HW * 3 * c, (int64_t)HW * c, 0, 0, 1.f,
                       nullptr, nullptr, bmm_impl(impl, HW, C), stream))
    return e;
  }
  if (tc) {
    if (int e = mas_pack_gemm_tc(proj_w, wpk, C, C, 0, stream)) return e;
    return mas_gemm_rows_packed(O, c, wpk, out, c, M, C, C, 1.f, proj_b, x, stats_part, stream);
  }
  return mas_gemm(O, proj_w, out, (int)M, C, C, 1, c, c, c, 0, 0, 0, 0, 1, 1.f, proj_b, x, impl, stream);
}

int mas_attnblock_backward(const float* dout, const float* x, int N, int HW, int C, int G, const float* mean, const float* rstd,
                           const float* norm_w, const float* norm_b, const float* q_w, const float* k_w, const float* v_w,
                           const float* proj_w, const float* hn, const float* qkv, const float* P, const float* O, float* dx,
                           float* dnorm_w, float* dnorm_b, float* dqkv_w, float* dqkv_b, float* dproj_w, float* dproj_b, float* dx_amax,
                           int impl, void* ws, size_t ws_bytes, void* stream) {
  MAS_REQUIRE(dout && x && mean && rstd && norm_w && norm_b && q_w && k_w && v_w && proj_w && hn && qkv && P && O && dx && dnorm_w &&
                  dnorm_b && dqkv_w && dqkv_b && dproj_w && dproj_b,
              "attnblock_backward: null pointer");
  MAS_REQUIRE(N > 0 && HW > 0 && C > 0 && G > 0 && C % G == 0, "attnblock_backward: bad shape");
  if (ws_bytes < mas_attnblock_ws_bytes(N, HW, C, G)) return fail(MAS_ERR_WORKSPACE, "attnblock_backward: workspace too small");
  const int64_t M = (int64_t)N * HW, c = C;
  const float scale = (float)pow((double)C, -0.5);
  const bool tc = rows_on_tc(impl, C, C);
  Carver cv{(char*)ws, ws_bytes};
  float* dO = cv.take(M * c);
  float* dhn = cv.take(M * c);
  float* dqkv = cv.take(M * 3 * c);
  float* dP = cv.take((size_t)N * HW * HW);
  float* wcat = cv.take(3 * c * c);
  float* wpk = cv.take(3 * c * c);
  if (!cv.ok) return fail(MAS_ERR_WORKSPACE, "attnblock_backward: workspace too small");
  void* scratch = cv.p;
  const size_t scratch_bytes = cv.left;
  // proj_out: dO = dout . Wp ; dWp = dout^T . O
  if (tc) {
    if (int e = mas_pack_gemm_tc(proj_w, wpk, C, C, 1, stream)) return e;
    if (int e = mas_gemm_rows_packed(dout, c, wpk, dO, c, M, C, C, 1.f, nullptr, nullptr, nullptr, stream)) return e;
  } else if (int e = mas_gemm(dout, proj_w, dO, (int)M, C, C, 1, c, c, c, 0, 0, 0, 0, 0, 1.f, nullptr, nullptr, impl, stream)) {
    return e;
  }
  if (int e = mas_conv1x1_wgrad(O, c, dout, c, M, C, C, dproj_w, dproj_b, impl, scratch, scratch_bytes, stream)) return e;
  const int64_t sP = (int64_t)HW * HW, sQ = (int64_t)HW * 3 * c, sO = (int64_t)HW * c;
  // dV[j,c] = sum_i P[i,j] dO[i,c]
  if (int e = mas_gemm(P, dO, dqkv + 2 * c, HW, C, HW, N, HW, c, 3 * c, sP, sO, sQ, 1, 0, 1.f, nullptr, nullptr, bmm_impl(impl, HW, C), stream)) return e;
  // dP[i,j] = sum_c dO[i,c] V[j,c]
  if (int e = mas_gemm(dO, qkv + 2 * c, dP, HW, HW, C, N, c, 3 * c, HW, sO, sQ, sP, 0, 1, 1.f, nullptr, nullptr, bmm_impl(impl, HW, C), stream)) return e;
  if (int e = mas_softmax_backward(P, dP, dP, (int64_t)N * HW, HW, scale, stream)) return e;  // dP <- dS (times c^-0.5)
  // dQ[i,c] = sum_j dS[i,j] K[j,c] ; dK[j,c] = sum_i dS[i,j] Q[i,c]
  if (int e = mas_gemm(dP, qkv + c, dqkv, HW, C, HW, N, HW, 3 * c, 3 * c, sP, sQ, sQ, 0, 0, 1.f, nullptr, nullptr, bmm_impl(impl, HW, C), stream)) return e;
  if (int e = mas_gemm(dP, qkv, dqkv + c, HW, C, HW, N, HW, 3 * c, 3 * c, sP, sQ, sQ, 1, 0, 1.f, nullptr, nullptr, bmm_impl(impl, HW, C), stream)) return e;
  // dhn = [dq dk dv] . [Wq; Wk; Wv]   (one contraction over K = 3C)
  if (tc && (3 * C) % 32 == 0) {
    cat3_kernel<<<296, 256, 0, S(stream)>>>(q_w, k_w, v_w, wcat, c * c, nullptr, nullptr, nullptr, nullptr, 0);
    if (int e = launched("attn_cat3")) return e;
    if (int e = mas_pack_gemm_tc(wcat, wpk, 3 * C, C, 1, stream)) return e;
    if (int e = mas_gemm_rows_packed(dqkv, 3 * c, wpk, dhn, c, M, C, 3 * C, 1.f, nullptr, nullptr, nullptr, stream)) return e;
  } else {
    const float* ws_[3] = {q_w, k_w, v_w};
    for (int i = 0; i < 3; ++i)
      if (int e = mas_gemm(dqkv + i * c, ws_[i], dhn, (int)M, C, C, 1, 3 * c, c, c, 0, 0, 0, 0, 0, 1.f, nullptr, i ? dhn : nullptr, impl,
                           stream))
        return e;
  }
  // [dWq; dWk; dWv] = dqkv^T . hn, biases = column sums of dqkv
  if (int e = mas_conv1x1_wgrad(hn, c, dqkv, 3 * c, M, C, 3 * C, dqkv_w, dqkv_b, impl, scratch, scratch_bytes, stream)) return e;
  // GroupNorm (no activation) backward, + dout for the residual branch
  return mas_gn_backward(dhn, x, mean, rstd, norm_w, norm_b, dout, dx, dnorm_w, dnorm_b, nullptr, 0, dx_amax, nullptr, nullptr, nullptr, N, HW, C, G, 0, scratch, scratch_bytes,
                         stream);
}

}  // extern "C"
