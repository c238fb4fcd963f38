// C-ABI dispatch for the contraction entry points (include/mas_b200.h): picks the wgmma path
// (contract_tc.cu) when the shape is eligible and impl allows, else the fp32 SIMT path.
#include "mas_common.cuh"

namespace mas {
int conv3x3_fprop_simt_launch(const float* x, mas_tensor4 xs, const float* w, const float* bias, const float* res, float* y,
                              mas_tensor4 ys, int mode, int ks, cudaStream_t st);
size_t conv_wgrad_simt_ws(mas_tensor4 xs, mas_tensor4 dys, int ks);
int conv_wgrad_simt_launch(const float* x, mas_tensor4 xs, const float* dy, mas_tensor4 dys, float* dw, int mode, int ks, void* ws,
                           size_t ws_bytes, cudaStream_t st);
int gemm_simt_launch(const float* A, const float* B, float* C, int M, int N, int K, int batch, int64_t lda, int64_t ldb, int64_t ldc,
                     int64_t sa, int64_t sb, int64_t sc, int ta, int tb, float alpha, const float* bias, const float* res,
                     cudaStream_t st);
// wgmma path; return MAS_ERR_UNSUPPORTED (without touching g_err semantics) when not eligible

int gemm_tc_launch(const float* A, const float* B, float* C, int M, int N, int K, int batch, int64_t lda, int64_t ldb, int64_t ldc,
                   int64_t sa, int64_t sb, int64_t sc, int ta, int tb, float alpha, const float* bias, const float* res,
                   cudaStream_t st);
size_t conv_wgrad_tc_ws(mas_tensor4 xs, mas_tensor4 dys, int mode);
bool conv_wgrad_tc_eligible(mas_tensor4 xs, mas_tensor4 dys, int mode);
int conv_wgrad_tc_launch(const float* x, mas_tensor4 xs, const float* dy, mas_tensor4 dys, float* dw, float* dbias, int mode,
                         const float* gn_table, int gn_silu, int f16, const float* dy_amax, int cout_rows, int x_f16, void* ws,
                         size_t ws_bytes, cudaStream_t st);
int gemm_tc3_launch(const float* A, const float* B, float* C, int M, int N, int K, int batch, int64_t lda, int64_t ldb, int64_t ldc,
                    int64_t sa, int64_t sb, int64_t sc, int ta, int tb, float alpha, const float* bias, const float* res,
                    cudaStream_t st);
int gemm_tc3_launch2(const float* A, const float* B, float* C, int M, int N, int K, int outer, int batch, int64_t lda, int64_t ldb,
                     int64_t ldc, int64_t sa2, int64_t sb2, int64_t sc2, int64_t sa, int64_t sb, int64_t sc, int ta, int tb, float alpha,
                     const float* bias, const float* res, int causal, cudaStream_t st);
size_t conv1x1_wgrad_tc_ws(int64_t M, int Cin, int Cout);
int conv1x1_wgrad_tc_launch(const float* x, int64_t ldx, const float* dy, int64_t ldy, int64_t M, int Cin, int Cout, float* dw,
                            float* dbias, void* ws, size_t ws_bytes, cudaStream_t st);
}  // namespace mas

using namespace mas;

extern "C" {
size_t mas_colsum_ws_bytes(mas_tensor4 t);
int mas_colsum(const float* x, mas_tensor4 t, float* out, void* ws, size_t ws_bytes, void* stream);

int mas_conv3x3_fprop(const float* x, mas_tensor4 xs, const float* w_packed, const float* bias, const float* residual, float* y,
                      mas_tensor4 ys, int mode, int impl, void* stream) {
  MAS_REQUIRE(x && w_packed && y, "conv3x3_fprop: null pointer");
  (void)impl;  // the tensor path takes differently packed weights: see mas_conv3x3_fprop_tc
  return conv3x3_fprop_simt_launch(x, xs, w_packed, bias, residual, y, ys, mode, 3, S(stream));
}

static size_t align256(size_t v) { return (v + 255) / 256 * 256; }

size_t mas_conv3x3_wgrad_ws_bytes(mas_tensor4 xs, mas_tensor4 dys, int mode) {
  size_t a = conv_wgrad_simt_ws(xs, dys, 3), b = conv_wgrad_tc_ws(xs, dys, mode);
  return align256(a > b ? a : b) + mas_colsum_ws_bytes(dys);
}

int mas_conv3x3_wgrad(const float* x, mas_tensor4 xs, const float* dy, mas_tensor4 dys, float* dw_oihw, float* dbias, int mode,
                      int impl, const float* gn_table, int gn_silu, void* ws, size_t ws_bytes, void* stream) {
  MAS_REQUIRE(x && dy && dw_oihw, "conv3x3_wgrad: null pointer");
  if (ws_bytes < mas_conv3x3_wgrad_ws_bytes(xs, dys, mode)) return fail(MAS_ERR_WORKSPACE, "conv3x3_wgrad: workspace too small");
  size_t a = conv_wgrad_simt_ws(xs, dys, 3), b = conv_wgrad_tc_ws(xs, dys, mode);
  size_t main_bytes = align256(a > b ? a : b);
  int e = MAS_ERR_UNSUPPORTED;
  if (impl != MAS_IMPL_SIMT) {
    e = conv_wgrad_tc_launch(x, xs, dy, dys, dw_oihw, dbias, mode, gn_table, gn_silu, 0, nullptr, (int)dys.c, 0, ws, main_bytes, S(stream));
    if (e != MAS_OK && (e != MAS_ERR_UNSUPPORTED || impl == MAS_IMPL_TC)) return e;
    if (e == MAS_OK) return MAS_OK;  // the tensor path also produced dbias
  }
  if (e == MAS_ERR_UNSUPPORTED) {
    if (gn_table) return fail(MAS_ERR_UNSUPPORTED, "conv3x3_wgrad: the fused GroupNorm prologue needs the tensor path (shape not eligible)");
    e = conv_wgrad_simt_launch(x, xs, dy, dys, dw_oihw, mode, 3, ws, main_bytes, S(stream));
    if (e) return e;
  }
  if (dbias) return mas_colsum(dy, dys, dbias, (char*)ws + main_bytes, ws_bytes - main_bytes, stream);
  return MAS_OK;
}

int mas_conv3x3_wgrad_tc_eligible(mas_tensor4 xs, mas_tensor4 dys, int mode) { return conv_wgrad_tc_eligible(xs, dys, mode) ? 1 : 0; }

int mas_conv3x3_wgrad_tc16(const void* x, int x_is_f16, mas_tensor4 xs, const float* dy, mas_tensor4 dys, float* dw_oihw, float* dbias,
                           int mode, const float* gn_table, int gn_silu, const float* dy_amax, int cout_rows, void* ws,
                           size_t ws_bytes, void* stream) {
  MAS_REQUIRE(x && dy && dw_oihw, "conv3x3_wgrad_tc16: null pointer");
  if (ws_bytes < mas_conv3x3_wgrad_ws_bytes(xs, dys, mode)) return fail(MAS_ERR_WORKSPACE, "conv3x3_wgrad_tc16: workspace too small");
  size_t a = conv_wgrad_simt_ws(xs, dys, 3), b = conv_wgrad_tc_ws(xs, dys, mode);
  return conv_wgrad_tc_launch((const float*)x, xs, dy, dys, dw_oihw, dbias, mode, gn_table, gn_silu, 1, dy_amax, cout_rows, x_is_f16, ws,
                              align256(a > b ? a : b), S(stream));
}

static mas_tensor4 rows_t4(int64_t M, int C, int64_t ld) {
  mas_tensor4 t;
  t.n = 1; t.h = 1; t.w = M; t.c = C;
  t.sn = M * ld; t.sh = M * ld; t.sw = ld; t.sc = 1;
  return t;
}
size_t mas_conv1x1_wgrad_ws_bytes(int64_t M, int Cin, int Cout) {
  size_t a = conv_wgrad_simt_ws(rows_t4(M, Cin, Cin), rows_t4(M, Cout, Cout), 1), b = conv1x1_wgrad_tc_ws(M, Cin, Cout);
  return align256(a > b ? a : b) + mas_colsum_ws_bytes(rows_t4(M, Cout, Cout));
}
int mas_conv1x1_wgrad(const float* x, int64_t ldx, const float* dy, int64_t ldy, int64_t M, int Cin, int Cout, float* dw,
                      float* dbias, int impl, void* ws, size_t ws_bytes, void* stream) {
  MAS_REQUIRE(x && dy && dw && M > 0 && ldx >= Cin && ldy >= Cout, "conv1x1_wgrad: bad arguments");
  if (ws_bytes < mas_conv1x1_wgrad_ws_bytes(M, Cin, Cout)) return fail(MAS_ERR_WORKSPACE, "conv1x1_wgrad: workspace too small");
  mas_tensor4 xs = rows_t4(M, Cin, ldx), ds = rows_t4(M, Cout, ldy);
  size_t a = conv_wgrad_simt_ws(rows_t4(M, Cin, Cin), rows_t4(M, Cout, Cout), 1), b = conv1x1_wgrad_tc_ws(M, Cin, Cout);
  size_t main_bytes = align256(a > b ? a : b);
  if (impl != MAS_IMPL_SIMT) {
    int e = conv1x1_wgrad_tc_launch(x, ldx, dy, ldy, M, Cin, Cout, dw, dbias, ws, main_bytes, S(stream));
    if (e == MAS_OK) return MAS_OK;
    if (e != MAS_ERR_UNSUPPORTED || impl == MAS_IMPL_TC) return e;
  }
  if (int e = conv_wgrad_simt_launch(x, xs, dy, ds, dw, MAS_CONV_S1, 1, ws, main_bytes, S(stream))) return e;
  if (dbias) return mas_colsum(dy, ds, dbias, (char*)ws + main_bytes, ws_bytes - main_bytes, stream);
  return MAS_OK;
}

int mas_gemm(const float* A, const float* B, float* C, int M, int N, int K, int batch, int64_t lda, int64_t ldb, int64_t ldc,
             int64_t stride_a, int64_t stride_b, int64_t stride_c, int trans_a, int trans_b, float alpha, const float* bias,
             const float* residual, int impl, void* stream) {
  MAS_REQUIRE(A && B && C && M > 0 && N > 0 && K > 0 && batch > 0, "gemm: bad arguments");
  if (impl == MAS_IMPL_TC3)   // explicit selection (the AttnBlock path does): never chosen by MAS_IMPL_AUTO
    return gemm_tc3_launch(A, B, C, M, N, K, batch, lda, ldb, ldc, stride_a, stride_b, stride_c, trans_a, trans_b, alpha, bias, residual,
                           S(stream));
  if (impl != MAS_IMPL_SIMT) {
    int e = gemm_tc_launch(A, B, C, M, N, K, batch, lda, ldb, ldc, stride_a, stride_b, stride_c, trans_a, trans_b, alpha, bias,
                           residual, S(stream));
    if (e != MAS_ERR_UNSUPPORTED || impl == MAS_IMPL_TC) return e;
  }
  return gemm_simt_launch(A, B, C, M, N, K, batch, lda, ldb, ldc, stride_a, stride_b, stride_c, trans_a, trans_b, alpha, bias,
                          residual, S(stream));
}

// outer x batch matrices, matrix (o, i) at o * outer_stride_? + i * stride_? (heads inside a fused [B, S, 3H] activation):
// one launch on the 3xTF32 kernel; the other implementations run one plain batched call per outer index.
int mas_gemm_batched2(const float* A, const float* B, float* C, int M, int N, int K, int outer, int batch, int64_t lda, int64_t ldb,
                      int64_t ldc, int64_t outer_stride_a, int64_t outer_stride_b, int64_t outer_stride_c, int64_t stride_a,
                      int64_t stride_b, int64_t stride_c, int trans_a, int trans_b, float alpha, int impl, int causal, void* stream) {
  MAS_REQUIRE(A && B && C && M > 0 && N > 0 && K > 0 && batch > 0 && outer > 0, "gemm_batched2: bad arguments");
  if (impl == MAS_IMPL_TC3)   // causal (see the header): a hint - the other implementations contract the (zero) blocks too
    return gemm_tc3_launch2(A, B, C, M, N, K, outer, batch, lda, ldb, ldc, outer_stride_a, outer_stride_b, outer_stride_c, stride_a,
                            stride_b, stride_c, trans_a, trans_b, alpha, nullptr, nullptr, causal, S(stream));
  for (int o = 0; o < outer; ++o) {
    const int e = mas_gemm(A + (int64_t)o * outer_stride_a, B + (int64_t)o * outer_stride_b, C + (int64_t)o * outer_stride_c, M, N, K,
                           batch, lda, ldb, ldc, stride_a, stride_b, stride_c, trans_a, trans_b, alpha, nullptr, nullptr, impl, stream);
    if (e) return e;
  }
  return MAS_OK;
}

}  // extern "C"
