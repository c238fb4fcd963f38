/* mas_b200.h — C-ABI of the H100-native VQ-IMG hot path (libmas_b200.so).
 *
 * The reference (CasualGANPapers/Make-A-Scene) is pure Python/PyTorch and has NO native interface;
 * every arithmetic step of its hot path is a stock ATen/cuDNN/cuBLAS call issued from
 * models/modules.py and models/vqvae.py.  Each entry point below replaces one such call site and
 * cites it (file:line relative to the reference root).  SURVEY.md 8(b) is the contract:
 *   - extern "C", plain pointers and sizes, no torch / C++ types in any signature;
 *   - every pointer is a DEVICE pointer unless the name ends in _host;
 *   - no hidden allocation, no hidden synchronisation: scratch comes from the caller (ws/ws_bytes,
 *     size from the matching *_ws_bytes function), work is enqueued on `stream` (a cudaStream_t
 *     passed as void*) and the call returns immediately;
 *   - return value: 0 = ok, <0 = error (MAS_ERR_*); mas_last_error() gives a thread-local message.
 *
 * Activation layout: fp32 "NHWC" (channels innermost).  Where an entry takes explicit element
 * strides (sn, sh, sw, sc) any layout — including the reference's NCHW — is accepted, which is how
 * the first/last convolutions read/write NCHW images without a transposing copy.
 */
#ifndef MAS_B200_H_
#define MAS_B200_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define MAS_OK 0
#define MAS_ERR_INVALID_ARG (-1)
#define MAS_ERR_UNSUPPORTED (-2)
#define MAS_ERR_LAUNCH (-3)
#define MAS_ERR_WORKSPACE (-4)

/* Input-coordinate maps of the 3x3 convolution family (modules.py:44-81). */
#define MAS_CONV_S1 0 /* stride 1, pad 1                       — nn.Conv2d(k=3,s=1,p=1), modules.py:93-104 */
#define MAS_CONV_S2 1 /* pad (0,1,0,1) + stride 2, pad 0       — Downsample.forward, modules.py:74-78      */
#define MAS_CONV_UP 2 /* nearest x2 upsample then stride 1 p1  — Upsample.forward, modules.py:55-59        */
#define MAS_CONV_ZS 3 /* zero-stuffed x2 input (data gradient of MAS_CONV_S2), stride 1 pad 1             */
/* Phase-decomposed forms of MAS_CONV_UP / MAS_CONV_S2 (mas_conv3x3_phase_tc16h); mas_conv3x3_tc_eligible(xs, ys, mode) with
 * the layer's input / output shapes answers whether both the forward and the data gradient can take them. */
#define MAS_CONV_UP_PHASE 4
#define MAS_CONV_S2_PHASE 5

/* Implementation selector for the contraction kernels. */
#define MAS_IMPL_AUTO 0  /* wgmma (TF32 operands, fp32 accumulate) when the shape is eligible, else SIMT */
#define MAS_IMPL_SIMT 1  /* fp32 FFMA kernels (exact fp32; also the on-GPU checker for the tensor path)      */
#define MAS_IMPL_TC 2    /* wgmma only; MAS_ERR_UNSUPPORTED if the shape is not eligible                   */
#define MAS_IMPL_TC3 3   /* mas_gemm only, explicit selection: fp32-accurate 3xTF32 operand-split wgmma GEMM
                          * (csrc/contract_tc3.cu; the AttnBlock token contractions run on it)                  */

typedef struct mas_tensor4 {
  int64_t n, h, w, c;     /* logical extents */
  int64_t sn, sh, sw, sc; /* element strides */
} mas_tensor4;

int mas_version(void);
const char* mas_last_error(void);
/* Number of kernels this library has launched in the calling process (bench.py's gpu_launches). */
int64_t mas_launch_count(void);
/* ... of which kernels that issue wgmma tensor-core MMAs (the driver's evidence that the tensor path ran). */
int64_t mas_tc_launch_count(void);

/* Measurement aid for bench.py: runs a pure-FFMA kernel (16 independent chains per thread, 148*4 blocks of 512 threads,
 * 128*iters FMAs per thread); *flops_out_host (HOST pointer, may be NULL) receives the FLOPs of one launch. `scratch`
 * needs 148*4*512 floats (never written). Timed by the caller with CUDA events => the fp32 FMA-pipe peak at the
 * clocks the GPU actually runs. */
int mas_ffma_probe(float* scratch, int iters, double* flops_out_host, void* stream);

/* ---- layout helpers (boundary only; the VQBASE path itself never transposes) ------------------- */
int mas_copy_strided(const float* x, mas_tensor4 xs, float* y, mas_tensor4 ys, void* stream);

/* NCHW (contiguous) -> channels-last with CP >= C channels, the extra ones zero (a 159-channel segmentation map becomes a
 * 160-channel operand of the tensor-core convolution); y = x * g[0] with g a device scalar (a loss's upstream gradient). */
int mas_nchw_to_nhwc_pad(const float* x_nchw, float* y_nhwc, int N, int C, int CP, int H, int W, void* stream);
int mas_scale_by(const float* x, const float* g, float* y, int64_t n, void* stream);

/* ---- GroupNorm(32, C, eps=1e-6) + optional SiLU — Normalize / nonlinearity, modules.py:35-41 ------
 * x, y: [N, HW, C] NHWC.  mean/rstd: [N*G].  silu=1 fuses x*sigmoid(x) (modules.py:122,126,194-196).
 * round_tf32=1 rounds y to TF32 (round-to-nearest) so that a following tensor-core contraction sees
 * correctly rounded operands; round_tf32=2: y receives fp16 values (N*HW*C halves: the shadow mas_conv3x3_fprop_tc16h reads).  Backward: dx = GN/SiLU input gradient (+ dx_add elementwise when not NULL, which
 * folds the residual-branch gradient of ResnetBlock/AttnBlock, modules.py:136,191); dgamma/dbeta are overwritten. */
size_t mas_gn_ws_bytes(int N, int HW, int C, int G);
int mas_gn_stats(const float* x, int N, int HW, int C, int G, float eps, float* mean, float* rstd,
                 void* ws, size_t ws_bytes, void* stream);
int mas_gn_apply(const float* x, const float* mean, const float* rstd, const float* gamma,
                 const float* beta, float* y, int N, int HW, int C, int G, int silu, int round_tf32,
                 void* stream);
int mas_gn_backward(const float* dy, const float* x, const float* mean, const float* rstd,
                    const float* gamma, const float* beta, const float* dx_add, float* dx, float* dgamma,
                    float* dbeta, void* act_out, int act_f16, float* dx_amax, const float* add_amax, void* dx_f16,
                    float* dx_bound, int N, int HW, int C, int G, int silu, void* ws, size_t ws_bytes, void* stream);
/* act_out (or NULL): also writes act(GN(x)), the operand of the following weight gradient - as fp32, or with act_f16 != 0
 * as fp16 (what mas_conv3x3_wgrad_tc16(..., x_is_f16 = 1) stages without converting); dx_amax (or NULL): device
 * scalar receiving max|dx| (what mas_amax(dx) would return), for the fp16-operand kernels that consume dx.  dx_f16 (or NULL): also write dx as an fp16 channels-last
 * shadow for mas_conv3x3_fprop_tc16h, scaled by the power of two derived from *dx_bound - a rigorous bound on max|dx| that
 * is known before the apply pass: rstd*(max|dy*silu'*gamma| + |B| + max|xhat|*|A|) over (image, group), the two maxima
 * collected by the first pass, plus *add_amax = max|dx_add| (required with dx_add); dx_bound is written for the consumer. */
/* out = a + b (gradient of x+h where the two branches cannot be fused). */
int mas_add(const float* a, const float* b, float* out, int64_t n, void* stream);
/* Standalone Swish module (modules.py:194-196). */
int mas_silu_forward(const float* x, float* y, int64_t n, void* stream);
int mas_silu_backward(const float* dy, const float* x, float* dx, int64_t n, void* stream);

/* ---- 3x3 convolution family — nn.Conv2d / Downsample / Upsample, modules.py:44-81,93-104 ----------
 * w_packed: [9*Cin, Cout] row-major, row index (ty*3+tx)*Cin+ci (mas_pack_conv3x3 builds it from the
 * reference's [Cout,Cin,3,3] parameter; flip_transpose=1 builds the data-gradient form
 * [9*Cout, Cin] with taps flipped).  y = conv(x) + bias + residual (bias/residual may be NULL;
 * residual has y's strides).  x and y carry explicit strides. */
int mas_pack_conv3x3(const float* w_oihw, float* w_packed, int Cout, int Cin, int flip_transpose,
                     int round_tf32, void* stream);
int mas_conv3x3_fprop(const float* x, mas_tensor4 xs, const float* w_packed, const float* bias,
                      const float* residual, float* y, mas_tensor4 ys, int mode, int impl, void* stream);
/* Tensor-core (wgmma, TF32 operands / fp32 accumulate) form of the same convolution for dense NHWC
 * tensors with Cin % 8 == 0, Cout % 128 == 0, Hout % 16 == 0, Wout % 8 == 0 and mode S1 / UP / ZS
 * (mas_conv3x3_tc_eligible).  w_tc comes from mas_pack_conv3x3_tc (transpose=1: data-gradient operand with
 * flipped taps); the packed image is what one cp.async.bulk per pipeline stage drops into shared memory. */
int mas_conv3x3_tc_eligible(mas_tensor4 xs, mas_tensor4 ys, int mode);
int mas_pack_conv3x3_tc(const float* w_oihw, float* w_tc, int Cout, int Cin, int transpose, void* stream);
/* Fusions on the tensor path (north_star: "fused GroupNorm+SiLU+Conv2d tiles"):
 *  gn_table  [N,Cin,2] (mas_gn_table) or NULL — the A-operand producers apply a = act(x*sc + sh) while staging, so the
 *            normalised/activated tensor of modules.py:121-126 is never written; gn_silu selects the Swish.
 *  stats_part or NULL — the epilogue also emits per-(tile, 32-row group, channel quad) sum / sum of squares of the
 *            stored output, [tiles][4][Cout/4][2] floats with tiles = N*(Hout/16)*(Wout/8); mas_gn_finalize_partials
 *            turns them into the NEXT GroupNorm's mean/rstd (deterministic), replacing a full read of the tensor. */
int mas_conv3x3_fprop_tc(const float* x, mas_tensor4 xs, const float* w_tc, const float* bias,
                         const float* residual, float* y, mas_tensor4 ys, int mode, const float* gn_table,
                         int gn_silu, float* stats_part, void* stream);
/* fp16-operand form of the same kernel (wgmma kind::f16, fp32 accumulate): an fp16 significand has the 11 bits of a TF32
 * one, so the rounding of the operands is the same as on the TF32 path, while one MMA instruction (and one byte of
 * shared-memory operand traffic, the kernel's limiter) carries twice the FLOPs.  The narrower exponent range is handled by
 * a power-of-two operand scale derived ON THE DEVICE from x_amax (a device scalar holding max|x|, from mas_amax; NULL = no
 * scaling, right for post-GroupNorm activations): x*s is converted with round-to-nearest (saturating), the epilogue
 * multiplies by 1/s, both exact.  Needs Cin % 16 == 0 on top of mas_conv3x3_tc_eligible.  w_tc16 comes from
 * mas_pack_conv3x3_tc16: 9*Cout*Cin halves ([n_tile][k_chunk][tap][k/8][128][8]); with w_tc16_dgrad != NULL the forward
 * packing goes to w_tc16 and the data-gradient packing (transpose = 1) to w_tc16_dgrad in one pass over the weight. */
int mas_amax(const float* x, int64_t n, float* out, void* stream);
int mas_pack_conv3x3_tc16(const float* w_oihw, void* w_tc16, void* w_tc16_dgrad, int Cout, int Cin, int transpose,
                          void* stream);
int mas_conv3x3_fprop_tc16(const float* x, mas_tensor4 xs, const void* w_tc16, const float* bias,
                           const float* residual, float* y, mas_tensor4 ys, int mode, const float* gn_table,
                           int gn_silu, float* stats_part, const float* x_amax, void* stream);
/* TMA-fed form of the fp16-operand 3x3 stride-1 convolution (csrc/conv_tma.cu; nn.Conv2d 3x3, modules.py:93-104, forward and
 * data gradient): the A operand is read by the copy engine from an fp16 channels-last "shadow" x_f16 [N][H][W][Cin] of the
 * (already activated) input - written by mas_gn_apply(round_tf32 = 2), mas_gn_backward(dx_f16) or mas_to_half - so no thread
 * of the kernel touches the operands.  x_amax: the device scalar the shadow's power-of-two scale was derived from (NULL for an
 * unscaled shadow).  Eligible: dense NHWC, Cin % 64 == 0, H % 16 == 0, W % 8 == 0, Cout % 4 == 0 (weights / bias packed for
 * round_up(Cout, 128) rows).  Same packed weights (mas_pack_conv3x3_tc16), residual and GroupNorm-statistics epilogues as
 * mas_conv3x3_fprop_tc16.  mas_to_half: y = fp16(x * s), s = the power-of-two operand scale of *amax (NULL: 1). */
int mas_conv3x3_tc16h_eligible(mas_tensor4 xs, mas_tensor4 ys);
int mas_conv3x3_fprop_tc16h(const void* x_f16, mas_tensor4 xs, const void* w_tc16, const float* bias,
                            const float* residual, float* y, mas_tensor4 ys, float* stats_part,
                            const float* x_amax, void* stream);
int mas_to_half(const float* x, void* y_f16, int64_t n, const float* amax, void* stream);
/* Upsample / Downsample convolution (mode MAS_CONV_UP_PHASE / MAS_CONV_S2_PHASE) in phase-decomposed form on the same TMA-fed
 * kernel: the Upsample is four 2x2 convolutions of the low-resolution input (taps summed per output phase), the Downsample
 * reads the four phase planes of its input with 4 / 2 / 2 / 1 of the nine taps each.  transpose = 0: forward (x_f16 the
 * layer input, y its output, bias optional); transpose = 1: data gradient (x_f16 the output-gradient shadow, y = dx, no
 * bias).  Phase planes are read through tensor-map strides: no copy of any of them is made.  Weights: the
 * mas_pack_conv3x3_phase16 image of the same mode and transpose (Upsample 16 Cout Cin halves, Downsample 9 Cout Cin);
 * combined taps are summed in fp32 and rounded to fp16 once.  Eligible: see MAS_CONV_UP_PHASE. */
int mas_pack_conv3x3_phase16(const float* w_oihw, void* w_ph16, int Cout, int Cin, int mode, int transpose, void* stream);
int mas_conv3x3_phase_tc16h(const void* x_f16, mas_tensor4 xs, const void* w_ph16, const float* bias, float* y,
                            mas_tensor4 ys, int mode, int transpose, const float* x_amax, void* stream);
/* Weight (and bias) gradient of the same layer from two fp16 shadows, phase-decomposed on the TMA-fed weight-gradient
 * kernel: x_f16 the layer input (xs), scaled by the power-of-two operand scale of *x_amax (NULL: unscaled); dy_f16 the output
 * gradient (dys), scaled by that of *dy_amax.  The Upsample runs 16 per-phase 2 x 2 correlations of the low-resolution x
 * and sums them into the nine taps in a fixed order; the Downsample runs each of the nine taps once over a phase plane of
 * x.  dw_oihw [Cout][Cin][3][3] and dbias [Cout] (or NULL) are overwritten; deterministic (no atomics).  ws: at least
 * mas_conv3x3_phase_wgrad_tc16_ws_bytes(xs, dys, mode) bytes (0: the shape is not eligible, see MAS_CONV_UP_PHASE). */
size_t mas_conv3x3_phase_wgrad_tc16_ws_bytes(mas_tensor4 xs, mas_tensor4 dys, int mode);
int mas_conv3x3_phase_wgrad_tc16(const void* x_f16, mas_tensor4 xs, const float* x_amax, const void* dy_f16,
                                 mas_tensor4 dys, const float* dy_amax, float* dw_oihw, float* dbias, int mode, void* ws,
                                 size_t ws_bytes, void* stream);
/* Both packings of one weight (transpose = 0 and 1 of mas_pack_conv3x3_tc) in a single pass; Cout % 128 == Cin % 128 == 0. */
int mas_pack_conv3x3_tc_pair(const float* w_oihw, float* w_tc_fwd, float* w_tc_dgrad, int Cout, int Cin, void* stream);
int mas_gn_finalize_partials(const float* part, int tiles_per_image, int N, int C, int G, int64_t hw, float eps,
                             float* mean, float* rstd, void* stream);
int mas_gn_table(const float* mean, const float* rstd, const float* gamma, const float* beta, int N, int C, int G,
                 float* table, void* stream);
/* Row GEMM on the tensor path for 1x1 convolutions: C[M,N] = alpha * A[M,K] . W^T + bias + residual with W
 * [N,K] row-major packed by mas_pack_gemm_tc (transpose=1 packs W^T for the data gradient: N<->K).
 * Needs N % 128 == 0 and K % 32 == 0 (after the optional transpose). */
int mas_pack_gemm_tc(const float* w_nk, float* w_tc, int N, int K, int transpose, void* stream);
int mas_gemm_rows_packed(const float* A, int64_t lda, const float* w_tc, float* C, int64_t ldc, int64_t M, int N,
                         int K, float alpha, const float* bias, const float* residual, float* stats_part,
                         void* stream);  /* stats_part as above with 128-row tiles: [M/128][4][N/4][2] */
/* Row GEMM on fp16 operands read by the copy engine (csrc/gemm_tma.cu; nn.Linear forward / data gradient, transformer.py:17-56):
 * y[M,N] = alpha * x[M,K] . W^T (+bias +residual), x_f16 a dense [M,K] fp16 copy of x (mas_to_half, scaled by the power-of-two
 * operand scale of *x_amax when x_amax != NULL: the epilogue undoes it), w_tc16 from mas_pack_gemm_tc16 (transpose=1 packs W^T:
 * the data gradient dx = dy . W).  Needs K % 64 == 0; output features padded to 128 inside the packed image (N % 128 == 0 for
 * the packer).  fp16 operands carry the same 11-bit significand as the TF32 path; fp32 accumulate. */
int mas_pack_gemm_tc16(const float* w_nk, void* w_tc16, int N, int K, int transpose, void* stream);
int mas_gemm_rows_f16(const void* x_f16, int64_t M, int K, const void* w_tc16, float* y, int64_t ldy, int N, const float* bias,
                      const float* residual, const float* x_amax, float alpha, void* stream);
/* Weight gradient of the same layer from the two fp16 copies: dw[N,K] = dy^T . x (reduction over the M rows; dy^T through tensor
 * memory, x tiles as the copy engine lands them, split-K partials in ws reduced in a fixed order), dbias[N] = column sums of dy
 * (may be NULL).  x_f16 [M,K] / dy_f16 [M,N] dense, scaled by the operand scales of *x_amax / *dy_amax (NULL: unscaled).
 * Needs N % 128 == 0 and K % 128 == 0. */
size_t mas_wgrad_rows_f16_ws_bytes(int64_t M, int N, int K);
int mas_wgrad_rows_f16(const void* x_f16, const void* dy_f16, int64_t M, int N, int K, float* dw, float* dbias,
                       const float* x_amax, const float* dy_amax, void* ws, size_t ws_bytes, void* stream);
/* Diagnostic: wgmma D[128x32] = A[128x8].B[32x8]^T (TF32, 2 x m64) with A from shared memory (a_src=0) or registers
 * (a_src=1) and B K-major (b_layout=0) or MN-major (1; 2 = LBO/SBO fields swapped). Used by the tests to pin the
 * descriptor conventions the production kernels rely on. b_layout=99: B descriptor bits (sm_100 encoding) /
 * start offset are taken verbatim from raw_* and the B region holds its own word indices (address reveal). */
int mas_tc_probe(const float* A, const float* B, float* D, int a_src, int b_layout, uint64_t raw_desc,
                 uint32_t raw_idesc, int raw_off, void* stream);
/* fp16 address-reveal form: D[k][n] (k < 16, n < N; D is [128][N]) = index of the half the tensor core reads for element
 * (n, k) of a B operand described by the raw descriptor (MN-major when bit 16 of raw_idesc is set, N = 8 x bits 17-22 of
 * raw_idesc, 32 or 128), from a region filled with 0..2047. */
int mas_tc_probe16(float* D, uint64_t raw_desc, uint32_t raw_idesc, int raw_off, void* stream);
/* Weight gradient, written in the reference's [Cout,Cin,3,3] layout; dbias [Cout] may be NULL.
 * x is the convolution's (already normalised+activated) input, dy the output gradient. */
size_t mas_conv3x3_wgrad_ws_bytes(mas_tensor4 xs, mas_tensor4 dys, int mode);
int mas_conv3x3_wgrad(const float* x, mas_tensor4 xs, const float* dy, mas_tensor4 dys, float* dw_oihw,
                      float* dbias, int mode, int impl, const float* gn_table, int gn_silu, void* ws,
                      size_t ws_bytes, void* stream);
/* fp16-operand tensor-core form (see mas_conv3x3_fprop_tc16): dy is scaled by a power of two derived on the device from
 * dy_amax (device scalar from mas_amax, or NULL), x (or act(GroupNorm(x)) with gn_table) is converted unscaled.
 * MAS_ERR_UNSUPPORTED unless mas_conv3x3_wgrad_tc_eligible (dense NHWC, Cin % 32 == 0, Cout % 128 == 0, H, W % 8 == 0,
 * mode S1 / UP).  Workspace: mas_conv3x3_wgrad_ws_bytes.  dbias (may be NULL) is produced too.
 * cout_rows = rows of dw_oihw / dbias: dys.c normally; with dys.c % 128 != 0 (a multiple of 4) pass round_up(dys.c, 128) and
 * buffers of that many rows - the TMA copy of dy zero-fills the missing channels and the extra rows come out zero.  x_is_f16 carries operand flags: bit 0 - x holds fp16
 * (mas_gn_apply(round_tf32 = 2) / mas_gn_backward(act_f16)); bit 1 - dy is the fp16 shadow written by mas_gn_backward(dx_f16),
 * already scaled by the power of two of *dy_amax (= that call's dx_bound). */
int mas_conv3x3_wgrad_tc_eligible(mas_tensor4 xs, mas_tensor4 dys, int mode);
int mas_conv3x3_wgrad_tc16(const void* x, int x_is_f16, mas_tensor4 xs, const float* dy, mas_tensor4 dys, float* dw_oihw,
                           float* dbias, int mode, const float* gn_table, int gn_silu, const float* dy_amax, int cout_rows,
                           void* ws, size_t ws_bytes, void* stream);   /* x_is_f16: x holds fp16 (dense NHWC, no gn_table) */  /* gn_table: x is re-activated on the fly (tensor path only) */
/* Weight gradient of a 1x1 convolution: dw[Cout,Cin] = dy^T x over M rows (split over rows, deterministic);
 * dbias [Cout] may be NULL. x [M,Cin] and dy [M,Cout] are row-major with row pitches ldx / ldy (elements). */
size_t mas_conv1x1_wgrad_ws_bytes(int64_t M, int Cin, int Cout);
int mas_conv1x1_wgrad(const float* x, int64_t ldx, const float* dy, int64_t ldy, int64_t M, int Cin, int Cout,
                      float* dw, float* dbias, int impl, void* ws, size_t ws_bytes, void* stream);
/* Edge convolutions (3x3, stride 1, pad 1) with exactly 3 channels on one side — conv_in / conv_out of Encoder/Decoder
 * (modules.py:219,364).  The 3-channel tensor carries explicit strides (the caller's NCHW image / reconstruction);
 * the wide tensor is dense NHWC.  small_cin_fprop with flip_transpose=1 and w = the [3,C,3,3] weight of conv_out is
 * conv_out's data gradient.  Weight/bias gradients are deterministic (persistent blocks + ordered reduction). */
int mas_edge_small_cin_fprop(const float* xs, mas_tensor4 xst, const float* w, const float* bias, float* y,
                             mas_tensor4 yst, int flip_transpose, void* stream);
int mas_edge_small_cout_fprop(const float* a, mas_tensor4 at, const float* w, const float* bias, float* ys,
                              mas_tensor4 yst, void* stream);
size_t mas_edge_wgrad_ws_bytes(int Cbig);
int mas_edge_small_cin_wgrad(const float* xs, mas_tensor4 xst, const float* dy, mas_tensor4 dyt, float* dw,
                             float* dbias, void* ws, size_t ws_bytes, void* stream);
int mas_edge_small_cout_wgrad(const float* a, mas_tensor4 at, const float* dys, mas_tensor4 dyt, float* dw,
                              float* dbias, void* ws, size_t ws_bytes, void* stream);
/* Stride-2 convolution (Downsample, modules.py:74-78) on the stride-1 tensor kernels: space-to-depth of the input
 * ([N,H,W,C] -> [N,H/2,W/2,4C]) turns it into a 2x2-tap unit-stride convolution, run as a 3x3 convolution with the
 * remapped weight W9 [Cout,4C,3,3] (mas_s2d_pack_weights); mas_s2d_unpack_wgrad maps dW9 back to dW [Cout,C,3,3]. */
int mas_space_to_depth(const float* x, float* y, int N, int H, int W, int C, void* stream);
int mas_s2d_pack_weights(const float* w, float* w9, int Cout, int C, void* stream);
int mas_s2d_unpack_wgrad(const float* dw9, float* dw, int Cout, int C, void* stream);
/* 2x2 sum pooling: data gradient of the nearest x2 upsample (modules.py:56). x [N,2H,2W,C] -> y [N,H,W,C]. */
int mas_sumpool2x2(const float* x, float* y, int N, int H, int W, int C, void* stream);

/* ---- batched GEMM — Conv2d 1x1 (modules.py:113-117,145-164; vqvae.py:15,18) and torch.bmm
 * (modules.py:179,186).  Row-major.  C[b] = alpha * op(A[b]) * op(B[b]) + bias[n] + residual[b].
 * op(A) is M x K, op(B) is K x N; trans_a: A stored K x M; trans_b: B stored N x K.
 * lda/ldb/ldc row pitches, stride_* batch pitches (elements); bias/residual may be NULL
 * (residual shares C's ldc / stride_c). */
int mas_gemm(const float* A, const float* B, float* C, int M, int N, int K, int batch, int64_t lda,
             int64_t ldb, int64_t ldc, int64_t stride_a, int64_t stride_b, int64_t stride_c, int trans_a,
             int trans_b, float alpha, const float* bias, const float* residual, int impl, void* stream);
/* Two-level batch: outer x batch matrices, matrix (o, i) at o * outer_stride_? + i * stride_? - the heads of a fused
 * [B, S, 3H] q|k|v activation (transformer.py:77-103) in ONE launch on the 3xTF32 kernel (impl = MAS_IMPL_TC3, outer * batch
 * <= 65535); other impl values run one mas_gemm per outer index.  No bias / residual.
 * causal: structure hint for the square (queries x keys, key <= query) attention matrices - identically-zero K chunks and
 * output tiles are skipped by the 3xTF32 kernel (other implementations ignore it; results are the same because the skipped
 * operand blocks are zero / the skipped outputs are never consumed): 0 none; 1 A[m][k] = 0 for k > m (ctx = P v, dQ = dS k);
 * 2 A stored [K][M] with A[k][m] = 0 for k < m (dV = P^T dO, dK = dS^T q); 3 outputs with n > m unused, whole tiles above the
 * diagonal are written as zeros (S = q k^T, dP = dO v^T). */
int mas_gemm_batched2(const float* A, const float* B, float* C, int M, int N, int K, int outer, int batch, int64_t lda,
                      int64_t ldb, int64_t ldc, int64_t outer_stride_a, int64_t outer_stride_b, int64_t outer_stride_c,
                      int64_t stride_a, int64_t stride_b, int64_t stride_c, int trans_a, int trans_b, float alpha, int impl,
                      int causal, void* stream);
/* Column sums of a strided [N,H,W,C] view (bias gradients): out[c] = sum_{n,h,w} x[n,h,w,c]. Deterministic. */
size_t mas_colsum_ws_bytes(mas_tensor4 t);
int mas_colsum(const float* x, mas_tensor4 t, float* out, void* ws, size_t ws_bytes, void* stream);

/* ---- AttnBlock softmax over keys — modules.py:180-181,185 ------------------------------------------
 * rows x cols row-major; forward is in place capable (p may alias s). backward: ds = p*(dp - sum(dp*p))*scale. */
int mas_softmax_forward(const float* s, float* p, int64_t rows, int cols, void* stream);
int mas_softmax_backward(const float* p, const float* dp, float* ds, int64_t rows, int cols, float scale,
                         void* stream);

/* ---- AttnBlock as one unit — replaces AttnBlock.forward (modules.py:167-191) and its autograd graph ------
 * x, hn, O, out, dout, dx: [N*HW, C] NHWC rows; qkv: [N*HW, 3C] (q | k | v per row); P: [N, HW, HW] softmax over keys.
 * mean/rstd: GroupNorm(G) statistics of x (mas_gn_stats or a producer's statistics epilogue).  Weights in the
 * reference layout ([C, C(,1,1)] row-major, biases [C]).  hn, qkv, P, O are outputs of the forward that the caller
 * keeps for the backward.  stats_part (or NULL): statistics partials of `out` for the next GroupNorm
 * ([N*HW/128][4][C/4][2], tensor path and HW % 128 == 0 only).  dqkv_w [3C, C] / dqkv_b [3C] hold the q, k, v gradients
 * back to back.  The 1x1 convolutions use the wgmma row GEMM / weight-gradient kernels when C % 128 == 0 (impl as
 * MAS_IMPL_*); QK^T, PV and their gradients are strict fp32 like torch.bmm (modules.py:180,186). */
size_t mas_attnblock_ws_bytes(int N, int HW, int C, int G);
int mas_attnblock_forward(const float* x, int N, int HW, int C, int G, const float* mean, const float* rstd,
                          const float* norm_w, const float* norm_b, const float* q_w, const float* q_b,
                          const float* k_w, const float* k_b, const float* v_w, const float* v_b,
                          const float* proj_w, const float* proj_b, float* hn, float* qkv, float* P, float* O,
                          float* out, float* stats_part, int impl, void* ws, size_t ws_bytes, void* stream);
int mas_attnblock_backward(const float* dout, const float* x, int N, int HW, int C, int G, const float* mean,
                           const float* rstd, const float* norm_w, const float* norm_b, const float* q_w,
                           const float* k_w, const float* v_w, const float* proj_w, const float* hn,
                           const float* qkv, const float* P, const float* O, float* dx, float* dnorm_w,
                           float* dnorm_b, float* dqkv_w, float* dqkv_b, float* dproj_w, float* dproj_b,
                           float* dx_amax /* or NULL: max|dx|, see mas_gn_backward */, int impl, void* ws,
                           size_t ws_bytes, void* stream);

/* ---- (Sync)BatchNorm for quant_conv[1] — vqvae.py:16 ---------------------------------------------------
 * x [R, C] NHWC rows.  mas_bn_stats writes LOCAL [sum(C), sumsq(C), R] as fp64 (2*C+1 doubles: the last one is the
 * local row count); the caller all-reduces those 2*C+1 numbers across ranks over NCCL, then mas_bn_finalize turns the
 * global sums into mean / invstd (biased variance) and updates running_mean / running_var (unbiased,
 * momentum; either may be NULL) exactly like nn.SyncBatchNorm; count <= 0 means "read the reduced count from
 * stats[2*C]" (ranks with different batch sizes, no host round trip).  Backward: mas_bn_backward_reduce writes the
 * LOCAL [sum_dy(C), sum_dy_xhat(C), R] (fp64, 2*C+1) for the second all-reduce; mas_bn_backward_apply consumes the
 * global sums for dx (inv_count <= 0: 1 / sums_global[2*C]) and the local sums for dgamma/dbeta (DDP all-reduces
 * parameter grads itself). */
int mas_bn_stats(const float* x, int64_t R, int C, double* stats_out, void* stream);
int mas_bn_finalize(const double* stats, double count, int C, float eps, float momentum, float* mean,
                    float* invstd, float* running_mean, float* running_var, void* stream);
/* eval mode: invstd = 1/sqrt(running_var + eps) for mas_bn_apply (nn.BatchNorm2d.eval()) */
int mas_bn_invstd(const float* running_var, float eps, float* invstd, int C, void* stream);
int mas_bn_apply(const float* x, const float* mean, const float* invstd, const float* gamma,
                 const float* beta, float* y, int64_t R, int C, void* stream);
int mas_bn_backward_reduce(const float* dy, const float* x, const float* mean, const float* invstd,
                           int64_t R, int C, double* sums_out, void* stream);
int mas_bn_backward_apply(const float* dy, const float* x, const float* mean, const float* invstd,
                          const float* gamma, const double* sums_global, const double* sums_local,
                          double inv_count, float* dx, float* dgamma, float* dbeta, int64_t R, int C,
                          void* stream);

/* ---- PatchGAN discriminator — losses/discriminator.py:21-35 ---------------------------------------------
 * nn.Conv2d(k=4, s in {1, 2}, p=1) (+ LeakyReLU(0.2) after the first one), nn.BatchNorm2d + LeakyReLU(0.2) (plain, per-call
 * batch statistics), csrc/conv4x4.cu and csrc/norm.cu.  The convolutions are exact-fp32 SIMT implicit GEMMs over explicit
 * strides and any channel counts (the first reads the caller's NCHW image, the last has Cout = 1).
 * mas_pack_conv4x4: [Cout,Cin,4,4] -> transpose 0: [(4kh+kw)*Cin + ci][co] (forward operand); transpose 1:
 * [(4kh+kw)*Cout + co][ci] (data-gradient operand).
 * mas_conv4x4: y = conv(x) (+bias[co] when bias != NULL), then LeakyReLU(act_slope) when act != 0.  ys.h = (xs.h - 2) / stride + 1.
 * mas_conv4x4_dgrad: dx of that convolution from dy (any strides: an expanded loss gradient with zero strides is fine).
 * mas_conv4x4_wgrad: dw [Cout,Cin,4,4] (OIHW), deterministic (split over pixels, ordered reduction); bias gradients are
 * mas_colsum(dy).  Workspace: mas_conv4x4_wgrad_ws_bytes.
 * mas_lrelu_backward: dx = dy * (y > 0 ? 1 : slope) with y the LeakyReLU output (dense, n elements).
 * BatchNorm2d + LeakyReLU: mas_bn_stats, then mas_bn_finalize(count = 0) (momentum, eps, unbiased running variance as
 * nn.BatchNorm2d), then mas_bn_apply_lrelu: y = LeakyReLU(slope)(BN(x)).  Backward from dy = dL/dy, y the forward output:
 * mas_bn_backward_reduce_lrelu writes [sum_dz(C), sum_dz_xhat(C), R] of dz = dy * LeakyReLU'(y) (row chunks, then an ordered
 * sum: deterministic; workspace mas_bn_backward_reduce_lrelu_ws_bytes), and
 * mas_bn_backward_apply_lrelu writes dx and (when dgamma != NULL) dgamma / dbeta from those sums.  Eval mode: mas_bn_invstd
 * of the running variance with the running mean in mas_bn_apply_lrelu. */
int mas_pack_conv4x4(const float* w_oihw, float* w_packed, int Cout, int Cin, int transpose, void* stream);
int mas_conv4x4(const float* x, mas_tensor4 xs, const float* w_packed, const float* bias, float* y, mas_tensor4 ys, int stride,
                float act_slope, int act, void* stream);
int mas_conv4x4_dgrad(const float* dy, mas_tensor4 dys, const float* w_packed_t, float* dx, mas_tensor4 dxs, int stride,
                      void* stream);
size_t mas_conv4x4_wgrad_ws_bytes(mas_tensor4 xs, mas_tensor4 dys);
int mas_conv4x4_wgrad(const float* x, mas_tensor4 xs, const float* dy, mas_tensor4 dys, float* dw_oihw, int stride, void* ws,
                      size_t ws_bytes, void* stream);
int mas_lrelu_backward(const float* dy, const float* y, float slope, float* dx, int64_t n, void* stream);
/* Tensor-core route of the 4x4 convolution (dense NHWC, Cout % 128 == 0, stride 2 with even extents): it is the 3x3 stride-1
 * pad-1 convolution of the 4*Cin-channel shift map X'(i, j, (2p + q)*Cin + c) = x(s*i + p, s*j + q, c) (0 outside x;
 * X' is H/s x W/s) with the remapped weight W3 [Cout, 4*Cin, 3, 3]: 4x4 tap kh is the 3x3 tap a of plane p with
 * kh = 2a - 1 + p at stride 2 (16 of the 36 taps), kh = a (p = 0) for kh < 3 and (a, p) = (2, 1) for kh = 3 at stride 1.
 * So the forward, data gradient and weight gradient run on mas_conv3x3_fprop_tc16 / mas_conv3x3_wgrad_tc16 (fp16 operands,
 * power-of-two scales from device-side amax, fp32 accumulate).  At stride 1 the 3x3 output is H x W: its last row and column
 * are dropped (the layer's output is the H-1 x W-1 view), and the output gradient handed to the data / weight gradient must be
 * zero there.  mas_conv4x4_shift_map writes X' (dense); mas_conv4x4_shift_map_adjoint writes dx from dX' (sum over the up to
 * four X' positions that read each x element); mas_conv4x4_remap_weight: to3x3 = 1 writes W3 from w [Cout,Cin,4,4],
 * to3x3 = 0 writes dw [Cout,Cin,4,4] from dW3. */
int mas_conv4x4_shift_map(const float* x, mas_tensor4 xs, float* y, int stride, void* stream);
int mas_conv4x4_shift_map_adjoint(const float* dmap, float* dx, mas_tensor4 dxs, int stride, void* stream);
int mas_conv4x4_remap_weight(const float* src, float* dst, int Cout, int Cin, int stride, int to3x3, void* stream);
int mas_bn_apply_lrelu(const float* x, const float* mean, const float* invstd, const float* gamma, const float* beta, float slope,
                       float* y, int64_t R, int C, void* stream);
size_t mas_bn_backward_reduce_lrelu_ws_bytes(int64_t R, int C);
int mas_bn_backward_reduce_lrelu(const float* dy, const float* y, float slope, const float* x, const float* mean,
                                 const float* invstd, int64_t R, int C, double* sums_out, void* ws, size_t ws_bytes,
                                 void* stream);
int mas_bn_backward_apply_lrelu(const float* dy, const float* y, float slope, const float* x, const float* mean,
                                const float* invstd, const float* gamma, const double* sums, float* dx, float* dgamma,
                                float* dbeta, int64_t R, int C, void* stream);

/* ---- Codebook (vector quantiser) — modules.py:470-473,501-517 ---------------------------------------
 * z: [R, D] latent rows (NHWC order, R = B*h*w), E: [K, D] codebook.
 * idx_out[r] = argmin_k ( (|z_r|^2 + |e_k|^2) - 2 z_r.e_k ), fp32, the reference's association and
 * first-index tie-break (modules.py:501-505).  zq_out[r] = E[idx] (modules.py:506).
 * loss_out (1 float) = (1+beta) * mean((zq - z)^2)  (modules.py:509; both terms are numerically equal
 * in the forward).  The distance matrix is never materialised. */
/* mas_vq_forward picks the arg-min with a tensor-core FILTER (csrc/vq_tc.cu: 2 x fp16 operand split, 3 MMAs per K step,
 * the four best candidates per row) followed by an exact fp32 re-evaluation of every row whose runner-up lies within a
 * rigorous error margin of the best candidate - the indices are those of the exact-fp32 FFMA kernel, bit for bit - when
 * D % 32 == 0 and the latent tile fits shared memory (D <= 256); otherwise, or after mas_vq_select_path(0), the FFMA kernel
 * evaluates every (row, code) pair.  mas_vq_select_path is process-wide (A/B measurements, tests). */
int mas_vq_select_path(int use_tensor_core_filter);
size_t mas_vq_ws_bytes(int64_t R, int K, int D);
int mas_vq_forward(const float* z, const float* E, int64_t R, int K, int D, float beta, int64_t* idx_out,
                   float* zq_out, float* loss_out, void* ws, size_t ws_bytes, void* stream);
/* Backward (modules.py:509-512): grad_z = g_zq + g_loss*(2/(R*D))*(z - zq);
 * grad_E[k] += g_loss*(2*beta/(R*D)) * sum_{r: idx_r = k} (e_k - z_r).  grad_E must be zeroed by the caller. */
/* Same gather + loss + straight-through value for CALLER-SUPPLIED code indices (the argmin is skipped): teacher-forced
 * quantisation, e.g. re-evaluating the codebook loss of stored codes (modules.py:506-512 with idx given). */
int mas_vq_forward_given(const float* z, const float* E, const int64_t* idx_in, int64_t R, int K, int D, float beta,
                         float* zq_out, float* loss_out, void* ws, size_t ws_bytes, void* stream);
/* Lloyd update step for Codebook re-initialisation (modules.py:487-499, replacing the un-installed fast_pytorch_kmeans;
 * the assignment step is mas_vq_forward): centres_new[k] = mean of the rows x[r] with idx[r] == k (an empty cluster keeps
 * centres_old[k]); shift_out (device scalar, may be NULL) = |centres_new - centres_old|_F. */
size_t mas_kmeans_ws_bytes(int K, int D);
int mas_kmeans_update(const float* x, const int64_t* idx, int64_t n, int K, int D, const float* centres_old,
                      float* centres_new, float* shift_out, void* ws, size_t ws_bytes, void* stream);
int mas_vq_backward(const float* g_zq, const float* g_loss, const float* z, const float* E,
                    const int64_t* idx, int64_t R, int K, int D, float beta, float* grad_z, float* grad_E,
                    void* stream);
/* get_codebook_entry gather (modules.py:519-528): out[r] = E[idx[r]]. */
int mas_vq_gather(const float* E, const int64_t* idx, int64_t R, int K, int D, float* out, void* stream);

/* ---- tier 2: token transformer (models/transformer.py) ---------------------------------------------------------
 * LayerNorm over the last dimension of x [R,H] (+ optional fused residual add: y = LN(x) + residual, the sandwich-LN
 * pattern of transformer.py:183-208); tanh-GELU (transformer.py:11-14); causal softmax over [mats, rows, cols] score
 * matrices (row i sees columns 0..i+cols-rows; transformer.py:57-71,90); fused token + position embedding sum written
 * into rows [off, off+seg) of each length-`total` sequence (transformer.py:350-364). Linear layers / attention
 * contractions go through mas_gemm_rows_packed / mas_gemm / mas_conv1x1_wgrad. */
int mas_layernorm_forward(const float* x, const float* gamma, const float* beta, const float* residual, float* y,
                          float* mean, float* rstd, int64_t R, int H, float eps, void* stream);
/* Two chained LayerNorms of a decode step (inference, R <= 64 rows): y1 = residual + LN1(x) (residual may be NULL) and
 * y2 = LN2(y1) - the sandwich LayerNorm and the next sub-layer's input LayerNorm (transformer.py:183-208) in one launch. */
int mas_layernorm2_forward(const float* x, const float* gamma1, const float* beta1, const float* residual, float* y1,
                           const float* gamma2, const float* beta2, float* y2, int64_t R, int H, float eps1, float eps2,
                           void* stream);
size_t mas_layernorm_ws_bytes(int64_t R, int H);
int mas_layernorm_backward(const float* dy, const float* x, const float* mean, const float* rstd,
                           const float* gamma, float* dx, float* dgamma, float* dbeta, int64_t R, int H, void* ws,
                           size_t ws_bytes, void* stream);
int mas_gelu_forward(const float* x, float* y, int64_t n, void* stream);
int mas_gelu_backward(const float* dy, const float* x, float* dx, int64_t n, void* stream);
int mas_softmax_causal_forward(const float* s, float* p, int64_t mats, int rows, int cols, void* stream);
/* ds = p * (dp - sum_visible(dp * p)) * scale on the visible columns (0..i+cols-rows) of each row, zeros beyond; dp is not read
 * beyond the visible columns (the causal dP GEMM leaves whole tiles unwritten there); ds may alias dp. */
int mas_softmax_causal_backward(const float* p, const float* dp, float* ds, int64_t mats, int rows, int cols, float scale,
                                void* stream);
int mas_embed3_forward(const float* t0, const int64_t* id0, const float* t1, const int64_t* id1, const float* t2,
                       const int64_t* id2, float* out, int64_t R, int H, int seg, int total, int off, void* stream);
int mas_embed3_backward(const float* dout, const int64_t* id0, float* d0, const int64_t* id1, float* d1,
                        const int64_t* id2, float* d2, int64_t R, int H, int seg, int total, int off, void* stream);
/* Causal self-attention core of the token transformer, fused (transformer.py:77-103; csrc/attn_causal.cu): per (sequence,
 * head, 128-query tile) S = q k^T * scale in registers -> causal softmax on the accumulator fragment -> P (written once, [B,heads,S,S],
 * zeros above the diagonal: the backward reads it) -> ctx = P v accumulated in registers.  qkv [B,S,3*heads*hd] fused
 * q|k|v, ctx [B,S,heads*hd], amax = device scalar max|qkv| (mas_amax).  Needs hd == 64 and S % 128 == 0
 * (MAS_ERR_UNSUPPORTED otherwise: the caller runs the GEMM / softmax sequence).  2 x fp16 operand split = fp32-level accuracy. */
int mas_attn_causal_forward(const float* qkv, const float* amax, float* P, float* ctx, int B, int S, int heads, int hd,
                            float scale, void* stream);
/* Token cross-entropy, train.py:150-153 (F.cross_entropy(logits.view(-1, V), img_token.view(-1)), mean reduction):
 * logits [R, V] with row pitch ld, target int64 [R] (outside [0, V): row ignored like ignore_index).  forward writes the
 * per-row losses, the per-row logsumexp (kept for the backward) and out[0] = mean loss, out[1] = counted rows.
 * backward: dlogits[r, c] = (softmax(logits_r)[c] - [c == target_r]) * dloss[0] / out[1]; dlogits may alias logits. */
int mas_ce_forward(const float* logits, int64_t ld, const int64_t* target, float* loss_rows, float* lse, float* out,
                   int64_t R, int V, void* stream);
int mas_ce_backward(const float* logits, int64_t ld, const int64_t* target, const float* lse, const float* stat,
                    const float* dloss, float* dlogits, int64_t ldd, int64_t R, int V, void* stream);

/* ---- Autoregressive sampling with a KV cache (SURVEY.md 8f-3) ---------------------------------------------
 * The reference has no working cached path (models/transformer.py:73-115 vs :176-210; train.py never samples); the
 * specification is its non-cached forward (transformer.py:77-103, 216-244): a decode step reproduces the logits the
 * full causal forward gives at that position.
 * mas_linear_small: y[r,n] = act(sum_k x[r,k] W[n,k] + b[n]) for R <= 8 rows (cond + uncond streams), strict fp32,
 *   W [N,K] row-major (nn.Linear layout) streamed once; act 0 = none, 1 = tanh-GELU (transformer.py:11-14).
 * mas_kv_append: k / v thirds of a fused qkv activation [R,T,3H] -> caches [R,heads,Tmax,hd] at pos0..pos0+T-1.
 * mas_attn_decode: softmax(q k^T / sqrt(hd)) v for ONE query per (row, head) (qkv [R,3H]) over the first `len`
 *   cached positions; ctx [R,H].  mas_cfg_mix: out = uncond + scale * (cond - uncond) (classifier-free guidance). */
int mas_linear_small(const float* x, int64_t ldx, const float* W, const float* bias, float* y, int64_t ldy, int R, int N,
                     int K, int act, void* stream);
int mas_kv_append(const float* qkv, int R, int T, int heads, int hd, float* kcache, float* vcache, int Tmax, int pos0,
                  void* stream);
int mas_attn_decode(const float* qkv, const float* kcache, const float* vcache, float* ctx, int R, int heads, int hd,
                    int Tmax, int len, void* stream);
/* mas_attn_decode with the cache append folded in: the k / v thirds of qkv [R,3H] are stored at position pos and the query
 * attends over positions 0..pos (one launch per layer instead of mas_kv_append + mas_attn_decode). */
int mas_attn_decode_append(const float* qkv, float* kcache, float* vcache, float* ctx, int R, int heads, int hd, int Tmax,
                           int pos, void* stream);
int mas_cfg_mix(const float* cond, const float* uncond, float* out, int64_t n, float scale, void* stream);
/* Token draw of the sampler (replaces the div / topk / where / softmax / multinomial chain of generate()): per row,
 * z = logits / temperature, entries below the top_k-th largest value dropped (top_k <= 0 or >= V: none), p = softmax(z),
 * tokens[r] = first index whose running sum of p exceeds u[r] (u in [0,1): caller-supplied uniforms, device floats). */
int mas_sample_topk(const float* logits, int64_t ld, int R, int V, float temperature, int top_k, const float* u,
                    int64_t* tokens, void* stream);

/* ---- weighted BCE-with-logits (VQ-SEG loss, losses/loss_seg.py:15-22) — "next" row ------------------
 * logits/target: strided [N,H,W,C] views; pos_weight [C]; loss_out = mean over all elements. grad may be NULL. */
int mas_bce_logits(const float* logits, mas_tensor4 ls, const float* target, mas_tensor4 ts,
                   const float* pos_weight, float* loss_out, float* grad, mas_tensor4 gs, float grad_scale,
                   void* ws, size_t ws_bytes, void* stream);
size_t mas_bce_ws_bytes(mas_tensor4 ls);
/* The VQ-SEG step's own layouts: logits channels-last with channel pitch CP >= C (the padded output of the decoder's last
 * convolution), target NCHW (the data loader's maps), W % 32 == 0.  mas_bce_cl_forward: loss = mean over N*C*H*W.
 * mas_bce_cl_backward: grad[n,h,w,c] = g[0] * dloss/dlogit (g: device scalar from autograd, NULL = 1), pad channels
 * written as 0 - so the loss's backward runs here, not in the host framework (losses/loss_seg.py:15-22). */
size_t mas_bce_cl_ws_bytes(int N, int H, int W);
int mas_bce_cl_forward(const float* logits, const float* target_nchw, const float* pos_weight, int N, int C, int CP, int H,
                       int W, float* loss_out, void* ws, size_t ws_bytes, void* stream);
int mas_bce_cl_backward(const float* logits, const float* target_nchw, const float* pos_weight, const float* g, int N, int C,
                        int CP, int H, int W, float* grad, void* stream);


/* ---- LPIPS perceptual loss (losses/lpips.py; csrc/lpips.cu) ------------------------------------------------------------
 * The thirteen VGG16 3x3 convolutions (lpips.py:106-111, torchvision vgg16 features[0:30]) run on the 3x3 family above
 * (mas_conv3x3_fprop_tc16 / mas_conv3x3_fprop, mas_edge_small_cin_fprop / mas_edge_small_cout_fprop for conv1_1); these
 * entries are the rest of LPIPS.forward (lpips.py:66-73) and its data gradient.  Activations are channels-last fp32 over
 * ONE batch of 2B images, real first then fake.
 * mas_lpips_prep: ScalingLayer (lpips.py:81-82), (x - shift) / scale of NCHW real and fake [B,3,H,W] -> out [2B,H,W,3].
 * mas_lpips_relu: nn.ReLU (features 1, 3, 6, ...) in place on n floats; amax (or NULL) = max of the result.
 * mas_lpips_maxpool: nn.MaxPool2d(2, 2) (features 4, 9, 16, 23), floor mode: x [N,H,W,C] -> y [N,H/2,W/2,C]; amax as above.
 * mas_lpips_head_forward: for tap [2B,H,W,C] (relu1_2 .. relu5_3), part[b][k] (k < mas_lpips_head_blocks()) = partial sums
 *   over pixels of sum_c w_lin[c] (n_real - n_fake)^2, n = f / (sqrt(sum_c f^2) + 1e-10) (norm_tensor, lpips.py:128-135;
 *   NetLinLayer, lpips.py:90-96; Dropout is the identity in eval mode).
 * mas_lpips_head_finalize: out[b] = sum over the five taps, in order, of sum_k part[l][b][k] / hw_l (spatial_average and the
 *   sum of lpips.py:73); part [5][B][mas_lpips_head_blocks()].
 * mas_lpips_tap_backward: d p_b / d (pre-ReLU tap) for a unit seed on every p_b, for the G images g0 .. g0+G-1 of the 2B
 *   batch (their partners: the other half), plus the gradient dpool [G,H/2,W/2,C] of the following max-pool (NULL: none)
 *   at the first maximum of each window; ReLU mask as a select (a pixel whose tap vector is all zero writes 0).
 *   dz [G,H,W,C]; amax (or NULL) = max|dz|.
 * mas_lpips_relu_backward: dx = y > 0 ? dy : 0 (threshold_backward; dx may alias dy); amax as above.
 * mas_lpips_prep_backward: ScalingLayer backward, dxp [G,H,W,3] -> J [G,3,H,W] = dxp / scale.
 * mas_lpips_scale_jacobian: out[b, :] = g[b * g_stride] * J[b, :] (per image of `per` floats): every traversal of the
 *   graph after the one that computed J. */
int mas_lpips_prep(const float* real, const float* fake, const float* shift, const float* scale, float* out, int B, int H, int W,
                   void* stream);
int mas_lpips_relu(float* y, int64_t n, float* amax, void* stream);
int mas_lpips_maxpool(const float* x, float* y, int N, int H, int W, int C, float* amax, void* stream);
int mas_lpips_head_blocks(void);
int mas_lpips_head_forward(const float* tap, const float* w_lin, int B, int H, int W, int C, double* part, void* stream);
int mas_lpips_head_finalize(const double* part, int B, int64_t hw0, int64_t hw1, int64_t hw2, int64_t hw3, int64_t hw4, float* out,
                            void* stream);
int mas_lpips_tap_backward(const float* tap, const float* w_lin, int B, int H, int W, int C, int g0, int G, const float* dpool,
                           float* dz, float* amax, void* stream);
int mas_lpips_relu_backward(const float* dy, const float* y, float* dx, int64_t n, float* amax, void* stream);
int mas_lpips_prep_backward(const float* dxp, const float* scale, float* J, int G, int H, int W, void* stream);
int mas_lpips_scale_jacobian(const float* J, const float* g, int64_t g_stride, float* out, int B, int64_t per, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* MAS_B200_H_ */
