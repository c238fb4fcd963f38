// Shared declarations of the edge-convolution kernels (edge.cu: generic channel counts; edge_quad.cu: Cbig % 128 == 0).
#pragma once
#include "mas_common.cuh"

namespace mas {
constexpr int SC = 3;  // the "small" channel count

struct EdgeGeom {
  int N, H, W, Cbig;
  int64_t sn, sh, sw, sc;  // strides of the SMALL-channel tensor (image / reconstruction / its gradient)
};

// register-tiled variants (lane = four wide-side channels, warp = a 2-row strip walked with a sliding 4x3 window)
constexpr int EDGE_Q_BLOCKS = NUM_SMS;  // persistent blocks of the weight-gradient kernels = rows of their partial buffer
int small_cin_fprop_q_launch(const float* xs, const float* w, const float* bias, float* y, const EdgeGeom& g, int flipT, cudaStream_t st);
int small_cout_fprop_q_launch(const float* a, const float* w, const float* bias, float* ys, const EdgeGeom& g, cudaStream_t st);
int small_cin_wgrad_q_launch(const float* xs, const float* dy, float* part, const EdgeGeom& g, cudaStream_t st);   // part [EDGE_Q_BLOCKS][28][Cbig]
int small_cout_wgrad_q_launch(const float* a, const float* dys, float* part, const EdgeGeom& g, cudaStream_t st);  // part [EDGE_Q_BLOCKS][30][Cbig]
}  // namespace mas
