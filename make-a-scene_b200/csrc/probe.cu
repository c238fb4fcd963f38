// Measurement aid (bench.py): the fp32 FFMA rate this GPU sustains at its current clocks — the denominator for kernels
// that are bound by the FMA pipe (the exact-fp32 VQ distance kernel). Not part of the model path.
#include "mas_common.cuh"

namespace mas {
// 16 independent accumulator chains per thread, 4 warps per scheduler: the FMA pipe is the only limiter
__global__ void __launch_bounds__(512) ffma_probe_kernel(float* __restrict__ out, int iters, float a, float b) {
  float acc[16];
#pragma unroll
  for (int j = 0; j < 16; ++j) acc[j] = (float)(threadIdx.x + j);
  for (int i = 0; i < iters; ++i) {
#pragma unroll
    for (int u = 0; u < 8; ++u)
#pragma unroll
      for (int j = 0; j < 16; ++j) acc[j] = fmaf(acc[j], a, b);
  }
  float s = 0.f;
#pragma unroll
  for (int j = 0; j < 16; ++j) s += acc[j];
  if (s == 123.456f) out[blockIdx.x * blockDim.x + threadIdx.x] = s;   // never true: keeps the chains alive
}
}  // namespace mas

using namespace mas;

extern "C" {
// Launches the probe; *flops_out (host) receives the FLOPs one launch executes (2 per FMA).
int mas_ffma_probe(float* scratch, int iters, double* flops_out_host, void* stream) {
  MAS_REQUIRE(scratch && iters > 0, "ffma_probe: bad arguments");
  const int blocks = NUM_SMS * 4, threads = 512;
  ffma_probe_kernel<<<blocks, threads, 0, S(stream)>>>(scratch, iters, 0.999f, 0.001f);
  if (flops_out_host) *flops_out_host = 2.0 * 16 * 8 * (double)iters * blocks * threads;
  return launched("ffma_probe");
}
}
