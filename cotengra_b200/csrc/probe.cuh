// probe.cuh -- register-resident microbenchmarks for the fp64 roofline
// denominators (the m16n8k4 DMMA the fp64 tensor-core kernels issue, and the
// DFMA pipe) on the current device.  Include after gett_kernels.cuh.
#pragma once
#include <cuda_runtime.h>

namespace ctgb {

__global__ void __launch_bounds__(256) probe_dmma_kernel(double* sink, int iters) {
  double c[8][2][2];
#pragma unroll
  for (int i = 0; i < 8; ++i) c[i][0][0] = c[i][0][1] = c[i][1][0] = c[i][1][1] = 0.0;
  double a = 1.0 + threadIdx.x * 1e-9, b = 1.0 - threadIdx.x * 1e-9;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < 8; ++i) dmma16x8x4(c[i][0], c[i][1], a, a, b);
  }
  double s = 0.0;
#pragma unroll
  for (int i = 0; i < 8; ++i) s += c[i][0][0] + c[i][0][1] + c[i][1][0] + c[i][1][1];
  if (s == 123.456) sink[0] = s;
}

__global__ void __launch_bounds__(256) probe_dfma_kernel(double* sink, int iters) {
  double c[8];
#pragma unroll
  for (int i = 0; i < 8; ++i) c[i] = i;
  const double a = 1.0000001, b = 1e-9 * threadIdx.x;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < 8; ++i) c[i] = fma(c[i], a, b);
  }
  double s = 0.0;
#pragma unroll
  for (int i = 0; i < 8; ++i) s += c[i];
  if (s == 123.456) sink[0] = s;
}

}  // namespace ctgb
