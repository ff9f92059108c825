// DMMA throughput vs occupancy / independent chains / instruction shape (dev microbenchmark)
#include <cstdio>
#include <cuda_runtime.h>
template <int CH>
__global__ void k884(double* sink, int iters) {
  double c[CH][2];
#pragma unroll
  for (int i = 0; i < CH; ++i) c[i][0] = c[i][1] = 0.0;
  double a = 1.0 + threadIdx.x * 1e-9, b = 1.0 - threadIdx.x * 1e-9;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < CH; ++i)
      asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
                   : "+d"(c[i][0]), "+d"(c[i][1]) : "d"(a), "d"(b));
  }
  double s = 0; 
#pragma unroll
  for (int i = 0; i < CH; ++i) s += c[i][0] + c[i][1];
  if (s == 123.456) sink[0] = s;
}
#if defined(TRY_BIG)
template <int CH>
__global__ void k16816(double* sink, int iters) {
  double c[CH][4];
#pragma unroll
  for (int i = 0; i < CH; ++i) c[i][0] = c[i][1] = c[i][2] = c[i][3] = 0.0;
  double a0 = 1.0 + threadIdx.x * 1e-9, b0 = 1.0 - threadIdx.x * 1e-9;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < CH; ++i)
      asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7,%8,%9,%10,%11}, {%12,%13,%14,%15}, {%0,%1,%2,%3};\n"
                   : "+d"(c[i][0]), "+d"(c[i][1]), "+d"(c[i][2]), "+d"(c[i][3])
                   : "d"(a0), "d"(a0), "d"(a0), "d"(a0), "d"(a0), "d"(a0), "d"(a0), "d"(a0), "d"(b0), "d"(b0), "d"(b0), "d"(b0));
  }
  double s = 0;
#pragma unroll
  for (int i = 0; i < CH; ++i) s += c[i][0] + c[i][1] + c[i][2] + c[i][3];
  if (s == 123.456) sink[0] = s;
}
#endif
template <typename F>
void run(const char* name, F launch, double flop) {
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  launch(); cudaDeviceSynchronize();
  cudaEventRecord(e0); launch(); cudaEventRecord(e1); cudaEventSynchronize(e1);
  float ms; cudaEventElapsedTime(&ms, e0, e1);
  printf("%-34s %8.3f ms  %6.2f TFLOP/s\n", name, ms, flop / ms / 1e9);
}
int main() {
  double* sink; cudaMalloc(&sink, 64);
  int sms = 0, iters = 8192;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  for (int warps : {4, 8, 16, 32}) {
    for (int blocks : {1, 2}) {
      char nm[64];
      double f8 = 512.0 * iters * warps * blocks * sms;
      snprintf(nm, 64, "m8n8k4 ch=8  warps=%d x%d", warps, blocks);
      run(nm, [&] { k884<8><<<sms * blocks, warps * 32>>>(sink, iters); }, f8 * 8);
      snprintf(nm, 64, "m8n8k4 ch=32 warps=%d x%d", warps, blocks);
      run(nm, [&] { k884<32><<<sms * blocks, warps * 32>>>(sink, iters); }, f8 * 32);
#if defined(TRY_BIG)
      snprintf(nm, 64, "m16n8k16 ch=8 warps=%d x%d", warps, blocks);
      run(nm, [&] { k16816<8><<<sms * blocks, warps * 32>>>(sink, iters); }, 2.0 * 16 * 8 * 16 * iters * warps * blocks * sms * 8);
#endif
    }
  }
  return 0;
}
