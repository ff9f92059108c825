// DMMA throughput per f64 instruction shape vs warps per SM and independent accumulator
// chains (dev microbenchmark).  Build: nvcc -O3 -gencode arch=compute_90a,code=sm_90a
// dmma_occ.cu -o dmma_occ.  Warps 4 and 8 are one and two warps per SM sub-partition.
#include <cstdio>
#include <cuda_runtime.h>

// SHAPE: 0 = m8n8k4, 1 = m16n8k4, 2 = m16n8k8, 3 = m16n8k16
template <int SHAPE> struct Shape;
template <> struct Shape<0> { static constexpr int M = 8, N = 8, K = 4, NA = 1, NB = 1, NC = 2; };
template <> struct Shape<1> { static constexpr int M = 16, N = 8, K = 4, NA = 2, NB = 1, NC = 4; };
template <> struct Shape<2> { static constexpr int M = 16, N = 8, K = 8, NA = 4, NB = 2, NC = 4; };
template <> struct Shape<3> { static constexpr int M = 16, N = 8, K = 16, NA = 8, NB = 4, NC = 4; };

template <int SHAPE>
__device__ __forceinline__ void mma(double* c, double a, double b) {
  if constexpr (SHAPE == 0)
    asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
                 : "+d"(c[0]), "+d"(c[1]) : "d"(a), "d"(b));
  else if constexpr (SHAPE == 1)
    asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};\n"
                 : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3]) : "d"(a), "d"(a), "d"(b));
  else if constexpr (SHAPE == 2)
    asm volatile("mma.sync.aligned.m16n8k8.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, "
                 "{%0,%1,%2,%3};\n"
                 : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3]) : "d"(a), "d"(a), "d"(a), "d"(a), "d"(b), "d"(b));
  else
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, "
                 "{%4,%5,%6,%7,%8,%9,%10,%11}, {%12,%13,%14,%15}, {%0,%1,%2,%3};\n"
                 : "+d"(c[0]), "+d"(c[1]), "+d"(c[2]), "+d"(c[3])
                 : "d"(a), "d"(a), "d"(a), "d"(a), "d"(a), "d"(a), "d"(a), "d"(a), "d"(b), "d"(b), "d"(b), "d"(b));
}

template <int SHAPE, int CH>
__global__ void kmma(double* sink, int iters) {
  constexpr int NC = Shape<SHAPE>::NC;
  double c[CH][NC];
#pragma unroll
  for (int i = 0; i < CH; ++i)
#pragma unroll
    for (int e = 0; e < NC; ++e) c[i][e] = 0.0;
  double a = 1.0 + threadIdx.x * 1e-9, b = 1.0 - threadIdx.x * 1e-9;
  for (int it = 0; it < iters; ++it) {
#pragma unroll
    for (int i = 0; i < CH; ++i) mma<SHAPE>(c[i], a, b);
  }
  double s = 0;
#pragma unroll
  for (int i = 0; i < CH; ++i)
#pragma unroll
    for (int e = 0; e < NC; ++e) s += c[i][e];
  if (s == 123.456) sink[0] = s;
}

template <typename F>
void run(const char* name, F launch, double flop) {
  launch();
  if (cudaGetLastError() != cudaSuccess) {  // e.g. more registers than the block size allows
    printf("%-36s launch refused\n", name);
    return;
  }
  cudaDeviceSynchronize();
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0);
  cudaEventCreate(&e1);
  cudaEventRecord(e0);
  launch();
  cudaEventRecord(e1);
  cudaEventSynchronize(e1);
  float ms;
  cudaEventElapsedTime(&ms, e0, e1);
  printf("%-36s %8.3f ms  %6.2f TFLOP/s\n", name, ms, flop / ms / 1e9);
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
}

template <int SHAPE, int CH>
void shape_row(const char* sname, double* sink, int sms, int warps, int blocks, int iters) {
  using S = Shape<SHAPE>;
  char nm[64];
  snprintf(nm, 64, "%-9s ch=%-2d warps=%-2d x%d", sname, CH, warps, blocks);
  const double flop = 2.0 * S::M * S::N * S::K * CH * (double)iters * warps * blocks * sms;
  run(nm, [&] { kmma<SHAPE, CH><<<sms * blocks, warps * 32>>>(sink, iters); }, flop);
}

int main() {
  double* sink;
  cudaMalloc(&sink, 64);
  int sms = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  cudaDeviceProp prop;
  cudaGetDeviceProperties(&prop, 0);
  printf("%s, %d SMs\n", prop.name, sms);
  // iters scale with 1/K, so every shape does the same work per chain
  for (int warps : {4, 8, 16}) {
    for (int blocks : {1, 2}) {
      shape_row<0, 8>("m8n8k4", sink, sms, warps, blocks, 8192);
      shape_row<0, 16>("m8n8k4", sink, sms, warps, blocks, 8192);
      shape_row<1, 8>("m16n8k4", sink, sms, warps, blocks, 8192);
      shape_row<1, 16>("m16n8k4", sink, sms, warps, blocks, 8192);
      shape_row<2, 8>("m16n8k8", sink, sms, warps, blocks, 4096);
      shape_row<2, 16>("m16n8k8", sink, sms, warps, blocks, 4096);
      shape_row<3, 8>("m16n8k16", sink, sms, warps, blocks, 2048);
      shape_row<3, 16>("m16n8k16", sink, sms, warps, blocks, 2048);
    }
  }
  cudaError_t err = cudaDeviceSynchronize();
  if (err != cudaSuccess) {
    printf("error: %s\n", cudaGetErrorString(err));
    return 1;
  }
  return 0;
}
