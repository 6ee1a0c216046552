// Latency / throughput of mma.sync.m16n8k32.s32.u8.s8 (IMMA.16832) and of the LDS -> LOP3 -> IMMA chain on sm_90a.
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o imma_lat imma_lat.cu && ./imma_lat
#include <cstdio>
#include <cuda_runtime.h>
__device__ __forceinline__ void imma(int (&d)[4], unsigned a0, unsigned a1, unsigned a2, unsigned a3, unsigned b0, unsigned b1) {
  asm volatile("mma.sync.aligned.m16n8k32.row.col.s32.u8.s8.s32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};"
      : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]) : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "r"(b0), "r"(b1));
}
template <int kChains>
__global__ void k_lat(long long* out, int iters, unsigned seed) {
  int d[kChains][4];
#pragma unroll
  for (int c = 0; c < kChains; ++c) { d[c][0] = d[c][1] = d[c][2] = d[c][3] = 0; }
  unsigned a = seed + threadIdx.x, b = seed * 3 + threadIdx.x;
  long long t0 = clock64();
  for (int i = 0; i < iters; ++i) {
#pragma unroll
    for (int c = 0; c < kChains; ++c) imma(d[c], a, a ^ 1, a ^ 2, a ^ 3, b, b ^ 5);
  }
  long long t1 = clock64();
  int s = 0;
#pragma unroll
  for (int c = 0; c < kChains; ++c) s += d[c][0] + d[c][1] + d[c][2] + d[c][3];
  if (threadIdx.x == 0 && blockIdx.x == 0) { out[0] = t1 - t0; out[1] = s; }
}
int main() {
  long long* d; cudaMalloc(&d, 16); long long h[2];
  const int iters = 2000;
  for (int warps : {1, 2, 4, 8, 16}) {
    k_lat<1><<<1, 32 * warps>>>(d, iters, 7); cudaMemcpy(h, d, 16, cudaMemcpyDeviceToHost);
    printf("{\"chains\":1,\"warps\":%d,\"cycles_per_imma_per_warp\":%.2f}\n", warps, double(h[0]) / iters);
    k_lat<2><<<1, 32 * warps>>>(d, iters, 7); cudaMemcpy(h, d, 16, cudaMemcpyDeviceToHost);
    printf("{\"chains\":2,\"warps\":%d,\"cycles_per_imma_per_warp\":%.2f}\n", warps, double(h[0]) / iters / 2);
    k_lat<4><<<1, 32 * warps>>>(d, iters, 7); cudaMemcpy(h, d, 16, cudaMemcpyDeviceToHost);
    printf("{\"chains\":4,\"warps\":%d,\"cycles_per_imma_per_warp\":%.2f}\n", warps, double(h[0]) / iters / 4);
  }
  return 0;
}
