// FP64 tensor-core rate: mma.sync.m8n8k4.f64 with 8 independent accumulator tiles per warp,
// nw warps on one sub-partition (warps 0,4,8,12) or spread over the four sub-partitions (warps 0..nw-1);
// compare with the same warps issuing DFMAs (256 FMAs per DMMA = 8 warp-wide DFMAs).
#include <cstdio>
#include <cuda_runtime.h>
__device__ __forceinline__ void dmma(double& c0, double& c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}
__global__ void k(double* out, long long* cyc, int iters, int mode, int nw, int same_sub) {
  const int warp = threadIdx.x >> 5;
  const int mine = same_sub ? ((warp & 3) == 0 && (warp >> 2) < nw) : (warp < nw);
  if (!mine) return;
  double c[16];
  for (int q = 0; q < 16; ++q) c[q] = q;
  double a = 1.0 + threadIdx.x * 1e-9, b = 1.0000001;
  const long long t0 = clock64();
  if (mode == 0) {
    for (int i = 0; i < iters; ++i)
#pragma unroll
      for (int q = 0; q < 8; ++q) dmma(c[2 * q], c[2 * q + 1], a, b);
  } else if (mode == 1) {   // dependent chain: latency
    for (int i = 0; i < iters; ++i)
#pragma unroll
      for (int q = 0; q < 8; ++q) dmma(c[0], c[1], a, b);
  } else {
    for (int i = 0; i < iters; ++i)
#pragma unroll
      for (int q = 0; q < 16; ++q) c[q] = fma(c[q], b, a);
  }
  const long long t1 = clock64();
  double s = 0;
  for (int q = 0; q < 16; ++q) s += c[q];
  if (s == 1.2345) out[threadIdx.x] = s;
  if (threadIdx.x == 0) *cyc = t1 - t0;
}
int main() {
  double* out; long long* cyc; long long h;
  cudaMalloc(&out, 8192); cudaMalloc(&cyc, 8);
  const int iters = 2000;
  for (int same = 1; same >= 0; --same)
    for (int nw = 1; nw <= 4; nw *= 2)
      for (int mode = 0; mode < 3; ++mode) {
        for (int rep = 0; rep < 2; ++rep) { k<<<1, 512>>>(out, cyc, iters, mode, nw, same); cudaDeviceSynchronize(); }
        cudaMemcpy(&h, cyc, 8, cudaMemcpyDeviceToHost);
        const double per = h / (double)(iters * (mode == 2 ? 16 : 8));
        printf("%s nw=%d %-28s cycles per instr (warp 0) %.2f\n", same ? "one sub-partition " : "four sub-partitions", nw,
               mode == 0 ? "DMMA m8n8k4, 8 independent" : (mode == 1 ? "DMMA m8n8k4, dependent" : "DFMA, 16 independent"), per);
      }
  printf("%s\n", cudaGetErrorString(cudaGetLastError()));
}
