// Latency of the 6x6 pivot-chain variants of k_solve, one warp alone on an SM (cycles per call).
// nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o chol chol.cu && ./chol
#include <cstdio>
#include <cuda_runtime.h>

__device__ __forceinline__ double fast_rsqrt(double a) {
  double y;
  asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(a));
  const double h = 0.5 * a;
  y = fma(y, fma(-h * y, y, 0.5), y);
  y = fma(y, fma(-h * y, y, 0.5), y);
  return y;
}
__device__ __forceinline__ double fast_rcp(double a) {
  double y;
  asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(a));
  double e = fma(-a, y, 1.0);
  y = fma(y, e, y);
  e = fma(-a, y, 1.0);
  y = fma(y, e, y);
  return y;
}
__device__ __forceinline__ double fast_rcp1(double a) {   // one Newton step
  double y;
  asm("rcp.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(a));
  double e = fma(-a, y, 1.0);
  y = fma(y, e, y);
  return y;
}

template <int MODE>
__device__ __forceinline__ double chol_warp(double a, int lane) {
  int u = lane < 21 ? lane : 20;
  const int r = (u >= 1) + (u >= 3) + (u >= 6) + (u >= 10) + (u >= 15);
  const int c = u - r * (r + 1) / 2;
  const int rb = r * (r + 1) / 2, cb = c * (c + 1) / 2;
  double dvc = 1.;
#pragma unroll
  for (int p = 0; p < 6; ++p) {
    const double dv = __shfl_sync(0xffffffffu, a, p * (p + 1) / 2 + p);
    const double x = __shfl_sync(0xffffffffu, a, rb + p);
    const double y = __shfl_sync(0xffffffffu, a, cb + p);
    double inv;
    if (MODE == 0) inv = fast_rcp(dv);
    else if (MODE == 1) inv = fast_rcp1(dv);
    else inv = 1.0 / dv;
    const double upd = fma(-(x * y), inv, a);
    a = (c > p) ? upd : a;
    dvc = (c == p) ? dv : dvc;
  }
  return a * fast_rsqrt(dvc);
}

__device__ __forceinline__ double chol_regs(double seed) {
  double a[21], l[21];
#pragma unroll
  for (int i = 0; i < 21; ++i) a[i] = seed * 0.01 * (i + 1);
#pragma unroll
  for (int r = 0; r < 6; ++r) a[r * (r + 1) / 2 + r] += 10.;
#pragma unroll
  for (int c = 0; c < 6; ++c) {
    const double dv = a[c * (c + 1) / 2 + c];
    const double ri = fast_rsqrt(dv);
    l[c * (c + 1) / 2 + c] = dv * ri;
#pragma unroll
    for (int r = c + 1; r < 6; ++r) l[r * (r + 1) / 2 + c] = a[r * (r + 1) / 2 + c] * ri;
#pragma unroll
    for (int r = c + 1; r < 6; ++r)
#pragma unroll
      for (int c2 = c + 1; c2 <= r; ++c2) a[r * (r + 1) / 2 + c2] -= l[r * (r + 1) / 2 + c] * l[c2 * (c2 + 1) / 2 + c];
  }
  double s = 0;
#pragma unroll
  for (int i = 0; i < 21; ++i) s += l[i];
  return s;
}

template <int MODE>
__global__ void k(double* out, long long* cyc, int iters, int noise_warps) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  if (warp > 0) {   // background load on the other warps: independent DFMA streams
    if (warp <= noise_warps) {
      double acc[8] = {1, 2, 3, 4, 5, 6, 7, 8};
      for (int i = 0; i < iters * 40; ++i)
#pragma unroll
        for (int q = 0; q < 8; ++q) acc[q] = fma(acc[q], 1.0000001, 0.5);
      double s = 0;
      for (int q = 0; q < 8; ++q) s += acc[q];
      if (s == 12345.) out[threadIdx.x] = s;
    }
    return;
  }
  double v = 1.0 + lane * 1e-3;
  const long long t0 = clock64();
  for (int i = 0; i < iters; ++i) {
    if (MODE == 3) v = chol_regs(v) * 1e-3 + 1.0;
    else {
      int u = lane < 21 ? lane : 20;
      const int r = (u >= 1) + (u >= 3) + (u >= 6) + (u >= 10) + (u >= 15);
      const int c = u - r * (r + 1) / 2;
      const double a = (r == c ? 10. : 0.) + 0.01 * v;
      v = chol_warp<MODE>(a, lane) * 1e-3 + 1.0;
    }
  }
  const long long t1 = clock64();
  if (lane == 0) { *cyc = (t1 - t0) / iters; out[0] = v; }
}

__global__ void k_dep(double* out, long long* cyc, int iters, int kind) {
  double v = 1.0 + threadIdx.x * 1e-3;
  const long long t0 = clock64();
  if (kind == 0) for (int i = 0; i < iters; ++i) v = fma(v, 1.0000001, 0.5);
  if (kind == 1) for (int i = 0; i < iters; ++i) { double y; asm volatile("rcp.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(v)); v = y; }
  if (kind == 2) for (int i = 0; i < iters; ++i) v = __shfl_sync(0xffffffffu, v, (threadIdx.x + 1) & 31);
  if (kind == 3) for (int i = 0; i < iters; ++i) { double y; asm volatile("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(v)); v = y; }
  if (kind == 4) for (int i = 0; i < iters; ++i) v = (threadIdx.x & 1) ? v * 1.0000001 : v;   // select
  const long long t1 = clock64();
  if (threadIdx.x == 0) { *cyc = (t1 - t0); out[0] = v; }
  if (v == 123.456) out[1] = v;
}

int main() {
  double* out; long long* cyc;
  cudaMalloc(&out, 8 * 1024); cudaMalloc(&cyc, 8);
  long long h;
  const char* names[4] = {"warp chol, rcp 2 Newton", "warp chol, rcp 1 Newton", "warp chol, IEEE division", "register chol (redundant lanes)"};
  for (int noise = 0; noise <= 12; noise += 4) {
    for (int m = 0; m < 4; ++m) {
      for (int rep = 0; rep < 2; ++rep) {
        if (m == 0) k<0><<<1, 512>>>(out, cyc, 200, noise);
        if (m == 1) k<1><<<1, 512>>>(out, cyc, 200, noise);
        if (m == 2) k<2><<<1, 512>>>(out, cyc, 200, noise);
        if (m == 3) k<3><<<1, 512>>>(out, cyc, 200, noise);
        cudaDeviceSynchronize();
      }
      cudaMemcpy(&h, cyc, 8, cudaMemcpyDeviceToHost);
      printf("noise warps %2d  %-34s %6lld cycles\n", noise, names[m], h);
    }
  }
  const char* dn[5] = {"DFMA", "MUFU.RCP64H", "SHFL.64", "MUFU.RSQ64H", "select"};
  for (int kind = 0; kind < 5; ++kind) {
    for (int rep = 0; rep < 2; ++rep) { k_dep<<<1, 32>>>(out, cyc, 1000, kind); cudaDeviceSynchronize(); }
    cudaMemcpy(&h, cyc, 8, cudaMemcpyDeviceToHost);
    printf("dependent %-12s %.1f cycles\n", dn[kind], h / 1000.0);
  }
  printf("%s\n", cudaGetErrorString(cudaGetLastError()));
  return 0;
}
