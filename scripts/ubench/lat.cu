// Micro-benchmarks that size the design: dependent-issue latency of FP64 ops (sm_90a),
// FP64 throughput per SM, RED.F64 throughput.  Build: nvcc -gencode arch=compute_90a,code=sm_90a -O3 lat.cu -o lat
#include <cstdio>
#include <cuda_runtime.h>

__global__ void k_lat(double* out, long long* cyc, double a, double b) {
  double x = a;
  long long t0 = clock64();
#pragma unroll 1
  for (int i = 0; i < 256; ++i) {
    x = fma(x, b, a); x = fma(x, b, a); x = fma(x, b, a); x = fma(x, b, a);
    x = fma(x, b, a); x = fma(x, b, a); x = fma(x, b, a); x = fma(x, b, a);
  }
  long long t1 = clock64();
  double y = a;
#pragma unroll 1
  for (int i = 0; i < 256; ++i) {
    y = y + b; y = y + b; y = y + b; y = y + b; y = y + b; y = y + b; y = y + b; y = y + b;
  }
  long long t2 = clock64();
  float f = (float)a;
#pragma unroll 1
  for (int i = 0; i < 256; ++i) {
    f = fmaf(f, (float)b, 1.f); f = fmaf(f, (float)b, 1.f); f = fmaf(f, (float)b, 1.f); f = fmaf(f, (float)b, 1.f);
    f = fmaf(f, (float)b, 1.f); f = fmaf(f, (float)b, 1.f); f = fmaf(f, (float)b, 1.f); f = fmaf(f, (float)b, 1.f);
  }
  long long t3 = clock64();
  double z = a + 2.;
#pragma unroll 1
  for (int i = 0; i < 64; ++i) { z = rsqrt(z) + 1.5; z = rsqrt(z) + 1.5; z = rsqrt(z) + 1.5; z = rsqrt(z) + 1.5; }
  long long t4 = clock64();
  double w = a + 2.;
#pragma unroll 1
  for (int i = 0; i < 64; ++i) {
    double r;
    asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(w)); w = r + 1.5;
    asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(w)); w = r + 1.5;
    asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(w)); w = r + 1.5;
    asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(w)); w = r + 1.5;
  }
  long long t5 = clock64();
  double s = a;
#pragma unroll 1
  for (int i = 0; i < 256; ++i) { s = __shfl_xor_sync(0xffffffffu, s, 1) + 0.; s = __shfl_xor_sync(0xffffffffu, s, 2) + 0.; }
  long long t6 = clock64();
  if (threadIdx.x == 0) {
    cyc[0] = (t1 - t0); cyc[1] = (t2 - t1); cyc[2] = (t3 - t2); cyc[3] = (t4 - t3); cyc[4] = (t5 - t4); cyc[5] = t6 - t5;
  }
  out[threadIdx.x] = x + y + f + z + w + s;
}

// throughput: many independent FMAs per thread, full SM
__global__ void k_tput(double* out, double a, double b, int iters) {
  double x0 = a, x1 = a + 1, x2 = a + 2, x3 = a + 3, x4 = a + 4, x5 = a + 5, x6 = a + 6, x7 = a + 7;
  for (int i = 0; i < iters; ++i) {
    x0 = fma(x0, b, a); x1 = fma(x1, b, a); x2 = fma(x2, b, a); x3 = fma(x3, b, a);
    x4 = fma(x4, b, a); x5 = fma(x5, b, a); x6 = fma(x6, b, a); x7 = fma(x7, b, a);
  }
  out[blockIdx.x * blockDim.x + threadIdx.x] = x0 + x1 + x2 + x3 + x4 + x5 + x6 + x7;
}

__global__ void k_red(double* dst, int n, int iters, int stride) {
  const int t = blockIdx.x * blockDim.x + threadIdx.x;
  for (int i = 0; i < iters; ++i) atomicAdd(dst + ((size_t)(t * stride + i * 977) % n), 1.0);
}

int main() {
  double* out; long long* cyc;
  cudaMalloc(&out, 1 << 24); cudaMalloc(&cyc, 64);
  for (int rep = 0; rep < 2; ++rep) k_lat<<<1, 32>>>(out, cyc, 1.0000001, 0.9999999);
  long long h[6]; cudaMemcpy(h, cyc, sizeof h, cudaMemcpyDeviceToHost);
  printf("dependent latency (cycles): DFMA %.1f  DADD %.1f  FFMA %.1f  rsqrt(double)+add %.1f  rsqrt.approx.f64+add %.1f  shfl64+add %.1f\n",
         h[0] / 2048.0, h[1] / 2048.0, h[2] / 2048.0, h[3] / 256.0, h[4] / 256.0, h[5] / 512.0);
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  const int iters = 4096;
  int sms = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  for (int warps = 4; warps <= 32; warps *= 2) {
    k_tput<<<sms, warps * 32>>>(out, 1.0000001, 0.9999999, iters);
    cudaEventRecord(e0); k_tput<<<sms, warps * 32>>>(out, 1.0000001, 0.9999999, iters); cudaEventRecord(e1);
    cudaEventSynchronize(e1); float ms; cudaEventElapsedTime(&ms, e0, e1);
    printf("FP64 FMA throughput, %d CTAs x %2d warps, 8 indep chains: %.2f TFLOP/s\n", sms, warps, 2.0 * 8 * iters * (double)sms * warps * 32 / (ms * 1e-3) / 1e12);
  }
  for (int stride = 1; stride <= 64; stride *= 8) {
    const int n = 1 << 21;
    k_red<<<sms * 8, 256>>>(out, n, 64, stride);
    cudaEventRecord(e0); k_red<<<sms * 8, 256>>>(out, n, 64, stride); cudaEventRecord(e1);
    cudaEventSynchronize(e1); float ms; cudaEventElapsedTime(&ms, e0, e1);
    printf("RED.F64 lane stride %2d doubles over 16 MB: %.1f G atomics/s\n", stride, (double)sms * 8 * 256 * 64 / (ms * 1e-3) / 1e9);
  }
  printf("%s\n", cudaGetErrorString(cudaDeviceSynchronize()));
  return 0;
}
