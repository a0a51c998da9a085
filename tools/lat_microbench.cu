// Single-warp dependent-chain latencies on sm_90a (cycles per op): DFMA, DMUL->DFMA, SHFL(64-bit)->DFMA, MUFU.RCP64H+2 Newton,
// DMMA m8n8k4 accumulate chain, 5 independent DMMA accumulators, LDS->DFMA, and issue throughput of independent SHFL / DFMA.
#include <cstdio>
#include <cuda_runtime.h>
__device__ __forceinline__ void dmma(double& c0, double& c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}
__global__ void k(double* out, long long* cyc, double seed) {
  __shared__ double sm[1024];
  const int lane = threadIdx.x & 31;
  for (int i = threadIdx.x; i < 1024; i += blockDim.x) sm[i] = seed + i * 1e-9;
  __syncthreads();
  double x = seed, y = seed * 0.5, acc = 0;
  long long t0, t1;
  const int N = 256;
  // 1. dependent DFMA
  t0 = clock64();
#pragma unroll 16
  for (int i = 0; i < N; ++i) x = fma(x, y, 1e-3);
  t1 = clock64(); if (lane == 0) cyc[0] = (t1 - t0); acc += x;
  // 2. dependent SHFL(double) + DFMA
  t0 = clock64();
#pragma unroll 16
  for (int i = 0; i < N; ++i) { double v = __shfl_sync(0xffffffffu, x, (i + 1) & 31); x = fma(v, y, 1e-3); }
  t1 = clock64(); if (lane == 0) cyc[1] = (t1 - t0); acc += x;
  // 3. rcp approx + 2 newton (dependent chain through d)
  x = 1.5;
  t0 = clock64();
#pragma unroll 8
  for (int i = 0; i < N; ++i) { double r; asm volatile("rcp.approx.ftz.f64 %0, %1;" : "=d"(r) : "d"(x)); r = fma(r, fma(-x, r, 1.0), r); r = fma(r, fma(-x, r, 1.0), r); x = r + 1.0; }
  t1 = clock64(); if (lane == 0) cyc[2] = (t1 - t0); acc += x;
  // 4. DMMA accumulate chain (1 accumulator)
  double c0 = 0, c1 = 0, a = seed, b = seed * 0.25;
  t0 = clock64();
#pragma unroll 16
  for (int i = 0; i < N; ++i) dmma(c0, c1, a, b);
  t1 = clock64(); if (lane == 0) cyc[3] = (t1 - t0); acc += c0 + c1;
  // 5. DMMA 5 independent accumulators (5*N dmmas)
  double d0[5] = {0, 0, 0, 0, 0}, d1[5] = {0, 0, 0, 0, 0};
  t0 = clock64();
#pragma unroll 8
  for (int i = 0; i < N; ++i) {
#pragma unroll
    for (int q = 0; q < 5; ++q) dmma(d0[q], d1[q], a, b);
  }
  t1 = clock64(); if (lane == 0) cyc[4] = (t1 - t0);
  for (int q = 0; q < 5; ++q) acc += d0[q] + d1[q];
  // 6. LDS -> DFMA dependent (address depends on result)
  int idx = lane;
  x = seed;
  t0 = clock64();
#pragma unroll 16
  for (int i = 0; i < N; ++i) { double v = sm[idx]; x = fma(v, y, x); idx = (idx + 33 + (int)(x > 1e300)) & 1023; }
  t1 = clock64(); if (lane == 0) cyc[5] = (t1 - t0); acc += x;
  // 7. independent SHFLs (throughput): 8 independent streams
  double s[8]; for (int q = 0; q < 8; ++q) s[q] = seed + q;
  t0 = clock64();
#pragma unroll 4
  for (int i = 0; i < N; ++i) {
#pragma unroll
    for (int q = 0; q < 8; ++q) s[q] = __shfl_sync(0xffffffffu, s[q], (lane + 1) & 31);
  }
  t1 = clock64(); if (lane == 0) cyc[6] = (t1 - t0);
  for (int q = 0; q < 8; ++q) acc += s[q];
  // 8. independent DFMA throughput: 8 streams
  for (int q = 0; q < 8; ++q) s[q] = seed + q;
  t0 = clock64();
#pragma unroll 4
  for (int i = 0; i < N; ++i) {
#pragma unroll
    for (int q = 0; q < 8; ++q) s[q] = fma(s[q], y, 1e-3);
  }
  t1 = clock64(); if (lane == 0) cyc[7] = (t1 - t0);
  for (int q = 0; q < 8; ++q) acc += s[q];
  // 9. DMUL dependent
  x = 1.0000001;
  t0 = clock64();
#pragma unroll 16
  for (int i = 0; i < N; ++i) x = x * y;
  t1 = clock64(); if (lane == 0) cyc[8] = (t1 - t0); acc += x;
  // 10. LDS broadcast + DFMA dependent through value only (fixed address pattern, pipelined loads)
  x = seed;
  t0 = clock64();
#pragma unroll 16
  for (int i = 0; i < N; ++i) { double v = sm[(i * 7) & 1023]; x = fma(v, y, x); }
  t1 = clock64(); if (lane == 0) cyc[9] = (t1 - t0); acc += x;
  out[threadIdx.x] = acc;
}
int main() {
  double* out; long long* cyc;
  cudaMalloc(&out, 1024 * 8); cudaMalloc(&cyc, 16 * 8);
  const char* names[10] = {"dependent DFMA", "dependent SHFL64+DFMA", "rcp.approx+2 Newton (+DADD)", "DMMA chain (1 acc)", "DMMA x5 indep acc (per k-step of 5)",
                           "dependent LDS(addr)+DFMA", "8 indep SHFL64 (per 8)", "8 indep DFMA (per 8)", "dependent DMUL", "LDS(indep)+DFMA chain"};
  for (int warps = 1; warps <= 4; warps *= 4) {
    k<<<1, 32 * warps>>>(out, cyc, 0.3); cudaDeviceSynchronize();
    k<<<1, 32 * warps>>>(out, cyc, 0.3); cudaDeviceSynchronize();
    long long h[16]; cudaMemcpy(h, cyc, 16 * 8, cudaMemcpyDeviceToHost);
    printf("== %d warp(s) in the CTA (cycles per iteration, N=256)\n", warps);
    for (int i = 0; i < 10; ++i) printf("%-40s %8.1f\n", names[i], h[i] / 256.0);
  }
  printf("%s\n", cudaGetErrorString(cudaGetLastError()));
  return 0;
}
