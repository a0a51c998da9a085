// Microbenchmark: FP64 DFMA vs DMMA (mma.sync.m8n8k4.f64) throughput on sm_90a.
// Decides whether the Riccati GEMMs use tensor-pipe DMMA or CUDA-core DFMA.
#include <cstdio>
#include <cuda_runtime.h>

__global__ void dfma_kernel(double* out, int iters, double a, double b) {
  double x0 = threadIdx.x, x1 = x0 + 1, x2 = x0 + 2, x3 = x0 + 3, x4 = x0 + 4, x5 = x0 + 5, x6 = x0 + 6, x7 = x0 + 7;
  for (int i = 0; i < iters; ++i) {
    x0 = fma(x0, a, b); x1 = fma(x1, a, b); x2 = fma(x2, a, b); x3 = fma(x3, a, b);
    x4 = fma(x4, a, b); x5 = fma(x5, a, b); x6 = fma(x6, a, b); x7 = fma(x7, a, b);
  }
  out[blockIdx.x * blockDim.x + threadIdx.x] = x0 + x1 + x2 + x3 + x4 + x5 + x6 + x7;
}

__device__ __forceinline__ void dmma(double& c0, double& c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};\n"
               : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}

__global__ void dmma_kernel(double* out, int iters, double a, double b) {
  double c[8][2];
  for (int j = 0; j < 8; ++j) { c[j][0] = threadIdx.x + j; c[j][1] = j; }
  for (int i = 0; i < iters; ++i) {
#pragma unroll
    for (int j = 0; j < 8; ++j) dmma(c[j][0], c[j][1], a, b);
  }
  double s = 0;
  for (int j = 0; j < 8; ++j) s += c[j][0] + c[j][1];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

// smem-fed DFMA: 3x3 register tile, operands from shared (models the GEMM inner loop)
__global__ void dfma_smem_kernel(double* out, int iters) {
  __shared__ double A[36 * 36], B[36 * 36];
  for (int i = threadIdx.x; i < 36 * 36; i += blockDim.x) { A[i] = 1e-3 * i; B[i] = 1e-3 * (i % 7); }
  __syncthreads();
  int t = threadIdx.x % 144; int ti = (t % 12) * 3, tj = (t / 12) * 3;
  double c[3][3] = {};
  for (int it = 0; it < iters; ++it) {
#pragma unroll 4
    for (int k = 0; k < 36; ++k) {
      double a0 = A[k * 36 + ti], a1 = A[k * 36 + ti + 1], a2 = A[k * 36 + ti + 2];
      double b0 = B[k * 36 + tj], b1 = B[k * 36 + tj + 1], b2 = B[k * 36 + tj + 2];
      c[0][0] = fma(a0, b0, c[0][0]); c[0][1] = fma(a0, b1, c[0][1]); c[0][2] = fma(a0, b2, c[0][2]);
      c[1][0] = fma(a1, b0, c[1][0]); c[1][1] = fma(a1, b1, c[1][1]); c[1][2] = fma(a1, b2, c[1][2]);
      c[2][0] = fma(a2, b0, c[2][0]); c[2][1] = fma(a2, b1, c[2][1]); c[2][2] = fma(a2, b2, c[2][2]);
    }
  }
  double s = 0; for (int i = 0; i < 3; ++i) for (int j = 0; j < 3; ++j) s += c[i][j];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

int main() {
  cudaDeviceProp p; cudaGetDeviceProperties(&p, 0);
  printf("device %s sms=%d clock=%d kHz\n", p.name, p.multiProcessorCount, p.clockRate);
  double* out; cudaMalloc(&out, sizeof(double) * 132 * 64 * 1024);
  cudaEvent_t e0, e1; cudaEventCreate(&e0); cudaEventCreate(&e1);
  float ms;
  for (int threads : {128, 256, 512, 1024}) {
    int blocks = 132 * (2048 / threads);
    int iters = 20000;
    dfma_kernel<<<blocks, threads>>>(out, 100, 1.0000001, 1e-9);
    cudaDeviceSynchronize();
    cudaEventRecord(e0); dfma_kernel<<<blocks, threads>>>(out, iters, 1.0000001, 1e-9); cudaEventRecord(e1);
    cudaEventSynchronize(e1); cudaEventElapsedTime(&ms, e0, e1);
    double fl = 2.0 * 8 * iters * (double)blocks * threads;
    printf("DFMA  threads=%4d blocks=%5d: %.3f ms  %.2f TFLOP/s\n", threads, blocks, ms, fl / ms * 1e-9);
    dmma_kernel<<<blocks, threads>>>(out, 100, 1.0000001, 1e-9);
    cudaDeviceSynchronize();
    int it2 = 5000;
    cudaEventRecord(e0); dmma_kernel<<<blocks, threads>>>(out, it2, 1.0000001, 1e-9); cudaEventRecord(e1);
    cudaEventSynchronize(e1); cudaEventElapsedTime(&ms, e0, e1);
    double fl2 = 2.0 * 256 * 8 * it2 * (double)blocks * (threads / 32);
    printf("DMMA  threads=%4d blocks=%5d: %.3f ms  %.2f TFLOP/s\n", threads, blocks, ms, fl2 / ms * 1e-9);
  }
  for (int threads : {160, 288}) {
    for (int bps : {1, 2, 4, 6}) {
      int blocks = 132 * bps; int iters = 2000;
      dfma_smem_kernel<<<blocks, threads>>>(out, 10);
      cudaDeviceSynchronize();
      cudaEventRecord(e0); dfma_smem_kernel<<<blocks, threads>>>(out, iters); cudaEventRecord(e1);
      cudaEventSynchronize(e1); cudaEventElapsedTime(&ms, e0, e1);
      double fl = 2.0 * 9 * 36 * iters * (double)blocks * threads;
      printf("DFMA-smem3x3 threads=%d blocks/SM=%d: %.3f ms  %.2f TFLOP/s\n", threads, bps, ms, fl / ms * 1e-9);
    }
  }
  printf("err=%s\n", cudaGetErrorString(cudaGetLastError()));
  return 0;
}
