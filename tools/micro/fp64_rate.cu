// Micro-benchmark: fp64 FMA throughput of sm_90a through the CUDA cores (DFMA) and through the
// tensor cores (mma.sync.m8n8k4.f64 -> DMMA): the comparison behind building the Lanczos block
// product (eigh_lanczos.cu, k_symm_dmma) on DMMA.
//   nvcc -gencode arch=compute_90a,code=sm_90a -O3 -o fp64_rate tools/micro/fp64_rate.cu && ./fp64_rate
#include <cstdio>
#include <cuda_runtime.h>

constexpr int ITERS = 4096;

__global__ void k_dfma(double* out, double a, double b) {
  double acc[16];
#pragma unroll
  for (int i = 0; i < 16; ++i) acc[i] = threadIdx.x * 1e-3 + i;
  for (int it = 0; it < ITERS; ++it) {
#pragma unroll
    for (int i = 0; i < 16; ++i) acc[i] = fma(acc[i], a, b);
  }
  double s = 0;
#pragma unroll
  for (int i = 0; i < 16; ++i) s += acc[i];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

__global__ void k_dmma(double* out, double a, double b) {
  double c[8][2];
#pragma unroll
  for (int i = 0; i < 8; ++i) c[i][0] = c[i][1] = threadIdx.x * 1e-3 + i;
  for (int it = 0; it < ITERS; ++it) {
#pragma unroll
    for (int i = 0; i < 8; ++i)
      asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};"
                   : "+d"(c[i][0]), "+d"(c[i][1]) : "d"(a), "d"(b));
  }
  double s = 0;
#pragma unroll
  for (int i = 0; i < 8; ++i) s += c[i][0] + c[i][1];
  out[blockIdx.x * blockDim.x + threadIdx.x] = s;
}

int main() {
  int sms = 0;
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, 0);
  double* out;
  const int threads = 256, blocks = sms * 8;
  cudaMalloc(&out, sizeof(double) * threads * blocks);
  cudaEvent_t e0, e1;
  cudaEventCreate(&e0); cudaEventCreate(&e1);
  for (int rep = 0; rep < 2; ++rep) {
    float ms;
    cudaEventRecord(e0);
    k_dfma<<<blocks, threads>>>(out, 0.999999, 1e-9);
    cudaEventRecord(e1); cudaEventSynchronize(e1); cudaEventElapsedTime(&ms, e0, e1);
    const double fma_dfma = (double)blocks * threads * ITERS * 16;
    printf("DFMA: %.3f ms  %.2f TFLOP/s (2 flop per FMA)\n", ms, 2 * fma_dfma / ms / 1e9);
    cudaEventRecord(e0);
    k_dmma<<<blocks, threads>>>(out, 0.999999, 1e-9);
    cudaEventRecord(e1); cudaEventSynchronize(e1); cudaEventElapsedTime(&ms, e0, e1);
    const double fma_dmma = (double)blocks * (threads / 32) * ITERS * 8 * 256;
    printf("DMMA m8n8k4: %.3f ms  %.2f TFLOP/s\n", ms, 2 * fma_dmma / ms / 1e9);
  }
  printf("%s\n", cudaGetErrorString(cudaGetLastError()));
  return 0;
}
