// SIMT validation GEMM: C = A B^T with fp32 operands and fp64 accumulation (every fp32 x fp32
// product is exact in fp64).  This is NOT the product path for large N -- that is the wgmma
// kernel in gemm_wgmma.cu -- it is the on-device reference the tensor-core kernel is tested
// against, and the engine used for matrices too small to fill a 128x128 tensor-core tile.
//
//   utils.py:35-39        affinity = (Xn Xn^T + 1) / 2      -> EPI_AFFINITY
//   refinement.py:232-234 Diffuse: Y Y^T                    -> EPI_PLAIN
#include "common.cuh"

namespace sc {

constexpr int SB = 64;   // block tile
constexpr int SK = 16;   // k step

enum { EPI_PLAIN = 0, EPI_AFFINITY = 1 };

template <int EPI>
__global__ void __launch_bounds__(256)
k_gemm_nt_simt(const float* __restrict__ A, int64_t lda, const float* __restrict__ B,
               int64_t ldb, int64_t M, int64_t N, int64_t K, float* __restrict__ C, int64_t ldc,
               float* __restrict__ rowmax_offdiag) {
  __shared__ float As[SK][SB + 4];
  __shared__ float Bs[SK][SB + 4];
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  const int64_t m0 = (int64_t)blockIdx.y * SB, n0 = (int64_t)blockIdx.x * SB;
  const int lr = threadIdx.x >> 2;          // 0..63 : tile row loaded by this thread
  const int lk = (threadIdx.x & 3) * 4;     // 0,4,8,12
  double acc[4][4];
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) acc[i][j] = 0.0;

  for (int64_t k0 = 0; k0 < K; k0 += SK) {
    float av[4], bv[4];
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const int64_t k = k0 + lk + t;
      av[t] = (m0 + lr < M && k < K) ? A[(m0 + lr) * lda + k] : 0.0f;
      bv[t] = (n0 + lr < N && k < K) ? B[(n0 + lr) * ldb + k] : 0.0f;
    }
    __syncthreads();
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      As[lk + t][lr] = av[t];
      Bs[lk + t][lr] = bv[t];
    }
    __syncthreads();
#pragma unroll
    for (int k = 0; k < SK; ++k) {
      double a[4], b[4];
#pragma unroll
      for (int i = 0; i < 4; ++i) a[i] = (double)As[k][ty * 4 + i];
#pragma unroll
      for (int j = 0; j < 4; ++j) b[j] = (double)Bs[k][tx * 4 + j];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = fma(a[i], b[j], acc[i][j]);
    }
  }
#pragma unroll
  for (int i = 0; i < 4; ++i) {
    const int64_t r = m0 + ty * 4 + i;
    if (r >= M) continue;
    float rmax = 0.0f;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int64_t c = n0 + tx * 4 + j;
      if (c >= N) continue;
      float v;
      if (EPI == EPI_AFFINITY) v = (float)((acc[i][j] + 1.0) / 2.0);   // utils.py:39
      else v = (float)acc[i][j];
      C[r * ldc + c] = v;
      if (EPI == EPI_AFFINITY && r != c) rmax = fmaxf(rmax, v);
    }
    if (EPI == EPI_AFFINITY && rowmax_offdiag) atomic_max_nonneg(rowmax_offdiag + r, rmax);
  }
}

int gemm_nt_simt(int epi, const float* A, int64_t lda, const float* B, int64_t ldb, int64_t M,
                 int64_t N, int64_t K, float* C, int64_t ldc, float* rowmax_offdiag,
                 cudaStream_t st) {
  const dim3 grid((unsigned)((N + SB - 1) / SB), (unsigned)((M + SB - 1) / SB));
  SC_REQUIRE(grid.y <= 65535u, "gemm_nt_simt: M too large for the SIMT validation engine");
  if (epi == EPI_AFFINITY)
    k_gemm_nt_simt<EPI_AFFINITY><<<grid, 256, 0, st>>>(A, lda, B, ldb, M, N, K, C, ldc,
                                                       rowmax_offdiag);
  else
    k_gemm_nt_simt<EPI_PLAIN><<<grid, 256, 0, st>>>(A, lda, B, ldb, M, N, K, C, ldc, nullptr);
  sc::launched();
  SC_LAUNCH_CHECK();
  return 0;
}

}  // namespace sc
