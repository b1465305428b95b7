// Shared helpers for the spectralcluster_b200 CUDA sources (sm_90a only).
#pragma once

#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <cstdio>
#include <cstdarg>
#include <cmath>

#include "../../include/spectralcluster_b200.h"

constexpr int SC_GEMM_PACE_SLOTS = 16;

struct sc_context {
  int device;
  int sm_count;
  size_t smem_optin;
  int cc_major, cc_minor;
  // device counters for the GEMM producers' pacing checkpoints: a ring of SC_GEMM_PACE_SLOTS, one
  // per launch in turn, so that GEMMs in flight on different streams (two threads running
  // predict() on one context) do not count on each other's checkpoints
  unsigned int* gemm_pace;
  int gemm_sm_limit;   // 0 = all SMs; otherwise the persistent GEMM leaves SMs to concurrent NCCL kernels
};

namespace sc {

void set_error(const char* fmt, ...);
void launched(int n = 1);   // bumps the process-wide kernel launch counter (sc_launch_count)

#define SC_CUDA(expr)                                                                   \
  do {                                                                                  \
    cudaError_t _e = (expr);                                                            \
    if (_e != cudaSuccess) {                                                            \
      sc::set_error("%s:%d: %s failed: %s", __FILE__, __LINE__, #expr,                  \
                    cudaGetErrorString(_e));                                            \
      return 1;                                                                         \
    }                                                                                   \
  } while (0)

#define SC_REQUIRE(cond, ...)                                                           \
  do {                                                                                  \
    if (!(cond)) {                                                                      \
      sc::set_error(__VA_ARGS__);                                                       \
      return 2;                                                                         \
    }                                                                                   \
  } while (0)

#define SC_LAUNCH_CHECK() SC_CUDA(cudaGetLastError())

inline cudaStream_t as_stream(void* s) { return reinterpret_cast<cudaStream_t>(s); }

inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }
// fp32 matrix usable with 128-bit accesses: 16-byte aligned base, leading dimension % 4 == 0
inline bool vec_ok_f32(const void* p, int64_t ld) { return aligned16(p) && (ld % 4) == 0; }
// fp16 plane written with 128-bit stores / read by TMA: 16-byte aligned base, ld % 8 == 0
inline bool vec_ok_f16(const void* p, int64_t ld) { return aligned16(p) && (ld % 8) == 0; }

// RAII stream-ordered scratch.
struct Scratch {
  void* p = nullptr;
  cudaStream_t st = nullptr;
  cudaError_t alloc(size_t bytes, cudaStream_t s) {
    st = s;
    if (bytes == 0) bytes = 16;
    return cudaMallocAsync(&p, bytes, s);
  }
  ~Scratch() {
    if (p) cudaFreeAsync(p, st);
  }
  template <typename T>
  T* as() { return reinterpret_cast<T*>(p); }
};

__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}
__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ double warp_maxd(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmax(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// Block-wide reductions; `red` is shared scratch of at least 32 elements.  All threads get the
// result.  blockDim.x must be a multiple of 32.
__device__ __forceinline__ float block_max(float v, float* red) {
  v = warp_max(v);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  __syncthreads();
  if (lane == 0) red[wid] = v;
  __syncthreads();
  float r = (lane < nw) ? red[lane] : -INFINITY;
  r = warp_max(r);
  return r;
}
__device__ __forceinline__ double block_sum(double v, double* red) {
  v = warp_sum(v);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  __syncthreads();
  if (lane == 0) red[wid] = v;
  __syncthreads();
  double r = (lane < nw) ? red[lane] : 0.0;
  r = warp_sum(r);
  return r;
}
__device__ __forceinline__ double block_maxd(double v, double* red) {
  v = warp_maxd(v);
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = blockDim.x >> 5;
  __syncthreads();
  if (lane == 0) red[wid] = v;
  __syncthreads();
  double r = (lane < nw) ? red[lane] : -INFINITY;
  r = warp_maxd(r);
  return r;
}

// atomic max for non-negative floats (bit pattern order == value order); NaN is not ordered.
__device__ __forceinline__ void atomic_max_nonneg(float* addr, float v) {
  atomicMax(reinterpret_cast<int*>(addr), __float_as_int(v));
}

// value = hi + lo, both fp16 (lo absorbs the rounding error of hi).
__device__ __forceinline__ void split_half(float v, __half& hi, __half& lo) {
  hi = __float2half_rn(v);
  lo = __float2half_rn(v - __half2float(hi));
}

// streaming (read-once) 128-bit load that does not pollute L1
__device__ __forceinline__ float4 ld_stream4(const float* p) {
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0,%1,%2,%3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w)
               : "l"(p));
  return r;
}

__device__ __forceinline__ float ld_stream1(const float* p) {
  float r;
  asm volatile("ld.global.nc.L1::no_allocate.f32 %0, [%1];" : "=f"(r) : "l"(p));
  return r;
}

// squared distance in sklearn's expanded form (_euclidean_distances): |c|^2 - 2 x.c + |x|^2, >= 0
__device__ __forceinline__ double sqdist_expanded(const double* __restrict__ x, int64_t i,
                                                  int64_t kd, const double* __restrict__ c,
                                                  double csq, double xsq_i) {
  double dot = 0.0;
  for (int64_t f = 0; f < kd; ++f) dot = fma(x[i * kd + f], c[f], dot);
  const double v = csq - 2.0 * dot + xsq_i;
  return v > 0.0 ? v : 0.0;
}

// C[8x8] += A[8x4] B[4x8] on the fp64 tensor cores (mma.sync m8n8k4; SASS DMMA).  Lane l holds
// A[l/4][l%4], B[l%4][l/4] (B column-major) and C[l/4][2(l%4)], C[l/4][2(l%4)+1] in (c0, c1).
__device__ __forceinline__ void dmma_m8n8k4(double& c0, double& c1, double a, double b) {
  asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};"
               : "+d"(c0), "+d"(c1)
               : "d"(a), "d"(b));
}

}  // namespace sc
