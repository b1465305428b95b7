// Row-wise / element-wise kernels of the refinement sequence and the Laplacian.
// All of these are HBM-bound: one CTA per matrix row, 128-bit coalesced loads,
// warp-shuffle reductions, second touch of a row served from L2.
//
// Reference operators replaced (file:line under /root/reference/spectralcluster):
//   utils.py:32-33        row L2 normalisation          -> k_normalize_rows (fp16/bf16/fp32/fp64 rows)
//   refinement.py:145-151 CropDiagonal                  -> k_crop_diagonal
//   refinement.py:182-210 RowWiseThreshold              -> k_row_threshold (+ radix select)
//   refinement.py:219-226 Symmetrize                    -> k_symmetrize
//   refinement.py:240-245 RowWiseNormalize              -> k_row_normalize
//   laplacian.py:24-60    compute_laplacian             -> k_laplacian
#include "common.cuh"

#include <cuda_bf16.h>

namespace sc {

// ------------------------------------------------------------------ normalise rows
// Every input dtype widens exactly to fp64, so an fp16 row gives what its fp64 upcast gives and a
// bf16 row what its fp32 upcast gives.
__device__ __forceinline__ double to_f64(float v) { return (double)v; }
__device__ __forceinline__ double to_f64(double v) { return v; }
__device__ __forceinline__ double to_f64(__half v) { return (double)__half2float(v); }
__device__ __forceinline__ double to_f64(__nv_bfloat16 v) { return (double)__bfloat162float(v); }

template <typename T>
__global__ void k_normalize_rows(const T* __restrict__ x, int64_t n, int64_t d, int64_t ldx,
                                 float* __restrict__ xn, int64_t ldxn, __half* __restrict__ hi,
                                 __half* __restrict__ lo, int64_t ldh) {
  const int64_t row = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (row >= n) return;
  const T* r = x + row * ldx;
  double ss = 0.0;
  for (int64_t j = lane; j < d; j += 32) {
    const double v = to_f64(r[j]);
    ss += v * v;
  }
  ss = warp_sum(ss);
  const double nrm = sqrt(ss);
  for (int64_t j = lane; j < d; j += 32) {
    const float f = (float)(to_f64(r[j]) / nrm);
    if (xn) xn[row * ldxn + j] = f;
    if (hi) {
      __half h, l;
      split_half(f, h, l);
      hi[row * ldh + j] = h;
      lo[row * ldh + j] = l;
    }
  }
}

// ------------------------------------------------------------------ crop diagonal
// diag_out (optional) receives the new diagonal; out (optional) the full matrix.  Row blockIdx.x
// of `a` is row row0 + blockIdx.x of the matrix (a row panel; row0 = 0 for the whole matrix).
__global__ void k_crop_diagonal(const float* a, int64_t n, int64_t lda, float* out, int64_t ldo,
                                float* __restrict__ diag_out, int64_t row0) {
  __shared__ float red[32];
  const int64_t i = row0 + blockIdx.x;
  const float* r = a + (int64_t)blockIdx.x * lda;
  float m = 0.0f;  // the zeroed diagonal takes part in the max (refinement.py:148-149)
  // 128-bit loads when the row is 16-byte aligned (every matrix the Python host allocates)
  const bool vec = ((lda & 3) == 0) && ((reinterpret_cast<uintptr_t>(a) & 15) == 0);
  const int64_t n4 = vec ? (n & ~(int64_t)3) : 0;
  for (int64_t j = (int64_t)threadIdx.x * 4; j < n4; j += (int64_t)blockDim.x * 4) {
    const float4 q = *reinterpret_cast<const float4*>(r + j);
    if (i < j || i > j + 3) {
      m = fmaxf(m, fmaxf(fmaxf(q.x, q.y), fmaxf(q.z, q.w)));
    } else {
      if (j != i) m = fmaxf(m, q.x);
      if (j + 1 != i) m = fmaxf(m, q.y);
      if (j + 2 != i) m = fmaxf(m, q.z);
      if (j + 3 != i) m = fmaxf(m, q.w);
    }
  }
  for (int64_t j = n4 + threadIdx.x; j < n; j += blockDim.x)
    if (j != i) m = fmaxf(m, r[j]);
  m = block_max(m, red);
  if (diag_out && threadIdx.x == 0) diag_out[blockIdx.x] = m;
  if (out) {
    float* o = out + (int64_t)blockIdx.x * ldo;
    if (out == a) {
      if (threadIdx.x == 0) o[i] = m;
    } else {
      const bool ovec = vec && ((ldo & 3) == 0) && ((reinterpret_cast<uintptr_t>(out) & 15) == 0);
      const int64_t o4 = ovec ? n4 : 0;
      for (int64_t j = (int64_t)threadIdx.x * 4; j < o4; j += (int64_t)blockDim.x * 4) {
        float4 q = *reinterpret_cast<const float4*>(r + j);
        if (i >= j && i <= j + 3) {
          if (j == i) q.x = m;
          else if (j + 1 == i) q.y = m;
          else if (j + 2 == i) q.z = m;
          else q.w = m;
        }
        *reinterpret_cast<float4*>(o + j) = q;
      }
      for (int64_t j = o4 + threadIdx.x; j < n; j += blockDim.x) o[j] = (j == i) ? m : r[j];
    }
  }
}

// ------------------------------------------------------------------ radix select (Percentile)
__device__ __forceinline__ uint32_t order_key(float v) {
  const uint32_t b = __float_as_uint(v);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float key_value(uint32_t k) {
  const uint32_t b = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
  return __uint_as_float(b);
}

// k-th smallest (0-based) of row r (diagonal read as 0 if zero_diag).  All threads return it.
__device__ float row_select(const float* r, int64_t n, int64_t diag, bool zero_diag, int64_t k,
                            unsigned int* hist /*256*/, unsigned int* bcast /*2*/) {
  uint32_t prefix = 0, mask = 0;
  int64_t want = k;
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int t = threadIdx.x; t < 256; t += blockDim.x) hist[t] = 0;
    __syncthreads();
    for (int64_t j = threadIdx.x; j < n; j += blockDim.x) {
      const float v = (zero_diag && j == diag) ? 0.0f : r[j];
      const uint32_t key = order_key(v);
      if ((key & mask) == prefix) atomicAdd(&hist[(key >> shift) & 255u], 1u);
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      int64_t cum = 0;
      int b = 0;
      for (; b < 256; ++b) {
        if (cum + (int64_t)hist[b] > want) break;
        cum += hist[b];
      }
      if (b > 255) b = 255;
      bcast[0] = (unsigned int)b;
      bcast[1] = (unsigned int)cum;
    }
    __syncthreads();
    prefix |= (bcast[0] << shift);
    mask |= (255u << shift);
    want -= (int64_t)bcast[1];
    __syncthreads();
  }
  return key_value(prefix);
}

// ------------------------------------------------------------------ row-wise threshold
__global__ void k_row_threshold(const float* __restrict__ a, int64_t n, int64_t lda, int type,
                                float p, double q, float mult, int binarize, int preserve_diag,
                                float* __restrict__ out, int64_t ldo) {
  __shared__ float red[32];
  __shared__ unsigned int hist[256];
  __shared__ unsigned int bcast[2];
  const int64_t i = blockIdx.x;
  const float* r = a + i * lda;
  float* o = out + i * ldo;
  double cut;
  if (type == SC_THRESHOLD_ROWMAX) {
    float m = -INFINITY;
    for (int64_t j = threadIdx.x; j < n; j += blockDim.x) {
      const float v = (preserve_diag && j == i) ? 0.0f : r[j];
      m = fmaxf(m, v);
    }
    m = block_max(m, red);
    cut = (double)(m * p);                       // refinement.py:189-191 evaluated in fp32
  } else {
    // np.percentile(row, 100 p), default 'linear' method (refinement.py:194-195)
    const double h = q * (double)(n - 1);
    int64_t k0 = (int64_t)floor(h);
    if (k0 < 0) k0 = 0;
    if (k0 > n - 1) k0 = n - 1;
    const int64_t k1 = (k0 + 1 < n) ? k0 + 1 : k0;
    const double t = h - (double)k0;
    const float v0 = row_select(r, n, i, preserve_diag != 0, k0, hist, bcast);
    const float v1 = (k1 == k0) ? v0 : row_select(r, n, i, preserve_diag != 0, k1, hist, bcast);
    const double d = (double)v1 - (double)v0;
    cut = (t >= 0.5) ? (double)v1 - d * (1.0 - t) : (double)v0 + d * t;   // numpy _lerp
  }
  auto rule = [&](float x, int64_t j) -> float {
    const float v = (preserve_diag && j == i) ? 0.0f : x;
    float y;
    if ((double)v < cut) y = v * mult;
    else y = binarize ? 1.0f : v;
    if (preserve_diag && j == i) y = 1.0f;
    return y;
  };
  const bool vec = ((reinterpret_cast<uintptr_t>(r) & 15) == 0) && ((reinterpret_cast<uintptr_t>(o) & 15) == 0);
  const int64_t n4 = vec ? (n & ~(int64_t)3) : 0;
  for (int64_t j = (int64_t)threadIdx.x * 4; j < n4; j += (int64_t)blockDim.x * 4) {
    const float4 q = *reinterpret_cast<const float4*>(r + j);
    *reinterpret_cast<float4*>(o + j) =
        make_float4(rule(q.x, j), rule(q.y, j + 1), rule(q.z, j + 2), rule(q.w, j + 3));
  }
  for (int64_t j = n4 + threadIdx.x; j < n; j += blockDim.x) o[j] = rule(r[j], j);
}

// ------------------------------------------------------------------ symmetrize
__global__ void k_symmetrize(const float* __restrict__ a, int64_t n, int64_t lda, int type,
                             float* __restrict__ out, int64_t ldo) {
  __shared__ float s1[32][33];
  __shared__ float s2[32][33];
  const int64_t bi = (int64_t)blockIdx.y * 32, bj = (int64_t)blockIdx.x * 32;
  for (int r = threadIdx.y; r < 32; r += blockDim.y) {
    const int64_t i = bi + r, j = bj + threadIdx.x;
    s1[r][threadIdx.x] = (i < n && j < n) ? a[i * lda + j] : 0.0f;
    const int64_t ti = bj + r, tj = bi + threadIdx.x;   // transposed tile
    s2[r][threadIdx.x] = (ti < n && tj < n) ? a[ti * lda + tj] : 0.0f;
  }
  __syncthreads();
  for (int r = threadIdx.y; r < 32; r += blockDim.y) {
    const int64_t i = bi + r, j = bj + threadIdx.x;
    if (i < n && j < n) {
      const float x = s1[r][threadIdx.x], y = s2[threadIdx.x][r];
      out[i * ldo + j] = (type == SC_SYMMETRIZE_MAX) ? fmaxf(x, y) : 0.5f * (x + y);
    }
  }
}

// ------------------------------------------------------------------ transpose (rectangular)
__global__ void k_transpose(const float* __restrict__ src, int64_t rows, int64_t cols, int64_t lds,
                            float* __restrict__ dst, int64_t ldd) {
  __shared__ float tile[32][33];
  const int64_t r0 = (int64_t)blockIdx.y * 32, c0 = (int64_t)blockIdx.x * 32;
  for (int r = threadIdx.y; r < 32; r += blockDim.y) {
    const int64_t i = r0 + r, j = c0 + threadIdx.x;
    tile[r][threadIdx.x] = (i < rows && j < cols) ? src[i * lds + j] : 0.0f;
  }
  __syncthreads();
  for (int r = threadIdx.y; r < 32; r += blockDim.y) {
    const int64_t j = c0 + r, i = r0 + threadIdx.x;     // dst[j][i] = src[i][j]
    if (i < rows && j < cols) dst[j * ldd + i] = tile[threadIdx.x][r];
  }
}

// ------------------------------------------------------------------ split planes
__global__ void k_split_planes(const float* __restrict__ a, int64_t n, int64_t lda,
                               __half* __restrict__ hi, __half* __restrict__ lo, int64_t ldh) {
  const int64_t i = blockIdx.x;   // rows on grid.x (grid.y is limited to 65535)
  const int64_t j = ((int64_t)blockIdx.y * blockDim.x + threadIdx.x) * 4;
  if (j >= n) return;
  const float* r = a + i * lda + j;
  float v[4];
  if (j + 3 < n) {
    const float4 q = *reinterpret_cast<const float4*>(r);
    v[0] = q.x; v[1] = q.y; v[2] = q.z; v[3] = q.w;
  } else {
    for (int t = 0; t < 4; ++t) v[t] = (j + t < n) ? r[t] : 0.0f;
  }
  for (int t = 0; t < 4; ++t) {
    if (j + t < n) {
      __half h, l;
      split_half(v[t], h, l);
      hi[i * ldh + j + t] = h;
      lo[i * ldh + j + t] = l;
    }
  }
}

// ------------------------------------------------------------------ row statistics
__global__ void k_row_stats(const float* __restrict__ a, int64_t n /*columns*/, int64_t lda,
                            double* __restrict__ rowmax, double* __restrict__ rowsum) {
  __shared__ double red[32];
  const int64_t i = blockIdx.x;
  const float* r = a + i * lda;
  double m = -INFINITY, s = 0.0;
  const int64_t n4 = n & ~(int64_t)3;
  for (int64_t j = (int64_t)threadIdx.x * 4; j < n4; j += (int64_t)blockDim.x * 4) {
    const float4 q = ld_stream4(r + j);
    m = fmax(m, (double)fmaxf(fmaxf(q.x, q.y), fmaxf(q.z, q.w)));
    s += ((double)q.x + (double)q.y) + ((double)q.z + (double)q.w);
  }
  for (int64_t j = n4 + threadIdx.x; j < n; j += blockDim.x) {
    m = fmax(m, (double)r[j]);
    s += (double)r[j];
  }
  m = block_maxd(m, red);
  s = block_sum(s, red);
  if (threadIdx.x == 0) {
    if (rowmax) rowmax[i] = m;
    if (rowsum) rowsum[i] = s;
  }
}

// ------------------------------------------------------------------ bounds of the Diffuse rows
// One read of the fp16 plane of Y (non-negative, 256 threads per row, 8 columns per thread, so one
// warp covers one 256-column group per step): per row the group norms |y_i^g| (fp64 sum of squares
// rounded up, stored as fp32 rounded up), a lower bound of the diagonal |y_i|^2 of S = Y Y^T (fp64,
// every addition rounded down; fp16 squares are exact in fp64, so it is the exact diagonal unless
// the row spans more than 2^53 in magnitude) and the row sums c_i (fp64).
constexpr int BOUND_GROUP = 256;

__device__ __forceinline__ double warp_sum_rd(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = __dadd_rd(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

__global__ void __launch_bounds__(256) k_row_group_bounds(const __half* __restrict__ y, int64_t n,
                                                          int64_t ldy, float* __restrict__ norms,
                                                          int G, double* __restrict__ diag_lb,
                                                          double* __restrict__ rowsum) {
  __shared__ double red[32];
  const int64_t i = blockIdx.x;
  const __half* r = y + i * ldy;
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  double lo = 0.0, s = 0.0;
  for (int64_t c0 = 0; c0 < n; c0 += 256 * 8) {
    const int64_t j = c0 + (int64_t)threadIdx.x * 8;
    double up = 0.0;
    if (j < n) {
      const uint4 q = __ldg(reinterpret_cast<const uint4*>(r + j));
      const __half* h = reinterpret_cast<const __half*>(&q);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const double v = (j + e < n) ? (double)__half2float(h[e]) : 0.0;
        up = __fma_ru(v, v, up);
        lo = __fma_rd(v, v, lo);
        s += v;
      }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) up = __dadd_ru(up, __shfl_xor_sync(0xffffffffu, up, o));
    const int64_t g = c0 / BOUND_GROUP + w;
    if (lane == 0 && g < G) norms[i * G + g] = __double2float_ru(__dsqrt_ru(up));
  }
  lo = warp_sum_rd(lo);
  __syncthreads();
  if (lane == 0) red[w] = lo;
  __syncthreads();
  lo = (lane < 8) ? red[lane] : 0.0;
  lo = warp_sum_rd(lo);
  s = block_sum(s, red);
  if (threadIdx.x == 0) {
    diag_lb[i] = lo;
    rowsum[i] = s;
  }
}

// dst row r = src row perm[r] (fp16, whole rows of `cols` elements, cols % 8 == 0)
__global__ void k_gather_rows_f16(const __half* __restrict__ src, int64_t lds,
                                  const int* __restrict__ perm, int64_t cols,
                                  __half* __restrict__ dst, int64_t ldd) {
  const int64_t r = blockIdx.x;
  const uint4* in = reinterpret_cast<const uint4*>(src + (int64_t)perm[r] * lds);
  uint4* out = reinterpret_cast<uint4*>(dst + r * ldd);
  for (int64_t j = threadIdx.x; j < cols / 8; j += blockDim.x) out[j] = __ldg(in + j);
}

// ------------------------------------------------------------------ single-cluster statistics
// fallback_clusterer.check_single_cluster (fallback_clusterer.py:127-187) needs three reductions
// of the affinity: its minimum (AllAffinity, :143), the minimum of the first super-diagonal
// (NeighborAffinity, :148-150) and np.std over all n^2 entries (AffinityStd, :154).  One
// streaming pass, fp64 accumulation; per-row partials, then a single-block finish.  The factored
// route, which never stores the affinity, runs the same row kernel over row panels: a panel's row r
// is matrix row row_begin + r, and with `nb` each row also records a[i][i+1] for the finish.
__global__ void k_affinity_row_stats(const float* __restrict__ a, int64_t n, int64_t lda,
                                     int64_t row_begin, double* __restrict__ part /*[3][n]*/,
                                     double* __restrict__ nb /*[n] or null*/) {
  __shared__ double red[32];
  const int64_t i = row_begin + blockIdx.x;
  const float* r = a + (int64_t)blockIdx.x * lda;
  double mn = INFINITY, s = 0.0, q2 = 0.0;
  const int64_t n4 = n & ~(int64_t)3;
  for (int64_t j = (int64_t)threadIdx.x * 4; j < n4; j += (int64_t)blockDim.x * 4) {
    const float4 q = ld_stream4(r + j);
    mn = fmin(mn, (double)fminf(fminf(q.x, q.y), fminf(q.z, q.w)));
    s += ((double)q.x + (double)q.y) + ((double)q.z + (double)q.w);
    q2 += ((double)q.x * q.x + (double)q.y * q.y) + ((double)q.z * q.z + (double)q.w * q.w);
  }
  for (int64_t j = n4 + threadIdx.x; j < n; j += blockDim.x) {
    const double x = (double)r[j];
    mn = fmin(mn, x);
    s += x;
    q2 += x * x;
  }
  mn = -block_maxd(-mn, red);
  s = block_sum(s, red);
  q2 = block_sum(q2, red);
  if (threadIdx.x == 0) {
    part[i] = mn;
    part[n + i] = s;
    part[2 * n + i] = q2;
    if (nb) nb[i] = i + 1 < n ? (double)r[i + 1] : INFINITY;
  }
}

// out[0] = min, out[1] = sum, out[2] = sum of squares, out[3] = min_i a[i][i+1] (+inf if n == 1),
// the neighbours read from `a` or, with a == null, from the row kernel's part[3 n + i]
__global__ void k_affinity_stats_finish(const double* __restrict__ part, const float* __restrict__ a,
                                        int64_t n, int64_t lda, double* __restrict__ out) {
  __shared__ double red[32];
  double mn = INFINITY, s = 0.0, q2 = 0.0, nb = INFINITY;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
    mn = fmin(mn, part[i]);
    s += part[n + i];
    q2 += part[2 * n + i];
    if (i + 1 < n) nb = fmin(nb, a ? (double)a[i * lda + i + 1] : part[3 * n + i]);
  }
  mn = -block_maxd(-mn, red);
  s = block_sum(s, red);
  q2 = block_sum(q2, red);
  nb = -block_maxd(-nb, red);
  if (threadIdx.x == 0) {
    out[0] = mn;
    out[1] = s;
    out[2] = q2;
    out[3] = nb;
  }
}

// ------------------------------------------------------------------ constraint operators
// constraint.py:95-164.  AffinityIntegration is one element-wise pass; ConstraintPropagation is a
// handful of dense products (host-orchestrated, on the GEMM engines) around these element-wise
// helpers.
//   mode 0: out = np.maximum(a, q)                AffinityIntegration(Max)      :112-113
//   mode 1: out = (a + q) / 2                     AffinityIntegration(Average)  :114-115
//   mode 2: out = q > 0 ? 1 - (1 - q)(1 - a) : (1 + q) a   propagation, eq. (4) :156-163
__global__ void k_constraint_combine(const float* __restrict__ a, int64_t lda,
                                     const float* __restrict__ q, int64_t ldq, int64_t n, int mode,
                                     float* __restrict__ out, int64_t ldo) {
  const int64_t i = blockIdx.y;
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const float x = a[i * lda + j], c = q[i * ldq + j];
  float r;
  if (mode == 0) r = (x >= c || x != x) ? x : c;   // np.maximum: a NaN operand propagates
  else if (mode == 1) r = 0.5f * (x + c);
  else r = (c > 0.0f) ? 1.0f - (1.0f - c) * (1.0f - x) : (1.0f + c) * x;
  out[i * ldo + j] = r;
}

// out = alpha * diag(r) x diag(c) + beta * I   (r, c fp64 vectors or NULL = ones)
__global__ void k_scale_shift(const float* __restrict__ x, int64_t ldx, int64_t n,
                              const double* __restrict__ r, const double* __restrict__ c,
                              double alpha, double beta, float* __restrict__ out, int64_t ldo) {
  const int64_t i = blockIdx.y;
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  double v = alpha * (double)x[i * ldx + j] * (r ? r[i] : 1.0) * (c ? c[j] : 1.0);
  if (i == j) v += beta;
  out[i * ldo + j] = (float)v;
}

// ------------------------------------------------------------------ row-wise normalise
__global__ void k_row_normalize(const float* __restrict__ a, int64_t n, int64_t lda,
                                float* __restrict__ out, int64_t ldo) {
  __shared__ float red[32];
  const int64_t i = blockIdx.x;
  const float* r = a + i * lda;
  float m = -INFINITY;
  float* o = out + i * ldo;
  const bool vec = ((reinterpret_cast<uintptr_t>(r) & 15) == 0) && ((reinterpret_cast<uintptr_t>(o) & 15) == 0);
  const int64_t n4 = vec ? (n & ~(int64_t)3) : 0;
  for (int64_t j = (int64_t)threadIdx.x * 4; j < n4; j += (int64_t)blockDim.x * 4) {
    const float4 q = *reinterpret_cast<const float4*>(r + j);
    m = fmaxf(m, fmaxf(fmaxf(q.x, q.y), fmaxf(q.z, q.w)));
  }
  for (int64_t j = n4 + threadIdx.x; j < n; j += blockDim.x) m = fmaxf(m, r[j]);
  m = block_max(m, red);
  for (int64_t j = (int64_t)threadIdx.x * 4; j < n4; j += (int64_t)blockDim.x * 4) {
    const float4 q = *reinterpret_cast<const float4*>(r + j);
    *reinterpret_cast<float4*>(o + j) = make_float4(q.x / m, q.y / m, q.z / m, q.w / m);   // refinement.py:244
  }
  for (int64_t j = n4 + threadIdx.x; j < n; j += blockDim.x) o[j] = r[j] / m;
}

// ------------------------------------------------------------------ Laplacian (materialised)
__global__ void k_laplacian(const float* __restrict__ w, int64_t n, int64_t ldw, int type,
                            double eps, const double* __restrict__ deg, float* __restrict__ out,
                            int64_t ldo) {
  const int64_t i = blockIdx.x;
  const int64_t j = (int64_t)blockIdx.y * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const double wij = (double)w[i * ldw + j];
  const double lij = ((i == j) ? deg[i] : 0.0) - wij;             // laplacian.py:42
  double v;
  if (type == SC_LAPLACIAN_AFFINITY) v = wij;
  else if (type == SC_LAPLACIAN_UNNORMALIZED) v = lij;
  else if (type == SC_LAPLACIAN_RANDOMWALK) v = (1.0 / (deg[i] + eps)) * lij;   // :51-53
  else v = ((1.0 / (sqrt(deg[i]) + eps)) * lij) * (1.0 / (sqrt(deg[j]) + eps));  // :56-58
  out[i * ldo + j] = (float)v;
}

// CropDiagonal values of the rows [row_begin, row_begin + rows) held by the panel `a`.
int crop_diagonal_rows(const float* a, int64_t n, int64_t lda, int64_t row_begin, int64_t rows,
                       float* diag_out, cudaStream_t st) {
  k_crop_diagonal<<<(unsigned)rows, 256, 0, st>>>(a, n, lda, nullptr, 0, diag_out, row_begin);
  sc::launched();
  SC_LAUNCH_CHECK();
  return 0;
}

}  // namespace sc

// ====================================================================== C ABI
using namespace sc;

extern "C" int sc_normalize_rows_typed(sc_context* ctx, const void* x, int x_dtype, int64_t n,
                                       int64_t d, int64_t ldx, float* xn, int64_t ldxn, void* hi,
                                       void* lo, int64_t ldh, void* stream) {
  SC_REQUIRE(ctx && x && n > 0 && d > 0, "sc_normalize_rows: bad arguments");
  SC_REQUIRE((hi == nullptr) == (lo == nullptr), "sc_normalize_rows: hi/lo must come together");
  const int warps = 8;
  const unsigned grid = (unsigned)((n + warps - 1) / warps);
  cudaStream_t st = as_stream(stream);
  __half* h = (__half*)hi;
  __half* l = (__half*)lo;
  switch (x_dtype) {
    case SC_DTYPE_F32:
      k_normalize_rows<float><<<grid, warps * 32, 0, st>>>((const float*)x, n, d, ldx, xn, ldxn,
                                                            h, l, ldh);
      break;
    case SC_DTYPE_F64:
      k_normalize_rows<double><<<grid, warps * 32, 0, st>>>((const double*)x, n, d, ldx, xn, ldxn,
                                                             h, l, ldh);
      break;
    case SC_DTYPE_F16:
      k_normalize_rows<__half><<<grid, warps * 32, 0, st>>>((const __half*)x, n, d, ldx, xn, ldxn,
                                                             h, l, ldh);
      break;
    case SC_DTYPE_BF16:
      k_normalize_rows<__nv_bfloat16><<<grid, warps * 32, 0, st>>>(
          (const __nv_bfloat16*)x, n, d, ldx, xn, ldxn, h, l, ldh);
      break;
    default:
      SC_REQUIRE(false, "sc_normalize_rows_typed: unknown dtype %d", x_dtype);
  }
  sc::launched();
  SC_LAUNCH_CHECK();
  return 0;
}

extern "C" int sc_normalize_rows(sc_context* ctx, const void* x, int x_is_f64, int64_t n,
                                 int64_t d, int64_t ldx, float* xn, int64_t ldxn, void* hi,
                                 void* lo, int64_t ldh, void* stream) {
  return sc_normalize_rows_typed(ctx, x, x_is_f64 ? SC_DTYPE_F64 : SC_DTYPE_F32, n, d, ldx, xn,
                                 ldxn, hi, lo, ldh, stream);
}

extern "C" int sc_crop_diagonal(sc_context* ctx, const float* a, int64_t n, int64_t lda,
                                float* out, int64_t ldo, void* stream) {
  SC_REQUIRE(ctx && a && out && n > 0, "sc_crop_diagonal: bad arguments");
  k_crop_diagonal<<<(unsigned)n, 256, 0, as_stream(stream)>>>(a, n, lda, out, ldo, nullptr, 0); sc::launched();
  SC_LAUNCH_CHECK();
  return 0;
}

extern "C" int sc_crop_diagonal_values(sc_context* ctx, const float* a, int64_t n, int64_t lda,
                                       float* diag_out, void* stream) {
  SC_REQUIRE(ctx && a && diag_out && n > 0, "sc_crop_diagonal_values: bad arguments");
  k_crop_diagonal<<<(unsigned)n, 256, 0, as_stream(stream)>>>(a, n, lda, nullptr, 0, diag_out, 0); sc::launched();
  SC_LAUNCH_CHECK();
  return 0;
}

extern "C" int sc_row_threshold(sc_context* ctx, const float* a, int64_t n, int64_t lda,
                                int type, double p, double mult, int binarize,
                                int preserve_diagonal, float* out, int64_t ldo, void* stream) {
  SC_REQUIRE(ctx && a && out && n > 0, "sc_row_threshold: bad arguments");
  SC_REQUIRE(type == SC_THRESHOLD_ROWMAX || type == SC_THRESHOLD_PERCENTILE,
             "Unsupported thresholding_type");
  const double q = (p * 100.0) / 100.0;   // the reference passes p*100 to np.percentile
  k_row_threshold<<<(unsigned)n, 256, 0, as_stream(stream)>>>(
      a, n, lda, type, (float)p, q, (float)mult, binarize, preserve_diagonal, out, ldo); sc::launched();
  SC_LAUNCH_CHECK();
  return 0;
}

extern "C" int sc_symmetrize(sc_context* ctx, const float* a, int64_t n, int64_t lda, int type,
                             float* out, int64_t ldo, void* stream) {
  SC_REQUIRE(ctx && a && out && n > 0 && a != out, "sc_symmetrize: bad arguments");
  SC_REQUIRE(type == SC_SYMMETRIZE_MAX || type == SC_SYMMETRIZE_AVERAGE,
             "Unsupported symmetrize_type.");
  const unsigned t = (unsigned)((n + 31) / 32);
  k_symmetrize<<<dim3(t, t), dim3(32, 8), 0, as_stream(stream)>>>(a, n, lda, type, out, ldo); sc::launched();
  SC_LAUNCH_CHECK();
  return 0;
}

extern "C" int sc_split_planes(sc_context* ctx, const float* a, int64_t n, int64_t lda, void* hi,
                               void* lo, int64_t ldh, void* stream) {
  SC_REQUIRE(ctx && a && hi && lo && n > 0, "sc_split_planes: bad arguments");
  SC_REQUIRE(vec_ok_f32(a, lda), "sc_split_planes: `a` needs a 16-byte aligned base and lda %% 4 == 0");
  const unsigned gx = (unsigned)((n + 1023) / 1024);
  k_split_planes<<<dim3((unsigned)n, gx), 256, 0, as_stream(stream)>>>(a, n, lda, (__half*)hi,
                                                                        (__half*)lo, ldh); sc::launched();
  SC_LAUNCH_CHECK();
  return 0;
}

extern "C" int sc_row_stats(sc_context* ctx, const float* a, int64_t n, int64_t lda,
                            double* rowmax, double* rowsum, void* stream) {
  SC_REQUIRE(ctx && a && n > 0, "sc_row_stats: bad arguments");
  SC_REQUIRE(vec_ok_f32(a, lda), "sc_row_stats: `a` needs a 16-byte aligned base and lda %% 4 == 0");
  k_row_stats<<<(unsigned)n, 256, 0, as_stream(stream)>>>(a, n, lda, rowmax, rowsum); sc::launched();
  SC_LAUNCH_CHECK();
  return 0;
}

extern "C" int sc_affinity_stats(sc_context* ctx, const float* a, int64_t n, int64_t lda,
                                 double* out_host, void* stream) {
  SC_REQUIRE(ctx && a && out_host && n > 0, "sc_affinity_stats: bad arguments");
  SC_REQUIRE(vec_ok_f32(a, lda), "sc_affinity_stats: `a` needs a 16-byte aligned base and lda %% 4 == 0");
  cudaStream_t st = as_stream(stream);
  Scratch part;
  SC_CUDA(part.alloc(sizeof(double) * (size_t)(3 * n + 4), st));
  double* p = part.as<double>();
  k_affinity_row_stats<<<(unsigned)n, 256, 0, st>>>(a, n, lda, 0, p, nullptr); sc::launched();
  k_affinity_stats_finish<<<1, 1024, 0, st>>>(p, a, n, lda, p + 3 * n); sc::launched();
  SC_LAUNCH_CHECK();
  SC_CUDA(cudaMemcpyAsync(out_host, p + 3 * n, sizeof(double) * 4, cudaMemcpyDeviceToHost, st));
  SC_CUDA(cudaStreamSynchronize(st));
  return 0;
}

extern "C" int sc_affinity_stats_rows(sc_context* ctx, const float* panel, int64_t rows, int64_t n,
                                      int64_t ldp, int64_t row_begin, double* part, void* stream) {
  SC_REQUIRE(ctx && panel && part && n > 0 && rows > 0 && row_begin >= 0 && row_begin + rows <= n &&
             ldp >= n, "sc_affinity_stats_rows: bad arguments");
  SC_REQUIRE(vec_ok_f32(panel, ldp),
             "sc_affinity_stats_rows: `panel` needs a 16-byte aligned base and ldp %% 4 == 0");
  k_affinity_row_stats<<<(unsigned)rows, 256, 0, as_stream(stream)>>>(panel, n, ldp, row_begin,
                                                                       part, part + 3 * n);
  sc::launched();
  SC_LAUNCH_CHECK();
  return 0;
}

extern "C" int sc_affinity_stats_finish(sc_context* ctx, double* part, int64_t n, double* out_host,
                                        void* stream) {
  SC_REQUIRE(ctx && part && out_host && n > 0, "sc_affinity_stats_finish: bad arguments");
  cudaStream_t st = as_stream(stream);
  k_affinity_stats_finish<<<1, 1024, 0, st>>>(part, nullptr, n, 0, part + 4 * n); sc::launched();
  SC_LAUNCH_CHECK();
  SC_CUDA(cudaMemcpyAsync(out_host, part + 4 * n, sizeof(double) * 4, cudaMemcpyDeviceToHost, st));
  SC_CUDA(cudaStreamSynchronize(st));
  return 0;
}

extern "C" int sc_row_stats_block(sc_context* ctx, const float* a, int64_t rows, int64_t cols,
                                  int64_t lda, double* rowmax, double* rowsum, void* stream) {
  SC_REQUIRE(ctx && a && rows > 0 && cols > 0, "sc_row_stats_block: bad arguments");
  SC_REQUIRE(vec_ok_f32(a, lda), "sc_row_stats_block: `a` needs a 16-byte aligned base and lda %% 4 == 0");
  k_row_stats<<<(unsigned)rows, 256, 0, as_stream(stream)>>>(a, cols, lda, rowmax, rowsum);
  sc::launched();
  SC_LAUNCH_CHECK();
  return 0;
}

extern "C" int sc_transpose(sc_context* ctx, const float* src, int64_t rows, int64_t cols,
                            int64_t lds, float* dst, int64_t ldd, void* stream) {
  SC_REQUIRE(ctx && src && dst && rows > 0 && cols > 0 && src != dst, "sc_transpose: bad arguments");
  const dim3 grid((unsigned)((cols + 31) / 32), (unsigned)((rows + 31) / 32));
  SC_REQUIRE(grid.y <= 65535u, "sc_transpose: too many rows");
  k_transpose<<<grid, dim3(32, 8), 0, as_stream(stream)>>>(src, rows, cols, lds, dst, ldd);
  sc::launched();
  SC_LAUNCH_CHECK();
  return 0;
}

extern "C" int sc_row_normalize(sc_context* ctx, const float* a, int64_t n, int64_t lda,
                                float* out, int64_t ldo, void* stream) {
  SC_REQUIRE(ctx && a && out && n > 0, "sc_row_normalize: bad arguments");
  k_row_normalize<<<(unsigned)n, 256, 0, as_stream(stream)>>>(a, n, lda, out, ldo); sc::launched();
  SC_LAUNCH_CHECK();
  return 0;
}

extern "C" int sc_laplacian(sc_context* ctx, const float* w, int64_t n, int64_t ldw, int type,
                            double eps, float* out, int64_t ldo, void* stream) {
  SC_REQUIRE(ctx && w && out && n > 0, "sc_laplacian: bad arguments");
  SC_REQUIRE(type >= SC_LAPLACIAN_AFFINITY && type <= SC_LAPLACIAN_GRAPHCUT,
             "Unsupported laplacian_type.");
  SC_REQUIRE(vec_ok_f32(w, ldw), "sc_laplacian: `w` needs a 16-byte aligned base and ldw %% 4 == 0");
  cudaStream_t st = as_stream(stream);
  Scratch deg;
  SC_CUDA(deg.alloc(sizeof(double) * (size_t)n, st));
  k_row_stats<<<(unsigned)n, 256, 0, st>>>(w, n, ldw, nullptr, deg.as<double>()); sc::launched();
  SC_LAUNCH_CHECK();
  const unsigned gx = (unsigned)((n + 255) / 256);
  k_laplacian<<<dim3((unsigned)n, gx), 256, 0, st>>>(w, n, ldw, type, eps, deg.as<double>(), out,
                                                     ldo); sc::launched();
  SC_LAUNCH_CHECK();
  return 0;
}

extern "C" int sc_constraint_combine(sc_context* ctx, const float* a, int64_t lda, const float* q,
                                     int64_t ldq, int64_t n, int mode, float* out, int64_t ldo,
                                     void* stream) {
  SC_REQUIRE(ctx && a && q && out && n > 0 && mode >= 0 && mode <= 2, "sc_constraint_combine: bad arguments");
  SC_REQUIRE(n <= 65535, "sc_constraint_combine: n too large for the element-wise grid");
  k_constraint_combine<<<dim3((unsigned)((n + 255) / 256), (unsigned)n), 256, 0, as_stream(stream)>>>(
      a, lda, q, ldq, n, mode, out, ldo); sc::launched();
  SC_LAUNCH_CHECK();
  return 0;
}

extern "C" int sc_scale_shift(sc_context* ctx, const float* x, int64_t ldx, int64_t n,
                              const double* row_scale, const double* col_scale, double alpha,
                              double beta, float* out, int64_t ldo, void* stream) {
  SC_REQUIRE(ctx && x && out && n > 0, "sc_scale_shift: bad arguments");
  SC_REQUIRE(n <= 65535, "sc_scale_shift: n too large for the element-wise grid");
  k_scale_shift<<<dim3((unsigned)((n + 255) / 256), (unsigned)n), 256, 0, as_stream(stream)>>>(
      x, ldx, n, row_scale, col_scale, alpha, beta, out, ldo); sc::launched();
  SC_LAUNCH_CHECK();
  return 0;
}

extern "C" int sc_row_group_bounds(sc_context* ctx, const void* y_hi, int64_t n, int64_t ldy,
                                   float* norms, int64_t groups, double* diag_lb, double* rowsum,
                                   void* stream) {
  SC_REQUIRE(ctx && y_hi && norms && diag_lb && rowsum && n > 0 &&
             groups == (n + BOUND_GROUP - 1) / BOUND_GROUP, "sc_row_group_bounds: bad arguments");
  SC_REQUIRE(vec_ok_f16(y_hi, ldy) && ldy >= n, "sc_row_group_bounds: y_hi needs a 16-byte aligned "
             "base and ldy %% 8 == 0");
  k_row_group_bounds<<<(unsigned)n, 256, 0, as_stream(stream)>>>(
      (const __half*)y_hi, n, ldy, norms, (int)groups, diag_lb, rowsum);
  sc::launched();
  SC_LAUNCH_CHECK();
  return 0;
}

extern "C" int sc_gather_rows_f16(sc_context* ctx, const void* src, int64_t lds, const int* perm,
                                  int64_t rows, int64_t cols, void* dst, int64_t ldd,
                                  void* stream) {
  SC_REQUIRE(ctx && src && perm && dst && rows > 0 && cols > 0 && cols % 8 == 0 && cols <= lds &&
             cols <= ldd, "sc_gather_rows_f16: bad arguments");
  SC_REQUIRE(vec_ok_f16(src, lds) && vec_ok_f16(dst, ldd),
             "sc_gather_rows_f16: 16-byte aligned bases and leading dimensions %% 8 == 0");
  k_gather_rows_f16<<<(unsigned)rows, 256, 0, as_stream(stream)>>>(
      (const __half*)src, lds, perm, cols, (__half*)dst, ldd);
  sc::launched();
  SC_LAUNCH_CHECK();
  return 0;
}
