// GaussianBlur (refinement.py:160-162 == scipy.ndimage.gaussian_filter(a, sigma), separable
// correlate1d along axis 0 then axis 1, mode='reflect', truncate=4.0) as a shared-memory tiled
// stencil, with three epilogues so that the ICASSP-2018 chain
//     CropDiagonal -> GaussianBlur -> RowWiseThreshold(RowMax) -> Symmetrize
// costs 12 B per matrix element of HBM traffic (SURVEY.md 8(d)):
//   pass 1  EPI_STATS : read A (diag <- crop vector), blur on the fly, emit row maxima only
//   pass 2  EPI_THRSYM: read A again, blur again, apply the threshold/symmetrize rule with
//                       (m_i, m_j), write Y as split fp16 planes (4 B/element) and/or fp32
//   EPI_STORE materialises B for the generic (unfused) operator API.
// The blur is recomputed rather than stored: 18 FMAs per element are free next to 4+4 bytes.
//
// Whole-matrix, symmetric input (the single-GPU hot path) goes one step further (EPI_UPPER +
// k_thrsym_upper): B = blur(A) is symmetric, so only the tiles that touch the upper triangle are
// blurred -- ONCE.  Pass 1 reads half of A, stores that half of B and folds both the row maxima
// and the column maxima of every tile into m (m_i = max_j B_ij needs the lower half only through
// B_ji).  Pass 2 is element-wise on the stored half of B and writes Y(i,j) and Y(j,i) (transposed
// through shared memory).  HBM traffic 2 + 2 + 2 + 4 = 10 B per element of the matrix (the
// contract figure is 12) and half the filter arithmetic of the two-pass form; both kernels were
// issue-bound, not bandwidth-bound.
//
// Two kernels: k_blur_tile<R> (compile-time radius, register sliding windows; R=4 is sigma=1,
// the configuration every BASELINE config uses) and k_blur_generic (run-time radius <= 64).
#include "common.cuh"

#include <cstdlib>

namespace sc {

constexpr int kMaxRadius = 64;

struct BlurArgs {
  const float* a;          // rows [in_row_base, ...) of the global n x n matrix
  int64_t n, lda;
  // Row block (multi-GPU row sharding; the single-GPU case is 0, n, 0, 0): outputs are produced
  // for global rows [row_begin, row_end); output buffers start at global row out_row_base.
  // Vectors (diag, m, rowmax_out) are indexed by GLOBAL row/column.
  int64_t row_begin, row_end, in_row_base, out_row_base;
  const float* diag;       // optional replacement of a[i][i]
  int radius;
  float* out;              // EPI_STORE
  int64_t ldo;
  float* rowmax_out;       // EPI_STORE (optional) / EPI_STATS
  // threshold + symmetrize epilogue
  const float* m;          // row maxima of the blurred matrix
  float p, mult;
  int binarize, preserve_diag, sym_type, stats_zero_diag;
  int tiles_per_cta;       // column tiles swept by one CTA of k_blur_band (cp.async pipeline)
  float* y;
  int64_t ldy;
  __half* hi;
  __half* lo;
  int64_t ldh;
};

struct BlurWeights {
  float w[2 * kMaxRadius + 1];
};

enum { EPI_STORE = 0, EPI_STATS = 1, EPI_THRSYM = 2, EPI_UPPER = 3 };

// scipy 'reflect' (half-sample symmetric, period 2n): d c b a | a b c d | d c b a
__device__ __forceinline__ int64_t reflect_index(int64_t i, int64_t n) {
  const int64_t period = 2 * n;
  i %= period;
  if (i < 0) i += period;
  return (i < n) ? i : (period - 1 - i);
}

__device__ __forceinline__ float threshold_rule(float b, float m, float p, float mult,
                                                int binarize) {
  return (b < m * p) ? b * mult : (binarize ? 1.0f : b);
}

// One output element (i, j) with blurred value b.  Returns the value that takes part in the
// row maximum (EPI_STORE / EPI_STATS).
template <int EPI>
__device__ __forceinline__ float blur_epilogue(const BlurArgs& g, int64_t i, int64_t j, float b) {
  if (EPI == EPI_STORE) {
    g.out[(i - g.out_row_base) * g.ldo + j] = b;
    return b;
  } else if (EPI == EPI_STATS) {
    return (g.stats_zero_diag && i == j) ? 0.0f : b;   // RowWiseThreshold preserve_diagonal
  } else {
    float yv;
    if (g.preserve_diag && i == j) {
      yv = 1.0f;                                        // refinement.py:208-209
    } else {
      const float t1 = threshold_rule(b, g.m[i], g.p, g.mult, g.binarize);
      const float t2 = threshold_rule(b, g.m[j], g.p, g.mult, g.binarize);
      yv = (g.sym_type == SC_SYMMETRIZE_MAX) ? fmaxf(t1, t2) : 0.5f * (t1 + t2);
    }
    if (g.y) g.y[(i - g.out_row_base) * g.ldy + j] = yv;
    if (g.hi) {
      __half h, l;
      split_half(yv, h, l);
      g.hi[(i - g.out_row_base) * g.ldh + j] = h;
      g.lo[(i - g.out_row_base) * g.ldh + j] = l;
    }
    return yv;
  }
}

__device__ __forceinline__ float load_input(const BlurArgs& g, int64_t gr, int64_t gc) {
  if (g.diag && gr == gc) return g.diag[gr];
  return g.a[(gr - g.in_row_base) * g.lda + gc];
}

// ------------------------------------------------------------------ generic radius
constexpr int GTH = 32, GTW = 64, GTHREADS = 256;

template <int EPI>
__global__ void __launch_bounds__(GTHREADS)
k_blur_generic(const BlurArgs g, const BlurWeights bw) {
  extern __shared__ float smem[];
  const int R = g.radius;
  const int IW = GTW + 2 * R, IH = GTH + 2 * R;
  float* in = smem;                 // [IH][IW]
  float* mid = smem + IH * IW;      // [GTH][IW]
  const int64_t row0 = g.row_begin + (int64_t)blockIdx.y * GTH, col0 = (int64_t)blockIdx.x * GTW;
  for (int idx = threadIdx.x; idx < IH * IW; idx += GTHREADS) {
    const int r = idx / IW, c = idx - r * IW;
    const int64_t gr = reflect_index(row0 - R + r, g.n), gc = reflect_index(col0 - R + c, g.n);
    in[idx] = load_input(g, gr, gc);
  }
  __syncthreads();
  for (int idx = threadIdx.x; idx < GTH * IW; idx += GTHREADS) {   // axis 0 (down the rows)
    const int r = idx / IW, c = idx - r * IW;
    float acc = 0.0f;
    for (int k = 0; k <= 2 * R; ++k) acc = fmaf(bw.w[k], in[(r + k) * IW + c], acc);
    mid[idx] = acc;
  }
  __syncthreads();
  for (int idx = threadIdx.x; idx < GTH * GTW; idx += GTHREADS) {  // axis 1 + epilogue
    const int r = idx / GTW, c = idx - r * GTW;                     // a warp = half a row
    float acc = 0.0f;
    for (int k = 0; k <= 2 * R; ++k) acc = fmaf(bw.w[k], mid[r * IW + c + k], acc);
    const int64_t i = row0 + r, j = col0 + c;
    float v = 0.0f;
    if (i < g.row_end && j < g.n) v = blur_epilogue<EPI>(g, i, j, acc);
    if (EPI != EPI_THRSYM && g.rowmax_out) {
      v = fmaxf(v, 0.0f);
      v = warp_max(v);
      if ((threadIdx.x & 31) == 0 && i < g.row_end) atomic_max_nonneg(g.rowmax_out + i, v);
    }
  }
}

// ------------------------------------------------------------------ compile-time radius
// Tile = 32 x 128 outputs, 288 threads (9 warps), two barriers per tile:
//   fill      (40 x 136 halo'd input, 128-bit global loads into shared memory)
//   vertical  thread = (column, 16-row strip): a 24-deep register window slides down the column;
//             lanes run along columns -> conflict-free reads of `in`, conflict-free writes of `mid`
//   horizontal thread = (row, 16-column strip): 24-deep window along the row of `mid` (pitch 137,
//             odd, so lanes running along rows hit 32 different banks); the 16 outputs stay in
//             registers and go straight into the epilogue -- 64 contiguous bytes of fp32 (or 32 B
//             per fp16 plane) per thread, whole 32-byte sectors, no staging pass.
// Shared-memory traffic: ~22 B per output element (was ~34 with the transposed staging), i.e.
// below the 4+8 B/element of HBM traffic the two passes of the fused chain are allowed.
constexpr int TTH = 32, TTW = 128, TTHREADS = 288, VSTRIP = 16, HSTRIP = 16;

template <int EPI>
__device__ __forceinline__ void epilogue16(const BlurArgs& g, int64_t i, int64_t j0,
                                           const float (&b)[HSTRIP], float& rmax) {
  const bool full = (j0 + HSTRIP <= g.n);
  if (EPI == EPI_STATS) {
    float v = rmax;
#pragma unroll
    for (int t = 0; t < HSTRIP; ++t) {
      float x = b[t];
      if (!full && j0 + t >= g.n) x = 0.0f;
      if (g.stats_zero_diag && i == j0 + t) x = 0.0f;   // RowWiseThreshold preserve_diagonal
      v = fmaxf(v, x);
    }
    rmax = v;
    return;
  }
  const int64_t io = i - g.out_row_base;
  if (EPI == EPI_UPPER) {
    // edge / diagonal tiles of the symmetric pass: store B, row maximum in the register, column
    // maxima by one atomic per element (O(N) such tiles out of N^2/4096)
    float* dst = g.out + io * g.ldo + j0;
    float v = rmax;
#pragma unroll
    for (int t = 0; t < HSTRIP; ++t) {
      if (!full && j0 + t >= g.n) continue;
      dst[t] = b[t];
      const float x = (g.stats_zero_diag && i == j0 + t) ? 0.0f : b[t];
      v = fmaxf(v, x);
      atomic_max_nonneg(g.rowmax_out + j0 + t, fmaxf(x, 0.0f));
    }
    rmax = v;
    return;
  }
  if (EPI == EPI_STORE) {
    float* dst = g.out + io * g.ldo + j0;
    if (full) {
#pragma unroll
      for (int q = 0; q < HSTRIP / 4; ++q)
        *reinterpret_cast<float4*>(dst + 4 * q) =
            make_float4(b[4 * q], b[4 * q + 1], b[4 * q + 2], b[4 * q + 3]);
    } else {
#pragma unroll
      for (int t = 0; t < HSTRIP; ++t)
        if (j0 + t < g.n) dst[t] = b[t];
    }
    if (g.rowmax_out) {
      float v = 0.0f;
#pragma unroll
      for (int t = 0; t < HSTRIP; ++t)
        if (full || j0 + t < g.n) v = fmaxf(v, b[t]);
      atomic_max_nonneg(g.rowmax_out + i, v);
    }
    return;
  }
  // EPI_THRSYM: y = sym(thr(b, m_i), thr(b, m_j))  (SURVEY.md A.3)
  const float cut_i = g.m[i] * g.p;
  float y[HSTRIP];
#pragma unroll
  for (int q = 0; q < HSTRIP / 4; ++q) {
    float mj[4];
    if (full) {
      const float4 v = *reinterpret_cast<const float4*>(g.m + j0 + 4 * q);   // warp-broadcast
      mj[0] = v.x; mj[1] = v.y; mj[2] = v.z; mj[3] = v.w;
    } else {
#pragma unroll
      for (int t = 0; t < 4; ++t) mj[t] = (j0 + 4 * q + t < g.n) ? g.m[j0 + 4 * q + t] : 0.0f;
    }
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      const float x = b[4 * q + t];
      const float keep = g.binarize ? 1.0f : x;
      const float small = x * g.mult;
      const float t1 = (x < cut_i) ? small : keep;
      const float t2 = (x < mj[t] * g.p) ? small : keep;
      y[4 * q + t] = (g.sym_type == SC_SYMMETRIZE_MAX) ? fmaxf(t1, t2) : 0.5f * (t1 + t2);
    }
  }
  if (g.preserve_diag) {
#pragma unroll
    for (int t = 0; t < HSTRIP; ++t)
      if (i == j0 + t) y[t] = 1.0f;                       // refinement.py:208-209
  }
  if (full) {
    if (g.y) {
      float* dst = g.y + io * g.ldy + j0;
#pragma unroll
      for (int q = 0; q < HSTRIP / 4; ++q)
        *reinterpret_cast<float4*>(dst + 4 * q) =
            make_float4(y[4 * q], y[4 * q + 1], y[4 * q + 2], y[4 * q + 3]);
    }
    if (g.hi) {
      uint32_t hw[HSTRIP / 2], lw[HSTRIP / 2];
#pragma unroll
      for (int q = 0; q < HSTRIP / 2; ++q) {
        const __half2 h = __floats2half2_rn(y[2 * q], y[2 * q + 1]);
        const float2 f = __half22float2(h);
        const __half2 l = __floats2half2_rn(y[2 * q] - f.x, y[2 * q + 1] - f.y);
        hw[q] = *reinterpret_cast<const uint32_t*>(&h);
        lw[q] = *reinterpret_cast<const uint32_t*>(&l);
      }
      uint4* hd = reinterpret_cast<uint4*>(g.hi + io * g.ldh + j0);
      uint4* ld = reinterpret_cast<uint4*>(g.lo + io * g.ldh + j0);
      hd[0] = make_uint4(hw[0], hw[1], hw[2], hw[3]);
      hd[1] = make_uint4(hw[4], hw[5], hw[6], hw[7]);
      ld[0] = make_uint4(lw[0], lw[1], lw[2], lw[3]);
      ld[1] = make_uint4(lw[4], lw[5], lw[6], lw[7]);
    }
  } else {
#pragma unroll
    for (int t = 0; t < HSTRIP; ++t) {
      if (j0 + t >= g.n) continue;
      if (g.y) g.y[io * g.ldy + j0 + t] = y[t];
      if (g.hi) {
        __half h, l;
        split_half(y[t], h, l);
        g.hi[io * g.ldh + j0 + t] = h;
        g.lo[io * g.ldh + j0 + t] = l;
      }
    }
  }
}

__device__ __forceinline__ void cp_async16(float* smem_dst, const float* gmem_src) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;"
               ::"r"((uint32_t)__cvta_generic_to_shared(smem_dst)), "l"(gmem_src)
               : "memory");
}
__device__ __forceinline__ void cp_async_commit() {
  asm volatile("cp.async.commit_group;" ::: "memory");
}
template <int N>
__device__ __forceinline__ void cp_async_wait() {
  asm volatile("cp.async.wait_group %0;" ::"n"(N) : "memory");
}

template <int R>
struct TileGeom {
  static constexpr int IW = TTW + 2 * R, IH = TTH + 2 * R, MP = IW + 1;
  static_assert(IW % 4 == 0 && R % 4 == 0, "vector fill needs 16-byte aligned tile origins");
  static_assert(IW * (TTH / VSTRIP) <= TTHREADS && TTH * (TTW / HSTRIP) <= TTHREADS,
                "one work item per thread in both passes");
};

template <int R>
__device__ __forceinline__ bool tile_is_vec(const BlurArgs& g, int64_t row0, int64_t col0) {
  return (row0 >= R) && (col0 >= R) && (row0 + TTH + R <= g.n) && (col0 + TTW + R <= g.n) &&
         ((g.lda & 3) == 0) && ((reinterpret_cast<uintptr_t>(g.a) & 15) == 0);
}

// Stage the halo'd input tile into `in`.  Interior tiles go through cp.async (16-byte copies
// that complete in the background: the caller commits the group and waits before use); edge
// tiles take the synchronous path with reflected indices.
template <int R>
__device__ __forceinline__ void tile_fill(const BlurArgs& g, int64_t row0, int64_t col0,
                                          float* in) {
  using G = TileGeom<R>;
  const int tid = threadIdx.x;
  if (tile_is_vec<R>(g, row0, col0)) {
    const float* src = g.a + (row0 - R - g.in_row_base) * g.lda + (col0 - R);
    for (int idx = tid; idx < G::IH * (G::IW / 4); idx += TTHREADS) {
      const int r = idx / (G::IW / 4), q = idx - r * (G::IW / 4);
      cp_async16(in + r * G::IW + 4 * q, src + (int64_t)r * g.lda + 4 * q);
    }
  } else {
    for (int idx = tid; idx < G::IH * G::IW; idx += TTHREADS) {
      const int r = idx / G::IW, c = idx - r * G::IW;
      const int64_t gr = reflect_index(row0 - R + r, g.n), gc = reflect_index(col0 - R + c, g.n);
      in[idx] = load_input(g, gr, gc);      // applies the diagonal override itself
    }
  }
}

// Both separable passes + epilogue on a staged tile.  The caller has made `in` visible to the
// whole block (cp.async.wait_group + __syncthreads) and guarantees nobody still reads `mid`.
template <int R, int EPI>
__device__ __forceinline__ void tile_compute(const BlurArgs& g, const float (&w)[2 * R + 1],
                                             int64_t row0, int64_t col0, float* in, float* mid,
                                             float& rmax) {
  using G = TileGeom<R>;
  const int tid = threadIdx.x;
  if (g.diag && tile_is_vec<R>(g, row0, col0)) {
    // fused CropDiagonal on the vector path: patch the diagonal elements inside the halo'd tile
    const int64_t lo = (row0 > col0 ? row0 : col0) - R;
    const int64_t hi = ((row0 + TTH < col0 + TTW) ? row0 + TTH : col0 + TTW) + R;
    if (lo < hi) {                                     // block-uniform
      for (int64_t d = lo + tid; d < hi; d += TTHREADS)
        in[(d - (row0 - R)) * G::IW + (d - (col0 - R))] = g.diag[d];
      __syncthreads();
    }
  }
  if (tid < G::IW * (TTH / VSTRIP)) {
    const int c = tid % G::IW, r0 = (tid / G::IW) * VSTRIP;
    float win[VSTRIP + 2 * R];
#pragma unroll
    for (int k = 0; k < VSTRIP + 2 * R; ++k) win[k] = in[(r0 + k) * G::IW + c];
#pragma unroll
    for (int o = 0; o < VSTRIP; ++o) {
      float acc = 0.0f;
#pragma unroll
      for (int k = 0; k <= 2 * R; ++k) acc = fmaf(w[k], win[o + k], acc);
      mid[(r0 + o) * G::MP + c] = acc;
    }
  }
  __syncthreads();
  if (tid < TTH * (TTW / HSTRIP)) {
    const int r = tid % TTH, c0 = (tid / TTH) * HSTRIP;
    float win[HSTRIP + 2 * R];
#pragma unroll
    for (int k = 0; k < HSTRIP + 2 * R; ++k) win[k] = mid[r * G::MP + c0 + k];
    float b[HSTRIP];
#pragma unroll
    for (int o = 0; o < HSTRIP; ++o) {
      float acc = 0.0f;
#pragma unroll
      for (int k = 0; k <= 2 * R; ++k) acc = fmaf(w[k], win[o + k], acc);
      b[o] = acc;
    }
    const int64_t i = row0 + r, j0 = col0 + c0;
    if (i < g.row_end && j0 < g.n) epilogue16<EPI>(g, i, j0, b, rmax);
  }
}

// ---- fast path: interior, off-diagonal, full tiles (all but O(N) of the N^2/4096 tiles).
// Everything that does not change from tile to tile inside a band is hoisted into FastCtx, and
// nothing is bounds-checked: the general tile_fill / tile_compute above remain the fallback for
// edge tiles, tiles that touch the diagonal (CropDiagonal patch, preserve_diagonal) and ragged
// row blocks.
template <int R>
struct FastCtx {
  static constexpr int FILL_ITERS = (TileGeom<R>::IH * (TileGeom<R>::IW / 4) + TTHREADS - 1) / TTHREADS;
  int fill_smem[FILL_ITERS];   // float offset inside the tile buffer (-1: no copy this round)
  int fill_gofs[FILL_ITERS];   // element offset from the tile's first source element
  int v_in, v_mid;             // vertical pass: first input / output element (-1: idle)
  int h_mid, h_c0;             // horizontal pass: first `mid` element (-1: idle), strip column
  float cut_i;                 // m[i] * p of this thread's output row (EPI_THRSYM)
  float* y_row;                // output row bases of this thread's row
  __half* hi_row;
  __half* lo_row;
  float* out_row;
};

template <int R>
__device__ __forceinline__ bool tile_is_fast(const BlurArgs& g, int64_t row0, int64_t col0) {
  if (!tile_is_vec<R>(g, row0, col0)) return false;
  if (col0 + TTW > g.n || row0 + TTH > g.row_end) return false;
  // tiles whose halo'd footprint meets the diagonal take the general path
  const int64_t lo = (row0 > col0 ? row0 : col0) - R;
  const int64_t hi = ((row0 + TTH < col0 + TTW) ? row0 + TTH : col0 + TTW) + R;
  return lo >= hi;
}

template <int R>
__device__ __forceinline__ void fast_fill(const FastCtx<R>& c, const float* src, float* in) {
#pragma unroll
  for (int k = 0; k < FastCtx<R>::FILL_ITERS; ++k)
    if (c.fill_smem[k] >= 0) cp_async16(in + c.fill_smem[k], src + c.fill_gofs[k]);
}

template <int R, int EPI>
__device__ __forceinline__ void fast_compute(const BlurArgs& g, const FastCtx<R>& c,
                                             const float (&w)[2 * R + 1], int64_t col0,
                                             const float* in, float* mid, float& rmax) {
  using G = TileGeom<R>;
  if (c.v_in >= 0) {
    float win[VSTRIP + 2 * R];
#pragma unroll
    for (int k = 0; k < VSTRIP + 2 * R; ++k) win[k] = in[c.v_in + k * G::IW];
#pragma unroll
    for (int o = 0; o < VSTRIP; ++o) {
      float acc = 0.0f;
#pragma unroll
      for (int k = 0; k <= 2 * R; ++k) acc = fmaf(w[k], win[o + k], acc);
      mid[c.v_mid + o * G::MP] = acc;
    }
  }
  __syncthreads();
  if (c.h_mid >= 0) {
    float win[HSTRIP + 2 * R];
#pragma unroll
    for (int k = 0; k < HSTRIP + 2 * R; ++k) win[k] = mid[c.h_mid + k];
    float b[HSTRIP];
#pragma unroll
    for (int o = 0; o < HSTRIP; ++o) {
      float acc = 0.0f;
#pragma unroll
      for (int k = 0; k <= 2 * R; ++k) acc = fmaf(w[k], win[o + k], acc);
      b[o] = acc;
    }
    const int64_t j0 = col0 + c.h_c0;
    if (EPI == EPI_STATS) {
      float v = rmax;
#pragma unroll
      for (int t = 0; t < HSTRIP; ++t) v = fmaxf(v, b[t]);
      rmax = v;
    } else if (EPI == EPI_UPPER) {
#pragma unroll
      for (int q = 0; q < HSTRIP / 4; ++q)
        *reinterpret_cast<float4*>(c.out_row + j0 + 4 * q) =
            make_float4(b[4 * q], b[4 * q + 1], b[4 * q + 2], b[4 * q + 3]);
      float v = rmax;
#pragma unroll
      for (int t = 0; t < HSTRIP; ++t) v = fmaxf(v, b[t]);
      rmax = v;
      // Column maxima of the tile: the lanes of this warp are its 32 rows, each holding the same 16
      // columns.  The blurred values are non-negative, so their bit patterns order like signed
      // integers and one REDUX.MAX per column reduces across the warp (16 instructions; the
      // shuffle butterfly before it took ~95); lane t keeps column t and issues its atomic.
      const int lane = threadIdx.x & 31;
      float cm = 0.0f;
#pragma unroll
      for (int t = 0; t < HSTRIP; ++t) {
        const int mx = __reduce_max_sync(0xffffffffu, __float_as_int(fmaxf(b[t], 0.0f)));
        if (lane == t) cm = __int_as_float(mx);
      }
      if (lane < HSTRIP) atomic_max_nonneg(g.rowmax_out + j0 + lane, cm);
    } else if (EPI == EPI_STORE) {
#pragma unroll
      for (int q = 0; q < HSTRIP / 4; ++q)
        *reinterpret_cast<float4*>(c.out_row + j0 + 4 * q) =
            make_float4(b[4 * q], b[4 * q + 1], b[4 * q + 2], b[4 * q + 3]);
      if (g.rowmax_out) {
        float v = 0.0f;
#pragma unroll
        for (int t = 0; t < HSTRIP; ++t) v = fmaxf(v, b[t]);
        atomic_max_nonneg(g.rowmax_out + (c.out_row - g.out) / g.ldo + g.out_row_base, v);
      }
    } else {
      float y[HSTRIP];
#pragma unroll
      for (int q = 0; q < HSTRIP / 4; ++q) {
        const float4 mq = *reinterpret_cast<const float4*>(g.m + j0 + 4 * q);   // warp-broadcast
        const float mj[4] = {mq.x, mq.y, mq.z, mq.w};
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          const float x = b[4 * q + t];
          const float keep = g.binarize ? 1.0f : x;
          const float small = x * g.mult;
          const float t1 = (x < c.cut_i) ? small : keep;
          const float t2 = (x < mj[t] * g.p) ? small : keep;
          y[4 * q + t] = (g.sym_type == SC_SYMMETRIZE_MAX) ? fmaxf(t1, t2) : 0.5f * (t1 + t2);
        }
      }
      if (c.y_row) {
#pragma unroll
        for (int q = 0; q < HSTRIP / 4; ++q)
          *reinterpret_cast<float4*>(c.y_row + j0 + 4 * q) =
              make_float4(y[4 * q], y[4 * q + 1], y[4 * q + 2], y[4 * q + 3]);
      }
      if (c.hi_row) {
        uint32_t hw[HSTRIP / 2], lw[HSTRIP / 2];
#pragma unroll
        for (int q = 0; q < HSTRIP / 2; ++q) {
          const __half2 h = __floats2half2_rn(y[2 * q], y[2 * q + 1]);
          const float2 f = __half22float2(h);
          const __half2 l = __floats2half2_rn(y[2 * q] - f.x, y[2 * q + 1] - f.y);
          hw[q] = *reinterpret_cast<const uint32_t*>(&h);
          lw[q] = *reinterpret_cast<const uint32_t*>(&l);
        }
        uint4* hd = reinterpret_cast<uint4*>(c.hi_row + j0);
        uint4* ld = reinterpret_cast<uint4*>(c.lo_row + j0);
        hd[0] = make_uint4(hw[0], hw[1], hw[2], hw[3]);
        hd[1] = make_uint4(hw[4], hw[5], hw[6], hw[7]);
        ld[0] = make_uint4(lw[0], lw[1], lw[2], lw[3]);
        ld[1] = make_uint4(lw[4], lw[5], lw[6], lw[7]);
      }
    }
  }
}

// One CTA per (32-row band, run of `tiles_per_cta` column tiles), 2-deep cp.async pipeline: the
// loads of tile t+1 are in flight while tile t is filtered, so every resident CTA always has
// ~22 KB outstanding (3 CTAs/SM) -- the first, load-then-compute version left HBM idle during
// the two filter passes and ran latency-bound at ~28% of the roofline.
//   EPI_STATS : row maxima of the blurred band, one register per thread, no atomics
//   EPI_THRSYM/EPI_STORE : the band's output rows
template <int R, int EPI>
__global__ void __launch_bounds__(TTHREADS)
k_blur_band(const BlurArgs g, const BlurWeights bw) {
  using G = TileGeom<R>;
  extern __shared__ float smem[];
  __shared__ float part[TTW / HSTRIP][TTH];
  float* in0 = smem;
  float* in1 = smem + G::IH * G::IW;
  float* mid = smem + 2 * G::IH * G::IW;
  float w[2 * R + 1];
#pragma unroll
  for (int k = 0; k <= 2 * R; ++k) w[k] = bw.w[k];
  float rmax = 0.0f;
  const int tid = threadIdx.x;
  const int64_t row0 = g.row_begin + (int64_t)blockIdx.x * TTH;
  // blockIdx.y selects a run of `tiles_per_cta` column tiles of the band
  const int ntiles = (int)((g.n + TTW - 1) / TTW);
  // EPI_UPPER: only the column tiles that touch the upper triangle of this band
  const int tx_first = (EPI == EPI_UPPER) ? (int)(row0 / TTW) : 0;
  const int tx0 = tx_first + blockIdx.y * g.tiles_per_cta;
  if (tx0 >= ntiles) return;                                   // block-uniform
  const int ntx = min(ntiles, tx0 + g.tiles_per_cta);

  // ---- per-thread invariants of the band
  FastCtx<R> c;
#pragma unroll
  for (int k = 0; k < FastCtx<R>::FILL_ITERS; ++k) {
    const int idx = tid + k * TTHREADS;
    const int r = idx / (G::IW / 4), q = idx - r * (G::IW / 4);
    const bool on = idx < G::IH * (G::IW / 4);
    c.fill_smem[k] = on ? r * G::IW + 4 * q : -1;
    c.fill_gofs[k] = on ? (int)(r * g.lda) + 4 * q : 0;      // < 40 * lda: fits 32 bits
  }
  {
    const bool von = tid < G::IW * (TTH / VSTRIP);
    const int vc = tid % G::IW, vr0 = (tid / G::IW) * VSTRIP;
    c.v_in = von ? vr0 * G::IW + vc : -1;
    c.v_mid = vr0 * G::MP + vc;
    const bool hon = tid < TTH * (TTW / HSTRIP);
    const int hr = tid % TTH;
    c.h_c0 = (tid / TTH) * HSTRIP;
    c.h_mid = hon ? hr * G::MP + c.h_c0 : -1;
    const int64_t i = row0 + hr;
    const bool row_ok = hon && i < g.row_end;
    const int64_t io = i - g.out_row_base;
    c.cut_i = (EPI == EPI_THRSYM && row_ok) ? g.m[i] * g.p : 0.0f;
    c.y_row = (row_ok && g.y) ? g.y + io * g.ldy : nullptr;
    c.hi_row = (row_ok && g.hi) ? g.hi + io * g.ldh : nullptr;
    c.lo_row = (row_ok && g.hi) ? g.lo + io * g.ldh : nullptr;
    c.out_row = (row_ok && g.out) ? g.out + io * g.ldo : nullptr;
  }
  const float* band_src = g.a + (row0 - R - g.in_row_base) * g.lda - R;   // + col0 per tile

  // tile_is_fast(row0, tx * TTW) for every tile of the band, reduced to four 32-bit compares per
  // tile (the per-tile form -- a dozen 64-bit compares evaluated twice per tile by every thread --
  // was a sixth of the kernel's instructions): the band-level
  // conditions once, the first/last tile with a complete halo, and the run of tiles whose halo'd
  // footprint meets the diagonal.
  const bool band_fast = (row0 >= R) && (row0 + TTH + R <= g.n) && (row0 + TTH <= g.row_end) &&
                         ((g.lda & 3) == 0) && ((reinterpret_cast<uintptr_t>(g.a) & 15) == 0);
  const int tx_fast_max = (g.n >= R + TTW) ? (int)((g.n - R) / TTW) - 1 : -1;   // col0 + TTW + R <= n
  const int64_t dq = row0 - TTW - 2 * R, dp = row0 + TTH + 2 * R;
  const int diag_lo = dq < 0 ? 0 : (int)(dq / TTW) + 1;     // first tile with col0 > row0 - TTW - 2R
  const int diag_hi = (int)((dp - 1) / TTW);                 // last tile with col0 < row0 + TTH + 2R
  auto is_fast = [&](int tx) {
    return band_fast && tx >= 1 && tx <= tx_fast_max && (tx < diag_lo || tx > diag_hi);
  };

  auto stage = [&](int tx, float* buf) {
    const int64_t col0 = (int64_t)tx * TTW;
    if (is_fast(tx)) fast_fill<R>(c, band_src + col0, buf);
    else tile_fill<R>(g, row0, col0, buf);
  };
  stage(tx0, in0);
  cp_async_commit();
  for (int tx = tx0; tx < ntx; ++tx) {
    float* cur = ((tx - tx0) & 1) ? in1 : in0;
    float* nxt = ((tx - tx0) & 1) ? in0 : in1;
    if (tx + 1 < ntx) {
      stage(tx + 1, nxt);                                     // `nxt` was last read two tiles ago
      cp_async_commit();
      cp_async_wait<1>();                                     // tile tx has landed
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();   // tile tx visible; everybody is out of the previous horizontal pass
    const int64_t col0 = (int64_t)tx * TTW;
    if (is_fast(tx)) fast_compute<R, EPI>(g, c, w, col0, cur, mid, rmax);
    else tile_compute<R, EPI>(g, w, row0, col0, cur, mid, rmax);
  }
  if (EPI == EPI_STATS || EPI == EPI_UPPER) {
    if (threadIdx.x < TTH * (TTW / HSTRIP)) part[threadIdx.x / TTH][threadIdx.x % TTH] = rmax;
    __syncthreads();
    if (threadIdx.x < TTH) {
      float v = 0.0f;
#pragma unroll
      for (int s8 = 0; s8 < TTW / HSTRIP; ++s8) v = fmaxf(v, part[s8][threadIdx.x]);
      const int64_t i = row0 + threadIdx.x;
      if (i < g.row_end) {
        if (EPI == EPI_STATS && gridDim.y == 1) g.rowmax_out[i] = v;
        else atomic_max_nonneg(g.rowmax_out + i, v);   // caller zero-fills
      }
    }
  }
}

// ------------------------------------------------------------------ no blur (sigma == 0)
template <int EPI>
__global__ void k_noblur(const BlurArgs g) {
  const int64_t i = g.row_begin + blockIdx.x;
  float vmax = 0.0f;
  for (int64_t j = (int64_t)blockIdx.y * blockDim.x + threadIdx.x; j < g.n;
       j += (int64_t)gridDim.y * blockDim.x) {
    const float v = blur_epilogue<EPI>(g, i, j, load_input(g, i, j));
    vmax = fmaxf(vmax, v);
  }
  if (EPI != EPI_THRSYM && g.rowmax_out) {
    vmax = warp_max(fmaxf(vmax, 0.0f));
    if ((threadIdx.x & 31) == 0) atomic_max_nonneg(g.rowmax_out + i, vmax);
  }
}

// ------------------------------------------------------------------ symmetric pass 2
// Element-wise threshold + symmetrize on the stored upper half of B (EPI_UPPER), 64 x 64 tiles
// with TI <= TJ: y = rule(b, m_i, m_j) is symmetric in (i, j), so the tile is written directly and,
// for TI < TJ, once more transposed (through shared memory, 128-byte row segments of the planes).
// A diagonal tile (TI == TJ) evaluates its lower half from the stored upper elements, so every pair
// (i, j), (j, i) comes from the one b[min(i, j), max(i, j)] and Y is bitwise symmetric.
constexpr int UT = 64;

struct UpperArgs {
  const float* b;
  int64_t n, ldb;
  const float* m;
  float p, mult;
  int binarize, preserve_diag, sym_type;
  float* y;
  int64_t ldy;
  __half* hi;
  __half* lo;
  int64_t ldh;
  int tiles;                 // ceil(n / UT)
};

__device__ __forceinline__ void store_y4(const UpperArgs& g, int64_t i, int64_t j, const float (&y)[4],
                                         bool full4) {
  if (full4) {
    if (g.y) *reinterpret_cast<float4*>(g.y + i * g.ldy + j) = make_float4(y[0], y[1], y[2], y[3]);
    if (g.hi) {
      const __half2 h0 = __floats2half2_rn(y[0], y[1]), h1 = __floats2half2_rn(y[2], y[3]);
      *reinterpret_cast<uint2*>(g.hi + i * g.ldh + j) =
          make_uint2(*reinterpret_cast<const uint32_t*>(&h0), *reinterpret_cast<const uint32_t*>(&h1));
      if (g.lo) {          // a single-MMA Diffuse reads only the hi plane
        const float2 f0 = __half22float2(h0), f1 = __half22float2(h1);
        const __half2 l0 = __floats2half2_rn(y[0] - f0.x, y[1] - f0.y);
        const __half2 l1 = __floats2half2_rn(y[2] - f1.x, y[3] - f1.y);
        *reinterpret_cast<uint2*>(g.lo + i * g.ldh + j) =
            make_uint2(*reinterpret_cast<const uint32_t*>(&l0), *reinterpret_cast<const uint32_t*>(&l1));
      }
    }
  } else {
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      if (j + t >= g.n) continue;
      if (g.y) g.y[i * g.ldy + j + t] = y[t];
      if (g.hi) {
        __half h, l;
        split_half(y[t], h, l);
        g.hi[i * g.ldh + j + t] = h;
        if (g.lo) g.lo[i * g.ldh + j + t] = l;
      }
    }
  }
}

// (A run-based variant -- one CTA per tile row x 8 tile columns, the next tile's loads prefetched
// into registers -- was slower than this one-tile-per-CTA form: the extra registers cost more
// occupancy than the prefetch wins.  The limiter is DRAM page locality of the 128-byte transposed
// row segments.)
__global__ void __launch_bounds__(256)
k_thrsym_upper(const UpperArgs g) {
  __shared__ float tile[UT][UT + 1];
  // linear index -> (TI, TJ) with TI <= TJ: row TI of the triangle starts at TI*T - TI(TI-1)/2
  const int64_t T = g.tiles, idx = blockIdx.x;
  int64_t ti = (int64_t)(((2.0 * T + 1.0) - sqrt((2.0 * T + 1.0) * (2.0 * T + 1.0) - 8.0 * (double)idx)) * 0.5);
  while (ti > 0 && ti * T - ti * (ti - 1) / 2 > idx) --ti;
  while ((ti + 1) * T - (ti + 1) * ti / 2 <= idx) ++ti;
  const int64_t tj = ti + (idx - (ti * T - ti * (ti - 1) / 2));
  const int64_t row0 = ti * UT, col0 = tj * UT;
  const bool diag_tile = (ti == tj);
  const int tr = threadIdx.x >> 4, tc = (threadIdx.x & 15) * 4;
  const int64_t j = col0 + tc;
  const bool full4 = (j + 3 < g.n);
  float mj[4] = {0.0f, 0.0f, 0.0f, 0.0f};
  if (full4) {
    const float4 v = *reinterpret_cast<const float4*>(g.m + j);
    mj[0] = v.x; mj[1] = v.y; mj[2] = v.z; mj[3] = v.w;
  } else {
#pragma unroll
    for (int t = 0; t < 4; ++t) mj[t] = (j + t < g.n) ? g.m[j + t] : 0.0f;
  }
#pragma unroll
  for (int t = 0; t < 4; ++t) mj[t] *= g.p;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int r = tr + 16 * k;
    const int64_t i = row0 + r;
    float y[4] = {0.0f, 0.0f, 0.0f, 0.0f};
    if (i < g.n) {
      float bv[4] = {0.0f, 0.0f, 0.0f, 0.0f};
      if (full4) {
        const float4 v = ld_stream4(g.b + i * g.ldb + j);
        bv[0] = v.x; bv[1] = v.y; bv[2] = v.z; bv[3] = v.w;
      } else {
#pragma unroll
        for (int t = 0; t < 4; ++t) bv[t] = (j + t < g.n) ? g.b[i * g.ldb + j + t] : 0.0f;
      }
      if (diag_tile) {
        // below the diagonal, the mirror of the upper element: the computed blur is not bitwise
        // symmetric, and Y(i, j) must equal Y(j, i) = rule(b[j, i], m_j, m_i) exactly
#pragma unroll
        for (int t = 0; t < 4; ++t)
          if (j + t < i) bv[t] = g.b[(j + t) * g.ldb + i];
      }
      const float cut_i = g.m[i] * g.p;
#pragma unroll
      for (int t = 0; t < 4; ++t) {
        const float x = bv[t];
        const float keep = g.binarize ? 1.0f : x;
        const float small = x * g.mult;
        const float t1 = (x < cut_i) ? small : keep;
        const float t2 = (x < mj[t]) ? small : keep;
        y[t] = (g.sym_type == SC_SYMMETRIZE_MAX) ? fmaxf(t1, t2) : 0.5f * (t1 + t2);
        if (g.preserve_diag && diag_tile && i == j + t) y[t] = 1.0f;      // refinement.py:208-209
      }
      store_y4(g, i, j, y, full4);
    }
    if (!diag_tile) {
      tile[r][tc] = y[0]; tile[r][tc + 1] = y[1]; tile[r][tc + 2] = y[2]; tile[r][tc + 3] = y[3];
    }
  }
  if (diag_tile) return;                                       // block-uniform
  __syncthreads();
  // transposed write: row (col0 + r') of Y, columns row0 + 4 c' .. +3
  const int64_t jm = row0 + tc;
  const bool full4m = (jm + 3 < g.n);
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int r = tr + 16 * k;
    const int64_t i = col0 + r;
    if (i >= g.n) continue;
    const float y[4] = {tile[tc][r], tile[tc + 1][r], tile[tc + 2][r], tile[tc + 3][r]};
    store_y4(g, i, jm, y, full4m);
  }
}

static int make_weights(double sigma, BlurWeights& bw, int& radius) {
  // scipy _gaussian_kernel1d: radius = int(truncate*sigma + 0.5), exp(-x^2/(2 sigma^2)) / sum
  radius = (int)(4.0 * sigma + 0.5);
  if (radius > kMaxRadius) return 1;
  double w[2 * kMaxRadius + 1], sum = 0.0;
  for (int k = -radius; k <= radius; ++k) {
    w[k + radius] = std::exp(-0.5 / (sigma * sigma) * (double)k * (double)k);
    sum += w[k + radius];
  }
  for (int k = 0; k <= 2 * radius; ++k) bw.w[k] = (float)(w[k] / sum);
  return 0;
}

static int check_outputs(const BlurArgs& g) {
  SC_REQUIRE(!g.y || vec_ok_f32(g.y, g.ldy), "blur: `y` needs a 16-byte aligned base and ldy %% 4 == 0");
  SC_REQUIRE(!g.out || vec_ok_f32(g.out, g.ldo), "blur: `out` needs a 16-byte aligned base and ldo %% 4 == 0");
  SC_REQUIRE(!g.hi || (vec_ok_f16(g.hi, g.ldh) && vec_ok_f16(g.lo, g.ldh)),
             "blur: the fp16 planes need 16-byte aligned bases and ldh %% 8 == 0");
  SC_REQUIRE(!g.m || aligned16(g.m), "blur: the row-maximum vector needs a 16-byte aligned base");
  return 0;
}

template <int EPI>
static int launch_blur(const sc_context* ctx, BlurArgs& g, double sigma, cudaStream_t st) {
  if (int rc = check_outputs(g)) return rc;
  if (sigma <= 1e-15) {     // scipy: "if sigma > 1e-15 ... else output[...] = input[...]"
    const unsigned gy = (unsigned)std::min<int64_t>((g.n + 1023) / 1024, 64);
    k_noblur<EPI><<<dim3((unsigned)(g.row_end - g.row_begin), gy), 256, 0, st>>>(g); sc::launched();
    SC_LAUNCH_CHECK();
    return 0;
  }
  BlurWeights bw;
  int radius;
  SC_REQUIRE(make_weights(sigma, bw, radius) == 0,
             "sc_gaussian_blur: sigma %g needs radius > %d", sigma, kMaxRadius);
  g.radius = radius;
  if (radius == 0) {        // a single tap of weight 1
    const unsigned gy = (unsigned)std::min<int64_t>((g.n + 1023) / 1024, 64);
    k_noblur<EPI><<<dim3((unsigned)(g.row_end - g.row_begin), gy), 256, 0, st>>>(g); sc::launched();
    SC_LAUNCH_CHECK();
    return 0;
  }
  if (radius == 4) {
    constexpr int R = 4;
    const size_t smem = sizeof(float) * (2 * (TTH + 2 * R) * (TTW + 2 * R) +
                                         TTH * (TTW + 2 * R + 1));
    auto kband = k_blur_band<R, EPI>;
    SC_CUDA(cudaFuncSetAttribute(kband, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const int ntiles = (int)((g.n + TTW - 1) / TTW);
    static int tpc_env = -1;
    if (tpc_env < 0) {
      const char* e = getenv("SCB_BLUR_TILES_PER_CTA");
      tpc_env = e ? atoi(e) : 0;
    }
    // the upper-triangle pass uses short runs of 2 tiles (they balance the ragged band ends of the
    // triangle); the two-pass kernels sweep runs of 4
    g.tiles_per_cta = tpc_env > 0 ? tpc_env : (EPI == EPI_UPPER ? 2 : 4);
    if (g.tiles_per_cta > ntiles) g.tiles_per_cta = ntiles;
    const unsigned gy = (unsigned)((ntiles + g.tiles_per_cta - 1) / g.tiles_per_cta);
    const dim3 grid((unsigned)((g.row_end - g.row_begin + TTH - 1) / TTH), gy);
    kband<<<grid, TTHREADS, smem, st>>>(g, bw);
    sc::launched();
    SC_LAUNCH_CHECK();
    return 0;
  }
  const size_t smem = sizeof(float) * ((size_t)(GTH + 2 * radius) * (GTW + 2 * radius) +
                                       (size_t)GTH * (GTW + 2 * radius));
  SC_REQUIRE(smem <= ctx->smem_optin, "sc_gaussian_blur: tile needs %zu B of shared memory", smem);
  auto kern = k_blur_generic<EPI>;
  SC_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const dim3 grid((unsigned)((g.n + GTW - 1) / GTW),
                  (unsigned)((g.row_end - g.row_begin + GTH - 1) / GTH));
  kern<<<grid, GTHREADS, smem, st>>>(g, bw); sc::launched();
  SC_LAUNCH_CHECK();
  return 0;
}

}  // namespace sc

using namespace sc;

static void whole_matrix(BlurArgs& g) {
  g.row_begin = 0; g.row_end = g.n; g.in_row_base = 0; g.out_row_base = 0;
}

static int check_block(int64_t n, int64_t in_row_base, int64_t in_rows, int64_t row_begin,
                       int64_t row_end, int radius) {
  SC_REQUIRE(0 <= row_begin && row_begin < row_end && row_end <= n, "blur block: bad row range");
  SC_REQUIRE((row_end - row_begin) % 32 == 0 || row_end == n,
             "blur block: the row count must be a multiple of 32 unless the block ends the matrix");
  // every input row the block can touch (after reflection at the matrix edges) must be resident
  const int64_t need_lo = row_begin - radius < 0 ? 0 : row_begin - radius;
  const int64_t need_hi = row_end + radius > n ? n : row_end + radius;
  SC_REQUIRE(in_row_base <= need_lo && in_row_base + in_rows >= need_hi,
             "blur block: input rows [%lld, %lld) do not cover the halo [%lld, %lld)",
             (long long)in_row_base, (long long)(in_row_base + in_rows), (long long)need_lo,
             (long long)need_hi);
  return 0;
}

extern "C" int sc_gaussian_blur(sc_context* ctx, const float* a, int64_t n, int64_t lda,
                                const float* diag_override, double sigma, float* out,
                                int64_t ldo, float* rowmax_out, void* stream) {
  SC_REQUIRE(ctx && a && n > 0, "sc_gaussian_blur: bad arguments");
  SC_REQUIRE(out || rowmax_out, "sc_gaussian_blur: nothing to compute");
  SC_REQUIRE(n <= 65535LL * 32, "sc_gaussian_blur: n too large for the tile grid");
  BlurArgs g = {};
  g.a = a; g.n = n; g.lda = lda; g.diag = diag_override;
  g.out = out; g.ldo = ldo; g.rowmax_out = rowmax_out;
  whole_matrix(g);
  if (out) return launch_blur<EPI_STORE>(ctx, g, sigma, as_stream(stream));
  return launch_blur<EPI_STATS>(ctx, g, sigma, as_stream(stream));
}

// statistics pass with the diagonal read as zero (RowWiseThreshold preserve_diagonal)
extern "C" int sc_gaussian_blur_rowmax(sc_context* ctx, const float* a, int64_t n, int64_t lda,
                                       const float* diag_override, double sigma,
                                       int zero_diagonal, float* rowmax_out, void* stream) {
  SC_REQUIRE(ctx && a && rowmax_out && n > 0, "sc_gaussian_blur_rowmax: bad arguments");
  BlurArgs g = {};
  g.a = a; g.n = n; g.lda = lda; g.diag = diag_override;
  g.rowmax_out = rowmax_out; g.stats_zero_diag = zero_diagonal;
  whole_matrix(g);
  return launch_blur<EPI_STATS>(ctx, g, sigma, as_stream(stream));
}

extern "C" int sc_blur_threshold_symmetrize(sc_context* ctx, const float* a, int64_t n,
                                            int64_t lda, const float* diag_override,
                                            double sigma, const float* rowmax, double p,
                                            double mult, int binarize, int preserve_diagonal,
                                            int sym_type, float* y, int64_t ldy, void* hi,
                                            void* lo, int64_t ldh, void* stream) {
  SC_REQUIRE(ctx && a && rowmax && n > 0, "sc_blur_threshold_symmetrize: bad arguments");
  SC_REQUIRE(y || (hi && lo), "sc_blur_threshold_symmetrize: no output given");
  SC_REQUIRE((hi == nullptr) == (lo == nullptr), "hi/lo must come together");
  SC_REQUIRE(sym_type == SC_SYMMETRIZE_MAX || sym_type == SC_SYMMETRIZE_AVERAGE,
             "Unsupported symmetrize_type.");
  BlurArgs g = {};
  g.a = a; g.n = n; g.lda = lda; g.diag = diag_override;
  g.m = rowmax; g.p = (float)p; g.mult = (float)mult; g.binarize = binarize;
  g.preserve_diag = preserve_diagonal; g.sym_type = sym_type;
  g.y = y; g.ldy = ldy; g.hi = (__half*)hi; g.lo = (__half*)lo; g.ldh = ldh;
  whole_matrix(g);
  return launch_blur<EPI_THRSYM>(ctx, g, sigma, as_stream(stream));
}

// ---- row-block variants (multi-GPU row sharding, SURVEY.md 8(e)): `a` holds global rows
// [in_row_base, in_row_base + in_rows) -- the owned rows plus the blur halo, recomputed locally
// from the embeddings instead of exchanged; outputs cover global rows [row_begin, row_end) and are
// written to buffers whose row 0 is global row `row_begin`.  diag_override / rowmax vectors are
// indexed by global row.
extern "C" int sc_gaussian_blur_rowmax_block(sc_context* ctx, const float* a, int64_t n,
                                             int64_t lda, int64_t in_row_base, int64_t in_rows,
                                             int64_t row_begin, int64_t row_end,
                                             const float* diag_override, double sigma,
                                             int zero_diagonal, float* rowmax_out,
                                             void* stream) {
  SC_REQUIRE(ctx && a && rowmax_out && n > 0, "sc_gaussian_blur_rowmax_block: bad arguments");
  const int radius = sigma > 1e-15 ? (int)(4.0 * sigma + 0.5) : 0;
  if (int rc = check_block(n, in_row_base, in_rows, row_begin, row_end, radius)) return rc;
  BlurArgs g = {};
  g.a = a; g.n = n; g.lda = lda; g.diag = diag_override;
  g.rowmax_out = rowmax_out; g.stats_zero_diag = zero_diagonal;
  g.row_begin = row_begin; g.row_end = row_end; g.in_row_base = in_row_base;
  g.out_row_base = row_begin;
  return launch_blur<EPI_STATS>(ctx, g, sigma, as_stream(stream));
}

extern "C" int sc_blur_threshold_symmetrize_block(
    sc_context* ctx, const float* a, int64_t n, int64_t lda, int64_t in_row_base, int64_t in_rows,
    int64_t row_begin, int64_t row_end, const float* diag_override, double sigma,
    const float* rowmax, double p, double mult, int binarize, int preserve_diagonal, int sym_type,
    float* y, int64_t ldy, void* hi, void* lo, int64_t ldh, void* stream) {
  SC_REQUIRE(ctx && a && rowmax && n > 0, "sc_blur_threshold_symmetrize_block: bad arguments");
  SC_REQUIRE(y || (hi && lo), "sc_blur_threshold_symmetrize_block: no output given");
  SC_REQUIRE((hi == nullptr) == (lo == nullptr), "hi/lo must come together");
  SC_REQUIRE(sym_type == SC_SYMMETRIZE_MAX || sym_type == SC_SYMMETRIZE_AVERAGE,
             "Unsupported symmetrize_type.");
  const int radius = sigma > 1e-15 ? (int)(4.0 * sigma + 0.5) : 0;
  if (int rc = check_block(n, in_row_base, in_rows, row_begin, row_end, radius)) return rc;
  BlurArgs g = {};
  g.a = a; g.n = n; g.lda = lda; g.diag = diag_override;
  g.m = rowmax; g.p = (float)p; g.mult = (float)mult; g.binarize = binarize;
  g.preserve_diag = preserve_diagonal; g.sym_type = sym_type;
  g.y = y; g.ldy = ldy; g.hi = (__half*)hi; g.lo = (__half*)lo; g.ldh = ldh;
  g.row_begin = row_begin; g.row_end = row_end; g.in_row_base = in_row_base;
  g.out_row_base = row_begin;
  return launch_blur<EPI_THRSYM>(ctx, g, sigma, as_stream(stream));
}

// ---- symmetric whole-matrix pair (single-GPU hot path).  Pass 1: b_out <- the tiles of blur(a)
// that touch the upper triangle (the rest of b_out is left untouched), m_out[i] <- max_j blur(a)[i,j]
// assembled from the row AND column maxima of those tiles.  Requires a symmetric `a` and sigma
// with radius 4 (sigma in [0.875, 1.125), every BASELINE configuration); the caller falls back to
// sc_gaussian_blur_rowmax + sc_blur_threshold_symmetrize otherwise.
extern "C" int sc_blur_upper_rowmax(sc_context* ctx, const float* a, int64_t n, int64_t lda,
                                    const float* diag_override, double sigma, int zero_diagonal,
                                    float* b_out, int64_t ldb, float* rowmax_out, void* stream) {
  SC_REQUIRE(ctx && a && b_out && rowmax_out && n > 0, "sc_blur_upper_rowmax: bad arguments");
  SC_REQUIRE(sigma > 1e-15 && (int)(4.0 * sigma + 0.5) == 4,
             "sc_blur_upper_rowmax: the symmetric pass is built for radius 4 (sigma ~ 1)");
  SC_REQUIRE(n <= 65535LL * 32, "sc_blur_upper_rowmax: n too large for the tile grid");
  BlurArgs g = {};
  g.a = a; g.n = n; g.lda = lda; g.diag = diag_override;
  g.out = b_out; g.ldo = ldb; g.rowmax_out = rowmax_out; g.stats_zero_diag = zero_diagonal;
  whole_matrix(g);
  SC_CUDA(cudaMemsetAsync(rowmax_out, 0, sizeof(float) * n, as_stream(stream)));
  return launch_blur<EPI_UPPER>(ctx, g, sigma, as_stream(stream));
}

// Pass 2: y / planes <- sym(thr(b, m_i), thr(b, m_j)) for the WHOLE matrix from the upper tiles of b.
extern "C" int sc_threshold_symmetrize_upper(sc_context* ctx, const float* b, int64_t n, int64_t ldb,
                                             const float* rowmax, double p, double mult,
                                             int binarize, int preserve_diagonal, int sym_type,
                                             float* y, int64_t ldy, void* hi, void* lo, int64_t ldh,
                                             void* stream) {
  SC_REQUIRE(ctx && b && rowmax && n > 0, "sc_threshold_symmetrize_upper: bad arguments");
  SC_REQUIRE(y || hi, "sc_threshold_symmetrize_upper: no output given");
  SC_REQUIRE(hi || !lo, "sc_threshold_symmetrize_upper: a lo plane needs its hi plane");
  SC_REQUIRE(sym_type == SC_SYMMETRIZE_MAX || sym_type == SC_SYMMETRIZE_AVERAGE,
             "Unsupported symmetrize_type.");
  SC_REQUIRE(vec_ok_f32(b, ldb) && aligned16(rowmax), "sc_threshold_symmetrize_upper: `b` / rowmax alignment");
  UpperArgs g = {};
  g.b = b; g.n = n; g.ldb = ldb; g.m = rowmax; g.p = (float)p; g.mult = (float)mult;
  g.binarize = binarize; g.preserve_diag = preserve_diagonal; g.sym_type = sym_type;
  g.y = y; g.ldy = ldy; g.hi = (__half*)hi; g.lo = (__half*)lo; g.ldh = ldh;
  SC_REQUIRE(!y || vec_ok_f32(y, ldy), "sc_threshold_symmetrize_upper: `y` alignment");
  SC_REQUIRE(!hi || (vec_ok_f16(hi, ldh) && (!lo || vec_ok_f16(lo, ldh))), "sc_threshold_symmetrize_upper: plane alignment");
  g.tiles = (int)((n + UT - 1) / UT);
  const int64_t pairs = (int64_t)g.tiles * (g.tiles + 1) / 2;
  SC_REQUIRE(pairs < (1LL << 31), "sc_threshold_symmetrize_upper: n too large for the tile grid");
  k_thrsym_upper<<<(unsigned)pairs, 256, 0, as_stream(stream)>>>(g); sc::launched();
  SC_LAUNCH_CHECK();
  return 0;
}
