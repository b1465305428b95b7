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
// Whole-matrix, symmetric input goes one step further.  The single-GPU hot path (k_blur_pair) blurs
// only the upper triangle, twice: pass 1 keeps the row and column maxima, pass 2 writes Y and its
// mirror -- 2 + 2 + 2 B per element of the matrix for the hi plane, no B in memory.  The stored-B
// form stays for callers that pass a B (EPI_UPPER + k_thrsym_upper): B = blur(A) is symmetric,
// so only the tiles that touch the upper triangle are blurred -- once.  Pass 1 reads half of A, stores that half of B and folds both the row maxima
// and the column maxima of every tile into m (m_i = max_j B_ij needs the lower half only through
// B_ji).  Pass 2 is element-wise on the stored half of B and writes Y(i,j) and Y(j,i) (transposed
// through shared memory).  HBM traffic 2 + 2 + 2 + 2 = 8 B per element of the matrix when only the
// hi plane of Y is written (a single-MMA Diffuse follows; 10 B with the lo plane, the contract
// figure is 12) and half the filter arithmetic of the two-pass form; both kernels were
// issue-bound, not bandwidth-bound.
//
// Kernels: k_blur_band<4, EPI> (compile-time radius 4 = sigma ~ 1, the configuration every
// BASELINE config uses: register sliding windows, cp.async pipeline), k_blur_generic<EPI>
// (run-time radius <= 64), k_noblur<EPI> (radius 0 and sigma <= 1e-15), k_thrsym_upper and
// k_blur_pair<PASS2> (radius 4).
#include "common.cuh"

#include <cstdlib>

namespace sc {

constexpr int kMaxRadius = 64;

// The threshold/symmetrize rule and the Y outputs, shared by every kernel that writes Y.
struct RuleArgs {
  const float* m;          // row maxima of the blurred matrix
  float p, mult;
  int binarize, preserve_diag, sym_type;
  float* y;                // fp32 Y (optional)
  int64_t ldy;
  __half* hi;              // split fp16 planes of Y (optional; lo optional even with hi)
  __half* lo;
  int64_t ldh;
};

struct BlurArgs {
  const float* a;          // rows [in_row_base, ...) of the global n x n matrix
  int64_t n, lda;
  // Row block (multi-GPU row sharding; the single-GPU case is 0, n, 0, 0): outputs are produced
  // for global rows [row_begin, row_end); output buffers start at global row out_row_base.
  // Vectors (diag, m, rowmax_out) are indexed by GLOBAL row/column.
  int64_t row_begin, row_end, in_row_base, out_row_base;
  const float* diag;       // optional replacement of a[i][i]
  int radius;
  float* out;              // EPI_STORE / EPI_UPPER
  int64_t ldo;
  float* rowmax_out;       // EPI_STORE (optional) / EPI_STATS / EPI_UPPER
  int stats_zero_diag;
  int tiles_per_cta;       // column tiles swept by one CTA of k_blur_band (cp.async pipeline)
  RuleArgs r;              // EPI_THRSYM
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

// y = sym(thr(b, m_i), thr(b, m_j)), thr(b, m) = b < m p ? b mult : (binarize ? 1 : b)
// (SURVEY.md A.3).  Every caller forms the cuts as the fp32 products m_i * p and m_j * p.
// `diag` marks the element (i, i), which preserve_diagonal sets to 1 (refinement.py:208-209).
__device__ __forceinline__ float thrsym_rule(const RuleArgs& r, float b, float cut_i, float cut_j,
                                             bool diag) {
  const float keep = r.binarize ? 1.0f : b;
  const float small = b * r.mult;
  const float t1 = (b < cut_i) ? small : keep;
  const float t2 = (b < cut_j) ? small : keep;
  const float y = (r.sym_type == SC_SYMMETRIZE_MAX) ? fmaxf(t1, t2) : 0.5f * (t1 + t2);
  return (diag && r.preserve_diag) ? 1.0f : y;
}

// dst[0 .. N) <- w[] (N 32-bit words, dst aligned to the store): 128-bit stores, or one 64-bit store
// for N = 2.  Written as PTX because the compiler, given the same stores as C++, merged the
// identical epilogues of the edge and interior tiles of k_blur_band and split the first 128-bit
// store of every run into four 32-bit ones, which made the kernels 1.5x slower.
template <int N>
__device__ __forceinline__ void store_words(void* dst, const uint32_t (&w)[N]) {
  static_assert(N == 2 || N % 4 == 0, "64-bit or 128-bit stores");
  if constexpr (N == 2) {
    asm volatile("st.global.v2.b32 [%0], {%1, %2};" ::"l"(dst), "r"(w[0]), "r"(w[1]) : "memory");
  } else {
#pragma unroll
    for (int q = 0; q < N / 4; ++q)
      asm volatile("st.global.v4.b32 [%0], {%1, %2, %3, %4};"
                   ::"l"(static_cast<uint32_t*>(dst) + 4 * q), "r"(w[4 * q]), "r"(w[4 * q + 1]),
                     "r"(w[4 * q + 2]), "r"(w[4 * q + 3])
                   : "memory");
  }
}

template <int N>
__device__ __forceinline__ void store_floats(float* dst, const float (&v)[N]) {
  uint32_t w[N];
#pragma unroll
  for (int t = 0; t < N; ++t) w[t] = __float_as_uint(v[t]);
  store_words<N>(dst, w);
}

// Y(io, j0 .. j0 + W - 1) <- y[]: fp32 and/or the split planes hi = fp16(y), lo = fp16(y - hi).
// A complete run (`full`) goes out as vector stores (W = 16: two 128-bit stores per plane, W = 4:
// one 64-bit store); otherwise element by element, stopping at column n.
template <int W>
__device__ __forceinline__ void store_y(const RuleArgs& r, int64_t io, int64_t j0,
                                        const float (&y)[W], bool full, int64_t n) {
  static_assert(W == 1 || W == 4 || W == 16, "runs of 1, 4 or 16 values");
  if constexpr (W > 1) {
    if (full) {
      if (r.y) store_floats<W>(r.y + io * r.ldy + j0, y);
      if (r.hi) {
        uint32_t hw[W / 2], lw[W / 2];
#pragma unroll
        for (int q = 0; q < W / 2; ++q) {
          const __half2 h = __floats2half2_rn(y[2 * q], y[2 * q + 1]);
          const float2 f = __half22float2(h);
          const __half2 l = __floats2half2_rn(y[2 * q] - f.x, y[2 * q + 1] - f.y);
          hw[q] = *reinterpret_cast<const uint32_t*>(&h);
          lw[q] = *reinterpret_cast<const uint32_t*>(&l);
        }
        store_words<W / 2>(r.hi + io * r.ldh + j0, hw);
        if (r.lo) store_words<W / 2>(r.lo + io * r.ldh + j0, lw);
      }
      return;
    }
  }
#pragma unroll
  for (int t = 0; t < W; ++t) {
    if (!full && j0 + t >= n) continue;
    if (r.y) r.y[io * r.ldy + j0 + t] = y[t];
    if (r.hi) {
      __half h, l;
      split_half(y[t], h, l);
      r.hi[io * r.ldh + j0 + t] = h;
      if (r.lo) r.lo[io * r.ldh + j0 + t] = l;
    }
  }
}

// One output element (i, j) with blurred value b.  Returns the value that takes part in the
// row maximum (EPI_STORE / EPI_STATS).
template <int EPI>
__device__ __forceinline__ float blur_epilogue(const BlurArgs& g, int64_t i, int64_t j, float b) {
  static_assert(EPI != EPI_UPPER, "the symmetric pass runs on k_blur_band only");
  if (EPI == EPI_STORE) {
    g.out[(i - g.out_row_base) * g.ldo + j] = b;
    return b;
  } else if (EPI == EPI_STATS) {
    return (g.stats_zero_diag && i == j) ? 0.0f : b;   // RowWiseThreshold preserve_diagonal
  } else {
    const float y[1] = {thrsym_rule(g.r, b, g.r.m[i] * g.r.p, g.r.m[j] * g.r.p, i == j)};
    store_y<1>(g.r, i - g.out_row_base, j, y, true, g.n);
    return y[0];
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

// The 16 blurred values b[] of row i, columns j0 .. j0 + 15.  Edge tiles (EDGE) check the columns
// against n and the diagonal; the interior tiles of the fast path are complete and off-diagonal,
// and all 32 lanes of each horizontal-pass warp reach the epilogue together.  `out_row` is row i of
// B for the fast path's stores (FastCtx).
template <int EPI, bool EDGE>
__device__ __forceinline__ void epilogue16(const BlurArgs& g, int64_t i, int64_t j0,
                                           const float (&b)[HSTRIP], float& rmax, float* out_row) {
  const bool full = !EDGE || j0 + HSTRIP <= g.n;
  const int64_t io = i - g.out_row_base;
  if (EPI == EPI_STATS || EPI == EPI_UPPER) {
    if (EPI == EPI_UPPER && !EDGE) store_floats<HSTRIP>(out_row + j0, b);
    // EPI_UPPER also stores B and folds the column maxima of the tile into m: by one atomic per
    // element on edge / diagonal tiles (O(N) such tiles out of N^2/4096)
#pragma unroll
    for (int t = 0; t < HSTRIP; ++t) {
      if (!full && j0 + t >= g.n) continue;
      // RowWiseThreshold preserve_diagonal
      const float x = (EDGE && g.stats_zero_diag && i == j0 + t) ? 0.0f : b[t];
      rmax = fmaxf(rmax, x);
      if (EPI == EPI_UPPER && EDGE) {
        g.out[io * g.ldo + j0 + t] = b[t];
        atomic_max_nonneg(g.rowmax_out + j0 + t, fmaxf(x, 0.0f));
      }
    }
    if (EPI == EPI_UPPER && !EDGE) {
      // The lanes of this warp are the tile's 32 rows, each holding the same 16 columns.  The
      // blurred values are non-negative, so their bit patterns order like signed integers and one
      // REDUX.MAX per column reduces across the warp (16 instructions; the shuffle butterfly
      // before it took ~95); lane t keeps column t and issues its atomic.
      const int lane = threadIdx.x & 31;
      float cm = 0.0f;
#pragma unroll
      for (int t = 0; t < HSTRIP; ++t) {
        const int mx = __reduce_max_sync(0xffffffffu, __float_as_int(fmaxf(b[t], 0.0f)));
        if (lane == t) cm = __int_as_float(mx);
      }
      if (lane < HSTRIP) atomic_max_nonneg(g.rowmax_out + j0 + lane, cm);
    }
    return;
  }
  if (EPI == EPI_STORE) {
    float* dst = (EDGE ? g.out + io * g.ldo : out_row) + j0;
    if (full) {
      store_floats<HSTRIP>(dst, b);
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
  // EPI_THRSYM
  const RuleArgs& r = g.r;
  const float cut_i = r.m[i] * r.p;
  // column of the diagonal element within the run (-1: none): one range test instead of sixteen
  // 64-bit compares, which the compiler hoists at a cost of ~30 registers
  const int dcol = (EDGE && i >= j0 && i < j0 + HSTRIP) ? (int)(i - j0) : -1;
  float y[HSTRIP];
#pragma unroll
  for (int q = 0; q < HSTRIP / 4; ++q) {
    float mj[4];
    if (full) {
      const float4 v = *reinterpret_cast<const float4*>(r.m + j0 + 4 * q);   // warp-broadcast
      mj[0] = v.x; mj[1] = v.y; mj[2] = v.z; mj[3] = v.w;
    } else {
#pragma unroll
      for (int t = 0; t < 4; ++t) mj[t] = (j0 + 4 * q + t < g.n) ? r.m[j0 + 4 * q + t] : 0.0f;
    }
#pragma unroll
    for (int t = 0; t < 4; ++t)
      y[4 * q + t] = thrsym_rule(r, b[4 * q + t], cut_i, mj[t] * r.p, dcol == 4 * q + t);
  }
  store_y<HSTRIP>(r, io, j0, y, full, g.n);
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

// One thread's share of the two filter passes of a tile.
struct PassOffsets {
  int v_in, v_mid;             // vertical pass: first input / output element (-1: idle)
  int h_mid, h_r, h_c0;        // horizontal pass: first `mid` element (-1: idle), row, strip column
};

template <int R>
__device__ __forceinline__ PassOffsets pass_offsets(int tid) {
  using G = TileGeom<R>;
  PassOffsets o;
  const int vc = tid % G::IW, vr0 = (tid / G::IW) * VSTRIP;
  o.v_in = tid < G::IW * (TTH / VSTRIP) ? vr0 * G::IW + vc : -1;
  o.v_mid = vr0 * G::MP + vc;
  o.h_r = tid % TTH;
  o.h_c0 = (tid / TTH) * HSTRIP;
  o.h_mid = tid < TTH * (TTW / HSTRIP) ? o.h_r * G::MP + o.h_c0 : -1;
  return o;
}

// ---- fast path: interior, off-diagonal, full tiles (all but O(N) of the N^2/4096 tiles).
// Everything that does not change from tile to tile inside a band is hoisted into FastCtx; the
// edge tiles recompute their pass offsets (cheaper than keeping them live across the edge path).
template <int R>
struct FastCtx {
  static constexpr int FILL_ITERS = (TileGeom<R>::IH * (TileGeom<R>::IW / 4) + TTHREADS - 1) / TTHREADS;
  int fill_smem[FILL_ITERS];   // float offset inside the tile buffer (-1: no copy this round)
  int fill_gofs[FILL_ITERS];   // element offset from the tile's first source element
  PassOffsets pass;
  // row of B this thread stores (EPI_STORE / EPI_UPPER).  With the address formed per tile, the
  // compiler shared it with the edge tiles' epilogue and the upper pass ran 1.15x slower.
  float* out_row;
};

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

template <int R>
__device__ __forceinline__ void fast_fill(const FastCtx<R>& c, const float* src, float* in) {
#pragma unroll
  for (int k = 0; k < FastCtx<R>::FILL_ITERS; ++k)
    if (c.fill_smem[k] >= 0) cp_async16(in + c.fill_smem[k], src + c.fill_gofs[k]);
}

// Vertical pass of one thread: a register window slides down a column of `in` (pitch IW) and
// VSTRIP outputs go down the same column of `mid` (pitch MP).
template <int R>
__device__ __forceinline__ void vertical_pass(const float (&w)[2 * R + 1], const float* in,
                                              float* mid) {
  using G = TileGeom<R>;
  float win[VSTRIP + 2 * R];
#pragma unroll
  for (int k = 0; k < VSTRIP + 2 * R; ++k) win[k] = in[k * G::IW];
#pragma unroll
  for (int o = 0; o < VSTRIP; ++o) {
    float acc = 0.0f;
#pragma unroll
    for (int k = 0; k <= 2 * R; ++k) acc = fmaf(w[k], win[o + k], acc);
    mid[o * G::MP] = acc;
  }
}

// Horizontal pass of one thread: HSTRIP outputs along a row of `mid`.
template <int R>
__device__ __forceinline__ void horizontal_pass(const float (&w)[2 * R + 1], const float* mid,
                                                float (&b)[HSTRIP]) {
  float win[HSTRIP + 2 * R];
#pragma unroll
  for (int k = 0; k < HSTRIP + 2 * R; ++k) win[k] = mid[k];
#pragma unroll
  for (int o = 0; o < HSTRIP; ++o) {
    float acc = 0.0f;
#pragma unroll
    for (int k = 0; k <= 2 * R; ++k) acc = fmaf(w[k], win[o + k], acc);
    b[o] = acc;
  }
}

// Both separable passes + epilogue on a staged tile.  The caller has made `in` visible to the
// whole block (cp.async.wait_group + __syncthreads) and guarantees nobody still reads `mid`.
// Edge tiles (EDGE) patch the diagonal into vector-filled tiles and bounds-check the outputs; the
// fast path does neither.
template <int R, int EPI, bool EDGE>
__device__ __forceinline__ void tile_compute(const BlurArgs& g, const PassOffsets& c,
                                             float* out_row, const float (&w)[2 * R + 1],
                                             int64_t row0, int64_t col0, float* in, float* mid,
                                             float& rmax) {
  using G = TileGeom<R>;
  if (EDGE && g.diag && tile_is_vec<R>(g, row0, col0)) {
    // fused CropDiagonal on the vector path: patch the diagonal elements inside the halo'd tile
    const int64_t lo = (row0 > col0 ? row0 : col0) - R;
    const int64_t hi = ((row0 + TTH < col0 + TTW) ? row0 + TTH : col0 + TTW) + R;
    if (lo < hi) {                                     // block-uniform
      for (int64_t d = lo + threadIdx.x; d < hi; d += TTHREADS)
        in[(d - (row0 - R)) * G::IW + (d - (col0 - R))] = g.diag[d];
      __syncthreads();
    }
  }
  if (c.v_in >= 0) vertical_pass<R>(w, in + c.v_in, mid + c.v_mid);
  __syncthreads();
  if (c.h_mid >= 0) {
    float b[HSTRIP];
    horizontal_pass<R>(w, mid + c.h_mid, b);
    const int64_t i = row0 + c.h_r, j0 = col0 + c.h_c0;
    if (!EDGE || (i < g.row_end && j0 < g.n)) epilogue16<EPI, EDGE>(g, i, j0, b, rmax, out_row);
  }
}

// One CTA per (32-row band, run of `tiles_per_cta` column tiles), 2-deep cp.async pipeline: the
// loads of tile t+1 are in flight while tile t is filtered, so every resident CTA always has
// ~22 KB outstanding (3 CTAs/SM) -- the first, load-then-compute version left HBM idle during
// the two filter passes and ran latency-bound at ~28% of the roofline.
//   EPI_STATS : row maxima of the blurred band, one register per thread, no atomics
//   EPI_THRSYM/EPI_STORE : the band's output rows
//   EPI_UPPER : the column tiles that touch the upper triangle: B stored, row and column maxima
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
  c.pass = pass_offsets<R>(tid);
  c.out_row = ((EPI == EPI_STORE || EPI == EPI_UPPER) && c.pass.h_mid >= 0 && row0 + c.pass.h_r < g.row_end)
                  ? g.out + (row0 + c.pass.h_r - g.out_row_base) * g.ldo : nullptr;
  const float* band_src = g.a + (row0 - R - g.in_row_base) * g.lda - R;   // + col0 per tile

  // tile_is_vec(row0, col0), the output rows inside the block and a halo'd footprint that misses
  // the diagonal, for every tile of the band, reduced to four 32-bit compares per tile (the
  // per-tile form -- a dozen 64-bit compares evaluated twice per tile by every thread -- was a
  // sixth of the kernel's instructions): the band-level conditions once, the first/last tile with
  // a complete halo, and the run of tiles whose halo'd footprint meets the diagonal.
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
    if (is_fast(tx)) tile_compute<R, EPI, false>(g, c.pass, c.out_row, w, row0, col0, cur, mid, rmax);
    else tile_compute<R, EPI, true>(g, pass_offsets<R>(tid), nullptr, w, row0, col0, cur, mid, rmax);
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
  const float* b;            // rows [b_row0, ...) of the upper tiles of B
  int64_t n, ldb, b_row0;
  int64_t pair0;             // linear index of the first tile pair (a row panel starts past 0)
  int tiles;                 // ceil(n / UT)
  RuleArgs r;
};

// (A run-based variant -- one CTA per tile row x 8 tile columns, the next tile's loads prefetched
// into registers -- was slower than this one-tile-per-CTA form: the extra registers cost more
// occupancy than the prefetch wins.  The limiter is DRAM page locality of the 128-byte transposed
// row segments.)
__global__ void __launch_bounds__(256)
k_thrsym_upper(const UpperArgs g) {
  __shared__ float tile[UT][UT + 1];
  const RuleArgs& r = g.r;
  // linear index -> (TI, TJ) with TI <= TJ: row TI of the triangle starts at TI*T - TI(TI-1)/2
  const int64_t T = g.tiles, idx = g.pair0 + blockIdx.x;
  int64_t ti = (int64_t)(((2.0 * T + 1.0) - sqrt((2.0 * T + 1.0) * (2.0 * T + 1.0) - 8.0 * (double)idx)) * 0.5);
  while (ti > 0 && ti * T - ti * (ti - 1) / 2 > idx) --ti;
  while ((ti + 1) * T - (ti + 1) * ti / 2 <= idx) ++ti;
  const int64_t tj = ti + (idx - (ti * T - ti * (ti - 1) / 2));
  const int64_t row0 = ti * UT, col0 = tj * UT;
  const bool diag_tile = (ti == tj);
  const int tr = threadIdx.x >> 4, tc = (threadIdx.x & 15) * 4;
  const int64_t j = col0 + tc;
  const bool full4 = (j + 3 < g.n);
  float cut_j[4] = {0.0f, 0.0f, 0.0f, 0.0f};
  if (full4) {
    const float4 v = *reinterpret_cast<const float4*>(r.m + j);
    cut_j[0] = v.x; cut_j[1] = v.y; cut_j[2] = v.z; cut_j[3] = v.w;
  } else {
#pragma unroll
    for (int t = 0; t < 4; ++t) cut_j[t] = (j + t < g.n) ? r.m[j + t] : 0.0f;
  }
#pragma unroll
  for (int t = 0; t < 4; ++t) cut_j[t] *= r.p;
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int rr = tr + 16 * k;
    const int64_t i = row0 + rr;
    float y[4] = {0.0f, 0.0f, 0.0f, 0.0f};
    if (i < g.n) {
      float bv[4] = {0.0f, 0.0f, 0.0f, 0.0f};
      if (full4) {
        const float4 v = ld_stream4(g.b + (i - g.b_row0) * g.ldb + j);
        bv[0] = v.x; bv[1] = v.y; bv[2] = v.z; bv[3] = v.w;
      } else {
#pragma unroll
        for (int t = 0; t < 4; ++t) bv[t] = (j + t < g.n) ? g.b[(i - g.b_row0) * g.ldb + j + t] : 0.0f;
      }
      if (diag_tile) {
        // below the diagonal, the mirror of the upper element: the computed blur is not bitwise
        // symmetric, and Y(i, j) must equal Y(j, i) = rule(b[j, i], m_j, m_i) exactly
#pragma unroll
        for (int t = 0; t < 4; ++t)
          if (j + t < i) bv[t] = g.b[(j + t - g.b_row0) * g.ldb + i];
      }
      const float cut_i = r.m[i] * r.p;
      const int64_t dcol = diag_tile ? i - j : -1;             // column of (i, i) in the run
#pragma unroll
      for (int t = 0; t < 4; ++t) y[t] = thrsym_rule(r, bv[t], cut_i, cut_j[t], dcol == t);
      store_y<4>(r, i, j, y, full4, g.n);
    }
    if (!diag_tile) {
      tile[rr][tc] = y[0]; tile[rr][tc + 1] = y[1]; tile[rr][tc + 2] = y[2]; tile[rr][tc + 3] = y[3];
    }
  }
  if (diag_tile) return;                                       // block-uniform
  __syncthreads();
  // transposed write: row (col0 + r') of Y, columns row0 + 4 c' .. +3
  const int64_t jm = row0 + tc;
  const bool full4m = (jm + 3 < g.n);
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    const int rr = tr + 16 * k;
    const int64_t i = col0 + rr;
    if (i >= g.n) continue;
    const float y[4] = {tile[tc][rr], tile[tc + 1][rr], tile[tc + 2][rr], tile[tc + 3][rr]};
    store_y<4>(r, i, jm, y, full4m, g.n);
  }
}

// ------------------------------------------------------------------ symmetric pair, blur recomputed
// The symmetric pair without a stored B: pass 1 (k_blur_pair<false>) folds the row and column maxima
// of blur(A) over the same elements EPI_UPPER folds -- row i from column 128 floor(i / 128) -- and
// pass 2 (k_blur_pair<true>) blurs the upper triangle again and writes Y(i, j) and Y(j, i), i <= j,
// from the one value rule(b[i, j], m_i, m_j).  Each b is the same fmaf chain as k_blur_band's
// (vertical taps, then horizontal, reflected edges, the crop substituted on read), so m and Y are
// bit for bit those of sc_blur_upper_rowmax + sc_threshold_symmetrize_upper.
//
// A warp owns a strip of 120 output columns and walks down a band of 256 rows with no barrier:
//   lane L loads the 4 columns c0 - 4 + 4L .. +3 of each input row (one 128-bit load; lanes 0 and 31
//     are the horizontal halo), PU rows per step with the next step's rows already in flight;
//   the vertical taps slide down a 16-row register window per column;
//   the horizontal taps take the 4 columns on each side from the neighbouring lanes (8 shuffles).
// Halo: 8 rows per 256 (3 %) from HBM; the 8 halo columns of a strip are the next strips' columns and
// come from L2.  Pass 2 writes Y(i, .) from registers and stages 16 rows of y per warp in shared memory
// so that Y(j, i0 .. i0 + 15) of the mirror goes out as whole 32-byte sectors of each plane.
// A CTA is 8 adjacent strips of one band; pass 1 combines their row maxima in shared memory, so there
// is one atomic per row per CTA and one per column per warp.
constexpr int PW = 8, PCOLS = 120, PTH = 256, PU = 4, PMB = 16;

struct PairArgs {
  const float* a;
  int64_t n, lda;
  const float* diag;       // optional replacement of a[i][i]
  float* m_out;            // pass 1: row maxima, zero-filled by the caller
  int zero_diag;           // pass 1: the diagonal folds as 0 (RowWiseThreshold preserve_diagonal)
  RuleArgs r;              // pass 2
};

// One warp's strip: columns [c0, c0 + PCOLS) of rows [r0, r0 + PTH).  FAST: interior and off the
// diagonal (no reflection, no crop, no per-element masks).
template <bool PASS2, bool FAST>
__device__ __forceinline__ void pair_strip(const PairArgs& g, const BlurWeights& bw, int64_t r0,
                                           int64_t c0, bool vec, float* part, float* ybuf) {
  constexpr int R = 4;
  const int lane = threadIdx.x & 31;
  const int64_t n = g.n;
  const int64_t cv0 = c0 - R + 4 * lane;                        // this lane's first (virtual) column
  const bool own = lane >= 1 && lane <= 30;
  int64_t pc[4];                                                // physical columns (reflected)
#pragma unroll
  for (int q = 0; q < 4; ++q) pc[q] = (FAST || vec) ? cv0 + q : reflect_index(cv0 + q, n);
  const bool crop = !FAST && g.diag != nullptr;

  float cut_j[4] = {0.0f, 0.0f, 0.0f, 0.0f};
  if (PASS2) {
#pragma unroll
    for (int q = 0; q < 4; ++q)
      cut_j[q] = (cv0 + q >= 0 && cv0 + q < n ? g.r.m[cv0 + q] : 0.0f) * g.r.p;
  }
  float cm[4] = {0.0f, 0.0f, 0.0f, 0.0f};                       // pass 1: column maxima

  auto load_row = [&](int64_t vr, float (&v)[4]) {
    const int64_t gr = (FAST || (vr >= 0 && vr < n)) ? vr : reflect_index(vr, n);
    const float* row = g.a + gr * g.lda;
    if (FAST || vec) {
      const float4 t = ld_stream4(row + cv0);
      v[0] = t.x; v[1] = t.y; v[2] = t.z; v[3] = t.w;
    } else {
#pragma unroll
      for (int q = 0; q < 4; ++q) v[q] = row[pc[q]];
    }
    if (crop) {
#pragma unroll
      for (int q = 0; q < 4; ++q)
        if (gr == pc[q]) v[q] = g.diag[gr];
    }
  };

  // output row i from the 9 input rows win[.][u .. u + 2R]
  auto row_out = [&](int64_t i, const float (&win)[4][PU + 2 * R], int u) {
    float mid[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      float acc = 0.0f;
#pragma unroll
      for (int k = 0; k <= 2 * R; ++k) acc = fmaf(bw.w[k], win[q][u + k], acc);
      mid[q] = acc;
    }
    float e[12];                                                // columns cv0 - 4 .. cv0 + 7
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      e[q] = __shfl_up_sync(0xffffffffu, mid[q], 1);
      e[4 + q] = mid[q];
      e[8 + q] = __shfl_down_sync(0xffffffffu, mid[q], 1);
    }
    float b[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      float acc = 0.0f;
#pragma unroll
      for (int k = 0; k <= 2 * R; ++k) acc = fmaf(bw.w[k], e[q + k], acc);
      b[q] = acc;
    }
    const int rl = (int)(i - r0);
    if (!PASS2) {
      // fold row i from column 128 floor(i / 128), the diagonal as 0 if asked (EPI_UPPER's set)
      const int64_t jlo = i & ~(int64_t)127;
      float v = 0.0f;
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const int64_t j = cv0 + q;
        float x = b[q];
        if (!FAST && g.zero_diag && i == j) x = 0.0f;
        if (!own || (!FAST && !(i < n && j < n && j >= jlo))) x = 0.0f;
        x = fmaxf(x, 0.0f);
        cm[q] = fmaxf(cm[q], x);
        v = fmaxf(v, x);
      }
      // non-negative floats order like their bit patterns: one REDUX.MAX for the strip's row
      const int mx = __reduce_max_sync(0xffffffffu, __float_as_int(v));
      if (lane == 0) part[rl] = __int_as_float(mx);
    } else {
      const RuleArgs& r = g.r;
      const float cut_i = r.m[(FAST || i < n) ? i : n - 1] * r.p;
      float y[4];
#pragma unroll
      for (int q = 0; q < 4; ++q)
        y[q] = thrsym_rule(r, b[q], cut_i, cut_j[q], !FAST && i == cv0 + q);
      // Y(i, j) for j >= i
      if (FAST || (i < n && cv0 >= i && cv0 + 3 < n)) {
        if (own) store_y<4>(r, i, cv0, y, true, n);
      } else if (own && i < n) {
#pragma unroll
        for (int q = 0; q < 4; ++q) {
          const float yq[1] = {y[q]};
          if (cv0 + q >= i && cv0 + q < n) store_y<1>(r, i, cv0 + q, yq, true, n);
        }
      }
      *reinterpret_cast<float4*>(ybuf + (rl & (PMB - 1)) * 128 + 4 * lane) =
          make_float4(y[0], y[1], y[2], y[3]);
    }
  };

  // pass 2: Y(j, i0 .. i0 + PMB - 1) <- the staged y(i0 .., j), for the strip's columns j > i
  auto flush = [&](int64_t i0) {
    __syncwarp();
#pragma unroll
    for (int rd = 0; rd < 4; ++rd) {
      const int cl = 4 + 32 * rd + lane;                        // column of the staging buffer
      const int64_t j = c0 + 32 * rd + lane;
      if (cl >= 4 + PCOLS || (!FAST && j >= n)) continue;
      float y[PMB];
#pragma unroll
      for (int t = 0; t < PMB; ++t) y[t] = ybuf[t * 128 + cl];
      if (FAST || i0 + PMB - 1 < j) {
        store_y<PMB>(g.r, j, i0, y, true, n);
      } else {
#pragma unroll
        for (int t = 0; t < PMB; ++t) {
          const float yt[1] = {y[t]};
          if (i0 + t < j) store_y<1>(g.r, j, i0 + t, yt, true, n);
        }
      }
    }
    __syncwarp();
  };

  // win[q][k] = input row i0 - R + k of the lane's column q, i0 = the step's first output row; the
  // next step's PU rows are in flight (nxt) while this step is filtered
  float win[4][PU + 2 * R];
  float nxt[PU][4];
#pragma unroll
  for (int k = 0; k < 2 * R; ++k) {
    float v[4];
    load_row(r0 - R + k, v);
#pragma unroll
    for (int q = 0; q < 4; ++q) win[q][k] = v[q];
  }
#pragma unroll
  for (int u = 0; u < PU; ++u) load_row(r0 + R + u, nxt[u]);
  for (int st = 0; st < PTH / PU; ++st) {
    const int64_t i0 = r0 + (int64_t)st * PU;
#pragma unroll
    for (int u = 0; u < PU; ++u)
#pragma unroll
      for (int q = 0; q < 4; ++q) win[q][2 * R + u] = nxt[u][q];
    if (st + 1 < PTH / PU) {
#pragma unroll
      for (int u = 0; u < PU; ++u) load_row(i0 + PU + R + u, nxt[u]);
    }
#pragma unroll
    for (int u = 0; u < PU; ++u) row_out(i0 + u, win, u);
#pragma unroll
    for (int q = 0; q < 4; ++q)
#pragma unroll
      for (int k = 0; k < 2 * R; ++k) win[q][k] = win[q][PU + k];
    if (PASS2 && ((st + 1) * PU) % PMB == 0) flush(i0 + PU - PMB);
  }
  if (!PASS2 && own) {
#pragma unroll
    for (int q = 0; q < 4; ++q)
      if (FAST || cv0 + q < n) atomic_max_nonneg(g.m_out + cv0 + q, cm[q]);
  }
}

template <bool PASS2>
__global__ void __launch_bounds__(PW * 32, 2)
k_blur_pair(const PairArgs g, const BlurWeights bw) {
  constexpr int R = 4;
  extern __shared__ float psmem[];     // pass 1: [PW][PTH] row maxima; pass 2: [PW][PMB][128] y
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t n = g.n;
  const int64_t r0 = (int64_t)blockIdx.x * PTH;
  // strips from the one holding column r0: every element the band needs lies right of it (PTH is a
  // multiple of 128)
  const int64_t s0 = r0 / PCOLS + (int64_t)blockIdx.y * PW;
  if (s0 * PCOLS >= n) return;                                  // block-uniform
  const int64_t c0 = (s0 + warp) * PCOLS;
  float* part = psmem + warp * PTH;
  float* ybuf = psmem + warp * (PMB * 128);
  if (c0 < n) {                                                 // warp-uniform
    const bool vec = c0 >= R && c0 + PCOLS + R <= n && (g.lda & 3) == 0 &&
                     (reinterpret_cast<uintptr_t>(g.a) & 15) == 0;
    if (vec && r0 >= R && r0 + PTH + R <= n && c0 >= r0 + PTH + 2 * R)
      pair_strip<PASS2, true>(g, bw, r0, c0, vec, part, ybuf);
    else
      pair_strip<PASS2, false>(g, bw, r0, c0, vec, part, ybuf);
  } else if (!PASS2) {
    for (int k = lane; k < PTH; k += 32) part[k] = 0.0f;
  }
  if (!PASS2) {
    __syncthreads();
    const int rl = threadIdx.x;                                 // PTH == blockDim.x
    if (r0 + rl < n) {
      float v = 0.0f;
#pragma unroll
      for (int w = 0; w < PW; ++w) v = fmaxf(v, psmem[w * PTH + rl]);
      atomic_max_nonneg(g.m_out + r0 + rl, v);
    }
  }
}

static_assert(PTH == PW * 32 && PTH % 128 == 0 && PTH % PMB == 0 && PMB % PU == 0,
              "band geometry");

// Launch one pass of the pair (radius 4 only; the weights come from make_weights).
template <bool PASS2>
static int launch_pair(const PairArgs& g, const BlurWeights& bw, cudaStream_t st) {
  const size_t smem = sizeof(float) * (PASS2 ? PW * PMB * 128 : PW * PTH);
  auto k = k_blur_pair<PASS2>;
  SC_CUDA(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int64_t nstrips = (g.n + PCOLS - 1) / PCOLS;
  const dim3 grid((unsigned)((g.n + PTH - 1) / PTH), (unsigned)((nstrips + PW - 1) / PW));
  k<<<grid, PW * 32, smem, st>>>(g, bw);
  sc::launched();
  SC_LAUNCH_CHECK();
  return 0;
}

// scipy _gaussian_kernel1d: radius = int(truncate * sigma + 0.5) with truncate = 4; sigma <= 1e-15
// copies the input ("if sigma > 1e-15 ... else output[...] = input[...]"), i.e. radius 0.
static int blur_radius(double sigma) { return sigma > 1e-15 ? (int)(4.0 * sigma + 0.5) : 0; }

// Weights exp(-x^2/(2 sigma^2)) / sum for radius > 0 (radius 0 runs k_noblur, which takes none).
static int make_weights(double sigma, BlurWeights& bw, int& radius) {
  radius = blur_radius(sigma);
  if (radius > kMaxRadius) return 1;
  if (radius == 0) return 0;
  double w[2 * kMaxRadius + 1], sum = 0.0;
  for (int k = -radius; k <= radius; ++k) {
    w[k + radius] = std::exp(-0.5 / (sigma * sigma) * (double)k * (double)k);
    sum += w[k + radius];
  }
  for (int k = 0; k <= 2 * radius; ++k) bw.w[k] = (float)(w[k] / sum);
  return 0;
}

template <int EPI>
static int launch_band(BlurArgs& g, const BlurWeights& bw, cudaStream_t st) {
  constexpr int R = 4;
  const size_t smem = sizeof(float) * (2 * (TTH + 2 * R) * (TTW + 2 * R) + TTH * (TTW + 2 * R + 1));
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

// The two-pass forms (EPI_STORE / EPI_STATS / EPI_THRSYM) at any radius.
template <int EPI>
static int launch_blur(const sc_context* ctx, BlurArgs& g, double sigma, cudaStream_t st) {
  static_assert(EPI != EPI_UPPER, "the symmetric pass launches k_blur_band directly");
  SC_REQUIRE(g.row_end - g.row_begin <= 65535LL * 32, "sc_gaussian_blur: n too large for the tile grid");
  BlurWeights bw;
  SC_REQUIRE(make_weights(sigma, bw, g.radius) == 0,
             "sc_gaussian_blur: sigma %g needs radius > %d", sigma, kMaxRadius);
  if (g.radius == 0) {      // a copy, or a single tap of weight 1
    const unsigned gy = (unsigned)std::min<int64_t>((g.n + 1023) / 1024, 64);
    k_noblur<EPI><<<dim3((unsigned)(g.row_end - g.row_begin), gy), 256, 0, st>>>(g); sc::launched();
    SC_LAUNCH_CHECK();
    return 0;
  }
  if (g.radius == 4) return launch_band<EPI>(g, bw, st);
  const size_t smem = sizeof(float) * ((size_t)(GTH + 2 * g.radius) * (GTW + 2 * g.radius) +
                                       (size_t)GTH * (GTW + 2 * g.radius));
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

// Output rows [row_begin, row_end) from input rows starting at global row in_row_base.
static BlurArgs blur_args(const float* a, int64_t n, int64_t lda, int64_t in_row_base,
                          int64_t row_begin, int64_t row_end, const float* diag_override) {
  BlurArgs g = {};
  g.a = a; g.n = n; g.lda = lda; g.diag = diag_override;
  g.row_begin = row_begin; g.row_end = row_end; g.in_row_base = in_row_base;
  g.out_row_base = row_begin;
  return g;
}

static int check_block(int64_t n, int64_t in_row_base, int64_t in_rows, int64_t row_begin,
                       int64_t row_end, double sigma) {
  SC_REQUIRE(0 <= row_begin && row_begin < row_end && row_end <= n, "blur block: bad row range");
  SC_REQUIRE((row_end - row_begin) % 32 == 0 || row_end == n,
             "blur block: the row count must be a multiple of 32 unless the block ends the matrix");
  // every input row the block can touch (after reflection at the matrix edges) must be resident
  const int radius = blur_radius(sigma);
  const int64_t need_lo = row_begin - radius < 0 ? 0 : row_begin - radius;
  const int64_t need_hi = row_end + radius > n ? n : row_end + radius;
  SC_REQUIRE(in_row_base <= need_lo && in_row_base + in_rows >= need_hi,
             "blur block: input rows [%lld, %lld) do not cover the halo [%lld, %lld)",
             (long long)in_row_base, (long long)(in_row_base + in_rows), (long long)need_lo,
             (long long)need_hi);
  return 0;
}

// The rule and the Y outputs of the three threshold/symmetrize entries (`lo` may be NULL here).
static int rule_args(const char* who, const float* rowmax, double p, double mult, int binarize,
                     int preserve_diagonal, int sym_type, float* y, int64_t ldy, void* hi,
                     void* lo, int64_t ldh, RuleArgs& r) {
  SC_REQUIRE(y || hi, "%s: no output given", who);
  SC_REQUIRE(hi || !lo, "%s: a lo plane needs its hi plane", who);
  SC_REQUIRE(sym_type == SC_SYMMETRIZE_MAX || sym_type == SC_SYMMETRIZE_AVERAGE,
             "Unsupported symmetrize_type.");
  SC_REQUIRE(aligned16(rowmax), "%s: the row-maximum vector needs a 16-byte aligned base", who);
  SC_REQUIRE(!y || vec_ok_f32(y, ldy), "%s: `y` needs a 16-byte aligned base and ldy %% 4 == 0", who);
  SC_REQUIRE(!hi || (vec_ok_f16(hi, ldh) && (!lo || vec_ok_f16(lo, ldh))),
             "%s: the fp16 planes need 16-byte aligned bases and ldh %% 8 == 0", who);
  r = RuleArgs{rowmax, (float)p, (float)mult, binarize, preserve_diagonal, sym_type,
               y, ldy, (__half*)hi, (__half*)lo, ldh};
  return 0;
}

extern "C" int sc_gaussian_blur(sc_context* ctx, const float* a, int64_t n, int64_t lda,
                                const float* diag_override, double sigma, float* out,
                                int64_t ldo, float* rowmax_out, void* stream) {
  SC_REQUIRE(ctx && a && n > 0, "sc_gaussian_blur: bad arguments");
  SC_REQUIRE(out || rowmax_out, "sc_gaussian_blur: nothing to compute");
  SC_REQUIRE(!out || vec_ok_f32(out, ldo), "blur: `out` needs a 16-byte aligned base and ldo %% 4 == 0");
  BlurArgs g = blur_args(a, n, lda, 0, 0, n, diag_override);
  g.out = out; g.ldo = ldo; g.rowmax_out = rowmax_out;
  if (out) return launch_blur<EPI_STORE>(ctx, g, sigma, as_stream(stream));
  return launch_blur<EPI_STATS>(ctx, g, sigma, as_stream(stream));
}

// ---- row blocks (multi-GPU row sharding, SURVEY.md 8(e)): `a` holds global rows
// [in_row_base, in_row_base + in_rows) -- the owned rows plus the blur halo, recomputed locally
// from the embeddings instead of exchanged; outputs cover global rows [row_begin, row_end) and are
// written to buffers whose row 0 is global row `row_begin`.  diag_override / rowmax vectors are
// indexed by global row.  The whole-matrix entries are the block [0, n) with the input at row 0.
static int blur_rowmax_rows(const char* who, sc_context* ctx, const float* a, int64_t n,
                            int64_t lda, int64_t in_row_base, int64_t in_rows, int64_t row_begin,
                            int64_t row_end, const float* diag_override, double sigma,
                            int zero_diagonal, float* rowmax_out, void* stream) {
  SC_REQUIRE(ctx && a && rowmax_out && n > 0, "%s: bad arguments", who);
  if (int rc = check_block(n, in_row_base, in_rows, row_begin, row_end, sigma)) return rc;
  BlurArgs g = blur_args(a, n, lda, in_row_base, row_begin, row_end, diag_override);
  g.rowmax_out = rowmax_out; g.stats_zero_diag = zero_diagonal;
  return launch_blur<EPI_STATS>(ctx, g, sigma, as_stream(stream));
}

static int blur_thrsym_rows(const char* who, sc_context* ctx, const float* a, int64_t n,
                            int64_t lda, int64_t in_row_base, int64_t in_rows, int64_t row_begin,
                            int64_t row_end, const float* diag_override, double sigma,
                            const float* rowmax, double p, double mult, int binarize,
                            int preserve_diagonal, int sym_type, float* y, int64_t ldy, void* hi,
                            void* lo, int64_t ldh, void* stream) {
  SC_REQUIRE(ctx && a && rowmax && n > 0, "%s: bad arguments", who);
  RuleArgs r;
  if (int rc = rule_args(who, rowmax, p, mult, binarize, preserve_diagonal, sym_type, y, ldy, hi,
                         lo, ldh, r))
    return rc;
  if (int rc = check_block(n, in_row_base, in_rows, row_begin, row_end, sigma)) return rc;
  BlurArgs g = blur_args(a, n, lda, in_row_base, row_begin, row_end, diag_override);
  g.r = r;
  return launch_blur<EPI_THRSYM>(ctx, g, sigma, as_stream(stream));
}

// statistics pass with the diagonal read as zero (RowWiseThreshold preserve_diagonal)
extern "C" int sc_gaussian_blur_rowmax(sc_context* ctx, const float* a, int64_t n, int64_t lda,
                                       const float* diag_override, double sigma,
                                       int zero_diagonal, float* rowmax_out, void* stream) {
  return blur_rowmax_rows("sc_gaussian_blur_rowmax", ctx, a, n, lda, 0, n, 0, n, diag_override,
                          sigma, zero_diagonal, rowmax_out, stream);
}

extern "C" int sc_gaussian_blur_rowmax_block(sc_context* ctx, const float* a, int64_t n,
                                             int64_t lda, int64_t in_row_base, int64_t in_rows,
                                             int64_t row_begin, int64_t row_end,
                                             const float* diag_override, double sigma,
                                             int zero_diagonal, float* rowmax_out,
                                             void* stream) {
  return blur_rowmax_rows("sc_gaussian_blur_rowmax_block", ctx, a, n, lda, in_row_base, in_rows,
                          row_begin, row_end, diag_override, sigma, zero_diagonal, rowmax_out,
                          stream);
}

extern "C" int sc_blur_threshold_symmetrize(sc_context* ctx, const float* a, int64_t n,
                                            int64_t lda, const float* diag_override,
                                            double sigma, const float* rowmax, double p,
                                            double mult, int binarize, int preserve_diagonal,
                                            int sym_type, float* y, int64_t ldy, void* hi,
                                            void* lo, int64_t ldh, void* stream) {
  return blur_thrsym_rows("sc_blur_threshold_symmetrize", ctx, a, n, lda, 0, n, 0, n,
                          diag_override, sigma, rowmax, p, mult, binarize, preserve_diagonal,
                          sym_type, y, ldy, hi, lo, ldh, stream);
}

extern "C" int sc_blur_threshold_symmetrize_block(
    sc_context* ctx, const float* a, int64_t n, int64_t lda, int64_t in_row_base, int64_t in_rows,
    int64_t row_begin, int64_t row_end, const float* diag_override, double sigma,
    const float* rowmax, double p, double mult, int binarize, int preserve_diagonal, int sym_type,
    float* y, int64_t ldy, void* hi, void* lo, int64_t ldh, void* stream) {
  return blur_thrsym_rows("sc_blur_threshold_symmetrize_block", ctx, a, n, lda, in_row_base,
                          in_rows, row_begin, row_end, diag_override, sigma, rowmax, p, mult,
                          binarize, preserve_diagonal, sym_type, y, ldy, hi, lo, ldh, stream);
}

// ---- symmetric whole-matrix pair (single-GPU hot path).  Pass 1: m_out[i] <- max_j blur(a)[i,j]
// assembled from the row AND column maxima of the tiles of blur(a) that touch the upper triangle;
// with b_out, those tiles are also stored (the rest of b_out is left untouched) for
// sc_threshold_symmetrize_upper, without it nothing else is written and
// sc_blur_threshold_symmetrize_upper blurs the tiles again.  Requires a symmetric `a` and sigma
// with radius 4 (sigma in [0.875, 1.125), every BASELINE configuration); the caller falls back to
// sc_gaussian_blur_rowmax + sc_blur_threshold_symmetrize otherwise.
extern "C" int sc_blur_upper_rowmax(sc_context* ctx, const float* a, int64_t n, int64_t lda,
                                    const float* diag_override, double sigma, int zero_diagonal,
                                    float* b_out, int64_t ldb, float* rowmax_out, void* stream) {
  SC_REQUIRE(ctx && a && rowmax_out && n > 0, "sc_blur_upper_rowmax: bad arguments");
  SC_REQUIRE(blur_radius(sigma) == 4,
             "sc_blur_upper_rowmax: the symmetric pass is built for radius 4 (sigma ~ 1)");
  SC_REQUIRE(n <= 65535LL * 32, "sc_blur_upper_rowmax: n too large for the tile grid");
  SC_REQUIRE(!b_out || vec_ok_f32(b_out, ldb),
             "blur: `out` needs a 16-byte aligned base and ldo %% 4 == 0");
  BlurWeights bw;
  int radius;
  make_weights(sigma, bw, radius);
  SC_CUDA(cudaMemsetAsync(rowmax_out, 0, sizeof(float) * n, as_stream(stream)));
  if (!b_out) {
    PairArgs p = {};
    p.a = a; p.n = n; p.lda = lda; p.diag = diag_override;
    p.m_out = rowmax_out; p.zero_diag = zero_diagonal;
    return launch_pair<false>(p, bw, as_stream(stream));
  }
  BlurArgs g = blur_args(a, n, lda, 0, 0, n, diag_override);
  g.out = b_out; g.ldo = ldb; g.rowmax_out = rowmax_out; g.stats_zero_diag = zero_diagonal;
  g.radius = radius;
  return launch_band<EPI_UPPER>(g, bw, as_stream(stream));
}

// Pass 2 without a stored B: the upper triangle of blur(a) again, then Y(i, j) and Y(j, i) from
// rule(b[min(i, j), max(i, j)], m_i, m_j) -- bit for bit sc_threshold_symmetrize_upper on the B
// that sc_blur_upper_rowmax stores.
extern "C" int sc_blur_threshold_symmetrize_upper(sc_context* ctx, const float* a, int64_t n,
                                                  int64_t lda, const float* diag_override,
                                                  double sigma, const float* rowmax, double p,
                                                  double mult, int binarize, int preserve_diagonal,
                                                  int sym_type, float* y, int64_t ldy, void* hi,
                                                  void* lo, int64_t ldh, void* stream) {
  const char* who = "sc_blur_threshold_symmetrize_upper";
  SC_REQUIRE(ctx && a && rowmax && n > 0, "%s: bad arguments", who);
  SC_REQUIRE(blur_radius(sigma) == 4, "%s: the symmetric pass is built for radius 4 (sigma ~ 1)",
             who);
  SC_REQUIRE(n <= 65535LL * PCOLS, "%s: n too large for the tile grid", who);
  PairArgs g = {};
  if (int rc = rule_args(who, rowmax, p, mult, binarize, preserve_diagonal, sym_type, y, ldy, hi,
                         lo, ldh, g.r))
    return rc;
  g.a = a; g.n = n; g.lda = lda; g.diag = diag_override;
  BlurWeights bw;
  int radius;
  make_weights(sigma, bw, radius);
  return launch_pair<true>(g, bw, as_stream(stream));
}

// Pass 2 over the tile pairs (TI, TJ), TI <= TJ, whose rows TI lie in [row_begin, row_end); `b`
// holds rows [row_begin, row_end) of the upper tiles of B.
static int thrsym_upper_rows(const char* who, sc_context* ctx, const float* b, int64_t n,
                             int64_t ldb, int64_t row_begin, int64_t row_end, const float* rowmax,
                             double p, double mult, int binarize, int preserve_diagonal,
                             int sym_type, float* y, int64_t ldy, void* hi, void* lo, int64_t ldh,
                             void* stream) {
  SC_REQUIRE(ctx && b && rowmax && n > 0, "%s: bad arguments", who);
  SC_REQUIRE(0 <= row_begin && row_begin < row_end && row_end <= n && row_begin % UT == 0 &&
             (row_end % UT == 0 || row_end == n),
             "%s: the row range must start on a multiple of %d and end on one or at n", who, UT);
  UpperArgs g = {};
  if (int rc = rule_args(who, rowmax, p, mult, binarize, preserve_diagonal, sym_type, y, ldy, hi,
                         lo, ldh, g.r))
    return rc;
  SC_REQUIRE(vec_ok_f32(b, ldb), "%s: `b` alignment", who);
  g.b = b; g.n = n; g.ldb = ldb; g.b_row0 = row_begin;
  g.tiles = (int)((n + UT - 1) / UT);
  const int64_t T = g.tiles, t0 = row_begin / UT, t1 = (row_end + UT - 1) / UT;
  g.pair0 = t0 * T - t0 * (t0 - 1) / 2;                     // first pair of tile row t0
  const int64_t pairs = t1 * T - t1 * (t1 - 1) / 2 - g.pair0;
  SC_REQUIRE(T * (T + 1) / 2 < (1LL << 31), "%s: n too large for the tile grid", who);
  k_thrsym_upper<<<(unsigned)pairs, 256, 0, as_stream(stream)>>>(g); sc::launched();
  SC_LAUNCH_CHECK();
  return 0;
}

// Pass 2: y / planes <- sym(thr(b, m_i), thr(b, m_j)) for the WHOLE matrix from the upper tiles of b.
extern "C" int sc_threshold_symmetrize_upper(sc_context* ctx, const float* b, int64_t n, int64_t ldb,
                                             const float* rowmax, double p, double mult,
                                             int binarize, int preserve_diagonal, int sym_type,
                                             float* y, int64_t ldy, void* hi, void* lo, int64_t ldh,
                                             void* stream) {
  return thrsym_upper_rows("sc_threshold_symmetrize_upper", ctx, b, n, ldb, 0, n, rowmax, p, mult,
                           binarize, preserve_diagonal, sym_type, y, ldy, hi, lo, ldh, stream);
}

// ---- row panels of the symmetric pair (one GPU, no N x N fp32 matrix).  Pass 1 over the rows
// [row_begin, row_end) of a panel `a` that holds global rows [in_row_base, in_row_base + in_rows):
// b_out (rows [row_begin, row_end)) <- the upper tiles of blur(a), and their row and column maxima
// are folded into rowmax_accum, which the caller zero-fills once for all panels.
extern "C" int sc_blur_upper_rowmax_block(sc_context* ctx, const float* a, int64_t n, int64_t lda,
                                          int64_t in_row_base, int64_t in_rows, int64_t row_begin,
                                          int64_t row_end, const float* diag_override,
                                          double sigma, int zero_diagonal, float* b_out,
                                          int64_t ldb, float* rowmax_accum, void* stream) {
  SC_REQUIRE(ctx && a && b_out && rowmax_accum && n > 0, "sc_blur_upper_rowmax_block: bad arguments");
  SC_REQUIRE(blur_radius(sigma) == 4,
             "sc_blur_upper_rowmax_block: the symmetric pass is built for radius 4 (sigma ~ 1)");
  SC_REQUIRE(row_begin % TTH == 0, "sc_blur_upper_rowmax_block: row_begin must be a multiple of %d", TTH);
  SC_REQUIRE(vec_ok_f32(b_out, ldb), "blur: `out` needs a 16-byte aligned base and ldo %% 4 == 0");
  if (int rc = check_block(n, in_row_base, in_rows, row_begin, row_end, sigma)) return rc;
  SC_REQUIRE(row_end - row_begin <= 65535LL * 32, "sc_blur_upper_rowmax_block: too many rows");
  BlurArgs g = blur_args(a, n, lda, in_row_base, row_begin, row_end, diag_override);
  g.out = b_out; g.ldo = ldb; g.rowmax_out = rowmax_accum; g.stats_zero_diag = zero_diagonal;
  BlurWeights bw;
  make_weights(sigma, bw, g.radius);
  return launch_band<EPI_UPPER>(g, bw, as_stream(stream));
}

// Pass 2 of a panel: the tile pairs whose first tile row lies in [row_begin, row_end), from the
// panel's upper tiles of B (rows [row_begin, row_end), as pass 1 wrote them); Y and its mirror go
// to the full-size outputs.
extern "C" int sc_threshold_symmetrize_upper_block(
    sc_context* ctx, const float* b, int64_t n, int64_t ldb, int64_t row_begin, int64_t row_end,
    const float* rowmax, double p, double mult, int binarize, int preserve_diagonal, int sym_type,
    float* y, int64_t ldy, void* hi, void* lo, int64_t ldh, void* stream) {
  return thrsym_upper_rows("sc_threshold_symmetrize_upper_block", ctx, b, n, ldb, row_begin,
                           row_end, rowmax, p, mult, binarize, preserve_diagonal, sym_type, y, ldy,
                           hi, lo, ldh, stream);
}
