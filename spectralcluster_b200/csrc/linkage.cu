// Complete- and average-linkage cosine agglomerative clustering (scikit-learn
// AgglomerativeClustering(metric="cosine", linkage="complete" / "average") = scipy pdist(x,
// "cosine") + scipy linkage(..., "complete" / "average")):
//   k_row_norms        |x_i| in fp64, one thread per row
//   k_cosine_dist      D = 1 - clamp(X X^T / (|x_i| |x_j|), -1, 1), fp64 tensor cores, upper 64x64
//                      tiles only, each tile stored and mirror-stored through shared memory
//   k_nn_chain<L>      scipy's nn_chain, every merge in one cooperative launch: each chain step is
//                      a row scan split across the grid (one CTA per SM), a grid barrier, and a
//                      redundant reduction of the per-CTA minima in every CTA; a merge adds a
//                      row + column update (the linkage's Lance-Williams rule) and one more barrier.
//   k_nn_chain_small<L> the same chain for n <= SC_NN_SMALL_MAX in one CTA: block barriers instead
//                      of grid barriers, sizes and chain in shared memory (stream-sized caches)
// and the centroids of the clusters found (utils.get_cluster_centroids, max_spectral_size):
//   k_centroid_order   stable counting sort of the row indices by cluster id, one warp
//   k_centroid_sums    per (cluster, column): fp64 sum of the members in row order, over the count
#include "common.cuh"

#include <climits>
#include <cooperative_groups.h>

namespace cg = cooperative_groups;
using namespace sc;

namespace {

constexpr int CD_T = 64;                 // output tile edge
constexpr int CD_KC = 32;                // k-chunk staged in shared memory
constexpr int CD_PITCH = CD_KC + 4;      // doubles; == 4 mod 16: conflict-free fragment loads
constexpr int CD_OUT_PITCH = CD_T + 1;   // doubles; transposed reads of the staged tile
constexpr int CD_SMEM = 2 * CD_T * CD_PITCH * (int)sizeof(double);
static_assert(CD_T * CD_OUT_PITCH <= 2 * CD_T * CD_PITCH, "staged tile must fit the operand tiles");

template <typename T>
__device__ __forceinline__ double load_x(const void* x, int64_t off) {
  return (double)reinterpret_cast<const T*>(x)[off];
}

// scipy's row norms: rounded squares summed in index order, no FMA, so that they agree bit for bit
__global__ void __launch_bounds__(256)
k_row_norms(const void* __restrict__ x, int is64, int64_t n, int64_t d, int64_t ldx,
            double* __restrict__ nrm) {
  const int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (row >= n) return;
  double s = 0.0;
  for (int64_t k = 0; k < d; ++k) {
    const double v = is64 ? load_x<double>(x, row * ldx + k) : load_x<float>(x, row * ldx + k);
    s = __dadd_rn(s, __dmul_rn(v, v));
  }
  nrm[row] = sqrt(s);
}

// One CTA per upper tile (blockIdx.y <= blockIdx.x); 8 warps x (8 rows x 64 columns) of DMMA.
__global__ void __launch_bounds__(256)
k_cosine_dist(const void* __restrict__ x, int is64, int64_t n, int64_t d, int64_t ldx,
              const double* __restrict__ nrm, double* __restrict__ dist, int64_t ldd,
              int* __restrict__ nonfinite) {
  if (blockIdx.y > blockIdx.x) return;
  extern __shared__ double cd_smem[];
  double* as = cd_smem;                         // rows r0.. : [64][CD_PITCH]
  double* bs = cd_smem + CD_T * CD_PITCH;       // rows c0.. : [64][CD_PITCH]
  const bool diag = blockIdx.y == blockIdx.x;
  const int64_t r0 = (int64_t)blockIdx.y * CD_T, c0 = (int64_t)blockIdx.x * CD_T;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int fr = lane >> 2, fk = lane & 3;
  double acc[8][2];
#pragma unroll
  for (int t = 0; t < 8; ++t) acc[t][0] = acc[t][1] = 0.0;
  for (int64_t k0 = 0; k0 < d; k0 += CD_KC) {
    for (int idx = threadIdx.x; idx < CD_T * CD_KC; idx += blockDim.x) {
      const int t = idx / CD_KC, k = idx - t * CD_KC;       // consecutive threads: consecutive k
      const bool kin = k0 + k < d;
      double av = 0.0, bv = 0.0;
      if (kin && r0 + t < n)
        av = is64 ? load_x<double>(x, (r0 + t) * ldx + k0 + k) : load_x<float>(x, (r0 + t) * ldx + k0 + k);
      if (kin && c0 + t < n)
        bv = is64 ? load_x<double>(x, (c0 + t) * ldx + k0 + k) : load_x<float>(x, (c0 + t) * ldx + k0 + k);
      as[t * CD_PITCH + k] = av;
      bs[t * CD_PITCH + k] = bv;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < CD_KC; kk += 4) {
      const double av = as[(warp * 8 + fr) * CD_PITCH + kk + fk];
#pragma unroll
      for (int t = 0; t < 8; ++t) dmma_m8n8k4(acc[t][0], acc[t][1], av, bs[(t * 8 + fr) * CD_PITCH + kk + fk]);
    }
    __syncthreads();
  }
  // stage the finished tile: out[i][j] = D[r0 + i][c0 + j]
  double* out = cd_smem;
  const int i = warp * 8 + fr;
  const double ni = (r0 + i < n) ? nrm[r0 + i] : 1.0;
  bool bad = false;
#pragma unroll
  for (int t = 0; t < 8; ++t) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int j = t * 8 + fk * 2 + h;
      const double nj = (c0 + j < n) ? nrm[c0 + j] : 1.0;
      double c = acc[t][h] / (ni * nj);
      if (c > 1.0) c = 1.0;                    // a NaN stays NaN (fmin/fmax would drop it)
      else if (c < -1.0) c = -1.0;
      double v = 1.0 - c;
      if (diag && i == j) v = 0.0;
      if (r0 + i < n && c0 + j < n && (!diag || j >= i) && !isfinite(v)) bad = true;
      out[i * CD_OUT_PITCH + j] = v;
    }
  }
  if (__syncthreads_or(bad) && threadIdx.x == 0) atomicExch(nonfinite, 1);
  // direct store, row-major and coalesced; a diagonal tile keeps its upper triangle
  for (int idx = threadIdx.x; idx < CD_T * CD_T; idx += blockDim.x) {
    const int a = idx / CD_T, b = idx - a * CD_T;
    if (r0 + a < n && c0 + b < n && (!diag || b >= a)) dist[(r0 + a) * ldd + c0 + b] = out[a * CD_OUT_PITCH + b];
  }
  // mirror store D[c0 + a][r0 + b] = out[b][a]; a diagonal tile fills its lower triangle
  for (int idx = threadIdx.x; idx < CD_T * CD_T; idx += blockDim.x) {
    const int a = idx / CD_T, b = idx - a * CD_T;
    if (c0 + a < n && r0 + b < n && (!diag || a > b)) dist[(c0 + a) * ldd + r0 + b] = out[b * CD_OUT_PITCH + a];
  }
}

constexpr int NN_THREADS = 512;

// (value, index) ordered by value, then by index: the first index holding the minimum.
__device__ __forceinline__ void take_min(double& v, int& i, double ov, int oi) {
  if (ov < v || (ov == v && oi < i)) { v = ov; i = oi; }
}

__device__ __forceinline__ void warp_min_idx(double& v, int& i) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double ov = __shfl_xor_sync(0xffffffffu, v, o);
    const int oi = __shfl_xor_sync(0xffffffffu, i, o);
    take_min(v, i, ov, oi);
  }
}

// The (value, index) minimum of a CTA's NN_THREADS pairs: each warp reduces its lanes, lane 0
// stages the warp's pair, and warp 0 reduces the staged pairs.  The result is valid in warp 0.
__device__ __forceinline__ void cta_min_idx(double& v, int& i, double* red_v, int* red_i) {
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  warp_min_idx(v, i);
  if (lane == 0) red_v[wid] = v, red_i[wid] = i;
  __syncthreads();
  if (wid == 0) {
    v = lane < NN_THREADS / 32 ? red_v[lane] : INFINITY;
    i = lane < NN_THREADS / 32 ? red_i[lane] : INT_MAX;
    warp_min_idx(v, i);
  }
}

enum class Linkage { Complete, Average };

// The Lance-Williams update of d(i, a u b) from d(i, a), d(i, b) and the sizes na, nb, nab = na + nb.
// Average is scipy's _average, (na d_ai + nb d_bi) / (na + nb), rounded step by step: a contracted
// FMA would round once less and break bitwise equality with scipy.
template <Linkage L>
__device__ __forceinline__ double merged_distance(double da, double db, double na, double nb,
                                                  double nab) {
  if constexpr (L == Linkage::Complete) return fmax(da, db);
  else return __ddiv_rn(__dadd_rn(__dmul_rn(na, da), __dmul_rn(nb, db)), nab);
}

// Every CTA runs the same chain bookkeeping on the same reduced values, so all agree on every
// decision without a broadcast.  D and size change inside the launch: they are read with
// ld.global.cg (L2, never a stale L1 line) and written with st.global.cg.
template <Linkage L>
__global__ void __launch_bounds__(NN_THREADS)
k_nn_chain(double* __restrict__ dist, int64_t n, int64_t ldd, int* __restrict__ size,
           int* __restrict__ chain, double* __restrict__ part_v, int* __restrict__ part_i,
           int64_t* __restrict__ m_xy, double* __restrict__ m_dist, int64_t* __restrict__ m_size) {
  cg::grid_group grid = cg::this_grid();
  __shared__ double red_v[NN_THREADS / 32];
  __shared__ int red_i[NN_THREADS / 32];
  __shared__ double s_min;
  __shared__ int s_y;
  const int G = gridDim.x;
  const int64_t per = (n + G - 1) / G;
  const int64_t beg = (int64_t)blockIdx.x * per;
  const int64_t end = beg + per < n ? beg + per : n;
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  int len = 0;            // chain length
  int x = -1, prev = -1;  // chain top and the element below it
  int lo = 0;             // every index below lo is retired (indices are never reactivated)
  int parity = 0;         // the partials are double-buffered: one barrier per step suffices
  for (int64_t k = 0; k < n - 1;) {
    if (len == 0) {
      while (__ldcg(size + lo) == 0) ++lo;
      x = lo, prev = -1, len = 1;
      if (threadIdx.x == 0) __stcg(chain, x);
    }
    // A merge in this step joins x and prev.  Average linkage weighs their rows by their sizes,
    // which CTA 0 rewrites in the merge phase while other CTAs may still update; so every thread
    // reads both sizes here.  The last size writes were fenced by the previous merge's barrier and
    // the next ones follow this step's barrier: no write can overlap these loads.
    int nx = 0, nprev = 0;
    if constexpr (L == Linkage::Average) {
      nx = __ldcg(size + x);
      nprev = prev >= 0 ? __ldcg(size + prev) : 0;
    }
    // ---- nearest active neighbour of x in this CTA's columns
    const double* row = dist + (int64_t)x * ldd;
    double bv = INFINITY;
    int bi = INT_MAX;
    for (int64_t i = beg + threadIdx.x; i < end; i += NN_THREADS) {
      if (i == x || __ldcg(size + i) == 0) continue;
      const double v = __ldcg(row + i);
      if (v < bv) bv = v, bi = (int)i;
    }
    warp_min_idx(bv, bi);
    if (lane == 0) red_v[wid] = bv, red_i[wid] = bi;
    __syncthreads();
    if (wid == 0) {
      bv = lane < NN_THREADS / 32 ? red_v[lane] : INFINITY;
      bi = lane < NN_THREADS / 32 ? red_i[lane] : INT_MAX;
      warp_min_idx(bv, bi);
      if (lane == 0) {
        __stcg(part_v + parity * G + blockIdx.x, bv);
        __stcg(part_i + parity * G + blockIdx.x, bi);
      }
    }
    grid.sync();
    // ---- every CTA reduces the G partials in the same order
    if (wid == 0) {
      bv = INFINITY, bi = INT_MAX;
      for (int b = lane; b < G; b += 32) take_min(bv, bi, __ldcg(part_v + parity * G + b), __ldcg(part_i + parity * G + b));
      warp_min_idx(bv, bi);
      if (lane == 0) {
        if (prev >= 0) {                       // the previous chain element wins a tie
          const double dp = __ldcg(row + prev);
          if (dp <= bv) bv = dp, bi = prev;
        }
        s_min = bv, s_y = bi;
      }
    }
    __syncthreads();
    parity ^= 1;
    const int y = s_y;
    const double dmin = s_min;
    __syncthreads();                           // s_y / s_min are rewritten by the next step
    if (y != prev) {                           // grow the chain
      if (threadIdx.x == 0) __stcg(chain + len, y);
      ++len, prev = x, x = y;
      continue;
    }
    // ---- merge x and y into max(x, y); retire min(x, y)
    const int a = x < y ? x : y, b = x < y ? y : x;
    const double* ra = dist + (int64_t)a * ldd;
    double* rb = dist + (int64_t)b * ldd;
    if constexpr (L == Linkage::Complete) {
      for (int64_t i = beg + threadIdx.x; i < end; i += NN_THREADS) {
        if (i == a || i == b || __ldcg(size + i) == 0) continue;
        const double v = fmax(__ldcg(ra + i), __ldcg(rb + i));
        __stcg(rb + i, v);
        __stcg(dist + i * ldd + b, v);
      }
    } else {
      const double na = a == x ? nx : nprev, nb = a == x ? nprev : nx, nab = nx + nprev;
      // not unrolled: the division's slow path is a subroutine call, and the values an unrolled
      // loop keeps live across it spill
#pragma unroll 1
      for (int64_t i = beg + threadIdx.x; i < end; i += NN_THREADS) {
        if (i == a || i == b || __ldcg(size + i) == 0) continue;
        // scipy's _average, (na d_ai + nb d_bi) / (na + nb), rounded step by step: a contracted
        // FMA would round once less and break bitwise equality with scipy
        const double v = __ddiv_rn(
            __dadd_rn(__dmul_rn(na, __ldcg(ra + i)), __dmul_rn(nb, __ldcg(rb + i))), nab);
        __stcg(rb + i, v);
        __stcg(dist + i * ldd + b, v);
      }
    }
    if (blockIdx.x == 0 && threadIdx.x == 0) {   // no CTA reads size[a] or size[b] in this phase
      const int sz = __ldcg(size + a) + __ldcg(size + b);
      m_xy[2 * k] = a, m_xy[2 * k + 1] = b, m_dist[k] = dmin, m_size[k] = sz;
      __stcg(size + b, sz);
      __stcg(size + a, 0);
    }
    grid.sync();
    ++k;
    len -= 2;
    if (len > 0) {
      x = __ldcg(chain + len - 1);
      prev = len > 1 ? __ldcg(chain + len - 2) : -1;
    }
  }
}

__global__ void k_fill_ones(int* p, int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = 1;
}

// k_nn_chain's chain, scan order, tie rules and updates in one CTA, for the small matrices of a
// stream, where k_nn_chain's grid barriers cost more than the scans.  Every thread keeps the same
// chain bookkeeping; sizes and the chain live in shared memory (2 n ints), and D is read and
// written with plain loads and stores, which __syncthreads orders within the CTA.  Every branch
// below depends only on values all threads share (k, len, x, prev, y), so every thread reaches
// every barrier, up to the last merge.  *status is 1 if a chain top had no neighbour below
// infinity (non-finite D), 0 otherwise.
template <Linkage L>
__global__ void __launch_bounds__(NN_THREADS)
k_nn_chain_small(double* dist, int n, int64_t ldd, int64_t* __restrict__ m_xy,
                 double* __restrict__ m_dist, int64_t* __restrict__ m_size,
                 int* __restrict__ status) {
  extern __shared__ int ns_smem[];
  int* size = ns_smem;          // [n]
  int* chain = ns_smem + n;     // [n]
  __shared__ double red_v[NN_THREADS / 32];
  __shared__ int red_i[NN_THREADS / 32];
  __shared__ double s_min;
  __shared__ int s_y;
  for (int i = threadIdx.x; i < n; i += NN_THREADS) size[i] = 1;
  if (threadIdx.x == 0) *status = 0;
  __syncthreads();
  int len = 0, x = -1, prev = -1, lo = 0;
  for (int k = 0; k < n - 1;) {
    if (len == 0) {
      while (size[lo] == 0) ++lo;
      x = lo, prev = -1, len = 1;
      if (threadIdx.x == 0) chain[0] = x;
    }
    // a merge in this step joins x and prev: their sizes, read before thread 0 rewrites them
    const int nx = size[x], nprev = prev >= 0 ? size[prev] : 0;
    const double* row = dist + (int64_t)x * ldd;
    double bv = INFINITY;
    int bi = INT_MAX;
    for (int i = threadIdx.x; i < n; i += NN_THREADS) {
      if (i == x || size[i] == 0) continue;
      const double v = row[i];
      if (v < bv) bv = v, bi = i;
    }
    cta_min_idx(bv, bi, red_v, red_i);
    if (threadIdx.x == 0) {
      if (prev >= 0) {                         // the previous chain element wins a tie
        const double dp = row[prev];
        if (dp <= bv) bv = dp, bi = prev;
      }
      s_min = bv, s_y = bi;
    }
    // the next writes of s_y / s_min and of the staged pairs follow the next step's first barrier,
    // which every thread reaches only after reading them here
    __syncthreads();
    const int y = s_y;
    const double dmin = s_min;
    if (y == INT_MAX) {
      if (threadIdx.x == 0) *status = 1;
      return;
    }
    if (y != prev) {                           // grow the chain
      if (threadIdx.x == 0) chain[len] = y;
      ++len, prev = x, x = y;
      continue;
    }
    // ---- merge x and y into max(x, y); retire min(x, y)
    const int a = x < y ? x : y, b = x < y ? y : x;
    const double* ra = dist + (int64_t)a * ldd;
    double* rb = dist + (int64_t)b * ldd;
    const double na = a == x ? nx : nprev, nb = a == x ? nprev : nx, nab = nx + nprev;
#pragma unroll 1
    for (int i = threadIdx.x; i < n; i += NN_THREADS) {
      if (i == a || i == b || size[i] == 0) continue;
      const double v = merged_distance<L>(ra[i], rb[i], na, nb, nab);
      rb[i] = v;
      dist[i * ldd + b] = v;
    }
    if (threadIdx.x == 0) {                    // no thread reads size[a] or size[b] in this phase
      const int sz = size[a] + size[b];
      m_xy[2 * k] = a, m_xy[2 * k + 1] = b, m_dist[k] = dmin, m_size[k] = sz;
      size[b] = sz;
      size[a] = 0;
    }
    __syncthreads();
    ++k;
    len -= 2;
    if (len > 0) {
      x = chain[len - 1];
      prev = len > 1 ? chain[len - 2] : -1;
    }
  }
}

}  // namespace

extern "C" int sc_cosine_distances_f64(sc_context* ctx, const void* x, int x_is_f64, int64_t n,
                                       int64_t d, int64_t ldx, double* dist, int64_t ldd,
                                       int* nonfinite_flag, void* stream) {
  SC_REQUIRE(ctx && x && dist && nonfinite_flag && n > 0 && d > 0 && ldx >= d && ldd >= n,
             "sc_cosine_distances_f64: bad arguments");
  const int64_t tiles = (n + CD_T - 1) / CD_T;
  SC_REQUIRE(tiles <= 65535, "sc_cosine_distances_f64: n = %lld is too large", (long long)n);
  cudaStream_t st = as_stream(stream);
  Scratch nrm;
  SC_CUDA(nrm.alloc(sizeof(double) * n, st));
  SC_CUDA(cudaMemsetAsync(nonfinite_flag, 0, sizeof(int), st));
  k_row_norms<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(x, x_is_f64, n, d, ldx, nrm.as<double>());
  SC_LAUNCH_CHECK();
  k_cosine_dist<<<dim3((unsigned)tiles, (unsigned)tiles), 256, CD_SMEM, st>>>(
      x, x_is_f64, n, d, ldx, nrm.as<double>(), dist, ldd, nonfinite_flag);
  SC_LAUNCH_CHECK();
  launched(2);
  return 0;
}

namespace {

template <Linkage L>
int nn_chain_linkage(const char* name, sc_context* ctx, double* dist, int64_t n, int64_t ldd,
                     int64_t* merge_xy, double* merge_dist, int64_t* merge_size, void* stream) {
  SC_REQUIRE(ctx && dist && merge_xy && merge_dist && merge_size && n >= 2 && n < INT_MAX &&
             ldd >= n, "%s: bad arguments", name);
  cudaStream_t st = as_stream(stream);
  int per_sm = 0;
  SC_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, k_nn_chain<L>, NN_THREADS, 0));
  SC_REQUIRE(per_sm >= 1, "%s: the NN-chain kernel does not fit on an SM", name);
  // one CTA per SM: every CTA takes part in every grid barrier and reduces every partial, so
  // more CTAs would only add barrier and reduction work to an O(n) scan
  const int64_t want = (n + NN_THREADS - 1) / NN_THREADS;
  const int grid = (int)(want < ctx->sm_count ? want : ctx->sm_count);
  const int64_t m = n - 1;
  Scratch size, chain, part_v, part_i, xy, md, ms;
  SC_CUDA(size.alloc(sizeof(int) * n, st));
  SC_CUDA(chain.alloc(sizeof(int) * n, st));
  SC_CUDA(part_v.alloc(sizeof(double) * 2 * grid, st));
  SC_CUDA(part_i.alloc(sizeof(int) * 2 * grid, st));
  SC_CUDA(xy.alloc(sizeof(int64_t) * 2 * m, st));
  SC_CUDA(md.alloc(sizeof(double) * m, st));
  SC_CUDA(ms.alloc(sizeof(int64_t) * m, st));
  k_fill_ones<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(size.as<int>(), n);
  SC_LAUNCH_CHECK();
  double* d_ = dist;
  int64_t n_ = n, ldd_ = ldd;
  int* size_ = size.as<int>();
  int* chain_ = chain.as<int>();
  double* pv_ = part_v.as<double>();
  int* pi_ = part_i.as<int>();
  int64_t* xy_ = xy.as<int64_t>();
  double* md_ = md.as<double>();
  int64_t* ms_ = ms.as<int64_t>();
  void* args[] = {&d_, &n_, &ldd_, &size_, &chain_, &pv_, &pi_, &xy_, &md_, &ms_};
  SC_CUDA(cudaLaunchCooperativeKernel((const void*)k_nn_chain<L>, dim3((unsigned)grid),
                                      dim3(NN_THREADS), args, 0, st));
  launched(2);
  SC_CUDA(cudaMemcpyAsync(merge_xy, xy_, sizeof(int64_t) * 2 * m, cudaMemcpyDeviceToHost, st));
  SC_CUDA(cudaMemcpyAsync(merge_dist, md_, sizeof(double) * m, cudaMemcpyDeviceToHost, st));
  SC_CUDA(cudaMemcpyAsync(merge_size, ms_, sizeof(int64_t) * m, cudaMemcpyDeviceToHost, st));
  SC_CUDA(cudaStreamSynchronize(st));
  return 0;
}

}  // namespace

extern "C" int sc_complete_linkage(sc_context* ctx, double* dist, int64_t n, int64_t ldd,
                                   int64_t* merge_xy, double* merge_dist, int64_t* merge_size,
                                   void* stream) {
  return nn_chain_linkage<Linkage::Complete>("sc_complete_linkage", ctx, dist, n, ldd, merge_xy,
                                             merge_dist, merge_size, stream);
}

extern "C" int sc_average_linkage(sc_context* ctx, double* dist, int64_t n, int64_t ldd,
                                  int64_t* merge_xy, double* merge_dist, int64_t* merge_size,
                                  void* stream) {
  return nn_chain_linkage<Linkage::Average>("sc_average_linkage", ctx, dist, n, ldd, merge_xy,
                                            merge_dist, merge_size, stream);
}

extern "C" int sc_nn_chain_small(sc_context* ctx, double* dist, int64_t n, int64_t ldd, int linkage,
                                 int64_t* merge_xy, double* merge_dist, int64_t* merge_size,
                                 void* stream) {
  SC_REQUIRE(ctx && dist && merge_xy && merge_dist && merge_size && n >= 2 && ldd >= n &&
             (linkage == SC_LINKAGE_COMPLETE || linkage == SC_LINKAGE_AVERAGE),
             "sc_nn_chain_small: bad arguments");
  SC_REQUIRE(n <= SC_NN_SMALL_MAX, "sc_nn_chain_small: n = %lld is above SC_NN_SMALL_MAX = %d",
             (long long)n, (int)SC_NN_SMALL_MAX);
  cudaStream_t st = as_stream(stream);
  const int64_t m = n - 1;
  // one scratch: xy [2m] int64 | size [m] int64 | distance [m] fp64 | status int
  Scratch out;
  SC_CUDA(out.alloc(sizeof(int64_t) * 4 * m + sizeof(int), st));
  int64_t* xy = out.as<int64_t>();
  int64_t* ms = xy + 2 * m;
  double* md = reinterpret_cast<double*>(ms + m);
  int* status = reinterpret_cast<int*>(md + m);
  static_assert(sizeof(int) * 2 * SC_NN_SMALL_MAX <= 48 * 1024,
                "sizes and chain fit the default dynamic shared memory");
  const size_t smem = sizeof(int) * 2 * n;
  auto kernel = linkage == SC_LINKAGE_COMPLETE ? k_nn_chain_small<Linkage::Complete>
                                               : k_nn_chain_small<Linkage::Average>;
  kernel<<<1, NN_THREADS, smem, st>>>(dist, (int)n, ldd, xy, md, ms, status);
  SC_LAUNCH_CHECK();
  launched(1);
  int bad = 0;
  SC_CUDA(cudaMemcpyAsync(merge_xy, xy, sizeof(int64_t) * 2 * m, cudaMemcpyDeviceToHost, st));
  SC_CUDA(cudaMemcpyAsync(merge_dist, md, sizeof(double) * m, cudaMemcpyDeviceToHost, st));
  SC_CUDA(cudaMemcpyAsync(merge_size, ms, sizeof(int64_t) * m, cudaMemcpyDeviceToHost, st));
  SC_CUDA(cudaMemcpyAsync(&bad, status, sizeof(int), cudaMemcpyDeviceToHost, st));
  SC_CUDA(cudaStreamSynchronize(st));
  SC_REQUIRE(!bad, "sc_nn_chain_small: a chain top has no nearest neighbour (non-finite distances)");
  return 0;
}

// ---- utils.get_cluster_centroids: np.add.at into fp64 sums, then division by np.bincount ----------
namespace {

// One warp walks the labels 32 at a time.  Lanes that hold the same id find each other with
// __match_any_sync; the lowest of them moves the id's cursor past all of them, and each lane's
// rank among them is the count of lower lanes, so every cluster lists its rows in increasing order.
// Pass 1 counts, a warp scan turns counts into offsets, pass 2 scatters.  Ids outside [0, k) are
// skipped.  off has k + 1 entries, cur k.
__global__ void __launch_bounds__(32)
k_centroid_order(const int64_t* __restrict__ labels, int64_t n, int64_t k, int64_t* off,
                 int64_t* cur, int* perm) {
  const int lane = threadIdx.x;
  const unsigned lower = (1u << lane) - 1u;
  for (int64_t c = lane; c < k; c += 32) cur[c] = 0;
  __syncwarp();
  for (int pass = 0; pass < 2; ++pass) {
    for (int64_t base = 0; base < n; base += 32) {
      const int64_t i = base + lane;
      const int64_t c = i < n ? labels[i] : -1;
      const bool valid = c >= 0 && c < k;
      const unsigned same = __match_any_sync(0xffffffffu, valid ? c : (int64_t)-1);
      if (valid) {
        const int64_t at = cur[c];
        if (pass == 1) perm[at + __popc(same & lower)] = (int)i;
        __syncwarp(same);
        if ((same & lower) == 0) cur[c] = at + __popc(same);
      }
      __syncwarp();
    }
    if (pass == 0) {
      // off = exclusive prefix sum of the counts; the cursors restart at the offsets
      int64_t carry = 0;
      for (int64_t c0 = 0; c0 < k; c0 += 32) {
        const int64_t c = c0 + lane;
        const int64_t v = c < k ? cur[c] : 0;
        int64_t incl = v;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
          const int64_t u = __shfl_up_sync(0xffffffffu, incl, o);
          if (lane >= o) incl += u;
        }
        if (c < k) off[c] = cur[c] = carry + incl - v;
        carry += __shfl_sync(0xffffffffu, incl, 31);
      }
      if (lane == 0) off[k] = carry;
      __syncwarp();
    }
  }
}

// Block (cluster c, 128 columns): sequential fp64 adds of the members in increasing row index,
// starting from 0.0 as np.add.at does into np.zeros, then one division by the member count (0 / 0
// = NaN for an id with no member, as numpy gives).
template <typename T>
__global__ void __launch_bounds__(128)
k_centroid_sums(const T* __restrict__ x, int64_t d, int64_t ldx, const int64_t* __restrict__ off,
                const int* __restrict__ perm, double* __restrict__ out, int64_t ldo) {
  const int64_t c = blockIdx.x;
  const int64_t j = (int64_t)blockIdx.y * blockDim.x + threadIdx.x;
  if (j >= d) return;
  const int64_t b = off[c], e = off[c + 1];
  double s = 0.0;
#pragma unroll 8
  for (int64_t r = b; r < e; ++r) s += (double)x[(int64_t)perm[r] * ldx + j];
  out[c * ldo + j] = s / (double)(e - b);
}

}  // namespace

extern "C" int sc_cluster_centroids(sc_context* ctx, const void* x, int x_is_f64, int64_t n,
                                    int64_t d, int64_t ldx, const int64_t* labels, int64_t k,
                                    double* out, int64_t ldo, void* stream) {
  SC_REQUIRE(ctx && x && labels && out && n > 0 && d > 0 && k > 0 && ldo >= d &&
             (n == 1 || ldx >= d), "sc_cluster_centroids: bad arguments");
  SC_REQUIRE(n <= INT_MAX && k <= INT_MAX && (d + 127) / 128 <= 65535,
             "sc_cluster_centroids: n = %lld, d = %lld or k = %lld is too large", (long long)n,
             (long long)d, (long long)k);
  cudaStream_t st = as_stream(stream);
  Scratch off, cur, perm;
  SC_CUDA(off.alloc(sizeof(int64_t) * (k + 1), st));
  SC_CUDA(cur.alloc(sizeof(int64_t) * k, st));
  SC_CUDA(perm.alloc(sizeof(int) * n, st));
  k_centroid_order<<<1, 32, 0, st>>>(labels, n, k, off.as<int64_t>(), cur.as<int64_t>(),
                                     perm.as<int>());
  SC_LAUNCH_CHECK();
  const dim3 grid((unsigned)k, (unsigned)((d + 127) / 128));
  if (x_is_f64)
    k_centroid_sums<double><<<grid, 128, 0, st>>>((const double*)x, d, ldx, off.as<int64_t>(),
                                                  perm.as<int>(), out, ldo);
  else
    k_centroid_sums<float><<<grid, 128, 0, st>>>((const float*)x, d, ldx, off.as<int64_t>(),
                                                 perm.as<int>(), out, ldo);
  SC_LAUNCH_CHECK();
  launched(2);
  return 0;
}
