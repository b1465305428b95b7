// The online "naive" clusterer (naive_clusterer.NaiveClusterer.predict over a whole sequence) in one
// launch of one thread-block cluster:
//   k_naive<T>   the open centroids are dealt round-robin over the cluster's CTAs (centroid c lives
//                in CTA c % G, slot c / G) and kept as fp64 running means in shared memory, or in the
//                caller's means buffer for slots beyond shared-memory capacity.  One step per
//                embedding: every warp scores its centroids (one warp per cosine), one block-level
//                argmax per CTA, the G partial argmaxes are exchanged over DSMEM behind one
//                barrier.cluster, and every warp of every CTA reduces them in the same order, so all
//                agree on the decision without a broadcast.  The owner CTA then opens or merges the
//                centroid.  The next embedding is fetched with cp.async while the current one is
//                scored.  No grid barrier, no host round trip per embedding.
#include "common.cuh"

#include <climits>
#include <cooperative_groups.h>

namespace cg = cooperative_groups;
using namespace sc;

namespace {

constexpr int NV_THREADS = 512;
constexpr int NV_WARPS = NV_THREADS / 32;
constexpr int NV_MAX_CTAS = 16;          // the largest (non-portable) thread-block cluster on sm_90
constexpr int NV_CTA_CENTROIDS = 64;     // centroids per CTA before another CTA joins the cluster

// The order of np.max / np.argmax over the cosines: a NaN is above every number (np.max returns
// it, np.argmax picks the first one), then the larger value, then the lower index.  It is a total
// order on distinct indices, so an argmax reduced in any order gives the same winner.
__device__ __forceinline__ bool ahead(double v, int i, double bv, int bi) {
  const bool n = isnan(v), bn = isnan(bv);
  if (n != bn) return n;
  if (!n && v != bv) return v > bv;
  return i < bi;
}

__device__ __forceinline__ void warp_argmax(double& v, int& i) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const double ov = __shfl_xor_sync(0xffffffffu, v, o);
    const int oi = __shfl_xor_sync(0xffffffffu, i, o);
    if (ahead(ov, oi, v, i)) v = ov, i = oi;
  }
}

template <int BYTES>
__device__ __forceinline__ void cp_async(void* smem, const void* gmem) {
  const unsigned s = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.ca.shared.global [%0], [%1], %2;" ::"r"(s), "l"(gmem), "n"(BYTES) : "memory");
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait_all() { asm volatile("cp.async.wait_all;" ::: "memory"); }

struct NaiveParams {
  const void* x;
  int64_t n, d, ldx;
  double threshold, adaptation;
  int64_t stop_at;           // > 0: stop before an embedding once this many clusters are open
  double* means;             // [capacity, ldm]: initial state in rows [0, c0); home of the centroids
  int64_t ldm;               //   that do not fit in shared memory
  int64_t* counts;           // [capacity]
  int64_t capacity, c0;
  double* norms;             // [capacity] scratch: |m_c|
  int64_t* labels;           // [n]
  int64_t* out;              // [3]: embeddings processed, clusters, 1 if the capacity was exceeded
  int slots;                 // centroid slots in each CTA's shared memory
};

// Sum of squares / dot product of one warp: lane l takes elements l, l + 32, ...; the xor-butterfly
// leaves the same (commutative) sum in every lane, and every warp of every CTA that evaluates it on
// the same data gets the same bits.
template <typename A, typename B>
__device__ __forceinline__ double warp_dot(const A* a, const B* b, int64_t d, int lane) {
  double s = 0.0;
  for (int64_t k = lane; k < d; k += 32) s = fma((double)a[k], (double)b[k], s);
  return warp_sum(s);
}

template <typename T>
__global__ void __launch_bounds__(NV_THREADS, 1)
k_naive(const NaiveParams p) {
  cg::cluster_group cluster = cg::this_cluster();
  extern __shared__ __align__(16) double nv_smem[];
  __shared__ double red_v[NV_WARPS];
  __shared__ int red_i[NV_WARPS];
  __shared__ double part_v[2];             // this CTA's argmax of a step (double-buffered), read
  __shared__ int part_i[2];                // by every CTA of the cluster over DSMEM
  const int G = (int)cluster.num_blocks(), rank = (int)cluster.block_rank();
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t d = p.d;
  double* slot_means = nv_smem;                                   // [slots][d]
  T* ebuf = reinterpret_cast<T*>(nv_smem + (int64_t)p.slots * d);  // [2][d]
  const T* x = reinterpret_cast<const T*>(p.x);
  auto row = [&](int64_t c) -> double* {                          // storage of a centroid this CTA owns
    const int64_t s = c / G;
    return s < p.slots ? slot_means + s * d : p.means + c * p.ldm;
  };

  // ---- initial state: this CTA's centroids into shared memory, and their norms
  for (int64_t c = rank; c < p.c0; c += G) {
    if (c / G >= p.slots) break;
    double* m = row(c);
    for (int64_t k = threadIdx.x; k < d; k += NV_THREADS) m[k] = p.means[c * p.ldm + k];
  }
  __syncthreads();
  for (int64_t c = rank + (int64_t)G * warp; c < p.c0; c += (int64_t)G * NV_WARPS) {
    const double* m = row(c);
    const double ss = warp_dot(m, m, d, lane);
    if (lane == 0) p.norms[c] = sqrt(ss);
  }
  for (int64_t k = threadIdx.x; k < d; k += NV_THREADS) cp_async<sizeof(T)>(ebuf + k, x + k);
  cp_async_commit();

  int64_t C = p.c0, t = 0;
  int parity = 0, overflow = 0;
  for (; t < p.n; ++t) {
    if (p.stop_at > 0 && C >= p.stop_at) break;
    cp_async_wait_all();
    __syncthreads();              // e_t has landed; the previous step is done with e_{t-1}'s buffer
    const T* e = ebuf + (t & 1) * d;
    if (t + 1 < p.n) {
      T* nxt = ebuf + ((t + 1) & 1) * d;
      const T* src = x + (t + 1) * p.ldx;
      for (int64_t k = threadIdx.x; k < d; k += NV_THREADS) cp_async<sizeof(T)>(nxt + k, src + k);
    }
    cp_async_commit();
    const double ne = sqrt(warp_dot(e, e, d, lane));
    // ---- cosine of every owned centroid: cos_c = (m_c . e) / (|m_c| |e|), as numpy evaluates it
    double bv = -INFINITY;
    int bi = INT_MAX;
    for (int64_t c = rank + (int64_t)G * warp; c < C; c += (int64_t)G * NV_WARPS) {
      const double dot = warp_dot(row(c), e, d, lane);
      const double cs = dot / (p.norms[c] * ne);
      if (ahead(cs, (int)c, bv, bi)) bv = cs, bi = (int)c;
    }
    if (lane == 0) red_v[warp] = bv, red_i[warp] = bi;
    __syncthreads();
    if (warp == 0) {
      bv = lane < NV_WARPS ? red_v[lane] : -INFINITY;
      bi = lane < NV_WARPS ? red_i[lane] : INT_MAX;
      warp_argmax(bv, bi);
      if (lane == 0) part_v[parity] = bv, part_i[parity] = bi;
    }
    // The partials are double-buffered: a CTA rewrites part[parity] two steps later, after the next
    // barrier, which every CTA reaches only once it has read this step's partials.
    cluster.sync();
    bv = lane < G ? *cluster.map_shared_rank(part_v + parity, lane) : -INFINITY;
    bi = lane < G ? *cluster.map_shared_rank(part_i + parity, lane) : INT_MAX;
    warp_argmax(bv, bi);
    parity ^= 1;
    // ---- the decision (identical in every warp of every CTA)
    const bool open = C == 0 || bv < p.threshold;        // a NaN maximum neither opens ...
    const int64_t label = open ? C : bi;
    if (open) {
      if (C == p.capacity) { overflow = 1; break; }
      if (rank == (int)(C % G)) {
        double* m = row(C);
        for (int64_t k = threadIdx.x; k < d; k += NV_THREADS) m[k] = (double)e[k];
        if (threadIdx.x == 0) p.norms[C] = ne, p.counts[C] = 1;
      }
      ++C;
    } else if (bv > p.adaptation && rank == (int)(label % G)) {   // ... nor merges
      double* m = row(label);
      const int64_t cnt = p.counts[label];
      const double a = (double)cnt, b = (double)(cnt + 1);
      // (m count + e) / (count + 1) rounded step by step like numpy: no contraction into an FMA
      for (int64_t k = threadIdx.x; k < d; k += NV_THREADS)
        m[k] = __ddiv_rn(__dadd_rn(__dmul_rn(m[k], a), (double)e[k]), b);
      __syncthreads();
      if (warp == 0) {
        const double ss = warp_dot(m, m, d, lane);
        if (lane == 0) p.norms[label] = sqrt(ss), p.counts[label] = cnt + 1;
      }
    }
    if (rank == 0 && threadIdx.x == 0) p.labels[t] = label;
  }
  cp_async_wait_all();
  __syncthreads();
  // ---- centroids held in shared memory back to the caller's means
  for (int64_t c = rank; c < C; c += G) {
    if (c / G >= p.slots) break;
    const double* m = row(c);
    for (int64_t k = threadIdx.x; k < d; k += NV_THREADS) p.means[c * p.ldm + k] = m[k];
  }
  if (rank == 0 && threadIdx.x == 0) p.out[0] = t, p.out[1] = C, p.out[2] = overflow;
  cluster.sync();                 // no CTA leaves while another may still read its partials
}

template <typename T>
int naive_launch(sc_context* ctx, NaiveParams p, cudaStream_t st) {
  // the most clusters this call can ever hold sizes the cluster of CTAs and their slots
  int64_t cmax = p.c0 + p.n;
  if (p.stop_at > 0) cmax = p.stop_at > p.c0 ? p.stop_at : p.c0;
  if (cmax > p.capacity) cmax = p.capacity;
  if (cmax < 1) cmax = 1;
  const size_t ebytes = 2 * (size_t)p.d * sizeof(T);
  const size_t reserve = 1024;            // static shared memory and the per-CTA system share
  SC_REQUIRE(ctx->smem_optin > ebytes + reserve, "sc_naive_cluster: d = %lld is too large",
             (long long)p.d);
  const int64_t max_slots = (int64_t)((ctx->smem_optin - ebytes - reserve) / (8 * (size_t)p.d));
  const void* fn = (const void*)k_naive<T>;
  SC_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
  int64_t want = (cmax + NV_CTA_CENTROIDS - 1) / NV_CTA_CENTROIDS;
  int G = (int)(want < NV_MAX_CTAS ? want : NV_MAX_CTAS);
  // Results do not depend on G (every cosine is one warp's fixed-order sum and the argmax order is
  // total), so a cluster the device cannot co-schedule is never launched: it is halved instead.
  for (;; G /= 2) {
    SC_REQUIRE(G >= 1, "sc_naive_cluster: not even a single-CTA cluster fits on an SM");
    const int64_t per = (cmax + G - 1) / G;
    p.slots = (int)(per < max_slots ? per : max_slots);
    const size_t smem = ebytes + 8 * (size_t)p.slots * (size_t)p.d;
    SC_CUDA(cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    cudaLaunchConfig_t cfg = {};
    cudaLaunchAttribute attr[1];
    attr[0].id = cudaLaunchAttributeClusterDimension;
    attr[0].val.clusterDim.x = (unsigned)G, attr[0].val.clusterDim.y = 1, attr[0].val.clusterDim.z = 1;
    cfg.gridDim = dim3((unsigned)G), cfg.blockDim = dim3(NV_THREADS);
    cfg.dynamicSmemBytes = smem, cfg.stream = st, cfg.attrs = attr, cfg.numAttrs = 1;
    int clusters = 0;
    SC_CUDA(cudaOccupancyMaxActiveClusters(&clusters, fn, &cfg));
    if (clusters < 1) continue;
    SC_CUDA(cudaLaunchKernelEx(&cfg, k_naive<T>, p));
    launched();
    return 0;
  }
}

}  // namespace

extern "C" int sc_naive_cluster(sc_context* ctx, const void* x, int x_is_f64, int64_t n, int64_t d,
                                int64_t ldx, double threshold, double adaptation_threshold,
                                int64_t stop_at, double* means, int64_t ldm, int64_t* counts,
                                int64_t capacity, int64_t initial_clusters, int64_t* labels,
                                int64_t* processed_host, int64_t* clusters_host, void* stream) {
  SC_REQUIRE(ctx && processed_host && clusters_host && n >= 0 && d > 0 && ldm >= d &&
                 initial_clusters >= 0 && capacity >= initial_clusters && capacity < INT_MAX &&
                 (n == 0 || (x && ldx >= d && labels)) && (capacity == 0 || (means && counts)),
             "sc_naive_cluster: bad arguments");
  cudaStream_t st = as_stream(stream);
  *processed_host = 0, *clusters_host = initial_clusters;
  if (n == 0) return 0;
  Scratch norms, out;
  SC_CUDA(norms.alloc(sizeof(double) * (capacity > 0 ? capacity : 1), st));
  SC_CUDA(out.alloc(sizeof(int64_t) * 3, st));
  NaiveParams p{x, n, d, ldx, threshold, adaptation_threshold, stop_at, means, ldm, counts,
                capacity, initial_clusters, norms.as<double>(), labels, out.as<int64_t>(), 0};
  const int rc = x_is_f64 ? naive_launch<double>(ctx, p, st) : naive_launch<float>(ctx, p, st);
  if (rc != 0) return rc;
  SC_LAUNCH_CHECK();
  int64_t res[3];
  SC_CUDA(cudaMemcpyAsync(res, out.as<int64_t>(), sizeof(res), cudaMemcpyDeviceToHost, st));
  SC_CUDA(cudaStreamSynchronize(st));
  SC_REQUIRE(res[2] == 0, "sc_naive_cluster: more than capacity = %lld clusters",
             (long long)capacity);
  *processed_host = res[0], *clusters_host = res[1];
  return 0;
}
