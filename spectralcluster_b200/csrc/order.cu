// Row order of the bounded Diffuse (DESIGN.md section 3), entirely on the device: spherical
// k-means (k <= 16) in fp32 on the rows' group-norm profiles, then a stable counting sort by label.  The
// order only decides which tiles of S = Y Y^T the bounded Diffuse skips, never a value, so no
// particular clustering is owed; what is owed is the same order on every call (reproducible tile
// counts and timings) and no host synchronisation between Y and the tile GEMM.
//
//   seeding     greedy farthest point from row 0: centre j is the first row of least cosine to its
//               nearest earlier centre (one pass over the profiles per centre)
//   passes      assign every row to the centre of largest cosine (first on ties), then each centre
//               becomes the normalised sum of its rows' unit profiles, summed per row chunk and
//               the chunks in order (no floating-point atomics); an empty cluster keeps its centre
//   sort        stable counting sort of the last labels: per-chunk counts, one exclusive scan in
//               (label, chunk) order, a rank inside the chunk from warp match masks
// Profiles that are all alike only repeat the first centre: every row then takes label 0 and the
// order is the natural one.
#include "common.cuh"

namespace sc {

constexpr int ORDER_MAXK = 16;
constexpr int ORDER_CHUNK = 256;   // rows per CTA of the assignment and sort kernels (8 warps)
constexpr int ORDER_UNROLL = 8;    // loads of a profile row a lane keeps in flight (G = 256: all)
constexpr int ORDER_ROWS = 4;      // rows a warp of the scan kernels has in flight

// rn[i] = 1 / |x_i| (0 for an all-zero profile); best[i] = cosine of row i to centre 0 = unit row 0
__global__ void __launch_bounds__(256) k_order_seed0(const float* __restrict__ x, int64_t n, int G,
                                                     float* __restrict__ rn, float* __restrict__ c) {
  const int64_t i = (int64_t)blockIdx.x * 8 + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (i >= n) return;
  float s = 0.f;
  for (int g0 = 0; g0 < G; g0 += 32 * ORDER_UNROLL) {
    float v[ORDER_UNROLL];
#pragma unroll
    for (int u = 0; u < ORDER_UNROLL; ++u) {
      const int g = g0 + lane + 32 * u;
      v[u] = g < G ? x[i * G + g] : 0.f;
    }
#pragma unroll
    for (int u = 0; u < ORDER_UNROLL; ++u) s = fmaf(v[u], v[u], s);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  const float r = s > 0.f ? rsqrtf(s) : 0.f;
  if (lane == 0) rn[i] = r;
  if (i == 0)
    for (int g = lane; g < G; g += 32) c[g] = x[g] * r;
}

// best[i] = max(best[i], cos(x_i, centre j-1)) (j == 1: the cosine itself); then the first row
// of least best in this CTA's rows -> part[blockIdx.x] = (value, row)
__global__ void __launch_bounds__(256) k_order_seed_scan(const float* __restrict__ x, int64_t n, int G,
                                                         const float* __restrict__ rn,
                                                         const float* __restrict__ cj, int first,
                                                         float* __restrict__ best,
                                                         float2* __restrict__ part) {
  __shared__ float sv[8];
  __shared__ int64_t si[8];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float bv = INFINITY;
  int64_t bi = n;
  for (int r = warp * ORDER_ROWS; r < ORDER_CHUNK; r += 8 * ORDER_ROWS) {
    const int64_t i0 = (int64_t)blockIdx.x * ORDER_CHUNK + r;
    if (i0 >= n) break;
    float s[ORDER_ROWS];
#pragma unroll
    for (int q = 0; q < ORDER_ROWS; ++q) s[q] = 0.f;
    for (int g0 = 0; g0 < G; g0 += 32 * ORDER_UNROLL) {
      float v[ORDER_ROWS][ORDER_UNROLL];                // the rows' loads in flight together
#pragma unroll
      for (int q = 0; q < ORDER_ROWS; ++q)
#pragma unroll
        for (int u = 0; u < ORDER_UNROLL; ++u) {
          const int g = g0 + lane + 32 * u;
          v[q][u] = (g < G && i0 + q < n) ? x[(i0 + q) * G + g] : 0.f;
        }
#pragma unroll
      for (int u = 0; u < ORDER_UNROLL; ++u) {
        const int g = g0 + lane + 32 * u;
        if (g < G) {
          const float cg = cj[g];
#pragma unroll
          for (int q = 0; q < ORDER_ROWS; ++q) s[q] = fmaf(v[q][u], cg, s[q]);
        }
      }
    }
#pragma unroll
    for (int q = 0; q < ORDER_ROWS; ++q) {
      const int64_t i = i0 + q;
      if (i >= n) break;
      float sq = s[q];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) sq += __shfl_xor_sync(0xffffffffu, sq, o);
      sq *= rn[i];
      const float v = first ? sq : fmaxf(best[i], sq);
      if (lane == 0) best[i] = v;
      if (v < bv) { bv = v; bi = i; }                   // a warp's rows in increasing order: first on ties
    }
  }
  if (lane == 0) { sv[warp] = bv; si[warp] = bi; }
  __syncthreads();
  if (threadIdx.x == 0) {
    for (int w = 1; w < 8; ++w)
      if (sv[w] < sv[0] || (sv[w] == sv[0] && si[w] < si[0])) { sv[0] = sv[w]; si[0] = si[w]; }
    part[blockIdx.x] = make_float2(sv[0], __int_as_float((int)si[0]));
  }
}

// centre j = the unit profile of the first row of least best over all CTAs' candidates
__global__ void __launch_bounds__(256) k_order_seed_pick(const float* __restrict__ x, int G,
                                                         const float* __restrict__ rn,
                                                         const float2* __restrict__ part, int parts,
                                                         float* __restrict__ cj) {
  __shared__ float sv[8];
  __shared__ int si[8];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  float bv = INFINITY;
  int bi = 0x7fffffff;
  for (int p = threadIdx.x; p < parts; p += blockDim.x) {
    const float v = part[p].x;
    const int i = __float_as_int(part[p].y);
    if (v < bv || (v == bv && i < bi)) { bv = v; bi = i; }
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {                    // (value, row) is a total order: any tree
    const float v = __shfl_xor_sync(0xffffffffu, bv, o);
    const int i = __shfl_xor_sync(0xffffffffu, bi, o);
    if (v < bv || (v == bv && i < bi)) { bv = v; bi = i; }
  }
  if (lane == 0) { sv[warp] = bv; si[warp] = bi; }
  __syncthreads();
  bv = sv[0];
  bi = si[0];
  for (int w = 1; w < 8; ++w)
    if (sv[w] < bv || (sv[w] == bv && si[w] < bi)) { bv = sv[w]; bi = si[w]; }
  const int64_t i = bi;
  for (int g = threadIdx.x; g < G; g += blockDim.x) cj[g] = x[i * G + g] * rn[i];
}

// labels of this CTA's rows (largest cosine, first centre on ties), and with `part` the per-centre
// sums of their unit profiles: part[blockIdx.x][j][g], each column summed by one thread in row order
__global__ void __launch_bounds__(256) k_order_assign(const float* __restrict__ x, int64_t n, int G, int k,
                                                      const float* __restrict__ rn,
                                                      const float* __restrict__ c,
                                                      int* __restrict__ labels,
                                                      float* __restrict__ part) {
  extern __shared__ float order_smem[];                 // centres [k][G], then sums [k][G]
  __shared__ int lab[ORDER_CHUNK];
  float* cs = order_smem;
  float* acc = order_smem + (size_t)k * G;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t r0 = (int64_t)blockIdx.x * ORDER_CHUNK;
  const int rows = (int)min((int64_t)ORDER_CHUNK, n - r0);
  for (int e = threadIdx.x; e < k * G; e += blockDim.x) {
    cs[e] = c[e];
    acc[e] = 0.f;
  }
  __syncthreads();
  for (int r = 2 * warp; r < rows; r += 16) {           // two rows per warp in flight
    const int nr = min(2, rows - r);
    const float* xr = x + (r0 + r) * G;
    float d[2][ORDER_MAXK];
#pragma unroll
    for (int q = 0; q < 2; ++q)
#pragma unroll
      for (int j = 0; j < ORDER_MAXK; ++j) d[q][j] = 0.f;
    for (int g0 = 0; g0 < G; g0 += 32 * ORDER_UNROLL) {
      float v[2][ORDER_UNROLL];
#pragma unroll
      for (int q = 0; q < 2; ++q)
#pragma unroll
        for (int u = 0; u < ORDER_UNROLL; ++u) {
          const int g = g0 + lane + 32 * u;
          v[q][u] = (g < G && q < nr) ? xr[q * G + g] : 0.f;
        }
#pragma unroll
      for (int u = 0; u < ORDER_UNROLL; ++u) {
        const int g = g0 + lane + 32 * u;
        if (g < G) {
#pragma unroll
          for (int j = 0; j < ORDER_MAXK; ++j) {
            if (j < k) {
              const float cg = cs[j * G + g];
              d[0][j] = fmaf(v[0][u], cg, d[0][j]);
              d[1][j] = fmaf(v[1][u], cg, d[1][j]);
            }
          }
        }
      }
    }
#pragma unroll
    for (int q = 0; q < 2; ++q) {
      int bj = 0;
      float bv = -INFINITY;
#pragma unroll
      for (int j = 0; j < ORDER_MAXK; ++j) {
        if (j < k) {
          float s = d[q][j];
#pragma unroll
          for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
          if (s > bv) { bv = s; bj = j; }
        }
      }
      if (lane == 0 && q < nr) {
        lab[r + q] = bj;
        labels[r0 + r + q] = bj;
      }
    }
  }
  if (!part) return;
  __syncthreads();
  for (int g = threadIdx.x; g < G; g += blockDim.x)
    for (int r = 0; r < rows; r += 16) {
      float v[16];                                      // 16 loads in flight, then the sums in row order
#pragma unroll
      for (int u = 0; u < 16; ++u) v[u] = r + u < rows ? x[(r0 + r + u) * G + g] * rn[r0 + r + u] : 0.f;
#pragma unroll
      for (int u = 0; u < 16; ++u)
        if (r + u < rows) acc[lab[r + u] * G + g] += v[u];
    }
  __syncthreads();
  float* out = part + (size_t)blockIdx.x * k * G;
  for (int e = threadIdx.x; e < k * G; e += blockDim.x) out[e] = acc[e];
}

// centre j (= blockIdx.x) <- the normalised sum of the chunks' sums, chunks in order; kept when empty
__global__ void __launch_bounds__(256) k_order_update(const float* __restrict__ part, int parts, int G, int k,
                                                      float* __restrict__ c) {
  extern __shared__ float order_smem[];                 // the summed centre [G]
  __shared__ float red[8];
  const int j = blockIdx.x;
  float ss = 0.f;
  for (int g = threadIdx.x; g < G; g += blockDim.x) {
    float s = 0.f;
#pragma unroll 16
    for (int p = 0; p < parts; ++p) s += part[((size_t)p * k + j) * G + g];
    order_smem[g] = s;
    ss = fmaf(s, s, ss);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) ss += __shfl_xor_sync(0xffffffffu, ss, o);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = ss;
  __syncthreads();
  float tot = 0.f;
  for (int w = 0; w < 8; ++w) tot += red[w];
  if (!(tot > 0.f)) return;
  const float inv = rsqrtf(tot);
  for (int g = threadIdx.x; g < G; g += blockDim.x) c[(size_t)j * G + g] = order_smem[g] * inv;
}

// stable rank of each row of this CTA's chunk among the chunk's rows of its label; with `base`
// null, only counts[blockIdx.x][label]; otherwise perm[base[blockIdx.x][label] + rank] = row
__global__ void __launch_bounds__(ORDER_CHUNK) k_order_rank(const int* __restrict__ labels, int64_t n, int k,
                                                            int* __restrict__ counts,
                                                            const int* __restrict__ base,
                                                            int* __restrict__ perm) {
  __shared__ int wc[8][ORDER_MAXK];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t i = (int64_t)blockIdx.x * ORDER_CHUNK + threadIdx.x;
  const int l = i < n ? labels[i] : ORDER_MAXK;       // past n: a label of its own, never counted
  for (int e = threadIdx.x; e < 8 * ORDER_MAXK; e += blockDim.x) wc[e / ORDER_MAXK][e % ORDER_MAXK] = 0;
  __syncthreads();
  const unsigned same = __match_any_sync(0xffffffffu, l);
  const int rank = __popc(same & ((1u << lane) - 1u));
  if (l < ORDER_MAXK && rank == 0) wc[warp][l] = __popc(same);
  __syncthreads();
  if (!base) {
    if (threadIdx.x < k) {
      int s = 0;
      for (int w = 0; w < 8; ++w) s += wc[w][threadIdx.x];
      counts[(size_t)blockIdx.x * k + threadIdx.x] = s;
    }
    return;
  }
  if (i >= n) return;
  int before = 0;
  for (int w = 0; w < warp; ++w) before += wc[w][l];
  perm[base[(size_t)blockIdx.x * k + l] + before + rank] = (int)i;
}

// base[chunk][j] = (rows of labels < j) + (rows of label j in earlier chunks): one CTA, k threads
__global__ void k_order_scan(const int* __restrict__ counts, int chunks, int k, int* __restrict__ base) {
  __shared__ int tot[ORDER_MAXK];
  const int j = threadIdx.x;
  int s = 0;
  if (j < k)
#pragma unroll 8
    for (int p = 0; p < chunks; ++p) {
      base[(size_t)p * k + j] = s;
      s += counts[(size_t)p * k + j];
    }
  if (j < ORDER_MAXK) tot[j] = s;
  __syncthreads();
  if (j >= k) return;
  int off = 0;
  for (int q = 0; q < j; ++q) off += tot[q];
#pragma unroll 8
  for (int p = 0; p < chunks; ++p) base[(size_t)p * k + j] += off;
}

// ---- hub-first order (sc_bound_order_hubs): within each cluster, rows by diagonal descending.
// Key = label (bits 52..55) | complement of the fp32 diagonal rounded down (bits 21..51) | row
// (bits 0..20): ascending keys are (label, diagonal descending, row), distinct for every row.
constexpr int HUB_SORT_LOCAL = 2048;   // keys a CTA sorts or merges in shared memory (1024 threads)

__global__ void k_hub_keys(const int* __restrict__ labels, const double* __restrict__ diag,
                           int64_t n, int64_t P, unsigned long long* __restrict__ keys) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P) return;
  if (i >= n) { keys[i] = ~0ull; return; }
  const unsigned d = __float_as_uint(__double2float_rd(diag[i])) & 0x7fffffffu;
  keys[i] = ((unsigned long long)labels[i] << 52) |
            ((unsigned long long)(0x7fffffffu - d) << 21) | (unsigned long long)i;
}

__device__ __forceinline__ void hub_cas(unsigned long long* s, int i, int j, bool asc) {
  const unsigned long long a = s[i], b = s[j];
  if ((a > b) == asc) { s[i] = b; s[j] = a; }
}

// bitonic steps with partner distance < L = min(P, HUB_SORT_LOCAL) in shared memory: stages
// 2..L from scratch (merge_k == 0), or the tail j = L/2 .. 1 of stage merge_k
__global__ void __launch_bounds__(1024) k_hub_sort_local(unsigned long long* __restrict__ keys,
                                                         int64_t P, int64_t merge_k) {
  __shared__ unsigned long long s[HUB_SORT_LOCAL];
  const int L = (int)min(P, (int64_t)HUB_SORT_LOCAL);
  const int64_t base = (int64_t)blockIdx.x * L;
  for (int i = threadIdx.x; i < L; i += blockDim.x) s[i] = keys[base + i];
  __syncthreads();
  for (int64_t k = merge_k ? merge_k : 2; k <= (merge_k ? merge_k : (int64_t)L); k <<= 1) {
    for (int j = (int)min(k >> 1, (int64_t)L >> 1); j > 0; j >>= 1) {
      for (int i = threadIdx.x; i < L; i += blockDim.x) {
        const int p = i ^ j;
        if (p > i) hub_cas(s, i, p, ((base + i) & k) == 0);
      }
      __syncthreads();
    }
  }
  for (int i = threadIdx.x; i < L; i += blockDim.x) keys[base + i] = s[i];
}

// one bitonic step of stage k at partner distance j >= HUB_SORT_LOCAL, in global memory
__global__ void k_hub_sort_step(unsigned long long* __restrict__ keys, int64_t P, int64_t k,
                                int64_t j) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= P) return;
  const int64_t p = i ^ j;
  if (p > i) {
    const unsigned long long a = keys[i], b = keys[p];
    if ((a > b) == ((i & k) == 0)) { keys[i] = b; keys[p] = a; }
  }
}

// perm = the rows of the sorted keys; starts[j] = base[0][j] (rows of labels < j), starts[k] = n
__global__ void k_hub_finish(const unsigned long long* __restrict__ keys, int64_t n,
                             const int* __restrict__ base, int k, int* __restrict__ perm,
                             int* __restrict__ starts) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) perm[i] = (int)(keys[i] & 0x1fffffull);
  if (i <= k) starts[i] = i < k ? base[i] : (int)n;
}

// The k-means of both orders: labels[i] of every row, with the seeding and passes described at
// the top of this file.  `buf` receives the scratch; labels, counts and base point into it.
struct OrderScratch {
  Scratch buf;
  int* labels;
  int* counts;
  int* base;
  int chunks;
};

static int order_labels(sc_context* ctx, const char* who, const float* norms, int64_t n,
                        int64_t groups, int k, int passes, size_t extra, OrderScratch& o,
                        cudaStream_t st) {
  const size_t smem = sizeof(float) * 2 * (size_t)k * (size_t)groups;
  SC_REQUIRE(smem <= ctx->smem_optin - 2 * sizeof(int) * ORDER_CHUNK,
             "%s: %d centres of %lld groups do not fit in shared memory", who, k, (long long)groups);
  const int G = (int)groups;
  const int chunks = (int)((n + ORDER_CHUNK - 1) / ORDER_CHUNK);
  const size_t cbytes = sizeof(float) * (size_t)k * G;
  const size_t pbytes = cbytes * (size_t)chunks;
  SC_CUDA(o.buf.alloc(extra + cbytes + pbytes + sizeof(float) * 2 * (size_t)n + sizeof(int) * (size_t)n +
                          sizeof(float2) * chunks + sizeof(int) * 2 * (size_t)chunks * k + 64, st));
  char* p = o.buf.as<char>() + extra;
  float* c = reinterpret_cast<float*>(p);                     p += cbytes;
  float* part = reinterpret_cast<float*>(p);                  p += pbytes;
  float* rn = reinterpret_cast<float*>(p);                    p += sizeof(float) * n;
  float* best = reinterpret_cast<float*>(p);                  p += sizeof(float) * n;
  int* labels = reinterpret_cast<int*>(p);                    p += sizeof(int) * n;
  p = reinterpret_cast<char*>((reinterpret_cast<uintptr_t>(p) + 15) & ~(uintptr_t)15);
  float2* cand = reinterpret_cast<float2*>(p);                p += sizeof(float2) * chunks;
  int* counts = reinterpret_cast<int*>(p);                    p += sizeof(int) * (size_t)chunks * k;
  int* base = reinterpret_cast<int*>(p);
  o.labels = labels;
  o.counts = counts;
  o.base = base;
  o.chunks = chunks;

  k_order_seed0<<<(unsigned)((n + 7) / 8), 256, 0, st>>>(norms, n, G, rn, c); sc::launched();
  for (int j = 1; j < k; ++j) {
    k_order_seed_scan<<<(unsigned)chunks, 256, 0, st>>>(norms, n, G, rn, c + (size_t)(j - 1) * G,
                                                         j == 1, best, cand); sc::launched();
    k_order_seed_pick<<<1, 256, 0, st>>>(norms, G, rn, cand, chunks, c + (size_t)j * G); sc::launched();
  }
  SC_CUDA(cudaFuncSetAttribute(k_order_assign, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  SC_CUDA(cudaFuncSetAttribute(k_order_update, cudaFuncAttributeMaxDynamicSharedMemorySize,
                               (int)(sizeof(float) * G)));
  for (int it = 0; it < passes; ++it) {
    const bool last = it == passes - 1;
    k_order_assign<<<(unsigned)chunks, 256, smem, st>>>(norms, n, G, k, rn, c, labels,
                                                        last ? nullptr : part); sc::launched();
    if (!last) {
      k_order_update<<<(unsigned)k, 256, sizeof(float) * G, st>>>(part, chunks, G, k, c); sc::launched();
    }
  }
  // per-chunk label counts and their exclusive scan in (label, chunk) order
  k_order_rank<<<(unsigned)chunks, ORDER_CHUNK, 0, st>>>(labels, n, k, counts, nullptr, nullptr); sc::launched();
  k_order_scan<<<1, ORDER_MAXK, 0, st>>>(counts, chunks, k, base); sc::launched();
  return 0;
}

}  // namespace sc

using namespace sc;

extern "C" int sc_bound_order(sc_context* ctx, const float* norms, int64_t n, int64_t groups, int k,
                              int passes, int* perm, void* stream) {
  SC_REQUIRE(ctx && norms && perm && n > 0 && n <= (1LL << 30) && groups > 0 && k >= 1 &&
             k <= ORDER_MAXK && passes >= 1, "sc_bound_order: bad arguments");
  cudaStream_t st = as_stream(stream);
  OrderScratch o;
  if (int r = order_labels(ctx, "sc_bound_order", norms, n, groups, k, passes, 0, o, st)) return r;
  k_order_rank<<<(unsigned)o.chunks, ORDER_CHUNK, 0, st>>>(o.labels, n, k, nullptr, o.base, perm); sc::launched();
  SC_LAUNCH_CHECK();
  return 0;
}

extern "C" int sc_bound_order_hubs(sc_context* ctx, const float* norms, int64_t n, int64_t groups,
                                   int k, int passes, const double* diag, int* perm, int* starts,
                                   void* stream) {
  SC_REQUIRE(ctx && norms && diag && perm && starts && n > 0 && n <= (1LL << 21) && groups > 0 &&
             k >= 1 && k <= ORDER_MAXK && passes >= 1, "sc_bound_order_hubs: bad arguments");
  cudaStream_t st = as_stream(stream);
  int64_t P = 2;
  while (P < n) P <<= 1;
  const size_t kbytes = sizeof(unsigned long long) * (size_t)P;
  OrderScratch o;
  if (int r = order_labels(ctx, "sc_bound_order_hubs", norms, n, groups, k, passes, kbytes, o, st))
    return r;
  unsigned long long* keys = o.buf.as<unsigned long long>();
  k_hub_keys<<<(unsigned)((P + 255) / 256), 256, 0, st>>>(o.labels, diag, n, P, keys); sc::launched();
  const int64_t L = P < HUB_SORT_LOCAL ? P : HUB_SORT_LOCAL;
  const unsigned blocks = (unsigned)(P / L);
  k_hub_sort_local<<<blocks, 1024, 0, st>>>(keys, P, 0); sc::launched();
  for (int64_t kk = 2 * L; kk <= P; kk <<= 1) {
    for (int64_t j = kk >> 1; j >= L; j >>= 1) {
      k_hub_sort_step<<<(unsigned)((P + 255) / 256), 256, 0, st>>>(keys, P, kk, j); sc::launched();
    }
    k_hub_sort_local<<<blocks, 1024, 0, st>>>(keys, P, kk); sc::launched();
  }
  k_hub_finish<<<(unsigned)((n + 256) / 256), 256, 0, st>>>(keys, n, o.base, k, perm, starts); sc::launched();
  SC_LAUNCH_CHECK();
  return 0;
}
