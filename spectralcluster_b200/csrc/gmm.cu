// fallback_clusterer.check_single_cluster, AffinityGmmBic (fallback_clusterer.py:158-178): the
// reductions behind scikit-learn's GaussianMixture(1) / (2) fits on the strict upper band
// affinity[np.triu_indices(n, offset)], one streaming pass each.  The control flow (KMeans++,
// Lloyd, EM, BIC) is host logic in spectralcluster_b200/gmm_bic.py.
//
// The band of row i is columns [j0, n), j0 = max(0, i + offset), of the fp32 [n, lda] matrix;
// nothing else is read (no padding, no column >= n).  The same passes read a packed band (the
// factored route, which never stores the matrix): row i's columns [c0, n), c0 = j0 & ~3, at
// band[row_off[i] ...] with row_off[i] % 4 == 0, so column j keeps its position mod 4 and every
// thread adds the same samples in the same order as on the dense matrix.  One CTA per row: the
// ragged head up to the next multiple of 4 is read scalar, the body with 128-bit loads, the tail
// (n % 4) scalar.  Each sample is
// promoted to fp64 and every operation and sum is fp64 (exp / log1p included).  Each CTA writes
// its row's partial sums to `work` (per-thread sequential sums, then the fixed block tree); one
// block sums the rows in a fixed order, so the result is the same bit for bit on every call.
#include "common.cuh"

namespace sc {

constexpr int GT = 256;           // threads per row CTA
constexpr int GF = 8;             // partial-sum fields per row
constexpr int GL = 1024;          // threads of the lookup block

struct GmmArgs {
  double p[16];
};

// flat index of the first band element of row i (the band size for i >= the last band row)
__host__ __device__ inline int64_t band_start(int64_t n, int64_t offset, int64_t i) {
  const int64_t rows = offset >= n ? 0 : (offset > 0 ? n - offset : n);
  const int64_t full = offset < 0 ? (-offset < n ? -offset : n) : 0;
  const int64_t a = i < full ? i : full;
  const int64_t b = i < rows ? i : rows;
  int64_t s = a * n;
  if (b > a) s += (b - a) * (n - offset) - (b * (b - 1) / 2 - a * (a - 1) / 2);
  return s;
}

// sklearn's Lloyd label in 1-D: argmin_k c_k^2 - 2 x c_k (no contraction), first minimum wins
__device__ __forceinline__ int lloyd_label(double x, double c0, double c1) {
  const double d0 = __dadd_rn(__dmul_rn(c0, c0), -2.0 * __dmul_rn(x, c0));
  const double d1 = __dadd_rn(__dmul_rn(c1, c1), -2.0 * __dmul_rn(x, c1));
  return d1 < d0 ? 1 : 0;
}

__device__ __forceinline__ double sqdist1(double x, double c) {
  return sqdist_expanded(&x, 0, 1, &c, __dmul_rn(c, c), __dmul_rn(x, x));
}

// -0.5 (log 2 pi + (x pc - mu pc)^2) + log pc + log w, in numpy's operation order
__device__ __forceinline__ double weighted_log_prob(double x, const double* q) {
  const double y = __dadd_rn(__dmul_rn(x, q[2]), -q[1]);
  const double lp = __dadd_rn(__dmul_rn(-0.5, __dadd_rn(1.8378770664093453, __dmul_rn(y, y))), q[3]);
  return __dadd_rn(lp, q[0]);
}

template <int MODE>
struct RowAcc {
  double v[GF];
  __device__ void init() {
#pragma unroll
    for (int f = 0; f < GF; ++f) v[f] = 0.0;
    if (MODE == SC_GMM_MOMENTS) {
      v[3] = INFINITY;
      v[4] = -INFINITY;
    }
  }
  __device__ __forceinline__ void add(float xf, const GmmArgs& g) {
    const double x = (double)xf;
    const double* p = g.p;
    if constexpr (MODE == SC_GMM_MOMENTS) {
      const double d = x - p[0];
      v[0] += 1.0;
      v[1] += d;
      v[2] = fma(d, d, v[2]);
      v[3] = fmin(v[3], x);
      v[4] = fmax(v[4], x);
      if (!isfinite(x)) v[5] += 1.0;
    } else if constexpr (MODE == SC_GMM_KPP) {
      const double xc = x - p[0];
      const double d0 = sqdist1(xc, p[1]);
      v[0] += d0;
      if (p[4] != 0.0) {
        v[1] += fmin(d0, sqdist1(xc, p[2]));
        v[2] += fmin(d0, sqdist1(xc, p[3]));
      }
    } else if constexpr (MODE == SC_GMM_LLOYD) {
      const double xc = x - p[0];
      const int l = lloyd_label(xc, p[1], p[2]);
      v[0] += (double)l;
      if (l) v[2] += xc;
      else v[1] += xc;
      if (p[5] != 0.0 && lloyd_label(xc, p[3], p[4]) != l) v[3] += 1.0;
    } else if constexpr (MODE == SC_GMM_LABELS) {
      const int l = lloyd_label(x - p[0], p[1], p[2]);
      v[0] += (double)l;
      if (l) {
        const double d = x - p[4];
        v[2] += x;
        v[4] = fma(d, d, v[4]);
      } else {
        const double d = x - p[3];
        v[1] += x;
        v[3] = fma(d, d, v[3]);
      }
    } else {   // SC_GMM_EM, SC_GMM_SCORE: p[0] = components, then 5 per component
      const double w0 = weighted_log_prob(x, p + 1);
      double lse = w0, w1 = 0.0;
      if (p[0] > 1.5) {
        w1 = weighted_log_prob(x, p + 6);
        const double hi = fmax(w0, w1), lo = fmin(w0, w1);
        lse = hi + log1p(exp(lo - hi));
      }
      v[0] += lse;
      if constexpr (MODE == SC_GMM_EM) {
        const double r0 = exp(w0 - lse);
        const double d0 = x - p[5];
        v[1] += r0;
        v[2] = fma(r0, x, v[2]);
        v[3] = fma(r0 * d0, d0, v[3]);
        if (p[0] > 1.5) {
          const double r1 = exp(w1 - lse);
          const double d1 = x - p[10];
          v[4] += r1;
          v[5] = fma(r1, x, v[5]);
          v[6] = fma(r1 * d1, d1, v[6]);
        }
      }
    }
  }
};

// Row accessors: row(i, j0) points at column 0 of band row i, valid from column j0 & ~3 on.
struct DenseRows {         // the [n, lda] matrix
  const float* __restrict__ a;
  int64_t lda;
  __device__ __forceinline__ const float* row(int64_t i, int64_t) const { return a + i * lda; }
};
struct PackedRows {        // the packed band: columns [c0, n) of row i at band + row_off[i]
  const float* __restrict__ band;
  const int64_t* __restrict__ row_off;
  __device__ __forceinline__ const float* row(int64_t i, int64_t j0) const {
    return band + (row_off[i] - (j0 & ~(int64_t)3));
  }
};

template <int MODE, class Rows>
__global__ void __launch_bounds__(GT) k_gmm_rows(Rows rows, int64_t n, int64_t offset, GmmArgs g,
                                                 double* __restrict__ part) {
  __shared__ double red[32];
  const int64_t i = blockIdx.x;
  const int64_t j0 = i + offset > 0 ? i + offset : 0;
  RowAcc<MODE> acc;
  acc.init();
  if (j0 < n) {
    const float* r = rows.row(i, j0);
    const int64_t jv = ((j0 + 3) & ~(int64_t)3) < n ? ((j0 + 3) & ~(int64_t)3) : n;
    const int64_t jend = n & ~(int64_t)3;
    for (int64_t j = j0 + threadIdx.x; j < jv; j += GT) acc.add(r[j], g);
    for (int64_t j = jv + 4 * (int64_t)threadIdx.x; j < jend; j += 4 * GT) {
      const float4 q = ld_stream4(r + j);
      // one add() in the loop body: EM's fp64 exp / log1p, inlined four times, spill
#pragma unroll 1
      for (int e = 0; e < 4; ++e) acc.add(e == 0 ? q.x : e == 1 ? q.y : e == 2 ? q.z : q.w, g);
    }
    for (int64_t j = (jv > jend ? jv : jend) + threadIdx.x; j < n; j += GT) acc.add(r[j], g);
  }
#pragma unroll
  for (int f = 0; f < GF; ++f) {
    double s;
    if (MODE == SC_GMM_MOMENTS && f == 3) s = -block_maxd(-acc.v[f], red);
    else if (MODE == SC_GMM_MOMENTS && f == 4) s = block_maxd(acc.v[f], red);
    else s = block_sum(acc.v[f], red);
    if (threadIdx.x == 0) part[(int64_t)f * n + i] = s;
  }
}

// out[f] = the fixed-order reduction of part[f][0..n) (min / max for the moments' fields 3, 4)
__global__ void k_gmm_finish(const double* __restrict__ part, int64_t n, int mode,
                             double* __restrict__ out) {
  __shared__ double red[32];
  for (int f = 0; f < GF; ++f) {
    const bool is_min = mode == SC_GMM_MOMENTS && f == 3, is_max = mode == SC_GMM_MOMENTS && f == 4;
    double s = is_min ? INFINITY : (is_max ? -INFINITY : 0.0);
    for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
      const double v = part[(int64_t)f * n + i];
      s = is_min ? fmin(s, v) : (is_max ? fmax(s, v) : s + v);
    }
    if (is_min) s = -block_maxd(-s, red);
    else if (is_max) s = block_maxd(s, red);
    else s = block_sum(s, red);
    if (threadIdx.x == 0) out[f] = s;
  }
}

// #{k < len : prefix(k) < target} for the running sum prefix(k) = base + sum_{t <= k} term(t),
// summed in GL chunks (sequential inside a chunk, chunk sums scanned by one thread), like
// k_kpp_candidates.  Also returns the exclusive prefix of element `count` (base if count == 0).
template <typename Term>
__device__ int64_t scan_count(int64_t len, double base, double target, Term term, double* chunk,
                              int64_t* s_count, double* s_prefix) {
  const int t = threadIdx.x;
  const int64_t per = (len + GL - 1) / GL;
  const int64_t lo = (int64_t)t * per < len ? (int64_t)t * per : len;
  const int64_t hi = lo + per < len ? lo + per : len;
  double s = 0.0;
  for (int64_t k = lo; k < hi; ++k) s += term(k);
  chunk[t] = s;
  if (t == 0) *s_count = 0;
  __syncthreads();
  if (t == 0) {
    double run = base;
    for (int b = 0; b < GL; ++b) {
      const double v = chunk[b];
      chunk[b] = run;
      run += v;
    }
  }
  __syncthreads();
  double run = chunk[t];
  long long cnt = 0;
  for (int64_t k = lo; k < hi; ++k) {
    run += term(k);
    if (run < target) ++cnt;
  }
  if (cnt) atomicAdd(reinterpret_cast<unsigned long long*>(s_count), (unsigned long long)cnt);
  __syncthreads();
  const int64_t total = *s_count;
  if (total < len && total >= lo && total < hi) {   // owner of the first element not below target
    double r = chunk[t];
    for (int64_t k = lo; k < total; ++k) r += term(k);
    *s_prefix = r;
  }
  __syncthreads();
  return total;
}

// Two lookups.  p[2] == 0: p[3], p[4] are flat band indices.  p[2] == 1: p[3], p[4] are targets
// u * pot of searchsorted(cumsum(d0), target) over the KMeans++ distances to the centre p[1] (centred
// by p[0]): first over the row sums the preceding SC_GMM_KPP pass left in work[0..n), then inside
// the row.  Both clip to m - 1.  out[q] = index, out[2 + q] = the sample (fp32 promoted).
template <class Rows>
__global__ void __launch_bounds__(GL) k_gmm_lookup(Rows band, int64_t n, int64_t offset, GmmArgs g,
                                                   const double* __restrict__ rowsum,
                                                   double* __restrict__ out) {
  __shared__ double chunk[GL];
  __shared__ int64_t s_count;
  __shared__ double s_prefix;
  const int64_t m = band_start(n, offset, n);
  const int64_t rows = offset >= n ? 0 : (offset > 0 ? n - offset : n);
  const double mean = g.p[0], c0 = g.p[1];
  for (int q = 0; q < 2; ++q) {
    int64_t idx;
    if (g.p[2] == 0.0) {
      idx = (int64_t)g.p[3 + q];
    } else {
      const double target = g.p[3 + q];
      const int64_t row = scan_count(rows, 0.0, target, [&](int64_t k) { return rowsum[k]; },
                                     chunk, &s_count, &s_prefix);
      if (row >= rows) {
        idx = m;
      } else {
        const double base = s_prefix;
        const int64_t j0 = row + offset > 0 ? row + offset : 0;
        const float* r = band.row(row, j0) + j0;
        const int64_t k = scan_count(n - j0, base, target,
                                     [&](int64_t t) { return sqdist1((double)r[t] - mean, c0); },
                                     chunk, &s_count, &s_prefix);
        idx = band_start(n, offset, row) + k;
      }
    }
    if (idx > m - 1) idx = m - 1;
    if (idx < 0) idx = 0;
    // row of idx: the last row whose band starts at or before idx
    int64_t lo = 0, hi = rows - 1;
    while (lo < hi) {
      const int64_t mid = (lo + hi + 1) / 2;
      if (band_start(n, offset, mid) <= idx) lo = mid;
      else hi = mid - 1;
    }
    const int64_t jl = lo + offset > 0 ? lo + offset : 0;
    const int64_t j = jl + idx - band_start(n, offset, lo);
    if (threadIdx.x == 0) {
      out[q] = (double)idx;
      out[2 + q] = (double)band.row(lo, jl)[j];
    }
    __syncthreads();
  }
}

// Rows [row_begin, row_begin + rows) of an fp32 panel (panel row r = matrix row row_begin + r)
// -> their packed band rows.  The slots [c0, j0) and [n, round_up(n, 4)) are NaN, so a pass that
// strays outside the band sums to a non-finite value.  One CTA per row, 128-bit loads and stores
// (c0, lda and row_off[i] are multiples of 4).
__global__ void __launch_bounds__(GT) k_gmm_band_pack(const float* __restrict__ panel, int64_t ldp,
                                                      int64_t row_begin, int64_t n, int64_t offset,
                                                      const int64_t* __restrict__ row_off,
                                                      float* __restrict__ band) {
  const int64_t i = row_begin + blockIdx.x;
  const int64_t j0 = i + offset > 0 ? i + offset : 0;
  if (j0 >= n) return;
  const int64_t c0 = j0 & ~(int64_t)3;
  const float* r = panel + (int64_t)blockIdx.x * ldp;
  float* o = band + row_off[i] - c0;
  const int64_t cend = (n + 3) & ~(int64_t)3;
  for (int64_t j = c0 + 4 * (int64_t)threadIdx.x; j < cend; j += 4 * GT) {
    float4 q = ld_stream4(r + j);
    if (j < j0 || j + 3 >= n) {
      q.x = (j < j0 || j >= n) ? NAN : q.x;
      q.y = (j + 1 < j0 || j + 1 >= n) ? NAN : q.y;
      q.z = (j + 2 < j0 || j + 2 >= n) ? NAN : q.z;
      q.w = (j + 3 < j0 || j + 3 >= n) ? NAN : q.w;
    }
    *reinterpret_cast<float4*>(o + j) = q;
  }
}

}  // namespace sc

using namespace sc;

template <int MODE, class Rows>
static void launch_rows(Rows rows, int64_t n, int64_t offset, const GmmArgs& g, double* part,
                        cudaStream_t st) {
  k_gmm_rows<MODE><<<(unsigned)n, GT, 0, st>>>(rows, n, offset, g, part);
  sc::launched();
}

// One pass of `mode` over the band behind `rows` (sc_gmm_band_pass, sc_gmm_band_pass_packed).
template <class Rows>
static int band_pass(const char* name, Rows rows, int64_t n, int64_t offset, int mode,
                     const double* params_host, double* work, double* out_host, void* stream) {
  SC_REQUIRE(offset < n - 1, "%s: offset must be below n - 1", name);
  SC_REQUIRE(n < (int64_t)1 << 31, "%s: n too large", name);
  SC_REQUIRE(mode >= SC_GMM_MOMENTS && mode <= SC_GMM_SCORE, "%s: unknown mode %d", name, mode);
  cudaStream_t st = as_stream(stream);
  GmmArgs g;
  for (int k = 0; k < 16; ++k) g.p[k] = params_host[k];
  double* out_dev = work + (size_t)GF * n;
  if (mode == SC_GMM_LOOKUP) {
    if (g.p[2] == 0.0) {
      const double m = (double)band_start(n, offset, n);
      SC_REQUIRE(g.p[3] >= 0.0 && g.p[3] < m && g.p[4] >= 0.0 && g.p[4] < m,
                 "%s: lookup index out of range", name);
    }
    k_gmm_lookup<<<1, GL, 0, st>>>(rows, n, offset, g, work, out_dev); sc::launched();
  } else {
    switch (mode) {
      case SC_GMM_MOMENTS: launch_rows<SC_GMM_MOMENTS>(rows, n, offset, g, work, st); break;
      case SC_GMM_KPP: launch_rows<SC_GMM_KPP>(rows, n, offset, g, work, st); break;
      case SC_GMM_LLOYD: launch_rows<SC_GMM_LLOYD>(rows, n, offset, g, work, st); break;
      case SC_GMM_LABELS: launch_rows<SC_GMM_LABELS>(rows, n, offset, g, work, st); break;
      case SC_GMM_EM: launch_rows<SC_GMM_EM>(rows, n, offset, g, work, st); break;
      default: launch_rows<SC_GMM_SCORE>(rows, n, offset, g, work, st); break;
    }
    k_gmm_finish<<<1, 1024, 0, st>>>(work, n, mode, out_dev); sc::launched();
  }
  SC_LAUNCH_CHECK();
  SC_CUDA(cudaMemcpyAsync(out_host, out_dev, sizeof(double) * GF, cudaMemcpyDeviceToHost, st));
  SC_CUDA(cudaStreamSynchronize(st));
  return 0;
}

extern "C" int sc_gmm_band_pass(sc_context* ctx, const float* a, int64_t n, int64_t lda,
                                int64_t offset, int mode, const double* params_host, double* work,
                                double* out_host, void* stream) {
  SC_REQUIRE(ctx && a && params_host && work && out_host && n > 0 && lda >= n,
             "sc_gmm_band_pass: bad arguments");
  SC_REQUIRE(vec_ok_f32(a, lda), "sc_gmm_band_pass: `a` needs a 16-byte aligned base and lda %% 4 == 0");
  return band_pass("sc_gmm_band_pass", DenseRows{a, lda}, n, offset, mode, params_host, work,
                   out_host, stream);
}

extern "C" int sc_gmm_band_pass_packed(sc_context* ctx, const float* band, const int64_t* row_off,
                                       int64_t n, int64_t offset, int mode,
                                       const double* params_host, double* work, double* out_host,
                                       void* stream) {
  SC_REQUIRE(ctx && band && row_off && params_host && work && out_host && n > 0,
             "sc_gmm_band_pass_packed: bad arguments");
  SC_REQUIRE(vec_ok_f32(band, 0), "sc_gmm_band_pass_packed: `band` needs a 16-byte aligned base");
  return band_pass("sc_gmm_band_pass_packed", PackedRows{band, row_off}, n, offset, mode,
                   params_host, work, out_host, stream);
}

extern "C" int sc_gmm_band_pack(sc_context* ctx, const float* panel, int64_t ldp, int64_t row_begin,
                                int64_t rows, int64_t n, int64_t offset, const int64_t* row_off,
                                float* band, void* stream) {
  SC_REQUIRE(ctx && panel && row_off && band && n > 0 && rows > 0 && row_begin >= 0 &&
             row_begin + rows <= n && ldp >= ((n + 3) & ~(int64_t)3),
             "sc_gmm_band_pack: bad arguments");
  SC_REQUIRE(vec_ok_f32(panel, ldp), "sc_gmm_band_pack: `panel` needs a 16-byte aligned base and ldp %% 4 == 0");
  SC_REQUIRE(vec_ok_f32(band, 0), "sc_gmm_band_pack: `band` needs a 16-byte aligned base");
  SC_REQUIRE(offset < n - 1, "sc_gmm_band_pack: offset must be below n - 1");
  k_gmm_band_pack<<<(unsigned)rows, GT, 0, as_stream(stream)>>>(panel, ldp, row_begin, n, offset,
                                                                row_off, band);
  sc::launched();
  SC_LAUNCH_CHECK();
  return 0;
}
