// custom_distance_kmeans.run_kmeans (custom_distance_kmeans.py:13-52) on the device, fp64.
//
// Stage 1 (custom_distance_kmeans.py:39-43) restates what scikit-learn 1.9.0's
//   KMeans(n_clusters=k, init="k-means++", max_iter=1, random_state=0, n_init="auto").fit(E)
// does to produce cluster_centers_ (sklearn/cluster/_kmeans.py: fit :1436-1560,
// _kmeans_plusplus :180-283, _kmeans_single_lloyd :630-758):
//   X = E - mean(E, axis 0); greedy k-means++ with 2+int(ln k) trials per centre, driven by the
//   caller's RandomState(0) draws; ONE Lloyd iteration (E-step argmin ||c||^2 - 2 x.c, first
//   minimum wins; M-step = mean of members); centres + mean.
// Stage 2 (custom_distance_kmeans.py:118-141, CustomKMeans.predict): <= max_iter+1 assignment
//   passes with scipy cdist 'cosine' (1 - u.v/(|u||v|), clipped) or 'euclidean', relative
//   improvement stop (tol 1e-3), centroid = mean of members, including the quirk that a cluster
//   whose only member is sample 0 keeps its centroid (`np.where(...)[0].any()`, :137-138).
// All reductions are deterministic (fixed thread->row assignment, tree reductions).
#include "common.cuh"

#include <algorithm>
#include <vector>

namespace sc {

constexpr int KT = 256;

struct KmState {
  double prev_mean;
  double pot;
  int done;
  int iters;
  int best_trial;
  int empty_cluster;
  int nonfinite;      // bit 0: an embedding element is NaN, bit 1: one is +-inf
  int singular;       // mahalanobis: the covariance of a pass had an exactly zero pivot
};

// Metric codes of sc_kmeans (include/spectralcluster_b200.h) and k_assign's template argument.
// KM_BUILTIN is the one kernel that serves the sklearn E-step (-1), cosine (0) and euclidean (1),
// chosen by its run-time `metric` argument; every other value is one scipy metric.
enum : int {
  KM_BUILTIN = -2,
  KM_COSINE = SC_KMEANS_COSINE,
  KM_EUCLIDEAN = SC_KMEANS_EUCLIDEAN,
  KM_SQEUCLIDEAN = SC_KMEANS_SQEUCLIDEAN,
  KM_CITYBLOCK = SC_KMEANS_CITYBLOCK,
  KM_CHEBYSHEV = SC_KMEANS_CHEBYSHEV,
  KM_CANBERRA = SC_KMEANS_CANBERRA,
  KM_BRAYCURTIS = SC_KMEANS_BRAYCURTIS,
  KM_CORRELATION = SC_KMEANS_CORRELATION,
  KM_JENSENSHANNON = SC_KMEANS_JENSENSHANNON,
  KM_SEUCLIDEAN = SC_KMEANS_SEUCLIDEAN,
  KM_MAHALANOBIS = SC_KMEANS_MAHALANOBIS,
};

// ---- centring ---------------------------------------------------------------------------
__global__ void k_col_mean(const double* __restrict__ e, int64_t n, int64_t kd,
                           double* __restrict__ mean) {
  __shared__ double red[32];
  const int64_t f = blockIdx.x;
  double s = 0.0;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) s += e[i * kd + f];
  s = block_sum(s, red);
  if (threadIdx.x == 0) mean[f] = s / (double)n;
}

// Also flags non-finite input in st->nonfinite: scikit-learn's fit refuses it (check_array).
__global__ void k_center(const double* __restrict__ e, int64_t n, int64_t kd,
                         const double* __restrict__ mean, double* __restrict__ x,
                         double* __restrict__ xsq, KmState* st) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double ss = 0.0;
  int bad = 0;
  for (int64_t f = 0; f < kd; ++f) {
    const double ef = e[i * kd + f];
    if (isnan(ef)) bad |= 1;
    else if (isinf(ef)) bad |= 2;
    const double v = ef - mean[f];
    x[i * kd + f] = v;
    ss += v * v;
  }
  xsq[i] = ss;
  if (bad) atomicOr(&st->nonfinite, bad);
}

// ---- k-means++ ---------------------------------------------------------------------------
// closest[i] = d2(x_i, x_first); partial sums per block -> part[block]
__global__ void k_kpp_first(const double* __restrict__ x, const double* __restrict__ xsq,
                            int64_t n, int64_t kd, int64_t first, double* __restrict__ closest,
                            double* __restrict__ part, double* __restrict__ centers) {
  __shared__ double red[32];
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const double* c = x + first * kd;
  double v = 0.0;
  if (i < n) {
    v = sqdist_expanded(x, i, kd, c, xsq[first], xsq[i]);
    closest[i] = v;
  }
  v = block_sum(v, red);
  if (threadIdx.x == 0) part[blockIdx.x] = v;
  if (blockIdx.x == 0)
    for (int64_t f = threadIdx.x; f < kd; f += blockDim.x) centers[f] = c[f];
}

// one block: pot = sum(part[0..nb)); also (re)used to pick the best trial
__global__ void k_kpp_reduce_pot(const double* __restrict__ part, int nb, KmState* st) {
  __shared__ double red[32];
  double s = 0.0;
  for (int b = threadIdx.x; b < nb; b += blockDim.x) s += part[b];
  s = block_sum(s, red);
  if (threadIdx.x == 0) st->pot = s;
}

// one block of 1024 threads: candidate ids = searchsorted(cumsum(closest), u * pot), clipped
__global__ void k_kpp_candidates(const double* __restrict__ closest, int64_t n,
                                 const double* __restrict__ u, int trials, const KmState* st,
                                 int* __restrict__ cand) {
  __shared__ double chunk_sum[1024];
  __shared__ int count[16];
  const int t = threadIdx.x;
  const int64_t per = (n + 1023) / 1024;
  const int64_t lo = (int64_t)t * per, hi = (lo + per < n) ? lo + per : n;
  double s = 0.0;
  for (int64_t i = lo; i < hi; ++i) s += closest[i];
  chunk_sum[t] = s;
  if (t < 16) count[t] = 0;
  __syncthreads();
  if (t == 0) {   // exclusive scan of 1024 partial sums, sequential like np.cumsum
    double run = 0.0;
    for (int b = 0; b < 1024; ++b) {
      const double v = chunk_sum[b];
      chunk_sum[b] = run;
      run += v;
    }
  }
  __syncthreads();
  const double pot = st->pot;
  double run = chunk_sum[t];
  int local[16];
  for (int q = 0; q < trials; ++q) local[q] = 0;
  for (int64_t i = lo; i < hi; ++i) {
    run += closest[i];                    // inclusive cumsum at i
    for (int q = 0; q < trials; ++q)
      if (run < u[q] * pot) ++local[q];   // searchsorted side='left': #{cum < value}
  }
  for (int q = 0; q < trials; ++q)
    if (local[q]) atomicAdd(&count[q], local[q]);
  __syncthreads();
  if (t < trials) {
    int c = count[t];
    if (c > (int)(n - 1)) c = (int)(n - 1);   // np.clip(..., None, n - 1)
    cand[t] = c;
  }
}

// newd[q][i] = min(closest[i], d2(x_i, x_cand[q])); part[q][block] = block sum
__global__ void k_kpp_trials(const double* __restrict__ x, const double* __restrict__ xsq,
                             int64_t n, int64_t kd, const double* __restrict__ closest,
                             const int* __restrict__ cand, int trials, double* __restrict__ newd,
                             double* __restrict__ part) {
  __shared__ double red[32];
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  for (int q = 0; q < trials; ++q) {
    const int64_t cq = cand[q];
    double v = 0.0;
    if (i < n) {
      v = sqdist_expanded(x, i, kd, x + cq * kd, xsq[cq], xsq[i]);
      v = fmin(closest[i], v);
      newd[(int64_t)q * n + i] = v;
    }
    v = block_sum(v, red);
    if (threadIdx.x == 0) part[(int64_t)q * gridDim.x + blockIdx.x] = v;
  }
}

// one block: potentials of the trials, argmin (first minimum), record centre c
__global__ void k_kpp_choose(const double* __restrict__ part, int nb, int trials,
                             const int* __restrict__ cand, const double* __restrict__ x,
                             int64_t kd, int center_idx, double* __restrict__ centers,
                             KmState* st) {
  __shared__ double red[32];
  __shared__ double pots[16];
  for (int q = 0; q < trials; ++q) {
    double s = 0.0;
    for (int b = threadIdx.x; b < nb; b += blockDim.x) s += part[(int64_t)q * nb + b];
    s = block_sum(s, red);
    if (threadIdx.x == 0) pots[q] = s;
  }
  __syncthreads();
  __shared__ int best;
  if (threadIdx.x == 0) {
    int b = 0;
    for (int q = 1; q < trials; ++q)
      if (pots[q] < pots[b]) b = q;
    best = b;
    st->best_trial = b;
    st->pot = pots[b];
  }
  __syncthreads();
  const double* c = x + (int64_t)cand[best] * kd;
  for (int64_t f = threadIdx.x; f < kd; f += blockDim.x) centers[(int64_t)center_idx * kd + f] = c[f];
}

__global__ void k_kpp_commit(const double* __restrict__ newd, int64_t n, const KmState* st,
                             double* __restrict__ closest) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) closest[i] = newd[(int64_t)st->best_trial * n + i];
}

// ---- Lloyd E-step (sklearn) and the custom-distance assignment ------------------------------
// scipy's cdist kernels (scipy/spatial/src/distance_impl.h) for one row x and one centroid c, in
// their order of operations.  `aux` is the per-pass parameter: V for seuclidean, VI (row-major)
// for mahalanobis.  Correlation is cosine on rows and centroids already centred by their own mean
// (k_row_centre), as scipy's _correlation_cdist_wrap.
template <int M>
__device__ __forceinline__ double scipy_dist(const double* __restrict__ x,
                                             const double* __restrict__ c, int64_t kd,
                                             const double* __restrict__ aux) {
  if constexpr (M == KM_SQEUCLIDEAN) {
    double s = 0.0;
    for (int64_t f = 0; f < kd; ++f) {
      const double d = x[f] - c[f];
      s = fma(d, d, s);
    }
    return s;
  } else if constexpr (M == KM_CITYBLOCK) {
    double s = 0.0;
    for (int64_t f = 0; f < kd; ++f) s += fabs(x[f] - c[f]);
    return s;
  } else if constexpr (M == KM_CHEBYSHEV) {
    double s = 0.0;
    for (int64_t f = 0; f < kd; ++f) s = fmax(s, fabs(x[f] - c[f]));
    return s;
  } else if constexpr (M == KM_CANBERRA) {
    double s = 0.0;
    for (int64_t f = 0; f < kd; ++f) {
      const double den = fabs(x[f]) + fabs(c[f]);
      if (den > 0.0) s += fabs(x[f] - c[f]) / den;   // a 0/0 term adds 0
    }
    return s;
  } else if constexpr (M == KM_BRAYCURTIS) {
    double num = 0.0, den = 0.0;
    for (int64_t f = 0; f < kd; ++f) {
      num += fabs(x[f] - c[f]);
      den += fabs(x[f] + c[f]);
    }
    return num / den;
  } else if constexpr (M == KM_CORRELATION) {
    double dot = 0.0, xn = 0.0, cn = 0.0;
    for (int64_t f = 0; f < kd; ++f) {
      dot = fma(x[f], c[f], dot);
      xn = fma(x[f], x[f], xn);
      cn = fma(c[f], c[f], cn);
    }
    double cosv = dot / (sqrt(xn) * sqrt(cn));
    if (fabs(cosv) > 1.0) cosv = copysign(1.0, cosv);
    return 1.0 - cosv;
  } else if constexpr (M == KM_JENSENSHANNON) {
    double ps = 0.0, qs = 0.0;
    for (int64_t f = 0; f < kd; ++f) {
      if (x[f] < 0.0 || c[f] < 0.0) return HUGE_VAL;
      ps += x[f];
      qs += c[f];
    }
    double s = 0.0;
    for (int64_t f = 0; f < kd; ++f) {
      const double p = x[f] / ps, q = c[f] / qs, m = (p + q) / 2.0;
      if (p > 0.0) s += p * log(p / m);
      if (q > 0.0) s += q * log(q / m);
    }
    return sqrt(s / 2.0);
  } else if constexpr (M == KM_SEUCLIDEAN) {
    double s = 0.0;
    for (int64_t f = 0; f < kd; ++f) {
      const double d = x[f] - c[f];
      s += d * d / aux[f];
    }
    return sqrt(s);
  } else {
    static_assert(M == KM_MAHALANOBIS, "unknown metric");
    double s = 0.0;
    for (int64_t a = 0; a < kd; ++a) {
      double w = 0.0;
      for (int64_t b = 0; b < kd; ++b) w = fma(aux[a * kd + b], x[b] - c[b], w);
      s = fma(x[a] - c[a], w, s);
    }
    return sqrt(s);
  }
}

// M = KM_BUILTIN, metric: -1 = sklearn E-step (|c|^2 - 2 x.c), 0 = cosine (scipy cdist),
// 1 = euclidean; the first minimum under `<` wins.  Any other M: that scipy metric (`metric` unused),
// argmin as np.argmin: the first NaN wins, otherwise the first minimum.
template <int M>
__global__ void k_assign(const double* __restrict__ x, int64_t n, int64_t kd,
                         const double* __restrict__ centers, int64_t k, int metric,
                         int* __restrict__ labels, double* __restrict__ part,
                         const KmState* st, const double* __restrict__ aux) {
  __shared__ double red[32];
  if (st->done) return;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  double best = 0.0;
  if constexpr (M != KM_BUILTIN) {
    if (i < n) {
      int arg = 0;
      for (int64_t c = 0; c < k; ++c) {
        const double dist = scipy_dist<M>(x + i * kd, centers + c * kd, kd, aux);
        if (c == 0 || dist < best || (isnan(dist) && !isnan(best))) {
          best = dist;
          arg = (int)c;
        }
      }
      labels[i] = arg;
    }
  } else if (i < n) {
    double xn = 0.0;
    if (metric == 0)
      for (int64_t f = 0; f < kd; ++f) xn = fma(x[i * kd + f], x[i * kd + f], xn);
    int arg = 0;
    for (int64_t c = 0; c < k; ++c) {
      const double* cc = centers + c * kd;
      double dist;
      if (metric == 1) {
        double s = 0.0;
        for (int64_t f = 0; f < kd; ++f) {
          const double df = x[i * kd + f] - cc[f];
          s = fma(df, df, s);
        }
        dist = sqrt(s);
      } else {
        double dot = 0.0, cn = 0.0;
        for (int64_t f = 0; f < kd; ++f) {
          dot = fma(x[i * kd + f], cc[f], dot);
          cn = fma(cc[f], cc[f], cn);
        }
        if (metric == 0) {
          double cosv = dot / (sqrt(xn) * sqrt(cn));
          if (fabs(cosv) > 1.0) cosv = copysign(1.0, cosv);   // scipy clips
          dist = 1.0 - cosv;
        } else {
          dist = cn - 2.0 * dot;
        }
      }
      if (c == 0 || dist < best) {   // argmin keeps the first minimum
        best = dist;
        arg = (int)c;
      }
    }
    labels[i] = arg;
  }
  double v = (i < n) ? best : 0.0;
  v = block_sum(v, red);
  if (threadIdx.x == 0) part[blockIdx.x] = v;
}

// grid (k, kd): sums[c][f] = sum over members of x[i][f]; counts[c] (and members other than
// sample 0) from the f == 0 column.  Fixed thread->row mapping: deterministic.
__global__ void k_cluster_sums(const double* __restrict__ x, int64_t n, int64_t kd,
                               const int* __restrict__ labels, double* __restrict__ sums,
                               int* __restrict__ counts, int* __restrict__ counts_nz,
                               const KmState* st) {
  __shared__ double red[32];
  if (st->done) return;
  const int c = blockIdx.x;
  const int64_t f = blockIdx.y;
  double s = 0.0, cnt = 0.0, cnz = 0.0;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
    if (labels[i] == c) {
      s += x[i * kd + f];
      cnt += 1.0;
      if (i != 0) cnz += 1.0;
    }
  }
  s = block_sum(s, red);
  if (threadIdx.x == 0) sums[(int64_t)c * kd + f] = s;
  if (f == 0) {
    cnt = block_sum(cnt, red);
    cnz = block_sum(cnz, red);
    if (threadIdx.x == 0) {
      counts[c] = (int)cnt;
      counts_nz[c] = (int)cnz;
    }
  }
}

// sklearn M-step + "centres += X_mean".  Flags empty clusters (relocation not restated).
__global__ void k_lloyd_update(const double* __restrict__ sums, const int* __restrict__ counts,
                               int64_t k, int64_t kd, const double* __restrict__ mean,
                               double* __restrict__ centers, KmState* st) {
  const int64_t idx = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= k * kd) return;
  const int64_t c = idx / kd, f = idx - c * kd;
  if (counts[c] == 0) {
    st->empty_cluster = 1;
    centers[idx] += mean[f];
  } else {
    centers[idx] = sums[idx] / (double)counts[c] + mean[f];
  }
}

// One thread: mean distance, stop rule (custom_distance_kmeans.py:126-133), else centroid update
// (:134-140) by the threads of the block.
__global__ void k_custom_step(const double* __restrict__ part, int nb, int64_t n,
                              const double* __restrict__ sums, const int* __restrict__ counts_nz,
                              int64_t k, int64_t kd, double tol, int64_t max_iter,
                              double* __restrict__ centers, const int* __restrict__ counts,
                              KmState* st) {
  __shared__ double red[32];
  __shared__ int stop;
  if (st->done) return;
  double s = 0.0;
  for (int b = threadIdx.x; b < nb; b += blockDim.x) s += part[b];
  s = block_sum(s, red);
  if (threadIdx.x == 0) {
    const double mean_d = s / (double)n;
    const double prev = st->prev_mean;
    const int it = st->iters;            // index of the assignment pass just finished
    const bool hit = (mean_d <= prev && mean_d >= (1.0 - tol) * prev) || (it == max_iter);
    st->iters = it + 1;
    if (hit) st->done = 1;
    else st->prev_mean = mean_d;
    stop = hit ? 1 : 0;
  }
  __syncthreads();
  if (stop) return;
  for (int64_t idx = threadIdx.x; idx < k * kd; idx += blockDim.x) {
    const int64_t c = idx / kd;
    if (counts_nz[c] > 0) centers[idx] = sums[idx] / (double)counts[c];
  }
}

__global__ void k_state_init(KmState* st) {
  st->prev_mean = 0.0;
  st->pot = 0.0;
  st->done = 0;
  st->iters = 0;
  st->best_trial = 0;
  st->empty_cluster = 0;
  st->nonfinite = 0;
  st->singular = 0;
}

// ---- per-pass parameters of the scipy metrics (scipy's validators recompute them every cdist) --
// correlation: dst[i] = src[i] - mean(src[i]) (XA - XA.mean(axis=1, keepdims=True)).  st may be
// NULL (the embeddings, centred once before the loop).
__global__ void k_row_centre(const double* __restrict__ src, int64_t rows, int64_t kd,
                             double* __restrict__ dst, const KmState* st) {
  if (st && st->done) return;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows) return;
  double s = 0.0;
  for (int64_t f = 0; f < kd; ++f) s += src[i * kd + f];
  const double mu = s / (double)kd;
  for (int64_t f = 0; f < kd; ++f) dst[i * kd + f] = src[i * kd + f] - mu;
}

// One block per column f of the stacked rows [E; C] (m = n + k rows): mu[f] = column mean and,
// when var is not NULL, var[f] = sum((x - mu)^2) / (m - 1) (np.var(vstack([E, C]), axis=0, ddof=1),
// seuclidean's V).
__global__ void k_stack_col_stats(const double* __restrict__ e, int64_t n,
                                  const double* __restrict__ c, int64_t k, int64_t kd,
                                  double* __restrict__ mu, double* __restrict__ var,
                                  const KmState* st) {
  __shared__ double red[32];
  if (st->done) return;
  const int64_t f = blockIdx.x, m = n + k;
  double s = 0.0;
  for (int64_t i = threadIdx.x; i < m; i += blockDim.x) s += i < n ? e[i * kd + f] : c[(i - n) * kd + f];
  s = block_sum(s, red);
  const double mean = s / (double)m;
  if (threadIdx.x == 0) mu[f] = mean;
  if (!var) return;
  double q = 0.0;
  for (int64_t i = threadIdx.x; i < m; i += blockDim.x) {
    const double d = (i < n ? e[i * kd + f] : c[(i - n) * kd + f]) - mean;
    q = fma(d, d, q);
  }
  q = block_sum(q, red);
  if (threadIdx.x == 0) var[f] = q / (double)(m - 1);
}

// grid (kd, kd), blocks with a <= b: cv[a][b] = cv[b][a] = sum((x_a - mu_a)(x_b - mu_b)) * (1/(m-1))
// over the stacked rows [E; C] (np.cov(vstack([E, C]).T)), so cv is exactly symmetric.
__global__ void k_stack_cov(const double* __restrict__ e, int64_t n, const double* __restrict__ c,
                            int64_t k, int64_t kd, const double* __restrict__ mu,
                            double* __restrict__ cv, const KmState* st) {
  __shared__ double red[32];
  const int64_t a = blockIdx.y, b = blockIdx.x;
  if (st->done || b < a) return;
  const int64_t m = n + k;
  double s = 0.0;
  for (int64_t i = threadIdx.x; i < m; i += blockDim.x) {
    const double* r = i < n ? e + i * kd : c + (i - n) * kd;
    s = fma(r[a] - mu[a], r[b] - mu[b], s);
  }
  s = block_sum(s, red);
  if (threadIdx.x == 0) {
    const double v = s * (1.0 / (double)(m - 1));
    cv[a * kd + b] = v;
    cv[b * kd + a] = v;
  }
}

// One CTA: vi = inv(a)^T (np.linalg.inv(CV).T), fp64 Gauss-Jordan elimination with partial
// pivoting.  The pivot is the first largest |a[i][p]| over i >= p (LAPACK's idamax) and the
// multipliers are a[i][p] / a[p][p], so the pivots are those of LAPACK's getrf: an exactly zero
// pivot is numpy's "Singular matrix", reported in st->singular (and the loop stops).  a is
// destroyed; b [kd*kd] and fac [kd] are scratch.
__global__ void k_inverse_t(double* __restrict__ a, double* __restrict__ b, double* __restrict__ fac,
                            int64_t kd, double* __restrict__ vi, KmState* st) {
  __shared__ double rv[32];
  __shared__ long long ri[32];
  __shared__ long long piv;
  if (st->done) return;
  const int tid = threadIdx.x, nt = blockDim.x, lane = tid & 31, wid = tid >> 5;
  for (int64_t idx = tid; idx < kd * kd; idx += nt) b[idx] = (idx / kd == idx % kd) ? 1.0 : 0.0;
  for (int64_t p = 0; p < kd; ++p) {
    __syncthreads();
    double bv = -1.0;
    long long bi = kd;
    for (int64_t i = p + tid; i < kd; i += nt) {
      const double v = fabs(a[i * kd + p]);
      if (v > bv) { bv = v; bi = i; }
    }
    for (int o = 16; o; o >>= 1) {   // larger |a| wins, the lower row on a tie
      const double ov = __shfl_xor_sync(0xffffffffu, bv, o);
      const long long oi = __shfl_xor_sync(0xffffffffu, bi, o);
      if (ov > bv || (ov == bv && oi < bi)) { bv = ov; bi = oi; }
    }
    if (lane == 0) { rv[wid] = bv; ri[wid] = bi; }
    __syncthreads();
    if (tid == 0) {
      for (int w = 1; w < nt / 32; ++w)
        if (rv[w] > rv[0] || (rv[w] == rv[0] && ri[w] < ri[0])) { rv[0] = rv[w]; ri[0] = ri[w]; }
      piv = ri[0];
    }
    __syncthreads();
    const int64_t r = piv;
    if (!(a[r * kd + p] != 0.0)) {
      if (tid == 0) { st->singular = 1; st->done = 1; }
      return;
    }
    if (r != p)
      for (int64_t q = tid; q < kd; q += nt) {
        double t = a[p * kd + q]; a[p * kd + q] = a[r * kd + q]; a[r * kd + q] = t;
        t = b[p * kd + q]; b[p * kd + q] = b[r * kd + q]; b[r * kd + q] = t;
      }
    __syncthreads();
    for (int64_t i = tid; i < kd; i += nt) fac[i] = i == p ? 0.0 : a[i * kd + p] / a[p * kd + p];
    __syncthreads();
    for (int64_t idx = tid; idx < kd * 2 * kd; idx += nt) {
      const int64_t i = idx / (2 * kd), q = idx - i * 2 * kd;
      if (i == p) continue;
      if (q < kd) {
        if (q > p) a[i * kd + q] = fma(-fac[i], a[p * kd + q], a[i * kd + q]);
      } else {
        b[i * kd + q - kd] = fma(-fac[i], b[p * kd + q - kd], b[i * kd + q - kd]);
      }
    }
  }
  __syncthreads();
  for (int64_t idx = tid; idx < kd * kd; idx += nt) {
    const int64_t i = idx / kd, j = idx - i * kd;
    vi[j * kd + i] = b[idx] / a[i * kd + i];
  }
}

__global__ void k_row_renorm(double* __restrict__ e, int64_t n, int64_t k) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double ss = 0.0;
  for (int64_t f = 0; f < k; ++f) ss = fma(e[i * k + f], e[i * k + f], ss);
  const double nrm = sqrt(ss);
  for (int64_t f = 0; f < k; ++f) e[i * k + f] /= nrm;
}

}  // namespace sc

using namespace sc;

namespace {

// The assignment pass of metric `metric` (>= 0) on stage 2's rows x and centroids c.
void launch_assign(int metric, int nb, cudaStream_t st, const double* x, int64_t n, int64_t kd,
                   const double* c, int64_t k, int* labels, double* part, const KmState* state,
                   const double* aux) {
#define SC_ASSIGN(M) k_assign<M><<<nb, KT, 0, st>>>(x, n, kd, c, k, metric, labels, part, state, aux)
  switch (metric) {
    case KM_COSINE:
    case KM_EUCLIDEAN: SC_ASSIGN(KM_BUILTIN); break;
    case KM_SQEUCLIDEAN: SC_ASSIGN(KM_SQEUCLIDEAN); break;
    case KM_CITYBLOCK: SC_ASSIGN(KM_CITYBLOCK); break;
    case KM_CHEBYSHEV: SC_ASSIGN(KM_CHEBYSHEV); break;
    case KM_CANBERRA: SC_ASSIGN(KM_CANBERRA); break;
    case KM_BRAYCURTIS: SC_ASSIGN(KM_BRAYCURTIS); break;
    case KM_CORRELATION: SC_ASSIGN(KM_CORRELATION); break;
    case KM_JENSENSHANNON: SC_ASSIGN(KM_JENSENSHANNON); break;
    case KM_SEUCLIDEAN: SC_ASSIGN(KM_SEUCLIDEAN); break;
    default: SC_ASSIGN(KM_MAHALANOBIS); break;
  }
#undef SC_ASSIGN
  sc::launched();
}

}  // namespace

extern "C" int sc_row_renorm(sc_context* ctx, double* e, int64_t n, int64_t k, void* stream) {
  SC_REQUIRE(ctx && e && n > 0 && k > 0, "sc_row_renorm: bad arguments");
  k_row_renorm<<<(unsigned)((n + KT - 1) / KT), KT, 0, as_stream(stream)>>>(e, n, k); sc::launched();
  SC_LAUNCH_CHECK();
  return 0;
}

extern "C" int sc_kmeans(sc_context* ctx, const double* e, int64_t n, int64_t k_dim, int64_t k,
                         int64_t first_center, const double* u_host, int64_t trials, int metric,
                         int64_t max_iter, double tol, int64_t* labels_host, int64_t* iters_host,
                         void* stream) {
  SC_REQUIRE(ctx && e && labels_host && n > 0 && k_dim > 0 && k > 0, "sc_kmeans: bad arguments");
  SC_REQUIRE(metric >= KM_COSINE && metric <= KM_MAHALANOBIS,
             "sc_kmeans: metric must be 0 (cosine) .. 10 (mahalanobis), got %d", metric);
  SC_REQUIRE(max_iter > 0, "Number of iterations should be a positive number, got %lld instead",
             (long long)max_iter);
  SC_REQUIRE(n >= k, "n_samples=%lld should be >= n_clusters=%lld", (long long)n, (long long)k);
  SC_REQUIRE(trials >= 1 && trials <= 16, "sc_kmeans: 1 <= trials <= 16");
  SC_REQUIRE(first_center >= 0 && first_center < n, "sc_kmeans: first_center out of range");
  SC_REQUIRE(k == 1 || u_host, "sc_kmeans: u_host missing");
  SC_REQUIRE(k * k_dim <= (1 << 24) && k <= 65535 && k_dim <= 65535, "sc_kmeans: k too large");
  cudaStream_t st = as_stream(stream);
  const int nb = (int)((n + KT - 1) / KT);

  Scratch buf, ibuf, sbuf;
  // doubles: mean[kd] x[n*kd] xsq[n] closest[n] newd[trials*n] part[trials*nb] centers[k*kd]
  //          sums[k*kd] u[(k-1)*trials]
  const size_t nd = (size_t)k_dim + (size_t)n * k_dim + 2 * (size_t)n + (size_t)trials * n +
                    (size_t)trials * nb + 2 * (size_t)k * k_dim + (size_t)(k > 1 ? (k - 1) : 1) * trials;
  SC_CUDA(buf.alloc(sizeof(double) * nd, st));
  double* mean = buf.as<double>();
  double* x = mean + k_dim;
  double* xsq = x + (size_t)n * k_dim;
  double* closest = xsq + n;
  double* newd = closest + n;
  double* part = newd + (size_t)trials * n;
  double* centers = part + (size_t)trials * nb;
  double* sums = centers + (size_t)k * k_dim;
  double* u_dev = sums + (size_t)k * k_dim;
  // ints: labels[n] counts[k] counts_nz[k] cand[16]
  SC_CUDA(ibuf.alloc(sizeof(int) * ((size_t)n + 2 * (size_t)k + 16), st));
  int* labels = ibuf.as<int>();
  int* counts = labels + n;
  int* counts_nz = counts + k;
  int* cand = counts_nz + k;
  SC_CUDA(sbuf.alloc(sizeof(KmState), st));
  KmState* state = sbuf.as<KmState>();
  // per-pass parameters of stage 2: correlation xc[n*kd] cc[k*kd]; seuclidean mu[kd] var[kd];
  // mahalanobis mu[kd] cv[kd*kd] work[kd*kd] vi[kd*kd] fac[kd]
  Scratch abuf;
  double *xc = nullptr, *cc = nullptr, *mu = nullptr, *var = nullptr, *cv = nullptr,
         *work = nullptr, *vi = nullptr, *fac = nullptr;
  const size_t kd2 = (size_t)k_dim * k_dim;
  if (metric == KM_CORRELATION) {
    SC_CUDA(abuf.alloc(sizeof(double) * ((size_t)n + k) * k_dim, st));
    xc = abuf.as<double>();
    cc = xc + (size_t)n * k_dim;
  } else if (metric == KM_SEUCLIDEAN) {
    SC_CUDA(abuf.alloc(sizeof(double) * 2 * (size_t)k_dim, st));
    mu = abuf.as<double>();
    var = mu + k_dim;
  } else if (metric == KM_MAHALANOBIS) {
    SC_CUDA(abuf.alloc(sizeof(double) * (3 * kd2 + 2 * (size_t)k_dim), st));
    mu = abuf.as<double>();
    fac = mu + k_dim;
    cv = fac + k_dim;
    work = cv + kd2;
    vi = work + kd2;
  }

  k_state_init<<<1, 1, 0, st>>>(state); sc::launched();
  if (k > 1)
    SC_CUDA(cudaMemcpyAsync(u_dev, u_host, sizeof(double) * (size_t)(k - 1) * trials,
                            cudaMemcpyHostToDevice, st));
  // ---- stage 1: scikit-learn seeding + one Lloyd iteration
  k_col_mean<<<(unsigned)k_dim, KT, 0, st>>>(e, n, k_dim, mean); sc::launched();
  k_center<<<nb, KT, 0, st>>>(e, n, k_dim, mean, x, xsq, state); sc::launched();
  k_kpp_first<<<nb, KT, 0, st>>>(x, xsq, n, k_dim, first_center, closest, part, centers); sc::launched();
  k_kpp_reduce_pot<<<1, KT, 0, st>>>(part, nb, state); sc::launched();
  SC_LAUNCH_CHECK();
  for (int64_t c = 1; c < k; ++c) {
    k_kpp_candidates<<<1, 1024, 0, st>>>(closest, n, u_dev + (c - 1) * trials, (int)trials, state,
                                         cand); sc::launched();
    k_kpp_trials<<<nb, KT, 0, st>>>(x, xsq, n, k_dim, closest, cand, (int)trials, newd, part); sc::launched();
    k_kpp_choose<<<1, KT, 0, st>>>(part, nb, (int)trials, cand, x, k_dim, (int)c, centers, state); sc::launched();
    k_kpp_commit<<<nb, KT, 0, st>>>(newd, n, state, closest); sc::launched();
  }
  SC_LAUNCH_CHECK();
  k_assign<KM_BUILTIN><<<nb, KT, 0, st>>>(x, n, k_dim, centers, k, -1, labels, part, state,
                                          nullptr); sc::launched();
  k_cluster_sums<<<dim3((unsigned)k, (unsigned)k_dim), KT, 0, st>>>(x, n, k_dim, labels, sums,
                                                                    counts, counts_nz, state); sc::launched();
  k_lloyd_update<<<(unsigned)((k * k_dim + KT - 1) / KT), KT, 0, st>>>(sums, counts, k, k_dim,
                                                                       mean, centers, state); sc::launched();
  SC_LAUNCH_CHECK();

  // ---- stage 2: CustomKMeans.predict on the un-centred embeddings
  KmState hs;
  if (metric == KM_MAHALANOBIS && n + k <= k_dim) {
    // scipy's validator refuses this at the first cdist, after the seeding has run (and after
    // scikit-learn's fit has refused non-finite input)
    SC_CUDA(cudaMemcpyAsync(&hs, state, sizeof(hs), cudaMemcpyDeviceToHost, st));
    SC_CUDA(cudaStreamSynchronize(st));
    SC_REQUIRE(!(hs.nonfinite & 1), "Input X contains NaN.");
    SC_REQUIRE(!hs.nonfinite, "Input X contains infinity or a value too large for dtype('float64').");
    SC_REQUIRE(false, "The number of observations (%lld) is too small; the covariance matrix is "
               "singular. For observations with %lld dimensions, at least %lld observations are "
               "required.", (long long)(n + k), (long long)k_dim, (long long)(k_dim + 1));
  }
  const double* xs = e;                 // the rows stage 2 measures
  const double* cs = centers;           // and the centroids
  const double* aux = var ? var : vi;
  if (metric == KM_CORRELATION) {
    k_row_centre<<<nb, KT, 0, st>>>(e, n, k_dim, xc, nullptr); sc::launched();
    xs = xc;
    cs = cc;
  }
  const unsigned kb = (unsigned)((k + KT - 1) / KT);
  int64_t launched = 0;
  for (;;) {
    const int batch = 4;
    for (int b = 0; b < batch; ++b) {
      if (metric == KM_CORRELATION) {
        k_row_centre<<<kb, KT, 0, st>>>(centers, k, k_dim, cc, state); sc::launched();
      } else if (metric == KM_SEUCLIDEAN || metric == KM_MAHALANOBIS) {
        k_stack_col_stats<<<(unsigned)k_dim, KT, 0, st>>>(e, n, centers, k, k_dim, mu, var, state); sc::launched();
      }
      if (metric == KM_MAHALANOBIS) {
        k_stack_cov<<<dim3((unsigned)k_dim, (unsigned)k_dim), KT, 0, st>>>(e, n, centers, k, k_dim, mu,
                                                                           cv, state); sc::launched();
        k_inverse_t<<<1, 1024, 0, st>>>(cv, work, fac, k_dim, vi, state); sc::launched();
      }
      launch_assign(metric, nb, st, xs, n, k_dim, cs, k, labels, part, state, aux);
      k_cluster_sums<<<dim3((unsigned)k, (unsigned)k_dim), KT, 0, st>>>(e, n, k_dim, labels, sums,
                                                                        counts, counts_nz, state); sc::launched();
      k_custom_step<<<1, KT, 0, st>>>(part, nb, n, sums, counts_nz, k, k_dim, tol, max_iter,
                                      centers, counts, state); sc::launched();
    }
    launched += batch;
    SC_LAUNCH_CHECK();
    SC_CUDA(cudaMemcpyAsync(&hs, state, sizeof(hs), cudaMemcpyDeviceToHost, st));
    SC_CUDA(cudaStreamSynchronize(st));
    // scikit-learn's wording (sklearn/utils/validation.py, _assert_all_finite): NaN first
    SC_REQUIRE(!(hs.nonfinite & 1), "Input X contains NaN.");
    SC_REQUIRE(!hs.nonfinite, "Input X contains infinity or a value too large for dtype('float64').");
    SC_REQUIRE(!hs.singular, "Singular matrix");   // np.linalg.inv's LinAlgError
    if (hs.done) break;
    SC_REQUIRE(launched <= max_iter + 8, "sc_kmeans: stop rule never fired (internal error)");
  }
  SC_REQUIRE(!hs.empty_cluster, "sc_kmeans: a k-means++ seed lost all members in the Lloyd step "
             "(duplicate points); scikit-learn's empty-cluster relocation is not restated");
  std::vector<int> lab((size_t)n);
  SC_CUDA(cudaMemcpyAsync(lab.data(), labels, sizeof(int) * (size_t)n, cudaMemcpyDeviceToHost, st));
  SC_CUDA(cudaStreamSynchronize(st));
  for (int64_t i = 0; i < n; ++i) labels_host[i] = lab[(size_t)i];
  if (iters_host) *iters_host = hs.iters;
  return 0;
}
