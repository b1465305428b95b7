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
// metric: -1 = sklearn E-step (|c|^2 - 2 x.c), 0 = cosine (scipy cdist), 1 = euclidean
__global__ void k_assign(const double* __restrict__ x, int64_t n, int64_t kd,
                         const double* __restrict__ centers, int64_t k, int metric,
                         int* __restrict__ labels, double* __restrict__ part,
                         const KmState* st) {
  __shared__ double red[32];
  if (st->done) return;
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  double best = 0.0;
  if (i < n) {
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
  SC_REQUIRE(metric == 0 || metric == 1, "sc_kmeans: metric must be 0 (cosine) or 1 (euclidean)");
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
  k_assign<<<nb, KT, 0, st>>>(x, n, k_dim, centers, k, -1, labels, part, state); sc::launched();
  k_cluster_sums<<<dim3((unsigned)k, (unsigned)k_dim), KT, 0, st>>>(x, n, k_dim, labels, sums,
                                                                    counts, counts_nz, state); sc::launched();
  k_lloyd_update<<<(unsigned)((k * k_dim + KT - 1) / KT), KT, 0, st>>>(sums, counts, k, k_dim,
                                                                       mean, centers, state); sc::launched();
  SC_LAUNCH_CHECK();

  // ---- stage 2: CustomKMeans.predict on the un-centred embeddings
  KmState hs;
  int64_t launched = 0;
  for (;;) {
    const int batch = 4;
    for (int b = 0; b < batch; ++b) {
      k_assign<<<nb, KT, 0, st>>>(e, n, k_dim, centers, k, metric, labels, part, state); sc::launched();
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
