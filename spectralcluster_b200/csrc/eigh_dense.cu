// Dense symmetric eigensolver, fp64, on the device: Householder tridiagonalisation + implicit QL
// with eigenvector accumulation, then back-transformation of the requested eigenvectors and the
// similarity map-back of SURVEY.md A.2.  Replaces utils.compute_sorted_eigenvectors
// (utils.py:44-71, np.linalg.eig = LAPACK geev) for the symmetrisable matrices of the hot path:
//
//      M = diag(delta) + sign * diag(left) S diag(right)        (what the reference decomposes)
//      T = diag(delta) + sign * c S c,  c = sqrt(left*right)    (symmetric, same spectrum)
//      v = E u / |E u|,  E = sqrt(left/right)                   (reference eigenvectors)
//
// This is the full-spectrum solver (O(n^3), everything resident: 2 n^2 doubles + the rotation
// log).  It serves small/medium n and the max_clusters=None scan of utils.py:100-102 that needs
// all eigenvalues; large n with a bounded cluster count goes to the Lanczos solver in
// eigh_lanczos.cu.
//
// Kernels
//   k_build_sym       T <- delta + sign * c S c                         (n^2, HBM)
//   k_hh_reflector    Householder vector of column j (one CTA)
//   k_hh_symv         p <- T22 v          (warp per row, the HBM/L2-bound half of tridiag)
//   k_hh_w            w <- tau p - (tau^2 p.v / 2) v
//   k_hh_rank2        T22 <- T22 - v w^T - w v^T
//   k_sturm_bisect    every eigenvalue of (d, e) by Sturm-count bisection, one thread each: the
//                     parallel route to the full spectrum (n > 256) -- O(n^2) work spread over n
//                     threads instead of one thread's 3 n^2 dependent rotations
//   k_invit_*         inverse iteration (pivoted LU of T - lambda I, one thread per requested
//                     vector, workspaces interleaved for coalescing) + modified Gram-Schmidt
//                     inside clusters of close eigenvalues, three rounds
//   k_tql_rotations   implicit QL on (d, e), state in shared memory; logs every Givens rotation
//                     (one thread, O(n^2)); used when many eigenvectors are wanted at small n
//   k_apply_rotations Z <- Z G_1 G_2 ...  (one thread per row of Z, rotations streamed)
//   k_backtransform   u <- H_0 ... H_{n-3} z, v <- E u / |E u|  (one CTA per eigenvector)
#include "common.cuh"

#include <algorithm>
#include <numeric>
#include <vector>

namespace sc {

__global__ void k_build_sym(const float* __restrict__ s, int64_t n, int64_t lds,
                            const double* __restrict__ delta, const double* __restrict__ left,
                            const double* __restrict__ right, double sign,
                            double* __restrict__ t) {
  const int64_t i = blockIdx.x;
  const double ci = sqrt((left ? left[i] : 1.0) * (right ? right[i] : 1.0));
  for (int64_t j = (int64_t)blockIdx.y * blockDim.x + threadIdx.x; j < n;
       j += (int64_t)gridDim.y * blockDim.x) {
    const double cj = sqrt((left ? left[j] : 1.0) * (right ? right[j] : 1.0));
    // symmetrise the fp32 input explicitly: S is symmetric only up to rounding
    const double sij = 0.5 * ((double)s[i * lds + j] + (double)s[j * lds + i]);
    double v = sign * ci * cj * sij;
    if (i == j && delta) v += delta[i];
    t[i * n + j] = v;
  }
}

// Row j of the (fully updated, symmetric) matrix holds column j; x = T[j, j+1:n].
__global__ void k_hh_reflector(double* __restrict__ t, int64_t n, int64_t j,
                               double* __restrict__ d, double* __restrict__ e,
                               double* __restrict__ tau, double* __restrict__ vbuf) {
  __shared__ double red[32];
  __shared__ double sh[2];
  const int64_t m = n - j - 1;
  double* x = t + j * n + j + 1;
  double ss = 0.0;
  for (int64_t i = 1 + threadIdx.x; i < m; i += blockDim.x) ss += x[i] * x[i];
  ss = block_sum(ss, red);
  if (threadIdx.x == 0) {
    const double alpha = x[0];
    d[j] = t[j * n + j];
    if (ss == 0.0) {
      tau[j] = 0.0;
      e[j] = alpha;
      sh[0] = 0.0;      // scale (unused)
      sh[1] = 0.0;      // tau
    } else {
      const double beta = -copysign(sqrt(alpha * alpha + ss), alpha);
      tau[j] = (beta - alpha) / beta;
      e[j] = beta;
      sh[0] = 1.0 / (alpha - beta);
      sh[1] = tau[j];
    }
  }
  __syncthreads();
  const double scale = sh[0];
  const bool trivial = (sh[1] == 0.0);
  for (int64_t i = threadIdx.x; i < m; i += blockDim.x) {
    double v;
    if (i == 0) v = 1.0;
    else v = trivial ? 0.0 : x[i] * scale;
    vbuf[i] = v;
    x[i] = v;            // reflector kept in row j for the back-transformation
  }
}

__global__ void k_hh_symv(const double* __restrict__ t, int64_t n, int64_t j,
                          const double* __restrict__ vbuf, double* __restrict__ pbuf) {
  const int64_t m = n - j - 1;
  const int64_t r = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (r >= m) return;
  const int lane = threadIdx.x & 31;
  const double* row = t + (j + 1 + r) * n + (j + 1);
  double acc = 0.0;
  for (int64_t k = lane; k < m; k += 32) acc = fma(row[k], vbuf[k], acc);
  acc = warp_sum(acc);
  if (lane == 0) pbuf[r] = acc;
}

__global__ void k_hh_w(const double* __restrict__ tau, int64_t j, int64_t m,
                       const double* __restrict__ vbuf, const double* __restrict__ pbuf,
                       double* __restrict__ wbuf) {
  __shared__ double red[32];
  const double tj = tau[j];
  double pv = 0.0;
  for (int64_t i = threadIdx.x; i < m; i += blockDim.x) pv += pbuf[i] * vbuf[i];
  pv = block_sum(pv, red);
  const double corr = 0.5 * tj * tj * pv;
  for (int64_t i = threadIdx.x; i < m; i += blockDim.x) wbuf[i] = tj * pbuf[i] - corr * vbuf[i];
}

__global__ void k_hh_rank2(double* __restrict__ t, int64_t n, int64_t j,
                           const double* __restrict__ vbuf, const double* __restrict__ wbuf) {
  const int64_t m = n - j - 1;
  const int64_t r = blockIdx.y;
  const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= m) return;
  const double vr = vbuf[r], wr = wbuf[r];
  t[(j + 1 + r) * n + (j + 1 + c)] -= vr * wbuf[c] + wr * vbuf[c];
}

// ------------------------------------------------------------------ blocked tridiagonalisation
// LAPACK's dsytrd/dlatrd scheme on the full (both triangles) fp64 matrix: inside a panel of NB
// columns the trailing matrix is NOT touched -- column j is brought up to date from the panel's
// (V, W) pairs, its reflector v_j is formed, p_j = A22 v_j streams the stale trailing matrix once
// (the memory-bound half: n^3/3 elements in all) and is corrected with the same pairs; after the
// panel A22 -= V W^T + W V^T is ONE rank-2NB update on the fp64 tensor cores (DMMA m8n8k4), which
// replaces NB read-modify-write sweeps of the trailing matrix by one.
constexpr int NB = 32;

// Column j = j0 + k of the panel.  V, W are [NB][n] (vector-major).  One CTA.
//   x[r]   = A[j][r] - sum_{i<k} (V_i[j] W_i[r] + W_i[j] V_i[r]),  r > j   (row j == column j)
//   d[j]   = A[j][j] - 2 sum_{i<k} V_i[j] W_i[j]
//   v (v[j+1] = 1), tau[j], e[j] = beta; v goes to row j of A (back-transformation), to V_k and vbuf
__global__ void __launch_bounds__(1024)
k_panel_column(double* __restrict__ a, int64_t n, int64_t j, int k, double* __restrict__ vv,
               double* __restrict__ ww, double* __restrict__ d, double* __restrict__ e,
               double* __restrict__ tau, double* __restrict__ vbuf) {
  __shared__ double red[32];
  __shared__ double sv[NB], sw[NB];
  __shared__ double sh[2];
  const int64_t m = n - j - 1;
  if (threadIdx.x < k) {
    sv[threadIdx.x] = vv[(int64_t)threadIdx.x * n + j];
    sw[threadIdx.x] = ww[(int64_t)threadIdx.x * n + j];
  }
  __syncthreads();
  double* x = a + j * n + j + 1;
  double ss = 0.0;
  for (int64_t i = threadIdx.x; i < m; i += blockDim.x) {
    const int64_t r = j + 1 + i;
    double val = x[i];
    for (int q = 0; q < k; ++q) val -= sv[q] * ww[(int64_t)q * n + r] + sw[q] * vv[(int64_t)q * n + r];
    x[i] = val;
    if (i > 0) ss += val * val;
  }
  ss = block_sum(ss, red);
  if (threadIdx.x == 0) {
    double dj = a[j * n + j];
    for (int q = 0; q < k; ++q) dj -= 2.0 * sv[q] * sw[q];
    d[j] = dj;
    const double alpha = x[0];
    if (ss == 0.0) {
      tau[j] = 0.0;
      e[j] = alpha;
      sh[0] = 0.0;
      sh[1] = 0.0;
    } else {
      const double beta = -copysign(sqrt(alpha * alpha + ss), alpha);
      tau[j] = (beta - alpha) / beta;
      e[j] = beta;
      sh[0] = 1.0 / (alpha - beta);
      sh[1] = tau[j];
    }
  }
  __syncthreads();
  const double scale = sh[0];
  const bool trivial = (sh[1] == 0.0);
  double* vk = vv + (int64_t)k * n;
  for (int64_t r = threadIdx.x; r <= j; r += blockDim.x) vk[r] = 0.0;
  for (int64_t i = threadIdx.x; i < m; i += blockDim.x) {
    const double v = (i == 0) ? 1.0 : (trivial ? 0.0 : x[i] * scale);
    vbuf[i] = v;
    x[i] = v;
    vk[j + 1 + i] = v;
  }
}

// p (from the stale trailing matrix) -> w_k.  One CTA of 32 warps: warp i takes the two dot
// products with (V_i, W_i); then every thread corrects and scales its rows.
__global__ void __launch_bounds__(1024)
k_panel_w(int64_t n, int64_t j, int k, const double* __restrict__ tau, const double* __restrict__ vv,
          double* __restrict__ ww, const double* __restrict__ vbuf, double* __restrict__ pbuf) {
  __shared__ double red[32];
  __shared__ double g1[NB], g2[NB];       // W_i^T v, V_i^T v
  const int64_t m = n - j - 1;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (warp < k) {
    const double* wi = ww + (int64_t)warp * n + j + 1;
    const double* vi = vv + (int64_t)warp * n + j + 1;
    double a1 = 0.0, a2 = 0.0;
    for (int64_t i = lane; i < m; i += 32) {
      const double v = vbuf[i];
      a1 = fma(wi[i], v, a1);
      a2 = fma(vi[i], v, a2);
    }
    a1 = warp_sum(a1);
    a2 = warp_sum(a2);
    if (lane == 0) { g1[warp] = a1; g2[warp] = a2; }
  }
  __syncthreads();
  double pv = 0.0;
  for (int64_t i = threadIdx.x; i < m; i += blockDim.x) {
    const int64_t r = j + 1 + i;
    double val = pbuf[i];
    for (int q = 0; q < k; ++q) val -= vv[(int64_t)q * n + r] * g1[q] + ww[(int64_t)q * n + r] * g2[q];
    pbuf[i] = val;
    pv = fma(val, vbuf[i], pv);
  }
  pv = block_sum(pv, red);
  const double tj = tau[j];
  const double corr = 0.5 * tj * tj * pv;
  double* wk = ww + (int64_t)k * n;
  for (int64_t r = threadIdx.x; r <= j; r += blockDim.x) wk[r] = 0.0;
  for (int64_t i = threadIdx.x; i < m; i += blockDim.x) wk[j + 1 + i] = tj * pbuf[i] - corr * vbuf[i];
}

// A[r][c] -= sum_{i<kc} (V_i[r] W_i[c] + W_i[r] V_i[c]) for r, c >= lo: C -= P Q^T with
// P = [V | W], Q = [W | V] (K = 2 kc), 64 x 64 tile per CTA, 8 warps x (8 rows x 64 columns), on the
// fp64 tensor cores (mma.sync m8n8k4; SASS DMMA).
constexpr int UPD_T = 64;
constexpr int UPD_PITCH = 2 * NB + 4;     // doubles; == 4 mod 16: conflict-free 64-bit fragment loads

__global__ void __launch_bounds__(256)
k_trailing_update(double* __restrict__ a, int64_t n, int64_t lo, int kc,
                  const double* __restrict__ vv, const double* __restrict__ ww) {
  extern __shared__ double upd_smem[];                       // P tile, Q tile: [64][UPD_PITCH] each
  double* ps = upd_smem;
  double* qs = upd_smem + UPD_T * UPD_PITCH;
  const int64_t r0 = lo + (int64_t)blockIdx.y * UPD_T, c0 = lo + (int64_t)blockIdx.x * UPD_T;
  const int kk = 2 * kc;
  for (int idx = threadIdx.x; idx < kk * UPD_T; idx += blockDim.x) {
    const int q = idx / UPD_T, t = idx - q * UPD_T;           // consecutive threads: consecutive rows
    const double* pv = (q < kc) ? vv + (int64_t)q * n : ww + (int64_t)(q - kc) * n;
    const double* qv = (q < kc) ? ww + (int64_t)q * n : vv + (int64_t)(q - kc) * n;
    ps[t * UPD_PITCH + q] = (r0 + t < n) ? pv[r0 + t] : 0.0;
    qs[t * UPD_PITCH + q] = (c0 + t < n) ? qv[c0 + t] : 0.0;
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int fr = lane >> 2, fk = lane & 3;                    // fragment row (or column) / k index
  double acc[8][2];
#pragma unroll
  for (int t = 0; t < 8; ++t) acc[t][0] = acc[t][1] = 0.0;
  for (int k0 = 0; k0 < kk; k0 += 4) {
    const double av = ps[(warp * 8 + fr) * UPD_PITCH + k0 + fk];
#pragma unroll
    for (int t = 0; t < 8; ++t) {
      const double bv = qs[(t * 8 + fr) * UPD_PITCH + k0 + fk];
      dmma_m8n8k4(acc[t][0], acc[t][1], av, bv);
    }
  }
  const int64_t row = r0 + warp * 8 + fr;
  if (row < n) {
#pragma unroll
    for (int t = 0; t < 8; ++t) {
      const int64_t col = c0 + t * 8 + fk * 2;
      double* dst = a + row * n + col;
      if (col + 1 < n) {
        double2 cur = *reinterpret_cast<double2*>(dst);
        cur.x -= acc[t][0];
        cur.y -= acc[t][1];
        *reinterpret_cast<double2*>(dst) = cur;
      } else if (col < n) {
        dst[0] -= acc[t][0];
      }
    }
  }
}

__global__ void k_hh_tail(const double* __restrict__ t, int64_t n, double* d, double* e,
                          double* tau) {
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  if (n >= 2) {
    d[n - 2] = t[(n - 2) * n + (n - 2)];
    e[n - 2] = t[(n - 2) * n + (n - 1)];
    tau[n - 2] = 0.0;
  }
  d[n - 1] = t[(n - 1) * n + (n - 1)];
  e[n - 1] = 0.0;
  tau[n - 1] = 0.0;
}

struct Sweep {
  int first_i;      // first rotation acts on columns (first_i, first_i + 1), then first_i - 1, ...
  int count;
  long long offset; // into the rotation log
};

struct QlStatus {
  long long n_rot;
  int n_sweeps;
  int status;       // 0 ok, 1 no convergence, 2 rotation log overflow, 3 sweep log overflow
};

// Implicit QL with Wilkinson shift (the classical tql2 recurrences, restated).  d: diagonal,
// e[i]: coupling between i and i+1 (e[n-1] = 0).  One thread; the rotations are logged so that
// the O(n^3) eigenvector update can run in parallel afterwards.
__global__ void k_tql_rotations(double* __restrict__ d_glob, double* __restrict__ e_glob, int n,
                                double* __restrict__ rc, double* __restrict__ rs,
                                long long rot_cap, Sweep* __restrict__ sweeps, int sweep_cap,
                                QlStatus* __restrict__ out, int use_smem) {
  // the recurrence is one dependent chain: keep its state (2 n doubles) in shared memory when it
  // fits -- every d[]/e[] access was a global round trip before (~1000 cycles per rotation)
  extern __shared__ double ql_state[];
  double* d = use_smem ? ql_state : d_glob;
  double* e = use_smem ? ql_state + n : e_glob;
  if (use_smem) {
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      d[i] = d_glob[i];
      e[i] = e_glob[i];
    }
    __syncthreads();
  }
  if (threadIdx.x != 0 || blockIdx.x != 0) return;
  const double eps = 2.220446049250313e-16;
  long long nrot = 0;
  int nsw = 0, status = 0;
  for (int l = 0; l < n && status == 0; ++l) {
    int iter = 0, m;
    do {
      for (m = l; m < n - 1; ++m) {
        const double dd = fabs(d[m]) + fabs(d[m + 1]);
        if (fabs(e[m]) <= eps * dd) break;
      }
      if (m != l) {
        if (iter++ == 60) { status = 1; break; }
        if (nsw >= sweep_cap) { status = 3; break; }
        if (nrot + (m - l) > rot_cap) { status = 2; break; }
        double g = (d[l + 1] - d[l]) / (2.0 * e[l]);
        double r = hypot(g, 1.0);
        g = d[m] - d[l] + e[l] / (g + copysign(r, g));
        double s = 1.0, c = 1.0, p = 0.0;
        const long long start = nrot;
        int i;
        for (i = m - 1; i >= l; --i) {
          double f = s * e[i];
          const double b = c * e[i];
          r = hypot(f, g);
          e[i + 1] = r;
          if (r == 0.0) {
            d[i + 1] -= p;
            e[m] = 0.0;
            break;
          }
          s = f / r;
          c = g / r;
          g = d[i + 1] - p;
          r = (d[i] - g) * s + 2.0 * c * b;
          p = s * r;
          d[i + 1] = g + p;
          g = c * r - b;
          rc[nrot] = c;
          rs[nrot] = s;
          ++nrot;
        }
        sweeps[nsw].first_i = m - 1;
        sweeps[nsw].count = (int)(nrot - start);
        sweeps[nsw].offset = start;
        ++nsw;
        if (r == 0.0 && i >= l) continue;
        d[l] -= p;
        e[l] = g;
        e[m] = 0.0;
      }
    } while (m != l);
  }
  out->n_rot = nrot;
  out->n_sweeps = nsw;
  out->status = status;
  if (use_smem)
    for (int i = 0; i < n; ++i) d_glob[i] = d[i];
}

// zt is Z transposed: zt[col * n + row]; thread = row.  Z starts as the identity.
__global__ void k_apply_rotations(double* __restrict__ zt, int64_t n,
                                  const Sweep* __restrict__ sweeps, int n_sweeps,
                                  const double* __restrict__ rc, const double* __restrict__ rs) {
  const int64_t k = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (k >= n) return;
  for (int sw = 0; sw < n_sweeps; ++sw) {
    const int i0 = sweeps[sw].first_i, cnt = sweeps[sw].count;
    const long long off = sweeps[sw].offset;
    if (cnt == 0) continue;
    double carry = zt[(int64_t)(i0 + 1) * n + k];
    int t = 0;
    // batches of 8: the loads are independent of the carry chain, issue them together
    for (; t + 8 <= cnt; t += 8) {
      double z[8];
#pragma unroll
      for (int u = 0; u < 8; ++u) z[u] = zt[(int64_t)(i0 - t - u) * n + k];
#pragma unroll
      for (int u = 0; u < 8; ++u) {
        const double c = rc[off + t + u], s = rs[off + t + u];
        zt[(int64_t)(i0 - t - u + 1) * n + k] = s * z[u] + c * carry;
        carry = c * z[u] - s * carry;
      }
    }
    for (; t < cnt; ++t) {
      const double c = rc[off + t], s = rs[off + t];
      const double zi = zt[(int64_t)(i0 - t) * n + k];
      zt[(int64_t)(i0 - t + 1) * n + k] = s * zi + c * carry;
      carry = c * zi - s * carry;
    }
    zt[(int64_t)(i0 - cnt + 1) * n + k] = carry;
  }
}

__global__ void k_identity(double* __restrict__ zt, int64_t n) {
  const int64_t i = blockIdx.x;
  for (int64_t j = threadIdx.x; j < n; j += blockDim.x) zt[i * n + j] = (i == j) ? 1.0 : 0.0;
}

// One CTA per requested eigenvector: u = H_0 H_1 ... H_{n-3} z ; v = E u / |E u|.
// t holds reflector j in row j (columns j+1..n-1).  u lives in dynamic shared memory.
__global__ void k_backtransform(const double* __restrict__ t, int64_t n,
                                const double* __restrict__ tau, const double* __restrict__ zt,
                                const int* __restrict__ sel, int64_t n_sel,
                                const double* __restrict__ left, const double* __restrict__ right,
                                double* __restrict__ v_out) {
  extern __shared__ double u[];
  __shared__ double red[32];
  const int64_t col = blockIdx.x;
  const double* z = zt + (int64_t)sel[col] * n;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) u[i] = z[i];
  __syncthreads();
  for (int64_t j = n - 3; j >= 0; --j) {
    const double tj = tau[j];
    if (tj == 0.0) continue;                      // uniform across the block
    const int64_t m = n - j - 1;
    const double* v = t + j * n + j + 1;
    double dot = 0.0;
    for (int64_t i = threadIdx.x; i < m; i += blockDim.x) dot += v[i] * u[j + 1 + i];
    dot = block_sum(dot, red);
    const double f = tj * dot;
    for (int64_t i = threadIdx.x; i < m; i += blockDim.x) u[j + 1 + i] -= f * v[i];
    __syncthreads();
  }
  double ss = 0.0;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
    const double ei = sqrt((left ? left[i] : 1.0) / (right ? right[i] : 1.0));
    const double x = ei * u[i];
    u[i] = x;
    ss += x * x;
  }
  ss = block_sum(ss, red);
  const double inv = 1.0 / sqrt(ss);
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) v_out[i * n_sel + col] = u[i] * inv;
}

// ------------------------------------------------------------------ bisection + inverse iteration
// Number of eigenvalues of the symmetric tridiagonal (d, e) that are < x (Sturm sequence of the
// LDL^T pivots; tiny pivots are pushed to -pivmin as in LAPACK's dstebz).
__device__ __forceinline__ int sturm_count(const double* __restrict__ d, const double* __restrict__ e2,
                                           int n, double x, double pivmin) {
  double q = d[0] - x;
  int cnt = (q < 0.0);
  for (int k = 1; k < n; ++k) {
    if (fabs(q) < pivmin) q = -pivmin;
    q = d[k] - x - e2[k - 1] / q;
    cnt += (q < 0.0);
  }
  return cnt;
}

// w[i] = i-th smallest eigenvalue, one thread per i, bisection on [lo, hi] (Gershgorin) until the
// interval no longer shrinks in fp64.
__global__ void k_sturm_bisect(const double* __restrict__ d, const double* __restrict__ e2, int n,
                               double lo, double hi, double pivmin, double* __restrict__ w) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double a = lo, b = hi;
  for (int it = 0; it < 200; ++it) {
    const double mid = 0.5 * (a + b);
    if (mid <= a || mid >= b) break;
    if (sturm_count(d, e2, n, mid, pivmin) > i) b = mid;
    else a = mid;
  }
  w[i] = 0.5 * (a + b);
}

__global__ void k_square(const double* __restrict__ e, int n, double* __restrict__ e2) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) e2[i] = e[i] * e[i];
}

// Workspace of vector v, array `arr` (0..4: a, b, c, d2, pivot flag), entry k: interleaved over
// the vectors so that the threads of a warp (one vector each) touch consecutive addresses.
#define IW(arr, k) ws[((size_t)(arr) * n + (k)) * nvec + v]

// Pivoted LU of T - lambda I (the dlagtf recurrences restated), one thread per vector.
__global__ void k_invit_factor(const double* __restrict__ d, const double* __restrict__ e, int n,
                               const double* __restrict__ lambda, int nvec,
                               double* __restrict__ ws) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= nvec) return;
  const double lam = lambda[v];
  for (int k = 0; k < n; ++k) {
    IW(0, k) = d[k] - lam;
    IW(1, k) = (k < n - 1) ? e[k] : 0.0;      // super-diagonal
    IW(2, k) = (k < n - 1) ? e[k] : 0.0;      // sub-diagonal, becomes the multipliers
    IW(3, k) = 0.0;                           // second super-diagonal created by pivoting
    IW(4, k) = 0.0;                           // 1 = rows k, k+1 were interchanged
  }
  double scale1 = fabs(IW(0, 0)) + fabs(IW(1, 0));
  for (int k = 0; k < n - 1; ++k) {
    const double ak = IW(0, k), ck = IW(2, k);
    double ak1 = IW(0, k + 1);
    double scale2 = fabs(ck) + fabs(ak1);
    if (k < n - 2) scale2 += fabs(IW(1, k + 1));
    const double piv1 = (ak == 0.0) ? 0.0 : fabs(ak) / scale1;
    if (ck == 0.0) {
      scale1 = scale2;
    } else {
      const double piv2 = fabs(ck) / scale2;
      if (piv2 <= piv1) {                      // no interchange
        scale1 = scale2;
        const double mult = ck / ak;
        IW(2, k) = mult;
        IW(0, k + 1) = ak1 - mult * IW(1, k);
      } else {                                 // interchange rows k and k+1
        const double mult = ak / ck;
        IW(4, k) = 1.0;
        IW(0, k) = ck;
        const double bk = IW(1, k);
        IW(0, k + 1) = bk - mult * ak1;
        if (k < n - 2) {
          const double bk1 = IW(1, k + 1);
          IW(3, k) = bk1;
          IW(1, k + 1) = -mult * bk1;
        }
        IW(1, k) = ak1;
        IW(2, k) = mult;
      }
    }
  }
}

// x <- (T - lambda I)^-1 x through the stored factors (dlagts, job -1 flavour: a vanishing pivot
// is replaced by +-pivmin instead of overflowing); x is [nvec][n], contiguous per vector.
__global__ void k_invit_solve(int n, int nvec, const double* __restrict__ ws, double pivmin,
                              double* __restrict__ x) {
  const int v = blockIdx.x * blockDim.x + threadIdx.x;
  if (v >= nvec) return;
  double* y = x + (size_t)v * n;
  for (int k = 1; k < n; ++k) {
    if (IW(4, k - 1) == 0.0) {
      y[k] -= IW(2, k - 1) * y[k - 1];
    } else {
      const double temp = y[k - 1];
      y[k - 1] = y[k];
      y[k] = temp - IW(2, k - 1) * y[k];
    }
  }
  for (int k = n - 1; k >= 0; --k) {
    double temp = y[k];
    if (k < n - 1) temp -= IW(1, k) * y[k + 1];
    if (k < n - 2) temp -= IW(3, k) * y[k + 2];
    double ak = IW(0, k);
    if (fabs(ak) < pivmin) ak = copysign(pivmin, ak == 0.0 ? 1.0 : ak);
    y[k] = temp / ak;
  }
}
#undef IW

__global__ void k_invit_start(double* __restrict__ x, int n, int nvec) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)n * nvec) return;
  uint64_t z = 0x51ED270B0ull + 0x9E3779B97F4A7C15ull * (uint64_t)(i + 1);   // splitmix64
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  z ^= z >> 31;
  x[i] = (double)(z >> 11) * (1.0 / 9007199254740992.0) + 0.25;
}

// One CTA per cluster of close eigenvalues [first, first+count): modified Gram-Schmidt in order,
// every vector scaled to unit norm (singletons are just normalised).
__global__ void k_invit_orthonormalize(double* __restrict__ x, int n,
                                       const int* __restrict__ cluster_first,
                                       const int* __restrict__ cluster_count) {
  __shared__ double red[32];
  const int first = cluster_first[blockIdx.x], count = cluster_count[blockIdx.x];
  for (int a = 0; a < count; ++a) {
    double* xa = x + (size_t)(first + a) * n;
    for (int b = 0; b < a; ++b) {
      const double* xb = x + (size_t)(first + b) * n;
      double dot = 0.0;
      for (int i = threadIdx.x; i < n; i += blockDim.x) dot += xa[i] * xb[i];
      dot = block_sum(dot, red);
      for (int i = threadIdx.x; i < n; i += blockDim.x) xa[i] -= dot * xb[i];
      __syncthreads();
    }
    double ss = 0.0;
    for (int i = threadIdx.x; i < n; i += blockDim.x) ss += xa[i] * xa[i];
    ss = block_sum(ss, red);
    const double inv = 1.0 / sqrt(ss);
    for (int i = threadIdx.x; i < n; i += blockDim.x) xa[i] *= inv;
    __syncthreads();
  }
}

// Global-memory twin of k_backtransform for n beyond the shared-memory budget: u is a per-vector
// scratch row in HBM/L2.
__global__ void k_backtransform_gmem(const double* __restrict__ t, int64_t n,
                                     const double* __restrict__ tau, const double* __restrict__ zt,
                                     const int* __restrict__ sel, int64_t n_sel,
                                     const double* __restrict__ left, const double* __restrict__ right,
                                     double* __restrict__ scratch, double* __restrict__ v_out) {
  __shared__ double red[32];
  const int64_t col = blockIdx.x;
  const double* z = zt + (int64_t)sel[col] * n;
  double* u = scratch + col * n;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) u[i] = z[i];
  __syncthreads();
  for (int64_t j = n - 3; j >= 0; --j) {
    const double tj = tau[j];
    if (tj == 0.0) continue;
    const int64_t m = n - j - 1;
    const double* v = t + j * n + j + 1;
    double dot = 0.0;
    for (int64_t i = threadIdx.x; i < m; i += blockDim.x) dot += v[i] * u[j + 1 + i];
    dot = block_sum(dot, red);
    const double f = tj * dot;
    for (int64_t i = threadIdx.x; i < m; i += blockDim.x) u[j + 1 + i] -= f * v[i];
    __syncthreads();
  }
  double ss = 0.0;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
    const double ei = sqrt((left ? left[i] : 1.0) / (right ? right[i] : 1.0));
    const double x = ei * u[i];
    u[i] = x;
    ss += x * x;
  }
  ss = block_sum(ss, red);
  const double inv = 1.0 / sqrt(ss);
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) v_out[i * n_sel + col] = u[i] * inv;
}

}  // namespace sc

using namespace sc;

typedef int64_t (*sc_pick_fn)(void* user, const double* w_sorted, int64_t n_values, void** v_dev_out);

extern "C" int sc_eigh_dense(sc_context* ctx, const float* s, int64_t n, int64_t lds,
                             const double* delta, const double* left, const double* right,
                             double sign, int which, int64_t n_values, int64_t n_vectors,
                             double* w_host, double* v_dev, sc_pick_fn pick, void* user,
                             void* stream) {
  SC_REQUIRE(ctx && s && n > 0 && w_host, "sc_eigh_dense: bad arguments");
  SC_REQUIRE(n_values >= 0 && n_values <= n && n_vectors >= 0 && n_vectors <= n_values,
             "sc_eigh_dense: need 0 <= n_vectors <= n_values <= n");
  SC_REQUIRE(pick || n_vectors == 0 || v_dev, "sc_eigh_dense: v_dev missing");
  SC_REQUIRE(n <= 32768, "sc_eigh_dense: n=%lld exceeds the dense solver limit (32768: 8 n^2 B of "
             "fp64 working matrix); use sc_eigh_extremal", (long long)n);
  cudaStream_t st = as_stream(stream);
  const size_t nn = (size_t)n * (size_t)n;

  Scratch T, Zt, vec, rc, rs, sw, stat, selbuf;
  SC_CUDA(T.alloc(sizeof(double) * nn, st));
  SC_CUDA(vec.alloc(sizeof(double) * (size_t)n * 8, st));
  double* d = vec.as<double>();
  double* e = d + n;
  double* tau = e + n;
  double* vbuf = tau + n;
  double* pbuf = vbuf + n;
  double* wbuf = pbuf + n;
  double* e2 = wbuf + n;
  double* wall = e2 + n;

  const unsigned gy = (unsigned)std::min<int64_t>((n + 255) / 256, 64);
  k_build_sym<<<dim3((unsigned)n, gy), 256, 0, st>>>(s, n, lds, delta, left, right, sign,
                                                    T.as<double>()); sc::launched();
  SC_LAUNCH_CHECK();
  if (n < 256 || (n & 1)) {
    // small (or odd-sized: the update uses 16-byte accesses) matrices: unblocked, rank-2 update per column
    for (int64_t j = 0; j + 2 < n; ++j) {
      const int64_t m = n - j - 1;
      k_hh_reflector<<<1, 512, 0, st>>>(T.as<double>(), n, j, d, e, tau, vbuf); sc::launched();
      k_hh_symv<<<(unsigned)((m + 7) / 8), 256, 0, st>>>(T.as<double>(), n, j, vbuf, pbuf); sc::launched();
      k_hh_w<<<1, 512, 0, st>>>(tau, j, m, vbuf, pbuf, wbuf); sc::launched();
      k_hh_rank2<<<dim3((unsigned)((m + 255) / 256), (unsigned)m), 256, 0, st>>>(T.as<double>(), n,
                                                                                  j, vbuf, wbuf); sc::launched();
    }
  } else {
    Scratch panel;
    SC_CUDA(panel.alloc(sizeof(double) * 2 * NB * (size_t)n, st));
    double* vv = panel.as<double>();
    double* ww = vv + (size_t)NB * n;
    const size_t upd_smem = sizeof(double) * 2 * UPD_T * UPD_PITCH;
    SC_CUDA(cudaFuncSetAttribute(k_trailing_update, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)upd_smem));
    for (int64_t j0 = 0; j0 + 2 < n; j0 += NB) {
      int kc = 0;
      for (; kc < NB && j0 + kc + 2 < n; ++kc) {
        const int64_t j = j0 + kc, m = n - j - 1;
        k_panel_column<<<1, 1024, 0, st>>>(T.as<double>(), n, j, kc, vv, ww, d, e, tau, vbuf); sc::launched();
        k_hh_symv<<<(unsigned)((m + 7) / 8), 256, 0, st>>>(T.as<double>(), n, j, vbuf, pbuf); sc::launched();
        k_panel_w<<<1, 1024, 0, st>>>(n, j, kc, tau, vv, ww, vbuf, pbuf); sc::launched();
      }
      const int64_t lo = j0 + kc;                 // first row / column of the trailing matrix
      const unsigned tiles = (unsigned)((n - lo + UPD_T - 1) / UPD_T);
      if (tiles > 0) {
        k_trailing_update<<<dim3(tiles, tiles), 256, upd_smem, st>>>(T.as<double>(), n, lo, kc, vv, ww);
        sc::launched();
      }
    }
  }
  SC_LAUNCH_CHECK();
  k_hh_tail<<<1, 32, 0, st>>>(T.as<double>(), n, d, e, tau); sc::launched();
  SC_LAUNCH_CHECK();

  // Which route to the spectrum: implicit QL logs O(n^2) rotations from ONE thread and pays off only
  // when (nearly) all eigenvectors are wanted at small n (the rotations rebuild Z for every row
  // in parallel); everything else -- in particular the full-spectrum scan of max_clusters=None
  // (utils.py:100-102) -- takes bisection + inverse iteration, which is parallel over eigenvalues.
  const bool use_ql = (n <= 256) || (!pick && n_vectors > 64 && n <= 16384);
  std::vector<double> dh((size_t)n);
  QlStatus hs = {};
  if (use_ql) {
    const long long rot_cap = 2LL * n * n + 1024;
    const int sweep_cap = (int)std::min<long long>(64LL * n + 64, 2000000000LL);
    SC_CUDA(rc.alloc(sizeof(double) * (size_t)rot_cap, st));
    SC_CUDA(rs.alloc(sizeof(double) * (size_t)rot_cap, st));
    SC_CUDA(sw.alloc(sizeof(Sweep) * (size_t)sweep_cap, st));
    SC_CUDA(stat.alloc(sizeof(QlStatus), st));
    const size_t ql_smem = sizeof(double) * 2 * (size_t)n;
    const int in_smem = ql_smem <= ctx->smem_optin ? 1 : 0;
    if (in_smem)
      SC_CUDA(cudaFuncSetAttribute(k_tql_rotations, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                   (int)ql_smem));
    k_tql_rotations<<<1, 256, in_smem ? ql_smem : 0, st>>>(d, e, (int)n, rc.as<double>(),
                                                          rs.as<double>(), rot_cap, sw.as<Sweep>(),
                                                          sweep_cap, stat.as<QlStatus>(), in_smem);
    sc::launched();
    SC_LAUNCH_CHECK();
    SC_CUDA(cudaMemcpyAsync(&hs, stat.p, sizeof(hs), cudaMemcpyDeviceToHost, st));
    SC_CUDA(cudaMemcpyAsync(dh.data(), d, sizeof(double) * (size_t)n, cudaMemcpyDeviceToHost, st));
    SC_CUDA(cudaStreamSynchronize(st));
    SC_REQUIRE(hs.status == 0, "sc_eigh_dense: implicit QL failed (status %d: 1=no convergence, "
               "2=rotation log overflow, 3=sweep log overflow)", hs.status);
  } else {
    // Gershgorin interval and the pivot floor from (d, e) on the host (2 n doubles)
    std::vector<double> eh((size_t)n);
    SC_CUDA(cudaMemcpyAsync(dh.data(), d, sizeof(double) * (size_t)n, cudaMemcpyDeviceToHost, st));
    SC_CUDA(cudaMemcpyAsync(eh.data(), e, sizeof(double) * (size_t)n, cudaMemcpyDeviceToHost, st));
    SC_CUDA(cudaStreamSynchronize(st));
    double lo = dh[0], hi = dh[0], emax = 0.0;
    for (int64_t i = 0; i < n; ++i) {
      const double r = (i > 0 ? std::fabs(eh[(size_t)i - 1]) : 0.0) + (i + 1 < n ? std::fabs(eh[(size_t)i]) : 0.0);
      lo = std::min(lo, dh[(size_t)i] - r);
      hi = std::max(hi, dh[(size_t)i] + r);
      emax = std::max(emax, std::fabs(eh[(size_t)i]));
    }
    const double tnorm = std::max(std::fabs(lo), std::fabs(hi));
    const double pivmin = std::max(2.2250738585072014e-308 * std::max(1.0, emax * emax), 1e-300);
    const double margin = 2.0 * tnorm * 2.220446049250313e-16 * (double)n + 2.0 * pivmin;
    k_square<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(e, (int)n, e2); sc::launched();
    k_sturm_bisect<<<(unsigned)((n + 63) / 64), 64, 0, st>>>(d, e2, (int)n, lo - margin, hi + margin,
                                                            pivmin, wall); sc::launched();
    SC_LAUNCH_CHECK();
    SC_CUDA(cudaMemcpyAsync(dh.data(), wall, sizeof(double) * (size_t)n, cudaMemcpyDeviceToHost, st));
    SC_CUDA(cudaStreamSynchronize(st));
  }

  // host: order the spectrum (argsort of +-w, utils.py:62-67)
  std::vector<int> order((size_t)n);
  std::iota(order.begin(), order.end(), 0);
  if (which == SC_EIG_LARGEST)
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return dh[a] > dh[b]; });
  else
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return dh[a] < dh[b]; });
  for (int64_t i = 0; i < n_values; ++i) w_host[i] = dh[(size_t)order[(size_t)i]];

  if (pick) {                      // the caller decides how many eigenvectors it needs from w
    void* out = nullptr;
    n_vectors = pick(user, w_host, n_values, &out);
    SC_REQUIRE(n_vectors >= 0 && n_vectors <= n_values && (n_vectors == 0 || out),
               "sc_eigh_dense: the pick callback returned a bad count / buffer");
    v_dev = static_cast<double*>(out);
  }
  if (n_vectors == 0) return 0;

  Scratch zsel, bt_scratch;
  const double* zrows = nullptr;          // eigenvectors of the tridiagonal, one per row of length n
  std::vector<int> sel((size_t)n_vectors);
  if (use_ql) {
    SC_CUDA(Zt.alloc(sizeof(double) * nn, st));
    k_identity<<<(unsigned)n, 256, 0, st>>>(Zt.as<double>(), n); sc::launched();
    SC_LAUNCH_CHECK();
    if (hs.n_sweeps > 0) {
      k_apply_rotations<<<(unsigned)((n + 63) / 64), 64, 0, st>>>(
          Zt.as<double>(), n, sw.as<Sweep>(), hs.n_sweeps, rc.as<double>(), rs.as<double>()); sc::launched();
      SC_LAUNCH_CHECK();
    }
    zrows = Zt.as<double>();
    for (int64_t i = 0; i < n_vectors; ++i) sel[(size_t)i] = order[(size_t)i];
  } else {
    // inverse iteration for the first n_vectors eigenvalues of the requested order
    const int nv = (int)n_vectors;
    Scratch lam, ws, cf, cc;
    SC_CUDA(lam.alloc(sizeof(double) * (size_t)nv, st));
    SC_CUDA(ws.alloc(sizeof(double) * 5 * (size_t)n * (size_t)nv, st));
    SC_CUDA(zsel.alloc(sizeof(double) * (size_t)n * (size_t)nv, st));
    std::vector<double> lh((size_t)nv);
    double tnorm = 0.0;
    for (int64_t i = 0; i < n; ++i) tnorm = std::max(tnorm, std::fabs(dh[(size_t)i]));
    tnorm = std::max(tnorm, 1e-300);
    // clusters of close eigenvalues (dstein's 1e-3 |T| rule) are orthogonalised together; members
    // are nudged apart by a few ulps so that their factorizations differ
    std::vector<int> cfirst, ccount;
    for (int i = 0; i < nv; ++i) {
      lh[(size_t)i] = dh[(size_t)order[(size_t)i]];
      const bool close = i > 0 && std::fabs(lh[(size_t)i] - dh[(size_t)order[(size_t)i - 1]]) <= 1e-3 * tnorm;
      if (close) {
        ++ccount.back();
        const double sep = 10.0 * 2.220446049250313e-16 * tnorm;
        const double dir = (which == SC_EIG_LARGEST) ? -1.0 : 1.0;
        if (std::fabs(lh[(size_t)i] - lh[(size_t)i - 1]) < sep) lh[(size_t)i] = lh[(size_t)i - 1] + dir * sep;
      } else {
        cfirst.push_back(i);
        ccount.push_back(1);
      }
    }
    SC_CUDA(cf.alloc(sizeof(int) * cfirst.size(), st));
    SC_CUDA(cc.alloc(sizeof(int) * ccount.size(), st));
    SC_CUDA(cudaMemcpyAsync(lam.p, lh.data(), sizeof(double) * (size_t)nv, cudaMemcpyHostToDevice, st));
    SC_CUDA(cudaMemcpyAsync(cf.p, cfirst.data(), sizeof(int) * cfirst.size(), cudaMemcpyHostToDevice, st));
    SC_CUDA(cudaMemcpyAsync(cc.p, ccount.data(), sizeof(int) * ccount.size(), cudaMemcpyHostToDevice, st));
    const double pivmin = 2.220446049250313e-16 * tnorm;
    const unsigned gv = (unsigned)((nv + 31) / 32);
    k_invit_factor<<<gv, 32, 0, st>>>(d, e, (int)n, lam.as<double>(), nv, ws.as<double>()); sc::launched();
    k_invit_start<<<(unsigned)(((int64_t)n * nv + 255) / 256), 256, 0, st>>>(zsel.as<double>(), (int)n, nv); sc::launched();
    for (int round = 0; round < 3; ++round) {
      k_invit_solve<<<gv, 32, 0, st>>>((int)n, nv, ws.as<double>(), pivmin, zsel.as<double>()); sc::launched();
      k_invit_orthonormalize<<<(unsigned)cfirst.size(), 256, 0, st>>>(zsel.as<double>(), (int)n,
                                                                      cf.as<int>(), cc.as<int>()); sc::launched();
    }
    SC_LAUNCH_CHECK();
    SC_CUDA(cudaStreamSynchronize(st));     // the host vectors above feed async copies
    zrows = zsel.as<double>();
    for (int64_t i = 0; i < n_vectors; ++i) sel[(size_t)i] = (int)i;
  }
  SC_CUDA(selbuf.alloc(sizeof(int) * (size_t)n_vectors, st));
  SC_CUDA(cudaMemcpyAsync(selbuf.p, sel.data(), sizeof(int) * (size_t)n_vectors,
                          cudaMemcpyHostToDevice, st));
  const size_t smem = sizeof(double) * (size_t)n;
  if (smem <= ctx->smem_optin) {
    SC_CUDA(cudaFuncSetAttribute(k_backtransform, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                 (int)smem));
    k_backtransform<<<(unsigned)n_vectors, 256, smem, st>>>(T.as<double>(), n, tau, zrows,
                                                            selbuf.as<int>(), n_vectors, left,
                                                            right, v_dev); sc::launched();
  } else {
    SC_CUDA(bt_scratch.alloc(sizeof(double) * (size_t)n * (size_t)n_vectors, st));
    k_backtransform_gmem<<<(unsigned)n_vectors, 512, 0, st>>>(T.as<double>(), n, tau, zrows,
                                                              selbuf.as<int>(), n_vectors, left, right,
                                                              bt_scratch.as<double>(), v_dev); sc::launched();
  }
  SC_LAUNCH_CHECK();
  SC_CUDA(cudaStreamSynchronize(st));   // `sel` must outlive the H2D copy
  return 0;
}
