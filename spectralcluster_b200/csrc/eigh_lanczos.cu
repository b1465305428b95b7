// Extremal symmetric eigensolver for large N: thick-restart BLOCK Lanczos (band form, symmetric
// block Krylov-Schur) with full re-orthogonalisation, on the implicit operator
//
//      Op x = delta .* x + sign * c .* (S (c .* x)),   c = sqrt(left*right)
//
// (the symmetrised form of the matrix the reference hands to np.linalg.eig at utils.py:59, see
// SURVEY.md A.2 and eigh_dense.cu).  Only `n_values` eigenpairs at one end are wanted
// (utils.compute_number_of_clusters reads w[0..max_clusters], utils.py:100-102), so the
// 4/3 N^3 tridiagonalisation (>= 47 s of HBM traffic at N = 65,536) is replaced by O(100s) of
// matrix-vector products, each ONE streaming pass over the fp32 matrix S:
//
//   k_symm_dmma + k_symm_reduce   Y = S T for a block of b <= 16 vectors: ONE pass over the fp32
//                   matrix per block (4 B/element of HBM traffic for b matrix-vector products) on
//                   the fp64 tensor cores.  A block of b >= (number of wanted pairs) vectors also
//                   makes the solver find every copy of a repeated eigenvalue (a single start
//                   vector with full re-orthogonalisation can only ever see one).
//                   k_symm_dmma_f16 is the same product on an fp16 matrix (the factored operator).
//   k_block_proj / k_block_axpy   block classical Gram-Schmidt (twice) of the b products against
//                   the N x m basis, then Cholesky-QR (twice) inside the block
//   k_proj / k_axpy_basis   the same one vector at a time, for a rank-deficient block
//   k_combine       thick restart V <- V Z
// The m x m projected problem (m <= 128) is solved on the host by Householder tridiagonalisation
// and implicit QL (tred2/tql2).
//
// More pairs than one solve finds (max_clusters=None, or max_clusters >= 32, above the dense
// solver's N) come in windows (sc_eigh_extremal_locked, driven by eigen_windows.py): each window
// solves for the next 16 pairs of Op restricted to the complement of the pairs already found (the
// locked set, orthogonalised out of every block with k_block_proj / k_block_axpy in chunks of
// LOCK_CHUNK vectors: about four reads of N x L x 8 bytes per pass over S) and appends its Ritz
// vectors to that set; sc_eigh_mapback turns the selected ones into eigenvectors of M.
//
// The sc_krylov_* primitives at the end serve the general (non-symmetric) eigen path of arnoldi.py.
#include "common.cuh"

#include <algorithm>
#include <cstdlib>
#include <cstring>
#include <numeric>
#include <type_traits>
#include <vector>

namespace sc {

constexpr int SYMV_ROWS = 8;       // rows per CTA (one warp each)
constexpr int SYMV_CHUNK = 2048;   // multiple of 256   // columns of t staged in shared memory per step

// y = S t for one vector: the matrix-vector product of sc_krylov_matvec (general eigen path)
__global__ void __launch_bounds__(SYMV_ROWS * 32)
k_symv_f32_f64(const float* __restrict__ s, int64_t rows, int64_t n, int64_t lds,
               const double* __restrict__ t, double* __restrict__ y) {
  // y[0..rows) = S[0..rows, 0..n) t   (rows == n on one GPU; a row block when sharded)
  __shared__ double ts[SYMV_CHUNK];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t row = (int64_t)blockIdx.x * SYMV_ROWS + warp;
  const float* r = s + (row < rows ? row : 0) * lds;
  double acc0 = 0.0, acc1 = 0.0;
  for (int64_t c0 = 0; c0 < n; c0 += SYMV_CHUNK) {
    const int64_t len = (n - c0 < SYMV_CHUNK) ? (n - c0) : SYMV_CHUNK;
    __syncthreads();
    for (int64_t j = threadIdx.x; j < SYMV_CHUNK; j += blockDim.x) ts[j] = (j < len) ? t[c0 + j] : 0.0;
    __syncthreads();
    if (row < rows) {
      // lanes walk consecutive columns (coalesced 128 B per warp load, conflict-free shared
      // reads); 8 independent loads in flight per lane
      const float* rc = r + c0;
      for (int64_t j = lane; j < len; j += 256) {
        float q[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) q[u] = (j + 32 * u < len) ? ld_stream1(rc + j + 32 * u) : 0.0f;
#pragma unroll
        for (int u = 0; u < 8; u += 2) {
          acc0 = fma((double)q[u], ts[j + 32 * u], acc0);          // ts is zero past len
          acc1 = fma((double)q[u + 1], ts[j + 32 * (u + 1)], acc1);
        }
      }
    }
  }
  double acc = warp_sum(acc0 + acc1);
  if (row < rows && lane == 0) y[row] = acc;
}

// ---- block product: fp64 tensor cores (mma.sync.m8n8k4.f64, SASS DMMA) fed from a cp.async ring
// (2 stages x 2 CTAs per SM).  A DFMA form needs one 64-bit shared load per 4 FMAs of each lane
// (shared-memory-bound); here the S tile is staged in shared memory (108 KB in flight per SM), a B
// fragment (one T value per lane) serves four row groups, and the FP64 pipe is the only busy unit:
// 16 vectors' worth of DMMA per 4 columns whatever b <= 16 is.
//   CTA = 8 warps x 32 rows (4 row groups of 8) = 256 rows; work item = (row block, column split);
//   stage = 256 rows x 32 columns of S (fp32, row pitch 36 floats: conflict-free A fragments)
//         + b vectors x 32 columns of T (fp64, row pitch 36 doubles: conflict-free B fragments).
//   Column splits keep >= ~6 work items per SM; their partial products are summed in a fixed order
//   by k_symm_reduce (every rank of a sharded run must get bit-identical vectors).
constexpr int SYMM_ROWS = 256, SYMM_COLS = 32, SYMM_SP = 36, SYMM_TP = 36, SYMM_MAXB = 16;
constexpr int SYMM_S_FLOATS = SYMM_ROWS * SYMM_SP;                       // 9,216 floats = 36,864 B
constexpr int SYMM_STAGE_BYTES = SYMM_S_FLOATS * 4 + SYMM_MAXB * SYMM_TP * 8;   // + 4,608 B
constexpr int SYMM_STAGES = 2;     // x 41,472 B: two CTAs (16 warps) per SM
template <typename T> struct SymmElem;
template <> struct SymmElem<float> { static constexpr int SP = SYMM_SP; };

__device__ __forceinline__ double to_f64(float x) { return (double)x; }
__device__ __forceinline__ double to_f64(__half x) { return (double)__half2float(x); }

__device__ __forceinline__ void cp_async16_zfill(void* dst, const void* src, int src_bytes) {
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;"
               ::"r"((uint32_t)__cvta_generic_to_shared(dst)), "l"(src), "r"(src_bytes) : "memory");
}

template <typename T>
__global__ void __launch_bounds__(256, 2)
k_symm_dmma(const T* __restrict__ s, int64_t rows, int64_t n, int64_t lds,
            const double* __restrict__ t /*[b][ldt]*/, int64_t ldt, int b, int row_blocks,
            int64_t cols_per_split, double* __restrict__ partial /*[split][b][rows_pad]*/,
            int64_t rows_pad) {
  extern __shared__ __align__(16) unsigned char symm_smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int rb = blockIdx.x % row_blocks, split = blockIdx.x / row_blocks;
  const int64_t row0 = (int64_t)rb * SYMM_ROWS;
  const int64_t c_begin = (int64_t)split * cols_per_split;
  const int64_t c_end = min(n, c_begin + cols_per_split);
  const int chunks = (int)((c_end - c_begin + SYMM_COLS - 1) / SYMM_COLS);
  constexpr int SP = SymmElem<T>::SP, GR = 16 / (int)sizeof(T);   // elements per 16-byte granule
  auto stage_s = [&](int st) { return reinterpret_cast<T*>(symm_smem + (size_t)st * SYMM_STAGE_BYTES); };
  auto stage_t = [&](int st) {
    return reinterpret_cast<double*>(symm_smem + (size_t)st * SYMM_STAGE_BYTES + SYMM_S_FLOATS * 4);
  };
  // fill: 256 rows x 8 (fp16: 4) 16-byte granules of S, 8 (4) per thread; b rows x 16 granules of T
  auto fill = [&](int ch, int st) {
    const int64_t c0 = c_begin + (int64_t)ch * SYMM_COLS;
    T* ss = stage_s(st);
    constexpr int GPR = SYMM_COLS / GR;                // granules per row
#pragma unroll
    for (int k = 0; k < SYMM_ROWS * GPR / 256; ++k) {
      const int idx = threadIdx.x + k * 256;
      const int r = idx / GPR, q = idx % GPR;
      const int64_t gr = (row0 + r < rows) ? row0 + r : rows - 1;
      const int64_t gc = c0 + GR * q;
      int64_t valid = c_end - gc;
      valid = valid < 0 ? 0 : (valid > GR ? GR : valid);
      cp_async16_zfill(ss + r * SP + GR * q, s + gr * lds + (valid > 0 ? gc : 0),
                       (int)valid * (int)sizeof(T));
    }
    double* ts = stage_t(st);
    for (int idx = threadIdx.x; idx < b * 16; idx += 256) {
      const int p = idx >> 4, q = idx & 15;
      const int64_t gc = c0 + 2 * q;
      int64_t valid = c_end - gc;
      valid = valid < 0 ? 0 : (valid > 2 ? 2 : valid);
      cp_async16_zfill(ts + p * SYMM_TP + 2 * q, t + (int64_t)p * ldt + (valid > 0 ? gc : 0), (int)valid * 8);
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  double acc[4][2][2];
#pragma unroll
  for (int g = 0; g < 4; ++g)
#pragma unroll
    for (int h = 0; h < 2; ++h) acc[g][h][0] = acc[g][h][1] = 0.0;
  const int fr = lane >> 2, fk = lane & 3;
  const bool n1_live = (8 + fr) < b;                    // second n-tile: vectors 8..15
  const bool n0_live = fr < b;
  const bool two_tiles = b > 8;                         // block-uniform
#pragma unroll
  for (int st = 0; st < SYMM_STAGES - 1; ++st) {
    if (st < chunks) fill(st, st);
    else asm volatile("cp.async.commit_group;" ::: "memory");
  }
  for (int ch = 0; ch < chunks; ++ch) {
    asm volatile("cp.async.wait_group %0;" ::"n"(SYMM_STAGES - 2) : "memory");
    __syncthreads();                                    // chunk ch landed; stage (ch-1)%S is free
    if (ch + SYMM_STAGES - 1 < chunks) fill(ch + SYMM_STAGES - 1, (ch + SYMM_STAGES - 1) % SYMM_STAGES);
    else asm volatile("cp.async.commit_group;" ::: "memory");
    const T* ss = stage_s(ch % SYMM_STAGES) + (warp * 32 + fr) * SP + fk;
    const double* ts = stage_t(ch % SYMM_STAGES) + fk;
#pragma unroll
    for (int ks = 0; ks < SYMM_COLS / 4; ++ks) {
      const double b0 = n0_live ? ts[fr * SYMM_TP + 4 * ks] : 0.0;
      const double b1 = n1_live ? ts[(8 + fr) * SYMM_TP + 4 * ks] : 0.0;
#pragma unroll
      for (int g = 0; g < 4; ++g) {
        const double a = to_f64(ss[g * 8 * SP + 4 * ks]);
        asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};"
                     : "+d"(acc[g][0][0]), "+d"(acc[g][0][1]) : "d"(a), "d"(b0));
        if (two_tiles)                                  // b <= 8: the second n-tile would be all zeros
          asm volatile("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0, %1}, {%2}, {%3}, {%0, %1};"
                       : "+d"(acc[g][1][0]), "+d"(acc[g][1][1]) : "d"(a), "d"(b1));
      }
    }
  }
  // C fragment: row = fr of the group, vectors 8 h + 2 fk + {0, 1}
  double* out = partial + (int64_t)split * b * rows_pad;
#pragma unroll
  for (int g = 0; g < 4; ++g) {
    const int64_t row = row0 + warp * 32 + g * 8 + fr;
    if (row >= rows) continue;
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int p = 8 * h + 2 * fk + e;
        if (p < b) out[(int64_t)p * rows_pad + row] = acc[g][h][e];
      }
  }
}

// The same block product on an fp16 matrix (the factored operator Y (Y T) of
// sc_eigh_extremal_factored, its windows and the row sums of the bounded Diffuse), with the same
// work items, column splits and k order, so every output is bit for bit what k_symm_dmma gives on
// the fp32 upcast (fp16 -> fp64 is exact).  Two things differ from the fp32 kernel:
//   stage = 256 rows x 64 columns of fp16 (128 B per row: whole L2 lines; a 64 B half line per row
//           and stage streams at about 1.95 TB/s, a 128 B line at 3.05 TB/s on the H100) at a row
//           pitch of 72 halves (144 B: 16-byte aligned rows, and the eight rows of an A fragment
//           land on distinct bank quads), + b vectors x 64 columns of T at a pitch of 68 doubles;
//   MMA   = mma.sync.m16n8k4.f64: the two m8n8k4 steps of row groups g and g + 1 on the same four
//           columns in one instruction.  Issued as separate m8n8k4 steps, the MMAs alone (stages
//           loaded once and reused, no HBM traffic) take ~4.4 ms per pass over a 65,536^2 fp16
//           matrix at any b, well above the 2.6 ms HBM floor; paired they take 2.3-2.45 ms.
constexpr int SYMH_COLS = 64, SYMH_SP = 72, SYMH_TP = 68;
constexpr int SYMH_S_BYTES = SYMM_ROWS * SYMH_SP * 2;                       // 36,864 B
constexpr int SYMH_STAGE_BYTES = SYMH_S_BYTES + SYMM_MAXB * SYMH_TP * 8;    // + 8,704 B
constexpr int SYMH_STAGES = 2;     // x 45,568 B: two CTAs (16 warps) per SM

__global__ void __launch_bounds__(256, 2)
k_symm_dmma_f16(const __half* __restrict__ s, int64_t rows, int64_t n, int64_t lds,
                const double* __restrict__ t /*[b][ldt]*/, int64_t ldt, int b, int row_blocks,
                int64_t cols_per_split, double* __restrict__ partial /*[split][b][rows_pad]*/,
                int64_t rows_pad) {
  extern __shared__ __align__(16) unsigned char symm_smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int rb = blockIdx.x % row_blocks, split = blockIdx.x / row_blocks;
  const int64_t row0 = (int64_t)rb * SYMM_ROWS;
  const int64_t c_begin = (int64_t)split * cols_per_split;
  const int64_t c_end = min(n, c_begin + cols_per_split);
  const int chunks = (int)((c_end - c_begin + SYMH_COLS - 1) / SYMH_COLS);
  auto stage_s = [&](int st) { return reinterpret_cast<__half*>(symm_smem + (size_t)st * SYMH_STAGE_BYTES); };
  auto stage_t = [&](int st) {
    return reinterpret_cast<double*>(symm_smem + (size_t)st * SYMH_STAGE_BYTES + SYMH_S_BYTES);
  };
  // fill: 256 rows x 8 16-byte granules of S, 8 per thread; b rows x 32 granules of T.  Past c_end
  // both are zero-filled: the extra k steps at the end of a split add exact zeros.
  auto fill = [&](int ch, int st) {
    const int64_t c0 = c_begin + (int64_t)ch * SYMH_COLS;
    __half* ss = stage_s(st);
#pragma unroll
    for (int k = 0; k < SYMM_ROWS * (SYMH_COLS / 8) / 256; ++k) {
      const int idx = threadIdx.x + k * 256;
      const int r = idx / (SYMH_COLS / 8), q = idx % (SYMH_COLS / 8);
      const int64_t gr = (row0 + r < rows) ? row0 + r : rows - 1;
      const int64_t gc = c0 + 8 * q;
      int64_t valid = c_end - gc;
      valid = valid < 0 ? 0 : (valid > 8 ? 8 : valid);
      cp_async16_zfill(ss + r * SYMH_SP + 8 * q, s + gr * lds + (valid > 0 ? gc : 0), (int)valid * 2);
    }
    double* ts = stage_t(st);
    for (int idx = threadIdx.x; idx < b * (SYMH_COLS / 2); idx += 256) {
      const int p = idx / (SYMH_COLS / 2), q = idx % (SYMH_COLS / 2);
      const int64_t gc = c0 + 2 * q;
      int64_t valid = c_end - gc;
      valid = valid < 0 ? 0 : (valid > 2 ? 2 : valid);
      cp_async16_zfill(ts + p * SYMH_TP + 2 * q, t + (int64_t)p * ldt + (valid > 0 ? gc : 0), (int)valid * 8);
    }
    asm volatile("cp.async.commit_group;" ::: "memory");
  };
  double acc[4][2][2];
#pragma unroll
  for (int g = 0; g < 4; ++g)
#pragma unroll
    for (int h = 0; h < 2; ++h) acc[g][h][0] = acc[g][h][1] = 0.0;
  const int fr = lane >> 2, fk = lane & 3;
  const bool n1_live = (8 + fr) < b;                    // second n-tile: vectors 8..15
  const bool n0_live = fr < b;
  const bool two_tiles = b > 8;                         // block-uniform
#pragma unroll
  for (int st = 0; st < SYMH_STAGES - 1; ++st) {
    if (st < chunks) fill(st, st);
    else asm volatile("cp.async.commit_group;" ::: "memory");
  }
  for (int ch = 0; ch < chunks; ++ch) {
    asm volatile("cp.async.wait_group %0;" ::"n"(SYMH_STAGES - 2) : "memory");
    __syncthreads();                                    // chunk ch landed; stage (ch-1)%S is free
    if (ch + SYMH_STAGES - 1 < chunks) fill(ch + SYMH_STAGES - 1, (ch + SYMH_STAGES - 1) % SYMH_STAGES);
    else asm volatile("cp.async.commit_group;" ::: "memory");
    const __half* ss = stage_s(ch % SYMH_STAGES) + (warp * 32 + fr) * SYMH_SP + fk;
    const double* ts = stage_t(ch % SYMH_STAGES) + fk;
#pragma unroll
    for (int ks = 0; ks < SYMH_COLS / 4; ++ks) {
      const double b0 = n0_live ? ts[fr * SYMH_TP + 4 * ks] : 0.0;
      const double b1 = n1_live ? ts[(8 + fr) * SYMH_TP + 4 * ks] : 0.0;
#pragma unroll
      for (int g = 0; g < 4; g += 2) {
        // A fragment of m16n8k4: rows fr (group g) and 8 + fr (group g + 1), column fk
        const double a0 = to_f64(ss[g * 8 * SYMH_SP + 4 * ks]);
        const double a1 = to_f64(ss[(g + 1) * 8 * SYMH_SP + 4 * ks]);
        asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0, %1, %2, %3}, {%4, %5}, {%6}, "
                     "{%0, %1, %2, %3};"
                     : "+d"(acc[g][0][0]), "+d"(acc[g][0][1]), "+d"(acc[g + 1][0][0]), "+d"(acc[g + 1][0][1])
                     : "d"(a0), "d"(a1), "d"(b0));
        if (two_tiles)                                  // b <= 8: the second n-tile would be all zeros
          asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0, %1, %2, %3}, {%4, %5}, {%6}, "
                       "{%0, %1, %2, %3};"
                       : "+d"(acc[g][1][0]), "+d"(acc[g][1][1]), "+d"(acc[g + 1][1][0]), "+d"(acc[g + 1][1][1])
                       : "d"(a0), "d"(a1), "d"(b1));
      }
    }
  }
  // C fragment: row = fr of the group, vectors 8 h + 2 fk + {0, 1} (that of m8n8k4 per group)
  double* out = partial + (int64_t)split * b * rows_pad;
#pragma unroll
  for (int g = 0; g < 4; ++g) {
    const int64_t row = row0 + warp * 32 + g * 8 + fr;
    if (row >= rows) continue;
#pragma unroll
    for (int h = 0; h < 2; ++h)
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int p = 8 * h + 2 * fk + e;
        if (p < b) out[(int64_t)p * rows_pad + row] = acc[g][h][e];
      }
  }
}

// y[p][row] = sum over the column splits, in order
__global__ void k_symm_reduce(const double* __restrict__ partial, int splits, int b, int64_t rows,
                              int64_t rows_pad, double* __restrict__ y, int64_t ldy) {
  const int64_t row = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int p = blockIdx.y;
  if (row >= rows) return;
  double acc = 0.0;
  for (int sp = 0; sp < splits; ++sp) acc += partial[((int64_t)sp * b + p) * rows_pad + row];
  y[(int64_t)p * ldy + row] = acc;
}

// scratch the caller provides for the block product: doubles
static size_t block_product_scratch_doubles(int64_t rows, int64_t n, int b, int sm_count,
                                            int* splits_out, int64_t* cols_per_split_out) {
  const int64_t row_blocks = (rows + SYMM_ROWS - 1) / SYMM_ROWS;
  int64_t splits = (6LL * sm_count + row_blocks - 1) / row_blocks;
  const int64_t max_splits = (n + 2047) / 2048;           // at least 2,048 columns per work item
  if (splits > max_splits) splits = max_splits;
  if (splits < 1) splits = 1;
  int64_t cps = (n + splits - 1) / splits;
  cps = (cps + SYMM_COLS - 1) / SYMM_COLS * SYMM_COLS;
  splits = (n + cps - 1) / cps;
  *splits_out = (int)splits;
  *cols_per_split_out = cps;
  const int64_t rows_pad = (rows + 1) & ~(int64_t)1;
  return (size_t)splits * b * rows_pad;
}

// Y = S T (k_symm_dmma or, for fp16, k_symm_dmma_f16, then k_symm_reduce); `scratch`, `splits` and `cols_per_split` come from
// block_product_scratch_doubles
template <typename T>
static int launch_block_product(int b, const T* s, int64_t rows, int64_t n, int64_t lds,
                                const double* t, int64_t ldt, double* y, int64_t ldy, double* scratch,
                                int splits, int64_t cols_per_split, cudaStream_t st) {
  SC_REQUIRE(b >= 1 && b <= SYMM_MAXB && ldt % 2 == 0 && (reinterpret_cast<uintptr_t>(t) & 15) == 0 &&
             (lds * (int64_t)sizeof(T)) % 16 == 0 && (reinterpret_cast<uintptr_t>(s) & 15) == 0,
             "sc_eigh_extremal: internal (block product alignment)");
  const int row_blocks = (int)((rows + SYMM_ROWS - 1) / SYMM_ROWS);
  const int64_t rows_pad = (rows + 1) & ~(int64_t)1;
  if constexpr (std::is_same<T, __half>::value) {
    const size_t smem = (size_t)SYMH_STAGES * SYMH_STAGE_BYTES;
    SC_CUDA(cudaFuncSetAttribute(k_symm_dmma_f16, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_symm_dmma_f16<<<(unsigned)(row_blocks * splits), 256, smem, st>>>(s, rows, n, lds, t, ldt, b, row_blocks,
                                                                    cols_per_split, scratch, rows_pad);
  } else {
    const size_t smem = (size_t)SYMM_STAGES * SYMM_STAGE_BYTES;
    SC_CUDA(cudaFuncSetAttribute(k_symm_dmma<T>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_symm_dmma<T><<<(unsigned)(row_blocks * splits), 256, smem, st>>>(s, rows, n, lds, t, ldt, b, row_blocks,
                                                                  cols_per_split, scratch, rows_pad);
  }
  sc::launched();
  k_symm_reduce<<<dim3((unsigned)((rows + 255) / 256), (unsigned)b), 256, 0, st>>>(scratch, splits, b, rows,
                                                                                 rows_pad, y, ldy);
  sc::launched();
  return 0;
}

// t_p = c .* x_p for the vectors p = blockIdx.y of a block (contiguous, stride n)
__global__ void k_prescale(const double* __restrict__ x, const double* __restrict__ left,
                           const double* __restrict__ right, int64_t n, double* __restrict__ t,
                           int64_t ldt) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const double c = sqrt((left ? left[i] : 1.0) * (right ? right[i] : 1.0));
  t[(int64_t)blockIdx.y * ldt + i] = c * x[(int64_t)blockIdx.y * n + i];
}

// w_p = flip * (delta .* x_p + sign * c .* y_p).  The products are stored in slabs of `slab_len`
// rows, [slab][vector][slab_len] (one slab per rank when the matrix is row-sharded; a single slab
// of n rows otherwise): element i of vector p sits at (i / slab_len) * nb * slab_len + p * slab_len
// + i % slab_len.
__global__ void k_postscale(const double* __restrict__ x, const double* __restrict__ y,
                            int64_t slab_len, int nb, const double* __restrict__ delta,
                            const double* __restrict__ left, const double* __restrict__ right,
                            double sign, double flip, int64_t n, double* __restrict__ w) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int p = blockIdx.y;
  const int64_t o = (int64_t)p * n + i;
  const int64_t yi = (i / slab_len) * nb * slab_len + (int64_t)p * slab_len + i % slab_len;
  const double c = sqrt((left ? left[i] : 1.0) * (right ? right[i] : 1.0));
  w[o] = flip * ((delta ? delta[i] * x[o] : 0.0) + sign * c * y[yi]);
}

// Transposed block product over local rows: partial[split][p][c] = sum over the rows r of the
// split of y[r, c] t[p][r] (fp16 -> fp64 exactly, fp64 accumulation in row order).  One thread per
// column, so a warp reads 64 contiguous bytes of a row; t is read uniformly (a broadcast).
template <int B>
__global__ void __launch_bounds__(256)
k_colprod_f16(const __half* __restrict__ y, int64_t rows, int64_t n, int64_t ldy,
              const double* __restrict__ t, int64_t ldt, int b, int64_t rows_per_split,
              double* __restrict__ partial) {
  const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n) return;
  const int64_t r0 = (int64_t)blockIdx.y * rows_per_split;
  const int64_t r1 = min(rows, r0 + rows_per_split);
  double acc[B];
#pragma unroll
  for (int p = 0; p < B; ++p) acc[p] = 0.0;
  for (int64_t r = r0; r < r1; ++r) {
    const double v = (double)__half2float(y[r * ldy + c]);
#pragma unroll
    for (int p = 0; p < B; ++p)
      if (p < b) acc[p] = fma(v, t[(int64_t)p * ldt + r], acc[p]);
  }
  double* out = partial + (int64_t)blockIdx.y * b * n;
#pragma unroll
  for (int p = 0; p < B; ++p)
    if (p < b) out[(int64_t)p * n + c] = acc[p];
}

template <int B>
static void launch_colprod(const __half* y, int64_t rows, int64_t n, int64_t ldy, const double* t,
                           int64_t ldt, int b, int splits, int64_t rows_per_split, double* partial,
                           cudaStream_t st) {
  k_colprod_f16<B><<<dim3((unsigned)((n + 255) / 256), (unsigned)splits), 256, 0, st>>>(
      y, rows, n, ldy, t, ldt, b, rows_per_split, partial);
  sc::launched();
}

// z[p][c] = sum over the splits, in order, of partial[split][p][c] (z: stride n)
__global__ void k_colprod_reduce(const double* __restrict__ partial, int splits, int b, int64_t n,
                                 double* __restrict__ z) {
  const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= n) return;
  const int p = blockIdx.y;
  double acc = 0.0;
  for (int sp = 0; sp < splits; ++sp) acc += partial[((int64_t)sp * b + p) * n + c];
  z[(int64_t)p * n + c] = acc;
}

// row splits of the transposed block product: enough CTAs to fill the device
static int colprod_splits(int64_t rows, int64_t n, int sm_count) {
  const int64_t col_blocks = (n + 255) / 256;
  int64_t splits = (8LL * sm_count + col_blocks - 1) / col_blocks;
  const int64_t max_splits = (rows + 255) / 256;           // at least 256 rows per split
  return (int)std::max<int64_t>(1, std::min(splits, max_splits));
}

// t[p][i] = y[i / slab_len][p][i % slab_len]: gathered slabs back to vector-major (stride ldt)
__global__ void k_unslab(const double* __restrict__ y, int64_t slab_len, int nb, int64_t n,
                         double* __restrict__ t, int64_t ldt) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int p = blockIdx.y;
  t[(int64_t)p * ldt + i] = y[(i / slab_len) * nb * slab_len + (int64_t)p * slab_len + i % slab_len];
}

// h[j] = <V_j, w>, one CTA per basis vector (deterministic tree reduction)
__global__ void k_proj(const double* __restrict__ v, int64_t n, const double* __restrict__ w,
                       double* __restrict__ h) {
  __shared__ double red[32];
  const double* vj = v + (int64_t)blockIdx.x * n;
  double s = 0.0;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) s = fma(vj[i], w[i], s);
  s = block_sum(s, red);
  if (threadIdx.x == 0) h[blockIdx.x] = s;
}

// w -= sum_j h[j] V_j
__global__ void k_axpy_basis(const double* __restrict__ v, int64_t n, int nvec,
                             const double* __restrict__ h, double* __restrict__ w) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double acc = w[i];
  for (int j = 0; j < nvec; ++j) acc = fma(-h[j], v[(int64_t)j * n + i], acc);
  w[i] = acc;
}

__global__ void k_norm2(const double* __restrict__ w, int64_t n, double* __restrict__ out) {
  __shared__ double red[32];
  double s = 0.0;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) s = fma(w[i], w[i], s);
  s = block_sum(s, red);
  if (threadIdx.x == 0) out[0] = s;
}

// w (device, length n) <- w orthogonalised against the cnt basis vectors v[0..cnt) by classical
// Gram-Schmidt applied twice; h1 / h2 (device, cnt each) take the coefficients of the two sweeps and
// nrm (device) the squared norm of what is left.  Copies h1, h2 to h1_host, h2_host when those are
// given and the norm to *nrm2_host.  One stream synchronisation.
static int gram_schmidt2(const double* v, int64_t n, int cnt, double* w, double* h1, double* h2,
                         double* nrm, double* h1_host, double* h2_host, double* nrm2_host,
                         cudaStream_t st) {
  const unsigned gn = (unsigned)((n + 255) / 256);
  if (cnt > 0) {
    k_proj<<<(unsigned)cnt, 256, 0, st>>>(v, n, w, h1); sc::launched();
    k_axpy_basis<<<gn, 256, 0, st>>>(v, n, cnt, h1, w); sc::launched();
    k_proj<<<(unsigned)cnt, 256, 0, st>>>(v, n, w, h2); sc::launched();
    k_axpy_basis<<<gn, 256, 0, st>>>(v, n, cnt, h2, w); sc::launched();
  }
  k_norm2<<<1, 1024, 0, st>>>(w, n, nrm); sc::launched();
  SC_LAUNCH_CHECK();
  if (h1_host && cnt > 0) {
    SC_CUDA(cudaMemcpyAsync(h1_host, h1, sizeof(double) * cnt, cudaMemcpyDeviceToHost, st));
    SC_CUDA(cudaMemcpyAsync(h2_host, h2, sizeof(double) * cnt, cudaMemcpyDeviceToHost, st));
  }
  SC_CUDA(cudaMemcpyAsync(nrm2_host, nrm, sizeof(double), cudaMemcpyDeviceToHost, st));
  SC_CUDA(cudaStreamSynchronize(st));
  return 0;
}

__global__ void k_scale_into(const double* __restrict__ w, int64_t n, double alpha,
                             double* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = alpha * w[i];
}

__global__ void k_random_vec(double* __restrict__ w, int64_t n, uint64_t seed) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint64_t z = seed + 0x9E3779B97F4A7C15ull * (uint64_t)(i + 1);   // splitmix64
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  z ^= z >> 31;
  w[i] = (double)(z >> 11) * (1.0 / 9007199254740992.0) - 0.5;
}

// out[p] = sum_q z[q*ldz + p] V_q  for p in [p0, p0+8) : thick restart / Ritz vectors
__global__ void k_combine(const double* __restrict__ v, int64_t n, int m,
                          const double* __restrict__ z, int ldz, int n_out,
                          double* __restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int p0 = blockIdx.y * 8;
  if (i >= n) return;
  double acc[8] = {0, 0, 0, 0, 0, 0, 0, 0};
  for (int q = 0; q < m; ++q) {
    const double x = v[(int64_t)q * n + i];
#pragma unroll
    for (int p = 0; p < 8; ++p)
      if (p0 + p < n_out) acc[p] = fma(z[q * ldz + p0 + p], x, acc[p]);
  }
#pragma unroll
  for (int p = 0; p < 8; ++p)
    if (p0 + p < n_out) out[(int64_t)(p0 + p) * n + i] = acc[p];
}

// ---- block Gram-Schmidt: all b products of a pass are orthogonalised together, so the O(N m b)
// vector work runs as a few grid-wide kernels per pass instead of 6 launches and one host
// synchronisation per vector (at N = 65,536 the per-vector form cost more than the four passes
// over S themselves: one CTA per basis vector streaming 2 x 512 KB).
//
// partial[c][j][p] = sum_{i in chunk c} V_j[i] W_p[i]   (j < cnt, p < B); fixed chunking and a
// fixed-order second stage keep the result bit-reproducible (every rank of a sharded run must
// take the same decisions).
constexpr int BP_CHUNK = 256;      // rows per CTA
constexpr int BP_WARPS = 8;
constexpr int LOCK_CHUNK = 128;    // locked vectors per block projection (16 KB of coefficients)

template <int B>
__global__ void __launch_bounds__(BP_WARPS * 32)
k_block_proj(const double* __restrict__ v, int64_t n, int cnt, const double* __restrict__ w,
             double* __restrict__ partial) {
  __shared__ double ws[B][BP_CHUNK];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int64_t i0 = (int64_t)blockIdx.x * BP_CHUNK;
  for (int idx = threadIdx.x; idx < B * BP_CHUNK; idx += BP_WARPS * 32) {
    const int p = idx / BP_CHUNK, t = idx - p * BP_CHUNK;
    ws[p][t] = (i0 + t < n) ? w[(int64_t)p * n + i0 + t] : 0.0;
  }
  __syncthreads();
  for (int j = warp; j < cnt; j += BP_WARPS) {
    const double* vj = v + (int64_t)j * n + i0;
    double x[BP_CHUNK / 32];
#pragma unroll
    for (int t = 0; t < BP_CHUNK / 32; ++t) x[t] = (i0 + lane + 32 * t < n) ? vj[lane + 32 * t] : 0.0;
    double acc[B];
#pragma unroll
    for (int p = 0; p < B; ++p) {
      double a = 0.0;
#pragma unroll
      for (int t = 0; t < BP_CHUNK / 32; ++t) a = fma(x[t], ws[p][lane + 32 * t], a);
      acc[p] = warp_sum(a);
    }
    if (lane == 0) {
      double* out = partial + ((int64_t)blockIdx.x * cnt + j) * B;
#pragma unroll
      for (int p = 0; p < B; ++p) out[p] = acc[p];
    }
  }
}

// h[j*B + p] = sum_c partial[c][j][p], chunks in order
__global__ void k_block_proj_reduce(const double* __restrict__ partial, int chunks, int total,
                                    double* __restrict__ h) {
  const int idx = blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= total) return;
  double s = 0.0;
  for (int c = 0; c < chunks; ++c) s += partial[(int64_t)c * total + idx];
  h[idx] = s;
}

// W_p -= sum_j h[j*B + p] V_j   (p < B)
template <int B>
__global__ void __launch_bounds__(256)
k_block_axpy(const double* __restrict__ v, int64_t n, int cnt, const double* __restrict__ h,
             double* __restrict__ w) {
  extern __shared__ double hs[];                      // [cnt][B]
  for (int idx = threadIdx.x; idx < cnt * B; idx += blockDim.x) hs[idx] = h[idx];
  __syncthreads();
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double acc[B];
#pragma unroll
  for (int p = 0; p < B; ++p) acc[p] = w[(int64_t)p * n + i];
  for (int j = 0; j < cnt; ++j) {
    const double x = v[(int64_t)j * n + i];
#pragma unroll
    for (int p = 0; p < B; ++p) acc[p] = fma(-hs[j * B + p], x, acc[p]);
  }
#pragma unroll
  for (int p = 0; p < B; ++p) w[(int64_t)p * n + i] = acc[p];
}

// b random vectors at once (vector p = blockIdx.y)
__global__ void k_random_block(double* __restrict__ w, int64_t n, uint64_t seed) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  uint64_t z = seed + 0x9E3779B97F4A7C15ull * (uint64_t)(i + 1) + 0xD1B54A32D192ED03ull * (uint64_t)(blockIdx.y + 1);
  z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
  z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
  z ^= z >> 31;
  w[(int64_t)blockIdx.y * n + i] = (double)(z >> 11) * (1.0 / 9007199254740992.0) - 0.5;
}

template <int B>
static int launch_block_proj(const double* v, int64_t n, int cnt, const double* w, double* partial,
                             double* h, cudaStream_t st) {
  const int chunks = (int)((n + BP_CHUNK - 1) / BP_CHUNK);
  k_block_proj<B><<<chunks, BP_WARPS * 32, 0, st>>>(v, n, cnt, w, partial); sc::launched();
  const int total = cnt * B;
  k_block_proj_reduce<<<(total + 127) / 128, 128, 0, st>>>(partial, chunks, total, h); sc::launched();
  return 0;
}

template <int B>
static int launch_block_axpy(const double* v, int64_t n, int cnt, const double* h, double* w,
                             cudaStream_t st) {
  k_block_axpy<B><<<(unsigned)((n + 255) / 256), 256, sizeof(double) * cnt * B, st>>>(v, n, cnt, h, w);
  sc::launched();
  return 0;
}

#define SC_BLOCK_DISPATCH(b, CALL)                                     \
  switch (b) {                                                         \
    case 4: { constexpr int B_ = 4; CALL; } break;                     \
    case 8: { constexpr int B_ = 8; CALL; } break;                     \
    case 12: { constexpr int B_ = 12; CALL; } break;                   \
    default: { constexpr int B_ = 16; CALL; } break;                   \
  }

// Upper-triangular Cholesky factor of the b x b Gram matrix g (row-major): g = R^T R.  Returns
// false when a pivot falls below 1e-12 of the largest diagonal entry (a block that is rank
// deficient to 1e-6: Cholesky-QR would lose orthogonality, the caller takes the vector-by-vector
// path, which also knows how to continue past an exhausted invariant subspace).
static bool cholesky_upper(const double* g, int b, std::vector<double>& r) {
  r.assign((size_t)b * b, 0.0);
  double dmax = 0.0;
  for (int p = 0; p < b; ++p) dmax = std::max(dmax, g[(size_t)p * b + p]);
  if (!(dmax > 0.0)) return false;
  for (int p = 0; p < b; ++p) {
    for (int q = 0; q <= p; ++q) {
      double acc = g[(size_t)q * b + p];
      for (int k = 0; k < q; ++k) acc -= r[(size_t)k * b + q] * r[(size_t)k * b + p];
      if (q < p) {
        r[(size_t)q * b + p] = acc / r[(size_t)q * b + q];
      } else {
        if (!(acc > 1e-12 * dmax)) return false;
        r[(size_t)p * b + p] = std::sqrt(acc);
      }
    }
  }
  return true;
}

// inverse of an upper-triangular b x b matrix (row-major), into `inv` with leading dimension ld
static void invert_upper(const std::vector<double>& r, int b, double* inv, int ld) {
  for (int i = 0; i < b; ++i)
    for (int j = 0; j < b; ++j) inv[(size_t)i * ld + j] = 0.0;
  for (int j = 0; j < b; ++j) {
    inv[(size_t)j * ld + j] = 1.0 / r[(size_t)j * b + j];
    for (int i = j - 1; i >= 0; --i) {
      double acc = 0.0;
      for (int k = i + 1; k <= j; ++k) acc += r[(size_t)i * b + k] * inv[(size_t)k * ld + j];
      inv[(size_t)i * ld + j] = -acc / r[(size_t)i * b + i];
    }
  }
}

// v_out[i, col] = E_i u_src[i] / |E u_src|  (row-major [n, n_out]), src = cols ? cols[col] : col;
// one CTA per output column
__global__ void k_mapback(const double* __restrict__ u, int64_t n, int n_out,
                          const double* __restrict__ left, const double* __restrict__ right,
                          const int* __restrict__ cols, double* __restrict__ v_out) {
  __shared__ double red[32];
  const int col = blockIdx.x;
  const double* uc = u + (int64_t)(cols ? cols[col] : col) * n;
  double ss = 0.0;
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
    const double e = sqrt((left ? left[i] : 1.0) / (right ? right[i] : 1.0));
    const double x = e * uc[i];
    ss = fma(x, x, ss);
  }
  ss = block_sum(ss, red);
  const double inv = 1.0 / sqrt(ss);
  for (int64_t i = threadIdx.x; i < n; i += blockDim.x) {
    const double e = sqrt((left ? left[i] : 1.0) / (right ? right[i] : 1.0));
    v_out[i * n_out + col] = e * uc[i] * inv;
  }
}

// Host eigensolver of the small projected matrix (m <= 128): Householder tridiagonalisation with
// accumulated reflectors, then implicit-shift QL (the classic tred2/tql2 pair, O(m^3) with a
// small constant -- cyclic Jacobi took tens of milliseconds at m = 96).  `a` is row-major and is
// destroyed; eigenvalues come back ascending in w, eigenvectors in the COLUMNS of z.
static bool small_eigh(std::vector<double>& a, int m, std::vector<double>& w,
                       std::vector<double>& z) {
  std::vector<double> e(m, 0.0);
  w.assign(m, 0.0);
  z = a;
  auto Z = [&](int i, int j) -> double& { return z[(size_t)i * m + j]; };
  // --- tridiagonalise (rows are annihilated from the last one up)
  for (int i = m - 1; i > 0; --i) {
    const int l = i - 1;
    double h = 0.0, scale = 0.0;
    if (l > 0) {
      for (int k = 0; k <= l; ++k) scale += std::fabs(Z(i, k));
      if (scale == 0.0) {
        e[i] = Z(i, l);
      } else {
        for (int k = 0; k <= l; ++k) {
          Z(i, k) /= scale;
          h += Z(i, k) * Z(i, k);
        }
        double f = Z(i, l);
        const double g = (f >= 0.0) ? -std::sqrt(h) : std::sqrt(h);
        e[i] = scale * g;
        h -= f * g;
        Z(i, l) = f - g;
        f = 0.0;
        for (int j = 0; j <= l; ++j) {
          Z(j, i) = Z(i, j) / h;
          double g2 = 0.0;
          for (int k = 0; k <= j; ++k) g2 += Z(j, k) * Z(i, k);
          for (int k = j + 1; k <= l; ++k) g2 += Z(k, j) * Z(i, k);
          e[j] = g2 / h;
          f += e[j] * Z(i, j);
        }
        const double hh = f / (h + h);
        for (int j = 0; j <= l; ++j) {
          const double fj = Z(i, j);
          const double gj = e[j] - hh * fj;
          e[j] = gj;
          for (int k = 0; k <= j; ++k) Z(j, k) -= fj * e[k] + gj * Z(i, k);
        }
      }
    } else {
      e[i] = Z(i, l);
    }
    w[i] = h;
  }
  w[0] = 0.0;
  e[0] = 0.0;
  for (int i = 0; i < m; ++i) {                 // accumulate the transformation
    const int l = i - 1;
    if (w[i] != 0.0) {
      for (int j = 0; j <= l; ++j) {
        double g = 0.0;
        for (int k = 0; k <= l; ++k) g += Z(i, k) * Z(k, j);
        for (int k = 0; k <= l; ++k) Z(k, j) -= g * Z(k, i);
      }
    }
    w[i] = Z(i, i);
    Z(i, i) = 1.0;
    for (int j = 0; j <= l; ++j) Z(j, i) = Z(i, j) = 0.0;
  }
  // --- implicit QL on (w, e)
  for (int i = 1; i < m; ++i) e[i - 1] = e[i];
  e[m - 1] = 0.0;
  for (int l = 0; l < m; ++l) {
    int iter = 0, mm;
    do {
      for (mm = l; mm < m - 1; ++mm) {
        const double dd = std::fabs(w[mm]) + std::fabs(w[mm + 1]);
        if (std::fabs(e[mm]) <= 2.3e-16 * dd) break;
      }
      if (mm != l) {
        if (++iter > 200) return false;
        double g = (w[l + 1] - w[l]) / (2.0 * e[l]);
        double r = std::hypot(g, 1.0);
        g = w[mm] - w[l] + e[l] / (g + (g >= 0.0 ? std::fabs(r) : -std::fabs(r)));
        double sn = 1.0, cs = 1.0, pp = 0.0;
        int i;
        for (i = mm - 1; i >= l; --i) {
          double f = sn * e[i];
          const double bb = cs * e[i];
          r = std::hypot(f, g);
          e[i + 1] = r;
          if (r == 0.0) {
            w[i + 1] -= pp;
            e[mm] = 0.0;
            break;
          }
          sn = f / r;
          cs = g / r;
          g = w[i + 1] - pp;
          r = (w[i] - g) * sn + 2.0 * cs * bb;
          pp = sn * r;
          w[i + 1] = g + pp;
          g = cs * r - bb;
          for (int k = 0; k < m; ++k) {
            f = Z(k, i + 1);
            Z(k, i + 1) = sn * Z(k, i) + cs * f;
            Z(k, i) = cs * Z(k, i) - sn * f;
          }
        }
        if (r == 0.0 && i >= l) continue;
        w[l] -= pp;
        e[l] = g;
        e[mm] = 0.0;
      }
    } while (mm != l);
  }
  return true;
}

}  // namespace sc

using namespace sc;

typedef int (*sc_gather_fn)(void* user, int count);

// Shared implementation.  Unsharded: rows == n, row_begin == 0, y_ext == NULL.  Row-sharded: `s`
// holds the rows [row_begin, row_begin+rows) of S and rank `slab` of `slabs`; every block product
// writes its slab of y_ext -- laid out [slab][vector][slab_len], so that one all-gather of
// contiguous slabs completes it -- and calls gather(user, b); everything else runs replicated on
// full-length vectors, so every rank takes identical decisions.
//
// Band (block) Lanczos with full re-orthogonalisation.  Basis v_0..v_{J-1}; the operator has been
// applied to the first P of them ("processed"), J = P + b.  One step multiplies the block
// v_P..v_{P+b-1} (ONE pass over S), then orthogonalises the b products against the whole basis
// (block classical Gram-Schmidt, twice) and among themselves (Cholesky-QR, twice), giving b new
// basis vectors; a rank-deficient block goes one vector at a time instead.  T = V^T Op V is
// banded (plus the arrow left by a thick restart); Ritz pairs come from T[0:P,0:P], their
// residuals from the coupling rows T[P:P+b, 0:P].
//
// Locked set (windowed solve): `locked` holds n_locked orthonormal vectors of the symmetrised
// space (vector-major, stride n) spanning eigenpairs found by earlier windows.  The start block,
// every random direction and every product block are orthogonalised against it (classical
// Gram-Schmidt, twice), so the solver finds the next n_values extremal pairs of Op restricted to
// the complement; their Ritz vectors are appended at locked[n_locked..).  A residual counts as
// converged when it is <= tol * max(|theta|max, scale): the complement's spectrum can sit far
// below the operator's scale (a rank-deficient matrix leaves a cluster of rounding-level values),
// and relative to the operator's scale is the accuracy its callers need.
// Factored operator (sc_eigh_extremal_factored): `s` is NULL and yh = Y (fp16, symmetric) stands
// for S = Y Y^T; every block product is Y (Y T) through an [b][n] fp64 intermediate, two passes of
// 2 B per element over Y.  Row-sharded factored operator (sc_eigh_extremal_factored_sharded): yh
// holds the local rows of Y; Y^T T is summed over the ranks (gather(user, -b)) and Y (Y^T T) is
// all-gathered (gather(user, b)): two collectives per pass.
static int lanczos_impl(sc_context* ctx, const float* s, const __half* yh, int64_t rows,
                        int64_t row_begin,
                        int64_t n, int64_t lds, const double* delta, const double* left,
                        const double* right, double sign, int which, int64_t n_values,
                        int64_t n_vectors, double tol, int64_t max_matvecs, double* y_ext,
                        int slab, int64_t slab_len, sc_gather_fn gather, void* user,
                        double* locked, int64_t n_locked, double scale,
                        double* w_host, double* v_dev, int64_t* stats_host, void* stream) {
  SC_REQUIRE(ctx && (s != nullptr) != (yh != nullptr) && w_host && n > 0,
             "sc_eigh_extremal: bad arguments");
  SC_REQUIRE(!yh || (rows == n && y_ext == nullptr) || (y_ext && gather),
             "sc_eigh_extremal: internal (factored operator)");
  SC_REQUIRE(n_values >= 1 && n_values <= 32 && n_vectors >= 0 && n_vectors <= n_values,
             "sc_eigh_extremal: need 1 <= n_values <= 32 and n_vectors <= n_values");
  SC_REQUIRE(n_vectors == 0 || v_dev, "sc_eigh_extremal: v_dev missing");
  SC_REQUIRE(s ? ((reinterpret_cast<uintptr_t>(s) & 15) == 0 && lds % 4 == 0)
               : ((reinterpret_cast<uintptr_t>(yh) & 15) == 0 && lds % 8 == 0),
             "sc_eigh_extremal: S needs a 16-byte aligned base and lds %% 4 == 0 (Y: lds %% 8 == 0)");
  SC_REQUIRE(n_locked >= 0 && (n_locked == 0 || locked), "sc_eigh_extremal: bad locked set");
  const int nev = (int)n_values;
  const int b = sc_eigh_block_size(n_values);
  const int m = 6 * b;                               // processed vectors before a thick restart
  const int jmax = m + b;                            // basis capacity
  const int keep_extra = std::max(8, nev / 2);
  SC_REQUIRE(n - n_locked >= 2 * (int64_t)jmax, "sc_eigh_extremal: n=%lld (%lld locked) too small "
             "for the Lanczos basis (%d); use sc_eigh_dense", (long long)n, (long long)n_locked, jmax);
  if (tol <= 0) tol = 1e-9;
  if (max_matvecs <= 0) max_matvecs = 20000;
  cudaStream_t st = as_stream(stream);
  const double flip = (which == SC_EIG_LARGEST) ? 1.0 : -1.0;

  Scratch vb, vb2, work, small;
  SC_CUDA(vb.alloc(sizeof(double) * (size_t)jmax * n, st));
  SC_CUDA(vb2.alloc(sizeof(double) * (size_t)jmax * n, st));
  const int64_t ldtb = (n + 1) & ~(int64_t)1;      // even: 16-byte aligned rows for cp.async
  SC_CUDA(work.alloc(sizeof(double) * (size_t)(ldtb + 2 * n + (yh ? ldtb : 0)) * b, st));
  SC_CUDA(small.alloc(sizeof(double) * (size_t)(2 * jmax + 8 + jmax * 64 + 2 * jmax * 16 + 256), st));
  const int bp_chunks = (int)((n + BP_CHUNK - 1) / BP_CHUNK);
  Scratch part;
  const int proj_rows = n_locked > 0 ? std::max(jmax, LOCK_CHUNK) : jmax;
  SC_CUDA(part.alloc(sizeof(double) * (size_t)bp_chunks * proj_rows * 16, st));
  double* partial = part.as<double>();
  // locked-set coefficients: one chunk of the block form, or the whole set for one vector
  Scratch lock_small;
  if (n_locked > 0)
    SC_CUDA(lock_small.alloc(sizeof(double) * (size_t)(LOCK_CHUNK * 16 + 2 * n_locked), st));
  double* lh_dev = lock_small.as<double>();
  double* V = vb.as<double>();
  double* V2 = vb2.as<double>();
  double* tb = work.as<double>();                  // [b][ldtb] prescaled block
  double* yb = tb + (size_t)b * ldtb;              // [b][n] products (unsharded)
  double* wb = yb + (size_t)b * n;                 // [b][n] Op applied, being orthogonalised
  double* mid = wb + (size_t)b * n;                // [b][ldtb] Y T of the factored operator
  double* h_dev = small.as<double>();              // [jmax]
  double* h2_dev = h_dev + jmax;                   // [jmax]
  double* nrm_dev = h2_dev + jmax;                 // [1] (+pad)
  double* z_dev = nrm_dev + 8;                     // [jmax x 64]
  double* hb1_dev = z_dev + (size_t)jmax * 64;     // [jmax x b] block Gram-Schmidt coefficients
  double* hb2_dev = hb1_dev + (size_t)jmax * 16;   // [jmax x b] second sweep
  double* g_dev = hb2_dev + (size_t)jmax * 16;     // [b x b] Gram matrix of the block
  // where the block product lands and how postscale finds element i of vector p
  double* y_base = y_ext ? y_ext : yb;
  const int64_t y_slab_len = y_ext ? slab_len : n;
  double* y_mine = y_base + (y_ext ? (size_t)slab * b * slab_len : 0);

  const unsigned gn = (unsigned)((n + 255) / 256);
  const int ldt = jmax;
  std::vector<double> T((size_t)ldt * ldt, 0.0), hh(jmax), hh2(jmax);
  auto Tat = [&](int i, int j) -> double& { return T[(size_t)i * ldt + j]; };
  double nrm2 = 0.0;
  uint64_t reseed = 1;

  // W (b vectors at stride n) <- W orthogonalised against the locked set: classical Gram-Schmidt
  // twice, each sweep in chunks of LOCK_CHUNK locked vectors (the block kernels' coefficient
  // tile); the coefficients are dropped, Op restricted to the complement is what is solved
  auto deflate_block = [&](double* w) -> int {
    for (int sweep = 0; sweep < 2; ++sweep)
      for (int64_t j0 = 0; j0 < n_locked; j0 += LOCK_CHUNK) {
        const int cnt = (int)std::min<int64_t>(LOCK_CHUNK, n_locked - j0);
        const double* u = locked + (size_t)j0 * n;
        SC_BLOCK_DISPATCH(b, {
          if (int rc = launch_block_proj<B_>(u, n, cnt, w, partial, lh_dev, st)) return rc;
          if (int rc = launch_block_axpy<B_>(u, n, cnt, lh_dev, w, st)) return rc;
        });
      }
    return 0;
  };

  // V[at] <- a fresh random direction orthogonal to the locked set and to V[0..at)
  auto random_direction = [&](int at) -> int {
    double* w = wb;                                  // scratch: callers are done with wb[0]
    k_random_vec<<<gn, 256, 0, st>>>(w, n, 0x5CB200ull + 7919ull * reseed++); sc::launched();
    if (n_locked > 0)
      if (int rc = gram_schmidt2(locked, n, (int)n_locked, w, lh_dev, lh_dev + n_locked, nrm_dev,
                                 nullptr, nullptr, &nrm2, st))
        return rc;
    if (int rc = gram_schmidt2(V, n, at, w, h_dev, h2_dev, nrm_dev, nullptr, nullptr, &nrm2, st))
      return rc;
    k_scale_into<<<gn, 256, 0, st>>>(w, n, 1.0 / std::sqrt(nrm2), V + (size_t)at * n); sc::launched();
    return 0;
  };

  // ---- block forms (see k_block_proj): Gram matrix of a block, Cholesky-QR twice
  std::vector<double> hb1((size_t)jmax * 16), hb2((size_t)jmax * 16), gram((size_t)16 * 16);
  std::vector<double> zk1((size_t)16 * 64), zk2((size_t)16 * 64), R1, R2, Rtot((size_t)16 * 16);
  auto gram_of = [&](const double* w) -> int {       // gram <- W^T W (host), one synchronisation
    SC_BLOCK_DISPATCH(b, if (int rc = launch_block_proj<B_>(w, n, b, w, partial, g_dev, st)) return rc);
    SC_LAUNCH_CHECK();
    SC_CUDA(cudaMemcpyAsync(gram.data(), g_dev, sizeof(double) * b * b, cudaMemcpyDeviceToHost, st));
    SC_CUDA(cudaStreamSynchronize(st));
    return 0;
  };
  // q_out <- orthonormal basis of span(W) by Cholesky-QR applied twice, W = Q Rtot; `gram` already
  // holds W^T W.  Returns 0, or -1 when the block is (numerically) rank deficient -- W untouched.
  // tmp: b x n scratch, distinct from w and q_out.
  auto cholqr2 = [&](const double* w, double* tmp, double* q_out, int* status) -> int {
    *status = -1;
    if (!cholesky_upper(gram.data(), b, R1)) return 0;
    invert_upper(R1, b, zk1.data(), 64);
    SC_CUDA(cudaMemcpyAsync(z_dev, zk1.data(), sizeof(double) * (size_t)b * 64, cudaMemcpyHostToDevice, st));
    k_combine<<<dim3(gn, (unsigned)((b + 7) / 8)), 256, 0, st>>>(w, n, b, z_dev, 64, b, tmp); sc::launched();
    if (int rc = gram_of(tmp)) return rc;
    if (!cholesky_upper(gram.data(), b, R2)) return 0;
    invert_upper(R2, b, zk2.data(), 64);
    SC_CUDA(cudaMemcpyAsync(z_dev + 16 * 64, zk2.data(), sizeof(double) * (size_t)b * 64,
                            cudaMemcpyHostToDevice, st));
    k_combine<<<dim3(gn, (unsigned)((b + 7) / 8)), 256, 0, st>>>(tmp, n, b, z_dev + 16 * 64, 64, b, q_out); sc::launched();
    SC_LAUNCH_CHECK();
    for (int i = 0; i < b; ++i)
      for (int j = 0; j < b; ++j) {
        double acc = 0.0;
        for (int k = i; k <= j; ++k) acc += R2[(size_t)i * b + k] * R1[(size_t)k * b + j];
        Rtot[(size_t)i * b + j] = (j >= i) ? acc : 0.0;
      }
    *status = 0;
    return 0;
  };

  // start block: b random orthonormal vectors
  {
    k_random_block<<<dim3(gn, b), 256, 0, st>>>(wb, n, 0x5CB200ull + 7919ull * reseed++); sc::launched();
    int status = -1;
    if (int rc = deflate_block(wb)) return rc;
    if (int rc = gram_of(wb)) return rc;
    if (int rc = cholqr2(wb, tb, V, &status)) return rc;
    if (status != 0)
      for (int p = 0; p < b; ++p)
        if (int rc = random_direction(p)) return rc;
  }

  const bool trace = std::getenv("SCB_LANCZOS_TRACE") != nullptr;
  int prod_splits = 1;
  int64_t prod_cols = n;
  Scratch prod_buf;
  SC_CUDA(prod_buf.alloc(sizeof(double) * block_product_scratch_doubles(rows, n, b, ctx->sm_count,
                                                                        &prod_splits, &prod_cols), st));
  // transposed block product of the row-sharded factored operator
  const int colp_splits = (yh && y_ext) ? colprod_splits(rows, n, ctx->sm_count) : 0;
  const int64_t colp_rows = colp_splits ? (rows + colp_splits - 1) / colp_splits : 0;
  Scratch colp_buf;
  if (colp_splits) SC_CUDA(colp_buf.alloc(sizeof(double) * (size_t)colp_splits * b * n, st));
  int P = 0, J = b;
  int64_t matvecs = 0, restarts = 0, passes = 0;
  int converged = 0, mm = 0;
  std::vector<double> theta, Z;

  // Rayleigh-Ritz on T[0:sz,0:sz]; Ritz values sorted descending.  Returns how many of the first
  // nev pairs have residual |T[sz:sz+b, 0:sz] z| <= tol * max|theta|.
  auto ritz = [&](int sz) -> int {
    std::vector<double> A((size_t)sz * sz);
    for (int r = 0; r < sz; ++r)
      for (int c = 0; c < sz; ++c) A[(size_t)r * sz + c] = 0.5 * (Tat(r, c) + Tat(c, r));
    std::vector<double> wv, zv;
    if (!small_eigh(A, sz, wv, zv)) return -1;
    std::vector<int> ord(sz);
    std::iota(ord.begin(), ord.end(), 0);
    std::stable_sort(ord.begin(), ord.end(), [&](int x, int y) { return wv[x] > wv[y]; });
    theta.assign(sz, 0.0);
    Z.assign((size_t)sz * sz, 0.0);
    for (int p = 0; p < sz; ++p) {
      theta[p] = wv[ord[p]];
      for (int q = 0; q < sz; ++q) Z[(size_t)q * sz + p] = zv[(size_t)q * sz + ord[p]];
    }
    mm = sz;
    double tmax = scale;
    for (int p = 0; p < sz; ++p) tmax = std::max(tmax, std::fabs(theta[p]));
    int ok = 0;
    for (int p = 0; p < nev && p < sz; ++p) {
      double r2 = 0.0;
      for (int i = 0; i < b; ++i) {
        double acc = 0.0;
        for (int q = 0; q < sz; ++q) acc += Tat(sz + i, q) * Z[(size_t)q * sz + p];
        r2 += acc * acc;
      }
      if (trace) fprintf(stderr, "%s%.2e", p ? " " : "[sc lanczos] pass residuals/|theta|max: ", std::sqrt(r2) / tmax);
      if (std::sqrt(r2) <= tol * tmax) {
        if (ok == p) ++ok;
      } else if (!trace) {
        break;
      }
    }
    if (trace) fprintf(stderr, "  (basis %d, converged %d of %d)\n", sz, ok, nev);
    return ok;
  };

  for (;;) {
    // ---- one pass over S: W = flip * Op V[P..P+b)
    k_prescale<<<dim3(gn, b), 256, 0, st>>>(V + (size_t)P * n, left, right, n, tb, ldtb); sc::launched();
    if (yh && y_ext) {
      // row-sharded factored operator: this rank's share of Z = Y^T T, Y[R,:]^T T[R], into
      // y_ext[0 .. b n) (vector-major, stride n), summed over the ranks by gather(user, -b) and
      // copied into `mid`; then Y[R,:] Z, row block R of Y Y^T T.  No symmetry of Y is assumed.
      SC_BLOCK_DISPATCH(b, launch_colprod<B_>(yh, rows, n, lds, tb + row_begin, ldtb, b, colp_splits,
                                                colp_rows, colp_buf.as<double>(), st));
      k_colprod_reduce<<<dim3(gn, b), 256, 0, st>>>(colp_buf.as<double>(), colp_splits, b, n, y_ext);
      sc::launched();
      SC_LAUNCH_CHECK();
      SC_REQUIRE(gather(user, -b) == 0, "sc_eigh_extremal_sharded: the gather callback failed");
      k_unslab<<<dim3(gn, b), 256, 0, st>>>(y_ext, n, b, n, mid, ldtb); sc::launched();
      if (int rc = launch_block_product(b, yh, rows, n, lds, mid, ldtb, y_mine, y_slab_len,
                                        prod_buf.as<double>(), prod_splits, prod_cols, st)) return rc;
    } else if (yh) {
      if (int rc = launch_block_product(b, yh, rows, n, lds, tb, ldtb, mid, ldtb,
                                        prod_buf.as<double>(), prod_splits, prod_cols, st)) return rc;
      if (int rc = launch_block_product(b, yh, rows, n, lds, mid, ldtb, y_mine, y_slab_len,
                                        prod_buf.as<double>(), prod_splits, prod_cols, st)) return rc;
    } else if (int rc = launch_block_product(b, s, rows, n, lds, tb, ldtb, y_mine, y_slab_len,
                                             prod_buf.as<double>(), prod_splits, prod_cols, st)) {
      return rc;
    }
    SC_LAUNCH_CHECK();
    if (gather) SC_REQUIRE(gather(user, b) == 0, "sc_eigh_extremal_sharded: the gather callback failed");
    k_postscale<<<dim3(gn, b), 256, 0, st>>>(V + (size_t)P * n, y_base, y_slab_len, b, delta, left,
                                             right, sign, flip, n, wb); sc::launched();
    matvecs += b;
    ++passes;
    if (int rc = deflate_block(wb)) return rc;
    // ---- block classical Gram-Schmidt (twice) of all b products against the basis, then
    // Cholesky-QR (twice) inside the block: T[0:J, P:P+b] = V^T W, T[J:J+b, P:P+b] = R
    SC_BLOCK_DISPATCH(b, {
      if (int rc = launch_block_proj<B_>(V, n, J, wb, partial, hb1_dev, st)) return rc;
      if (int rc = launch_block_axpy<B_>(V, n, J, hb1_dev, wb, st)) return rc;
      if (int rc = launch_block_proj<B_>(V, n, J, wb, partial, hb2_dev, st)) return rc;
      if (int rc = launch_block_axpy<B_>(V, n, J, hb2_dev, wb, st)) return rc;
    });
    SC_CUDA(cudaMemcpyAsync(hb1.data(), hb1_dev, sizeof(double) * (size_t)J * b, cudaMemcpyDeviceToHost, st));
    SC_CUDA(cudaMemcpyAsync(hb2.data(), hb2_dev, sizeof(double) * (size_t)J * b, cudaMemcpyDeviceToHost, st));
    // and against the locked set once more: what is left is small when the Krylov space nears an
    // invariant subspace, and the locked components the first pass left at rounding level would
    // grow by 1/|W| when it is normalised.  At the smallest end the locked directions are the
    // extremal ones of the deflated operator (Op restricted to the complement is 0 on them), so
    // any such growth is found.
    if (int rc = deflate_block(wb)) return rc;
    if (int rc = gram_of(wb)) return rc;
    for (int p = 0; p < b; ++p)
      for (int q = 0; q < J; ++q) {
        const double v = hb1[(size_t)q * b + p] + hb2[(size_t)q * b + p];
        Tat(q, P + p) = v;
        Tat(P + p, q) = v;
      }
    int qr_status = -1;
    if (int rc = cholqr2(wb, tb, V + (size_t)J * n, &qr_status)) return rc;
    if (qr_status == 0) {
      for (int p = 0; p < b; ++p)
        for (int q = 0; q <= p; ++q) {
          Tat(J + q, P + p) = Rtot[(size_t)q * b + p];
          Tat(P + p, J + q) = Rtot[(size_t)q * b + p];
        }
      J += b;
    }
    // ---- rank-deficient block (an invariant subspace is complete, or an eigenvalue is repeated
    // more often than the block is wide): one vector at a time, each yields one new basis vector
    for (int p = 0; p < b && qr_status != 0; ++p) {
      double* w = wb + (size_t)p * n;
      const int col = P + p;
      if (int rc = gram_schmidt2(V, n, J, w, h_dev, h2_dev, nrm_dev, hh.data(), hh2.data(), &nrm2, st))
        return rc;
      if (n_locked > 0)                              // as above, before the division by beta
        if (int rc = gram_schmidt2(locked, n, (int)n_locked, w, lh_dev, lh_dev + n_locked, nrm_dev,
                                   nullptr, nullptr, &nrm2, st))
          return rc;
      for (int q = 0; q < J; ++q) {
        const double v = hh[q] + hh2[q];
        Tat(q, col) += v;
        if (q != col) Tat(col, q) += v;
      }
      double beta = std::sqrt(nrm2);
      double scale = std::fabs(Tat(col, col));
      for (int q = 0; q < J; ++q) scale = std::max(scale, std::fabs(Tat(q, col)));
      if (!(beta > 1e-12 * (scale + 1e-300))) {
        // the product lies in the span of the basis (an invariant subspace is complete, or an
        // eigenvalue is repeated more often than the block is wide): continue with a fresh
        // direction, coupled to nothing
        if (int rc = random_direction(J)) return rc;
        beta = 0.0;
      } else {
        k_scale_into<<<gn, 256, 0, st>>>(w, n, 1.0 / beta, V + (size_t)J * n); sc::launched();
      }
      Tat(J, col) = beta;
      Tat(col, J) = beta;
      ++J;
    }
    P += b;
    converged = ritz(P);
    SC_REQUIRE(converged >= 0, "sc_eigh_extremal: the projected eigenproblem did not converge");
    if (converged >= nev || matvecs >= max_matvecs) break;
    if (P + b > m) {
      // ---- thick restart: keep the leading Ritz vectors and the unprocessed block
      const int keep = std::min(m - b, nev + keep_extra);
      SC_REQUIRE(keep <= 64 && keep < P, "sc_eigh_extremal: internal (restart size)");
      std::vector<double> zk((size_t)P * 64, 0.0);
      for (int q = 0; q < P; ++q)
        for (int p = 0; p < keep; ++p) zk[(size_t)q * 64 + p] = Z[(size_t)q * P + p];
      SC_CUDA(cudaMemcpyAsync(z_dev, zk.data(), sizeof(double) * (size_t)P * 64,
                              cudaMemcpyHostToDevice, st));
      k_combine<<<dim3(gn, (unsigned)((keep + 7) / 8)), 256, 0, st>>>(V, n, P, z_dev, 64, keep, V2); sc::launched();
      SC_CUDA(cudaMemcpyAsync(V2 + (size_t)keep * n, V + (size_t)P * n, sizeof(double) * (size_t)n * b,
                              cudaMemcpyDeviceToDevice, st));
      SC_CUDA(cudaStreamSynchronize(st));      // zk lives on the host stack frame
      std::swap(V, V2);
      // coupling of the unprocessed block to the kept Ritz vectors: C = T[P:P+b, 0:P] Z[:, :keep]
      std::vector<double> C((size_t)b * keep, 0.0);
      for (int i = 0; i < b; ++i)
        for (int p = 0; p < keep; ++p) {
          double acc = 0.0;
          for (int q = 0; q < P; ++q) acc += Tat(P + i, q) * Z[(size_t)q * P + p];
          C[(size_t)i * keep + p] = acc;
        }
      std::fill(T.begin(), T.end(), 0.0);
      for (int p = 0; p < keep; ++p) Tat(p, p) = theta[p];
      for (int i = 0; i < b; ++i)
        for (int p = 0; p < keep; ++p) {
          Tat(keep + i, p) = C[(size_t)i * keep + p];
          Tat(p, keep + i) = C[(size_t)i * keep + p];
        }
      P = keep;
      J = keep + b;
      ++restarts;
    }
  }
  for (int p = 0; p < nev; ++p) w_host[p] = flip * theta[p];
  if (locked) {                                      // Ritz vectors of the window join the set
    std::vector<double> zk((size_t)mm * 64, 0.0);
    for (int q = 0; q < mm; ++q)
      for (int p = 0; p < nev; ++p) zk[(size_t)q * 64 + p] = Z[(size_t)q * mm + p];
    SC_CUDA(cudaMemcpyAsync(z_dev, zk.data(), sizeof(double) * (size_t)mm * 64,
                            cudaMemcpyHostToDevice, st));
    k_combine<<<dim3(gn, (unsigned)((nev + 7) / 8)), 256, 0, st>>>(V, n, mm, z_dev, 64, nev,
                                                                  locked + (size_t)n_locked * n); sc::launched();
    SC_LAUNCH_CHECK();
    SC_CUDA(cudaStreamSynchronize(st));
  }
  if (n_vectors > 0) {
    std::vector<double> zk((size_t)mm * 64, 0.0);
    for (int q = 0; q < mm; ++q)
      for (int p = 0; p < (int)n_vectors; ++p) zk[(size_t)q * 64 + p] = Z[(size_t)q * mm + p];
    SC_CUDA(cudaMemcpyAsync(z_dev, zk.data(), sizeof(double) * (size_t)mm * 64,
                            cudaMemcpyHostToDevice, st));
    k_combine<<<dim3(gn, (unsigned)((n_vectors + 7) / 8)), 256, 0, st>>>(V, n, mm, z_dev, 64,
                                                                        (int)n_vectors, V2); sc::launched();
    k_mapback<<<(unsigned)n_vectors, 512, 0, st>>>(V2, n, (int)n_vectors, left, right, nullptr, v_dev); sc::launched();
    SC_LAUNCH_CHECK();
    SC_CUDA(cudaStreamSynchronize(st));
  }
  if (stats_host) {
    stats_host[0] = matvecs;
    stats_host[1] = restarts;
    stats_host[2] = converged;
    stats_host[3] = passes;
  }
  SC_REQUIRE(converged >= nev, "sc_eigh_extremal: only %d of %d eigenpairs converged to %g in "
             "%lld matrix-vector products", converged, nev, tol, (long long)matvecs);
  return 0;
}

extern "C" int sc_block_product(sc_context* ctx, const float* s, int64_t rows, int64_t n, int64_t lds,
                                const double* t, int64_t ldt, int b, double* y, int64_t ldy,
                                void* stream) {
  SC_REQUIRE(ctx && s && t && y && rows > 0 && n > 0 && b >= 1 && b <= SYMM_MAXB && ldt >= n && ldy >= rows,
             "sc_block_product: bad arguments");
  cudaStream_t st = as_stream(stream);
  int splits = 1;
  int64_t cols = n;
  Scratch buf;
  SC_CUDA(buf.alloc(sizeof(double) * block_product_scratch_doubles(rows, n, b, ctx->sm_count, &splits, &cols), st));
  if (int rc = launch_block_product(b, s, rows, n, lds, t, ldt, y, ldy, buf.as<double>(), splits, cols, st)) return rc;
  SC_LAUNCH_CHECK();
  return 0;
}

extern "C" int sc_eigh_block_size(int64_t n_values) {
  return n_values <= 4 ? 4 : (n_values <= 8 ? 8 : (n_values <= 12 ? 12 : 16));
}

extern "C" int sc_eigh_extremal(sc_context* ctx, const float* s, int64_t n, int64_t lds,
                                const double* delta, const double* left, const double* right,
                                double sign, int which, int64_t n_values, int64_t n_vectors,
                                double tol, int64_t max_matvecs, double* w_host, double* v_dev,
                                int64_t* stats_host, void* stream) {
  return lanczos_impl(ctx, s, nullptr, n, 0, n, lds, delta, left, right, sign, which, n_values,
                      n_vectors, tol, max_matvecs, nullptr, 0, 0, nullptr, nullptr, nullptr, 0, 0.0,
                      w_host, v_dev, stats_host, stream);
}

extern "C" int sc_eigh_extremal_factored(sc_context* ctx, const void* y_hi, int64_t n, int64_t ldy,
                                         const double* delta, const double* left,
                                         const double* right, double sign, int which,
                                         int64_t n_values, int64_t n_vectors, double tol,
                                         int64_t max_matvecs, double* w_host, double* v_dev,
                                         int64_t* stats_host, void* stream) {
  SC_REQUIRE(y_hi, "sc_eigh_extremal_factored: y_hi missing");
  return lanczos_impl(ctx, nullptr, (const __half*)y_hi, n, 0, n, ldy, delta, left, right, sign,
                      which, n_values, n_vectors, tol, max_matvecs, nullptr, 0, 0, nullptr, nullptr,
                      nullptr, 0, 0.0, w_host, v_dev, stats_host, stream);
}

extern "C" int sc_block_product_f16(sc_context* ctx, const void* s, int64_t rows, int64_t n,
                                    int64_t lds, const double* t, int64_t ldt, int b, double* y,
                                    int64_t ldy, void* stream) {
  SC_REQUIRE(ctx && s && t && y && rows > 0 && n > 0 && b >= 1 && b <= SYMM_MAXB && ldt >= n && ldy >= rows,
             "sc_block_product_f16: bad arguments");
  SC_REQUIRE(lds % 8 == 0 && (reinterpret_cast<uintptr_t>(s) & 15) == 0,
             "sc_block_product_f16: `s` needs a 16-byte aligned base and lds %% 8 == 0");
  cudaStream_t st = as_stream(stream);
  int splits = 1;
  int64_t cols = n;
  Scratch buf;
  SC_CUDA(buf.alloc(sizeof(double) * block_product_scratch_doubles(rows, n, b, ctx->sm_count, &splits, &cols), st));
  if (int rc = launch_block_product(b, (const __half*)s, rows, n, lds, t, ldt, y, ldy, buf.as<double>(),
                                    splits, cols, st)) return rc;
  SC_LAUNCH_CHECK();
  return 0;
}

extern "C" int sc_eigh_extremal_locked(sc_context* ctx, const float* s, int64_t n, int64_t lds,
                                       const double* delta, const double* left, const double* right,
                                       double sign, int which, int64_t n_values, double tol,
                                       int64_t max_matvecs, double scale, double* locked,
                                       int64_t n_locked, double* w_host, int64_t* stats_host,
                                       void* stream) {
  SC_REQUIRE(locked, "sc_eigh_extremal_locked: locked buffer missing");
  return lanczos_impl(ctx, s, nullptr, n, 0, n, lds, delta, left, right, sign, which, n_values, 0, tol,
                      max_matvecs, nullptr, 0, 0, nullptr, nullptr, locked, n_locked, scale, w_host,
                      nullptr, stats_host, stream);
}

// One window of the windowed solve on the factored operator S = Y Y^T (S never formed).  The
// scratch of lanczos_impl holds both at once: `mid` (the Y T intermediate) sits after `wb` in
// `work` and is touched only by the block product, while the locked-set deflation uses `partial`
// (sized for LOCK_CHUNK rows) and `lock_small`, neither of which the block product reads.
extern "C" int sc_eigh_extremal_locked_factored(sc_context* ctx, const void* y_hi, int64_t n,
                                                int64_t ldy, const double* delta,
                                                const double* left, const double* right,
                                                double sign, int which, int64_t n_values,
                                                double tol, int64_t max_matvecs, double scale,
                                                double* locked, int64_t n_locked, double* w_host,
                                                int64_t* stats_host, void* stream) {
  SC_REQUIRE(y_hi, "sc_eigh_extremal_locked_factored: y_hi missing");
  SC_REQUIRE(locked, "sc_eigh_extremal_locked_factored: locked buffer missing");
  return lanczos_impl(ctx, nullptr, (const __half*)y_hi, n, 0, n, ldy, delta, left, right, sign,
                      which, n_values, 0, tol, max_matvecs, nullptr, 0, 0, nullptr, nullptr, locked,
                      n_locked, scale, w_host, nullptr, stats_host, stream);
}

extern "C" int sc_eigh_mapback(sc_context* ctx, const double* u, int64_t n, const int* cols_host,
                               int64_t k, const double* left, const double* right, double* v_out,
                               void* stream) {
  SC_REQUIRE(ctx && u && cols_host && v_out && n > 0 && k > 0, "sc_eigh_mapback: bad arguments");
  cudaStream_t st = as_stream(stream);
  Scratch cols;
  SC_CUDA(cols.alloc(sizeof(int) * (size_t)k, st));
  SC_CUDA(cudaMemcpyAsync(cols.as<int>(), cols_host, sizeof(int) * (size_t)k, cudaMemcpyHostToDevice, st));
  k_mapback<<<(unsigned)k, 512, 0, st>>>(u, n, (int)k, left, right, cols.as<int>(), v_out); sc::launched();
  SC_LAUNCH_CHECK();
  SC_CUDA(cudaStreamSynchronize(st));             // cols_host may be released on return
  return 0;
}

extern "C" int sc_eigh_extremal_sharded(sc_context* ctx, const float* s_block, int64_t rows,
                                        int64_t row_begin, int64_t n, int64_t lds,
                                        const double* delta, const double* left,
                                        const double* right, double sign, int which,
                                        int64_t n_values, int64_t n_vectors, double tol,
                                        int64_t max_matvecs, double* y_slabs, int slab,
                                        int64_t slab_len, sc_gather_fn gather, void* user,
                                        double* w_host, double* v_dev, int64_t* stats_host,
                                        void* stream) {
  SC_REQUIRE(s_block && y_slabs && gather && rows > 0 && row_begin >= 0 && row_begin + rows <= n,
             "sc_eigh_extremal_sharded: bad arguments");
  SC_REQUIRE(slab >= 0 && slab_len > 0 && row_begin == (int64_t)slab * slab_len && rows <= slab_len,
             "sc_eigh_extremal_sharded: rank `slab` must own rows [slab*slab_len, +rows)");
  return lanczos_impl(ctx, s_block, nullptr, rows, row_begin, n, lds, delta, left, right, sign, which,
                      n_values, n_vectors, tol, max_matvecs, y_slabs, slab, slab_len, gather, user,
                      nullptr, 0, 0.0, w_host, v_dev, stats_host, stream);
}

// One window of the windowed solve on a row-sharded S.  The locked set is full length and
// replicated on every rank: its deflation runs on the gathered products, like the rest of the
// O(n m b) vector work, so only the block product reads the local rows.
extern "C" int sc_eigh_extremal_locked_sharded(sc_context* ctx, const float* s_block, int64_t rows,
                                               int64_t row_begin, int64_t n, int64_t lds,
                                               const double* delta, const double* left,
                                               const double* right, double sign, int which,
                                               int64_t n_values, double tol, int64_t max_matvecs,
                                               double scale, double* locked, int64_t n_locked,
                                               double* y_slabs, int slab, int64_t slab_len,
                                               sc_gather_fn gather, void* user, double* w_host,
                                               int64_t* stats_host, void* stream) {
  SC_REQUIRE(s_block && y_slabs && gather && locked && rows > 0 && row_begin >= 0 &&
             row_begin + rows <= n, "sc_eigh_extremal_locked_sharded: bad arguments");
  SC_REQUIRE(slab >= 0 && slab_len > 0 && row_begin == (int64_t)slab * slab_len && rows <= slab_len,
             "sc_eigh_extremal_locked_sharded: rank `slab` must own rows [slab*slab_len, +rows)");
  return lanczos_impl(ctx, s_block, nullptr, rows, row_begin, n, lds, delta, left, right, sign, which,
                      n_values, 0, tol, max_matvecs, y_slabs, slab, slab_len, gather, user, locked,
                      n_locked, scale, w_host, nullptr, stats_host, stream);
}

// Row-sharded factored operator: `y_rows` holds rows [row_begin, row_begin+rows) of Y (fp16 hi
// plane) and S = Y Y^T is never formed.  Every pass over the operator is two half-products:
// Y[R,:]^T T[R], summed over the ranks by gather(user, -b), and Y[R,:] Z, all-gathered by
// gather(user, b).
extern "C" int sc_eigh_extremal_factored_sharded(sc_context* ctx, const void* y_rows, int64_t rows,
                                                 int64_t row_begin, int64_t n, int64_t ldy,
                                                 const double* delta, const double* left,
                                                 const double* right, double sign, int which,
                                                 int64_t n_values, int64_t n_vectors, double tol,
                                                 int64_t max_matvecs, double* y_slabs, int slab,
                                                 int64_t slab_len, sc_gather_fn gather, void* user,
                                                 double* w_host, double* v_dev, int64_t* stats_host,
                                                 void* stream) {
  SC_REQUIRE(y_rows && y_slabs && gather && rows > 0 && row_begin >= 0 && row_begin + rows <= n,
             "sc_eigh_extremal_factored_sharded: bad arguments");
  SC_REQUIRE(slab >= 0 && slab_len > 0 && row_begin == (int64_t)slab * slab_len && rows <= slab_len,
             "sc_eigh_extremal_factored_sharded: rank `slab` must own rows [slab*slab_len, +rows)");
  return lanczos_impl(ctx, nullptr, (const __half*)y_rows, rows, row_begin, n, ldy, delta, left,
                      right, sign, which, n_values, n_vectors, tol, max_matvecs, y_slabs, slab,
                      slab_len, gather, user, nullptr, 0, 0.0, w_host, v_dev, stats_host, stream);
}

// One window of the windowed solve on the row-sharded factored operator (locked set replicated).
extern "C" int sc_eigh_extremal_locked_factored_sharded(
    sc_context* ctx, const void* y_rows, int64_t rows, int64_t row_begin, int64_t n, int64_t ldy,
    const double* delta, const double* left, const double* right, double sign, int which,
    int64_t n_values, double tol, int64_t max_matvecs, double scale, double* locked,
    int64_t n_locked, double* y_slabs, int slab, int64_t slab_len, sc_gather_fn gather, void* user,
    double* w_host, int64_t* stats_host, void* stream) {
  SC_REQUIRE(y_rows && y_slabs && gather && locked && rows > 0 && row_begin >= 0 &&
             row_begin + rows <= n, "sc_eigh_extremal_locked_factored_sharded: bad arguments");
  SC_REQUIRE(slab >= 0 && slab_len > 0 && row_begin == (int64_t)slab * slab_len && rows <= slab_len,
             "sc_eigh_extremal_locked_factored_sharded: rank `slab` must own rows "
             "[slab*slab_len, +rows)");
  return lanczos_impl(ctx, nullptr, (const __half*)y_rows, rows, row_begin, n, ldy, delta, left,
                      right, sign, which, n_values, 0, tol, max_matvecs, y_slabs, slab, slab_len,
                      gather, user, locked, n_locked, scale, w_host, nullptr, stats_host, stream);
}

// ---------------------------------------------------------------------------------------------
// Krylov primitives for the GENERAL (non-symmetrisable) eigen path (SURVEY.md 8(f)-1;
// utils.py:59-61 is np.linalg.eig + .real).  The N-length work -- products with the fp32 matrix,
// Gram-Schmidt against the basis, Ritz-vector assembly -- runs here; the Krylov-Schur recurrence
// itself (a small m x m real Schur form per restart) is host logic in
// spectralcluster_b200/arnoldi.py.
extern "C" int sc_krylov_matvec(sc_context* ctx, const float* a, int64_t rows, int64_t n, int64_t lda,
                                const double* x, double* y, void* stream) {
  SC_REQUIRE(ctx && a && x && y && rows > 0 && n > 0, "sc_krylov_matvec: bad arguments");
  k_symv_f32_f64<<<(unsigned)((rows + SYMV_ROWS - 1) / SYMV_ROWS), SYMV_ROWS * 32, 0, as_stream(stream)>>>(
      a, rows, n, lda, x, y); sc::launched();
  SC_LAUNCH_CHECK();
  return 0;
}

// w <- w - V (V^T w), twice (classical Gram-Schmidt with re-orthogonalisation) against the `count`
// basis vectors V[0..count) (each of length n, contiguous); h_host[count] receives the summed
// coefficients, nrm2_host the squared norm of what is left.  SYNCHRONOUS.
extern "C" int sc_krylov_orthogonalize(sc_context* ctx, const double* v, int64_t n, int64_t count,
                                       double* w, double* h_host, double* nrm2_host, void* stream) {
  SC_REQUIRE(ctx && w && nrm2_host && n > 0 && count >= 0 && (count == 0 || (v && h_host)),
             "sc_krylov_orthogonalize: bad arguments");
  cudaStream_t st = as_stream(stream);
  Scratch small;
  SC_CUDA(small.alloc(sizeof(double) * (size_t)(2 * count + 8), st));
  double* h1 = small.as<double>();
  double* h2 = h1 + count;
  double* nrm = h2 + count;
  std::vector<double> a((size_t)count), b((size_t)count);
  if (int rc = gram_schmidt2(v, n, (int)count, w, h1, h2, nrm, a.data(), b.data(), nrm2_host, st))
    return rc;
  for (int64_t q = 0; q < count; ++q) h_host[q] = a[q] + b[q];
  return 0;
}

extern "C" int sc_krylov_scale(sc_context* ctx, const double* w, int64_t n, double alpha, double* out,
                               void* stream) {
  SC_REQUIRE(ctx && w && out && n > 0, "sc_krylov_scale: bad arguments");
  k_scale_into<<<(unsigned)((n + 255) / 256), 256, 0, as_stream(stream)>>>(w, n, alpha, out); sc::launched();
  SC_LAUNCH_CHECK();
  return 0;
}

extern "C" int sc_krylov_random(sc_context* ctx, double* w, int64_t n, int64_t seed, void* stream) {
  SC_REQUIRE(ctx && w && n > 0, "sc_krylov_random: bad arguments");
  k_random_vec<<<(unsigned)((n + 255) / 256), 256, 0, as_stream(stream)>>>(w, n, 0x5CB200ull + 7919ull * (uint64_t)seed);
  sc::launched();
  SC_LAUNCH_CHECK();
  return 0;
}

// out[p] = sum_q z_host[q*k + p] V_q for p < k <= 64 (Ritz vectors / restart basis).  out holds k
// vectors of length n and must not alias v.  SYNCHRONOUS.
extern "C" int sc_krylov_combine(sc_context* ctx, const double* v, int64_t n, int64_t m,
                                 const double* z_host, int64_t k, double* out, void* stream) {
  SC_REQUIRE(ctx && v && z_host && out && n > 0 && m > 0 && k > 0 && k <= 64 && out != v,
             "sc_krylov_combine: bad arguments");
  cudaStream_t st = as_stream(stream);
  Scratch zs;
  SC_CUDA(zs.alloc(sizeof(double) * (size_t)m * 64, st));
  std::vector<double> zk((size_t)m * 64, 0.0);
  for (int64_t q = 0; q < m; ++q)
    for (int64_t p = 0; p < k; ++p) zk[(size_t)q * 64 + p] = z_host[(size_t)q * k + p];
  SC_CUDA(cudaMemcpyAsync(zs.as<double>(), zk.data(), sizeof(double) * (size_t)m * 64,
                          cudaMemcpyHostToDevice, st));
  k_combine<<<dim3((unsigned)((n + 255) / 256), (unsigned)((k + 7) / 8)), 256, 0, st>>>(
      v, n, (int)m, zs.as<double>(), 64, (int)k, out); sc::launched();
  SC_LAUNCH_CHECK();
  SC_CUDA(cudaStreamSynchronize(st));
  return 0;
}

// v_out[i, col] = u_col[i] / |u_col|: `k` vectors of length n (contiguous) -> unit-norm columns of
// a row-major [n, k] array (the layout k-means reads).
extern "C" int sc_krylov_columns(sc_context* ctx, const double* u, int64_t n, int64_t k, double* v_out,
                                 void* stream) {
  SC_REQUIRE(ctx && u && v_out && n > 0 && k > 0, "sc_krylov_columns: bad arguments");
  k_mapback<<<(unsigned)k, 512, 0, as_stream(stream)>>>(u, n, (int)k, nullptr, nullptr, nullptr, v_out); sc::launched();
  SC_LAUNCH_CHECK();
  return 0;
}
