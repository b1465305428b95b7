/*
 * spectralcluster_b200 -- C ABI of the H100-native SpectralClusterer.predict() hot path.
 *
 * The reference (wq2012/SpectralCluster v0.2.22) is pure Python and has no FFI:
 * its drop-in boundary is the Python object surface (SURVEY.md 8(b)).  This header
 * is the boundary underneath our Python mirror of that surface: one entry point per
 * reference operator, bound with ctypes by spectralcluster_b200/_native.py.  Every
 * declaration cites the reference function (file:line under /root/reference) whose
 * arithmetic it replaces.
 *
 * Conventions
 *   - every function returns 0 on success, non-zero on failure; the message is
 *     available from sc_last_error() (thread local).
 *   - all matrix pointers are DEVICE pointers (cudaMalloc'ed by the caller --
 *     the Python host uses torch tensors purely as device buffers), row-major,
 *     with an explicit leading dimension `ld` counted in elements.  fp32 matrices
 *     need ld % 4 == 0 and 16-byte aligned bases; fp16 planes need ld % 8 == 0.
 *   - `stream` is a cudaStream_t passed as void* (0 = default stream).  Calls are
 *     asynchronous unless stated otherwise.
 *   - "split fp16 planes" (hi, lo): value = hi + lo with hi = fp16(value),
 *     lo = fp16(value - hi): the operand format of the wgmma GEMMs (three
 *     kind::f16 MMAs hi*hi + hi*lo + lo*hi reproduce an fp32-accurate product).
 */
#ifndef SPECTRALCLUSTER_B200_H_
#define SPECTRALCLUSTER_B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SC_ABI_VERSION 2

/* enums mirror the reference's enum *names* (values are ours) */
enum sc_threshold_type { SC_THRESHOLD_ROWMAX = 0, SC_THRESHOLD_PERCENTILE = 1 }; /* refinement.py:21-27 */
enum sc_symmetrize_type { SC_SYMMETRIZE_MAX = 0, SC_SYMMETRIZE_AVERAGE = 1 };    /* refinement.py:30-36 */
enum sc_laplacian_type {                                                          /* laplacian.py:9-21 */
  SC_LAPLACIAN_AFFINITY = 0, SC_LAPLACIAN_UNNORMALIZED = 1,
  SC_LAPLACIAN_RANDOMWALK = 2, SC_LAPLACIAN_GRAPHCUT = 3
};
enum sc_gemm_engine {
  SC_GEMM_TCGEN05 = 0,   /* tensor cores (wgmma f16) on split planes, TMA-fed (product path) */
  SC_GEMM_SIMT_F64ACC = 1 /* SIMT fp32 operands, fp64 accumulation (validation path, small N) */
};
enum sc_gemm_precision {
  SC_GEMM_SPLIT3 = 0,    /* hi*hi + hi*lo + lo*hi : ~2^-22 relative per product */
  SC_GEMM_SINGLE = 1,    /* hi*hi only            : ~2^-11 relative per product */
  SC_GEMM_SPLIT2 = 2     /* (hi+lo)*hi : B rounded to fp16, zero-mean 2^-12 per product */
};
enum sc_which_end { SC_EIG_LARGEST = 0, SC_EIG_SMALLEST = 1 };
/* element type of an input matrix (F32 / F64 agree with the x_is_f64 flags of older entries) */
enum sc_dtype { SC_DTYPE_F32 = 0, SC_DTYPE_F64 = 1, SC_DTYPE_F16 = 2, SC_DTYPE_BF16 = 3 };

typedef struct sc_context sc_context;

int sc_abi_version(void);
const char* sc_last_error(void);
/* Number of CUDA kernels this library has launched in this process (bench.py's gpu_launches). */
long long sc_launch_count(void);

/* One context per (process, device).  Owns nothing the caller can see except
 * cached device properties and stream-ordered scratch. */
int sc_context_create(int device, sc_context** out);
int sc_context_destroy(sc_context* ctx);
int sc_context_sm_count(const sc_context* ctx);
/* Cap the CTA count of the persistent GEMM (0 = every SM) so that communication kernels issued
 * concurrently (NCCL send/recv in the sharded pipeline) find free SMs. */
int sc_context_set_gemm_sm_limit(sc_context* ctx, int sms);

/* ---- utils.compute_affinity_matrix (utils.py:20-41) --------------------------------- */
/* Row L2-normalisation (utils.py:32-33).  x is [n,d] fp32 (x_is_f64=0) or fp64 (=1) on the
 * device.  Norms are accumulated in fp64.  Any of xn (fp32 [n,ldxn]) and hi/lo (fp16
 * [n,ldh]) may be NULL.  Zero rows give NaN like the reference. */
int sc_normalize_rows(sc_context* ctx, const void* x, int x_is_f64, int64_t n, int64_t d,
                      int64_t ldx, float* xn, int64_t ldxn, void* hi, void* lo, int64_t ldh,
                      void* stream);

/* sc_normalize_rows on rows of any sc_dtype (x_dtype), read in place with row stride ldx and unit
 * column stride.  Each element widens exactly to fp64, so fp16 rows give bit for bit the outputs
 * of sc_normalize_rows on their fp64 upcast, and bf16 rows those of their fp32 upcast
 * (SpectralClusterer.predict on a CUDA tensor: no widened N x d staging copy). */
int sc_normalize_rows_typed(sc_context* ctx, const void* x, int x_dtype, int64_t n, int64_t d,
                            int64_t ldx, float* xn, int64_t ldxn, void* hi, void* lo,
                            int64_t ldh, void* stream);

/* A = (Xn Xn^T + 1) / 2 (utils.py:35-39).  engine TCGEN05 reads the split planes,
 * engine SIMT reads xn.  If rowmax_offdiag != NULL it receives max_j!=i A[i,j] clamped at 0
 * (the CropDiagonal value, refinement.py:148-150) -- it must be zero-filled by the caller. */
int sc_affinity_cosine(sc_context* ctx, int engine, int precision, const float* xn, int64_t ldxn,
                       const void* hi, const void* lo, int64_t ldh, int64_t n, int64_t d,
                       float* a, int64_t lda, float* rowmax_offdiag, void* stream);

/* ---- refinement.py operators --------------------------------------------------------- */
/* CropDiagonal.refine (refinement.py:145-151): out = a with diag[i] = max(0, max_{j!=i} a[i,j]).
 * out may alias a. */
int sc_crop_diagonal(sc_context* ctx, const float* a, int64_t n, int64_t lda, float* out,
                     int64_t ldo, void* stream);

/* Only the new diagonal of CropDiagonal (the vector the fused blur pass substitutes on read). */
int sc_crop_diagonal_values(sc_context* ctx, const float* a, int64_t n, int64_t lda,
                            float* diag_out, void* stream);

/* GaussianBlur.refine (refinement.py:160-162) == scipy.ndimage.gaussian_filter(a, sigma):
 * separable, axis 0 then axis 1, mode='reflect', truncate=4.0 (radius int(4*sigma+0.5)),
 * weights computed in fp64.  sigma <= 1e-15 copies.  diag_override (may be NULL) replaces
 * a[i,i] on read (fused CropDiagonal).  out == NULL runs the statistics-only pass.
 * rowmax_out (may be NULL; caller zero-fills; values must be >= 0) receives max_j out[i,j]. */
int sc_gaussian_blur(sc_context* ctx, const float* a, int64_t n, int64_t lda,
                     const float* diag_override, double sigma, float* out, int64_t ldo,
                     float* rowmax_out, void* stream);

/* Statistics-only pass of the blur: rowmax_out[i] = max_j blur(a)[i,j], with the diagonal read
 * as zero when zero_diagonal != 0 (RowWiseThreshold's preserve_diagonal, refinement.py:185-186). */
int sc_gaussian_blur_rowmax(sc_context* ctx, const float* a, int64_t n, int64_t lda,
                            const float* diag_override, double sigma, int zero_diagonal,
                            float* rowmax_out, void* stream);

/* RowWiseThreshold.refine (refinement.py:182-210), any option combination. */
int sc_row_threshold(sc_context* ctx, const float* a, int64_t n, int64_t lda, int type, double p,
                     double mult, int binarize, int preserve_diagonal, float* out, int64_t ldo,
                     void* stream);

/* Symmetrize.refine (refinement.py:219-226).  out must not alias a. */
int sc_symmetrize(sc_context* ctx, const float* a, int64_t n, int64_t lda, int type, float* out,
                  int64_t ldo, void* stream);

/* Fused GaussianBlur -> RowWiseThreshold(RowMax) -> Symmetrize for a SYMMETRIC input
 * (SURVEY.md A.3): y[i,j] = sym(t(b, m_i), t(b, m_j)), b = blur(a)[i,j], t = the threshold rule
 * with row maxima `rowmax` (from the statistics-only pass of sc_gaussian_blur).  sigma <= 1e-15
 * skips the blur.  Writes fp32 `y` and/or split planes (either may be NULL). */
int sc_blur_threshold_symmetrize(sc_context* ctx, const float* a, int64_t n, int64_t lda,
                                 const float* diag_override, double sigma, const float* rowmax,
                                 double p, double mult, int binarize, int preserve_diagonal,
                                 int sym_type, float* y, int64_t ldy, void* hi, void* lo,
                                 int64_t ldh, void* stream);

/* The same chain for a SYMMETRIC whole matrix with the blur evaluated on the tiles that touch the
 * upper triangle only (blur(a) is symmetric): sc_blur_upper_rowmax assembles rowmax[i] =
 * max_j b[i,j], b = blur(a), from the row and column maxima of those tiles (zero-fills rowmax
 * itself).  With b_out it also stores those tiles of b (the rest of b_out is left untouched) and
 * sc_threshold_symmetrize_upper writes the whole y from them (fp32 and/or planes; lo may be NULL
 * when only the hi plane is wanted, i.e. for a single-MMA Diffuse), mirroring every tile.  With
 * b_out == NULL nothing but rowmax is written, and sc_blur_threshold_symmetrize_upper blurs the
 * upper triangle of a again and writes y and its mirror -- bit for bit the same y, with no b in
 * memory: 2 + 2 + 2 B of HBM traffic per matrix element for the hi plane alone.  Radius-4 blur
 * only (int(4*sigma+0.5) == 4). */
int sc_blur_upper_rowmax(sc_context* ctx, const float* a, int64_t n, int64_t lda,
                         const float* diag_override, double sigma, int zero_diagonal, float* b_out,
                         int64_t ldb, float* rowmax_out, void* stream);
int sc_threshold_symmetrize_upper(sc_context* ctx, const float* b, int64_t n, int64_t ldb,
                                  const float* rowmax, double p, double mult, int binarize,
                                  int preserve_diagonal, int sym_type, float* y, int64_t ldy,
                                  void* hi, void* lo, int64_t ldh, void* stream);
int sc_blur_threshold_symmetrize_upper(sc_context* ctx, const float* a, int64_t n, int64_t lda,
                                       const float* diag_override, double sigma,
                                       const float* rowmax, double p, double mult, int binarize,
                                       int preserve_diagonal, int sym_type, float* y, int64_t ldy,
                                       void* hi, void* lo, int64_t ldh, void* stream);

/* fp32 [n,n] -> split fp16 planes (for matrices that did not come out of the fused pass). */
int sc_split_planes(sc_context* ctx, const float* a, int64_t n, int64_t lda, void* hi, void* lo,
                    int64_t ldh, void* stream);

/* Diffuse.refine (refinement.py:232-234): s = y y^T.  rowmax (fp32) / rowsum (fp64), both or
 * neither (tensor-core engine only), receive max_j s[i,j] and sum_j s[i,j] from the GEMM epilogue: the
 * reductions of the following RowWiseNormalize (refinement.py:243) and of the Laplacian degree
 * (laplacian.py:41) without another pass over S.  The fused maximum assumes max_j s[i,j] >= 0,
 * which holds for every y (s[i,i] = |y_i|^2).  s == NULL (tensor-core engine, rowmax given) is the
 * statistics-only form: the same GEMM and epilogue reductions, bit for bit, with no store of S. */
int sc_diffuse(sc_context* ctx, int engine, int precision, const float* y, int64_t ldy,
               const void* hi, const void* lo, int64_t ldh, int64_t n, float* s, int64_t lds,
               float* rowmax, double* rowsum, void* stream);

/* ---- bounded Diffuse (DESIGN.md section 5): the row maxima of S = Y Y^T, Y >= 0 and bitwise
 * symmetric, from only the tiles that can hold one.
 * sc_row_group_bounds: one pass over the fp16 plane y_hi [n, ldy]: norms[i * groups + g] = |y_i^g|
 * over the 256-column groups g < groups = ceil(n / 256) (fp32, rounded up), diag_lb[i] <= |y_i|^2
 * (fp64, rounded down) and rowsum[i] = sum_j y_ij (fp64).
 * sc_gather_rows_f16: dst row r = src row perm[r], `cols` fp16 elements (cols % 8 == 0).
 * sc_diffuse_tile_list: the tiles (128 x 192, those the symmetric sc_diffuse launch enumerates) of
 * the product of the permuted rows Y[perm] whose bound from norms and diag_lb (both indexed by the
 * original row) does not rule out a row maximum, packed m << 16 | n in the launch's rasterised
 * order into tiles (room for ceil(n/128) * ceil(n/192) entries); *count (device) receives their
 * number and *total (device) the number of tiles the full launch computes.  n <= 2^20.
 * sc_diffuse_rowmax_tiles: rowmax[perm[r]] = max over the listed tiles of row r of Y[perm] Y[perm]^T,
 * yp_hi = the gathered Y[perm]; every element is the statistics-only sc_diffuse(SC_GEMM_SINGLE)
 * element bit for bit, so rowmax equals its row maxima.  No host synchronisation. */
int sc_row_group_bounds(sc_context* ctx, const void* y_hi, int64_t n, int64_t ldy, float* norms,
                        int64_t groups, double* diag_lb, double* rowsum, void* stream);
int sc_gather_rows_f16(sc_context* ctx, const void* src, int64_t lds, const int* perm, int64_t rows,
                       int64_t cols, void* dst, int64_t ldd, void* stream);
int sc_diffuse_tile_list(sc_context* ctx, const float* norms, int64_t groups, const double* diag_lb,
                         const int* perm, int64_t n, uint32_t* tiles, int* count, int* total,
                         void* stream);
int sc_diffuse_rowmax_tiles(sc_context* ctx, const void* yp_hi, int64_t ldh, int64_t n,
                            const uint32_t* tiles, const int* count, const int* perm,
                            float* rowmax, void* stream);
/* sc_bound_order: the row order of the bounded Diffuse from the group-norm profiles norms [n, groups]
 * (those of sc_row_group_bounds): spherical k-means with k <= 16 centres (greedy farthest-point
 * seeds from row 0, `passes` assignments) and a stable sort by label; perm (device int32 [n])
 * receives the rows in that order.  Deterministic, and enqueued only (no host synchronisation).
 * Profiles that are all alike give the natural order. */
int sc_bound_order(sc_context* ctx, const float* norms, int64_t n, int64_t groups, int k, int passes,
                   int* perm, void* stream);
/* Hub-first bounded Diffuse (DESIGN.md section 3).
 * sc_bound_order_hubs: the clusters of sc_bound_order, each re-sorted by its diagonal (diag, fp64,
 * compared as fp32 rounded down) descending, ties by row; perm receives the rows in that order and
 * starts (device int32 [k + 1]) the first position of each cluster, starts[k] = n.  The first row
 * of a non-empty cluster is its hub.  Deterministic, enqueued only.  n <= 2^21.
 * sc_diffuse_hub_tiles: phase 1, the tiles of each non-empty cluster's hub row block against the
 * column blocks holding its rows, in the rasterised order and format of sc_diffuse_tile_list.
 * sc_diffuse_tile_list_rows: phase 2, given rowmax = the maxima phase 1 folded (indexed by the
 * original row): the tiles that straddle the diagonal or that the per-row rule keeps, minus the
 * phase-1 tiles; *total receives the number of tiles of the full launch.
 * sc_diffuse_rowmax_tiles_fold: sc_diffuse_rowmax_tiles folding into rowmax as it stands instead
 * of zeroing it first. */
int sc_bound_order_hubs(sc_context* ctx, const float* norms, int64_t n, int64_t groups, int k,
                        int passes, const double* diag, int* perm, int* starts, void* stream);
int sc_diffuse_hub_tiles(sc_context* ctx, const int* starts, int k, int64_t n, uint32_t* tiles,
                         int* count, void* stream);
int sc_diffuse_tile_list_rows(sc_context* ctx, const float* norms, int64_t groups, const int* perm,
                              int64_t n, const float* rowmax, const int* starts, int k,
                              uint32_t* tiles, int* count, int* total, void* stream);
int sc_diffuse_rowmax_tiles_fold(sc_context* ctx, const void* yp_hi, int64_t ldh, int64_t n,
                                 const uint32_t* tiles, const int* count, const int* perm,
                                 float* rowmax, void* stream);

/* Row maxima and row sums (fp64) of an fp32 matrix: the reductions of
 * RowWiseNormalize (refinement.py:243) and of the degree (laplacian.py:41). */
int sc_row_stats(sc_context* ctx, const float* a, int64_t n, int64_t lda, double* rowmax,
                 double* rowsum, void* stream);

/* The reductions behind fallback_clusterer.check_single_cluster (fallback_clusterer.py:127-187):
 * out_host[0] = min a, [1] = sum a, [2] = sum a^2 over all n^2 entries (np.std, :154),
 * [3] = min_i a[i][i+1] (np.diag(affinity, k=1).min(), :148-150).  SYNCHRONOUS. */
int sc_affinity_stats(sc_context* ctx, const float* a, int64_t n, int64_t lda, double* out_host,
                      void* stream);

/* The same reductions over an affinity that is never stored (the factored route), built in row
 * panels.  sc_affinity_stats_rows takes rows [row_begin, row_begin + rows) of the affinity as the
 * fp32 panel [rows, ldp] and writes their per-row partials into the DEVICE fp64 buffer part
 * [4 n + 4] (the row kernel of sc_affinity_stats, plus a[i][i+1] per row).  Once every row has
 * been through it, sc_affinity_stats_finish reduces part in sc_affinity_stats's fixed order, so
 * out_host[0..4) equals what sc_affinity_stats returns on the whole matrix, bit for bit.
 * sc_affinity_stats_finish is SYNCHRONOUS. */
int sc_affinity_stats_rows(sc_context* ctx, const float* panel, int64_t rows, int64_t n,
                           int64_t ldp, int64_t row_begin, double* part, void* stream);
int sc_affinity_stats_finish(sc_context* ctx, double* part, int64_t n, double* out_host,
                             void* stream);

/* RowWiseNormalize.refine (refinement.py:240-245), materialised.  out may alias a. */
int sc_row_normalize(sc_context* ctx, const float* a, int64_t n, int64_t lda, float* out,
                     int64_t ldo, void* stream);

/* ---- laplacian.compute_laplacian (laplacian.py:24-60), materialised in fp32 ----------- */
int sc_laplacian(sc_context* ctx, const float* w, int64_t n, int64_t ldw, int type, double eps,
                 float* out, int64_t ldo, void* stream);

/* ---- row-block variants for the row-sharded multi-GPU pipeline (SURVEY.md 8(e)) ------------- */
/* Rows [row_begin, row_begin+row_count) of the affinity (utils.py:35-39) from the split planes of
 * ALL n normalised embeddings.  rowmax_offdiag_block is indexed by local row. */
int sc_affinity_cosine_block(sc_context* ctx, int precision, const void* hi, const void* lo,
                             int64_t ldh, int64_t n, int64_t d, int64_t row_begin,
                             int64_t row_count, float* a_block, int64_t lda,
                             float* rowmax_offdiag_block, void* stream);
/* ---- row panels of the single-GPU factored route (no N x N fp32 matrix is ever allocated).
 * sc_affinity_cosine_panel: rows [row_begin, row_begin+row_count) of the sc_affinity_cosine
 * matrix (tensor-core engine), equal to them bit for bit -- row_begin % 128 == 0, so the panel's
 * tiles are the whole-matrix tiles, those below the diagonal stored as the transpose of their
 * mirror tile as the symmetric launch stores them.  crop_panel (may be NULL) receives the
 * CropDiagonal values of those rows, indexed from row_begin.
 * sc_blur_upper_rowmax_block: pass 1 of the symmetric blur pair (sc_blur_upper_rowmax) for the
 * output rows [row_begin, row_end) (row_begin % 32 == 0) of a panel `a` holding global rows
 * [in_row_base, in_row_base+in_rows), halo included; b_out holds rows [row_begin, row_end) of the
 * upper tiles of blur(a).  Their row and column maxima are folded into rowmax_accum (global
 * length n), which is NOT reset: zero it once, then run every panel.
 * sc_threshold_symmetrize_upper_block: pass 2 (sc_threshold_symmetrize_upper) for the 64 x 64
 * tile pairs (TI, TJ >= TI) whose rows TI lie in [row_begin, row_end) (row_begin % 64 == 0,
 * row_end % 64 == 0 or row_end == n), from such a b panel; y / hi / lo are the full-size outputs
 * and receive Y(i,j) and its mirror Y(j,i). */
int sc_affinity_cosine_panel(sc_context* ctx, int precision, const void* hi, const void* lo,
                             int64_t ldh, int64_t n, int64_t d, int64_t row_begin,
                             int64_t row_count, float* a_panel, int64_t lda, float* crop_panel,
                             void* stream);
int sc_blur_upper_rowmax_block(sc_context* ctx, const float* a, int64_t n, int64_t lda,
                               int64_t in_row_base, int64_t in_rows, int64_t row_begin,
                               int64_t row_end, const float* diag_override, double sigma,
                               int zero_diagonal, float* b_out, int64_t ldb, float* rowmax_accum,
                               void* stream);
int sc_threshold_symmetrize_upper_block(sc_context* ctx, const float* b, int64_t n, int64_t ldb,
                                        int64_t row_begin, int64_t row_end, const float* rowmax,
                                        double p, double mult, int binarize,
                                        int preserve_diagonal, int sym_type, float* y, int64_t ldy,
                                        void* hi, void* lo, int64_t ldh, void* stream);
/* Blur statistics / blur+threshold+symmetrize for global rows [row_begin, row_end) when `a` holds
 * global rows [in_row_base, in_row_base+in_rows) (owned rows + the blur halo, recomputed locally
 * rather than exchanged).  Output buffers start at global row row_begin; diag_override, rowmax and
 * rowmax_out are indexed by GLOBAL row.  (row_end-row_begin) % 32 == 0 unless row_end == n. */
int sc_gaussian_blur_rowmax_block(sc_context* ctx, const float* a, int64_t n, int64_t lda,
                                  int64_t in_row_base, int64_t in_rows, int64_t row_begin,
                                  int64_t row_end, const float* diag_override, double sigma,
                                  int zero_diagonal, float* rowmax_out, void* stream);
int sc_blur_threshold_symmetrize_block(sc_context* ctx, const float* a, int64_t n, int64_t lda,
                                       int64_t in_row_base, int64_t in_rows, int64_t row_begin,
                                       int64_t row_end, const float* diag_override, double sigma,
                                       const float* rowmax, double p, double mult, int binarize,
                                       int preserve_diagonal, int sym_type, float* y, int64_t ldy,
                                       void* hi, void* lo, int64_t ldh, void* stream);
/* Row maxima / sums of a rectangular [rows, cols] block (local rows of a sharded matrix). */
int sc_row_stats_block(sc_context* ctx, const float* a, int64_t rows, int64_t cols, int64_t lda,
                       double* rowmax, double* rowsum, void* stream);
/* dst[cols, rows] = src[rows, cols]^T (the mirrored S blocks exchanged between ranks). */
int sc_transpose(sc_context* ctx, const float* src, int64_t rows, int64_t cols, int64_t lds,
                 float* dst, int64_t ldd, void* stream);
/* c[m,n] = (a_hi+a_lo)[m,k] (b_hi+b_lo)[n,k]^T : one (row block) x (peer row block) piece of
 * Diffuse (refinement.py:232-234) in the sharded pipeline.  c_mirror (may be NULL) additionally
 * receives the transpose, c_mirror[j*ldm + i] = c[i,j], from the same epilogue: it may point into
 * a PEER GPU's row block of S (sc_ipc_open), which is how the symmetric half of the sharded
 * product reaches its owner over NVLink without a separate exchange step. */
int sc_gemm_nt_planes(sc_context* ctx, int precision, const void* a_hi, const void* a_lo,
                      int64_t lda, int64_t m, const void* b_hi, const void* b_lo, int64_t ldb,
                      int64_t n, int64_t k, float* c, int64_t ldc, float* c_mirror, int64_t ldm,
                      void* stream);

/* Row statistics of the single-MMA product a_hi[m,k] b_hi[n,k]^T without storing it: rowmax[i]
 * (fp32) and rowsum[i] (fp64) for i < m are FOLDED INTO (maximum and sum, not reset; start them at
 * 0 -- the products are non-negative) so that a row block of S = Y Y^T can be streamed over column
 * chunks.  a_hi == b_hi with m == n takes the symmetric launch of sc_diffuse (upper tiles, mirrored
 * column statistics).  fp16 operands: 16-byte aligned bases, lda/ldb % 8 == 0.  The row-sharded
 * factored route's RowWiseNormalize maxima and Laplacian degrees. */
int sc_diffuse_stats_block(sc_context* ctx, const void* a_hi, int64_t lda, int64_t m,
                           const void* b_hi, int64_t ldb, int64_t n, int64_t k, float* rowmax,
                           double* rowsum, void* stream);

/* ---- constraint operators (constraint.py:95-164) ---------------------------------------------- */
/* Element-wise: mode 0 max(a, q) (AffinityIntegration Max, :112-113); 1 (a + q)/2 (Average,
 * :114-115); 2 q > 0 ? 1 - (1 - q)(1 - a) : (1 + q) a (the propagation's final adjustment,
 * :156-163, q = the propagated constraint matrix).  out may alias a. */
int sc_constraint_combine(sc_context* ctx, const float* a, int64_t lda, const float* q, int64_t ldq,
                          int64_t n, int mode, float* out, int64_t ldo, void* stream);
/* out = alpha * diag(row_scale) x diag(col_scale) + beta * I (fp64 scale vectors, NULL = ones): the
 * D^-1/2 A D^-1/2 normalisation (:145-147) and the I - alpha A / 2I - P steps of the Newton-Schulz
 * inverse that replaces np.linalg.inv (:151).  out may alias x. */
int sc_scale_shift(sc_context* ctx, const float* x, int64_t ldx, int64_t n, const double* row_scale,
                   const double* col_scale, double alpha, double beta, float* out, int64_t ldo,
                   void* stream);
/* c[m,n] = a[m,k] b[n,k]^T, fp32 operands, fp64 accumulation (SIMT engine): the products of the
 * propagation (:151-153) for matrices too small for a tensor-core tile. */
int sc_gemm_nt_f32(sc_context* ctx, const float* a, int64_t lda, const float* b, int64_t ldb,
                   int64_t m, int64_t n, int64_t k, float* c, int64_t ldc, void* stream);

/* ---- peer memory (one process per GPU, NVLink/NVSwitch) ------------------------------------ */
/* CUDA IPC: export the allocation that contains dev_ptr (64-byte handle + byte offset of dev_ptr
 * inside it); open it in another process of the same box (peer access is enabled lazily); close
 * every mapping this process opened.  No reference counterpart (SURVEY.md section 1). */
int sc_ipc_export(sc_context* ctx, const void* dev_ptr, void* handle_out, int64_t* offset_out);
int sc_ipc_open(sc_context* ctx, const void* handle, int64_t offset, void** out);
int sc_ipc_close_all(sc_context* ctx);
/* cudaMemcpyAsync(cudaMemcpyDefault) on `stream`: with a peer-mapped source the copy engines pull
 * the bytes over NVLink and no SM is involved. */
int sc_memcpy_async(sc_context* ctx, void* dst, const void* src, int64_t bytes, void* stream);

/* ---- utils.compute_sorted_eigenvectors (utils.py:44-71) ------------------------------ */
/* The matrix decomposed is M = diag(delta) + sign * diag(left) S diag(right) with S symmetric
 * fp32 and left,right > 0 (SURVEY.md A.2); delta/left/right are fp64 device vectors, NULL
 * meaning zeros/ones/ones.  M is similar to the symmetric delta + sign * c S c, c = sqrt(left*
 * right); reference eigenvectors are v = E u / |E u|, E = sqrt(left/right).
 * Eigenvalues are returned sorted (descending for LARGEST, ascending for SMALLEST) in
 * w_host[0..n_values); unit-norm eigenvectors of M for the first n_vectors of them go to
 * v_dev, fp64 row-major [n, n_vectors].  SYNCHRONOUS (returns after the stream drains).
 *
 * sc_eigh_dense: Householder tridiagonalisation in fp64 on the device, then the full spectrum
 * (n_values <= n <= 32768) by Sturm-count bisection (one thread per eigenvalue) with inverse
 * iteration for the requested eigenvectors, or by implicit QL when (nearly) all eigenvectors are
 * wanted at small n.  sc_eigh_extremal: thick-restart block Lanczos on the implicit operator
 * (fp32 S streamed from HBM once per block of vectors, fp64 vectors), n_values <= 32 << n.
 * stats_host[4] = {matrix-vector products, restarts, converged pairs, passes over S}. */
/* sc_eigh_dense with pick != NULL: once the sorted eigenvalues are in w_host the callback decides
 * how many eigenvectors are needed (the eigengap of utils.py:74-130 runs on the host) and hands
 * back the device buffer [n, count] for them; n_vectors / v_dev are then ignored. */
typedef int64_t (*sc_pick_fn)(void* user, const double* w_sorted, int64_t n_values, void** v_dev_out);
int sc_eigh_dense(sc_context* ctx, const float* s, int64_t n, int64_t lds, const double* delta,
                  const double* left, const double* right, double sign, int which,
                  int64_t n_values, int64_t n_vectors, double* w_host, double* v_dev,
                  sc_pick_fn pick, void* user, void* stream);
int sc_eigh_extremal(sc_context* ctx, const float* s, int64_t n, int64_t lds, const double* delta,
                     const double* left, const double* right, double sign, int which,
                     int64_t n_values, int64_t n_vectors, double tol, int64_t max_matvecs,
                     double* w_host, double* v_dev, int64_t* stats_host, void* stream);

/* One window of a windowed extremal solve: sc_eigh_extremal restricted to the complement of the
 * n_locked orthonormal vectors locked[0..n_locked) of the SYMMETRISED space (fp64, vector-major,
 * stride n).  Finds the next n_values (<= 32) extremal eigenvalues of M into w_host and APPENDS
 * their symmetrised-space Ritz vectors at locked[n_locked..n_locked+n_values) (the buffer must
 * hold them), so the caller only advances n_locked.  A residual is converged when it is <= tol *
 * max(largest |Ritz value|, scale): pass the magnitude of M's extremal eigenvalue once known.
 * stats_host[4] as sc_eigh_extremal.  SYNCHRONOUS. */
int sc_eigh_extremal_locked(sc_context* ctx, const float* s, int64_t n, int64_t lds,
                            const double* delta, const double* left, const double* right,
                            double sign, int which, int64_t n_values, double tol,
                            int64_t max_matvecs, double scale, double* locked, int64_t n_locked,
                            double* w_host, int64_t* stats_host, void* stream);

/* Eigenvectors of M from symmetrised-space vectors: v_out[:, j] = E u_c / |E u_c| with
 * c = cols_host[j], u_c = u + c * n, E = sqrt(left / right) (NULL = 1); v_out fp64 row-major
 * [n, k].  SYNCHRONOUS. */
int sc_eigh_mapback(sc_context* ctx, const double* u, int64_t n, const int* cols_host, int64_t k,
                    const double* left, const double* right, double* v_out, void* stream);

/* Block size b (vectors multiplied per pass over S) the extremal solver uses for n_values pairs. */
int sc_eigh_block_size(int64_t n_values);

/* Row-sharded variant: `s_block` holds rows [row_begin, row_begin+rows) of S, and this rank is
 * slab `slab` of a partition into slabs of `slab_len` rows (row_begin == slab * slab_len).  Every
 * block product writes b = sc_eigh_block_size(n_values) partial vectors into this rank's slab of
 * y_slabs, laid out [slab][vector][slab_len] (room for (number of slabs) * b * slab_len doubles),
 * and calls gather(user, b), which must all-gather the slabs across the ranks on `stream` (b * N
 * doubles per pass over S); all other work is replicated, so every rank returns identical results.
 * delta/left/right and the outputs are full length, as in sc_eigh_extremal. */
typedef int (*sc_gather_fn)(void* user, int count);
int sc_eigh_extremal_sharded(sc_context* ctx, const float* s_block, int64_t rows, int64_t row_begin,
                             int64_t n, int64_t lds, const double* delta, const double* left,
                             const double* right, double sign, int which, int64_t n_values,
                             int64_t n_vectors, double tol, int64_t max_matvecs, double* y_slabs,
                             int slab, int64_t slab_len, sc_gather_fn gather, void* user,
                             double* w_host, double* v_dev, int64_t* stats_host, void* stream);

/* One window of a windowed solve on a row-sharded S: sc_eigh_extremal_locked with the row block,
 * slabs and gather callback of sc_eigh_extremal_sharded.  locked[0..n_locked) is full length and
 * replicated on every rank (the deflation runs on the gathered products); the window's Ritz
 * vectors are appended at locked[n_locked..), identically on every rank.  SYNCHRONOUS. */
int sc_eigh_extremal_locked_sharded(sc_context* ctx, const float* s_block, int64_t rows,
                                    int64_t row_begin, int64_t n, int64_t lds, const double* delta,
                                    const double* left, const double* right, double sign,
                                    int which, int64_t n_values, double tol, int64_t max_matvecs,
                                    double scale, double* locked, int64_t n_locked,
                                    double* y_slabs, int slab, int64_t slab_len,
                                    sc_gather_fn gather, void* user, double* w_host,
                                    int64_t* stats_host, void* stream);

/* Row-sharded FACTORED operator: as sc_eigh_extremal_sharded, with S = Y Y^T never formed.
 * `y_rows` holds rows [row_begin, row_begin+rows) of Y's fp16 hi plane (16-byte aligned, ldy % 8
 * == 0).  Every pass is two half-products.  First this rank's share of Z = Y^T T, Y[R,:]^T T[R],
 * is written to y_slabs[0 .. b N) (vector-major, stride N) and gather(user, -b) is called: it must
 * SUM those b N doubles over the ranks in place, leaving bitwise the same result on every rank (an
 * all-reduce).  Then Y[R,:] Z is written to this rank's slab and gather(user, b) all-gathers it as
 * in sc_eigh_extremal_sharded.  Y need not be symmetric. */
int sc_eigh_extremal_factored_sharded(sc_context* ctx, const void* y_rows, int64_t rows,
                                      int64_t row_begin, int64_t n, int64_t ldy,
                                      const double* delta, const double* left, const double* right,
                                      double sign, int which, int64_t n_values, int64_t n_vectors,
                                      double tol, int64_t max_matvecs, double* y_slabs, int slab,
                                      int64_t slab_len, sc_gather_fn gather, void* user,
                                      double* w_host, double* v_dev, int64_t* stats_host,
                                      void* stream);

/* One window of a windowed solve on the row-sharded factored operator: the arguments of
 * sc_eigh_extremal_locked_sharded with `y_rows` / `ldy` in place of `s_block` / `lds`. */
int sc_eigh_extremal_locked_factored_sharded(sc_context* ctx, const void* y_rows, int64_t rows,
                                             int64_t row_begin, int64_t n, int64_t ldy,
                                             const double* delta, const double* left,
                                             const double* right, double sign, int which,
                                             int64_t n_values, double tol, int64_t max_matvecs,
                                             double scale, double* locked, int64_t n_locked,
                                             double* y_slabs, int slab, int64_t slab_len,
                                             sc_gather_fn gather, void* user, double* w_host,
                                             int64_t* stats_host, void* stream);

/* The block product of the extremal solver on its own (the O(N^2) part of what replaces
 * np.linalg.eig at utils.py:59): y[p][0..rows) = s[0..rows, 0..n) t[p][0..n) for p < b <= 16; `s` fp32
 * row-major (16-byte aligned, lds % 4 == 0), `t` / `y` fp64 vector-major with leading dimensions
 * ldt (even, t 16-byte aligned) / ldy.  One pass over `s`; products on the fp64 tensor cores,
 * column splits summed in a fixed order (bit-reproducible).  Used by sc_eigh_extremal[_sharded];
 * exported so that the kernel has its own parity test against a float64 product. */
int sc_block_product(sc_context* ctx, const float* s, int64_t rows, int64_t n, int64_t lds,
                     const double* t, int64_t ldt, int b, double* y, int64_t ldy, void* stream);

/* sc_block_product with an fp16 matrix `s` (16-byte aligned, lds % 8 == 0), converted exactly to
 * fp64 for the products: the block product of the factored operator below. */
int sc_block_product_f16(sc_context* ctx, const void* s, int64_t rows, int64_t n, int64_t lds,
                         const double* t, int64_t ldt, int b, double* y, int64_t ldy, void* stream);

/* sc_eigh_extremal on the factored operator S = Y Y^T, where y_hi is the fp16 hi plane of a
 * bitwise-symmetric Y (n x n, leading dimension ldy % 8 == 0) and S is never formed: each block
 * product is Y (Y T) by two sc_block_product_f16 passes through an [b][n] fp64 intermediate (2 + 2
 * B per element, the bytes of one pass over an fp32 S).  fp16 -> fp64 is exact, so this is the
 * exact product of Y up to the fp64 accumulation; a stored S is its fp32-accumulated rounding.
 * Arguments and results otherwise as sc_eigh_extremal.  SYNCHRONOUS. */
int sc_eigh_extremal_factored(sc_context* ctx, const void* y_hi, int64_t n, int64_t ldy,
                              const double* delta, const double* left, const double* right,
                              double sign, int which, int64_t n_values, int64_t n_vectors,
                              double tol, int64_t max_matvecs, double* w_host, double* v_dev,
                              int64_t* stats_host, void* stream);

/* One window of a windowed solve on the factored operator: sc_eigh_extremal_locked with `y_hi` /
 * `ldy` (as in sc_eigh_extremal_factored) in place of `s` / `lds`.  Finds the next n_values
 * extremal eigenvalues of M on the complement of locked[0..n_locked) and appends their
 * symmetrised-space Ritz vectors at locked[n_locked..).  SYNCHRONOUS. */
int sc_eigh_extremal_locked_factored(sc_context* ctx, const void* y_hi, int64_t n, int64_t ldy,
                                     const double* delta, const double* left, const double* right,
                                     double sign, int which, int64_t n_values, double tol,
                                     int64_t max_matvecs, double scale, double* locked,
                                     int64_t n_locked, double* w_host, int64_t* stats_host,
                                     void* stream);

/* ---- Krylov primitives of the general (non-symmetrisable) eigen path: utils.py:59-61 is
 * np.linalg.eig + .real; sequences such as [RowWiseThreshold] alone leave a genuinely
 * non-symmetric matrix (SURVEY.md 8(f)-1).  The Krylov-Schur recurrence is host logic
 * (spectralcluster_b200/arnoldi.py); everything of length n runs here.  Vectors are fp64, basis
 * vectors contiguous (vector q at v + q*n).
 *   matvec        y[rows] = a[rows, n] x            (fp32 matrix streamed once, fp64 accumulate)
 *   orthogonalize w -= V (V^T w) twice; h_host[count] = coefficients, *nrm2_host = |w|^2  (SYNC)
 *   scale         out = alpha * w
 *   random        w = a reproducible pseudo-random direction
 *   combine       out[p] = sum_q z_host[q*k + p] v[q], p < k <= 64                          (SYNC)
 *   columns       v_out[n, k] row-major <- the k vectors of u, each scaled to unit norm */
int sc_krylov_matvec(sc_context* ctx, const float* a, int64_t rows, int64_t n, int64_t lda,
                     const double* x, double* y, void* stream);
int sc_krylov_orthogonalize(sc_context* ctx, const double* v, int64_t n, int64_t count, double* w,
                            double* h_host, double* nrm2_host, void* stream);
int sc_krylov_scale(sc_context* ctx, const double* w, int64_t n, double alpha, double* out,
                    void* stream);
int sc_krylov_random(sc_context* ctx, double* w, int64_t n, int64_t seed, void* stream);
int sc_krylov_combine(sc_context* ctx, const double* v, int64_t n, int64_t m, const double* z_host,
                      int64_t k, double* out, void* stream);
int sc_krylov_columns(sc_context* ctx, const double* u, int64_t n, int64_t k, double* v_out,
                      void* stream);

/* Rows of e[n,k] (fp64) scaled to unit L2 norm (spectral_clusterer.py:301-305). In place. */
int sc_row_renorm(sc_context* ctx, double* e, int64_t n, int64_t k, void* stream);

/* ---- custom_distance_kmeans.run_kmeans (custom_distance_kmeans.py:13-52, 85-141) ------ */
/* e is fp64 [n,k_dim] on the device.  Seeding = scikit-learn KMeans(init="k-means++",
 * max_iter=1, random_state=0, n_init="auto") restated on the device: `first_center` and the
 * uniform draws u[(k-1)*trials] come from the caller's np.random.RandomState(0) (host RNG
 * logic only).  metric is one of the SC_KMEANS_* codes below: stage 2 uses that scipy cdist metric
 * with scipy's special values (NaN, inf) and np.argmin's rule for the new codes (the first NaN
 * wins, else the first minimum).  seuclidean's V and mahalanobis's VI = inv(cov)^T are recomputed
 * every pass over the n + k stacked rows, as scipy's validators do; mahalanobis refuses
 * n + k <= k_dim with scipy's ValueError wording and fails with "Singular matrix" (numpy's
 * LinAlgError) on an exactly zero pivot.  minkowski with p = 2 is euclidean.  labels_host
 * int64[n].  SYNCHRONOUS.  iters_host (may be NULL) receives the number of assignment passes. */
enum {
  SC_KMEANS_COSINE = 0,
  SC_KMEANS_EUCLIDEAN = 1,
  SC_KMEANS_SQEUCLIDEAN = 2,
  SC_KMEANS_CITYBLOCK = 3,
  SC_KMEANS_CHEBYSHEV = 4,
  SC_KMEANS_CANBERRA = 5,
  SC_KMEANS_BRAYCURTIS = 6,
  SC_KMEANS_CORRELATION = 7,
  SC_KMEANS_JENSENSHANNON = 8,
  SC_KMEANS_SEUCLIDEAN = 9,
  SC_KMEANS_MAHALANOBIS = 10
};
int sc_kmeans(sc_context* ctx, const double* e, int64_t n, int64_t k_dim, int64_t k,
              int64_t first_center, const double* u_host, int64_t trials, int metric,
              int64_t max_iter, double tol, int64_t* labels_host, int64_t* iters_host,
              void* stream);

/* ---- AgglomerativeClustering(metric="cosine", linkage="complete") ------------------------
 * The max_spectral_size pre-clustering (spectral_clusterer.py:211-220) and the pre-clusterer of
 * MultiStageClusterer (multi_stage_clusterer.py:64,84).  scikit-learn runs it as
 * scipy.spatial.distance.pdist(x, "cosine") followed by scipy.cluster.hierarchy.linkage(...,
 * "complete"), i.e. scipy's _hierarchy.nn_chain; these two entries restate those two steps.  The
 * sort of the merges, the relabelling and the tree cut are host logic
 * (spectralcluster_b200/agglomerative.py). */

/* dist[i,j] = 1 - clamp(x_i.x_j / (|x_i| |x_j|), -1, 1) for all i, j < n: scipy's pdist(x, "cosine")
 * as a full symmetric fp64 matrix [n, ldd] (ldd >= n), 0 on the diagonal.  x is [n,d] fp32 (x_is_f64=0) or fp64 (=1), converted to double; norms are
 * sqrt(sum x^2).  Products on the fp64 tensor cores; only the upper tiles are computed and each
 * value is stored at (i,j) and (j,i), so dist is bitwise symmetric.  *nonfinite_flag (a device
 * int) is set to 1 if any entry is not finite (a zero row, for instance) and to 0 otherwise. */
int sc_cosine_distances_f64(sc_context* ctx, const void* x, int x_is_f64, int64_t n, int64_t d,
                            int64_t ldx, double* dist, int64_t ldd, int* nonfinite_flag,
                            void* stream);

/* Complete-linkage NN-chain (scipy/cluster/_hierarchy.pyx nn_chain) over the finite symmetric
 * fp64 matrix dist [n, ldd] (2 <= n < 2^31), all n - 1 merges in one cooperative launch.  The
 * chain starts at the lowest active index; the nearest neighbour of the chain top x is the argmin
 * of dist[x, i] over active i != x, where the previous chain element wins ties and otherwise the
 * lowest index does.  Mutual neighbours x < y merge into y (x is retired) and dist[y,:] =
 * dist[:,y] = max(dist[x,:], dist[y,:]).  Merge k, in chain order (unsorted, unrelabelled), goes to
 * the HOST arrays merge_xy[2k], merge_xy[2k+1] (x < y), merge_dist[k] and merge_size[k] (points
 * in the merged cluster).  dist is overwritten.  SYNCHRONOUS. */
int sc_complete_linkage(sc_context* ctx, double* dist, int64_t n, int64_t ldd, int64_t* merge_xy,
                        double* merge_dist, int64_t* merge_size, void* stream);

/* ---- utils.get_cluster_centroids (reference utils.py:159-177) ---------------------------------
 * The cluster centroids of the max_spectral_size pre-clustering on the device.  x is [n,d] fp32
 * (x_is_f64=0) or fp64 (=1) with row stride ldx and unit column stride; labels are n int64 ids
 * (device).  out [k, ldo] fp64 receives, per id c in [0, k), the sum of the rows labelled c
 * divided by their count: np.add.at into np.zeros fp64 sums, divided by np.bincount, bit for bit
 * (each (cluster, column) is a sequential fp64 sum in increasing row index, after a stable
 * counting sort of the rows by id).  An id with no row gives a NaN row; ids outside [0, k) are
 * skipped.  n < 2^31. */
int sc_cluster_centroids(sc_context* ctx, const void* x, int x_is_f64, int64_t n, int64_t d,
                         int64_t ldx, const int64_t* labels, int64_t k, double* out, int64_t ldo,
                         void* stream);

/* ---- AgglomerativeClustering(metric="cosine", linkage="average", distance_threshold=t) -------
 * The single-cluster check of SingleClusterCondition.FallbackClusterer with
 * FallbackClustererType.Agglomerative (fallback_clusterer.py:179-184) inside predict().  The
 * distances come from sc_cosine_distances_f64; the threshold cut is host logic.
 *
 * Average-linkage NN-chain: the same arguments, chain rules, outputs and contract as
 * sc_complete_linkage, except for the update after a merge of x < y with nx, ny points:
 * dist[y,i] = dist[i,y] = (nx dist[x,i] + ny dist[y,i]) / (nx + ny), each product, the sum and the
 * quotient rounded to nearest in turn (scipy's _average, no fused multiply-add).  SYNCHRONOUS. */
int sc_average_linkage(sc_context* ctx, double* dist, int64_t n, int64_t ldd, int64_t* merge_xy,
                       double* merge_dist, int64_t* merge_size, void* stream);

/* ---- NN-chain of a small matrix in one thread block -----------------------------------------
 * The matrices of MultiStageClusterer's steps (at most U2 = 600 rows by default) are too small for
 * the grid barriers of sc_complete_linkage / sc_average_linkage to pay off.  sc_nn_chain_small runs
 * the same chain in one thread block, with block barriers: for linkage SC_LINKAGE_COMPLETE it
 * returns exactly what sc_complete_linkage returns on the same dist, for SC_LINKAGE_AVERAGE exactly
 * what sc_average_linkage returns (same merges in the same chain order, same distances and sizes,
 * bit for bit), with the same arguments and contract otherwise.  2 <= n <= SC_NN_SMALL_MAX; a chain
 * top without a neighbour below infinity (non-finite dist) is an error.  SYNCHRONOUS. */
enum { SC_LINKAGE_COMPLETE = 0, SC_LINKAGE_AVERAGE = 1 };
enum { SC_NN_SMALL_MAX = 2048 };   /* the measured crossing: DESIGN.md §5 */
int sc_nn_chain_small(sc_context* ctx, double* dist, int64_t n, int64_t ldd, int linkage,
                      int64_t* merge_xy, double* merge_dist, int64_t* merge_size, void* stream);

/* ---- fallback_clusterer.check_single_cluster, AffinityGmmBic (fallback_clusterer.py:158-178) --
 * scikit-learn's GaussianMixture(1) and (2) fitted to affinity[np.triu_indices(n, offset)], as
 * one streaming reduction per step; the KMeans / EM / BIC control flow is host logic
 * (spectralcluster_b200/gmm_bic.py).  A pass reads the band j >= max(0, i + offset), j < n of the
 * fp32 matrix a [n, lda] and nothing else, promotes each sample x to fp64 and sums in fp64 in a
 * fixed order (repeated calls agree bit for bit).  params_host[16] and out_host[8] are HOST
 * arrays; work is a DEVICE fp64 buffer of 8 n + 8 elements, whose first n elements a KPP pass
 * leaves for the LOOKUP that follows it.  "Centred" means x - p[0].  SYNCHRONOUS.
 *   MOMENTS  p: shift s.  out: count, sum (x-s), sum (x-s)^2, min x, max x, #non-finite x.
 *   KPP      p: mean, c0, ca, cb, trials (0 or 2), centres centred.  With d(c) = sklearn's
 *            max(-2 x c + c^2 + x^2, 0) on centred x: out sum d(c0), sum min(d(c0), d(ca)),
 *            sum min(d(c0), d(cb)) (the last two only if trials == 2).
 *   LOOKUP   p: mean, c0, kind, v0, v1.  kind 0: v are flat band indices.  kind 1: v are targets
 *            t and the index is searchsorted(cumsum(d(c0)), t) (count of prefixes below t),
 *            summed row sums first, then within one row; clipped to m - 1.
 *            out: index(v0), index(v1), x at each index.
 *   LLOYD    p: mean, c0, c1, o0, o1, has_old (centred).  label(c) = argmin_k c_k^2 - 2 x c_k
 *            (first minimum).  out: #label 1, sum x over label 0, over label 1 (centred x),
 *            #label(c) != label(o) (0 without has_old).
 *   LABELS   p: mean, c0, c1, s0, s1.  out: #label 1, sum x over label 0, over 1 (x not
 *            centred), sum (x - s0)^2 over label 0, sum (x - s1)^2 over label 1.
 *   EM       p: K (1 or 2), then per component: log w, mu pc, pc, log pc, shift.  With
 *            w_k(x) = -0.5 (log 2 pi + (x pc - mu pc)^2) + log pc + log w and
 *            lse = logsumexp_k w_k, r_k = exp(w_k - lse): out sum lse, then per component
 *            sum r_k, sum r_k x, sum r_k (x - shift_k)^2.
 *   SCORE    p as EM.  out: sum lse. */
enum sc_gmm_mode {
  SC_GMM_MOMENTS = 0, SC_GMM_KPP = 1, SC_GMM_LOOKUP = 2, SC_GMM_LLOYD = 3, SC_GMM_LABELS = 4,
  SC_GMM_EM = 5, SC_GMM_SCORE = 6
};
int sc_gmm_band_pass(sc_context* ctx, const float* a, int64_t n, int64_t lda, int64_t offset,
                     int mode, const double* params_host, double* work, double* out_host,
                     void* stream);

/* The packed band, for an affinity that is never stored (the factored route).  Row i of the band,
 * j0 = max(0, i + offset) < n, keeps columns [c0, n), c0 = j0 & ~3, at band[row_off[i] ...], with
 * row_off[i] % 4 == 0 and row_off[i + 1] = row_off[i] + round_up(n - c0, 4) (0 for rows without
 * band elements); row_off is a DEVICE int64 array [n + 1] (gmm_bic.packed_row_offsets).  Column j
 * has the position mod 4 it has in a dense [n, lda] matrix, so sc_gmm_band_pass_packed reads the
 * same samples in the same order as sc_gmm_band_pass and returns the same out_host, bit for bit;
 * its modes, params, work and out are those of sc_gmm_band_pass.  SYNCHRONOUS.
 * sc_gmm_band_pack copies rows [row_begin, row_begin + rows) of the matrix, given as the fp32 panel
 * [rows, ldp] (ldp >= round_up(n, 4)), into their packed rows, with NaN in the slots [c0, j0) and
 * [n, round_up(n, 4)). */
int sc_gmm_band_pass_packed(sc_context* ctx, const float* band, const int64_t* row_off, int64_t n,
                            int64_t offset, int mode, const double* params_host, double* work,
                            double* out_host, void* stream);
int sc_gmm_band_pack(sc_context* ctx, const float* panel, int64_t ldp, int64_t row_begin,
                     int64_t rows, int64_t n, int64_t offset, const int64_t* row_off, float* band,
                     void* stream);

/* ---- naive_clusterer.NaiveClusterer (naive_clusterer.py:59-101) ------------------------------
 * The online clusterer over x[0..n) in one launch, and the single-cluster check of
 * SingleClusterCondition.FallbackClusterer with FallbackClustererType.Naive
 * (fallback_clusterer.py:179-184).  x is [n,d] fp32 (x_is_f64=0) or fp64 (=1), read as fp64.  For
 * each embedding e in turn: cos_c = (m_c . e) / (|m_c| |e|) over the open clusters; if max cos <
 * threshold (or none is open) cluster C opens with m_C = e, count 1; otherwise the label is the
 * first index of the maximum, and if that cosine > adaptation_threshold, m = (m count + e) /
 * (count + 1), each step rounded in turn (no FMA), and count += 1.  A NaN cosine ranks above every
 * number, as np.max / np.argmax have it: it is the label and neither opens nor merges.
 *
 * means (fp64 [capacity, ldm]) and counts (int64 [capacity]) are DEVICE buffers whose first
 * initial_clusters rows hold the state to continue from (0 = fresh); on return rows [0, C) hold the
 * final state.  stop_at > 0 stops before the next embedding as soon as stop_at clusters are open.
 * labels (DEVICE int64 [n]) receives the labels of the processed prefix; *processed_host and
 * *clusters_host (C) are HOST values.  capacity >= initial_clusters + n always suffices; a call
 * that would open more clusters than capacity fails.  SYNCHRONOUS. */
int sc_naive_cluster(sc_context* ctx, const void* x, int x_is_f64, int64_t n, int64_t d, int64_t ldx,
                     double threshold, double adaptation_threshold, int64_t stop_at, double* means,
                     int64_t ldm, int64_t* counts, int64_t capacity, int64_t initial_clusters,
                     int64_t* labels, int64_t* processed_host, int64_t* clusters_host,
                     void* stream);

#ifdef __cplusplus
}
#endif
#endif /* SPECTRALCLUSTER_B200_H_ */
