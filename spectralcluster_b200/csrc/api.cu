// Context, error reporting and the GEMM-backed entry points of the C ABI.
#include "common.cuh"

#include <algorithm>
#include <atomic>
#include <cstdlib>
#include <cstring>
#include <string>

namespace sc {

static thread_local char g_error[1024] = "";

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_error, sizeof(g_error), fmt, ap);
  va_end(ap);
}

static std::atomic<long long> g_launches{0};
void launched(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

// gemm_simt.cu
int gemm_nt_simt(int epi, const float* A, int64_t lda, const float* B, int64_t ldb, int64_t M,
                 int64_t N, int64_t K, float* C, int64_t ldc, float* rowmax_offdiag,
                 cudaStream_t st);
// gemm_wgmma.cu
int gemm_nt_wgmma(const sc_context* ctx, int epi, int precision, const __half* a_hi,
                  const __half* a_lo, int64_t lda, const __half* b_hi, const __half* b_lo,
                  int64_t ldb, int64_t M, int64_t N, int64_t K, float* C, int64_t ldc,
                  float* rowmax_offdiag, bool symmetric, int diag_shift, float* stat_rowmax,
                  double* stat_rowsum, float* mirror, int64_t ldm, cudaStream_t st);
int diffuse_tile_list(const float* norms, int G, const double* diag_lb, const int* perm,
                      int64_t n, uint32_t* list, int* count, int* total, cudaStream_t st);
int diffuse_rowmax_tiles(const sc_context* ctx, const __half* y_hi, int64_t ldh, int64_t n,
                         const uint32_t* list, const int* count, const int* row_map,
                         float* rowmax, bool fold, cudaStream_t st);
int diffuse_hub_tiles(const int* starts, int k, int64_t n, uint32_t* list, int* count,
                      cudaStream_t st);
int diffuse_tile_list_rows(const float* norms, int G, const int* perm, int64_t n,
                           const float* rowmax, const int* starts, int k, uint32_t* list,
                           int* count, int* total, cudaStream_t st);
// rowops.cu
int crop_diagonal_rows(const float* a, int64_t n, int64_t lda, int64_t row_begin, int64_t rows,
                       float* diag_out, cudaStream_t st);

}  // namespace sc

using namespace sc;

extern "C" int sc_abi_version(void) { return SC_ABI_VERSION; }

extern "C" const char* sc_last_error(void) { return g_error; }

extern "C" long long sc_launch_count(void) { return g_launches.load(std::memory_order_relaxed); }

extern "C" int sc_context_create(int device, sc_context** out) {
  SC_REQUIRE(out != nullptr, "sc_context_create: out is NULL");
  int count = 0;
  cudaError_t e = cudaGetDeviceCount(&count);
  if (e != cudaSuccess || count == 0) {
    set_error("sc_context_create: no CUDA device is visible (%s). spectralcluster_b200 has no "
              "CPU fallback.", cudaGetErrorString(e));
    return 1;
  }
  SC_REQUIRE(device >= 0 && device < count, "sc_context_create: device %d out of range [0,%d)",
             device, count);
  SC_CUDA(cudaSetDevice(device));
  cudaDeviceProp prop;
  SC_CUDA(cudaGetDeviceProperties(&prop, device));
  SC_REQUIRE(prop.major == 9 && prop.minor == 0, "sc_context_create: device %d is sm_%d%d; this "
             "library is built for sm_90a (H100) only", device, prop.major, prop.minor);
  sc_context* ctx = new sc_context();
  ctx->device = device;
  ctx->sm_count = prop.multiProcessorCount;
  ctx->smem_optin = prop.sharedMemPerBlockOptin;
  ctx->cc_major = prop.major;
  ctx->cc_minor = prop.minor;
  ctx->gemm_sm_limit = 0;
  ctx->gemm_pace = nullptr;
  if (!getenv("SCB_NO_GEMM_PACING") &&
      cudaMalloc(&ctx->gemm_pace, sizeof(unsigned int) * SC_GEMM_PACE_SLOTS) != cudaSuccess)
    ctx->gemm_pace = nullptr;
  // keep stream-ordered scratch inside the pool between calls (no trim at every sync)
  cudaMemPool_t pool;
  if (cudaDeviceGetDefaultMemPool(&pool, device) == cudaSuccess) {
    uint64_t keep = UINT64_MAX;
    cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
  }
  *out = ctx;
  return 0;
}

extern "C" int sc_context_destroy(sc_context* ctx) {
  if (ctx && ctx->gemm_pace) cudaFree(ctx->gemm_pace);
  delete ctx;
  return 0;
}

extern "C" int sc_context_sm_count(const sc_context* ctx) { return ctx ? ctx->sm_count : 0; }

extern "C" int sc_context_set_gemm_sm_limit(sc_context* ctx, int sms) {
  SC_REQUIRE(ctx && sms >= 0, "sc_context_set_gemm_sm_limit: bad arguments");
  ctx->gemm_sm_limit = sms;
  return 0;
}

extern "C" int sc_affinity_cosine(sc_context* ctx, int engine, int precision, const float* xn,
                                  int64_t ldxn, const void* hi, const void* lo, int64_t ldh,
                                  int64_t n, int64_t d, float* a, int64_t lda,
                                  float* rowmax_offdiag, void* stream) {
  SC_REQUIRE(ctx && a && n > 0 && d > 0, "sc_affinity_cosine: bad arguments");
  if (engine == SC_GEMM_SIMT_F64ACC) {
    SC_REQUIRE(xn, "sc_affinity_cosine: the SIMT engine needs the fp32 operand");
    return gemm_nt_simt(1, xn, ldxn, xn, ldxn, n, n, d, a, lda, rowmax_offdiag,
                        as_stream(stream));
  }
  SC_REQUIRE(engine == SC_GEMM_TCGEN05, "sc_affinity_cosine: unknown engine %d", engine);
  SC_REQUIRE(hi && (lo || precision == SC_GEMM_SINGLE),
             "sc_affinity_cosine: the tensor-core engine needs the split fp16 planes");
  return gemm_nt_wgmma(ctx, 1, precision, (const __half*)hi, (const __half*)lo, ldh,
                         (const __half*)hi, (const __half*)lo, ldh, n, n, d, a, lda,
                         rowmax_offdiag, /*symmetric=*/true, /*diag_shift=*/0, nullptr, nullptr,
                         nullptr, 0, as_stream(stream));
}

extern "C" int sc_diffuse(sc_context* ctx, int engine, int precision, const float* y,
                          int64_t ldy, const void* hi, const void* lo, int64_t ldh, int64_t n,
                          float* s, int64_t lds, float* rowmax, double* rowsum, void* stream) {
  SC_REQUIRE(ctx && (s || rowmax) && n > 0, "sc_diffuse: bad arguments");
  SC_REQUIRE((rowmax == nullptr) == (rowsum == nullptr), "sc_diffuse: rowmax/rowsum come together");
  SC_REQUIRE(s || engine == SC_GEMM_TCGEN05, "sc_diffuse: s == NULL needs the tensor-core engine");
  if (engine == SC_GEMM_SIMT_F64ACC) {
    SC_REQUIRE(y, "sc_diffuse: the SIMT engine needs the fp32 operand");
    SC_REQUIRE(!rowmax, "sc_diffuse: the SIMT engine has no fused row statistics");
    return gemm_nt_simt(0, y, ldy, y, ldy, n, n, n, s, lds, nullptr, as_stream(stream));
  }
  SC_REQUIRE(engine == SC_GEMM_TCGEN05, "sc_diffuse: unknown engine %d", engine);
  SC_REQUIRE(hi && (lo || precision == SC_GEMM_SINGLE),
             "sc_diffuse: the tensor-core engine needs the split fp16 planes");
  if (rowmax) {
    SC_CUDA(cudaMemsetAsync(rowmax, 0, sizeof(float) * n, as_stream(stream)));
    SC_CUDA(cudaMemsetAsync(rowsum, 0, sizeof(double) * n, as_stream(stream)));
  }
  return gemm_nt_wgmma(ctx, 0, precision, (const __half*)hi, (const __half*)lo, ldh,
                         (const __half*)hi, (const __half*)lo, ldh, n, n, n, s, lds, nullptr,
                         /*symmetric=*/true, /*diag_shift=*/0, rowmax, rowsum, nullptr, 0,
                         as_stream(stream));
}

// ---- bounded Diffuse: row maxima of S = Y Y^T from the tiles that can hold one ----------------
extern "C" int sc_diffuse_tile_list(sc_context* ctx, const float* norms, int64_t groups,
                                    const double* diag_lb, const int* perm, int64_t n,
                                    uint32_t* tiles, int* count, int* total, void* stream) {
  SC_REQUIRE(ctx && norms && diag_lb && perm && tiles && count && total && n > 0,
             "sc_diffuse_tile_list: bad arguments");
  return diffuse_tile_list(norms, (int)groups, diag_lb, perm, n, tiles, count, total,
                           as_stream(stream));
}

extern "C" int sc_diffuse_rowmax_tiles(sc_context* ctx, const void* yp_hi, int64_t ldh, int64_t n,
                                       const uint32_t* tiles, const int* count, const int* perm,
                                       float* rowmax, void* stream) {
  SC_REQUIRE(ctx && yp_hi && tiles && count && perm && rowmax && n > 0,
             "sc_diffuse_rowmax_tiles: bad arguments");
  return diffuse_rowmax_tiles(ctx, (const __half*)yp_hi, ldh, n, tiles, count, perm, rowmax,
                              false, as_stream(stream));
}

extern "C" int sc_diffuse_rowmax_tiles_fold(sc_context* ctx, const void* yp_hi, int64_t ldh,
                                            int64_t n, const uint32_t* tiles, const int* count,
                                            const int* perm, float* rowmax, void* stream) {
  SC_REQUIRE(ctx && yp_hi && tiles && count && perm && rowmax && n > 0,
             "sc_diffuse_rowmax_tiles_fold: bad arguments");
  return diffuse_rowmax_tiles(ctx, (const __half*)yp_hi, ldh, n, tiles, count, perm, rowmax,
                              true, as_stream(stream));
}

extern "C" int sc_diffuse_hub_tiles(sc_context* ctx, const int* starts, int k, int64_t n,
                                    uint32_t* tiles, int* count, void* stream) {
  SC_REQUIRE(ctx && starts && tiles && count && n > 0, "sc_diffuse_hub_tiles: bad arguments");
  return diffuse_hub_tiles(starts, k, n, tiles, count, as_stream(stream));
}

extern "C" int sc_diffuse_tile_list_rows(sc_context* ctx, const float* norms, int64_t groups,
                                         const int* perm, int64_t n, const float* rowmax,
                                         const int* starts, int k, uint32_t* tiles, int* count,
                                         int* total, void* stream) {
  SC_REQUIRE(ctx && norms && perm && rowmax && starts && tiles && count && total && n > 0,
             "sc_diffuse_tile_list_rows: bad arguments");
  return diffuse_tile_list_rows(norms, (int)groups, perm, n, rowmax, starts, k, tiles, count,
                                total, as_stream(stream));
}

// ---- row-block / general variants used by the row-sharded multi-GPU pipeline ----------------
extern "C" int sc_affinity_cosine_block(sc_context* ctx, int precision, const void* hi,
                                        const void* lo, int64_t ldh, int64_t n, int64_t d,
                                        int64_t row_begin, int64_t row_count, float* a_block,
                                        int64_t lda, float* rowmax_offdiag_block, void* stream) {
  SC_REQUIRE(ctx && hi && a_block && n > 0 && d > 0 && row_begin >= 0 && row_count > 0 &&
             row_begin + row_count <= n, "sc_affinity_cosine_block: bad arguments");
  SC_REQUIRE(lo || precision == SC_GEMM_SINGLE, "sc_affinity_cosine_block: lo plane missing");
  const __half* h = (const __half*)hi;
  const __half* l = (const __half*)lo;
  return gemm_nt_wgmma(ctx, 1, precision, h + row_begin * ldh, l ? l + row_begin * ldh : nullptr,
                         ldh, h, l, ldh, row_count, n, d, a_block, lda, rowmax_offdiag_block,
                         /*symmetric=*/false, /*diag_shift=*/(int)row_begin, nullptr, nullptr,
                         nullptr, 0, as_stream(stream));
}

// Rows [row_begin, row_begin + row_count) of the sc_affinity_cosine matrix, bit for bit: one
// 128-row strip at a time, the tiles on and above the diagonal computed directly and those below it
// as the transpose of their mirror tile, as the symmetric whole-matrix launch does.
extern "C" int sc_affinity_cosine_panel(sc_context* ctx, int precision, const void* hi,
                                        const void* lo, int64_t ldh, int64_t n, int64_t d,
                                        int64_t row_begin, int64_t row_count, float* a_panel,
                                        int64_t lda, float* crop_panel, void* stream) {
  SC_REQUIRE(ctx && hi && a_panel && n > 0 && d > 0 && row_begin >= 0 && row_count > 0 &&
             row_begin + row_count <= n, "sc_affinity_cosine_panel: bad arguments");
  SC_REQUIRE(row_begin % 128 == 0, "sc_affinity_cosine_panel: row_begin must be a multiple of 128");
  SC_REQUIRE(lo || precision == SC_GEMM_SINGLE, "sc_affinity_cosine_panel: lo plane missing");
  const __half* h = (const __half*)hi;
  const __half* l = (const __half*)lo;
  cudaStream_t st = as_stream(stream);
  for (int64_t s0 = row_begin; s0 < row_begin + row_count; s0 += 128) {
    const int64_t rows = std::min<int64_t>(128, row_begin + row_count - s0);   // rows of the panel
    float* strip = a_panel + (s0 - row_begin) * lda;
    // columns [s0, n): the diagonal tile and the tiles right of it
    if (int rc = gemm_nt_wgmma(ctx, 1, precision, h + s0 * ldh, l ? l + s0 * ldh : nullptr, ldh,
                               h + s0 * ldh, l ? l + s0 * ldh : nullptr, ldh, rows, n - s0, d,
                               strip + s0, lda, nullptr, /*symmetric=*/false, 0, nullptr, nullptr,
                               nullptr, 0, st))
      return rc;
    // columns [0, s0): tiles (rows of X[0, s0)) x (this strip), stored transposed only
    if (s0 > 0)
      if (int rc = gemm_nt_wgmma(ctx, 1, precision, h, l, ldh, h + s0 * ldh,
                                 l ? l + s0 * ldh : nullptr, ldh, s0, rows, d, nullptr, 0, nullptr,
                                 /*symmetric=*/false, 0, nullptr, nullptr, strip, lda, st))
        return rc;
  }
  if (crop_panel) return crop_diagonal_rows(a_panel, n, lda, row_begin, row_count, crop_panel, st);
  return 0;
}

extern "C" int sc_gemm_nt_planes(sc_context* ctx, int precision, const void* a_hi,
                                 const void* a_lo, int64_t lda, int64_t m, const void* b_hi,
                                 const void* b_lo, int64_t ldb, int64_t n, int64_t k, float* c,
                                 int64_t ldc, float* c_mirror, int64_t ldm, void* stream) {
  SC_REQUIRE(ctx && a_hi && b_hi && c && m > 0 && n > 0 && k > 0, "sc_gemm_nt_planes: bad arguments");
  SC_REQUIRE((a_lo && b_lo) || precision == SC_GEMM_SINGLE || (a_lo && precision == SC_GEMM_SPLIT2),
             "sc_gemm_nt_planes: lo planes missing");
  SC_REQUIRE(c_mirror == nullptr || ldm >= m, "sc_gemm_nt_planes: bad mirror leading dimension");
  return gemm_nt_wgmma(ctx, 0, precision, (const __half*)a_hi, (const __half*)a_lo, lda,
                         (const __half*)b_hi, (const __half*)b_lo, ldb, m, n, k, c, ldc, nullptr,
                         /*symmetric=*/true, /*diag_shift=*/0, nullptr, nullptr, c_mirror, ldm,
                         as_stream(stream));
}

// Row statistics of the single-MMA product a_hi[m,k] b_hi[n,k]^T, nothing stored: the epilogue of
// sc_diffuse(s == NULL) on a rectangular block.  rowmax (fp32) and rowsum (fp64) are indexed by the
// rows of a and are folded into, not reset, so that a row's statistics accumulate over column
// blocks.  When a and b are the same rows (a_hi == b_hi, m == n) the symmetric launch computes the
// upper tiles only and folds the mirrored column statistics, as sc_diffuse does.
extern "C" int sc_diffuse_stats_block(sc_context* ctx, const void* a_hi, int64_t lda, int64_t m,
                                      const void* b_hi, int64_t ldb, int64_t n, int64_t k,
                                      float* rowmax, double* rowsum, void* stream) {
  SC_REQUIRE(ctx && a_hi && b_hi && rowmax && rowsum && m > 0 && n > 0 && k > 0,
             "sc_diffuse_stats_block: bad arguments");
  return gemm_nt_wgmma(ctx, 0, SC_GEMM_SINGLE, (const __half*)a_hi, nullptr, lda,
                         (const __half*)b_hi, nullptr, ldb, m, n, k, nullptr, 0, nullptr,
                         /*symmetric=*/true, /*diag_shift=*/0, rowmax, rowsum, nullptr, 0,
                         as_stream(stream));
}

// c[m,n] = a[m,k] b[n,k]^T with fp32 operands on the SIMT engine (fp64 accumulation): the small-
// matrix twin of sc_gemm_nt_planes for the constraint propagation products (constraint.py:147-153).
extern "C" int sc_gemm_nt_f32(sc_context* ctx, const float* a, int64_t lda, const float* b,
                              int64_t ldb, int64_t m, int64_t n, int64_t k, float* c, int64_t ldc,
                              void* stream) {
  SC_REQUIRE(ctx && a && b && c && m > 0 && n > 0 && k > 0, "sc_gemm_nt_f32: bad arguments");
  return gemm_nt_simt(0, a, lda, b, ldb, m, n, k, c, ldc, nullptr, as_stream(stream));
}
