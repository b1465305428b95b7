// wgmma / TMA GEMM for sm_90a:  C[M,N] = A[M,K] * B[N,K]^T  (both operands K-major),
// the only two dense contractions of the hot path:
//   utils.py:35-39        affinity = (Xn Xn^T + 1)/2        K = d      (EPI_AFFINITY)
//   refinement.py:232-234 Diffuse  = Y Y^T                  K = N      (EPI_PLAIN)
//
// Operands are "split fp16 planes" (value = hi + lo).  Per 64-wide K block each consumer
// warpgroup issues
//     D += Ahi*Blo ; D += Alo*Bhi ; D += Ahi*Bhi          (wgmma kind f16, fp32 accum)
// which reproduces the fp32 product to ~2^-22 relative (the dropped lo*lo term is 2^-22) at the
// fp16 tensor-pipe rate.  SC_GEMM_SPLIT2 drops the B_lo plane (D += Alo*Bhi ; D += Ahi*Bhi: the
// missing Ahi*Blo term is a zero-mean 2^-12 relative perturbation per product that averages down
// with sqrt(K)); SC_GEMM_SINGLE issues only hi*hi (2^-11 on both sides).
//
// Structure (one CTA per SM, persistent, 384 threads = 3 warpgroups, 128 x BN output tile):
//   warpgroup 0  warp 0 lane 0 is the TMA producer: cp.async.bulk.tensor.2d (SWIZZLE_128B) of the
//                4 (or 3, 2) planes of a K block into a ring of stages, completion on an mbarrier
//                (expect_tx); paced against the other CTAs' producers through a global
//                checkpoint counter (see below)
//   warpgroups 1-2  consumers (setmaxnreg 232): each owns 64 rows of the tile and issues
//                wgmma.m64n{BN}k16 from shared-memory descriptors into a register chain
//                accumulator.  A chain is only CHUNK_KB K-blocks long; at its end the chain is
//                added, round-to-nearest, into a second register tile (the tensor core's fp32
//                accumulation truncates, so long chains drift low -- the two-level scheme keeps the
//                bias below 1e-6).  At the end of the tile the consumers run the fused epilogue
//                straight from registers: (x+1)/2 + off-diagonal row maximum (affinity), row
//                maximum / sum (Diffuse), the stores, and the mirrored (transposed) stores of the
//                symmetric variant.
// Tile width BN: the Diffuse products at one or two MMAs (EPI_PLAIN, SINGLE / SPLIT2) use
// 128 x 192 tiles.  Each consumer warpgroup reads its A half and all of B from shared memory per
// wgmma, so the wider tile moves ~14 % fewer shared-memory bytes and 17 % fewer L2 bytes per MMA;
// the chain and sum accumulators (96 + 96 registers per thread) still fit the 232 of setmaxnreg.
// SPLIT3 keeps 128 x 128 (at 192 its 72 KB stages would leave a ring of 2), and so does the
// affinity (K = d: bound by its stores, not by operand traffic).
// Tiles are rasterised in groups of 16 M-blocks so that a wave of CTAs shares 16 A-panels and ~8
// B-panels through L2.  The symmetric variant (C = Y Y^T) computes only the tiles that reach the
// upper triangle, tile (m, n) iff BN n + BN - 1 >= BM m, and stores the mirrored half from them.
#include "common.cuh"

#include <cuda.h>
#include <atomic>
#include <cstdlib>
#include <mutex>

namespace sc {

constexpr int BM = 128, BK = 64;                     // BK fp16 = 128 bytes = one swizzle row
constexpr int WG_M = 64;                             // rows of the tile per consumer warpgroup
constexpr int MMA_K = 16;
constexpr int A_PLANE_BYTES = BM * BK * 2;           // 16 KB
constexpr int GROUP_M = 16;
// K-blocks between pacing checkpoints of the producers.  The window the CTAs of a wave may drift
// apart is PACE_KB x ~0.4-0.8 MB of operand panels per K block; 32 keeps it well inside L2.
// Single-MMA Diffuse at N = 65,536 on uniform operands (H100 SXM, 700 W limit): 16 / 32 / 64 ->
// 535 / 527 / 518 ms, one run each; without pacing 1,380 ms.
constexpr int PACE_KB = 32;
constexpr int PACE_SPINS = 400;   // x 100 ns: bounded wait (a hint, never a dependency)
constexpr uint32_t SPIN_LIMIT = 1u << 27;            // trap instead of hanging the GPU
constexpr int NUM_CONSUMER_WARPS = 8;
constexpr int NUM_THREADS = 128 + NUM_CONSUMER_WARPS * 32;   // 384

static_assert(BM == 2 * WG_M, "two consumer warpgroups of 64 rows each");

enum { TC_EPI_PLAIN = 0, TC_EPI_AFFINITY = 1 };

// ---------------------------------------------------------------- PTX helpers
__device__ __forceinline__ uint32_t smem_u32(const void* p) {
  return (uint32_t)__cvta_generic_to_shared(p);
}
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes)
               : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t spins = 0;
  while (!mbar_try_wait(bar, parity)) {
    if (++spins > SPIN_LIMIT) __trap();
  }
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar,
                                            int32_t c_inner, int32_t c_outer) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes "
      "[%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"(map), "r"(bar), "r"(c_inner), "r"(c_outer)
      : "memory");
}

__device__ __forceinline__ void wgmma_fence() {
  asm volatile("wgmma.fence.sync.aligned;" ::: "memory");
}
__device__ __forceinline__ void wgmma_commit() {
  asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory");
}
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory");
}

// K-major, SWIZZLE_128B shared-memory matrix descriptor (sm_90 GMMA descriptor): start>>4 [0,14) |
// LBO>>4 [16,30) (=1, unused for swizzled K-major) | SBO>>4 [32,46) = 1024 B between 8-row
// groups | base offset [49,52) = 0 (stage buffers are 1024-byte aligned) | layout [62,64) = 1
// (SWIZZLE_128B).  Advancing K by 16 fp16 inside the swizzle atom adds 32 B to the start address.
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t smem_addr) {
  uint64_t d = 0;
  d |= (uint64_t)((smem_addr >> 4) & 0x3FFFu);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

// D[64 x BN] (+)= A[64 x 16] B[BN x 16]^T, fp16 in, fp32 accumulate; scale_d = 0 overwrites D.
// Fragment of thread t of the warpgroup: warp w = t / 32, lane l; d[4 j + 2 h + e] is row
// 16 w + l / 4 + 8 h, column 8 j + 2 (l % 4) + e, j < BN / 8.
template <int BN>
__device__ __forceinline__ void wgmma_m64k16(float (&d)[BN / 2], uint64_t adesc, uint64_t bdesc,
                                             uint32_t scale_d) {
  static_assert(BN == 128 || BN == 192, "wgmma tile width");
  if constexpr (BN == 128) {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %66, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
        "%64, %65, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]),
          "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]),
          "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),
          "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
          "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]),
          "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]),
          "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]),
          "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),
          "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]),
          "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]),
          "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
        : "l"(adesc), "l"(bdesc), "r"(scale_d));
  } else {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "setp.ne.b32 p, %98, 0;\n\t"
        "wgmma.mma_async.sync.aligned.m64n192k16.f32.f16.f16 "
        "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
        "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
        "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
        "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, "
        "%64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, "
        "%80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95}, "
        "%96, %97, p, 1, 1, 0, 0;\n\t}"
        : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]),
          "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]),
          "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),
          "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]),
          "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]),
          "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]),
          "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]),
          "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]),
          "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]),
          "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]),
          "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]),
          "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]),
          "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]),
          "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]),
          "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]),
          "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95])
        : "l"(adesc), "l"(bdesc), "r"(scale_d));
  }
}

struct TileCoord {
  int m_blk, n_blk;
};

// Rasterisation.  Full problem: groups of GROUP_M M-blocks sweep all N-blocks.  Symmetric
// problem (C = Y Y^T): only the tiles that reach the upper triangle (c >= r) are computed, i.e.
// tile (m, n) iff its last column BN n + BN - 1 >= its first row BM m; the rest is filled by
// mirrored stores.  group_start[g] is the first tile index of group g (host-computed with the
// same counting rule).  Any BN works here; BN is a multiple of 8 for the epilogue fragments.
constexpr int MAX_GROUPS = 160;
struct TileTable {
  int group_start[MAX_GROUPS + 1];
  int num_groups;
  int num_tiles;
};

template <int BN>
__host__ __device__ inline int sym_valid_mblocks(int g, int n_blk, int tiles_m) {
  // m blocks of group g that are valid for column block n_blk: BM m_blk <= BN n_blk + BN - 1
  int lim = (n_blk * BN + BN - 1) / BM + 1 - g * GROUP_M;
  const int avail = tiles_m - g * GROUP_M;
  if (lim > GROUP_M) lim = GROUP_M;
  if (lim > avail) lim = avail;
  return lim < 0 ? 0 : lim;
}

// first column block whose tiles reach the first row of group g
template <int BN>
__host__ __device__ inline int sym_first_nblk(int g) {
  return g * GROUP_M * BM / BN;
}

// Tile coordinates for a CTA that walks tile, tile + stride, tile + 2 stride, ...: the symmetric
// table search would cost ~1 k instructions per call, which is noise at K = N but not at K = d
// (affinity), so the cursor moves forward inside the (group, column block) enumeration instead
// of restarting it.
template <bool SYM, int BN>
struct TileCursor {
  int tiles_m, tiles_n;
  int g, nb, base;          // SYM: current group, column block, first tile index of (g, nb)
  __device__ __forceinline__ void init(int tm, int tn) {
    tiles_m = tm; tiles_n = tn; g = 0; nb = 0; base = 0;
  }
  __device__ __forceinline__ TileCoord at(int tile, const TileTable& tab) {
    TileCoord t;
    if (!SYM) {
      const int group = GROUP_M * tiles_n;
      const int gg = tile / group;
      const int first_m = gg * GROUP_M;
      const int gm = min(GROUP_M, tiles_m - first_m);
      const int r = tile - gg * group;
      t.m_blk = first_m + r % gm;
      t.n_blk = r / gm;
    } else {
      // tiles are visited in increasing order: move forward only
      while (g + 1 < tab.num_groups && tab.group_start[g + 1] <= tile) {
        ++g;
        nb = sym_first_nblk<BN>(g);
        base = tab.group_start[g];
      }
      for (;;) {
        const int cnt = sym_valid_mblocks<BN>(g, nb, tiles_m);
        if (tile - base < cnt) break;
        base += cnt;
        ++nb;
      }
      t.m_blk = g * GROUP_M + (tile - base);
      t.n_blk = nb;
    }
    return t;
  }
};

__device__ __forceinline__ TileCoord listed_tile(const uint32_t* __restrict__ list, int tile) {
  const uint32_t v = __ldg(list + tile);
  return TileCoord{(int)(v >> 16), (int)(v & 0xFFFFu)};
}

template <int PREC, int BN>
struct StageGeom {
  // planes of one K block in a stage: [A_hi][B_hi][A_lo (PREC>=2)][B_lo (PREC==3)], each a
  // multiple of the 1 KB swizzle atom.  BN = 192: 40 KB x 5 stages (single), 56 KB x 4 (split2).
  static constexpr int B_PLANE_BYTES = BN * BK * 2;
  static constexpr int BYTES =
      A_PLANE_BYTES * (PREC >= 2 ? 2 : 1) + B_PLANE_BYTES * (PREC == 3 ? 2 : 1);
  static constexpr int BUDGET = 227 * 1024 - 1024 - 256;
  static constexpr int STAGES = (BUDGET / BYTES) > 8 ? 8 : (BUDGET / BYTES);
};

template <int PREC, int EPI, bool SYM, int BN, bool LIST = false>
__global__ void __launch_bounds__(NUM_THREADS, 1)
k_gemm_wgmma(const __grid_constant__ CUtensorMap map_a_hi,
             const __grid_constant__ CUtensorMap map_a_lo,
             const __grid_constant__ CUtensorMap map_b_hi,
             const __grid_constant__ CUtensorMap map_b_lo,
             const __grid_constant__ TileTable tab, int M, int N, int K,
             float* __restrict__ C, int64_t ldc, float* __restrict__ rowmax_offdiag,
             int diag_shift, unsigned int* __restrict__ pace, int pace_kb,
             float* __restrict__ stat_rowmax, double* __restrict__ stat_rowsum,
             float* __restrict__ mirror_out, int64_t ldm, int aff_chunk_kb,
             const uint32_t* __restrict__ tile_list, const int* __restrict__ tile_count,
             const int* __restrict__ row_map) {
  constexpr int STAGES = StageGeom<PREC, BN>::STAGES;
  constexpr int STAGE_BYTES = StageGeom<PREC, BN>::BYTES;
  constexpr int B_PLANE_BYTES = StageGeom<PREC, BN>::B_PLANE_BYTES;
  constexpr int NACC = BN / 2;          // accumulator registers per thread and tile
  // The affinity stores its diagonal tiles whole, without the mask of the straddling tiles below:
  // that needs square tiles.
  static_assert(EPI == TC_EPI_PLAIN || BN == BM, "the affinity runs on square tiles");
  // K blocks per register chain.  Diffuse: 2 (split) / 4 (single).  Affinity (K = d):
  // `aff_chunk_kb` from the host, 1 by default -- the affinity feeds a threshold, so it gets the
  // shortest chains (SCB_AFFINITY_CHUNK_KB overrides).
  const int CHUNK_KB = (EPI == TC_EPI_AFFINITY) ? aff_chunk_kb : (PREC == 1 ? 4 : 2);
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~(uintptr_t)1023);
  uint64_t* bars = reinterpret_cast<uint64_t*>(smem + STAGES * STAGE_BYTES);
  uint64_t* full_bar = bars;
  uint64_t* empty_bar = bars + STAGES;

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int tiles_m = (M + BM - 1) / BM, tiles_n = (N + BN - 1) / BN;
  // LIST: the tiles come from a device list (tile_list[0, *tile_count), packed m_blk << 16 | n_blk,
  // in the rasterised order), row statistics are maxima only, stored through row_map
  static_assert(!LIST || (SYM && EPI == TC_EPI_PLAIN), "a tile list serves the symmetric Diffuse");
  const int num_tiles = LIST ? *tile_count : SYM ? tab.num_tiles : tiles_m * tiles_n;
  const int num_kb = (K + BK - 1) / BK;

  if (warp == 0 && lane == 0) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_a_hi) : "memory");
    asm volatile("prefetch.tensormap [%0];" ::"l"(&map_b_hi) : "memory");
    if (PREC >= 2) asm volatile("prefetch.tensormap [%0];" ::"l"(&map_a_lo) : "memory");
    if (PREC == 3) asm volatile("prefetch.tensormap [%0];" ::"l"(&map_b_lo) : "memory");
  }
  if (warp == 1 && lane == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(smem_u32(&full_bar[s]), 1);
      mbar_init(smem_u32(&empty_bar[s]), NUM_CONSUMER_WARPS);
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();

  if (warp < 4) {
    // the producer warpgroup gives its registers to the consumer warpgroups
    asm volatile("setmaxnreg.dec.sync.aligned.u32 40;");
    if (warp == 0 && lane == 0) {
      // ===================================================== TMA producer
      int stage = 0;
      uint32_t phase = 0;
      // Pacing: the CTAs of a wave share their A/B panels through L2 only while they stream K at
      // the same position.  Left alone they drift apart and every CTA re-reads its panels from
      // DRAM, so every pace_kb K-blocks each producer signs in on a global counter and waits --
      // bounded, it is only a hint -- until the whole grid has reached the same checkpoint.
      const int ck_per_tile = (num_kb + pace_kb - 1) / pace_kb;
      unsigned int passed = 0;
      TileCursor<SYM, BN> cursor;
      cursor.init(tiles_m, tiles_n);
      for (int round = 0; round * (int)gridDim.x < num_tiles; ++round) {
        const int tile = round * (int)gridDim.x + (int)blockIdx.x;
        if (tile >= num_tiles) {            // no tile in the last round: keep the targets reachable
          if (pace) atomicAdd(pace, (unsigned int)ck_per_tile);
          continue;
        }
        const TileCoord tc = LIST ? listed_tile(tile_list, tile) : cursor.at(tile, tab);
        const int row_a = tc.m_blk * BM, row_b = tc.n_blk * BN;
        for (int kb = 0; kb < num_kb; ++kb) {
          if (pace && kb % pace_kb == 0) {
            atomicAdd(pace, 1u);
            ++passed;
            const unsigned int target = passed * gridDim.x;
            for (int spin = 0; spin < PACE_SPINS; ++spin) {
              if (*reinterpret_cast<volatile unsigned int*>(pace) >= target) break;
              __nanosleep(100);
            }
          }
          mbar_wait(smem_u32(&empty_bar[stage]), phase ^ 1u);
          const uint32_t bar = smem_u32(&full_bar[stage]);
          const uint32_t base = smem_u32(smem + stage * STAGE_BYTES);
          const int k0 = kb * BK;
          mbar_expect_tx(bar, (uint32_t)STAGE_BYTES);
          tma_load_2d(base, &map_a_hi, bar, k0, row_a);
          tma_load_2d(base + A_PLANE_BYTES, &map_b_hi, bar, k0, row_b);
          if (PREC >= 2) tma_load_2d(base + A_PLANE_BYTES + B_PLANE_BYTES, &map_a_lo, bar, k0, row_a);
          if (PREC == 3)
            tma_load_2d(base + 2 * A_PLANE_BYTES + B_PLANE_BYTES, &map_b_lo, bar, k0, row_b);
          if (++stage == STAGES) { stage = 0; phase ^= 1u; }
        }
      }
    }
    return;
  }

  // ===================================================== consumer warpgroups
  asm volatile("setmaxnreg.inc.sync.aligned.u32 232;");
  const int wg = (warp - 4) >> 2;                       // rows [64 wg, +64) of the tile
  const int wq = warp & 3;                              // rows [16 wq, +16) of those
  int stage = 0;
  uint32_t phase = 0;
  float acc[NACC], sum[NACC];
#pragma unroll
  for (int i = 0; i < NACC; ++i) acc[i] = 0.0f;
  TileCursor<SYM, BN> cursor;
  cursor.init(tiles_m, tiles_n);
  for (int tile = blockIdx.x; tile < num_tiles; tile += gridDim.x) {
    const TileCoord tc = LIST ? listed_tile(tile_list, tile) : cursor.at(tile, tab);
#pragma unroll
    for (int i = 0; i < NACC; ++i) sum[i] = 0.0f;
    // One chain per pass of the outer loop.  Its end is a structural wait<0>, so the compiler sees
    // no path on which accumulator registers are read while a wgmma group is in flight (a wait
    // on a data-dependent branch makes ptxas drain the pipe at every K block).
    for (int kb0 = 0; kb0 < num_kb; kb0 += CHUNK_KB) {
      const int kb_end = min(kb0 + CHUNK_KB, num_kb);
      int pending = -1;                 // stage whose MMAs are issued but whose buffer is not freed
      for (int kb = kb0; kb < kb_end; ++kb) {
        const int in_chunk = kb - kb0;
        mbar_wait(smem_u32(&full_bar[stage]), phase);
        const uint32_t base = smem_u32(smem + stage * STAGE_BYTES);
        const uint32_t a_off = (uint32_t)(wg * WG_M * BK * 2);
        const uint64_t a_hi = make_smem_desc(base + a_off);
        const uint64_t b_hi = make_smem_desc(base + A_PLANE_BYTES);
        const uint64_t a_lo = make_smem_desc(base + A_PLANE_BYTES + B_PLANE_BYTES + a_off);
        const uint64_t b_lo = make_smem_desc(base + 2 * A_PLANE_BYTES + B_PLANE_BYTES);
        wgmma_fence();
        // The small cross products go first: the accumulation truncates each add to the
        // accumulator's current ulp, so terms added while the chain is still small cost almost
        // nothing; only the BK/16 hi*hi accumulates run at full magnitude.
        if (PREC == 3) {
#pragma unroll
          for (int kk = 0; kk < BK / MMA_K; ++kk) {
            const uint64_t adv = (uint64_t)(kk * MMA_K * 2 / 16);
            wgmma_m64k16<BN>(acc, a_hi + adv, b_lo + adv, (in_chunk | kk) ? 1u : 0u);
            wgmma_m64k16<BN>(acc, a_lo + adv, b_hi + adv, 1u);
          }
        } else if (PREC == 2) {
#pragma unroll
          for (int kk = 0; kk < BK / MMA_K; ++kk) {
            const uint64_t adv = (uint64_t)(kk * MMA_K * 2 / 16);
            wgmma_m64k16<BN>(acc, a_lo + adv, b_hi + adv, (in_chunk | kk) ? 1u : 0u);
          }
        }
#pragma unroll
        for (int kk = 0; kk < BK / MMA_K; ++kk) {
          const uint64_t adv = (uint64_t)(kk * MMA_K * 2 / 16);
          wgmma_m64k16<BN>(acc, a_hi + adv, b_hi + adv, (PREC >= 2 || in_chunk || kk) ? 1u : 0u);
        }
        wgmma_commit();
        // one group in flight: the previous K block's buffer is free once this one is queued
        wgmma_wait<1>();
        if (lane == 0 && pending >= 0) mbar_arrive(smem_u32(&empty_bar[pending]));
        pending = stage;
        if (++stage == STAGES) { stage = 0; phase ^= 1u; }
      }
      // chain complete: fold it into the tile, round-to-nearest
      wgmma_wait<0>();
      if (lane == 0) mbar_arrive(smem_u32(&empty_bar[pending]));
#pragma unroll
      for (int i = 0; i < NACC; ++i) sum[i] += acc[i];
    }

    // ---- epilogue, straight from the accumulator fragment: this thread holds rows r0 and r0 + 8
    // of the tile, columns 8 j + 2 (lane % 4) + {0, 1} for j < BN / 8.
    const int64_t r0 = (int64_t)tc.m_blk * BM + wg * WG_M + wq * 16 + (lane >> 2);
    const int64_t col0 = (int64_t)tc.n_blk * BN + 2 * (lane & 3);
    const int64_t tile_row0 = (int64_t)tc.m_blk * BM, tile_col0 = (int64_t)tc.n_blk * BN;
    const bool full = (tile_row0 + BM <= M) && (tile_col0 + BN <= N);     // CTA-uniform
    // Symmetric product: the tiles below the diagonal are skipped; every tile wholly above it also
    // stores its transpose.  A Diffuse tile that straddles the diagonal stores element (r, c) iff
    // c >= r and its mirror (c, r) iff c > r, so each element of C is written once, from one
    // accumulator, and C is bitwise symmetric; its row statistics take c >= r, the mirrored
    // column statistics r < c.  The affinity's square diagonal tiles store every element directly.
    // Both flags are CTA-uniform: the tiles wholly above the diagonal run unmasked.
    const bool above = SYM && tile_col0 >= tile_row0 + BM;
    const bool straddle = SYM && EPI == TC_EPI_PLAIN && !above;
    const bool mirror = above || straddle;
    // in a straddling tile, element (r0 + 8 h, col0 + x) lies on the diagonal iff x = diag + 8 h
    const int diag = (int)(r0 - col0);
    if (EPI == TC_EPI_AFFINITY) {
#pragma unroll
      for (int i = 0; i < NACC; ++i) sum[i] = fmaf(sum[i], 0.5f, 0.5f);   // (x + 1) / 2, utils.py:39
    }
    const bool row_stats = (EPI == TC_EPI_AFFINITY && rowmax_offdiag != nullptr) ||
                           (EPI == TC_EPI_PLAIN && stat_rowmax != nullptr);
    if (row_stats) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int64_t row = r0 + 8 * h;
        const int64_t dcol = row + diag_shift;          // this row's diagonal column (affinity)
        float mx = 0.0f, sm = 0.0f;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int64_t col = col0 + 8 * j + e;
            const float v = sum[4 * j + 2 * h + e];
            // columns past N: zero-filled operands (plain: 0, no effect on the sum or a
            // non-negative maximum; affinity: 0.5, excluded)
            if (EPI == TC_EPI_AFFINITY) {
              if (col != dcol && (full || col < N)) mx = fmaxf(mx, v);
            } else if (!straddle || 8 * j + e >= diag + 8 * h) {
              mx = fmaxf(mx, v);
              if (!LIST) sm += v;
            }
          }
        }
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
        if (EPI == TC_EPI_PLAIN && !LIST) {
          sm += __shfl_xor_sync(0xffffffffu, sm, 1);
          sm += __shfl_xor_sync(0xffffffffu, sm, 2);
        }
        if ((lane & 3) == 0 && row < M) {
          if (EPI == TC_EPI_AFFINITY) {
            atomic_max_nonneg(rowmax_offdiag + row, mx);
          } else if (LIST) {
            atomic_max_nonneg(stat_rowmax + row_map[row], mx);
          } else {
            atomic_max_nonneg(stat_rowmax + row, mx);
            atomicAdd(stat_rowsum + row, (double)sm);
          }
        }
      }
    }
    if (mirror && row_stats) {
      // the mirrored elements of column c form a piece of ROW c of C: column reductions over the
      // tile's rows (rows past M are skipped)
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
        for (int e = 0; e < 2; ++e) {
          const int64_t tr = col0 + 8 * j + e;
          float mx = 0.0f, sm = 0.0f;
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            if ((full || r0 + 8 * h < M) && (!straddle || 8 * j + e > diag + 8 * h)) {
              const float v = sum[4 * j + 2 * h + e];
              mx = fmaxf(mx, v);
              if (!LIST) sm += v;
            }
          }
#pragma unroll
          for (int o = 4; o < 32; o <<= 1) {
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
            if (EPI == TC_EPI_PLAIN && !LIST) sm += __shfl_xor_sync(0xffffffffu, sm, o);
          }
          if (lane < 4 && tr < N) {
            if (EPI == TC_EPI_AFFINITY) {
              atomic_max_nonneg(rowmax_offdiag + tr, mx);
            } else if (LIST) {
              atomic_max_nonneg(stat_rowmax + row_map[tr], mx);
            } else {
              atomic_max_nonneg(stat_rowmax + tr, mx);
              atomicAdd(stat_rowsum + tr, (double)sm);
            }
          }
        }
      }
    }
    // ---- stores: a warp's float2 store covers 8 rows x 32 contiguous bytes.  C == NULL keeps the
    // row statistics (and a mirrored block) only: nothing of C is written.
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const int64_t row = r0 + 8 * h;
      if (C == nullptr || (!full && row >= M)) continue;
      float* dst = C + row * ldc + col0;
#pragma unroll
      for (int j = 0; j < BN / 8; ++j) {
        const float2 v = make_float2(sum[4 * j + 2 * h], sum[4 * j + 2 * h + 1]);
        if (straddle && 8 * j < diag + 8 * h) {          // c < r comes from the mirror of (c, r)
          if (8 * j + 1 == diag + 8 * h) dst[8 * j + 1] = v.y;
        } else if (full || col0 + 8 * j + 1 < N) {
          *reinterpret_cast<float2*>(dst + 8 * j) = v;
        } else if (col0 + 8 * j < N) {
          dst[8 * j] = v.x;
        }
      }
    }
    // ---- transposed stores: the mirrored half of a symmetric product, or (row-sharded Diffuse)
    // the peer's block S(p,g) = S(g,p)^T mapped into this process by CUDA IPC, so that the
    // exchange rides on the GEMM epilogue tile by tile.  Lanes with the same lane % 4 hold 8
    // consecutive rows: every store instruction writes 4 x 32 contiguous bytes.
    float* tdst = mirror ? C : (!SYM ? mirror_out : nullptr);   // NULL when C is (stats only)
    const int64_t ldt = mirror ? ldc : ldm;
    if (tdst != nullptr) {
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int64_t row = r0 + 8 * h;
        if (!full && row >= M) continue;
#pragma unroll
        for (int j = 0; j < BN / 8; ++j) {
#pragma unroll
          for (int e = 0; e < 2; ++e) {
            const int64_t col = col0 + 8 * j + e;
            if ((full || col < N) && (!straddle || 8 * j + e > diag + 8 * h))
              tdst[col * ldt + row] = sum[4 * j + 2 * h + e];
          }
        }
      }
    }
  }
}

// ---------------------------------------------------------------- host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*,
                                  const cuuint64_t*, const cuuint64_t*, const cuuint32_t*,
                                  const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, []() {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) ==
            cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

// 2-D fp16 tensor [rows, k] with leading dimension ld (elements); box = BK x box_rows.
static int make_plane_map(CUtensorMap* map, const __half* ptr, int64_t rows, int64_t k,
                          int64_t ld, int box_rows) {
  EncodeTiledFn enc = get_encode_fn();
  SC_REQUIRE(enc != nullptr, "cuTensorMapEncodeTiled is not available from the driver");
  SC_REQUIRE((reinterpret_cast<uintptr_t>(ptr) & 15) == 0 && (ld * 2) % 16 == 0,
             "wgmma GEMM: fp16 planes need 16-byte aligned base and ld %% 8 == 0");
  const cuuint64_t dims[2] = {(cuuint64_t)k, (cuuint64_t)rows};
  const cuuint64_t strides[1] = {(cuuint64_t)ld * 2};
  const cuuint32_t box[2] = {(cuuint32_t)BK, (cuuint32_t)box_rows};
  const cuuint32_t estr[2] = {1, 1};
  const CUresult r = enc(map, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<__half*>(ptr), dims,
                         strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                         CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                         CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  SC_REQUIRE(r == CUDA_SUCCESS, "cuTensorMapEncodeTiled failed with CUresult %d", (int)r);
  return 0;
}

template <int BN>
static void build_tile_table(TileTable& tab, int tiles_m, int tiles_n) {
  tab.num_groups = (tiles_m + GROUP_M - 1) / GROUP_M;
  int total = 0;
  for (int g = 0; g < tab.num_groups; ++g) {
    tab.group_start[g] = total;
    for (int nb = sym_first_nblk<BN>(g); nb < tiles_n; ++nb)
      total += sym_valid_mblocks<BN>(g, nb, tiles_m);
  }
  tab.group_start[tab.num_groups] = total;
  tab.num_tiles = total;
}

template <int PREC, int EPI, bool SYM, int BN>
static int launch(const sc_context* ctx, const __half* a_hi, const __half* a_lo, int64_t lda,
                  const __half* b_hi, const __half* b_lo, int64_t ldb, int M, int N, int K,
                  float* C, int64_t ldc, float* rowmax, int diag_shift, float* stat_rowmax,
                  double* stat_rowsum, float* mirror, int64_t ldm, cudaStream_t st) {
  constexpr int STAGES = StageGeom<PREC, BN>::STAGES;
  constexpr int STAGE_BYTES = StageGeom<PREC, BN>::BYTES;
  static_assert(STAGES >= 2, "wgmma GEMM: the operand ring needs at least two stages");
  CUtensorMap ah, al, bh, bl;
  if (int r = make_plane_map(&ah, a_hi, M, K, lda, BM)) return r;
  if (int r = make_plane_map(&bh, b_hi, N, K, ldb, BN)) return r;
  al = ah;
  bl = bh;
  if (PREC >= 2) {
    SC_REQUIRE(a_lo, "wgmma GEMM: the lo plane of A is missing");
    if (int r = make_plane_map(&al, a_lo, M, K, lda, BM)) return r;
  }
  if (PREC == 3) {
    SC_REQUIRE(b_lo, "wgmma GEMM: the lo plane of B is missing");
    if (int r = make_plane_map(&bl, b_lo, N, K, ldb, BN)) return r;
  }
  const size_t smem = (size_t)STAGES * STAGE_BYTES + 1024 /*align*/ + 256 /*barriers*/;
  SC_REQUIRE(smem <= ctx->smem_optin, "wgmma GEMM needs %zu B of shared memory", smem);
  auto kern = k_gemm_wgmma<PREC, EPI, SYM, BN>;
  SC_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  const int tiles_m = (M + BM - 1) / BM, tiles_n = (N + BN - 1) / BN;
  TileTable tab = {};
  int tiles = tiles_m * tiles_n;
  if (SYM) {
    SC_REQUIRE((tiles_m + GROUP_M - 1) / GROUP_M <= MAX_GROUPS, "wgmma GEMM: N too large for "
               "the symmetric tile table");
    build_tile_table<BN>(tab, tiles_m, tiles_n);
    tiles = tab.num_tiles;
  }
  int sms = ctx->sm_count;
  if (ctx->gemm_sm_limit > 0 && ctx->gemm_sm_limit < sms) sms = ctx->gemm_sm_limit;
  const int grid = tiles < sms ? tiles : sms;
  unsigned int* pace = nullptr;
  static int pace_kb = 0;
  if (pace_kb == 0) {
    const char* e = getenv("SCB_GEMM_PACE_KB");
    pace_kb = (e && atoi(e) > 0) ? atoi(e) : PACE_KB;
  }
  if (ctx->gemm_pace && (K + BK - 1) / BK >= 2 * pace_kb && tiles > grid) {
    static std::atomic<unsigned int> pace_turn{0};
    pace = ctx->gemm_pace + (pace_turn.fetch_add(1) % SC_GEMM_PACE_SLOTS);
    SC_CUDA(cudaMemsetAsync(pace, 0, sizeof(unsigned int), st));
  }
  static int aff_chunk_kb = 0;
  if (aff_chunk_kb == 0) {
    const char* e = getenv("SCB_AFFINITY_CHUNK_KB");
    aff_chunk_kb = (e && atoi(e) > 0) ? atoi(e) : 1;
  }
  kern<<<grid, NUM_THREADS, smem, st>>>(ah, al, bh, bl, tab, M, N, K, C, ldc, rowmax, diag_shift,
                                        pace, pace_kb, stat_rowmax, stat_rowsum, mirror, ldm,
                                        aff_chunk_kb, nullptr, nullptr, nullptr);
  sc::launched();
  SC_LAUNCH_CHECK();
  return 0;
}

int gemm_nt_wgmma(const sc_context* ctx, int epi, int precision, const __half* a_hi,
                  const __half* a_lo, int64_t lda, const __half* b_hi, const __half* b_lo,
                  int64_t ldb, int64_t M, int64_t N, int64_t K, float* C, int64_t ldc,
                  float* rowmax_offdiag, bool symmetric, int diag_shift, float* stat_rowmax,
                  double* stat_rowsum, float* mirror, int64_t ldm, cudaStream_t st) {
  SC_REQUIRE(M > 0 && N > 0 && K > 0 && M < (1LL << 31) && N < (1LL << 31) && K < (1LL << 31),
             "wgmma GEMM: bad shape");
  SC_REQUIRE(C || stat_rowmax || mirror, "wgmma GEMM: nothing to write");
  SC_REQUIRE((reinterpret_cast<uintptr_t>(C) & 7) == 0 && ldc % 2 == 0,
             "wgmma GEMM: C needs an 8-byte aligned base and ldc %% 2 == 0");
  SC_REQUIRE(precision == SC_GEMM_SPLIT3 || precision == SC_GEMM_SPLIT2 ||
             precision == SC_GEMM_SINGLE, "wgmma GEMM: unknown precision %d", precision);
  SC_REQUIRE((stat_rowmax == nullptr) == (stat_rowsum == nullptr),
             "wgmma GEMM: the row statistics come together");
  const int m = (int)M, n = (int)N, k = (int)K;
  // C = Y Y^T is symmetric when both operands are the same matrix: compute the upper tiles only
  const bool sym = symmetric && a_hi == b_hi && a_lo == b_lo && M == N && lda == ldb;
  SC_REQUIRE(!(sym && mirror), "wgmma GEMM: a mirrored copy only makes sense for an off-diagonal block");
#define SC_TC_LAUNCH(PR, EP, BN_)                                                                \
  do {                                                                                           \
    if (sym)                                                                                     \
      return launch<PR, EP, true, BN_>(ctx, a_hi, a_lo, lda, b_hi, b_lo, ldb, m, n, k, C, ldc,   \
                                       rowmax_offdiag, diag_shift, stat_rowmax, stat_rowsum,     \
                                       mirror, ldm, st);                                         \
    return launch<PR, EP, false, BN_>(ctx, a_hi, a_lo, lda, b_hi, b_lo, ldb, m, n, k, C, ldc,    \
                                      rowmax_offdiag, diag_shift, stat_rowmax, stat_rowsum,      \
                                      mirror, ldm, st);                                          \
  } while (0)
  // tile width per product: see the header
  if (epi == TC_EPI_AFFINITY) {
    if (precision == SC_GEMM_SPLIT3) SC_TC_LAUNCH(3, TC_EPI_AFFINITY, 128);
    if (precision == SC_GEMM_SPLIT2) SC_TC_LAUNCH(2, TC_EPI_AFFINITY, 128);
    SC_TC_LAUNCH(1, TC_EPI_AFFINITY, 128);
  }
  if (precision == SC_GEMM_SPLIT3) SC_TC_LAUNCH(3, TC_EPI_PLAIN, 128);
  if (precision == SC_GEMM_SPLIT2) SC_TC_LAUNCH(2, TC_EPI_PLAIN, 192);
  SC_TC_LAUNCH(1, TC_EPI_PLAIN, 192);
#undef SC_TC_LAUNCH
}

// ---------------------------------------------------------------- bounded Diffuse (row maxima)
// RowWiseNormalize after Diffuse needs max_j S_ij of S = Y Y^T, and Y >= 0.  For 256-column groups
// g, S_ij = sum_g <y_i^g, y_j^g> <= sum_g |y_i^g| |y_j^g|, and every row's maximum is at least its
// diagonal S_ii = |y_i|^2.  A tile of the (row-permuted) product whose bound
//   u = sum_g max_{rows of the tile} |y^g| x max_{columns of the tile} |y^g|
// lies below the smallest diagonal of its rows and columns, l, holds no row maximum of either.  With
// the computed product within a factor (1 +- BOUND_EPS) of the exact one (DESIGN.md section 3), a
// tile is skipped iff u (1 + eps) < l (1 - eps); tiles that straddle the diagonal are always
// computed, so every S~_ii is.  u is accumulated in fp64 rounded up and l from diagonals rounded
// down, so the rule holds in floating point as it does in exact arithmetic.
constexpr int LIST_BN = 192;                       // the single-MMA Diffuse tile width
constexpr double BOUND_EPS = 1.0 / 1024;           // valid for K <= 2^20
constexpr int BOUND_MAX_K = 1 << 20;

// Maxima of the group norms and minimum of the diagonal lower bounds over each block of R rows of
// the permuted order (permuted row r is row perm[r]).
__global__ void k_block_bounds(const float* __restrict__ norms, int G,
                               const double* __restrict__ diag_lb, const int* __restrict__ perm,
                               int n, int R, float* __restrict__ bmax, double* __restrict__ bmin) {
  const int b = blockIdx.x;
  const int r0 = b * R, r1 = min(n, r0 + R);
  for (int g = threadIdx.x; g < G; g += blockDim.x) {
    float m = 0.0f;
    for (int r = r0; r < r1; ++r) m = fmaxf(m, norms[(int64_t)perm[r] * G + g]);
    bmax[(int64_t)b * G + g] = m;
  }
  if (threadIdx.x < 32) {
    double l = INFINITY;
    for (int r = r0 + (int)threadIdx.x; r < r1; r += 32) l = fmin(l, diag_lb[perm[r]]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) l = fmin(l, __shfl_xor_sync(0xffffffffu, l, o));
    if (threadIdx.x == 0) bmin[b] = l;
  }
}

// One warp per (m, n) tile: flags[m tiles_n + n] = 1 iff the tile is computed.
__global__ void k_tile_flags(const float* __restrict__ amax, const double* __restrict__ amin,
                             const float* __restrict__ bmax, const double* __restrict__ bmin, int G,
                             int tiles_m, int tiles_n, uint8_t* __restrict__ flags) {
  const int64_t id = (int64_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  const int lane = threadIdx.x & 31;
  if (id >= (int64_t)tiles_m * tiles_n) return;
  const int m = (int)(id / tiles_n), nb = (int)(id - (int64_t)m * tiles_n);
  const int64_t row0 = (int64_t)m * BM, col0 = (int64_t)nb * LIST_BN;
  bool keep;
  if (col0 + LIST_BN - 1 < row0) {
    keep = false;                                   // below the diagonal: never enumerated
  } else if (col0 < row0 + BM) {
    keep = true;                                    // straddles the diagonal
  } else {
    double u = 0.0;                                 // fp32 x fp32 is exact in fp64
    for (int g = lane; g < G; g += 32)
      u = __fma_ru((double)amax[(int64_t)m * G + g], (double)bmax[(int64_t)nb * G + g], u);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) u = __dadd_ru(u, __shfl_xor_sync(0xffffffffu, u, o));
    const double l = fmin(amin[m], bmin[nb]);
    keep = !(__dmul_ru(u, 1.0 + BOUND_EPS) < __dmul_rd(l, 1.0 - BOUND_EPS));
  }
  if (lane == 0) flags[id] = keep ? 1 : 0;
}

// One block: the flagged tiles in the rasterised order of the symmetric launch (TileCursor), packed
// m << 16 | n, their number in *count and the number of upper tiles in *total.
__global__ void k_tile_compact(const uint8_t* __restrict__ flags, int tiles_m, int tiles_n,
                               uint32_t* __restrict__ list, int* __restrict__ count,
                               int* __restrict__ total) {
  __shared__ int warp_tot[32];
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5, nw = blockDim.x >> 5;
  int base = 0, all = 0;
  const int groups = (tiles_m + GROUP_M - 1) / GROUP_M;
  for (int g = 0; g < groups; ++g) {
    const int nb0 = sym_first_nblk<LIST_BN>(g);
    const int span = (tiles_n - nb0) * GROUP_M;
    for (int c0 = 0; c0 < span; c0 += blockDim.x) {
      const int idx = c0 + (int)threadIdx.x;
      bool valid = false, keep = false;
      int m = 0, nb = 0;
      if (idx < span) {
        nb = nb0 + idx / GROUP_M;
        const int mi = idx % GROUP_M;
        valid = mi < sym_valid_mblocks<LIST_BN>(g, nb, tiles_m);
        m = g * GROUP_M + mi;
        keep = valid && flags[(int64_t)m * tiles_n + nb];
      }
      const unsigned bal = __ballot_sync(0xffffffffu, keep);
      if (lane == 0) warp_tot[w] = __popc(bal);
      __syncthreads();
      int off = 0, tot = 0;
      for (int i = 0; i < nw; ++i) {
        const int v = warp_tot[i];
        off += i < w ? v : 0;
        tot += v;
      }
      if (keep) list[base + off + __popc(bal & ((1u << lane) - 1u))] = ((uint32_t)m << 16) | nb;
      base += tot;
      all += __syncthreads_count(valid);            // also the barrier before warp_tot is reused
    }
  }
  if (threadIdx.x == 0) {
    *count = base;
    *total = all;
  }
}

int diffuse_tile_list(const float* norms, int G, const double* diag_lb, const int* perm,
                      int64_t n, uint32_t* list, int* count, int* total, cudaStream_t st) {
  SC_REQUIRE(n > 0 && n <= BOUND_MAX_K && G == (n + 255) / 256,
             "sc_diffuse_tile_list: n must lie in [1, 2^20] and G = ceil(n / 256)");
  const int tiles_m = (int)((n + BM - 1) / BM), tiles_n = (int)((n + LIST_BN - 1) / LIST_BN);
  Scratch amax, bmax, amin, bmin, flags;
  SC_CUDA(amax.alloc(sizeof(float) * tiles_m * G, st));
  SC_CUDA(bmax.alloc(sizeof(float) * tiles_n * G, st));
  SC_CUDA(amin.alloc(sizeof(double) * tiles_m, st));
  SC_CUDA(bmin.alloc(sizeof(double) * tiles_n, st));
  SC_CUDA(flags.alloc((size_t)tiles_m * tiles_n, st));
  k_block_bounds<<<tiles_m, 256, 0, st>>>(norms, G, diag_lb, perm, (int)n, BM, amax.as<float>(),
                                          amin.as<double>());
  k_block_bounds<<<tiles_n, 256, 0, st>>>(norms, G, diag_lb, perm, (int)n, LIST_BN,
                                          bmax.as<float>(), bmin.as<double>());
  const int64_t tiles = (int64_t)tiles_m * tiles_n;
  k_tile_flags<<<(unsigned)((tiles + 7) / 8), 256, 0, st>>>(
      amax.as<float>(), amin.as<double>(), bmax.as<float>(), bmin.as<double>(), G, tiles_m, tiles_n,
      flags.as<uint8_t>());
  k_tile_compact<<<1, 1024, 0, st>>>(flags.as<uint8_t>(), tiles_m, tiles_n, list, count, total);
  sc::launched(4);
  SC_LAUNCH_CHECK();
  return 0;
}

// ---- hub-first bounded Diffuse (DESIGN.md section 3).  The rows are ordered cluster by cluster,
// each cluster's row of largest diagonal (its hub) first; starts[c] is the first row of cluster c in
// that order, starts[k] = n.  Phase 1 computes, for every non-empty cluster [s, e), the tiles of the
// hub's row block against the column blocks that hold its rows: every row of the cluster then has
// its element with the hub folded into its maximum L_i.  Phase 2 keeps a tile iff it straddles the
// diagonal or some row i of it has (1 + eps) u_iJ >= L_i, u_iJ = sum_g |y_i^g| max_{j in J} |y_j^g|
// (or some column j the same with the roles swapped), and phase 1 did not compute it.
__device__ __forceinline__ bool is_hub_tile(int m, int c, const int* __restrict__ starts, int k) {
  for (int q = 0; q < k; ++q) {
    const int s = starts[q], e = starts[q + 1];
    if (e > s && s / BM == m && s / LIST_BN <= c && c <= (e - 1) / LIST_BN) return true;
  }
  return false;
}

// flags[m tiles_n + c]: phase 1 (rule_row == nullptr) = the hub tiles; phase 2 = the straddling
// tiles and those the row rule keeps, minus the hub tiles.  Tiles below the diagonal are never read.
__global__ void k_hub_tile_flags(const int* __restrict__ starts, int k, int tiles_m, int tiles_n,
                                 const uint8_t* __restrict__ rule_row,
                                 const uint8_t* __restrict__ rule_col, uint8_t* __restrict__ flags) {
  const int64_t id = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (id >= (int64_t)tiles_m * tiles_n) return;
  const int m = (int)(id / tiles_n), c = (int)(id - (int64_t)m * tiles_n);
  const bool hub = is_hub_tile(m, c, starts, k);
  bool keep;
  if (rule_row == nullptr)
    keep = hub;
  else if (hub || (int64_t)c * LIST_BN + LIST_BN - 1 < (int64_t)m * BM)
    keep = false;
  else
    keep = (int64_t)c * LIST_BN < (int64_t)m * BM + BM || rule_row[id] ||
           rule_col[(int64_t)c * tiles_m + m];
  flags[id] = keep ? 1 : 0;
}

// The per-row rule as one dense product over the permuted rows: CTA (b, t0) takes the R rows of
// block b and the other side's blocks t0 .. t0 + 31, whose group-norm maxima are omax [T, G].
// out[b T + t] = 1 iff some row i of block b has (1 + eps) sum_g |y_i^g| omax[t][g] >= L_i (fp64,
// every operation rounded up; L_i = rowmax[perm[i]] exactly).  row_side: block b is a row block
// (R = 128) against column blocks (192); otherwise a column block against row blocks.  Only the
// pairs that form a tile wholly above the diagonal are wanted; CTAs without one return at once.
constexpr int RULE_T = 32, RULE_GC = 32;

template <int R>
__global__ void __launch_bounds__(256) k_row_rule(const float* __restrict__ norms, int G,
                                                  const int* __restrict__ perm, int n,
                                                  const float* __restrict__ rowmax,
                                                  const float* __restrict__ omax, int T,
                                                  bool row_side, uint8_t* __restrict__ out) {
  constexpr int RO = (R == BM) ? LIST_BN : BM;      // rows per block of the other side
  constexpr int RQ = R / 16;                        // rows per thread
  __shared__ float sn[R][RULE_GC + 1];
  __shared__ float so[RULE_GC][RULE_T];
  __shared__ int fl[RULE_T];
  const int b = blockIdx.x, t0 = blockIdx.y * RULE_T;
  // wanted pair (b, t): row side  RO t >= R b + R;  column side  R b >= RO t + RO
  const bool any = row_side ? (int64_t)RO * min(T - 1, t0 + RULE_T - 1) >= (int64_t)R * b + R
                            : (int64_t)R * b >= (int64_t)RO * t0 + RO;
  if (!any) return;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  if (threadIdx.x < RULE_T) fl[threadIdx.x] = 0;
  double acc[RQ][2];
#pragma unroll
  for (int q = 0; q < RQ; ++q) acc[q][0] = acc[q][1] = 0.0;
  for (int g0 = 0; g0 < G; g0 += RULE_GC) {
    __syncthreads();
    for (int e = threadIdx.x; e < R * RULE_GC; e += blockDim.x) {
      const int r = e / RULE_GC, g = g0 + e % RULE_GC;
      const int i = b * R + r;
      sn[r][e % RULE_GC] = (i < n && g < G) ? norms[(int64_t)perm[i] * G + g] : 0.f;
    }
    for (int e = threadIdx.x; e < RULE_T * RULE_GC; e += blockDim.x) {
      const int t = e / RULE_GC, g = g0 + e % RULE_GC;
      so[e % RULE_GC][t] = (t0 + t < T && g < G) ? omax[(int64_t)(t0 + t) * G + g] : 0.f;
    }
    __syncthreads();
#pragma unroll 4
    for (int g = 0; g < RULE_GC; ++g) {
      const double o0 = (double)so[g][tx], o1 = (double)so[g][tx + 16];
#pragma unroll
      for (int q = 0; q < RQ; ++q) {
        const double v = (double)sn[ty + 16 * q][g];
        acc[q][0] = __fma_ru(v, o0, acc[q][0]);
        acc[q][1] = __fma_ru(v, o1, acc[q][1]);
      }
    }
  }
  bool k0 = false, k1 = false;
#pragma unroll
  for (int q = 0; q < RQ; ++q) {
    const int i = b * R + ty + 16 * q;
    if (i < n) {
      const double l = (double)rowmax[perm[i]];
      k0 |= !(__dmul_ru(acc[q][0], 1.0 + BOUND_EPS) < l);
      k1 |= !(__dmul_ru(acc[q][1], 1.0 + BOUND_EPS) < l);
    }
  }
  if (k0) fl[tx] = 1;
  if (k1) fl[tx + 16] = 1;
  __syncthreads();
  if (threadIdx.x < RULE_T && t0 + (int)threadIdx.x < T)
    out[(int64_t)b * T + t0 + threadIdx.x] = (uint8_t)fl[threadIdx.x];
}

int diffuse_hub_tiles(const int* starts, int k, int64_t n, uint32_t* list, int* count,
                      cudaStream_t st) {
  SC_REQUIRE(n > 0 && n <= BOUND_MAX_K && k >= 1 && k <= 16,
             "sc_diffuse_hub_tiles: n must lie in [1, 2^20] and k in [1, 16]");
  const int tiles_m = (int)((n + BM - 1) / BM), tiles_n = (int)((n + LIST_BN - 1) / LIST_BN);
  const int64_t tiles = (int64_t)tiles_m * tiles_n;
  Scratch flags, total;
  SC_CUDA(flags.alloc((size_t)tiles, st));
  SC_CUDA(total.alloc(sizeof(int), st));
  k_hub_tile_flags<<<(unsigned)((tiles + 255) / 256), 256, 0, st>>>(starts, k, tiles_m, tiles_n,
                                                                   nullptr, nullptr,
                                                                   flags.as<uint8_t>());
  k_tile_compact<<<1, 1024, 0, st>>>(flags.as<uint8_t>(), tiles_m, tiles_n, list, count,
                                     total.as<int>());
  sc::launched(2);
  SC_LAUNCH_CHECK();
  return 0;
}

int diffuse_tile_list_rows(const float* norms, int G, const int* perm, int64_t n,
                           const float* rowmax, const int* starts, int k, uint32_t* list,
                           int* count, int* total, cudaStream_t st) {
  SC_REQUIRE(n > 0 && n <= BOUND_MAX_K && G == (n + 255) / 256 && k >= 1 && k <= 16,
             "sc_diffuse_tile_list_rows: n must lie in [1, 2^20], G = ceil(n / 256), k in [1, 16]");
  const int tiles_m = (int)((n + BM - 1) / BM), tiles_n = (int)((n + LIST_BN - 1) / LIST_BN);
  const int64_t tiles = (int64_t)tiles_m * tiles_n;
  Scratch amax, bmax, amin, bmin, diag0, rule_row, rule_col, flags;
  SC_CUDA(amax.alloc(sizeof(float) * tiles_m * G, st));
  SC_CUDA(bmax.alloc(sizeof(float) * tiles_n * G, st));
  SC_CUDA(amin.alloc(sizeof(double) * tiles_m, st));
  SC_CUDA(bmin.alloc(sizeof(double) * tiles_n, st));
  SC_CUDA(diag0.alloc(sizeof(double) * n, st));
  SC_CUDA(rule_row.alloc((size_t)tiles, st));
  SC_CUDA(rule_col.alloc((size_t)tiles, st));
  SC_CUDA(flags.alloc((size_t)tiles, st));
  // the block maxima of the norms (the block minima of k_block_bounds are not used here: a zeroed
  // diagonal stands in for them)
  SC_CUDA(cudaMemsetAsync(diag0.p, 0, sizeof(double) * n, st));
  k_block_bounds<<<tiles_m, 256, 0, st>>>(norms, G, diag0.as<double>(), perm, (int)n, BM,
                                          amax.as<float>(), amin.as<double>());
  k_block_bounds<<<tiles_n, 256, 0, st>>>(norms, G, diag0.as<double>(), perm, (int)n, LIST_BN,
                                          bmax.as<float>(), bmin.as<double>());
  k_row_rule<BM><<<dim3(tiles_m, (tiles_n + RULE_T - 1) / RULE_T), 256, 0, st>>>(
      norms, G, perm, (int)n, rowmax, bmax.as<float>(), tiles_n, true, rule_row.as<uint8_t>());
  k_row_rule<LIST_BN><<<dim3(tiles_n, (tiles_m + RULE_T - 1) / RULE_T), 256, 0, st>>>(
      norms, G, perm, (int)n, rowmax, amax.as<float>(), tiles_m, false, rule_col.as<uint8_t>());
  k_hub_tile_flags<<<(unsigned)((tiles + 255) / 256), 256, 0, st>>>(
      starts, k, tiles_m, tiles_n, rule_row.as<uint8_t>(), rule_col.as<uint8_t>(),
      flags.as<uint8_t>());
  k_tile_compact<<<1, 1024, 0, st>>>(flags.as<uint8_t>(), tiles_m, tiles_n, list, count, total);
  sc::launched(6);
  SC_LAUNCH_CHECK();
  return 0;
}

int diffuse_rowmax_tiles(const sc_context* ctx, const __half* y_hi, int64_t ldh, int64_t n,
                         const uint32_t* list, const int* count, const int* row_map,
                         float* rowmax, bool fold, cudaStream_t st) {
  SC_REQUIRE(n > 0 && n <= BOUND_MAX_K, "sc_diffuse_rowmax_tiles: n must lie in [1, 2^20]");
  constexpr int PREC = 1, BN = LIST_BN;
  constexpr int STAGES = StageGeom<PREC, BN>::STAGES;
  constexpr int STAGE_BYTES = StageGeom<PREC, BN>::BYTES;
  CUtensorMap ah, bh;
  if (int r = make_plane_map(&ah, y_hi, n, n, ldh, BM)) return r;
  if (int r = make_plane_map(&bh, y_hi, n, n, ldh, BN)) return r;
  const size_t smem = (size_t)STAGES * STAGE_BYTES + 1024 /*align*/ + 256 /*barriers*/;
  SC_REQUIRE(smem <= ctx->smem_optin, "wgmma GEMM needs %zu B of shared memory", smem);
  auto kern = k_gemm_wgmma<PREC, TC_EPI_PLAIN, true, BN, true>;
  SC_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  if (!fold) SC_CUDA(cudaMemsetAsync(rowmax, 0, sizeof(float) * n, st));
  int grid = ctx->sm_count;
  if (ctx->gemm_sm_limit > 0 && ctx->gemm_sm_limit < grid) grid = ctx->gemm_sm_limit;
  // the tile count is on the device: pace whenever K is long enough (CTAs without a tile sign off
  // their checkpoints, as in the last round of the enumerated launch)
  unsigned int* pace = nullptr;
  if (ctx->gemm_pace && (n + BK - 1) / BK >= 2 * PACE_KB) {
    static std::atomic<unsigned int> pace_turn{0};
    pace = ctx->gemm_pace + (pace_turn.fetch_add(1) % SC_GEMM_PACE_SLOTS);
    SC_CUDA(cudaMemsetAsync(pace, 0, sizeof(unsigned int), st));
  }
  TileTable tab = {};
  kern<<<grid, NUM_THREADS, smem, st>>>(ah, ah, bh, bh, tab, (int)n, (int)n, (int)n, nullptr, 0,
                                        nullptr, 0, pace, PACE_KB, rowmax, nullptr, nullptr, 0, 1,
                                        list, count, row_map);
  sc::launched();
  SC_LAUNCH_CHECK();
  return 0;
}

}  // namespace sc
