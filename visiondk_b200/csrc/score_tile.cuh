// score_tile.cuh — the fp16 wgmma mainloop shared by retrieval's score kernel (retrieval.cu) and the DBSCAN Gram passes
// (cluster.cu): a 128-row A block resident in shared memory (kTileKB-wide K blocks, one per 64 columns of dim), 256-row B
// tiles streamed by TMA through a kTileStages-deep mbarrier ring, two consumer warpgroups of 64 rows each accumulating a
// 64 x 256 fp32 tile in registers, and the staging of the accumulator through shared memory 64 columns at a time.
#pragma once
#include "vdk_ptx.cuh"

namespace vdk {

constexpr int kTileM = 128;                            // A rows per tile (two consumer warpgroups)
constexpr int kTileN = 256;                            // B rows per tile (wgmma N)
constexpr int kTileKB = 64;                            // K per shared-memory block (one 128-byte swizzle row of fp16)
constexpr int kTileABlockBytes = kTileM * kTileKB * 2;  // 16 KB
constexpr int kTileBStageBytes = kTileN * kTileKB * 2;  // 32 KB
constexpr int kTileStages = 2;
constexpr int kTileStageLd = kTileKB + 1;               // fp32 pitch of a staged 128 x 64 chunk (odd: conflict-free row reads)

// Producer (one thread): B tiles t_lo .. t_hi - 1, tile t at row b_row0 + t * kTileN of `map_b`, through the ring.
__device__ __forceinline__ void tile_produce_b(uint8_t* smem_b, const CUtensorMap* map_b, uint64_t* full_bar, uint64_t* empty_bar,
                                               int num_kb, int b_row0, int t_lo, int t_hi, int& stage, uint32_t& phase) {
  for (int t = t_lo; t < t_hi; ++t) {
    const int row = b_row0 + t * kTileN;
    for (int kb = 0; kb < num_kb; ++kb) {
      mbar_wait<true>(&empty_bar[stage], phase ^ 1);
      mbar_arrive_expect_tx(&full_bar[stage], kTileBStageBytes);
      tma_load_2d(smem_b + stage * kTileBStageBytes, map_b, &full_bar[stage], kb * kTileKB, row, kEvictNormal);
      if (++stage == kTileStages) {
        stage = 0;
        phase ^= 1;
      }
    }
  }
}

// Consumer warpgroup cg: acc = A[64 cg .. 64 cg + 63] . B tile^T over num_kb K blocks.  Every stage is handed back to the
// producer (one arrival per warp) once the MMAs reading it have retired; on return all of this tile's MMAs have retired.
__device__ __forceinline__ void tile_mma(float (&acc)[kTileN / 2], const uint8_t* smem_a, const uint8_t* smem_b, uint64_t* full_bar,
                                         uint64_t* empty_bar, int num_kb, int cg, int lane, int& stage, uint32_t& phase) {
  int prev = -1;
  for (int kb = 0; kb < num_kb; ++kb) {
    mbar_wait<true>(&full_bar[stage], phase);
    const uint64_t da = wgmma_desc_k_sw128(smem_u32(smem_a + kb * kTileABlockBytes) + cg * 8192);
    const uint64_t db = wgmma_desc_k_sw128(smem_u32(smem_b + stage * kTileBStageBytes));
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < kTileKB / 16; ++k)
      wgmma_m64n256k16_ss<false, 0, 0>(acc, da + 2 * k, db + 2 * k, (kb | k) != 0 ? 1u : 0u);
    wgmma_commit();
    wgmma_wait<1>();
    if (prev >= 0 && lane == 0) mbar_arrive(&empty_bar[prev]);
    prev = stage;
    if (++stage == kTileStages) {
      stage = 0;
      phase ^= 1;
    }
  }
  wgmma_wait<0>();
  wgmma_fence_regs(acc);
  if (lane == 0) mbar_arrive(&empty_bar[prev]);
}

// Columns 64 cc .. 64 cc + 63 of the accumulator into the staging chunk [kTileM][kTileStageLd] (score bits); (frow, fcol): the
// thread's fragment row and column (vdk_wgmma.cuh's layout).
__device__ __forceinline__ void tile_stage_chunk(uint32_t* stage_sm, const float (&acc)[kTileN / 2], int cc, int frow, int fcol) {
#pragma unroll
  for (int jj = 0; jj < 8; ++jj) {
    const int j = cc * 8 + jj;
    stage_sm[frow * kTileStageLd + jj * 8 + fcol] = __float_as_uint(acc[4 * j]);
    stage_sm[frow * kTileStageLd + jj * 8 + fcol + 1] = __float_as_uint(acc[4 * j + 1]);
    stage_sm[(frow + 8) * kTileStageLd + jj * 8 + fcol] = __float_as_uint(acc[4 * j + 2]);
    stage_sm[(frow + 8) * kTileStageLd + jj * 8 + fcol + 1] = __float_as_uint(acc[4 * j + 3]);
  }
}

}  // namespace vdk
