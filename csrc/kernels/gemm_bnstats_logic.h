// Index and phase arithmetic of the wgmma GEMM + BN-statistics kernel (gemm_bnstats.cu), shared verbatim between the
// kernel and its host model (csrc/tests/gemm_pipeline_model.cc): pipeline ring state, persistent tile walk, the
// 128-byte-swizzled layout of the output staging buffer and the addressing of the per-CTA partial rows.
#pragma once
#include <stddef.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define B200_HD __host__ __device__ __forceinline__
#else
#define B200_HD inline
#endif

namespace b200mpi {
namespace gemm {

constexpr int BM = 128;          // rows per tile: two warpgroups x wgmma M = 64
constexpr int BK = 64;           // 64 bf16 = 128 bytes = one swizzle-128B row
constexpr int MMA_K = 16;        // K per wgmma.mma_async for 16-bit inputs
constexpr int kStages = 4;
constexpr uint32_t kBoxBytes = BM * 128;   // one TMA store box: 128 rows x 64 bf16

// stage index + phase bit of an mbarrier ring of n slots
struct Ring {
  int s = 0;
  uint32_t ph = 0;
  B200_HD void advance(int n) {
    if (++s == n) { s = 0; ph ^= 1u; }
  }
};

// Persistent schedule: CTA `cta` of `grid` owns column block cta % num_n for the whole kernel and visits the row blocks
// m_first, m_first + m_step, ... (< num_m); its column sums go to partial row m_first.
struct TileWalk {
  int n_blk, m_first, m_step, num_m;
  B200_HD TileWalk(int cta, int grid, int num_n, int M)
      : n_blk(cta % num_n), m_first(cta / num_n), m_step(grid / num_n), num_m((M + BM - 1) / BM) {}
};

// Staging buffer = BN/64 boxes of [128 rows x 64 bf16], each laid out the way a SWIZZLE_128B tensor map expects it:
// the 16-byte chunk index inside a 128-byte row is XORed with (row & 7).
// Byte offset of the 16-byte group holding tile row `row`, columns [32*c32 + 8*g, 32*c32 + 8*g + 8):
B200_HD uint32_t stage_group_byte(int row, int c32, int g) {
  const uint32_t lc = (uint32_t)((c32 & 1) * 4 + g);          // logical chunk inside the 64-column box
  return (uint32_t)(c32 >> 1) * kBoxBytes + (uint32_t)row * 128u + ((lc ^ (uint32_t)(row & 7)) << 4);
}
// Byte offset of element (row r, tile column col):
B200_HD uint32_t stage_elem_byte(int col, int r) {
  return (uint32_t)(col >> 6) * kBoxBytes + (uint32_t)r * 128u + ((((uint32_t)(col & 63) >> 3) ^ (uint32_t)(r & 7)) << 4) +
         (uint32_t)(col & 7) * 2u;
}
// Same layout for the operand tiles TMA writes (K-major, 64 elements = 128 bytes per row): element (r, k)
B200_HD uint32_t operand_elem_byte(int r, int k) {
  return (uint32_t)r * 128u + ((((uint32_t)k >> 3) ^ (uint32_t)(r & 7)) << 4) + (uint32_t)(k & 7) * 2u;
}
// partials[m_first][2 * global_column + {0: sum, 1: sum of squares}]
B200_HD size_t partial_index(int m_first, int N, int global_col) { return (size_t)m_first * 2 * (size_t)N + 2 * (size_t)global_col; }

}  // namespace gemm
}  // namespace b200mpi
