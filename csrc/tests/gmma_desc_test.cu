// Cross-check of the hand-packed wgmma shared-memory descriptor in csrc/kernels/gemm_bnstats.cu against the CuTe
// definitions (cute/arch/mma_sm90_desc.hpp, cute/atom/mma_traits_sm90_gmma.hpp from the CUTLASS headers). Host only.
// `make test_gmma_desc CUTLASS_INC=<cutlass include dir>`; tests/test_native_cpu.py runs it when the headers are present.
#include <cstdio>

#include <cute/tensor.hpp>
#include <cute/arch/mma_sm90_desc.hpp>
#include <cute/atom/mma_traits_sm90_gmma.hpp>

#include "../kernels/gemm_bnstats.cu"

using namespace cute;

int main() {
  int failed = 0;
  auto check = [&](const char* what, unsigned long long got, unsigned long long want) {
    printf("%-40s ours %016llx  want %016llx %s\n", what, got, want, got == want ? "ok" : "MISMATCH");
    if (got != want) failed++;
  };
  using bf16 = cutlass::bfloat16_t;
  // canonical K-major 128-byte-swizzle tile, the layout TMA (CU_TENSOR_MAP_SWIZZLE_128B, 64-element inner box) writes;
  // each warpgroup's A operand is a [64 x 64] half of the [128 x 64] stage, B is [BN x 64]
  alignas(1024) static bf16 tile[128 * 64];
  auto a128 = make_tensor(make_smem_ptr(tile), tile_to_shape(GMMA::Layout_K_SW128_Atom<bf16>{}, Shape<_128, _64>{}));
  auto a64 = make_tensor(make_smem_ptr(tile), tile_to_shape(GMMA::Layout_K_SW128_Atom<bf16>{}, Shape<_64, _64>{}));
  // one wgmma reads a K = 16 slice of the tile (CuTe's canonical GMMA_K layout)
  const unsigned long long addr_mask = ~0x3FFFull;   // the start-address field depends on the run-time address
  check("smem desc [64 x 64] (no addr)", b200mpi::gemm::make_desc_kmajor_sw128(0) & addr_mask, GMMA::make_gmma_desc<GMMA::Major::K>(local_tile(a64, Shape<_64, _16>{}, make_coord(0, 0))).desc_ & addr_mask);
  check("smem desc [128 x 64] (no addr)", b200mpi::gemm::make_desc_kmajor_sw128(0) & addr_mask, GMMA::make_gmma_desc<GMMA::Major::K>(local_tile(a128, Shape<_128, _16>{}, make_coord(0, 0))).desc_ & addr_mask);
  // self-checks against the PTX ISA encoding (CuTe cannot take a shared-memory address on the host): start address >> 4 in
  // bits [0,14), and one K = 16 slice of bf16 (32 bytes inside the swizzle atom) is +2 in that field
  check("address field (self-check, not CuTe)", b200mpi::gemm::make_desc_kmajor_sw128(0x2A400) & 0x3FFFull, 0x2A40ull);
  check("K advance +32 B (self-check, not CuTe)", (b200mpi::gemm::make_desc_kmajor_sw128(0x400) + 2) & 0x3FFFull, (0x400ull + 32) >> 4);
  // the epilogue writes the bf16 tile into shared memory by hand in the 128-byte-swizzle layout the TMA store expects:
  //   byte offset(row r, column j) = r*128 + ((j/8) ^ (r & 7))*16 + (j % 8)*2     (gemm_bnstats.cu, epilogue + column sums)
  {
    // CuTe applies Sw<3,4,3> to the byte address of the (1024-byte aligned) tile: compare real element addresses
    long bad = 0;
    const char* base = reinterpret_cast<const char*>(&a128(0, 0));
    for (int r = 0; r < 128; r++)
      for (int j = 0; j < 64; j++) {
        const unsigned long long theirs = (unsigned long long)(reinterpret_cast<const char*>(&a128(r, j)) - base);
        if (b200mpi::gemm::operand_elem_byte(r, j) != theirs) bad++;              // operand tiles as TMA writes them
        if (b200mpi::gemm::stage_elem_byte(j, r) != theirs) bad++;                // output staging, first 64-column box
        if (b200mpi::gemm::stage_elem_byte(64 + j, r) != theirs + b200mpi::gemm::kBoxBytes) bad++;   // second box
        if ((j & 7) == 0 && b200mpi::gemm::stage_group_byte(r, j >> 5, (j >> 3) & 3) != theirs) bad++;   // 16-byte groups
      }
    check("swizzled tile offsets (mismatches)", (unsigned long long)bad, 0);
  }
  printf(failed ? "gmma_desc_test: %d MISMATCH(ES)\n" : "gmma_desc_test: descriptors match CuTe\n", failed);
  return failed ? 1 : 0;
}
