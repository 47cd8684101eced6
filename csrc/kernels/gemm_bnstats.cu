// 1x1-convolution GEMM with BatchNorm statistics fused into the epilogue (sm_90a: TMA + wgmma + mbarrier).
//
//   Y[M,N] = X[M,K] . W[N,K]^T      bf16 in, fp32 accumulate in registers, bf16 out   (NHWC activations: M = N*H*W,
//                                                                                       K = Cin, N = Cout, W is the conv
//                                                                                       weight as stored)
//   partials[p][2n+0] += sum_m Y[m,n],  partials[p][2n+1] += sum_m Y[m,n]^2      (one row per CTA m-group, the layout the
//                                                                                  BN finalize kernel of bn_act.cu merges)
//
// Why: two thirds of ResNet's BatchNorm layers follow a 1x1 convolution. Their statistics pass re-reads the whole
// convolution output from HBM; here the tile is still in shared memory when its column sums are taken, so the pass
// disappears. The reference has no kernels at all (SURVEY.md §2.2) — this is part of the data plane the new framework adds.
//
// Structure (warp-specialised Hopper GEMM):
//   warp 8        TMA producer : cp.async.bulk.tensor loads of the X and W tiles (128B swizzle) into a 4-stage ring
//   warps 0..7    two consumer warpgroups; warpgroup g owns rows [64g, 64g+64) of the 128-row tile:
//                   wgmma.mma_async m64nBNk16 (bf16 x bf16 -> fp32 registers), one k-block in flight, each finished
//                   k-block releases its stage to the producer; then registers -> bf16 -> swizzled smem staging ->
//                   TMA store of the tile + column sums of the warpgroup's 64 rows from smem
// The producer runs ahead into the next tile while the consumers are in the epilogue.
// Persistent: CTA c owns column block c % num_n and walks m-blocks with stride grid/num_n, so every consumer thread keeps
// one column's running sums in registers for the whole kernel; the two warpgroups' sums are added in shared memory and
// a single partial row is written at the end (no atomics). Every wait is bounded and traps instead of hanging.
#include <cuda.h>
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include "../include/b200mpi.h"
#include "gemm_bnstats_logic.h"

namespace b200mpi {
namespace gemm {

constexpr int kConsumers = 256;              // two warpgroups
constexpr int kThreads = kConsumers + 32;    // + the TMA producer warp
constexpr int kMaxParts = 132;               // partial rows: at most one per SM (H100 SXM: 132 SMs)
constexpr uint32_t kABytes = BM * BK * 2;    // 16 KiB
constexpr long long kTimeoutCycles = 6000000000LL;  // ~3 s: a broken pipeline traps instead of hanging the GPU

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return static_cast<uint32_t>(__cvta_generic_to_shared(p)); }

// ---------------------------------------------------------------- mbarrier ----
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok;
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
      "selp.u32 %0, 1, 0, p;\n\t"
      "}"
      : "=r"(ok)
      : "r"(bar), "r"(parity)
      : "memory");
  return ok != 0;
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  if (mbar_try_wait(bar, parity)) return;
  const long long t0 = clock64();
  while (!mbar_try_wait(bar, parity)) {
    if (clock64() - t0 > kTimeoutCycles) asm volatile("trap;");
  }
}

// --------------------------------------------------------------------- TMA ----
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];" ::"r"(dst),
               "l"(reinterpret_cast<uint64_t>(map)), "r"(bar), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, uint32_t src, int c0, int c1) {
  asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];" ::"l"(reinterpret_cast<uint64_t>(map)),
               "r"(src), "r"(c0), "r"(c1)
               : "memory");
}
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(map)) : "memory");
}

// ------------------------------------------------------------------- wgmma ----
// Shared-memory matrix descriptor, K-major operand, 128-byte swizzle (cute/arch/mma_sm90_desc.hpp: GmmaDescriptor):
//   [0,14) start address >> 4 | [16,30) leading byte offset >> 4 (=1: unused for swizzled K-major) |
//   [32,46) stride byte offset >> 4 (=64: 8 rows x 128 B between core-matrix groups) | [49,52) base offset = 0 (every
//   operand tile starts on a 1024-byte swizzle atom) | [62,64) layout = 1 (SWIZZLE_128B)
__host__ __device__ __forceinline__ uint64_t make_desc_kmajor_sw128(uint32_t smem_addr) {
  return (uint64_t)((smem_addr >> 4) & 0x3FFFu) | ((uint64_t)1 << 16) | ((uint64_t)64 << 32) | ((uint64_t)1 << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }

// D[64 x BN] (+)= A[64 x 16] . B[BN x 16]^T, both operands K-major in swizzled smem. Accumulator fragment of thread
// (warp w of the warpgroup, lane l): d[4j + 2i + c] = D[16w + l/4 + 8i][8j + 2(l%4) + c]
template <int BN>
__device__ __forceinline__ void wgmma_bf16(float (&d)[BN / 2], uint64_t adesc, uint64_t bdesc, uint32_t accumulate);
template <>
__device__ __forceinline__ void wgmma_bf16<128>(float (&d)[64], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, "
      "%25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
      "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t"
      "}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
        "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),
        "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),
        "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]),
        "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]),
        "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]),
        "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(adesc), "l"(bdesc), "r"(accumulate)
      : "memory");
}

template <>
__device__ __forceinline__ void wgmma_bf16<64>(float (&d)[32], uint64_t adesc, uint64_t bdesc, uint32_t accumulate) {
  asm volatile(
      "{\n\t"
      ".reg .pred p;\n\t"
      "setp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k16.f32.bf16.bf16 "
      "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, "
      "%25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t"
      "}"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]),
        "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]),
        "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]),
        "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(adesc), "l"(bdesc), "r"(accumulate)
      : "memory");
}
__device__ __forceinline__ void cons_bar_sync() { asm volatile("bar.sync 1, %0;" ::"n"(kConsumers) : "memory"); }

__device__ __forceinline__ uint32_t pack_bf16(float lo, float hi) {
  __nv_bfloat162 h = __floats2bfloat162_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&h);
}

template <int BN>
struct Smem {
  static constexpr uint32_t kBBytes = BN * BK * 2;
  static constexpr uint32_t kStageBytes = kABytes + kBBytes;
  static constexpr uint32_t kOutBoxes = BN / 64;                  // TMA store boxes of [128 rows x 64 cols] (128 B inner)
  static constexpr uint32_t kOutBytes = kOutBoxes * kBoxBytes;
  static constexpr uint32_t kA = 0;
  static constexpr uint32_t kB = kStages * kABytes;
  static constexpr uint32_t kOut = kB + kStages * kBBytes;
  static constexpr uint32_t kSums = kOut + kOutBytes;             // [BN][2] fp32: warpgroup 1's column sums
  static constexpr uint32_t kBars = kSums + BN * 8;               // full[S], empty[S]
  static constexpr uint32_t kTotal = kBars + 2 * kStages * 8;
  static constexpr uint32_t kDynamic = kTotal + 1024;             // slack to align the base to 1024 B (swizzle atoms)
};

template <int BN>
__global__ void __launch_bounds__(kThreads, 1)
k_gemm_bnstats(const __grid_constant__ CUtensorMap tmX, const __grid_constant__ CUtensorMap tmW, const __grid_constant__ CUtensorMap tmY,
               float* __restrict__ partials, int M, int N, int K, int num_n) {
  using L = Smem<BN>;
  extern __shared__ uint8_t smem_raw[];
  const uint32_t base = (smem_u32(smem_raw) + 1023u) & ~1023u;
  uint8_t* base_ptr = smem_raw + (base - smem_u32(smem_raw));
  const uint32_t sA = base + L::kA, sB = base + L::kB, sOut = base + L::kOut, sBar = base + L::kBars;
  float* sums = reinterpret_cast<float*>(base_ptr + L::kSums);
  auto full_bar = [&](int s) { return sBar + 8u * s; };
  auto empty_bar = [&](int s) { return sBar + 8u * (kStages + s); };

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const TileWalk walk((int)blockIdx.x, (int)gridDim.x, num_n, M);
  const int m_first = walk.m_first, m_step = walk.m_step, num_m = walk.num_m;
  const int num_k = K / BK;
  const int n0 = walk.n_blk * BN;

  if (warp == kConsumers / 32 && lane == 0) {
    tma_prefetch_desc(&tmX);
    tma_prefetch_desc(&tmW);
    tma_prefetch_desc(&tmY);
    for (int s = 0; s < kStages; s++) {
      mbar_init(full_bar(s), 1);                   // producer's arrive.expect_tx (+ the TMA transaction bytes)
      mbar_init(empty_bar(s), kConsumers / 32);    // one arrive per consumer warp once its wgmma has read the stage
    }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();

  if (warp == kConsumers / 32) {
    // ===================================================== TMA producer ====
    if (lane == 0) {
      Ring st;
      for (int m_blk = m_first; m_blk < num_m; m_blk += m_step) {
        for (int kb = 0; kb < num_k; kb++) {
          mbar_wait(empty_bar(st.s), st.ph ^ 1u);
          mbar_arrive_expect_tx(full_bar(st.s), L::kStageBytes);
          tma_load_2d(sA + st.s * kABytes, &tmX, full_bar(st.s), kb * BK, m_blk * BM);
          tma_load_2d(sB + st.s * L::kBBytes, &tmW, full_bar(st.s), kb * BK, n0);
          st.advance(kStages);
        }
      }
    }
    return;
  }

  // =========================================================== consumers ====
  const int ct = threadIdx.x;                  // 0..255
  const int wg = warp >> 2;                    // rows [64 wg, 64 wg + 64) of every tile
  const int t = ct & 127;                      // thread `t` of each warpgroup owns column n0 + t for the statistics
  const bool col_owner = t < BN;
  const int frag_row = wg * 64 + (warp & 3) * 16 + (lane >> 2);
  float s1 = 0.f, s2 = 0.f;
  float d[BN / 2] = {};
  Ring st;
  for (int m_blk = m_first; m_blk < num_m; m_blk += m_step) {
    int prev = 0;
    for (int kb = 0; kb < num_k; kb++) {
      mbar_wait(full_bar(st.s), st.ph);
      wgmma_fence();
      const uint64_t adesc = make_desc_kmajor_sw128(sA + st.s * kABytes + (uint32_t)wg * 64u * 128u);
      const uint64_t bdesc = make_desc_kmajor_sw128(sB + st.s * L::kBBytes);
#pragma unroll
      for (int k = 0; k < BK / MMA_K; k++)  // +32 bytes along K inside the swizzle atom = +2 in the address field
        wgmma_bf16<BN>(d, adesc + (uint64_t)(2 * k), bdesc + (uint64_t)(2 * k), (kb | k) != 0 ? 1u : 0u);
      wgmma_commit();
      wgmma_wait<1>();                         // the previous k-block's MMAs are done reading their stage
      if (kb > 0) {
        __syncwarp();
        if (lane == 0) mbar_arrive(empty_bar(prev));
      }
      prev = st.s;
      st.advance(kStages);
    }
    wgmma_wait<0>();
    __syncwarp();
    if (lane == 0) mbar_arrive(empty_bar(prev));

    if (ct == 0) asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");  // previous tile's store has read the staging
    cons_bar_sync();                                                               // ... and its column sums are taken
    // fp32 fragment -> bf16 pairs in the swizzled staging layout (gemm_bnstats_logic.h)
#pragma unroll
    for (int j = 0; j < BN / 8; j++) {
      const int col = 8 * j + 2 * (lane & 3);
#pragma unroll
      for (int i = 0; i < 2; i++) {
        asm volatile("st.shared.b32 [%0], %1;" ::"r"(sOut + stage_elem_byte(col, frag_row + 8 * i)),
                     "r"(pack_bf16(d[4 * j + 2 * i], d[4 * j + 2 * i + 1]))
                     : "memory");
      }
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic-proxy writes -> visible to the TMA store
    cons_bar_sync();
    if (ct == 0) {
#pragma unroll
      for (int b = 0; b < (int)L::kOutBoxes; b++) tma_store_2d(&tmY, sOut + (uint32_t)b * kBoxBytes, n0 + b * 64, m_blk * BM);
      asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    }
    if (col_owner) {
      // column sums of the bf16-rounded tile (what the BN apply pass will read back). Rows past M are zero-filled by TMA.
#pragma unroll 8
      for (int r = wg * 64; r < wg * 64 + 64; r++) {
        uint16_t h;
        asm volatile("ld.shared.u16 %0, [%1];" : "=h"(h) : "r"(sOut + stage_elem_byte(t, r)));
        const float f = __uint_as_float((uint32_t)h << 16);
        s1 += f;
        s2 = fmaf(f, f, s2);
      }
    }
  }
  if (wg == 1 && col_owner) {
    sums[2 * t] = s1;
    sums[2 * t + 1] = s2;
  }
  cons_bar_sync();
  if (wg == 0 && col_owner && m_first < num_m) {
    float* row_out = partials + partial_index(m_first, N, n0 + t);
    row_out[0] = s1 + sums[2 * t];
    row_out[1] = s2 + sums[2 * t + 1];
  }
  if (ct == 0) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");  // stores landed before the CTA exits
}

// ------------------------------------------------------------------- host ----
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess && q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<EncodeTiledFn>(p);
  }
  return fn;
}

// row-major [rows, cols] bf16 matrix, box = [box_rows, 64 cols] with 128-byte swizzle
static bool make_map(CUtensorMap* map, const void* ptr, uint64_t rows, uint64_t cols, uint32_t box_rows) {
  EncodeTiledFn fn = encode_fn();
  if (!fn) return false;
  const cuuint64_t dims[2] = {cols, rows};              // innermost first
  const cuuint64_t strides[1] = {cols * 2};             // bytes, dims 1..rank-1
  const cuuint32_t box[2] = {64, box_rows};
  const cuuint32_t estr[2] = {1, 1};
  return fn(map, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, 2, const_cast<void*>(ptr), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
            CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE) == CUDA_SUCCESS;
}

static int sm_count() {
  static int n = 0;
  if (!n) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = kMaxParts;
  }
  return n;
}

template <int BN>
static int launch(const void* X, const void* W, void* Y, float* partials, int* parts_out, long long M, int N, int K, cudaStream_t s) {
  CUtensorMap tmX, tmW, tmY;
  if (!make_map(&tmX, X, (uint64_t)M, (uint64_t)K, BM) || !make_map(&tmW, W, (uint64_t)N, (uint64_t)K, BN) ||
      !make_map(&tmY, Y, (uint64_t)M, (uint64_t)N, BM))
    return B200MPI_ERR_CUDA;
  const int num_n = N / BN, num_m = (int)((M + BM - 1) / BM);
  int groups = (sm_count() < kMaxParts ? sm_count() : kMaxParts) / num_n;
  if (groups < 1) return B200MPI_ERR_UNSUPPORTED;
  if (groups > num_m) groups = num_m;
  static bool attr_set = false;
  if (!attr_set) {
    if (cudaFuncSetAttribute(k_gemm_bnstats<BN>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)Smem<BN>::kDynamic) != cudaSuccess)
      return B200MPI_ERR_CUDA;
    attr_set = true;
  }
  k_gemm_bnstats<BN><<<groups * num_n, kThreads, Smem<BN>::kDynamic, s>>>(tmX, tmW, tmY, partials, (int)M, N, K, num_n);
  if (parts_out) *parts_out = groups;
  return cudaGetLastError() == cudaSuccess ? 0 : B200MPI_ERR_CUDA;
}

}  // namespace gemm
}  // namespace b200mpi

extern "C" {

// M >= 128: every shape that ran on hardware had at least one full row tile (ragged tails - M = 196, 1000 - are covered); smaller
// problems (a 2x2 feature map at batch 4) are latency-bound anyway and stay with the library.
int b200mpi_gemm_bnstats_supported(long long M, int N, int K) {
  return (M >= 128 && M < (1LL << 31) - 128 && N >= 64 && N % 64 == 0 && K >= 64 && K % 64 == 0 &&
          N / (N % 128 == 0 ? 128 : 64) <= b200mpi::gemm::kMaxParts) ? 1 : 0;
}

// rows of per-column {sum, sum of squares} the kernel may write: one per m-group, at most one per SM
size_t b200mpi_gemm_bnstats_partial_floats(int N) { return (size_t)b200mpi::gemm::kMaxParts * 2 * (size_t)N; }

// Y = X . W^T (bf16, row-major, X [M,K], W [N,K], Y [M,N], all 16-byte aligned) and partials[parts][2N]; *parts = rows written.
int b200mpi_gemm_bnstats(const void* X, const void* W, void* Y, float* partials, int* parts, long long M, int N, int K, void* stream) {
  using namespace b200mpi::gemm;
  if (!b200mpi_gemm_bnstats_supported(M, N, K)) return B200MPI_ERR_UNSUPPORTED;
  if (((uintptr_t)X | (uintptr_t)W | (uintptr_t)Y) & 15) return B200MPI_ERR_INVALID;
  cudaStream_t s = (cudaStream_t)stream;
  return N % 128 == 0 ? launch<128>(X, W, Y, partials, parts, M, N, K, s) : launch<64>(X, W, Y, partials, parts, M, N, K, s);
}

}  // extern "C"
