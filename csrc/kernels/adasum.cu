// b200mpi Adasum allreduce for sm_90a: ONE kernel per tensor, slice-parallel over NVSwitch peer memory.
//
// Call site it serves (SURVEY.md section 2.5, K6): Horovod's op=hvd.Adasum, the --use-adasum flag of the reference's
// MNIST example (examples/v2beta1/horovod/tensorflow_mnist.py:31-32,126-133). In the reference stack this is Horovod's
// AdasumGpuAllreduceOp: an NCCL reduce-scatter, a host-driven MPI tree with one pair of dot-product allreduces per level,
// and an NCCL allgather. Here the whole tree runs inside one launch:
//
//   adasum(a, b) = (1 - a.b / (2 |a|^2)) a + (1 - a.b / (2 |b|^2)) b        (orthogonal gradients add, parallel ones average)
//
// folded over the ranks by distance doubling (level l combines the vectors of ranks g and g + 2^l, g a multiple of 2^(l+1)).
// Rank r owns slice r of EVERY vector:
//
//   phase 0   user input -> staging copy A (peer-readable), cross-rank barrier
//   level 0   rank r pulls slice r of all `world` copies over NVLink (ld.sys, all loads of a vector in flight), keeps them as
//             fp32 in its local work area W[q], and accumulates the partial (a.b, |a|^2, |b|^2) of the world/2 level-0 pairs
//   per level every CTA pushes its partial sums (fp64) into its own slot [pair][rank][cta] of every rank's dot board; after a
//             FULL barrier (same-index CTAs across ranks + all CTAs of this rank) each CTA adds the board up in a fixed order -
//             identical coefficients, bit for bit, on every CTA of every rank - and combines its part of the slice in W,
//             accumulating the partial dots of the next level in the same pass
//   last level the combined slice is packed back to T and stored into slice r of every rank's A (the all-gather half)
//   phase 2   cross-rank barrier, A -> user output
//
// Traffic per rank: S bytes pulled + S bytes pushed over NVLink (what a two-shot allreduce moves), log2(world) + 2 barriers;
// no host round trip, no O(world * S) gather on every rank as in the Python fallback (hvd/adasum.py). The dot board has one
// slot per (pair, source rank, source CTA) and every slot a launch reads was written in that launch, so nothing has to be
// zeroed between launches. All CTAs of a launch must be co-resident (spin barriers): the host caps the grid at kAdaMaxBlocks.
//
// Status: numerics test (8 / 4 / 2 virtual ranks against the fp64 tree) in tests/test_zzz_adasum_gpu.py, which sorts last
// in the GPU tier. hvd/adasum.py uses it only with B200MPI_ADASUM_KERNEL=1.
#include "kernels.h"

namespace b200mpi {

#define EMU_ARGS const KArgs& a = (emu != nullptr) ? emu[blockIdx.y] : a0

constexpr int kAdaMaxPairs = kMaxRanks / 2;   // pairs alive at one level
constexpr int kAdaWarps = kThreads / 32;

__device__ __forceinline__ double ld_sys_f64(const double* p) {
  double v;
  asm volatile("ld.relaxed.sys.global.f64 %0, [%1];" : "=d"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_sys_f64(double* p, double v) {
  asm volatile("st.relaxed.sys.global.f64 [%0], %1;" ::"l"(p), "d"(v) : "memory");
}
__device__ __forceinline__ uint32_t atom_add_acq_rel_gpu(uint32_t* p, uint32_t v) {
  uint32_t old;
  asm volatile("atom.acq_rel.gpu.global.add.u32 %0, [%1], %2;" : "=r"(old) : "l"(p), "r"(v) : "memory");
  return old;
}

// Barrier between all CTAs of THIS rank's grid (gridDim.x of them): a counter and a generation word in the rank's epoch
// array. The last CTA to arrive resets the counter and bumps the generation; nobody can reach the next instance before it
// has seen the bump, so the pair is reusable without host help (and across launches: a launch always leaves count == 0).
__device__ __forceinline__ void grid_barrier(const DevComm& c) {
  __syncthreads();
  if (threadIdx.x == 0) {
    uint32_t* cnt = c.epoch + kAdaEpochOff;
    uint32_t* gen = cnt + 1;
    const uint32_t g = ld_acquire_gpu(gen);
    if (atom_add_acq_rel_gpu(cnt, 1) == gridDim.x - 1) {
      *reinterpret_cast<volatile uint32_t*>(cnt) = 0;   // ordered before the release below
      st_release_gpu(gen, g + 1);
    } else {
      unsigned long long t0 = 0;
      uint32_t spins = 0;
      while (ld_acquire_gpu(gen) == g) {
        if ((++spins & 0x3ffu) == 0) {
          unsigned long long now = globaltimer_ns();
          if (t0 == 0) t0 = now;
          else if (now - t0 > c.timeout_ns) { *c.err = 1 + c.rank; break; }
        }
      }
    }
  }
  __syncthreads();
}

// CTA-wide sums of `n` (<= 3 * kAdaMaxPairs) per-thread doubles; the results land in out[0..n) (shared) for every thread.
__device__ __forceinline__ void block_sums(double* vals, int n, double (*warp_part)[3 * kAdaMaxPairs], double* out) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int k = 0; k < 3 * kAdaMaxPairs; k++) {   // unrolled with a guard: `vals` stays in registers
    if (k < n) {
      double v = vals[k];
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
      if (lane == 0) warp_part[warp][k] = v;
    }
  }
  __syncthreads();
  if (threadIdx.x < (unsigned)n) {
    double s = 0.0;
    for (int w = 0; w < kAdaWarps; w++) s += warp_part[w][threadIdx.x];
    out[threadIdx.x] = s;
  }
  __syncthreads();
}

template <int VN>
__device__ __forceinline__ void dots3(double* acc, const float* x, const float* y) {
  float d = 0.f, nx = 0.f, ny = 0.f;
#pragma unroll
  for (int j = 0; j < VN; j++) { d = fmaf(x[j], y[j], d); nx = fmaf(x[j], x[j], nx); ny = fmaf(y[j], y[j], ny); }
  acc[0] += (double)d; acc[1] += (double)nx; acc[2] += (double)ny;
}

template <typename T>
__global__ void __launch_bounds__(kThreads)
k_adasum(const __grid_constant__ KArgs a0, const KArgs* __restrict__ emu) {
  EMU_ARGS;
  constexpr int VN = VecTraits<T>::N;       // elements per 16-byte vector
  constexpr int V4 = VN / 4;                // float4s of fp32 work data per vector
  const int rank = a.c.rank, world = a.c.world;
  uint32_t e = a.c.epoch[blockIdx.x];
  const size_t per = a.per, nvec = a.nvec;
  char* const mine = a.buf.p[rank];
  char* const A_mine = mine + kAdaDotBytes;
  float4* const W = reinterpret_cast<float4*>(A_mine + (size_t)world * per * 16);   // [q][per][V4], local only
  const size_t wq = per * V4;               // float4s per work vector

  __shared__ double s_warp[kAdaWarps][3 * kAdaMaxPairs];
  __shared__ double s_part[3 * kAdaMaxPairs];
  __shared__ float s_coef[kAdaMaxPairs][2];

  const size_t t0 = (size_t)blockIdx.x * blockDim.x + threadIdx.x, tstride = (size_t)gridDim.x * blockDim.x;

  // ---- phase 0: user input -> A (every slice; same index -> CTA map as the phases below) ----
  for (int r = 0; r < world; r++) {
    const size_t base = (size_t)r * per;
    const size_t lim = base < nvec ? (nvec - base < per ? nvec - base : per) : 0;
    for (size_t i = t0; i < lim; i += tstride)
      *reinterpret_cast<uint4*>(A_mine + (base + i) * 16) = user_load(a.in, base + i, a.nbytes, a.in_aligned);
  }
  rank_barrier(a.c, ++e);

  const size_t base = (size_t)rank * per;
  const size_t lim = base < nvec ? (nvec - base < per ? nvec - base : per) : 0;
  double acc[3 * kAdaMaxPairs];
#pragma unroll
  for (int k = 0; k < 3 * kAdaMaxPairs; k++) acc[k] = 0.0;

  // ---- level 0 input: slice `rank` of every rank's A -> W[q] (fp32), partial dots of the pairs (2p, 2p+1) ----
  int np = world >> 1;                      // pairs at the current level
  for (size_t i = t0; i < lim; i += tstride) {
    uint4 v[kMaxRanks];
#pragma unroll
    for (int q = 0; q < kMaxRanks; q++)
      if (q < world) v[q] = ld_sys_v4(a.buf.p[q] + kAdaDotBytes + (base + i) * 16);
#pragma unroll
    for (int p = 0; p < kAdaMaxPairs; p++) {
      if (p < np) {
        float x[VN], y[VN];
        VecTraits<T>::unpack(v[2 * p], x);
        VecTraits<T>::unpack(v[2 * p + 1], y);
#pragma unroll
        for (int j = 0; j < V4; j++) {
          W[(size_t)(2 * p) * wq + i * V4 + j] = make_float4(x[4 * j], x[4 * j + 1], x[4 * j + 2], x[4 * j + 3]);
          W[(size_t)(2 * p + 1) * wq + i * V4 + j] = make_float4(y[4 * j], y[4 * j + 1], y[4 * j + 2], y[4 * j + 3]);
        }
        dots3<VN>(acc + 3 * p, x, y);
      }
    }
  }

  int pair_base = 0;                        // index of this level's first pair on the dot board
  for (int dist = 1; dist < world; dist <<= 1) {
    // ---- publish this CTA's partial sums in its slot of every rank's board ----
    block_sums(acc, 3 * np, s_warp, s_part);
    if (threadIdx.x < (unsigned)(3 * np)) {
      const int p = threadIdx.x / 3, k = threadIdx.x - 3 * p;
      const size_t slot = (((size_t)(pair_base + p) * kMaxRanks + rank) * kAdaMaxBlocks + blockIdx.x) * 3 + k;
      for (int q = 0; q < world; q++) st_sys_f64(reinterpret_cast<double*>(a.buf.p[q]) + slot, s_part[threadIdx.x]);
    }
    // ---- full barrier: same-index CTAs of all ranks, then all CTAs of this rank ----
    rank_barrier(a.c, ++e);
    grid_barrier(a.c);
    // ---- totals in a fixed order (warp w adds one of the 3*np numbers): the same bits everywhere ----
    {
      const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
      if (warp < 3 * np) {
        const int p = warp / 3, k = warp - 3 * p;
        const double* board = reinterpret_cast<const double*>(mine);
        const int entries = world * (int)gridDim.x;
        double s = 0.0;
        for (int j = lane; j < entries; j += 32) {
          const int src = j / (int)gridDim.x, cta = j - src * (int)gridDim.x;
          s += ld_sys_f64(board + (((size_t)(pair_base + p) * kMaxRanks + src) * kAdaMaxBlocks + cta) * 3 + k);
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0) s_part[warp] = s;
      }
      __syncthreads();
      if (threadIdx.x < (unsigned)np) {
        const double d = s_part[3 * threadIdx.x], na = s_part[3 * threadIdx.x + 1], nb = s_part[3 * threadIdx.x + 2];
        s_coef[threadIdx.x][0] = na > 0.0 ? (float)(1.0 - d / (2.0 * na)) : 1.0f;
        s_coef[threadIdx.x][1] = nb > 0.0 ? (float)(1.0 - d / (2.0 * nb)) : 1.0f;
      }
      __syncthreads();
    }
    // ---- combine: W[g] = ca W[g] + cb W[g + dist]; next level's partial dots in the same pass ----
#pragma unroll
    for (int k = 0; k < 3 * kAdaMaxPairs; k++) acc[k] = 0.0;
    const bool last = np == 1;
    for (size_t i = t0; i < lim; i += tstride) {
      float prev[VN];
#pragma unroll
      for (int p = 0; p < kAdaMaxPairs; p++) {
        if (p < np) {
          const size_t g = (size_t)p * 2 * dist, h = g + dist;
          const float ca = s_coef[p][0], cb = s_coef[p][1];
          float z[VN];
#pragma unroll
          for (int j = 0; j < V4; j++) {
            const float4 x = W[g * wq + i * V4 + j], y = W[h * wq + i * V4 + j];
            z[4 * j] = ca * x.x + cb * y.x; z[4 * j + 1] = ca * x.y + cb * y.y;
            z[4 * j + 2] = ca * x.z + cb * y.z; z[4 * j + 3] = ca * x.w + cb * y.w;
          }
          if (last) {
            const uint4 o = VecTraits<T>::pack(z);
            for (int q = 0; q < world; q++) st_peer_v4(a.buf.p[q] + kAdaDotBytes + (base + i) * 16, o);
          } else {
#pragma unroll
            for (int j = 0; j < V4; j++) W[g * wq + i * V4 + j] = make_float4(z[4 * j], z[4 * j + 1], z[4 * j + 2], z[4 * j + 3]);
            if (p & 1) dots3<VN>(acc + 3 * (p >> 1), prev, z);
            else {
#pragma unroll
              for (int j = 0; j < VN; j++) prev[j] = z[j];
            }
          }
        }
      }
    }
    pair_base += np;
    np >>= 1;
  }
  rank_barrier(a.c, ++e);

  // ---- phase 2: A -> user output ----
  for (int r = 0; r < world; r++) {
    const size_t b2 = (size_t)r * per;
    const size_t l2 = b2 < nvec ? (nvec - b2 < per ? nvec - b2 : per) : 0;
    for (size_t i = t0; i < l2; i += tstride)
      user_store(a.out, b2 + i, a.nbytes, a.out_aligned, ld_sys_v4(A_mine + (b2 + i) * 16));
  }
  if (threadIdx.x == 0) a.c.epoch[blockIdx.x] = e;
}

cudaError_t launch_adasum(const Launch& l, const KArgs& a, int dtype) {
  dim3 grid(l.blocks, l.emu_world > 0 ? l.emu_world : 1, 1);
  const KArgs* emu = l.emu_world > 0 ? l.emu_args : nullptr;
  switch (dtype) {
    case DT_F32: k_adasum<float><<<grid, kThreads, 0, l.stream>>>(a, emu); break;
    case DT_BF16: k_adasum<__nv_bfloat16><<<grid, kThreads, 0, l.stream>>>(a, emu); break;
    case DT_F16: k_adasum<__half><<<grid, kThreads, 0, l.stream>>>(a, emu); break;
    default: return cudaErrorInvalidValue;
  }
  return cudaGetLastError();
}

}  // namespace b200mpi
