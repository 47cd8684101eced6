// b200mpi collective kernels for sm_90a: NVSwitch peer-memory allreduce
// (push one-shot, pull/push two-shot, NVLS multimem), fused allreduce+SGD,
// allgather, broadcast, reduce-scatter, reduce, all-to-all, barrier.
//
// Call sites these serve in the reference's workloads (SURVEY.md §2.5):
//   K2 barrier        examples/v2beta1/pi/pi.cc:49
//   K3 broadcast      examples/v2beta1/horovod/tensorflow_mnist.py:143
//   K4 allreduce(avg) examples/v2beta1/horovod/tensorflow_mnist.py:133,
//                     examples/v2beta1/tensorflow-benchmarks/tensorflow-benchmarks.yaml:42
//   K5 allgather      Horovod API surface
// In the reference these are NCCL library calls plus a separate scale kernel;
// here the 1/N scale, the dtype handling and (optionally) the optimizer step
// run inside the same kernel that moves the bytes over NVLink.
//
// Work partition invariant (needed because CTAs only synchronise with the
// CTA of the same blockIdx.x on the other ranks): in every phase CTA b touches
// the vector indices C_b = { i : grid-stride from b } *within each slice*, so
// whatever CTA b reads after a barrier was written by CTA b of some rank.
#include "kernels.h"

namespace b200mpi {

#define EMU_ARGS const KArgs& a = (emu != nullptr) ? emu[blockIdx.y] : a0

__device__ __forceinline__ size_t gtid() { return (size_t)blockIdx.x * blockDim.x + threadIdx.x; }
__device__ __forceinline__ size_t gstride() { return (size_t)gridDim.x * blockDim.x; }
__device__ __forceinline__ int wrap(int x, int world) { return x >= world ? x - world : x; }

template <typename T>
__device__ __forceinline__ void accum(float* acc, const uint4& v, int op, bool first) {
  float f[VecTraits<T>::N];
  VecTraits<T>::unpack(v, f);
#pragma unroll
  for (int j = 0; j < VecTraits<T>::N; j++)
    acc[j] = first ? f[j] : (op == OP_SUM ? acc[j] + f[j] : (op == OP_MAX ? fmaxf(acc[j], f[j]) : fminf(acc[j], f[j])));
}

template <typename T>
__device__ __forceinline__ uint4 nvls_ld_reduce(const void* mc, int op) {
  if (MultiMem<T>::kHasMinMax) {
    if (op == OP_MAX) return MultiMem<T>::template ld_reduce<OP_MAX>(mc);
    if (op == OP_MIN) return MultiMem<T>::template ld_reduce<OP_MIN>(mc);
  }
  return MultiMem<T>::template ld_reduce<OP_SUM>(mc);
}

template <typename T>
__device__ __forceinline__ uint4 scale_vec(const uint4& v, float s) {
  float f[VecTraits<T>::N];
  VecTraits<T>::unpack(v, f);
#pragma unroll
  for (int j = 0; j < VecTraits<T>::N; j++) f[j] *= s;
  return VecTraits<T>::pack(f);
}

// ===========================================================================
// Two-shot allreduce. Rank r owns slice r: it pulls slice r from every peer
// (reduce-scatter), reduces in fp32, applies `scale`, and pushes the result
// into slice r of every peer (all-gather) — one kernel, two cross-rank
// barriers. MODE_NVLS replaces the N loads by one multimem.ld_reduce (the
// NVSwitch adds) and the N stores by one multimem.st (the switch fans out).
// STAGED: user pointers are copied into / out of the staging window here.
// ===========================================================================
template <typename T, int MODE, bool STAGED>
__global__ void __launch_bounds__(kThreads)
k_allreduce_twoshot(const __grid_constant__ KArgs a0, const KArgs* __restrict__ emu) {
  EMU_ARGS;
  const int rank = a.c.rank, world = a.c.world;
  uint32_t e = a.c.epoch[blockIdx.x];
  const size_t per = a.per, nvec = a.nvec;
  char* const mine = a.buf.p[rank];

  // U consecutive blockDim-sized chunks per CTA per trip: the SAME index->CTA map
  // in the copy-in, reduce and copy-out phases (partition invariant above).
  constexpr int U = (MODE == MODE_NVLS) ? 4 : 2;
  if (STAGED) {
    for (int r = 0; r < world; r++) {
      const size_t base = (size_t)r * per;
      const size_t lim = base < nvec ? (nvec - base < per ? nvec - base : per) : 0;
      for (size_t i0 = (size_t)blockIdx.x * blockDim.x * U + threadIdx.x; i0 < lim; i0 += gstride() * U) {
#pragma unroll
        for (int u = 0; u < U; u++) {
          const size_t i = i0 + (size_t)u * blockDim.x;
          if (i < lim)
            *reinterpret_cast<uint4*>(mine + (base + i) * 16) = user_load(a.in, base + i, a.nbytes, a.in_aligned);
        }
      }
    }
  }
  rank_barrier(a.c, ++e);

  {
    const size_t base = (size_t)rank * per;
    const size_t lim = base < nvec ? (nvec - base < per ? nvec - base : per) : 0;
    const bool do_scale = a.scale != 1.0f;
    if (MODE == MODE_NVLS) {
      char* const mc = a.buf.mc + base * 16;
      for (size_t i0 = (size_t)blockIdx.x * blockDim.x * U + threadIdx.x; i0 < lim; i0 += gstride() * U) {
        uint4 v[U];
#pragma unroll
        for (int u = 0; u < U; u++) {
          const size_t i = i0 + (size_t)u * blockDim.x;
          if (i < lim) v[u] = nvls_ld_reduce<T>(mc + i * 16, a.op);
        }
#pragma unroll
        for (int u = 0; u < U; u++) {
          const size_t i = i0 + (size_t)u * blockDim.x;
          if (i < lim) multimem_st_v4(mc + i * 16, do_scale ? scale_vec<T>(v[u], a.scale) : v[u]);
        }
      }
    } else {
      char* pp[kMaxRanks];
      char* po[kMaxRanks];   // where the result goes: the same region, or a second one (registered out-of-place user buffers)
#pragma unroll
      for (int k = 0; k < kMaxRanks; k++) {
        const int r = wrap(rank + (k < world ? k : 0), world);
        pp[k] = a.buf.p[r] + base * 16;
        po[k] = (a.param.p[0] ? a.param.p[r] : a.buf.p[r]) + base * 16;
      }
      for (size_t i0 = (size_t)blockIdx.x * blockDim.x * U + threadIdx.x; i0 < lim; i0 += gstride() * U) {
        uint4 v[U][kMaxRanks];
#pragma unroll
        for (int u = 0; u < U; u++) {
          const size_t i = i0 + (size_t)u * blockDim.x;
#pragma unroll
          for (int k = 0; k < kMaxRanks; k++)
            if (k < world && i < lim) v[u][k] = ld_sys_v4(pp[k] + i * 16);
        }
#pragma unroll
        for (int u = 0; u < U; u++) {
          const size_t i = i0 + (size_t)u * blockDim.x;
          if (i < lim) {
            float acc[VecTraits<T>::N];
#pragma unroll
            for (int k = 0; k < kMaxRanks; k++)
              if (k < world) accum<T>(acc, v[u][k], a.op, k == 0);
            if (do_scale) {
#pragma unroll
              for (int j = 0; j < VecTraits<T>::N; j++) acc[j] *= a.scale;
            }
            const uint4 o = VecTraits<T>::pack(acc);
#pragma unroll
            for (int k = 0; k < kMaxRanks; k++)
              if (k < world) st_peer_v4(po[k] + i * 16, o);
          }
        }
      }
    }
  }
  rank_barrier(a.c, ++e);

  if (STAGED) {
    for (int r = 0; r < world; r++) {
      const size_t base = (size_t)r * per;
      const size_t lim = base < nvec ? (nvec - base < per ? nvec - base : per) : 0;
      for (size_t i0 = (size_t)blockIdx.x * blockDim.x * U + threadIdx.x; i0 < lim; i0 += gstride() * U) {
        uint4 v[U];
#pragma unroll
        for (int u = 0; u < U; u++) {
          const size_t i = i0 + (size_t)u * blockDim.x;
          if (i < lim) v[u] = ld_sys_v4(mine + (base + i) * 16);
        }
#pragma unroll
        for (int u = 0; u < U; u++) {
          const size_t i = i0 + (size_t)u * blockDim.x;
          if (i < lim) user_store(a.out, base + i, a.nbytes, a.out_aligned, v[u]);
        }
      }
    }
  }
  if (threadIdx.x == 0) a.c.epoch[blockIdx.x] = e;
}

// ===========================================================================
// Pipelined staged collectives for arbitrary user pointers (the path the NCCL-ABI
// shim and hvd take for tensors that do not live in a symmetric window).
// The payload is cut into chunks; lane l owns chunks l, l+L, l+2L ... and is a
// chain of up to THREE CTAs that run concurrently and hand chunks on through flags:
//
//   ALLREDUCE       role 0  user input -> staging slot                          -> IN  (all ranks)
//                   role 1  wait IN; slice `rank` of the chunk: multimem.ld_reduce (or pull from every peer),
//                           scale, multimem.st (or peer stores) into every rank's slot -> RED (all ranks)
//                   role 2  wait RED; staging slot -> user output                -> local counter (frees the slot)
//   ALLGATHER       role 0  user input chunk -> region `rank` of EVERY rank's slot (multimem.st / peer stores),
//                           own block of the output written directly            -> IN  (all ranks)
//                   role 2  wait IN; regions of the other ranks -> user output   -> RED (all ranks: slot may be refilled)
//   REDUCE_SCATTER  role 0  all `world` blocks of the user input chunk -> own slot -> IN (all ranks)
//                   role 1  wait IN; region `rank`: ld_reduce / pull, scale -> user output -> RED (all ranks)
//   BROADCAST       role 0  (root) user buffer chunk -> every rank's slot        -> IN  (all ranks; non-roots signal at once)
//                   role 2  wait IN; (non-root) slot -> user buffer              -> RED (all ranks)
//
// so while chunk k is on NVLink, chunk k+1 is being copied in and chunk k-1 copied out: the local HBM copies that
// serialised the old staged kernels (three phases, two full barriers) disappear behind
// the link time. A slot is refilled for chunk k+depth only after every rank that reads or writes it for chunk k has
// said so (local counter for allreduce, RED flags otherwise). Flags only grow (per-role, per-lane counters persist in
// the epoch array and advance identically for all three roles), so the kernel is CUDA-graph capturable like the others.
// ===========================================================================
// ---- TMA bulk copies for the pipeline's local staging copies ------------------------------------------------------
// One elected thread moves a chunk global -> shared -> global with cp.async.bulk (SASS UBLKCP): a ring of kBulkNB
// buffers, up to kBulkNB/2 loads and kBulkNB/2 stores in flight (96 KB each way per CTA) with no registers and no
// warps tied up - a 512-thread CTA doing 16-byte loads/stores was slow enough to make the copy stages as slow as the NVLS stage they are supposed to hide behind.
constexpr int kBulkNB = 8;
constexpr uint32_t kBulkBytes = 24 * 1024;
constexpr size_t kPipeSmemBytes = (size_t)kBulkNB * kBulkBytes + 128;   // + mbarriers
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void bulk_mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t ok = 0;
  do {
    asm volatile(
        "{\n\t"
        ".reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t"
        "}"
        : "=r"(ok)
        : "r"(bar), "r"(parity)
        : "memory");
  } while (!ok);
}
// called by ONE thread. `pc` = pieces moved so far by this CTA (selects buffer and mbarrier phase); dst/src 16-byte aligned,
// bytes a multiple of 16. On return every store has been ISSUED; bulk_copy_drain() waits for them to land.
__device__ __forceinline__ void bulk_copy(char* dst, const char* src, size_t bytes, uint32_t ring, uint32_t bars, uint32_t& pc) {
  constexpr int LA = kBulkNB / 2;
  const size_t P = (bytes + kBulkBytes - 1) / kBulkBytes;
  for (size_t p = 0; p < P + LA; p++) {
    if (p >= (size_t)LA) {
      const size_t q = p - LA;
      const uint32_t g = pc + (uint32_t)q, sidx = g % kBulkNB;
      const uint32_t n = (uint32_t)(bytes - q * kBulkBytes < kBulkBytes ? bytes - q * kBulkBytes : kBulkBytes);
      bulk_mbar_wait(bars + sidx * 8, (g / kBulkNB) & 1u);
      asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst + q * kBulkBytes), "r"(ring + sidx * kBulkBytes), "r"(n) : "memory");
      asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    }
    if (p < P) {
      const uint32_t g = pc + (uint32_t)p, sidx = g % kBulkNB;
      const uint32_t n = (uint32_t)(bytes - p * kBulkBytes < kBulkBytes ? bytes - p * kBulkBytes : kBulkBytes);
      // the store that last read this buffer is at least kBulkNB - LA groups back
      asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(kBulkNB - LA) : "memory");
      asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bars + sidx * 8), "r"(n) : "memory");
      asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(ring + sidx * kBulkBytes),
                   "l"(src + p * kBulkBytes), "r"(n), "r"(bars + sidx * 8)
                   : "memory");
    }
  }
  pc += (uint32_t)P;
}
__device__ __forceinline__ void bulk_copy_drain() {
  asm volatile("cp.async.bulk.wait_group 0;" ::: "memory");
  asm volatile("fence.proxy.async;" ::: "memory");   // async-proxy writes before the generic-proxy flag that publishes them
}

// copy `len` vectors user -> staging (plain stores into local HBM), 8 loads in flight per thread.
// The aligned, full-vector case is a separate loop on purpose: user_load()'s byte-wise tail takes the address of its
// result, which parks the vector in local memory and makes every load wait for the previous one (measured with the
// in-kernel timeline: the bottleneck of the whole pipeline).
__device__ __forceinline__ void pipe_copy_in(char* dst, const char* ubase, size_t uvec0, size_t unbytes, bool ualigned, size_t len) {
  constexpr int U = 4;   // 32 KB in flight per CTA; 8 made the NVLS variants spill (128-register budget of 512-thread CTAs)
  if (ualigned && (uvec0 + len) * 16 <= unbytes) {
    const char* src = ubase + uvec0 * 16;
    for (size_t i0 = threadIdx.x; i0 < len; i0 += (size_t)blockDim.x * U) {
      uint4 v[U];
#pragma unroll
      for (int u = 0; u < U; u++) {
        const size_t i = i0 + (size_t)u * blockDim.x;
        if (i < len) v[u] = ld_stream_v4(src + i * 16);
      }
#pragma unroll
      for (int u = 0; u < U; u++) {
        const size_t i = i0 + (size_t)u * blockDim.x;
        if (i < len) *reinterpret_cast<uint4*>(dst + i * 16) = v[u];
      }
    }
    return;
  }
  for (size_t i = threadIdx.x; i < len; i += blockDim.x)
    *reinterpret_cast<uint4*>(dst + i * 16) = user_load(ubase, uvec0 + i, unbytes, ualigned);
}
__device__ __forceinline__ void pipe_copy_out(char* ubase, size_t uvec0, size_t unbytes, bool ualigned, const char* src, size_t len) {
  constexpr int U = 4;
  if (ualigned && (uvec0 + len) * 16 <= unbytes) {
    char* dst = ubase + uvec0 * 16;
    for (size_t i0 = threadIdx.x; i0 < len; i0 += (size_t)blockDim.x * U) {
      uint4 v[U];
#pragma unroll
      for (int u = 0; u < U; u++) {
        const size_t i = i0 + (size_t)u * blockDim.x;
        if (i < len) v[u] = ld_sys_v4(src + i * 16);
      }
#pragma unroll
      for (int u = 0; u < U; u++) {
        const size_t i = i0 + (size_t)u * blockDim.x;
        if (i < len) *reinterpret_cast<uint4*>(dst + i * 16) = v[u];
      }
    }
    return;
  }
  for (size_t i = threadIdx.x; i < len; i += blockDim.x)
    user_store(ubase, uvec0 + i, unbytes, ualigned, ld_sys_v4(src + i * 16));
}

// reduce `lim` vectors that every rank holds at byte offset `off` of its staging region; RESULT: `emit(i, vec)`
// NR = compile-time bound on the world size of the P2P variant: with 2 ranks eight vectors per thread are kept in
// flight (a peer load is ~3 us away; the link needs ~2 MB outstanding per direction), with up to 8 ranks two.
template <typename T, int MODE, int NR, typename Emit>
__device__ __forceinline__ void pipe_reduce(const KArgs& a, size_t off, size_t lim, Emit&& emit) {
  const int rank = a.c.rank, world = a.c.world;
  const bool do_scale = a.scale != 1.0f;
  if (MODE == MODE_NVLS) {
    constexpr int U = 4;
    const char* const mc = a.buf.mc + off;
    for (size_t i0 = threadIdx.x; i0 < lim; i0 += (size_t)blockDim.x * U) {
      uint4 v[U];
#pragma unroll
      for (int u = 0; u < U; u++) {
        const size_t i = i0 + (size_t)u * blockDim.x;
        if (i < lim) v[u] = nvls_ld_reduce<T>(mc + i * 16, a.op);
      }
#pragma unroll
      for (int u = 0; u < U; u++) {
        const size_t i = i0 + (size_t)u * blockDim.x;
        if (i < lim) emit(i, do_scale ? scale_vec<T>(v[u], a.scale) : v[u]);
      }
    }
  } else {
    constexpr int U = NR <= 2 ? 8 : 2;
    const char* pp[NR];
#pragma unroll
    for (int k = 0; k < NR; k++) pp[k] = a.buf.p[wrap(rank + (k < world ? k : 0), world)] + off;
    for (size_t i0 = threadIdx.x; i0 < lim; i0 += (size_t)blockDim.x * U) {
      uint4 v[U][NR];
#pragma unroll
      for (int u = 0; u < U; u++) {
        const size_t i = i0 + (size_t)u * blockDim.x;
#pragma unroll
        for (int k = 0; k < NR; k++)
          if (k < world && i < lim) v[u][k] = ld_sys_v4(pp[k] + i * 16);
      }
#pragma unroll
      for (int u = 0; u < U; u++) {
        const size_t i = i0 + (size_t)u * blockDim.x;
        if (i < lim) {
          float acc[VecTraits<T>::N];
#pragma unroll
          for (int k = 0; k < NR; k++)
            if (k < world) accum<T>(acc, v[u][k], a.op, k == 0);
          if (do_scale) {
#pragma unroll
            for (int q = 0; q < VecTraits<T>::N; q++) acc[q] *= a.scale;
          }
          emit(i, VecTraits<T>::pack(acc));
        }
      }
    }
  }
}

// store to the same staging byte offset on every rank (one multimem.st, or `world` peer stores)
template <int MODE, int NR>
__device__ __forceinline__ void pipe_store_all(const KArgs& a, size_t off, const uint4& v) {
  if (MODE == MODE_NVLS) {
    multimem_st_v4(a.buf.mc + off, v);
  } else {
    const int rank = a.c.rank, world = a.c.world;
#pragma unroll
    for (int k = 0; k < NR; k++)
      if (k < world) st_peer_v4(a.buf.p[wrap(rank + k, world)] + off, v);
  }
}

template <typename T, int MODE, int OP, int NR>
__global__ void __launch_bounds__(kThreads)
k_pipe(const __grid_constant__ KArgs a0, const KArgs* __restrict__ emu) {
  EMU_ARGS;
  const int rank = a.c.rank, world = a.c.world;
  const int L = a.lanes, D = a.depth;
  const int role = blockIdx.x / L, lane = blockIdx.x - role * L;
  const size_t Cv = a.per;                                     // vectors per chunk (of the per-rank payload)
  const size_t nchunks = (a.nvec + Cv - 1) / Cv;
  const uint32_t n_mine = nchunks > (size_t)lane ? (uint32_t)((nchunks - lane + L - 1) / L) : 0u;
  uint32_t* const ctr = a.c.epoch + kPipeEpochOff + (size_t)role * kPipeLanes + lane;
  uint32_t* const out_done = a.c.epoch + kPipeEpochOff + 3 * (size_t)kPipeLanes + lane;
  const uint32_t base = *ctr;
  const size_t row_in = kPipeSigOff + (size_t)lane * kMaxRanks;
  const size_t row_red = kPipeSigOff + ((size_t)kPipeLanes + lane) * kMaxRanks;
  const size_t row_done = kPipeSigOff + (2 * (size_t)kPipeLanes + lane) * kMaxRanks;
  char* const mine = a.buf.p[rank];
  constexpr bool kWide = OP == PIPE_ALLGATHER || OP == PIPE_REDUCE_SCATTER;   // slot = world regions of Cv vectors
  const size_t slot_vecs = kWide ? Cv * world : Cv;
  constexpr bool kUsesRole1 = OP == PIPE_ALLREDUCE || OP == PIPE_REDUCE_SCATTER;
  constexpr bool kUsesRole2 = OP != PIPE_REDUCE_SCATTER;
  const bool idle = (role == 1 && !kUsesRole1) || (role == 2 && !kUsesRole2);
  // TMA ring of the copy roles (dynamic shared memory: kBulkNB buffers + their mbarriers)
  extern __shared__ __align__(128) unsigned char pipe_smem[];
  const uint32_t ring = smem_u32(pipe_smem), bars = ring + kBulkNB * kBulkBytes;
  uint32_t pieces = 0;
  if (role != 1 && threadIdx.x == 0) {
    for (int b = 0; b < kBulkNB; b++) asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bars + b * 8), "r"(1) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
  }
  __syncthreads();
  const int last_role = kUsesRole2 ? 2 : 1;   // the role whose completion means: no rank touches this lane's slots any more
  // Ops whose FIRST action is a store into the peers' staging (allgather, broadcast) must know that every peer has left its
  // previous kernel: the barrier-based staged allreduce ends with a local copy-out from staging after its last barrier.
  // Entering this launch is that proof (stream order), so role 0 trades one ENTRY flag with everyone before it pushes.
  if ((OP == PIPE_ALLGATHER || OP == PIPE_BROADCAST) && role == 0 && n_mine > 0) {
    const size_t row_entry = kPipeSigOff + (3 * (size_t)kPipeLanes + lane) * kMaxRanks;
    flag_signal_all(a.c, row_entry, base + 1);
    flag_wait_all(a.c, row_entry, base + 1);
  }

  // optional timeline (B200MPI_PIPE_DEBUG): per (role, lane, chunk) the time the CTA started waiting, started working, finished
  unsigned long long* const dbg = a.dbg ? a.dbg + (((size_t)role * kPipeLanes + lane) * kPipeDbgChunks) * 3 : nullptr;
#define PIPE_STAMP(k) do { if (dbg && j < (uint32_t)kPipeDbgChunks && threadIdx.x == 0) dbg[j * 3 + (k)] = globaltimer_ns(); } while (0)
  for (uint32_t j = 0; j < n_mine && !idle; j++) {
    PIPE_STAMP(0);
    const size_t v0 = ((size_t)lane + (size_t)j * L) * Cv;            // first vector of the chunk in the payload
    const size_t len = a.nvec - v0 < Cv ? a.nvec - v0 : Cv;           // vectors in this chunk
    const size_t slot = ((size_t)lane * D + (j % D)) * slot_vecs;     // vector offset of the staging slot
    const uint32_t tgt = base + j + 1;
    if (role == 0) {
      if (j >= (uint32_t)D) {
        if (OP == PIPE_ALLREDUCE) local_wait(a.c, out_done, tgt - D);
        else flag_wait_all(a.c, row_red, tgt - D);
      }
      PIPE_STAMP(1);
      const bool bulk = a.in_aligned && (v0 + len) * 16 <= a.nbytes;   // whole chunk 16-byte aligned and inside the payload
      if (OP == PIPE_ALLREDUCE) {
        if (bulk) {
          if (threadIdx.x == 0) { bulk_copy(mine + slot * 16, a.in + v0 * 16, len * 16, ring, bars, pieces); bulk_copy_drain(); }
        } else {
          pipe_copy_in(mine + slot * 16, a.in, v0, a.nbytes, a.in_aligned, len);
        }
      } else if (OP == PIPE_REDUCE_SCATTER) {
        if (bulk) {
          if (threadIdx.x == 0) {
            for (int r = 0; r < world; r++)
              bulk_copy(mine + (slot + (size_t)r * Cv) * 16, a.in + (size_t)r * a.ustride + v0 * 16, len * 16, ring, bars, pieces);
            bulk_copy_drain();
          }
        } else {
          for (int r = 0; r < world; r++)
            pipe_copy_in(mine + (slot + (size_t)r * Cv) * 16, a.in + (size_t)r * a.ustride, v0, a.nbytes, a.in_aligned, len);
        }
      } else if (OP == PIPE_ALLGATHER || (OP == PIPE_BROADCAST && rank == a.root)) {
        // push: user chunk -> the same staging offset on every rank; allgather also writes its own output block directly
        const size_t dst = (slot + (OP == PIPE_ALLGATHER ? (size_t)rank * Cv : 0)) * 16;
        // the root of a broadcast is the only rank that pushes: twice the loads in flight per CTA
        constexpr int U = OP == PIPE_BROADCAST ? 8 : 4;
        const bool fast_in = a.in_aligned && (v0 + len) * 16 <= a.nbytes;
        const bool fast_out = a.out_aligned && (v0 + len) * 16 <= a.nbytes;
        const char* src = a.in + v0 * 16;
        char* own = OP == PIPE_ALLGATHER ? a.out + (size_t)rank * a.ustride + v0 * 16 : nullptr;
        for (size_t i0 = threadIdx.x; i0 < len; i0 += (size_t)blockDim.x * U) {
          uint4 v[U];
          if (fast_in) {
#pragma unroll
            for (int u = 0; u < U; u++) {
              const size_t i = i0 + (size_t)u * blockDim.x;
              if (i < len) v[u] = ld_stream_v4(src + i * 16);
            }
          } else {
            for (int u = 0; u < U; u++) {
              const size_t i = i0 + (size_t)u * blockDim.x;
              if (i < len) v[u] = user_load(a.in, v0 + i, a.nbytes, a.in_aligned);
            }
          }
#pragma unroll
          for (int u = 0; u < U; u++) {
            const size_t i = i0 + (size_t)u * blockDim.x;
            if (i < len) {
              pipe_store_all<MODE, NR>(a, dst + i * 16, v[u]);
              if (OP == PIPE_ALLGATHER) {
                if (fast_out) *reinterpret_cast<uint4*>(own + i * 16) = v[u];
                else user_store(a.out + (size_t)rank * a.ustride, v0 + i, a.nbytes, a.out_aligned, v[u]);
              }
            }
          }
        }
      }
      flag_signal_all(a.c, row_in, tgt);
      PIPE_STAMP(2);
    } else if (role == 1) {
      flag_wait_all(a.c, row_in, tgt);
      PIPE_STAMP(1);
      if (OP == PIPE_ALLREDUCE) {
        const size_t per = (len + world - 1) / world;
        const size_t sb = (size_t)rank * per;
        const size_t lim = sb < len ? (len - sb < per ? len - sb : per) : 0;
        const size_t off = (slot + sb) * 16;
        pipe_reduce<T, MODE, NR>(a, off, lim, [&](size_t i, const uint4& o) { pipe_store_all<MODE, NR>(a, off + i * 16, o); });
      } else {   // REDUCE_SCATTER: region `rank` of every rank's slot -> my output
        const size_t off = (slot + (size_t)rank * Cv) * 16;
        if (a.out_aligned && (v0 + len) * 16 <= a.nbytes) {
          char* const dst = a.out + v0 * 16;
          pipe_reduce<T, MODE, NR>(a, off, len, [&](size_t i, const uint4& o) { *reinterpret_cast<uint4*>(dst + i * 16) = o; });
        } else {
          pipe_reduce<T, MODE, NR>(a, off, len, [&](size_t i, const uint4& o) { user_store(a.out, v0 + i, a.nbytes, a.out_aligned, o); });
        }
      }
      flag_signal_all(a.c, row_red, tgt);
      PIPE_STAMP(2);
    } else {
      flag_wait_all(a.c, OP == PIPE_ALLREDUCE ? row_red : row_in, tgt);
      PIPE_STAMP(1);
      const bool bulk = a.out_aligned && (v0 + len) * 16 <= a.nbytes;
      // the slot was filled by remote (generic-proxy) stores observed through the flag acquire: order them before TMA reads
      if (bulk && threadIdx.x == 0) asm volatile("fence.proxy.async;" ::: "memory");
      if (OP == PIPE_ALLREDUCE) {
        if (bulk) {
          if (threadIdx.x == 0) { bulk_copy(a.out + v0 * 16, mine + slot * 16, len * 16, ring, bars, pieces); bulk_copy_drain(); }
        } else {
          pipe_copy_out(a.out, v0, a.nbytes, a.out_aligned, mine + slot * 16, len);
        }
        __syncthreads();
        if (threadIdx.x == 0) st_release_gpu(out_done, tgt);
      } else {
        if (OP == PIPE_ALLGATHER) {
          if (bulk) {
            if (threadIdx.x == 0) {
              for (int k = 1; k < world; k++) {     // own block was written by role 0
                const int r = wrap(rank + k, world);
                bulk_copy(a.out + (size_t)r * a.ustride + v0 * 16, mine + (slot + (size_t)r * Cv) * 16, len * 16, ring, bars, pieces);
              }
              bulk_copy_drain();
            }
          } else {
            for (int k = 1; k < world; k++) {
              const int r = wrap(rank + k, world);
              pipe_copy_out(a.out + (size_t)r * a.ustride, v0, a.nbytes, a.out_aligned, mine + (slot + (size_t)r * Cv) * 16, len);
            }
          }
        } else if (rank != a.root) {
          if (bulk) {
            if (threadIdx.x == 0) { bulk_copy(a.out + v0 * 16, mine + slot * 16, len * 16, ring, bars, pieces); bulk_copy_drain(); }
          } else {
            pipe_copy_out(a.out, v0, a.nbytes, a.out_aligned, mine + slot * 16, len);
          }
        }
        flag_signal_all(a.c, row_red, tgt);
      }
      PIPE_STAMP(2);
    }
  }
#undef PIPE_STAMP
  // Launch-completion handshake: a rank's kernel must not end before EVERY rank has finished with this lane's slots (peers
  // read and write them), otherwise the next launch on this stream - any kernel that uses the staging window, with any
  // slot geometry - could overwrite data a slower peer is still consuming. The last role tells all ranks it is done, role 0
  // (which finished first and would otherwise idle) waits for all of them.
  if (n_mine > 0) {
    if (role == last_role) flag_signal_all(a.c, row_done, base + n_mine);
    if (role == 0) flag_wait_all(a.c, row_done, base + n_mine);
  }
  if (threadIdx.x == 0) *ctr = base + n_mine;
}

// ===========================================================================
// Push one-shot allreduce (latency path). Every rank stores its input straight
// into a private slot of every peer's staging window, signals, then reduces
// the `world` slots that landed in its own HBM — one NVLink traversal and one
// flag per rank. Slots are double-buffered on a per-CTA use counter and the
// staging area is statically partitioned per CTA, so no trailing barrier is
// needed: a peer can only reach use k+2 of a CTA slot after this rank's kernel
// for use k has completed (see DESIGN.md "one-shot slot reuse").
// ===========================================================================
template <typename T>
__global__ void __launch_bounds__(kThreads)
k_allreduce_oneshot(const __grid_constant__ KArgs a0, const KArgs* __restrict__ emu) {
  EMU_ARGS;
  const int rank = a.c.rank, world = a.c.world;
  uint32_t e = a.c.epoch[blockIdx.x];
  const uint32_t use = a.c.epoch[kMaxBlocks + blockIdx.x];
  const size_t cap = a.per;  // vectors per (parity, block, rank) slot
  const size_t cv = (a.nvec + gridDim.x - 1) / gridDim.x;
  const size_t v0 = (size_t)blockIdx.x * cv;
  const size_t v1 = v0 + cv < a.nvec ? v0 + cv : a.nvec;
  const size_t slot0 = ((size_t)(use & 1u) * kOneshotBlocks + blockIdx.x) * world * cap;

  for (size_t i = v0 + threadIdx.x; i < v1; i += blockDim.x) {
    const uint4 v = user_load(a.in, i, a.nbytes, a.in_aligned);
    const size_t off = (slot0 + (size_t)rank * cap + (i - v0)) * 16;
#pragma unroll
    for (int k = 0; k < kMaxRanks; k++)
      if (k < world) st_peer_v4(a.buf.p[wrap(rank + k, world)] + off, v);
  }
  rank_barrier(a.c, ++e);

  const char* mine = a.buf.p[rank] + slot0 * 16;
  const bool do_scale = a.scale != 1.0f;
  for (size_t i = v0 + threadIdx.x; i < v1; i += blockDim.x) {
    uint4 v[kMaxRanks];
#pragma unroll
    for (int r = 0; r < kMaxRanks; r++)
      if (r < world) v[r] = ld_sys_v4(mine + ((size_t)r * cap + (i - v0)) * 16);
    float acc[VecTraits<T>::N];
#pragma unroll
    for (int r = 0; r < kMaxRanks; r++)
      if (r < world) accum<T>(acc, v[r], a.op, r == 0);
    if (do_scale) {
#pragma unroll
      for (int j = 0; j < VecTraits<T>::N; j++) acc[j] *= a.scale;
    }
    user_store(a.out, i, a.nbytes, a.out_aligned, VecTraits<T>::pack(acc));
  }
  if (threadIdx.x == 0) {
    a.c.epoch[blockIdx.x] = e;
    a.c.epoch[kMaxBlocks + blockIdx.x] = use + 1;
  }
}

// ===========================================================================
// Fused gradient allreduce + SGD. The reduce-scatter half of the two-shot
// produces the averaged gradient slice in registers; instead of writing it
// back, the owner applies weight decay + momentum + the parameter update to
// its fp32 slice (momentum lives only on the owner: 1/world of the state) and
// the all-gather half pushes the *updated parameters* to every rank. The
// gradient never returns to HBM and the optimizer kernel disappears.
// ===========================================================================
template <typename T, int MODE>
__global__ void __launch_bounds__(kThreads)
k_allreduce_sgd(const __grid_constant__ KArgs a0, const KArgs* __restrict__ emu) {
  EMU_ARGS;
  constexpr int N = VecTraits<T>::N;
  const int rank = a.c.rank, world = a.c.world;
  uint32_t e = a.c.epoch[blockIdx.x];
  const size_t per = a.per, nvec = a.nvec;
  rank_barrier(a.c, ++e);

  const size_t base = (size_t)rank * per;
  const size_t lim = base < nvec ? (nvec - base < per ? nvec - base : per) : 0;
  char* gp[kMaxRanks];
#pragma unroll
  for (int k = 0; k < kMaxRanks; k++) gp[k] = a.buf.p[wrap(rank + (k < world ? k : 0), world)] + base * 16;
  const char* gmc = a.buf.mc ? a.buf.mc + base * 16 : nullptr;
  const bool has_lowp = a.lowp.p[0] != nullptr;
  const float lr = a.hyper ? __ldg(a.hyper) : a.lr;
  const float mu = a.hyper ? __ldg(a.hyper + 1) : a.mu;
  const float wd = a.hyper ? __ldg(a.hyper + 2) : a.wd;

  // U vectors per thread per trip: U NVLink reduce-loads (or U x world peer loads) are issued before any
  // is consumed — with one vector per trip the NVLS variant was latency-bound.
  constexpr int U = (MODE == MODE_NVLS) ? 4 : 2;
  for (size_t i0 = (size_t)blockIdx.x * blockDim.x * U + threadIdx.x; i0 < lim; i0 += gstride() * U) {
    float gg[U][N];
    if (MODE == MODE_NVLS) {
      uint4 r[U];
#pragma unroll
      for (int u = 0; u < U; u++) {
        const size_t i = i0 + (size_t)u * blockDim.x;
        if (i < lim) r[u] = nvls_ld_reduce<T>(gmc + i * 16, OP_SUM);
      }
#pragma unroll
      for (int u = 0; u < U; u++) VecTraits<T>::unpack(r[u], gg[u]);
    } else {
      uint4 v[U][kMaxRanks];
#pragma unroll
      for (int u = 0; u < U; u++) {
        const size_t i = i0 + (size_t)u * blockDim.x;
#pragma unroll
        for (int k = 0; k < kMaxRanks; k++)
          if (k < world && i < lim) v[u][k] = ld_sys_v4(gp[k] + i * 16);
      }
#pragma unroll
      for (int u = 0; u < U; u++) {
#pragma unroll
        for (int k = 0; k < kMaxRanks; k++)
          if (k < world) accum<T>(gg[u], v[u][k], OP_SUM, k == 0);
      }
    }
#pragma unroll
    for (int u = 0; u < U; u++) {
      const size_t i = i0 + (size_t)u * blockDim.x;
      if (i >= lim) continue;
      float* g = gg[u];
      const size_t el = (base + i) * N;  // first element index of this vector
      float p[N], m[N];
      const float* pl = reinterpret_cast<const float*>(a.param.p[rank]) + el;
      float* ml = a.mom + i * N;
  #pragma unroll
      for (int q = 0; q < N / 4; q++) {
        float4 t = *reinterpret_cast<const float4*>(pl + 4 * q);
        p[4 * q] = t.x; p[4 * q + 1] = t.y; p[4 * q + 2] = t.z; p[4 * q + 3] = t.w;
        if (!a.first_step) {
          float4 s = *reinterpret_cast<const float4*>(ml + 4 * q);
          m[4 * q] = s.x; m[4 * q + 1] = s.y; m[4 * q + 2] = s.z; m[4 * q + 3] = s.w;
        }
      }
  #pragma unroll
      for (int j = 0; j < N; j++) {
        float gj = g[j] * a.scale + wd * p[j];
        float mj = a.first_step ? gj : mu * m[j] + gj;
        m[j] = mj;
        p[j] -= lr * (a.nesterov ? gj + mu * mj : mj);
      }
  #pragma unroll
      for (int q = 0; q < N / 4; q++) {
        *reinterpret_cast<float4*>(ml + 4 * q) = make_float4(m[4 * q], m[4 * q + 1], m[4 * q + 2], m[4 * q + 3]);
        const uint4 o = make_uint4(__float_as_uint(p[4 * q]), __float_as_uint(p[4 * q + 1]),
                                   __float_as_uint(p[4 * q + 2]), __float_as_uint(p[4 * q + 3]));
        const size_t boff = (el + 4 * q) * 4;
        if (MODE == MODE_NVLS) {
          multimem_st_v4(a.param.mc + boff, o);
        } else {
  #pragma unroll
          for (int k = 0; k < kMaxRanks; k++)
            if (k < world) st_peer_v4(a.param.p[wrap(rank + k, world)] + boff, o);
        }
      }
      if (has_lowp) {
        // bf16 shadow of the parameters for bf16-weight models: N bf16 = 2N bytes
        uint32_t w[N / 2];
  #pragma unroll
        for (int j = 0; j < N / 2; j++) {
          __nv_bfloat162 h = __floats2bfloat162_rn(p[2 * j], p[2 * j + 1]);
          w[j] = *reinterpret_cast<uint32_t*>(&h);
        }
        const size_t boff = el * 2;
  #pragma unroll
        for (int k = 0; k < kMaxRanks; k++) {
          if (k < world) {
            char* dst = a.lowp.p[wrap(rank + k, world)] + boff;
            if constexpr (N == 8) st_peer_v4(dst, make_uint4(w[0], w[1], w[2], w[3]));
            else *reinterpret_cast<uint2*>(dst) = make_uint2(w[0], w[1]);
          }
        }
      }
    }
  }
  rank_barrier(a.c, ++e);
  if (threadIdx.x == 0) a.c.epoch[blockIdx.x] = e;
}

// ===========================================================================
// Zero-copy collectives on a symmetric window region (no staging, no copy-out):
// the data already lives in peer-visible - and, when bound, multicast - memory.
// The region is `world` slices of `per` vectors; slice r belongs to rank r.
//   allgather       rank r's slice r -> slice r of every rank: ONE multimem.st per vector (the switch fans
//                   out, S/N bytes leave each GPU) or `world` peer stores
//   reduce_scatter  slice r of every rank -> reduced into rank r's slice r (or a user pointer):
//                   multimem.ld_reduce (the switch adds) or pulls from every peer
//   broadcast       the root's region -> every rank's region: multimem.st / peer stores
// Entry barrier: every rank's input is in place and nobody still reads what is about to be overwritten;
// exit barrier: everything has landed / everybody has read.
// ===========================================================================
template <int MODE>
__global__ void __launch_bounds__(kThreads)
k_allgather_sym(const __grid_constant__ KArgs a0, const KArgs* __restrict__ emu) {
  EMU_ARGS;
  const int rank = a.c.rank, world = a.c.world;
  uint32_t e = a.c.epoch[blockIdx.x];
  rank_barrier(a.c, ++e);
  const size_t base = (size_t)rank * a.per;
  const size_t lim = base < a.nvec ? (a.nvec - base < a.per ? a.nvec - base : a.per) : 0;
  // a.in: the slice comes from a separate buffer (registered user tensors) and must also land in this rank's own copy
  const char* src = a.in ? a.in : a.buf.p[rank] + base * 16;
  const int k0 = a.in ? 0 : 1;
  constexpr int U = 4;
  for (size_t i0 = (size_t)blockIdx.x * blockDim.x * U + threadIdx.x; i0 < lim; i0 += gstride() * U) {
    uint4 v[U];
#pragma unroll
    for (int u = 0; u < U; u++) {
      const size_t i = i0 + (size_t)u * blockDim.x;
      if (i < lim) v[u] = ld_stream_v4(src + i * 16);
    }
#pragma unroll
    for (int u = 0; u < U; u++) {
      const size_t i = i0 + (size_t)u * blockDim.x;
      if (i >= lim) continue;
      if (MODE == MODE_NVLS) {
        multimem_st_v4(a.buf.mc + (base + i) * 16, v[u]);
      } else {
#pragma unroll
        for (int k = 0; k < kMaxRanks; k++)
          if (k >= k0 && k < world) st_peer_v4(a.buf.p[wrap(rank + k, world)] + (base + i) * 16, v[u]);
      }
    }
  }
  rank_barrier(a.c, ++e);
  if (threadIdx.x == 0) a.c.epoch[blockIdx.x] = e;
}

template <typename T, int MODE>
__global__ void __launch_bounds__(kThreads)
k_reduce_scatter_sym(const __grid_constant__ KArgs a0, const KArgs* __restrict__ emu) {
  EMU_ARGS;
  const int rank = a.c.rank, world = a.c.world;
  uint32_t e = a.c.epoch[blockIdx.x];
  rank_barrier(a.c, ++e);
  const size_t base = (size_t)rank * a.per;
  const size_t lim = base < a.nvec ? (a.nvec - base < a.per ? a.nvec - base : a.per) : 0;
  const bool do_scale = a.scale != 1.0f;
  char* const dst = a.out ? a.out : a.buf.p[rank] + base * 16;   // user pointer (slice-sized) or in place
  if (MODE == MODE_NVLS) {
    constexpr int U = 4;
    const char* mc = a.buf.mc + base * 16;
    for (size_t i0 = (size_t)blockIdx.x * blockDim.x * U + threadIdx.x; i0 < lim; i0 += gstride() * U) {
      uint4 v[U];
#pragma unroll
      for (int u = 0; u < U; u++) {
        const size_t i = i0 + (size_t)u * blockDim.x;
        if (i < lim) v[u] = nvls_ld_reduce<T>(mc + i * 16, a.op);
      }
#pragma unroll
      for (int u = 0; u < U; u++) {
        const size_t i = i0 + (size_t)u * blockDim.x;
        if (i < lim) *reinterpret_cast<uint4*>(dst + i * 16) = do_scale ? scale_vec<T>(v[u], a.scale) : v[u];
      }
    }
  } else {
    constexpr int U = 2;
    const char* pp[kMaxRanks];
#pragma unroll
    for (int k = 0; k < kMaxRanks; k++) pp[k] = a.buf.p[wrap(rank + (k < world ? k : 0), world)] + base * 16;
    for (size_t i0 = (size_t)blockIdx.x * blockDim.x * U + threadIdx.x; i0 < lim; i0 += gstride() * U) {
      uint4 v[U][kMaxRanks];
#pragma unroll
      for (int u = 0; u < U; u++) {
        const size_t i = i0 + (size_t)u * blockDim.x;
#pragma unroll
        for (int k = 0; k < kMaxRanks; k++)
          if (k < world && i < lim) v[u][k] = ld_sys_v4(pp[k] + i * 16);
      }
#pragma unroll
      for (int u = 0; u < U; u++) {
        const size_t i = i0 + (size_t)u * blockDim.x;
        if (i >= lim) continue;
        float acc[VecTraits<T>::N];
#pragma unroll
        for (int k = 0; k < kMaxRanks; k++)
          if (k < world) accum<T>(acc, v[u][k], a.op, k == 0);
        if (do_scale) {
#pragma unroll
          for (int q = 0; q < VecTraits<T>::N; q++) acc[q] *= a.scale;
        }
        *reinterpret_cast<uint4*>(dst + i * 16) = VecTraits<T>::pack(acc);
      }
    }
  }
  rank_barrier(a.c, ++e);
  if (threadIdx.x == 0) a.c.epoch[blockIdx.x] = e;
}

template <int MODE>
__global__ void __launch_bounds__(kThreads)
k_broadcast_sym(const __grid_constant__ KArgs a0, const KArgs* __restrict__ emu) {
  EMU_ARGS;
  const int rank = a.c.rank, world = a.c.world;
  uint32_t e = a.c.epoch[blockIdx.x];
  rank_barrier(a.c, ++e);
  if (rank == a.root) {
    const char* src = a.buf.p[rank];
    constexpr int U = 4;
    for (size_t i0 = (size_t)blockIdx.x * blockDim.x * U + threadIdx.x; i0 < a.nvec; i0 += gstride() * U) {
      uint4 v[U];
#pragma unroll
      for (int u = 0; u < U; u++) {
        const size_t i = i0 + (size_t)u * blockDim.x;
        if (i < a.nvec) v[u] = ld_stream_v4(src + i * 16);
      }
#pragma unroll
      for (int u = 0; u < U; u++) {
        const size_t i = i0 + (size_t)u * blockDim.x;
        if (i >= a.nvec) continue;
        if (MODE == MODE_NVLS) {
          multimem_st_v4(a.buf.mc + i * 16, v[u]);
        } else {
#pragma unroll
          for (int k = 1; k < kMaxRanks; k++)
            if (k < world) st_peer_v4(a.buf.p[wrap(rank + k, world)] + i * 16, v[u]);
        }
      }
    }
  }
  rank_barrier(a.c, ++e);
  if (threadIdx.x == 0) a.c.epoch[blockIdx.x] = e;
}

// ===========================================================================
// Staged byte-wise collectives. Pattern: push/copy into staging -> barrier ->
// consume from own staging -> trailing barrier (staging is reused next call).
// ===========================================================================
__global__ void __launch_bounds__(kThreads)
k_allgather(const __grid_constant__ KArgs a0, const KArgs* __restrict__ emu) {
  EMU_ARGS;
  const int rank = a.c.rank, world = a.c.world;
  uint32_t e = a.c.epoch[blockIdx.x];
  const size_t per = a.per;
  for (size_t i = gtid(); i < a.nvec; i += gstride()) {
    const uint4 v = user_load(a.in, i, a.nbytes, a.in_aligned);
    const size_t off = ((size_t)rank * per + i) * 16;
#pragma unroll
    for (int k = 0; k < kMaxRanks; k++)
      if (k < world) st_peer_v4(a.buf.p[wrap(rank + k, world)] + off, v);
  }
  rank_barrier(a.c, ++e);
  const char* mine = a.buf.p[rank];
  for (int r = 0; r < world; r++)
    for (size_t i = gtid(); i < a.nvec; i += gstride())
      user_store(a.out + (size_t)r * a.ustride, i, a.nbytes, a.out_aligned, ld_sys_v4(mine + ((size_t)r * per + i) * 16));
  rank_barrier(a.c, ++e);
  if (threadIdx.x == 0) a.c.epoch[blockIdx.x] = e;
}

template <int MODE>
__global__ void __launch_bounds__(kThreads)
k_broadcast(const __grid_constant__ KArgs a0, const KArgs* __restrict__ emu) {
  EMU_ARGS;
  const int rank = a.c.rank, world = a.c.world;
  uint32_t e = a.c.epoch[blockIdx.x];
  if (rank == a.root) {
    for (size_t i = gtid(); i < a.nvec; i += gstride()) {
      const uint4 v = user_load(a.in, i, a.nbytes, a.in_aligned);
      if (MODE == MODE_NVLS) {
        multimem_st_v4(a.buf.mc + i * 16, v);
      } else {
#pragma unroll
        for (int k = 1; k < kMaxRanks; k++)
          if (k < world) st_peer_v4(a.buf.p[wrap(rank + k, world)] + i * 16, v);
      }
    }
  }
  rank_barrier(a.c, ++e);
  if (rank != a.root) {
    const char* mine = a.buf.p[rank];
    for (size_t i = gtid(); i < a.nvec; i += gstride())
      user_store(a.out, i, a.nbytes, a.out_aligned, ld_sys_v4(mine + i * 16));
  }
  rank_barrier(a.c, ++e);
  if (threadIdx.x == 0) a.c.epoch[blockIdx.x] = e;
}

template <typename T>
__global__ void __launch_bounds__(kThreads)
k_reduce_scatter(const __grid_constant__ KArgs a0, const KArgs* __restrict__ emu) {
  EMU_ARGS;
  const int rank = a.c.rank, world = a.c.world;
  uint32_t e = a.c.epoch[blockIdx.x];
  const size_t per = a.per;
  char* const mine = a.buf.p[rank];
  for (int r = 0; r < world; r++)
    for (size_t i = gtid(); i < a.nvec; i += gstride())
      *reinterpret_cast<uint4*>(mine + ((size_t)r * per + i) * 16) =
          user_load(a.in + (size_t)r * a.ustride, i, a.nbytes, a.in_aligned);
  rank_barrier(a.c, ++e);
  const bool do_scale = a.scale != 1.0f;
  for (size_t i = gtid(); i < a.nvec; i += gstride()) {
    uint4 v[kMaxRanks];
#pragma unroll
    for (int k = 0; k < kMaxRanks; k++)
      if (k < world) v[k] = ld_sys_v4(a.buf.p[k] + ((size_t)rank * per + i) * 16);
    float acc[VecTraits<T>::N];
#pragma unroll
    for (int k = 0; k < kMaxRanks; k++)
      if (k < world) accum<T>(acc, v[k], a.op, k == 0);
    if (do_scale) {
#pragma unroll
      for (int j = 0; j < VecTraits<T>::N; j++) acc[j] *= a.scale;
    }
    user_store(a.out, i, a.nbytes, a.out_aligned, VecTraits<T>::pack(acc));
  }
  rank_barrier(a.c, ++e);
  if (threadIdx.x == 0) a.c.epoch[blockIdx.x] = e;
}

template <typename T>
__global__ void __launch_bounds__(kThreads)
k_reduce(const __grid_constant__ KArgs a0, const KArgs* __restrict__ emu) {
  EMU_ARGS;
  const int rank = a.c.rank, world = a.c.world;
  uint32_t e = a.c.epoch[blockIdx.x];
  char* const mine = a.buf.p[rank];
  for (size_t i = gtid(); i < a.nvec; i += gstride())
    *reinterpret_cast<uint4*>(mine + i * 16) = user_load(a.in, i, a.nbytes, a.in_aligned);
  rank_barrier(a.c, ++e);
  if (rank == a.root) {
    const bool do_scale = a.scale != 1.0f;
    for (size_t i = gtid(); i < a.nvec; i += gstride()) {
      uint4 v[kMaxRanks];
#pragma unroll
      for (int k = 0; k < kMaxRanks; k++)
        if (k < world) v[k] = ld_sys_v4(a.buf.p[k] + i * 16);
      float acc[VecTraits<T>::N];
#pragma unroll
      for (int k = 0; k < kMaxRanks; k++)
        if (k < world) accum<T>(acc, v[k], a.op, k == 0);
      if (do_scale) {
#pragma unroll
        for (int j = 0; j < VecTraits<T>::N; j++) acc[j] *= a.scale;
      }
      user_store(a.out, i, a.nbytes, a.out_aligned, VecTraits<T>::pack(acc));
    }
  }
  rank_barrier(a.c, ++e);
  if (threadIdx.x == 0) a.c.epoch[blockIdx.x] = e;
}

__global__ void __launch_bounds__(kThreads)
k_alltoall(const __grid_constant__ KArgs a0, const KArgs* __restrict__ emu) {
  EMU_ARGS;
  const int rank = a.c.rank, world = a.c.world;
  uint32_t e = a.c.epoch[blockIdx.x];
  const size_t per = a.per;
  for (int k = 0; k < world; k++) {
    const int dst = wrap(rank + k, world);
    for (size_t i = gtid(); i < a.nvec; i += gstride())
      st_peer_v4(a.buf.p[dst] + ((size_t)rank * per + i) * 16,
                 user_load(a.in + (size_t)dst * a.ustride, i, a.nbytes, a.in_aligned));
  }
  rank_barrier(a.c, ++e);
  const char* mine = a.buf.p[rank];
  for (int r = 0; r < world; r++)
    for (size_t i = gtid(); i < a.nvec; i += gstride())
      user_store(a.out + (size_t)r * a.ustride, i, a.nbytes, a.out_aligned, ld_sys_v4(mine + ((size_t)r * per + i) * 16));
  rank_barrier(a.c, ++e);
  if (threadIdx.x == 0) a.c.epoch[blockIdx.x] = e;
}

__global__ void __launch_bounds__(kThreads)
k_barrier(const __grid_constant__ KArgs a0, const KArgs* __restrict__ emu) {
  EMU_ARGS;
  uint32_t e = a.c.epoch[blockIdx.x];
  rank_barrier(a.c, ++e);
  if (threadIdx.x == 0) a.c.epoch[blockIdx.x] = e;
}

// --------------------------------------------------------- local helpers ----
template <typename TI, typename TO>
__global__ void k_scale_cast(const TI* __restrict__ in, TO* __restrict__ out, size_t n, float scale) {
  for (size_t i = gtid(); i < n; i += gstride()) out[i] = static_cast<TO>(static_cast<float>(in[i]) * scale);
}
__global__ void k_fill_u32(uint32_t* p, uint32_t v, size_t n) {
  for (size_t i = gtid(); i < n; i += gstride()) p[i] = v;
}

// ------------------------------------------------------------- launchers ----
template <typename K>
static cudaError_t go(K kernel, const Launch& l, const KArgs& a) {
  dim3 grid(l.blocks, l.emu_world > 0 ? l.emu_world : 1, 1);
  kernel<<<grid, kThreads, 0, l.stream>>>(a, l.emu_world > 0 ? l.emu_args : nullptr);
  return cudaGetLastError();
}

#define DISPATCH_T(dtype, EXPR)                                   \
  switch (dtype) {                                                \
    case DT_F32: { using T = float; return EXPR; }                \
    case DT_BF16: { using T = __nv_bfloat16; return EXPR; }       \
    case DT_F16: { using T = __half; return EXPR; }               \
    default: return cudaErrorInvalidValue;                        \
  }

cudaError_t launch_allreduce_twoshot(const Launch& l, const KArgs& a, int dtype, int mode, bool staged) {
  if (mode == MODE_NVLS) {
    if (staged) DISPATCH_T(dtype, go(k_allreduce_twoshot<T, MODE_NVLS, true>, l, a))
    DISPATCH_T(dtype, go(k_allreduce_twoshot<T, MODE_NVLS, false>, l, a))
  }
  if (staged) DISPATCH_T(dtype, go(k_allreduce_twoshot<T, MODE_P2P, true>, l, a))
  DISPATCH_T(dtype, go(k_allreduce_twoshot<T, MODE_P2P, false>, l, a))
}
// launch with the TMA ring as dynamic shared memory (> 48 KB: opt in once per instantiation)
template <typename K>
static cudaError_t go_pipe(K kernel, const Launch& l, const KArgs& a) {
  // K is the same function-pointer type for every instantiation: remember the kernels already opted in by address
  static const void* done[64];
  static int ndone = 0;
  bool seen = false;
  for (int i = 0; i < ndone; i++) seen = seen || done[i] == (const void*)kernel;
  if (!seen) {
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kPipeSmemBytes);
    if (e != cudaSuccess) return e;
    if (ndone < 64) done[ndone++] = (const void*)kernel;
  }
  dim3 grid(l.blocks, l.emu_world > 0 ? l.emu_world : 1, 1);
  kernel<<<grid, kThreads, kPipeSmemBytes, l.stream>>>(a, l.emu_world > 0 ? l.emu_args : nullptr);
  return cudaGetLastError();
}
// kind: PIPE_* ; byte-wise kinds (allgather, broadcast) ignore dtype. P2P variants are specialised for world <= 2.
template <int OP>
static cudaError_t launch_pipe_t(const Launch& l, const KArgs& a, int dtype, int mode) {
  if (mode == MODE_NVLS) DISPATCH_T(dtype, go_pipe(k_pipe<T, MODE_NVLS, OP, kMaxRanks>, l, a))
  if (a.c.world <= 2) DISPATCH_T(dtype, go_pipe(k_pipe<T, MODE_P2P, OP, 2>, l, a))
  DISPATCH_T(dtype, go_pipe(k_pipe<T, MODE_P2P, OP, kMaxRanks>, l, a))
}
cudaError_t launch_pipe(const Launch& l, const KArgs& a, int kind, int dtype, int mode) {
  switch (kind) {
    case PIPE_ALLREDUCE: return launch_pipe_t<PIPE_ALLREDUCE>(l, a, dtype, mode);
    case PIPE_REDUCE_SCATTER: return launch_pipe_t<PIPE_REDUCE_SCATTER>(l, a, dtype, mode);
    case PIPE_ALLGATHER: return launch_pipe_t<PIPE_ALLGATHER>(l, a, DT_F32, mode);
    case PIPE_BROADCAST: return launch_pipe_t<PIPE_BROADCAST>(l, a, DT_F32, mode);
    default: return cudaErrorInvalidValue;
  }
}
cudaError_t launch_allreduce_oneshot(const Launch& l, const KArgs& a, int dtype) {
  DISPATCH_T(dtype, go(k_allreduce_oneshot<T>, l, a))
}
cudaError_t launch_allreduce_sgd(const Launch& l, const KArgs& a, int dtype, int mode) {
  if (mode == MODE_NVLS) DISPATCH_T(dtype, go(k_allreduce_sgd<T, MODE_NVLS>, l, a))
  DISPATCH_T(dtype, go(k_allreduce_sgd<T, MODE_P2P>, l, a))
}
cudaError_t launch_allgather(const Launch& l, const KArgs& a) { return go(k_allgather, l, a); }
cudaError_t launch_allgather_sym(const Launch& l, const KArgs& a, int mode) {
  return mode == MODE_NVLS ? go(k_allgather_sym<MODE_NVLS>, l, a) : go(k_allgather_sym<MODE_P2P>, l, a);
}
cudaError_t launch_broadcast_sym(const Launch& l, const KArgs& a, int mode) {
  return mode == MODE_NVLS ? go(k_broadcast_sym<MODE_NVLS>, l, a) : go(k_broadcast_sym<MODE_P2P>, l, a);
}
cudaError_t launch_reduce_scatter_sym(const Launch& l, const KArgs& a, int dtype, int mode) {
  if (mode == MODE_NVLS) DISPATCH_T(dtype, go(k_reduce_scatter_sym<T, MODE_NVLS>, l, a))
  DISPATCH_T(dtype, go(k_reduce_scatter_sym<T, MODE_P2P>, l, a))
}
cudaError_t launch_broadcast(const Launch& l, const KArgs& a, int mode) {
  return mode == MODE_NVLS ? go(k_broadcast<MODE_NVLS>, l, a) : go(k_broadcast<MODE_P2P>, l, a);
}
cudaError_t launch_reduce_scatter(const Launch& l, const KArgs& a, int dtype) {
  DISPATCH_T(dtype, go(k_reduce_scatter<T>, l, a))
}
cudaError_t launch_reduce(const Launch& l, const KArgs& a, int dtype) {
  DISPATCH_T(dtype, go(k_reduce<T>, l, a))
}
cudaError_t launch_alltoall(const Launch& l, const KArgs& a) { return go(k_alltoall, l, a); }
cudaError_t launch_barrier(const Launch& l, const KArgs& a) { return go(k_barrier, l, a); }

template <typename TI>
static cudaError_t scale_cast_out(cudaStream_t s, const void* in, void* out, int out_dt, size_t n, float scale) {
  const int blocks = (int)((n + 1023) / 1024 < 1184 ? (n + 1023) / 1024 : 1184);
  if (n == 0) return cudaSuccess;
  switch (out_dt) {
    case DT_F32: k_scale_cast<TI, float><<<blocks, 256, 0, s>>>((const TI*)in, (float*)out, n, scale); break;
    case DT_BF16: k_scale_cast<TI, __nv_bfloat16><<<blocks, 256, 0, s>>>((const TI*)in, (__nv_bfloat16*)out, n, scale); break;
    case DT_F16: k_scale_cast<TI, __half><<<blocks, 256, 0, s>>>((const TI*)in, (__half*)out, n, scale); break;
    default: return cudaErrorInvalidValue;
  }
  return cudaGetLastError();
}
cudaError_t launch_scale_cast(cudaStream_t s, const void* in, int in_dt, void* out, int out_dt, size_t n, float scale) {
  switch (in_dt) {
    case DT_F32: return scale_cast_out<float>(s, in, out, out_dt, n, scale);
    case DT_BF16: return scale_cast_out<__nv_bfloat16>(s, in, out, out_dt, n, scale);
    case DT_F16: return scale_cast_out<__half>(s, in, out, out_dt, n, scale);
    default: return cudaErrorInvalidValue;
  }
}
cudaError_t launch_fill_u32(cudaStream_t s, uint32_t* p, uint32_t v, size_t n) {
  if (n == 0) return cudaSuccess;
  k_fill_u32<<<(unsigned)((n + 255) / 256 < 1024 ? (n + 255) / 256 : 1024), 256, 0, s>>>(p, v, n);
  return cudaGetLastError();
}

}  // namespace b200mpi
