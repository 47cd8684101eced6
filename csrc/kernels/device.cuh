// b200mpi device-side primitives (sm_90a).
//
// Everything a collective kernel needs that is not the loop itself: the
// per-rank device context, .sys-scoped flag signalling between same-index CTAs
// of different ranks, 128-bit peer loads/stores, NVLS multimem wrappers and
// fp32-accumulate pack/unpack for f32 / bf16 / f16.
//
// Reference parity: this is the role NCCL's device primitives play underneath
// Horovod in the reference stack (SURVEY.md §2.5, §5.9); nothing here is
// derived from reference code (the reference tree has no device code at all).
#pragma once

#include <cuda_bf16.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

namespace b200mpi {

constexpr int kMaxRanks = 8;
constexpr int kMaxBlocks = 256;        // CTAs per rank that own a signal slot
constexpr int kThreads = 512;          // CTA size of every collective kernel
constexpr int kOneshotBlocks = 32;     // fixed staging partition of the push one-shot
// signal pad (u32 words): [kMaxBlocks][kMaxRanks]
constexpr size_t kSigWords = (size_t)kMaxBlocks * kMaxRanks;
// epoch array (u32 words): [0,kMaxBlocks) barrier epochs, [kMaxBlocks, 2*kMaxBlocks) one-shot use counts
constexpr size_t kEpochWords = 2 * (size_t)kMaxBlocks;
// Pipelined staged allreduce (k_allreduce_pipe): kPipeLanes independent lanes, each a chain of three CTAs
// (copy-in, reduce, copy-out) that hand chunks to each other through flags.
//   signal pad  : [kSigWords, kSigWords + 4*kPipeLanes*kMaxRanks)  IN-ready / REDUCED / DONE / ENTRY flags, [kind][lane][src rank]
//   epoch array : [kEpochWords, kEpochWords + 4*kPipeLanes)        chunks done so far per (role, lane), then the
//                                                                  local copy-out counter the copy-in CTA polls
constexpr int kPipeLanes = 44;           // 3 x 44 = 132 CTAs: one per H100 SM, so every lane is co-resident
constexpr size_t kPipeSigOff = kSigWords;
constexpr size_t kPipeSigWords = 4 * (size_t)kPipeLanes * kMaxRanks;
constexpr size_t kSigWordsTotal = kSigWords + kPipeSigWords;
constexpr size_t kPipeEpochOff = kEpochWords;
// Adasum (adasum.cu): counter + generation word of the barrier between the CTAs of one rank's grid
constexpr size_t kAdaEpochOff = kEpochWords + 4 * (size_t)kPipeLanes;
constexpr size_t kEpochWordsTotal = kAdaEpochOff + 2;

enum : int { OP_SUM = 0, OP_MAX = 1, OP_MIN = 2 };

struct DevComm {
  int rank;
  int world;
  uint32_t* sig[kMaxRanks];  // signal pad of every rank, mapped in this process
  uint32_t* epoch;           // local counters, kEpochWords
  int* err;                  // pinned host word, set non-zero on a device-side timeout
  unsigned long long timeout_ns;
};

struct Win {
  char* p[kMaxRanks];  // base of the (window + offset) region on every rank
  char* mc;            // multicast alias of the same region, or nullptr
};

// ---------------------------------------------------------------- flags ----
__device__ __forceinline__ void st_release_sys(uint32_t* p, uint32_t v) {
  asm volatile("st.release.sys.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_sys(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ void st_release_gpu(uint32_t* p, uint32_t v) {
  asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_gpu(const uint32_t* p) {
  uint32_t v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
__device__ __forceinline__ unsigned long long globaltimer_ns() {
  unsigned long long t;
  asm volatile("mov.u64 %0, %globaltimer;" : "=l"(t));
  return t;
}

// Cross-rank barrier between the CTAs with the same blockIdx.x on every rank.
// Called by all threads of the CTA. Thread p signals rank p's pad slot
// [block][my rank] with a release at .sys scope (cumulative over the CTA's
// earlier peer stores through the bar.sync) and spins with .sys acquires on
// its own slot [block][p]. Epochs only grow, so no reset traffic is needed and
// a late waiter can never miss a signal.
__device__ __forceinline__ void rank_barrier(const DevComm& c, uint32_t epoch) {
  __syncthreads();
  if (threadIdx.x < (unsigned)c.world) {
    const int peer = threadIdx.x;
    st_release_sys(c.sig[peer] + (size_t)blockIdx.x * kMaxRanks + c.rank, epoch);
    const uint32_t* mine = c.sig[c.rank] + (size_t)blockIdx.x * kMaxRanks + peer;
    unsigned long long t0 = 0;
    uint32_t spins = 0;
    while ((int32_t)(ld_acquire_sys(mine) - epoch) < 0) {
      if ((++spins & 0x3ffu) == 0) {  // watchdog (SURVEY.md §5.3): never hang the box
        unsigned long long now = globaltimer_ns();
        if (t0 == 0) t0 = now;
        else if (now - t0 > c.timeout_ns) {
          *c.err = 1 + peer;
          break;
        }
      }
    }
  }
  __syncthreads();
}

// One-directional variants of the barrier for pipelines: `flag_signal_all` publishes `value` in slot [src = me] of
// every rank's flag row (after the CTA's earlier stores, ordered by the bar.sync), `flag_wait_all` waits until every
// rank's slot of MY row reached `value`. `row` is the word offset of the row inside the signal pad.
__device__ __forceinline__ void flag_signal_all(const DevComm& c, size_t row, uint32_t value) {
  __syncthreads();
  if (threadIdx.x < (unsigned)c.world) st_release_sys(c.sig[threadIdx.x] + row + c.rank, value);
}
__device__ __forceinline__ void flag_wait_all(const DevComm& c, size_t row, uint32_t value) {
  if (threadIdx.x < (unsigned)c.world) {
    const int peer = threadIdx.x;
    const uint32_t* mine = c.sig[c.rank] + row + peer;
    unsigned long long t0 = 0;
    uint32_t spins = 0;
    while ((int32_t)(ld_acquire_sys(mine) - value) < 0) {
      if ((++spins & 0x3ffu) == 0) {
        unsigned long long now = globaltimer_ns();
        if (t0 == 0) t0 = now;
        else if (now - t0 > c.timeout_ns) { *c.err = 1 + peer; break; }
      }
    }
  }
  __syncthreads();
}
// same-GPU counter written by another CTA of this kernel
__device__ __forceinline__ void local_wait(const DevComm& c, const uint32_t* p, uint32_t value) {
  if (threadIdx.x == 0) {
    unsigned long long t0 = 0;
    uint32_t spins = 0;
    while ((int32_t)(ld_acquire_gpu(p) - value) < 0) {
      if ((++spins & 0x3ffu) == 0) {
        unsigned long long now = globaltimer_ns();
        if (t0 == 0) t0 = now;
        else if (now - t0 > c.timeout_ns) { *c.err = 1 + c.rank; break; }
      }
    }
  }
  __syncthreads();
}

// ------------------------------------------------------------ 128-bit IO ----
__device__ __forceinline__ uint4 ld_sys_v4(const void* p) {
  uint4 v;
  asm volatile("ld.relaxed.sys.global.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p)
               : "memory");
  return v;
}
__device__ __forceinline__ void st_peer_v4(void* p, const uint4& v) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y),
               "r"(v.z), "r"(v.w)
               : "memory");
}
__device__ __forceinline__ uint4 ld_stream_v4(const void* p) {  // local, read-once
  uint4 v;
  asm volatile("ld.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];"
               : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
               : "l"(p)
               : "memory");
  return v;
}

// ---------------------------------------------------- NVLS (multimem.*) ----
template <typename T>
struct MultiMem;
template <>
struct MultiMem<float> {
  static constexpr bool kHasMinMax = false;
  template <int OP>
  static __device__ __forceinline__ uint4 ld_reduce(const void* mc) {
    uint4 v;
    asm volatile("multimem.ld_reduce.relaxed.sys.global.add.v4.f32 {%0,%1,%2,%3}, [%4];"
                 : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w)
                 : "l"(mc)
                 : "memory");
    return v;
  }
};
template <>
struct MultiMem<__nv_bfloat16> {
  static constexpr bool kHasMinMax = true;
  template <int OP>
  static __device__ __forceinline__ uint4 ld_reduce(const void* mc) {
    uint4 v;
    if (OP == OP_SUM)
      asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.bf16x2 {%0,%1,%2,%3}, [%4];"
                   : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(mc) : "memory");
    else if (OP == OP_MAX)
      asm volatile("multimem.ld_reduce.relaxed.sys.global.max.v4.bf16x2 {%0,%1,%2,%3}, [%4];"
                   : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(mc) : "memory");
    else
      asm volatile("multimem.ld_reduce.relaxed.sys.global.min.v4.bf16x2 {%0,%1,%2,%3}, [%4];"
                   : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(mc) : "memory");
    return v;
  }
};
template <>
struct MultiMem<__half> {
  static constexpr bool kHasMinMax = true;
  template <int OP>
  static __device__ __forceinline__ uint4 ld_reduce(const void* mc) {
    uint4 v;
    if (OP == OP_SUM)
      asm volatile("multimem.ld_reduce.relaxed.sys.global.add.acc::f32.v4.f16x2 {%0,%1,%2,%3}, [%4];"
                   : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(mc) : "memory");
    else if (OP == OP_MAX)
      asm volatile("multimem.ld_reduce.relaxed.sys.global.max.v4.f16x2 {%0,%1,%2,%3}, [%4];"
                   : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(mc) : "memory");
    else
      asm volatile("multimem.ld_reduce.relaxed.sys.global.min.v4.f16x2 {%0,%1,%2,%3}, [%4];"
                   : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(mc) : "memory");
    return v;
  }
};
// One store, delivered by the switch to every rank bound to the multicast object.
__device__ __forceinline__ void multimem_st_v4(void* mc, const uint4& v) {
  asm volatile("multimem.st.relaxed.sys.global.v4.f32 [%0], {%1,%2,%3,%4};" ::"l"(mc), "r"(v.x),
               "r"(v.y), "r"(v.z), "r"(v.w)
               : "memory");
}

// ----------------------------------------- fp32-accumulate pack / unpack ----
template <typename T>
struct VecTraits;
template <>
struct VecTraits<float> {
  static constexpr int N = 4;
  static __device__ __forceinline__ void unpack(const uint4& v, float* f) {
    f[0] = __uint_as_float(v.x); f[1] = __uint_as_float(v.y);
    f[2] = __uint_as_float(v.z); f[3] = __uint_as_float(v.w);
  }
  static __device__ __forceinline__ uint4 pack(const float* f) {
    return make_uint4(__float_as_uint(f[0]), __float_as_uint(f[1]), __float_as_uint(f[2]),
                      __float_as_uint(f[3]));
  }
};
template <>
struct VecTraits<__nv_bfloat16> {
  static constexpr int N = 8;
  static __device__ __forceinline__ void unpack(const uint4& v, float* f) {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int i = 0; i < 4; i++) {
      f[2 * i] = __uint_as_float(w[i] << 16);
      f[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
    }
  }
  static __device__ __forceinline__ uint4 pack(const float* f) {
    uint32_t w[4];
#pragma unroll
    for (int i = 0; i < 4; i++) {
      __nv_bfloat162 h = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
      w[i] = *reinterpret_cast<uint32_t*>(&h);
    }
    return make_uint4(w[0], w[1], w[2], w[3]);
  }
};
template <>
struct VecTraits<__half> {
  static constexpr int N = 8;
  static __device__ __forceinline__ void unpack(const uint4& v, float* f) {
    const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
    for (int i = 0; i < 4; i++) {
      float2 t = __half22float2(*reinterpret_cast<const __half2*>(&w[i]));
      f[2 * i] = t.x; f[2 * i + 1] = t.y;
    }
  }
  static __device__ __forceinline__ uint4 pack(const float* f) {
    uint32_t w[4];
#pragma unroll
    for (int i = 0; i < 4; i++) {
      __half2 h = __floats2half2_rn(f[2 * i], f[2 * i + 1]);
      w[i] = *reinterpret_cast<uint32_t*>(&h);
    }
    return make_uint4(w[0], w[1], w[2], w[3]);
  }
};

template <int OP>
__device__ __forceinline__ float red(float a, float b) {
  if (OP == OP_SUM) return a + b;
  if (OP == OP_MAX) return fmaxf(a, b);
  return fminf(a, b);
}

// ------------------------------------ user-pointer <-> staging transfers ----
// Vector index `i` addresses bytes [16 i, 16 i + 16) of a buffer of `nbytes`.
// Fast path: 16-byte aligned base and a full vector. Slow path: byte loop
// (unaligned user pointer or ragged tail); missing bytes read as zero.
__device__ __forceinline__ uint4 user_load(const char* base, size_t i, size_t nbytes, bool aligned) {
  const size_t off = i * 16;
  if (aligned && off + 16 <= nbytes) return ld_stream_v4(base + off);
  uint4 v = make_uint4(0, 0, 0, 0);
  unsigned char* b = reinterpret_cast<unsigned char*>(&v);
  for (int k = 0; k < 16; k++)
    if (off + k < nbytes) b[k] = reinterpret_cast<const unsigned char*>(base)[off + k];
  return v;
}
__device__ __forceinline__ void user_store(char* base, size_t i, size_t nbytes, bool aligned, const uint4& v) {
  const size_t off = i * 16;
  if (aligned && off + 16 <= nbytes) {
    *reinterpret_cast<uint4*>(base + off) = v;
    return;
  }
  const unsigned char* b = reinterpret_cast<const unsigned char*>(&v);
  for (int k = 0; k < 16; k++)
    if (off + k < nbytes) reinterpret_cast<unsigned char*>(base)[off + k] = b[k];
}

}  // namespace b200mpi
