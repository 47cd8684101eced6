// Host-visible launch interface of the b200mpi collective kernels.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

#include "device.cuh"

namespace b200mpi {

struct KArgs {
  DevComm c;
  Win buf;          // staging region or symmetric user region (per-rank bases)
  // The grouped fused SGD reads no user pointers, so its two tables share these slots: KArgs keeps its size, and with
  // it the stride of the emulated ranks' argument array that every kernel indexes.
  union {
    const char* in;        // user input  (nullptr: data already in buf)
    const uint8_t* gmap;   // grouped SGD: group id of each fp32 vector of the region, indexed like `buf`
  };
  union {
    char* out;             // user output (nullptr: result stays in buf)
    const float* ghyper;   // grouped SGD: device table [G][3] of {lr, mu, wd}
  };
  size_t nbytes;    // payload bytes of one logical unit (op specific)
  size_t nvec;      // 16-byte vectors in the logical buffer
  size_t per;       // vectors per rank slice / slot
  // The weight average of the fused SGD / LARS steps shares this slot and `dbg` with fields those kernels never read:
  // appending them would grow KArgs, which moves the `emu` parameter and the emulated-args stride of every kernel.
  union {
    size_t ustride;   // byte stride between per-rank blocks in the user buffer
    float* ema;       // fused SGD / LARS with EMA: this rank's EMA slice, indexed like `mom`
  };
  float scale;
  int op;
  int root;
  int in_aligned;
  int out_aligned;
  // fused allreduce+SGD
  Win param;        // fp32 parameter window region
  Win lowp;         // optional bf16 parameter shadow (p[0]==nullptr: absent)
  float* mom;       // this rank's momentum slice
  float lr, mu, wd;
  const float* hyper;  // optional device {lr, mu, wd}: lets a captured CUDA graph follow LR schedules
  int nesterov;
  int first_step;
  // pipelined staged allreduce: lanes x {copy-in, reduce, copy-out} CTAs, `depth` staging slots of `per` vectors per lane
  int lanes;
  int depth;
  union {
    unsigned long long* dbg;   // optional timeline: [role 3][lane kPipeLanes][chunk kPipeDbgChunks][3] globaltimer ns
    const double* ema_sched;   // fused SGD / LARS with EMA: device {decay, updates so far} (ema_coef)
  };
};
constexpr int kPipeDbgChunks = 32;

struct Launch {
  cudaStream_t stream;
  int blocks;             // gridDim.x
  int emu_world;          // 0: real multi-process rank; >0: gridDim.y virtual ranks
  const KArgs* emu_args;  // device array of emu_world KArgs (emulated mode)
};

// ---- point-to-point (p2p.cu) -------------------------------------------------------------------------------------
constexpr size_t kP2PChunk = (size_t)1 << 20;                  // mailbox slot size
constexpr size_t kP2PDataBytes = (size_t)kMaxRanks * 2 * kP2PChunk;   // [src rank][2 slots]
constexpr int kP2PFlagStride = 32;                             // u32 words between flags: one 128-byte line each
constexpr size_t kP2PFlagBytes = (size_t)2 * kMaxRanks * 2 * kP2PFlagStride * sizeof(uint32_t);  // READY + ACK
constexpr size_t kP2PWindowBytes = kP2PDataBytes + kP2PFlagBytes;
constexpr int kMaxP2POps = 64;
enum : int { P2P_READY = 0, P2P_ACK = 1 };
// flag of slot 0 for stream (kind, r) inside the mailbox window whose base is `win`; slot 1 is kP2PFlagStride words on
__host__ __device__ inline uint32_t* p2p_flag(char* win, int kind, int r) {
  return reinterpret_cast<uint32_t*>(win + kP2PDataBytes) + ((size_t)kind * kMaxRanks + r) * 2 * kP2PFlagStride;
}
struct P2POp {
  const char* user;   // send: source buffer; receive: destination buffer
  size_t bytes;
  int peer;
  int is_send;
  uint32_t seq_off;   // chunks of earlier operations of this batch on the same (direction, peer) stream
};
struct P2PArgs {
  DevComm c;
  Win box;            // mailbox window of every rank
  uint32_t* cnt;      // device counters: [0,kMaxRanks) chunks sent to peer, [kMaxRanks, 2*kMaxRanks) chunks received from peer
  int nops;
  P2POp ops[kMaxP2POps];
};
struct P2PCommit { uint32_t n[2 * kMaxRanks]; };
cudaError_t launch_p2p_batch(cudaStream_t s, const P2PArgs& a, const P2PCommit& add);

enum : int { DT_F32 = 0, DT_BF16 = 1, DT_F16 = 2 };
enum : int { MODE_P2P = 0, MODE_NVLS = 1 };

// a = args of this rank (ignored in emulated mode where l.emu_args is used)
cudaError_t launch_allreduce_twoshot(const Launch& l, const KArgs& a, int dtype, int mode, bool staged);
enum : int { PIPE_ALLREDUCE = 0, PIPE_ALLGATHER = 1, PIPE_REDUCE_SCATTER = 2, PIPE_BROADCAST = 3 };
cudaError_t launch_pipe(const Launch& l, const KArgs& a, int kind, int dtype, int mode);
cudaError_t launch_allreduce_oneshot(const Launch& l, const KArgs& a, int dtype);
cudaError_t launch_allreduce_sgd(const Launch& l, const KArgs& a, int dtype, int mode);
// per-vector hyper-parameters from a.gmap / a.ghyper; fp32 gradients only
cudaError_t launch_allreduce_sgd_groups(const Launch& l, const KArgs& a, int mode);
// fp32 gradients, grouped or not (a.gmap), plus the weight average in a.ema / a.ema_sched
cudaError_t launch_allreduce_sgd_ema(const Launch& l, const KArgs& a, int mode, bool groups);
cudaError_t launch_allgather(const Launch& l, const KArgs& a);
cudaError_t launch_allgather_sym(const Launch& l, const KArgs& a, int mode);
cudaError_t launch_broadcast_sym(const Launch& l, const KArgs& a, int mode);
cudaError_t launch_reduce_scatter_sym(const Launch& l, const KArgs& a, int dtype, int mode);
cudaError_t launch_broadcast(const Launch& l, const KArgs& a, int mode);
cudaError_t launch_reduce_scatter(const Launch& l, const KArgs& a, int dtype);
cudaError_t launch_reduce(const Launch& l, const KArgs& a, int dtype);
cudaError_t launch_alltoall(const Launch& l, const KArgs& a);
cudaError_t launch_barrier(const Launch& l, const KArgs& a);
// Adasum (adasum.cu). Staging layout behind a.buf: [dot board kAdaDotBytes][A: world*per vectors of T][W: world*per vectors as fp32]
constexpr int kAdaMaxBlocks = 64;                                   // CTAs per rank (all co-resident: spin barriers)
constexpr size_t kAdaDotBytes = (size_t)96 << 10;                   // >= (kMaxRanks-1) pairs x kMaxRanks x kAdaMaxBlocks x 3 doubles
static_assert((size_t)(kMaxRanks - 1) * kMaxRanks * kAdaMaxBlocks * 3 * sizeof(double) <= kAdaDotBytes, "dot board too small");
cudaError_t launch_adasum(const Launch& l, const KArgs& a, int dtype);
// Fused allreduce + LARS (lars.cu): fp32 gradients, the group table of the grouped SGD, two launches per bucket.
constexpr int kLarsMaxParams = 1024;    // parameters per bucket (the trust ratios live in shared memory)
constexpr float kLarsEps = 1e-8f;
struct LarsArgs {
  const uint16_t* pmap;           // bucket-local parameter of each fp32 vector, indexed like KArgs::buf; non-decreasing,
                                  // bucket tails P
  const uint8_t* ptab;            // [P][2] {group, lars} of each parameter
  const float* ghyper;            // [G][3] {lr, mu, wd}
  Win board;                      // [P][world] float2 {sum g^2, sum w^2} on every rank
  char* scratch[kMaxRanks];       // per-rank scratch of lars_scratch_bytes (real mode: only [rank] is set)
  float* trust_out[kMaxRanks];    // optional [P] trust ratios per rank
  float eta;
  int P;
};
size_t lars_scratch_bytes(size_t per, int P);
cudaError_t launch_lars_norms(const Launch& l, const KArgs& a, const LarsArgs& L, int mode);
cudaError_t launch_lars_update(const Launch& l, const KArgs& a, const LarsArgs& L, int mode, bool ema = false);
// Learning-rate schedule (lr_schedule.cu): one CTA; reads the step count, writes each group's rate, stores count + 1.
enum : int { LR_CONSTANT = 0, LR_PIECEWISE = 1, LR_EXPONENTIAL = 2, LR_POLYNOMIAL = 3 };
constexpr int kLrMaxBoundaries = 64;
constexpr int kLrMaxGroups = 256;
cudaError_t launch_lr_schedule(cudaStream_t s, const double* sched, int form, int nb, long long* step, const double* base,
                               int G, float* hyper, float* group_hyper);
cudaError_t launch_scale_cast(cudaStream_t s, const void* in, int in_dt, void* out, int out_dt,
                              size_t count, float scale);
cudaError_t launch_fill_u32(cudaStream_t s, uint32_t* p, uint32_t v, size_t n);

}  // namespace b200mpi
