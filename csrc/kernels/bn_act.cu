// Fused BatchNorm(+residual add)+ReLU for channels-last bf16 activations (sm_90a).
//
// Why it exists: in the flagship step's launch list ATen's batch-norm +
// elementwise kernels take most of ResNet-101's device time, more than the
// convolutions (benchmarks/step_timeline.py lists it). The reference delegates the whole model to
// tf_cnn_benchmarks/cuDNN (SURVEY.md §2.5); here the memory-bound glue between
// convolutions is hand-written so every activation tensor is touched the
// minimum number of times:
//   forward : stats pass  (read x)                    + apply pass (read x [,res], write z, 1-bit mask)
//   backward: reduce pass (read dz, x, mask)          + elemt pass (read dz, x, mask, write dx [,dres])
// vs ATen: stats, normalise, (add,) relu  /  relu-bwd, reduce, elemt — 13 T of traffic per BN+ReLU
// layer becomes 8 T, and the extra passes partly hit the 50 MB L2.
//
// Layout: x is [M = N*H*W, C] (channels_last memory), bf16; statistics and
// affine parameters fp32. A thread owns 8 consecutive channels (one 16-byte
// vector); C/8 threads cover a row; a 256-thread CTA covers 2048/C rows per
// pass. Per-channel sums are accumulated in registers with a per-channel shift
// (first row) against cancellation, reduced through shared memory with all
// threads active, stored as one coalesced partial row per CTA (no atomics, no
// fences: a MEMBAR + same-address REDG tail costs microseconds per launch)
// and merged by a tiny finalize kernel —
// deterministic and CUDA-graph capturable.
#include <cuda_bf16.h>
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdlib.h>

#include "../include/b200mpi.h"

namespace b200mpi {
namespace bn {

constexpr int kThreadsBN = 256;
constexpr int kUnroll = 4;

__device__ __forceinline__ void unpack8(const uint4& v, float* f) {
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
  for (int i = 0; i < 4; i++) {
    f[2 * i] = __uint_as_float(w[i] << 16);
    f[2 * i + 1] = __uint_as_float(w[i] & 0xffff0000u);
  }
}
__device__ __forceinline__ uint4 pack8(const float* f) {
  uint32_t w[4];
#pragma unroll
  for (int i = 0; i < 4; i++) {
    __nv_bfloat162 h = __floats2bfloat162_rn(f[2 * i], f[2 * i + 1]);
    w[i] = *reinterpret_cast<uint32_t*>(&h);
  }
  return make_uint4(w[0], w[1], w[2], w[3]);
}
__device__ __forceinline__ uint4 ldg_stream(const uint4* p) {
  uint4 v;
  asm volatile("ld.global.L1::no_allocate.v4.u32 {%0,%1,%2,%3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p));
  return v;
}
__device__ __forceinline__ void stg_stream(uint4* p, const uint4& v) {
  asm volatile("st.global.L1::no_allocate.v4.u32 [%0], {%1,%2,%3,%4};" ::"l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

// workspace layout (floats): coef[4][C] | partials[kMaxParts][2C]
// The reduce-type kernels write one row of per-CTA partial sums (plain coalesced stores: no atomics,
// no fences, deterministic); a tiny finalize kernel merges the rows with all its threads in parallel.
constexpr int kMaxParts = 296;

// Intra-CTA reduction over the `rpp` row-groups, all threads active: output o = cg*16 + 2*j + stat
// is summed over q by thread o (conflict-free smem reads), then stored to this CTA's partial row.
__device__ __forceinline__ void block_reduce_to_partial(float (&s1)[8], float (&s2)[8], float* part_row, int C, int tpr, int r, int cg, int rpp) {
  __shared__ float red[kThreadsBN * 16];
  const int nout = tpr * 16;  // == 2C
#pragma unroll
  for (int j = 0; j < 8; j++) {
    red[r * nout + cg * 16 + 2 * j] = s1[j];
    red[r * nout + cg * 16 + 2 * j + 1] = s2[j];
  }
  __syncthreads();
  for (int o = threadIdx.x; o < nout; o += kThreadsBN) {
    float acc = 0.f;
    for (int q = 0; q < rpp; q++) acc += red[q * nout + o];
    part_row[o] = acc;
  }
}

// Merge `parts` partial rows. The finalize kernels are pure latency (a few KB of L2-resident data, 339 launches per
// ResNet-101 step: 9.2 us each = 3.1 ms in round 1's launch table), so the merge is laid out for the shortest dependent
// chain instead of for coalescing: a CTA owns 8 outputs (32 contiguous bytes per row) and its 256 threads are 32 row
// slots x 8 outputs, each slot walking rows slot, slot+32, ... with 4 loads in flight -> ceil(parts/128) rounds of L2
// latency (3 for the maximum of 296 rows; the 8-warps-x-32-outputs layout needed 10).
// Returns (for threads 0..7) the total for output blockIdx.x*8 + threadIdx.x.
constexpr int kMergeOut = 8;
__device__ __forceinline__ float merge_partials(const float* __restrict__ partials, int parts, int nout, int* out_index) {
  __shared__ float sm[8][kMergeOut + 1];
  const int oi = threadIdx.x & (kMergeOut - 1), slot = threadIdx.x >> 3;   // 32 slots
  const int o = blockIdx.x * kMergeOut + oi;
  float acc = 0.f;
  if (o < nout) {
    const float* p = partials + o;
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
    int b = slot;
    for (; b + 96 < parts; b += 128) {
      a0 += __ldcg(p + (size_t)b * nout);
      a1 += __ldcg(p + (size_t)(b + 32) * nout);
      a2 += __ldcg(p + (size_t)(b + 64) * nout);
      a3 += __ldcg(p + (size_t)(b + 96) * nout);
    }
    for (; b < parts; b += 32) a0 += __ldcg(p + (size_t)b * nout);
    acc = (a0 + a1) + (a2 + a3);
  }
  // the 4 slots of a warp that share an output: lanes oi, oi+8, oi+16, oi+24
  acc += __shfl_xor_sync(0xffffffffu, acc, 8);
  acc += __shfl_xor_sync(0xffffffffu, acc, 16);
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  if (lane < kMergeOut) sm[warp][lane] = acc;
  __syncthreads();
  float tot = 0.f;
  if (threadIdx.x < kMergeOut) {
#pragma unroll
    for (int w = 0; w < 8; w++) tot += sm[w][threadIdx.x];
  }
  *out_index = o;
  return tot;
}

// ---------------------------------------------------------------- forward ----
__global__ void __launch_bounds__(kThreadsBN)
k_bn_fwd_stats(const uint4* __restrict__ x, float* __restrict__ partials, long long M, int C, long long rows_per_cta) {
  const int tpr = C >> 3, rpp = kThreadsBN / tpr;
  const int r = threadIdx.x / tpr, cg = threadIdx.x % tpr;
  float K[8], s1[8], s2[8];
  unpack8(x[cg], K);  // per-channel shift = first row: sums of (x-K) do not cancel catastrophically
#pragma unroll
  for (int j = 0; j < 8; j++) s1[j] = s2[j] = 0.f;
  const long long m0 = (long long)blockIdx.x * rows_per_cta;
  const long long m1 = m0 + rows_per_cta < M ? m0 + rows_per_cta : M;
  for (long long m = m0 + r; m < m1; m += (long long)rpp * kUnroll) {
    uint4 v[kUnroll];
#pragma unroll
    for (int u = 0; u < kUnroll; u++) {
      const long long mm = m + (long long)u * rpp;
      if (mm < m1) v[u] = ldg_stream(x + mm * tpr + cg);
    }
#pragma unroll
    for (int u = 0; u < kUnroll; u++) {
      const long long mm = m + (long long)u * rpp;
      if (mm < m1) {
        float f[8];
        unpack8(v[u], f);
#pragma unroll
        for (int j = 0; j < 8; j++) {
          const float d = f[j] - K[j];
          s1[j] += d;
          s2[j] = fmaf(d, d, s2[j]);
        }
      }
    }
  }
  block_reduce_to_partial(s1, s2, partials + (size_t)blockIdx.x * 2 * C, C, tpr, r, cg, rpp);
}

// grid = ceil(2C/32): merges the partial rows, then the threads owning the (S1,S2) pair of a channel
// produce mean / invstd / running stats / affine coefficients a, b for the apply pass.
__global__ void __launch_bounds__(kThreadsBN)
k_bn_fwd_finalize(const __nv_bfloat16* __restrict__ x_row0, const float* __restrict__ partials, int parts, float* __restrict__ coef,
                  long long M, int C, const float* __restrict__ weight, const float* __restrict__ bias, float* running_mean,
                  float* running_var, float* save_mean, float* save_invstd, float eps, float momentum) {
  int o;
  const float tot = merge_partials(partials, parts, 2 * C, &o);
  if ((threadIdx.x >> 5) != 0) return;
  const float other = __shfl_xor_sync(0xffffffffu, tot, 1);  // lanes 2j / 2j+1 hold S1 / S2 of one channel
  if (threadIdx.x >= kMergeOut || o >= 2 * C || (o & 1)) return;
  const int cgi = o >> 4, j = (o & 15) >> 1, c = cgi * 8 + j;
  const float S1 = tot, S2 = other;
  const float inv_m = 1.0f / (float)M;
  const float k = x_row0 ? __bfloat162float(x_row0[c]) : 0.f;  // nullptr: partials are plain (unshifted) sums
  const float d = S1 * inv_m;
  const float mean = k + d;
  float var = fmaf(-d, d, S2 * inv_m);
  var = var > 0.f ? var : 0.f;
  const float invstd = rsqrtf(var + eps);
  save_mean[c] = mean;
  save_invstd[c] = invstd;
  if (running_mean) {
    running_mean[c] = (1.f - momentum) * running_mean[c] + momentum * mean;
    const float unbiased = M > 1 ? var * ((float)M / (float)(M - 1)) : var;
    running_var[c] = (1.f - momentum) * running_var[c] + momentum * unbiased;
  }
  const float a = (weight ? weight[c] : 1.f) * invstd;
  coef[c] = a;
  coef[C + c] = (bias ? bias[c] : 0.f) - mean * a;
}

template <bool RELU, bool RES>
__global__ void __launch_bounds__(kThreadsBN)
k_bn_fwd_apply(const uint4* __restrict__ x, const uint4* __restrict__ res, uint4* __restrict__ y, uint8_t* __restrict__ mask,
               const float* __restrict__ coef, long long M, int C, long long rows_per_cta) {
  const int tpr = C >> 3, rpp = kThreadsBN / tpr;
  const int r = threadIdx.x / tpr, cg = threadIdx.x % tpr;
  float a[8], b[8];
#pragma unroll
  for (int j = 0; j < 8; j++) {
    a[j] = coef[cg * 8 + j];
    b[j] = coef[C + cg * 8 + j];
  }
  const long long m0 = (long long)blockIdx.x * rows_per_cta;
  const long long m1 = m0 + rows_per_cta < M ? m0 + rows_per_cta : M;
  for (long long m = m0 + r; m < m1; m += (long long)rpp * kUnroll) {
    uint4 v[kUnroll], w[kUnroll];
#pragma unroll
    for (int u = 0; u < kUnroll; u++) {
      const long long mm = m + (long long)u * rpp;
      if (mm < m1) {
        v[u] = ldg_stream(x + mm * tpr + cg);
        if (RES) w[u] = ldg_stream(res + mm * tpr + cg);
      }
    }
#pragma unroll
    for (int u = 0; u < kUnroll; u++) {
      const long long mm = m + (long long)u * rpp;
      if (mm < m1) {
        float f[8], g[8];
        unpack8(v[u], f);
        if (RES) unpack8(w[u], g);
        unsigned bits = 0;
#pragma unroll
        for (int j = 0; j < 8; j++) {
          float z = fmaf(a[j], f[j], b[j]);
          if (RES) z += g[j];
          if (RELU) {
            bits |= (z > 0.f ? 1u : 0u) << j;
            z = z > 0.f ? z : 0.f;
          }
          f[j] = z;
        }
        stg_stream(y + mm * tpr + cg, pack8(f));
        if (RELU) mask[mm * tpr + cg] = (uint8_t)bits;
      }
    }
  }
}

// --------------------------------------------------------------- backward ----
template <bool RELU>
__global__ void __launch_bounds__(kThreadsBN)
k_bn_bwd_reduce(const uint4* __restrict__ dz, const uint4* __restrict__ x, const uint8_t* __restrict__ mask, float* __restrict__ partials,
                long long M, int C, long long rows_per_cta, const float* __restrict__ save_mean) {
  const int tpr = C >> 3, rpp = kThreadsBN / tpr;
  const int r = threadIdx.x / tpr, cg = threadIdx.x % tpr;
  float mu[8], s1[8], s2[8];
#pragma unroll
  for (int j = 0; j < 8; j++) {
    mu[j] = save_mean[cg * 8 + j];
    s1[j] = s2[j] = 0.f;
  }
  const long long m0 = (long long)blockIdx.x * rows_per_cta;
  const long long m1 = m0 + rows_per_cta < M ? m0 + rows_per_cta : M;
  for (long long m = m0 + r; m < m1; m += (long long)rpp * kUnroll) {
    uint4 g4[kUnroll], x4[kUnroll];
    unsigned mk[kUnroll];
#pragma unroll
    for (int u = 0; u < kUnroll; u++) {
      const long long mm = m + (long long)u * rpp;
      if (mm < m1) {
        g4[u] = ldg_stream(dz + mm * tpr + cg);
        x4[u] = ldg_stream(x + mm * tpr + cg);
        mk[u] = RELU ? mask[mm * tpr + cg] : 0xffu;
      }
    }
#pragma unroll
    for (int u = 0; u < kUnroll; u++) {
      const long long mm = m + (long long)u * rpp;
      if (mm < m1) {
        float g[8], f[8];
        unpack8(g4[u], g);
        unpack8(x4[u], f);
#pragma unroll
        for (int j = 0; j < 8; j++) {
          const float gj = (mk[u] >> j) & 1u ? g[j] : 0.f;
          s1[j] += gj;
          s2[j] = fmaf(gj, f[j] - mu[j], s2[j]);  // * invstd applied once at finalise
        }
      }
    }
  }
  block_reduce_to_partial(s1, s2, partials + (size_t)blockIdx.x * 2 * C, C, tpr, r, cg, rpp);
}

__global__ void __launch_bounds__(kThreadsBN)
k_bn_bwd_finalize(const float* __restrict__ partials, int parts, float* __restrict__ coef, long long M, int C,
                  const float* __restrict__ weight, const float* __restrict__ save_mean, const float* __restrict__ save_invstd,
                  float* dweight, float* dbias) {
  int o;
  const float tot = merge_partials(partials, parts, 2 * C, &o);
  if ((threadIdx.x >> 5) != 0) return;
  const float other = __shfl_xor_sync(0xffffffffu, tot, 1);
  if (threadIdx.x >= kMergeOut || o >= 2 * C || (o & 1)) return;
  const int cgi = o >> 4, j = (o & 15) >> 1, c = cgi * 8 + j;
  const float inv_m = 1.0f / (float)M;
  const float invstd = save_invstd[c];
  const float S1 = tot, S2 = other * invstd;  // sum g, sum g * xhat
  if (dbias) dbias[c] = S1;
  if (dweight) dweight[c] = S2;
  coef[c] = (weight ? weight[c] : 1.f) * invstd;  // a
  coef[C + c] = S1 * inv_m;                        // mean(g)
  coef[2 * C + c] = S2 * inv_m * invstd;           // mean(g*xhat) * invstd
  coef[3 * C + c] = save_mean[c];
}

template <bool RELU, bool RES>
__global__ void __launch_bounds__(kThreadsBN)
k_bn_bwd_elemt(const uint4* __restrict__ dz, const uint4* __restrict__ x, const uint8_t* __restrict__ mask, uint4* __restrict__ dx,
               uint4* __restrict__ dres, const float* __restrict__ coef, long long M, int C, long long rows_per_cta) {
  const int tpr = C >> 3, rpp = kThreadsBN / tpr;
  const int r = threadIdx.x / tpr, cg = threadIdx.x % tpr;
  float a[8], gm[8], c3[8], mu[8];
#pragma unroll
  for (int j = 0; j < 8; j++) {
    a[j] = coef[cg * 8 + j];
    gm[j] = coef[C + cg * 8 + j];
    c3[j] = coef[2 * C + cg * 8 + j];
    mu[j] = coef[3 * C + cg * 8 + j];
  }
  const long long m0 = (long long)blockIdx.x * rows_per_cta;
  const long long m1 = m0 + rows_per_cta < M ? m0 + rows_per_cta : M;
  for (long long m = m0 + r; m < m1; m += (long long)rpp * kUnroll) {
    uint4 g4[kUnroll], x4[kUnroll];
    unsigned mk[kUnroll];
#pragma unroll
    for (int u = 0; u < kUnroll; u++) {
      const long long mm = m + (long long)u * rpp;
      if (mm < m1) {
        g4[u] = ldg_stream(dz + mm * tpr + cg);
        x4[u] = ldg_stream(x + mm * tpr + cg);
        mk[u] = RELU ? mask[mm * tpr + cg] : 0xffu;
      }
    }
#pragma unroll
    for (int u = 0; u < kUnroll; u++) {
      const long long mm = m + (long long)u * rpp;
      if (mm < m1) {
        float g[8], f[8];
        unpack8(g4[u], g);
        unpack8(x4[u], f);
#pragma unroll
        for (int j = 0; j < 8; j++) {
          const float gj = (mk[u] >> j) & 1u ? g[j] : 0.f;
          g[j] = gj;                                              // gradient w.r.t. the residual branch
          f[j] = a[j] * (gj - gm[j] - (f[j] - mu[j]) * c3[j]);    // gradient w.r.t. the BN input
        }
        stg_stream(dx + mm * tpr + cg, pack8(f));
        if (RES) stg_stream(dres + mm * tpr + cg, pack8(g));
      }
    }
  }
}

static long long env_chunk(const char* name, long long dflt) {
  const char* v = getenv(name);
  return v && *v ? atoll(v) : dflt;
}
static long long reduce_chunk() { static long long v = env_chunk("B200MPI_BN_REDUCE_CHUNK", 64 << 10); return v; }
static long long elem_chunk() { static long long v = env_chunk("B200MPI_BN_ELEM_CHUNK", 64 << 10); return v; }

static void plan(long long M, int C, int cap, long long bytes_per_row, int* grid, long long* rows_per_cta, long long chunk) {
  const int tpr = C / 8, rpp = kThreadsBN / tpr;
  const long long min_rows = (long long)rpp * kUnroll;
  // >= `chunk` bytes of traffic per CTA: reduce-type kernels use 128 KiB (few partial rows to merge),
  // elementwise passes 32 KiB (more CTAs in flight, nothing to merge)
  long long by_bytes = (M * bytes_per_row + chunk - 1) / chunk;
  long long g = (M + min_rows - 1) / min_rows;
  if (g > by_bytes) g = by_bytes;
  if (g > cap) g = cap;
  if (g < 1) g = 1;
  long long rows = (M + g - 1) / g;
  rows = (rows + rpp - 1) / rpp * rpp;
  g = (M + rows - 1) / rows;
  *grid = (int)g;
  *rows_per_cta = rows;
}

}  // namespace bn
}  // namespace b200mpi

using namespace b200mpi::bn;

extern "C" {

size_t b200mpi_bn_workspace_floats(int C) { return (size_t)4 * C + (size_t)kMaxParts * 2 * C + 4; }

int b200mpi_bn_supported(long long M, int C) { return (C % 8 == 0 && C >= 8 && C / 8 <= kThreadsBN && kThreadsBN % (C / 8) == 0 && M >= 1) ? 1 : 0; }

int b200mpi_bn_act_fwd(const void* x, const void* residual, void* y, void* mask, const float* weight, const float* bias,
                       float* running_mean, float* running_var, float* save_mean, float* save_invstd, float* workspace,
                       long long M, int C, float eps, float momentum, int relu, void* stream_) {
  if (!b200mpi_bn_supported(M, C)) return B200MPI_ERR_UNSUPPORTED;
  cudaStream_t s = (cudaStream_t)stream_;
  float* coef = workspace;
  float* partials = workspace + 4 * C;
  int grid;
  long long rows;
  plan(M, C, kMaxParts, 2LL * C, &grid, &rows, reduce_chunk());
  k_bn_fwd_stats<<<grid, kThreadsBN, 0, s>>>((const uint4*)x, partials, M, C, rows);
  k_bn_fwd_finalize<<<(2 * C + kMergeOut - 1) / kMergeOut, kThreadsBN, 0, s>>>((const __nv_bfloat16*)x, partials, grid, coef, M, C, weight, bias,
                                                            running_mean, running_var, save_mean, save_invstd, eps, momentum);
  plan(M, C, 1184, (residual ? 6LL : 4LL) * C, &grid, &rows, elem_chunk());
  if (relu && residual) k_bn_fwd_apply<true, true><<<grid, kThreadsBN, 0, s>>>((const uint4*)x, (const uint4*)residual, (uint4*)y, (uint8_t*)mask, coef, M, C, rows);
  else if (relu) k_bn_fwd_apply<true, false><<<grid, kThreadsBN, 0, s>>>((const uint4*)x, nullptr, (uint4*)y, (uint8_t*)mask, coef, M, C, rows);
  else if (residual) k_bn_fwd_apply<false, true><<<grid, kThreadsBN, 0, s>>>((const uint4*)x, (const uint4*)residual, (uint4*)y, nullptr, coef, M, C, rows);
  else k_bn_fwd_apply<false, false><<<grid, kThreadsBN, 0, s>>>((const uint4*)x, nullptr, (uint4*)y, nullptr, coef, M, C, rows);
  return cudaGetLastError() == cudaSuccess ? 0 : B200MPI_ERR_CUDA;
}

// Forward with the statistics already reduced to `parts` rows of per-channel {sum, sum of squares} (unshifted) by the
// producer of x — the epilogue of the wgmma 1x1-convolution GEMM (gemm_bnstats.cu): finalize + apply only, the
// statistics pass over x is gone.
int b200mpi_bn_act_fwd_prestats(const void* x, const void* residual, void* y, void* mask, const float* weight, const float* bias,
                                float* running_mean, float* running_var, float* save_mean, float* save_invstd, float* workspace,
                                const float* partials, int parts, long long M, int C, float eps, float momentum, int relu,
                                void* stream_) {
  if (!b200mpi_bn_supported(M, C) || parts < 1 || !partials) return B200MPI_ERR_UNSUPPORTED;
  cudaStream_t s = (cudaStream_t)stream_;
  float* coef = workspace;
  int grid;
  long long rows;
  k_bn_fwd_finalize<<<(2 * C + kMergeOut - 1) / kMergeOut, kThreadsBN, 0, s>>>(nullptr, partials, parts, coef, M, C, weight, bias, running_mean,
                                                            running_var, save_mean, save_invstd, eps, momentum);
  plan(M, C, 1184, (residual ? 6LL : 4LL) * C, &grid, &rows, elem_chunk());
  if (relu && residual) k_bn_fwd_apply<true, true><<<grid, kThreadsBN, 0, s>>>((const uint4*)x, (const uint4*)residual, (uint4*)y, (uint8_t*)mask, coef, M, C, rows);
  else if (relu) k_bn_fwd_apply<true, false><<<grid, kThreadsBN, 0, s>>>((const uint4*)x, nullptr, (uint4*)y, (uint8_t*)mask, coef, M, C, rows);
  else if (residual) k_bn_fwd_apply<false, true><<<grid, kThreadsBN, 0, s>>>((const uint4*)x, (const uint4*)residual, (uint4*)y, nullptr, coef, M, C, rows);
  else k_bn_fwd_apply<false, false><<<grid, kThreadsBN, 0, s>>>((const uint4*)x, nullptr, (uint4*)y, nullptr, coef, M, C, rows);
  return cudaGetLastError() == cudaSuccess ? 0 : B200MPI_ERR_CUDA;
}

int b200mpi_bn_act_bwd(const void* dz, const void* x, const void* mask, void* dx, void* dres, const float* weight,
                       const float* save_mean, const float* save_invstd, float* dweight, float* dbias, float* workspace,
                       long long M, int C, int relu, void* stream_) {
  if (!b200mpi_bn_supported(M, C)) return B200MPI_ERR_UNSUPPORTED;
  cudaStream_t s = (cudaStream_t)stream_;
  float* coef = workspace;
  float* partials = workspace + 4 * C;
  int grid;
  long long rows;
  plan(M, C, kMaxParts, 4LL * C, &grid, &rows, reduce_chunk());
  if (relu) k_bn_bwd_reduce<true><<<grid, kThreadsBN, 0, s>>>((const uint4*)dz, (const uint4*)x, (const uint8_t*)mask, partials, M, C, rows, save_mean);
  else k_bn_bwd_reduce<false><<<grid, kThreadsBN, 0, s>>>((const uint4*)dz, (const uint4*)x, nullptr, partials, M, C, rows, save_mean);
  k_bn_bwd_finalize<<<(2 * C + kMergeOut - 1) / kMergeOut, kThreadsBN, 0, s>>>(partials, grid, coef, M, C, weight, save_mean, save_invstd, dweight, dbias);
  plan(M, C, 1184, (dres ? 8LL : 6LL) * C, &grid, &rows, elem_chunk());
  if (relu && dres) k_bn_bwd_elemt<true, true><<<grid, kThreadsBN, 0, s>>>((const uint4*)dz, (const uint4*)x, (const uint8_t*)mask, (uint4*)dx, (uint4*)dres, coef, M, C, rows);
  else if (relu) k_bn_bwd_elemt<true, false><<<grid, kThreadsBN, 0, s>>>((const uint4*)dz, (const uint4*)x, (const uint8_t*)mask, (uint4*)dx, nullptr, coef, M, C, rows);
  else if (dres) k_bn_bwd_elemt<false, true><<<grid, kThreadsBN, 0, s>>>((const uint4*)dz, (const uint4*)x, nullptr, (uint4*)dx, (uint4*)dres, coef, M, C, rows);
  else k_bn_bwd_elemt<false, false><<<grid, kThreadsBN, 0, s>>>((const uint4*)dz, (const uint4*)x, nullptr, (uint4*)dx, nullptr, coef, M, C, rows);
  return cudaGetLastError() == cudaSuccess ? 0 : B200MPI_ERR_CUDA;
}

}  // extern "C"
