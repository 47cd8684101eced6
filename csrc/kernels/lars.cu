// Fused gradient allreduce + LARS (You et al., 2017, "Large Batch Training of Convolutional Networks") for sm_90a.
//
// LARS is the grouped momentum SGD of k_allreduce_sgd with one extra factor per parameter tensor, the trust ratio
//
//   trust = eta * |w| / (|g| + wd * |w| + eps)     (1 when |w| or |g| is 0; eps = kLarsEps)
//   d = trust * (g + wd * w);   m = mu * m + d;   w -= lr * (nesterov ? d + mu * m : m)
//
// where g is the world-averaged gradient. No rank holds a whole layer's averaged gradient (rank r owns slice r of every
// bucket), so the norms need a cross-rank exchange before the update, and the step runs as two launches:
//
//   k_allreduce_lars_norms  entry barrier; the same slice loads and rank order of the sum as k_allreduce_sgd; the unscaled
//                           fp32 sum of the owned slice goes to a per-rank scratch (p.grad keeps its meaning); per
//                           bucket-local parameter the partial sum(scale*g)^2 and sum(w^2) over the slice. Per warp the
//                           partials are a segmented shuffle scan over 32 consecutive vectors (the parameter map is sorted),
//                           added to a per-warp row in shared memory; per CTA the warp rows are summed in warp order into a
//                           partial row in scratch. The last CTA to take a ticket (not a barrier: nobody waits for it)
//                           sums the CTA rows in CTA order and pushes this rank's [P][2] row into slot [p][rank] of every
//                           rank's norm board; it resets the ticket. Exit barrier: every board is complete.
//   k_lars_update           every CTA sums the board over ranks 0..world-1 and computes trust[P] in shared memory (the same
//                           bits on every CTA of every rank), then runs the update of k_allreduce_sgd<float, MODE, true>
//                           over the owned slice from the stored sum, pushes parameters and the bf16 shadow to every peer,
//                           and ends with a barrier (peers may read their parameters afterwards).
//
// Every sum has a fixed order and there are no float atomics, so all ranks and all runs agree bit for bit. For vectors of
// non-LARS parameters trust is exactly 1 and the update is written with the FMAs k_allreduce_sgd compiles to, so they come
// out bitwise equal to the grouped kernel.
//
// The trust contract, in fp32 throughout (tests/optimizer_oracle.py states it on the host), with S the fp32 sum of the
// ranks' gradients as in k_allreduce_sgd:
//   gs = fp32(S * scale)
//   sg, sp = fp32 sums of fmaf(gs, gs, .) / fmaf(w, w, .) over the parameter's elements of each slice, then over ranks
//            0..world-1 (the order within a slice follows the grid: the host can only bound it)
//   gn = sqrtf(sg), wn = sqrtf(sp)
//   t  = (wn > 0 && gn > 0) ? fdiv(fmul(eta, wn), fadd(fmaf(wd, wn, gn), kLarsEps)) : 1
//   d  = fmul(t, fmaf(S, scale, fmul(wd, p)))
// so NaN norms give t = 1 and an fp32 overflow of sg (gn = inf) gives t = 0.
//
// Extra HBM traffic over k_allreduce_sgd per rank: one read of the parameter slice (norms) and one write + one read of the
// sum scratch: 3 * S / world for S bytes of fp32 parameters.
#include "kernels.h"

namespace b200mpi {

#define EMU_ARGS const KArgs& a = (emu != nullptr) ? emu[blockIdx.y] : a0

constexpr int kLarsWarps = kThreads / 32;

__device__ __forceinline__ int lars_wrap(int x, int world) { return x >= world ? x - world : x; }
__device__ __forceinline__ size_t lars_gstride() { return (size_t)gridDim.x * blockDim.x; }

// Layout of one rank's scratch (lars_scratch_bytes): ticket, CTA partial rows [kMaxBlocks][P] of float2, slice sums.
__host__ __device__ inline size_t lars_rows_off() { return 256; }
__host__ __device__ inline size_t lars_sum_off(int P) { return lars_rows_off() + (((size_t)kMaxBlocks * P * 8 + 255) / 256) * 256; }
size_t lars_scratch_bytes(size_t per, int P) { return lars_sum_off(P) + per * 16; }
size_t lars_norms_smem(int P) { return (size_t)kLarsWarps * P * sizeof(float2); }

template <int MODE>
__global__ void __launch_bounds__(kThreads)
k_allreduce_lars_norms(const __grid_constant__ KArgs a0, const KArgs* __restrict__ emu, const __grid_constant__ LarsArgs L) {
  EMU_ARGS;
  extern __shared__ float2 lars_acc[];   // [warp][P]: this warp's partial {sum (scale g)^2, sum w^2} of each parameter
  const int rank = a.c.rank, world = a.c.world, P = L.P;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  uint32_t e = a.c.epoch[blockIdx.x];
  const size_t per = a.per, nvec = a.nvec;
  char* const scr = L.scratch[rank];
  uint32_t* const ticket = reinterpret_cast<uint32_t*>(scr);
  float2* const rows = reinterpret_cast<float2*>(scr + lars_rows_off());
  float* const sums = reinterpret_cast<float*>(scr + lars_sum_off(P));
  for (int k = threadIdx.x; k < kLarsWarps * P; k += blockDim.x) lars_acc[k] = make_float2(0.f, 0.f);
  rank_barrier(a.c, ++e);   // its __syncthreads also orders the zeroing before the first add

  const size_t base = (size_t)rank * per;
  const size_t lim = base < nvec ? (nvec - base < per ? nvec - base : per) : 0;
  const char* gmc = a.buf.mc ? a.buf.mc + base * 16 : nullptr;
  const float* pl = reinterpret_cast<const float*>(a.param.p[rank]) + base * 4;
  float2* const acc = lars_acc + (size_t)warp * P;

  constexpr int U = (MODE == MODE_NVLS) ? 4 : 2;
  // the loop runs on the warp's first index so that every lane takes part in the shuffles of every trip
  for (size_t w0 = (size_t)blockIdx.x * blockDim.x * U + (size_t)warp * 32; w0 < lim; w0 += lars_gstride() * U) {
    const size_t i0 = w0 + lane;
    float gg[U][4];
    if (MODE == MODE_NVLS) {
      uint4 r[U];
#pragma unroll
      for (int u = 0; u < U; u++) {
        const size_t i = i0 + (size_t)u * blockDim.x;
        if (i < lim) r[u] = MultiMem<float>::ld_reduce<OP_SUM>(gmc + i * 16);
      }
#pragma unroll
      for (int u = 0; u < U; u++) VecTraits<float>::unpack(r[u], gg[u]);
    } else {
      uint4 v[U][kMaxRanks];
#pragma unroll
      for (int u = 0; u < U; u++) {
        const size_t i = i0 + (size_t)u * blockDim.x;
#pragma unroll
        for (int k = 0; k < kMaxRanks; k++)
          if (k < world && i < lim) v[u][k] = ld_sys_v4(a.buf.p[lars_wrap(rank + k, world)] + (base + i) * 16);
      }
#pragma unroll
      for (int u = 0; u < U; u++) {
#pragma unroll
        for (int k = 0; k < kMaxRanks; k++) {
          if (k < world) {
            float f[4];
            VecTraits<float>::unpack(v[u][k], f);
#pragma unroll
            for (int j = 0; j < 4; j++) gg[u][j] = k == 0 ? f[j] : gg[u][j] + f[j];
          }
        }
      }
    }
#pragma unroll
    for (int u = 0; u < U; u++) {
      const size_t i = i0 + (size_t)u * blockDim.x;
      const bool in = i < lim;
      float sg = 0.f, sp = 0.f;
      int key = P;   // past the slice: the tail key, which no parameter has
      if (in) {
        key = __ldg(L.pmap + base + i);
        *reinterpret_cast<float4*>(sums + i * 4) = make_float4(gg[u][0], gg[u][1], gg[u][2], gg[u][3]);
        const float4 w = *reinterpret_cast<const float4*>(pl + i * 4);
        const float pw[4] = {w.x, w.y, w.z, w.w};
#pragma unroll
        for (int j = 0; j < 4; j++) {
          const float gs = gg[u][j] * a.scale;
          sg = __fmaf_rn(gs, gs, sg);
          sp = __fmaf_rn(pw[j], pw[j], sp);
        }
      }
      // segmented inclusive scan over the warp's 32 consecutive vectors: the map is sorted, so equal keys are contiguous
#pragma unroll
      for (int d = 1; d < 32; d <<= 1) {
        const float og = __shfl_up_sync(0xffffffffu, sg, d);
        const float op = __shfl_up_sync(0xffffffffu, sp, d);
        const int ok = __shfl_up_sync(0xffffffffu, key, d);
        if (lane >= d && ok == key) { sg += og; sp += op; }
      }
      const int next = __shfl_down_sync(0xffffffffu, key, 1);
      if ((lane == 31 || next != key) && key < P) {   // last lane of a segment: one writer per parameter and warp
        float2 t = acc[key];
        t.x += sg; t.y += sp;
        acc[key] = t;
      }
      __syncwarp();
    }
  }
  __syncthreads();
  for (int q = threadIdx.x; q < P; q += blockDim.x) {
    float2 t = lars_acc[q];
    for (int w = 1; w < kLarsWarps; w++) { t.x += lars_acc[(size_t)w * P + q].x; t.y += lars_acc[(size_t)w * P + q].y; }
    rows[(size_t)blockIdx.x * P + q] = t;
  }
  __threadfence();
  __syncthreads();
  __shared__ int last;
  if (threadIdx.x == 0) last = atomicAdd(ticket, 1u) == gridDim.x - 1;
  __syncthreads();
  if (last) {
    __threadfence();
    for (int q = threadIdx.x; q < P; q += blockDim.x) {
      float2 t = __ldcg(rows + q);
      for (unsigned b = 1; b < gridDim.x; b++) { const float2 s = __ldcg(rows + (size_t)b * P + q); t.x += s.x; t.y += s.y; }
      const size_t off = ((size_t)q * world + rank) * sizeof(float2);
#pragma unroll
      for (int k = 0; k < kMaxRanks; k++)
        if (k < world) *reinterpret_cast<float2*>(L.board.p[k] + off) = t;
    }
    if (threadIdx.x == 0) *ticket = 0;
  }
  rank_barrier(a.c, ++e);
  if (threadIdx.x == 0) a.c.epoch[blockIdx.x] = e;
}

// EMA: as k_allreduce_sgd's, the owner folds the updated parameters into its EMA slice a.ema.
template <int MODE, bool EMA = false>
__global__ void __launch_bounds__(kThreads)
k_lars_update(const __grid_constant__ KArgs a0, const KArgs* __restrict__ emu, const __grid_constant__ LarsArgs L) {
  EMU_ARGS;
  __shared__ float trust_s[kLarsMaxParams + 1];
  __shared__ uint8_t group_s[kLarsMaxParams + 1];
  const int rank = a.c.rank, world = a.c.world, P = L.P;
  uint32_t e = a.c.epoch[blockIdx.x];
  const size_t per = a.per, nvec = a.nvec;
  const float* const sums = reinterpret_cast<const float*>(L.scratch[rank] + lars_sum_off(P));
  const float2* const board = reinterpret_cast<const float2*>(L.board.p[rank]);
  for (int q = threadIdx.x; q <= P; q += blockDim.x) {
    float t = 1.0f;
    int grp = 0;
    if (q < P) {
      grp = __ldg(L.ptab + 2 * q);
      if (__ldg(L.ptab + 2 * q + 1)) {
        float sg = 0.f, sp = 0.f;
        for (int r = 0; r < world; r++) {
          const float2 v = __ldcg(board + (size_t)q * world + r);
          sg += v.x; sp += v.y;
        }
        const float gn = sqrtf(sg), wn = sqrtf(sp);
        const float wd = __ldg(L.ghyper + 3 * grp + 2);
        if (wn > 0.f && gn > 0.f) t = __fdiv_rn(__fmul_rn(L.eta, wn), __fadd_rn(__fmaf_rn(wd, wn, gn), kLarsEps));
      }
    }
    trust_s[q] = t;
    group_s[q] = (uint8_t)grp;
  }
  __syncthreads();
  if (blockIdx.x == 0 && L.trust_out[rank] != nullptr)
    for (int q = threadIdx.x; q < P; q += blockDim.x) L.trust_out[rank][q] = trust_s[q];

  const size_t base = (size_t)rank * per;
  const size_t lim = base < nvec ? (nvec - base < per ? nvec - base : per) : 0;
  const bool has_lowp = a.lowp.p[0] != nullptr;
  float ema_c = 0.f;
  if constexpr (EMA) ema_c = ema_coef(a.ema_sched);  // a.ema_sched aliases dbg: this kernel never reads dbg
  constexpr int U = (MODE == MODE_NVLS) ? 4 : 2;
  for (size_t i0 = (size_t)blockIdx.x * blockDim.x * U + threadIdx.x; i0 < lim; i0 += lars_gstride() * U) {
    int pid[U];
    float4 gv[U];
#pragma unroll
    for (int u = 0; u < U; u++) {
      const size_t i = i0 + (size_t)u * blockDim.x;
      if (i < lim) {
        pid[u] = __ldg(L.pmap + base + i);
        gv[u] = *reinterpret_cast<const float4*>(sums + i * 4);
      }
    }
#pragma unroll
    for (int u = 0; u < U; u++) {
      const size_t i = i0 + (size_t)u * blockDim.x;
      if (i >= lim) continue;
      const int q = pid[u] < P ? pid[u] : P;
      const float trust = trust_s[q];
      const float* h = L.ghyper + 3 * group_s[q];
      const float vlr = __ldg(h), vmu = __ldg(h + 1), vwd = __ldg(h + 2);
      const size_t el = (base + i) * 4;
      const float* pl = reinterpret_cast<const float*>(a.param.p[rank]) + el;
      float* ml = a.mom + i * 4;
      const float4 pt = *reinterpret_cast<const float4*>(pl);
      float4 mt = make_float4(0.f, 0.f, 0.f, 0.f);
      if (!a.first_step) mt = *reinterpret_cast<const float4*>(ml);
      float4 ev;  // EMA: this vector of the average, loaded with the parameters (a.ema aliases ustride: never read that here)
      if constexpr (EMA) ev = *reinterpret_cast<const float4*>(a.ema + i * 4);
      const float g[4] = {gv[u].x, gv[u].y, gv[u].z, gv[u].w};
      float p[4] = {pt.x, pt.y, pt.z, pt.w};
      float m[4] = {mt.x, mt.y, mt.z, mt.w};
#pragma unroll
      for (int j = 0; j < 4; j++) {
        // k_allreduce_sgd's expression, with its contraction spelled out: a trust of exactly 1 leaves it bit for bit
        const float dj = __fmul_rn(trust, __fmaf_rn(g[j], a.scale, __fmul_rn(vwd, p[j])));
        const float mj = a.first_step ? dj : __fmaf_rn(vmu, m[j], dj);
        m[j] = mj;
        p[j] = __fmaf_rn(-vlr, a.nesterov ? __fmaf_rn(vmu, mj, dj) : mj, p[j]);
      }
      if constexpr (EMA)
        *reinterpret_cast<float4*>(a.ema + i * 4) = make_float4(ema_update(ema_c, p[0], ev.x), ema_update(ema_c, p[1], ev.y),
                                                                ema_update(ema_c, p[2], ev.z), ema_update(ema_c, p[3], ev.w));
      *reinterpret_cast<float4*>(ml) = make_float4(m[0], m[1], m[2], m[3]);
      const uint4 o = make_uint4(__float_as_uint(p[0]), __float_as_uint(p[1]), __float_as_uint(p[2]), __float_as_uint(p[3]));
      const size_t boff = el * 4;
      if (MODE == MODE_NVLS) {
        multimem_st_v4(a.param.mc + boff, o);
      } else {
#pragma unroll
        for (int k = 0; k < kMaxRanks; k++)
          if (k < world) st_peer_v4(a.param.p[lars_wrap(rank + k, world)] + boff, o);
      }
      if (has_lowp) {
        const __nv_bfloat162 h0 = __floats2bfloat162_rn(p[0], p[1]), h1 = __floats2bfloat162_rn(p[2], p[3]);
        const uint2 w = make_uint2(*reinterpret_cast<const uint32_t*>(&h0), *reinterpret_cast<const uint32_t*>(&h1));
#pragma unroll
        for (int k = 0; k < kMaxRanks; k++)
          if (k < world) *reinterpret_cast<uint2*>(a.lowp.p[lars_wrap(rank + k, world)] + el * 2) = w;
      }
    }
  }
  rank_barrier(a.c, ++e);
  if (threadIdx.x == 0) a.c.epoch[blockIdx.x] = e;
}

template <typename K>
static cudaError_t go_lars(K kernel, const Launch& l, const KArgs& a, const LarsArgs& L, size_t smem) {
  if (smem > 48 * 1024) {
    cudaError_t e = cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
  }
  dim3 grid(l.blocks, l.emu_world > 0 ? l.emu_world : 1, 1);
  kernel<<<grid, kThreads, smem, l.stream>>>(a, l.emu_world > 0 ? l.emu_args : nullptr, L);
  return cudaGetLastError();
}

cudaError_t launch_lars_norms(const Launch& l, const KArgs& a, const LarsArgs& L, int mode) {
  const size_t smem = lars_norms_smem(L.P);
  if (mode == MODE_NVLS) return go_lars(k_allreduce_lars_norms<MODE_NVLS>, l, a, L, smem);
  return go_lars(k_allreduce_lars_norms<MODE_P2P>, l, a, L, smem);
}
cudaError_t launch_lars_update(const Launch& l, const KArgs& a, const LarsArgs& L, int mode, bool ema) {
  if (ema) {
    if (mode == MODE_NVLS) return go_lars(k_lars_update<MODE_NVLS, true>, l, a, L, 0);
    return go_lars(k_lars_update<MODE_P2P, true>, l, a, L, 0);
  }
  if (mode == MODE_NVLS) return go_lars(k_lars_update<MODE_NVLS>, l, a, L, 0);
  return go_lars(k_lars_update<MODE_P2P>, l, a, L, 0);
}

}  // namespace b200mpi
