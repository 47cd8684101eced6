// Learning-rate schedule of the data-parallel trainer for sm_90a: one single-CTA launch per synchronising step, on the
// compute stream before backward, that turns the step count k into each parameter group's rate for the step and writes it
// into the {lr, mu, wd} tables the fused SGD / LARS kernels read. Inside a captured CUDA graph every replay advances k.
//
// The contract (mpi_operator_b200/parallel/lr_schedule.py evaluates the same on the host):
//   m(k) = k / W                                                   k < W (warm-up)
//        = 1                                                       constant
//        = v[#{b in boundaries : b < k}]                           piecewise
//        = max(pow_int(factor, k / decay_steps), floor)            exponential (integer division: staircase)
//        = k < T ? end + (1 - end) * pow_int(1 - (k - W) / (T - W), power) : end     polynomial
//   lr_g = fp32_rn(base_g * m(k))
// Every floating-point operation is one float64 add, multiply or divide written with the _rn intrinsics, so nvcc cannot
// contract it into an FMA; pow_int is right-to-left binary exponentiation. Integer quantities (k, W, boundaries,
// decay_steps, T, power) are below 2^53 where they meet a float64 and are exact there.
//
// Table layout (float64, decoded with `form` and `nb` = number of boundaries):
//   [0] W, then  piecewise: [1, nb] boundaries, [nb + 1, 2 nb + 1] multipliers
//                exponential: decay_steps, factor, floor      polynomial: T, power, end
#include "kernels.h"

namespace b200mpi {

constexpr int kLrThreads = kLrMaxGroups;   // one thread per group row

static __device__ __forceinline__ double pow_int(double x, long long n) {
  double r = 1.0, b = x;
  while (n) {
    if (n & 1) r = __dmul_rn(r, b);
    b = __dmul_rn(b, b);
    n >>= 1;
  }
  return r;
}

static __device__ double lr_multiplier(const double* __restrict__ t, int form, int nb, long long k) {
  const long long W = __double2ll_rn(t[0]);
  if (k < W) return __ddiv_rn((double)k, (double)W);
  switch (form) {
    case LR_PIECEWISE: {
      int i = 0;
      for (int j = 0; j < nb; j++) i += __double2ll_rn(t[1 + j]) < k;
      return t[1 + nb + i];
    }
    case LR_EXPONENTIAL: {
      const double p = pow_int(t[2], k / __double2ll_rn(t[1])), floor = t[3];
      return p > floor ? p : floor;
    }
    case LR_POLYNOMIAL: {
      const long long T = __double2ll_rn(t[1]);
      const double end = t[3];
      if (k >= T) return end;
      const double u = __ddiv_rn((double)(k - W), (double)(T - W));
      return __dadd_rn(end, __dmul_rn(__dadd_rn(1.0, -end), pow_int(__dadd_rn(1.0, -u), __double2ll_rn(t[2]))));
    }
    default:
      return 1.0;
  }
}

// Thread 0 reads k, evaluates m(k) once and stores k + 1; after the barrier thread g writes group g's rate. Only the lr
// column of each row is written.
__global__ void __launch_bounds__(kLrThreads)
k_lr_schedule(const double* __restrict__ sched, int form, int nb, long long* __restrict__ step,
              const double* __restrict__ base, int G, float* __restrict__ hyper, float* __restrict__ group_hyper) {
  __shared__ double m;
  if (threadIdx.x == 0) {
    const long long k = *step;
    m = lr_multiplier(sched, form, nb, k);
    *step = k + 1;
    hyper[0] = __double2float_rn(__dmul_rn(base[0], m));
  }
  __syncthreads();
  const int g = threadIdx.x;
  if (group_hyper != nullptr && g < G) group_hyper[3 * g] = __double2float_rn(__dmul_rn(base[g], m));
}

cudaError_t launch_lr_schedule(cudaStream_t s, const double* sched, int form, int nb, long long* step, const double* base,
                               int G, float* hyper, float* group_hyper) {
  k_lr_schedule<<<1, kLrThreads, 0, s>>>(sched, form, nb, step, base, G, hyper, group_hyper);
  return cudaGetLastError();
}

}  // namespace b200mpi
