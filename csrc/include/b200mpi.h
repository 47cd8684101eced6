/*
 * b200mpi — Hopper-native (sm_90a) collective runtime (C ABI).
 *
 * This is the data plane that the reference delegates to external software
 * (Horovod -> NCCL inside user images; reference: examples/v2beta1/
 * tensorflow-benchmarks/tensorflow-benchmarks.yaml:26-42, SURVEY.md §2.5 K2-K7).
 * Here it is first-party: one process per GPU, peers mapped through CUDA VMM
 * (POSIX-fd export + SCM_RIGHTS) or cudaIpc, NVLS multicast objects when the
 * host exposes them, and hand-written sm_90a kernels that read/write peer
 * HBM directly over NVSwitch.
 *
 * All functions return 0 on success or a negative B200MPI_ERR_* code;
 * b200mpi_last_error() returns a thread-local human readable message.
 */
#ifndef B200MPI_H_
#define B200MPI_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200MPI_MAX_RANKS 8
#define B200MPI_VERSION "0.1.0"

typedef struct b200mpi_comm* b200mpi_comm_t;

typedef enum {
  B200MPI_F32 = 0,
  B200MPI_BF16 = 1,
  B200MPI_F16 = 2,
} b200mpi_dtype_t;

typedef enum {
  B200MPI_SUM = 0,
  B200MPI_MAX = 1,
  B200MPI_MIN = 2,
} b200mpi_op_t;

typedef enum {
  B200MPI_ALGO_AUTO = 0,
  B200MPI_ALGO_ONESHOT = 1, /* push one-shot: 1 NVLink traversal + flag   */
  B200MPI_ALGO_TWOSHOT = 2, /* reduce-scatter(pull) + all-gather(push)    */
  B200MPI_ALGO_NVLS = 3,    /* multimem.ld_reduce + multimem.st in-switch */
} b200mpi_algo_t;

enum {
  B200MPI_OK = 0,
  B200MPI_ERR_INVALID = -1,
  B200MPI_ERR_CUDA = -2,
  B200MPI_ERR_SYS = -3,
  B200MPI_ERR_TIMEOUT = -4,
  B200MPI_ERR_UNSUPPORTED = -5,
  B200MPI_ERR_PEER = -6,
};

/* flags for b200mpi_comm_init */
enum {
  B200MPI_FLAG_NO_MULTICAST = 1u << 0, /* never create NVLS multicast objects */
  B200MPI_FLAG_FORCE_IPC = 1u << 1,    /* cudaIpc instead of VMM fd export    */
  B200MPI_FLAG_NO_PIPE = 1u << 2,      /* user-pointer allreduce: never the pipelined kernel (chunked staged two-shot) */
};

const char* b200mpi_last_error(void);
const char* b200mpi_version(void);

/*
 * Multi-process communicator: `rank` of `world` on CUDA `device`. Ranks of the
 * same job find each other through the POSIX shm rendezvous segment
 * "/b200mpi-<job_id>" (replaces ssh + DNS + ncclUniqueId broadcast of the
 * reference stack, SURVEY.md §5.9). staging_bytes is the per-rank staging
 * window used by collectives on unregistered pointers (0 = default 64 MiB).
 */
int b200mpi_comm_init(b200mpi_comm_t* comm, int rank, int world, int device,
                      const char* job_id, size_t staging_bytes, unsigned flags);

/*
 * Emulated communicator: `world` virtual ranks inside ONE process on ONE
 * device. Every collective is a single launch with gridDim.y == world, each
 * y-slice of CTAs playing one rank. Exercises the exact same kernels with no
 * second GPU (unit tests, compute-sanitizer, ncu). Pointer arguments of the
 * collectives become arrays of `world` pointers (see each call).
 */
int b200mpi_comm_init_local(b200mpi_comm_t* comm, int world, int device,
                            size_t staging_bytes, unsigned flags);

int b200mpi_comm_destroy(b200mpi_comm_t comm);
int b200mpi_comm_rank(b200mpi_comm_t comm);
int b200mpi_comm_world(b200mpi_comm_t comm);
int b200mpi_comm_is_local(b200mpi_comm_t comm);
int b200mpi_comm_has_multicast(b200mpi_comm_t comm);
/* host-side barrier through the shm segment (no GPU work) */
int b200mpi_comm_host_barrier(b200mpi_comm_t comm);
/* host-side small allgather through the shm segment: each rank contributes
 * `bytes` (<= 256) and receives world*bytes. */
int b200mpi_comm_host_allgather(b200mpi_comm_t comm, const void* in, void* out, size_t bytes);
/* non-zero if a device-side wait timed out since the last call (watchdog) */
int b200mpi_comm_check_error(b200mpi_comm_t comm);
/* number of b200mpi kernels launched so far on this communicator */
uint64_t b200mpi_comm_launch_count(b200mpi_comm_t comm);
/* JSON counters by (op, algorithm): calls and payload bytes of every host-launched collective. snprintf-style:
 * writes at most cap-1 bytes + NUL, returns the full length. */
int b200mpi_comm_stats_json(b200mpi_comm_t comm, char* buf, size_t cap);

/*
 * Symmetric windows: every rank allocates `bytes`, all ranks map all peers,
 * and (when available) the window is bound to an NVLS multicast object.
 * Collective call. window ids are small integers, identical on all ranks.
 */
int b200mpi_window_alloc(b200mpi_comm_t comm, size_t bytes, int* win);
int b200mpi_window_free(b200mpi_comm_t comm, int win);
/* VA (in this process) of `rank`'s copy of the window; rank = -1 -> own copy.
 * In emulated mode `rank` selects the virtual rank. */
void* b200mpi_window_ptr(b200mpi_comm_t comm, int win, int rank);
void* b200mpi_window_mc_ptr(b200mpi_comm_t comm, int win);
size_t b200mpi_window_size(b200mpi_comm_t comm, int win);

/*
 * Exportable device allocations and windows built around them (what the NCCL-ABI shim's ncclMemAlloc /
 * ncclCommRegister map to): b200mpi_mem_alloc returns VMM memory of the current device that can be exported and bound
 * to a multicast object; b200mpi_window_adopt (COLLECTIVE: every rank passes its own allocation of the same size, in the
 * same order) maps the peers' allocations and binds them to an NVLS multicast object, after which the buffer is a
 * symmetric window: b200mpi_allreduce_sym & co. run zero-copy on it. b200mpi_mem_lookup: 1 if `p` lies in such an
 * allocation (base / size returned).
 */
int b200mpi_mem_alloc(size_t bytes, void** ptr);
int b200mpi_mem_free(void* ptr);
int b200mpi_mem_lookup(const void* p, void** base, size_t* size);
int b200mpi_window_adopt(b200mpi_comm_t comm, void* base, int* win);

/*
 * In-place allreduce on a symmetric window region [offset, offset+count*esz).
 * out = scale * reduce_over_ranks(in). `scale` is fused into the reduction
 * (1/world for Horovod's Average; reference call site: examples/v2beta1/
 * horovod/tensorflow_mnist.py:133). offset must be 16-byte aligned.
 */
int b200mpi_allreduce_sym(b200mpi_comm_t comm, int win, size_t offset, size_t count,
                          b200mpi_dtype_t dtype, b200mpi_op_t op, float scale,
                          b200mpi_algo_t algo, void* stream);

/*
 * Allreduce on arbitrary device pointers (staged through the comm's staging
 * window inside the same kernel). in == out allowed. In emulated mode `in`
 * and `out` are `const void* const*` / `void* const*` arrays of world ptrs.
 */
int b200mpi_allreduce(b200mpi_comm_t comm, const void* in, void* out, size_t count,
                      b200mpi_dtype_t dtype, b200mpi_op_t op, float scale,
                      b200mpi_algo_t algo, void* stream);

/* Fused gradient-allreduce + SGD(momentum, weight decay, nesterov) step:
 *   g   = scale * sum_r grad_r[i]           (each rank owns a 1/world slice)
 *   g  += wd * p ; m = mu*m + g ; p -= lr * (nesterov ? g + mu*m : m)
 * and the updated parameter slice is pushed to every rank's parameter window
 * (multimem.st on NVLS). Momentum is sharded: `momentum` points at this rank's
 * slice buffer of ceil(count/world) fp32 elements rounded up to 4
 * (b200mpi_slice_elems). grad window dtype = gdtype, param window fp32.
 * If `lowp_win` >= 0 a bf16 copy of the parameters is also pushed there.
 * Emulated mode: `momentum` is an array of world pointers. */
int b200mpi_allreduce_sgd_sym(b200mpi_comm_t comm, int grad_win, size_t grad_off,
                              int param_win, size_t param_off, int lowp_win, size_t lowp_off,
                              void* momentum, size_t count, b200mpi_dtype_t gdtype, float scale,
                              float lr, float mu, float wd, int nesterov, int first_step,
                              b200mpi_algo_t algo, void* stream);
/* Same step with parameter groups: vector i (4 fp32 elements) of the region is
 * updated with {lr, mu, wd} = group_hyper[3*g .. 3*g+2], g = group_map[i].
 * group_map is a device array of count/4 bytes for this region, every entry
 * < num_groups; group_hyper a device table of num_groups x 3 floats, read at
 * run time (a captured CUDA graph follows changes to it). Both NULL: exactly
 * b200mpi_allreduce_sgd_sym. Groups need gdtype == B200MPI_F32 and
 * 1 <= num_groups <= 256. Emulated mode: one map and table for all ranks. */
int b200mpi_allreduce_sgd_sym_groups(b200mpi_comm_t comm, int grad_win, size_t grad_off,
                                     int param_win, size_t param_off, int lowp_win, size_t lowp_off,
                                     void* momentum, size_t count, b200mpi_dtype_t gdtype, float scale,
                                     float lr, float mu, float wd, int nesterov, int first_step,
                                     b200mpi_algo_t algo, void* stream,
                                     const uint8_t* group_map, const float* group_hyper, int num_groups);
/* Same step with LARS (fp32 gradients): every parameter tensor q of the region
 * whose table row has lars != 0 scales its update direction by the trust ratio
 *   trust = eta*|w| / (|g| + wd*|w| + 1e-8)   (1 when |w| or |g| is 0)
 *   d = trust*(g + wd*w); m = first_step ? d : mu*m + d; w -= lr*(nesterov ? d + mu*m : m)
 * with g the averaged gradient and both norms over the whole tensor, before the
 * update; other parameters get exactly the grouped SGD step. Two launches on
 * `stream` (norms + board exchange, then the update); the gradient window is
 * only read.
 *   param_map    device [count/4] uint16: the parameter (0..num_params-1) of each
 *                vector, non-decreasing; vectors past the last parameter hold
 *                num_params.
 *   param_table  device [num_params][2] uint8 {group (< num_groups), lars}.
 *   group_hyper  device [num_groups][3] {lr, mu, wd}, read at run time.
 *   board_win    symmetric window holding num_params*world*2 floats at board_off.
 *   scratch      this rank's device scratch of scratch_bytes >=
 *                b200mpi_lars_scratch_bytes(count, world, num_params), zero-filled
 *                before its first use (the kernels leave it reusable).
 *   trust_out    optional device [num_params] floats: the trust ratios of this
 *                step (1 for non-LARS parameters).
 * 1 <= num_params <= 1024. Emulated mode: momentum, scratch and trust_out are
 * host arrays of world device pointers (trust_out may be NULL as a whole). */
int b200mpi_allreduce_lars_sym(b200mpi_comm_t comm, int grad_win, size_t grad_off,
                               int param_win, size_t param_off, int lowp_win, size_t lowp_off,
                               void* momentum, size_t count, b200mpi_dtype_t gdtype, float scale,
                               int nesterov, int first_step, b200mpi_algo_t algo, void* stream,
                               const float* group_hyper, int num_groups,
                               const uint16_t* param_map, const uint8_t* param_table, int num_params,
                               int board_win, size_t board_off, void* scratch, size_t scratch_bytes,
                               float eta, void* trust_out);
/* The grouped SGD step (group_map and group_hyper may both be NULL: the
 * ungrouped step) and the LARS step, each also keeping an exponential moving
 * average of the parameters (tf.train.ExponentialMovingAverage with
 * num_updates). Each launch reads ema_sched = device {d, k} (two doubles: the
 * decay and the number of parameter updates including this one) and applies
 *   c  = (float)(1 - min(d, (1 + k) / (10 + k)))     (in double, rounded once)
 *   e' = fmaf(c, p' - e, e)                           (p' the updated parameter)
 * to every element of this rank's slice. `ema` is laid out like `momentum`
 * (b200mpi_slice_elems fp32 elements) and never leaves the rank; the
 * parameter, momentum, shadow and trust-ratio results are those of the calls
 * without it. fp32 gradients only; ema and ema_sched must not be NULL.
 * Emulated mode: `ema` is a host array of world device pointers, ema_sched is
 * shared. */
int b200mpi_allreduce_sgd_sym_ema(b200mpi_comm_t comm, int grad_win, size_t grad_off,
                                  int param_win, size_t param_off, int lowp_win, size_t lowp_off,
                                  void* momentum, size_t count, b200mpi_dtype_t gdtype, float scale,
                                  float lr, float mu, float wd, int nesterov, int first_step,
                                  b200mpi_algo_t algo, void* stream,
                                  const uint8_t* group_map, const float* group_hyper, int num_groups,
                                  void* ema, const double* ema_sched);
int b200mpi_allreduce_lars_sym_ema(b200mpi_comm_t comm, int grad_win, size_t grad_off,
                                   int param_win, size_t param_off, int lowp_win, size_t lowp_off,
                                   void* momentum, size_t count, b200mpi_dtype_t gdtype, float scale,
                                   int nesterov, int first_step, b200mpi_algo_t algo, void* stream,
                                   const float* group_hyper, int num_groups,
                                   const uint16_t* param_map, const uint8_t* param_table, int num_params,
                                   int board_win, size_t board_off, void* scratch, size_t scratch_bytes,
                                   float eta, void* trust_out, void* ema, const double* ema_sched);
size_t b200mpi_lars_scratch_bytes(size_t count, int world, int num_params);
size_t b200mpi_slice_elems(size_t count, int world, b200mpi_dtype_t dtype);
/* Optional device-resident hyper-parameters {lr, momentum, weight_decay} (3 floats)
 * read by the fused kernels instead of the by-value arguments: a captured CUDA
 * graph then follows LR schedules without re-capture. NULL restores by-value. */
int b200mpi_set_hyper_ptr(b200mpi_comm_t comm, const float* device_hyper);
/* Learning-rate schedule step (one single-CTA launch on `stream`): reads the
 * device step counter k, evaluates the multiplier m(k) of the float64 device
 * table `schedule` in float64 and writes
 *   hyper[0] = fp32_rn(base[0] * m(k)),  group_hyper[3*g] = fp32_rn(base[g] * m(k))  (g < num_groups)
 * then stores k + 1. The momentum and weight-decay entries are not touched.
 * `form` (0 constant, 1 piecewise, 2 exponential, 3 polynomial) and
 * `num_boundaries` (piecewise: 0..64, otherwise 0) say how to decode the table:
 *   [0] warm-up steps W, then  piecewise: num_boundaries boundaries and
 *   num_boundaries + 1 multipliers; exponential: decay_steps, factor, floor;
 *   polynomial: total steps T, power, end.
 * mpi_operator_b200/parallel/lr_schedule.py states the contract and builds the
 * table. `base` holds num_groups (1..256) doubles; group_hyper ([num_groups][3]
 * floats) may be NULL, every other pointer may not. */
int b200mpi_lr_schedule(b200mpi_comm_t comm, const double* schedule, int form, int num_boundaries, int64_t* step,
                        const double* base, int num_groups, float* hyper, float* group_hyper, void* stream);

int b200mpi_broadcast(b200mpi_comm_t comm, void* buf, size_t count, b200mpi_dtype_t dtype,
                      int root, void* stream);
int b200mpi_broadcast_bytes(b200mpi_comm_t comm, void* buf, size_t bytes, int root, void* stream);
/* out has world*count elements */
int b200mpi_allgather(b200mpi_comm_t comm, const void* in, void* out, size_t count,
                      b200mpi_dtype_t dtype, void* stream);
/* in has world*count elements, out count */
int b200mpi_reduce_scatter(b200mpi_comm_t comm, const void* in, void* out, size_t count,
                           b200mpi_dtype_t dtype, b200mpi_op_t op, float scale, void* stream);
int b200mpi_reduce(b200mpi_comm_t comm, const void* in, void* out, size_t count,
                   b200mpi_dtype_t dtype, b200mpi_op_t op, float scale, int root, void* stream);
/* Adasum allreduce (Horovod op=hvd.Adasum) in one kernel; B200MPI_ERR_UNSUPPORTED when the world is not a power of two or
 * count * sizeof(dtype) > b200mpi_adasum_max_bytes(): callers then gather and fold the tree themselves */
int b200mpi_adasum(b200mpi_comm_t comm, const void* in, void* out, size_t count, b200mpi_dtype_t dtype, void* stream);
size_t b200mpi_adasum_max_bytes(b200mpi_comm_t comm, b200mpi_dtype_t dtype);
/* in/out have world*count elements; block j of in goes to rank j */
int b200mpi_alltoall(b200mpi_comm_t comm, const void* in, void* out, size_t count,
                     b200mpi_dtype_t dtype, void* stream);
int b200mpi_barrier(b200mpi_comm_t comm, void* stream);

/* fused local elementwise helpers used by the front-ends (same .so) */
int b200mpi_scale_cast(const void* in, b200mpi_dtype_t in_dtype, void* out,
                       b200mpi_dtype_t out_dtype, size_t count, float scale, void* stream);

/*
 * Fused BatchNorm(+residual add)+ReLU, training mode, channels-last bf16 activations
 * viewed as [M = N*H*W, C]; fp32 affine parameters and statistics (csrc/kernels/bn_act.cu).
 * forward: z = relu(bn(x) [+ residual]); writes a 1-bit/element ReLU mask ([M*C/8] bytes),
 * save_mean/save_invstd, updates running stats. backward: dx, optional dres (gradient of the
 * residual branch), dweight, dbias. `workspace`: b200mpi_bn_workspace_floats(C) floats,
 * zero-initialised once; the kernels leave it zeroed (CUDA-graph safe).
 */
size_t b200mpi_bn_workspace_floats(int C);
int b200mpi_bn_supported(long long M, int C);
int b200mpi_bn_act_fwd(const void* x, const void* residual, void* y, void* mask, const float* weight,
                       const float* bias, float* running_mean, float* running_var, float* save_mean,
                       float* save_invstd, float* workspace, long long M, int C, float eps, float momentum,
                       int relu, void* stream);
/* Same as b200mpi_bn_act_fwd but the per-channel statistics arrive as `parts` rows of {sum, sum of squares} (2*C floats
 * per row) produced by the epilogue of b200mpi_gemm_bnstats with x its output: row p holds the sums of x - x[128 p, c]
 * over the 128-row tiles p, p + parts, ... of x. No statistics pass over x. */
int b200mpi_bn_act_fwd_prestats(const void* x, const void* residual, void* y, void* mask, const float* weight, const float* bias,
                                float* running_mean, float* running_var, float* save_mean, float* save_invstd, float* workspace,
                                const float* partials, int parts, long long M, int C, float eps, float momentum, int relu,
                                void* stream);
/* Eval-mode forward: z = relu?(a x + b [+ residual]) with a = weight * rsqrt(running_var + eps) and b = bias - running_mean * a
 * (weight / bias NULL: 1 / 0), in fp32 with one bf16 rounding. Reads the running statistics and writes z only: no mask, no
 * workspace, no statistics. Same C as b200mpi_bn_supported, any M >= 1; x, residual, y 16-byte aligned. */
int b200mpi_bn_act_eval(const void* x, const void* residual, void* y, const float* weight, const float* bias,
                        const float* running_mean, const float* running_var, long long M, int C, float eps, int relu,
                        void* stream);
int b200mpi_bn_act_bwd(const void* dz, const void* x, const void* mask, void* dx, void* dres,
                       const float* weight, const float* save_mean, const float* save_invstd,
                       float* dweight, float* dbias, float* workspace, long long M, int C, int relu,
                       void* stream);
/* Same as b200mpi_bn_act_bwd but the reduction arrives as `parts` rows of {sum g, sum g*(x - save_mean)} (g = mask ⊙ dz,
 * 2*C floats per row) produced by the epilogue of the wgmma dgrad: no reduce pass over dz. */
int b200mpi_bn_act_bwd_prestats(const void* dz, const void* x, const void* mask, void* dx, void* dres, const float* weight,
                                const float* save_mean, const float* save_invstd, float* dweight, float* dbias, float* workspace,
                                const float* partials, int parts, long long M, int C, int relu, void* stream);

/* tuning */
int b200mpi_set_tuning(b200mpi_comm_t comm, size_t oneshot_max_bytes, size_t nvls_min_bytes,
                       int max_blocks, int timeout_ms);
int b200mpi_get_tuning(b200mpi_comm_t comm, size_t* oneshot_max_bytes, size_t* nvls_min_bytes,
                       int* max_blocks, int* timeout_ms);
/* which algorithm would AUTO pick */
/*
 * Zero-copy collectives on a symmetric window region (no staging, no copy-out). The region starts at `offset`
 * (16-byte aligned) and is `world` slices of `slice_bytes` (a multiple of 16); slice r belongs to rank r.
 *   allgather_sym       : every rank's slice r of its OWN copy ends up in slice r of every copy (multimem.st on NVLS)
 *   reduce_scatter_sym  : slice r of every copy is reduced (x scale) into rank r's `out` (slice-sized device pointer,
 *                         16-byte aligned) or, with out == NULL, in place into slice r of rank r's own copy
 *                         (multimem.ld_reduce on NVLS). Emulated mode: `out` is an array of world pointers.
 *   broadcast_sym       : the root's [offset, offset+bytes) replaces the same region of every copy
 */
int b200mpi_allgather_sym(b200mpi_comm_t comm, int win, size_t offset, size_t slice_bytes, void* stream);
int b200mpi_reduce_scatter_sym(b200mpi_comm_t comm, int win, size_t offset, size_t slice_count, b200mpi_dtype_t dtype,
                               b200mpi_op_t op, float scale, void* out, void* stream);
int b200mpi_broadcast_sym(b200mpi_comm_t comm, int win, size_t offset, size_t bytes, int root, void* stream);

/* Pipelined user-pointer allreduce (k_allreduce_pipe): messages of at least `min_bytes` (SIZE_MAX: keep) run as one
 * kernel of `lanes` x {copy-in, reduce, copy-out} CTAs with `depth` staging slots of `chunk_bytes` per lane.
 * Non-positive values keep the current setting. Env: B200MPI_PIPE_{MIN_BYTES,LANES_NVLS,LANES_P2P,DEPTH,CHUNK_BYTES}. */
int b200mpi_set_pipe(b200mpi_comm_t comm, size_t min_bytes, int lanes_nvls, int lanes_p2p, int depth, size_t chunk_bytes);
/* Debug timeline of the last pipelined launch (B200MPI_PIPE_DEBUG=1 when the communicator was created):
 * out[3 roles][48 lanes][32 chunks][3] = {wait begin, work begin, end} as %globaltimer ns. Returns u64 words written. */
size_t b200mpi_pipe_timeline(b200mpi_comm_t comm, unsigned long long* out, size_t cap);
/* Lazy registration of user buffers (cudaIpc) for the user-pointer collectives: mode 0 = never, 1 = where the zero-copy
 * P2P kernels win (default: world 2, paths without NVLS, allgather), 2 = whenever the buffers can be exported; calls below
 * `min_bytes` (SIZE_MAX: keep) always take the staged kernels. Env: B200MPI_REG, B200MPI_REG_MIN_BYTES. */
int b200mpi_set_reg(b200mpi_comm_t comm, int mode, size_t min_bytes);
int b200mpi_reg_stats(b200mpi_comm_t comm, uint64_t* zero_copy_calls, uint64_t* handles_opened, uint64_t* refused);
int b200mpi_select_algo(b200mpi_comm_t comm, size_t bytes, b200mpi_dtype_t dtype, b200mpi_op_t op,
                        int symmetric);

/* trace: per-collective records (op, bytes, algo, host enqueue ns) as JSONL */
/* Point-to-point (EXPERIMENTAL; the mailbox window is only allocated when B200MPI_P2P=1 is set for every rank at
 * communicator creation). A batch is executed by one kernel, one CTA per operation, so grouped exchanges cannot
 * deadlock on stream order; sends of up to 2 MiB complete without the matching receive (eager). */
typedef struct {
  const void* send; /* source buffer (is_send) */
  void* recv;       /* destination buffer (!is_send) */
  size_t bytes;
  int peer;
  int is_send;
} b200mpi_p2p_op_t;
int b200mpi_p2p_batch(b200mpi_comm_t comm, const b200mpi_p2p_op_t* ops, int nops, void* stream);
int b200mpi_send(b200mpi_comm_t comm, const void* buf, size_t bytes, int peer, void* stream);
int b200mpi_recv(b200mpi_comm_t comm, void* buf, size_t bytes, int peer, void* stream);
int b200mpi_comm_has_p2p(b200mpi_comm_t comm);

int b200mpi_trace_enable(b200mpi_comm_t comm, int on);
int b200mpi_trace_dump(b200mpi_comm_t comm, const char* path);

#ifdef __cplusplus
}
#endif
#endif /* B200MPI_H_ */
