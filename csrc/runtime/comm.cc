// b200mpi communicator: peer-memory windows (CUDA VMM + NVLS multicast, cudaIpc
// fallback), algorithm selection, kernel launch plumbing and the C ABI.
//
// Reference parity: SURVEY.md §5.9 (GPU-native replacement for the
// Horovod -> NCCL data plane the reference launches but does not contain).
#include <cuda.h>
#include <cuda_runtime.h>
#include <string.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <mutex>
#include <map>
#include <set>
#include <string>
#include <vector>

#include "../include/b200mpi.h"
#include "../kernels/kernels.h"
#include "rendezvous.h"

namespace b200mpi {

static thread_local std::string g_err;
static int fail(int code, const std::string& msg) {
  g_err = msg;
  if (getenv("B200MPI_DEBUG")) fprintf(stderr, "[b200mpi] error %d: %s\n", code, msg.c_str());
  return code;
}
#define CUDA_TRY(expr)                                                                         \
  do {                                                                                         \
    cudaError_t _e = (expr);                                                                   \
    if (_e != cudaSuccess)                                                                     \
      return fail(B200MPI_ERR_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e));       \
  } while (0)

// ---------------------------------------------------------------- driver ----
struct Driver {
  bool ok = false;
#define DRV(name) decltype(&name) name##_ = nullptr
  DRV(cuMemCreate); DRV(cuMemRelease); DRV(cuMemAddressReserve); DRV(cuMemAddressFree);
  DRV(cuMemMap); DRV(cuMemUnmap); DRV(cuMemSetAccess); DRV(cuMemExportToShareableHandle);
  DRV(cuMemImportFromShareableHandle); DRV(cuMemGetAllocationGranularity);
  DRV(cuMulticastCreate); DRV(cuMulticastAddDevice); DRV(cuMulticastBindMem);
  DRV(cuMulticastUnbind); DRV(cuMulticastGetGranularity); DRV(cuDeviceGetAttribute);
  DRV(cuGetErrorString); DRV(cuMemGetAddressRange); DRV(cuPointerGetAttribute);
#undef DRV
};
static Driver& driver() {
  static Driver d;
  static std::once_flag once;
  std::call_once(once, [] {
    cudaFree(0);
    bool all = true;
#define LOAD(name)                                                                               \
  do {                                                                                           \
    void* fn = nullptr;                                                                          \
    cudaDriverEntryPointQueryResult qr;                                                          \
    if (cudaGetDriverEntryPoint(#name, &fn, cudaEnableDefault, &qr) != cudaSuccess || !fn) {     \
      all = false;                                                                               \
      cudaGetLastError();                                                                        \
    }                                                                                            \
    d.name##_ = reinterpret_cast<decltype(&name)>(fn);                                           \
  } while (0)
    LOAD(cuMemCreate); LOAD(cuMemRelease); LOAD(cuMemAddressReserve); LOAD(cuMemAddressFree);
    LOAD(cuMemMap); LOAD(cuMemUnmap); LOAD(cuMemSetAccess); LOAD(cuMemExportToShareableHandle);
    LOAD(cuMemImportFromShareableHandle); LOAD(cuMemGetAllocationGranularity);
    LOAD(cuMulticastCreate); LOAD(cuMulticastAddDevice); LOAD(cuMulticastBindMem);
    LOAD(cuMulticastUnbind); LOAD(cuMulticastGetGranularity); LOAD(cuDeviceGetAttribute);
    LOAD(cuGetErrorString); LOAD(cuMemGetAddressRange); LOAD(cuPointerGetAttribute);
#undef LOAD
    d.ok = all;
  });
  return d;
}
static std::string cu_err(CUresult r) {
  const char* s = nullptr;
  if (driver().cuGetErrorString_) driver().cuGetErrorString_(r, &s);
  return s ? s : ("CUresult " + std::to_string((int)r));
}
#define CU_TRY(expr)                                                                 \
  do {                                                                               \
    CUresult _r = (expr);                                                            \
    if (_r != CUDA_SUCCESS) return fail(B200MPI_ERR_CUDA, std::string(#expr) + ": " + cu_err(_r)); \
  } while (0)

static size_t round_up(size_t x, size_t a) { return (x + a - 1) / a * a; }
static int env_int(const char* name, int dflt) {
  const char* v = getenv(name);
  return v && *v ? atoi(v) : dflt;
}
static size_t env_size(const char* name, size_t dflt) {
  const char* v = getenv(name);
  if (!v || !*v) return dflt;
  char* end = nullptr;
  double x = strtod(v, &end);
  if (end && (*end == 'k' || *end == 'K')) x *= 1024.0;
  else if (end && (*end == 'm' || *end == 'M')) x *= 1024.0 * 1024.0;
  else if (end && (*end == 'g' || *end == 'G')) x *= 1024.0 * 1024.0 * 1024.0;
  return (size_t)x;
}

// ---------------------------------------------------------------- window ----
struct Window {
  bool live = false;
  size_t bytes = 0;      // usable
  size_t mapped = 0;     // rounded to granularity
  bool vmm = false;
  char* ptr[kMaxRanks] = {};                          // local VA of each rank's copy
  CUmemGenericAllocationHandle h[kMaxRanks] = {};     // vmm handles (own + imported)
  char* mc = nullptr;
  CUmemGenericAllocationHandle mch = 0;
  bool adopted = false;   // own copy belongs to b200mpi_mem_alloc (ncclMemAlloc): never unmapped / released with the window
};

struct TraceRec { const char* op; size_t bytes; int algo; int blocks; uint64_t t_ns; };
// Per-communicator counters by (op, algorithm): what /metrics exports as b200mpi_collective_{calls,bytes}_total.
// `op` is a string literal, so pointer identity is the key; a handful of entries, linear scan.
struct OpStat { const char* op; int algo; uint64_t calls; uint64_t bytes; };
static const char* const kP2PName = "p2p";

}  // namespace b200mpi

using namespace b200mpi;

struct b200mpi_comm {
  int rank = 0, world = 1, device = 0;
  bool local = false;       // emulated: `world` virtual ranks in this process
  bool vmm = false;         // windows are VMM allocations (else cudaMalloc/cudaIpc)
  bool multicast = false;
  unsigned flags = 0;
  Rendezvous rv;
  std::vector<Window> wins;
  int sig_win = -1, stage_win = -1, p2p_win = -1;
  uint32_t* p2p_cnt = nullptr;       // device: chunks sent to / received from every peer (p2p.cu)
  uint32_t* epoch[kMaxRanks] = {};   // real mode: only [rank]
  int* err_host = nullptr;           // pinned, mapped
  int* err_dev = nullptr;
  KArgs* emu_ring = nullptr;
  int emu_slot = 0;
  static constexpr int kEmuRing = 64;
  // staging layout
  size_t stage_bytes = 0, oneshot_region = 0, oneshot_cap_vecs = 0, twoshot_off = 0, twoshot_bytes = 0;
  // tuning
  size_t oneshot_max = 256 << 10;
  size_t nvls_min = 0;
  int max_blocks = 64;
  int nvls_blocks = 16;  // the switch does the adds, so few CTAs are needed (not yet swept on H100)
  int timeout_ms = 30000;
  // pipelined staged allreduce (user pointers): from pipe_min bytes up; lanes per mode (each lane = 3 CTAs)
  size_t pipe_min = (size_t)8 << 20;
  int pipe_lanes_nvls = 32, pipe_lanes_p2p = 40, pipe_lanes_wide = 32, pipe_depth = 3;
  int pipe_p2p = 0;
  size_t pipe_chunk = (size_t)1 << 20;
  // user-pointer allreduce with NVLS available: below this size the registered zero-copy two-shot is preferred to the staging
  // pipeline. As a kernel it can be faster at mid sizes, but every call on the registered path pays a host agreement round (two
  // rendezvous allgathers, reg_exchange) that graph-replay timings do not show and that the eager callers of this path (torch
  // DDP buckets under the shim) would pay per bucket: 0 = always the pipeline. Not yet measured on H100.
  size_t pipe_pref_min = 0;
  // reduce-scatter: the registered pull instead of the NVLS pipeline once the message is large enough for the host agreement
  // round to disappear next to the kernel time (threshold not yet measured on H100)
  size_t rs_reg_min = (size_t)64 << 20;
  // lazy registration of user buffers (cudaIpc): peer mappings by (rank, allocation id); see reg_exchange()
  size_t reg_min = (size_t)8 << 20;
  int reg_mode = 1;  // 0 off, 1 where it wins (P2P paths: world 2; byte-wise ops), 2 always
  std::map<std::pair<int, unsigned long long>, char*> peer_maps;
  uint64_t reg_hits = 0, reg_opens = 0, reg_refused = 0;
  int n_adopted = 0;   // windows built around b200mpi_mem_alloc allocations (collective count: same on every rank)
  unsigned long long* pipe_dbg = nullptr;   // B200MPI_PIPE_DEBUG=1: device timeline buffer of the last k_pipe launch
  std::atomic<uint64_t> launches{0};
  bool trace_on = false;
  std::vector<TraceRec> trace;
  std::vector<OpStat> stats;
  uint32_t next_tag = 1;
  const float* hyper = nullptr;
};

namespace b200mpi {

static int emu_max_blocks(const b200mpi_comm* c) {
  // all gridDim.x * world CTAs of an emulated launch must be co-resident (1 CTA/SM worst case)
  int b = 132 / c->world;
  return b < 1 ? 1 : b;
}

static DevComm dev_comm(b200mpi_comm* c, int r) {
  DevComm d;
  d.rank = r;
  d.world = c->world;
  for (int p = 0; p < kMaxRanks; p++) d.sig[p] = p < c->world ? reinterpret_cast<uint32_t*>(c->wins[c->sig_win].ptr[p]) : nullptr;
  d.epoch = c->epoch[r];
  d.err = c->err_dev;
  d.timeout_ns = (unsigned long long)c->timeout_ms * 1000000ull;
  return d;
}

static Win win_region(b200mpi_comm* c, int win, size_t off) {
  Win w;
  const Window& W = c->wins[win];
  for (int p = 0; p < kMaxRanks; p++) w.p[p] = p < c->world ? W.ptr[p] + off : nullptr;
  w.mc = W.mc ? W.mc + off : nullptr;
  return w;
}

// Launch helper: real mode passes this rank's args by value; emulated mode
// uploads `world` arg blocks into a device ring and launches gridDim.y=world.
template <typename F>
static int run(b200mpi_comm* c, cudaStream_t stream, int blocks, const char* opname, size_t bytes, int algo,
               const std::vector<KArgs>& args, F&& launcher) {
  Launch l;
  l.stream = stream;
  l.blocks = blocks;
  l.emu_world = 0;
  l.emu_args = nullptr;
  if (c->local) {
    blocks = std::min(blocks, emu_max_blocks(c));
    l.blocks = blocks;
    KArgs* slot = c->emu_ring + (size_t)c->emu_slot * kMaxRanks;
    c->emu_slot = (c->emu_slot + 1) % b200mpi_comm::kEmuRing;
    if (c->emu_slot == 0) CUDA_TRY(cudaStreamSynchronize(stream));  // ring wrap: stay safe
    CUDA_TRY(cudaMemcpyAsync(slot, args.data(), sizeof(KArgs) * c->world, cudaMemcpyHostToDevice, stream));
    l.emu_world = c->world;
    l.emu_args = slot;
  }
  cudaError_t e = launcher(l, args[0]);
  if (e != cudaSuccess) return fail(B200MPI_ERR_CUDA, std::string(opname) + " launch: " + cudaGetErrorString(e));
  c->launches.fetch_add(1, std::memory_order_relaxed);
  {
    OpStat* st = nullptr;
    for (auto& x : c->stats) if (x.op == opname && x.algo == (algo & 3)) { st = &x; break; }
    if (!st) { c->stats.push_back(OpStat{opname, algo & 3, 0, 0}); st = &c->stats.back(); }
    st->calls++;
    st->bytes += bytes;
  }
  if (c->trace_on) c->trace.push_back(TraceRec{opname, bytes, algo, blocks, now_ns()});
  return 0;
}

static int esize(int dt) { return dt == B200MPI_F32 ? 4 : 2; }
static bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// ------------------------------------------------------ window allocation ----
static int window_alloc_local(b200mpi_comm* c, Window& W, size_t bytes) {
  W.bytes = bytes;
  W.mapped = round_up(bytes, 256);
  W.vmm = false;
  for (int r = 0; r < c->world; r++) {
    void* p = nullptr;
    CUDA_TRY(cudaMalloc(&p, W.mapped));
    CUDA_TRY(cudaMemset(p, 0, W.mapped));
    W.ptr[r] = (char*)p;
  }
  W.live = true;
  return 0;
}

static int window_alloc_ipc(b200mpi_comm* c, Window& W, size_t bytes) {
  W.bytes = bytes;
  W.mapped = round_up(bytes, 2 << 20);
  W.vmm = false;
  void* p = nullptr;
  CUDA_TRY(cudaMalloc(&p, W.mapped));
  CUDA_TRY(cudaMemset(p, 0, W.mapped));
  CUDA_TRY(cudaDeviceSynchronize());
  W.ptr[c->rank] = (char*)p;
  cudaIpcMemHandle_t mine;
  CUDA_TRY(cudaIpcGetMemHandle(&mine, p));
  std::vector<cudaIpcMemHandle_t> all(c->world);
  std::string err;
  if (c->rv.allgather(&mine, all.data(), sizeof(mine), c->timeout_ms, &err)) return fail(B200MPI_ERR_SYS, err);
  for (int r = 0; r < c->world; r++) {
    if (r == c->rank) continue;
    void* q = nullptr;
    CUDA_TRY(cudaIpcOpenMemHandle(&q, all[r], cudaIpcMemLazyEnablePeerAccess));
    W.ptr[r] = (char*)q;
  }
  W.live = true;
  return 0;
}

// `own`: an existing exportable VMM allocation of this rank to build the window around (b200mpi_window_adopt), or nullptr
struct OwnAlloc { CUmemGenericAllocationHandle h; char* ptr; size_t mapped; };
static int window_alloc_vmm(b200mpi_comm* c, Window& W, size_t bytes, bool want_mc, const OwnAlloc* own = nullptr) {
  Driver& d = driver();
  std::string err;
  CUmemAllocationProp prop;
  memset(&prop, 0, sizeof(prop));
  prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
  prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  prop.location.id = c->device;
  prop.requestedHandleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
  size_t gran = 0;
  CU_TRY(d.cuMemGetAllocationGranularity_(&gran, &prop, CU_MEM_ALLOC_GRANULARITY_RECOMMENDED));
  CUmulticastObjectProp mprop;
  memset(&mprop, 0, sizeof(mprop));
  if (want_mc) {
    mprop.numDevices = c->world;
    mprop.handleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
    mprop.size = round_up(bytes, gran);
    size_t mg = 0;
    if (d.cuMulticastGetGranularity_(&mg, &mprop, CU_MULTICAST_GRANULARITY_MINIMUM) == CUDA_SUCCESS && mg > gran) gran = mg;
  }
  W.bytes = bytes;
  W.mapped = round_up(bytes, gran);
  W.vmm = true;
  if (own) {
    if (own->mapped % gran) want_mc = false;   // not a multiple of the multicast granularity: peer mappings only
    W.mapped = own->mapped;
    W.adopted = true;
  }
  mprop.size = W.mapped;
  const uint32_t tag = c->next_tag;
  c->next_tag += 2;

  if (own) W.h[c->rank] = own->h;
  else CU_TRY(d.cuMemCreate_(&W.h[c->rank], W.mapped, &prop, 0));
  int myfd = -1;
  CU_TRY(d.cuMemExportToShareableHandle_(&myfd, W.h[c->rank], CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0));
  for (int r = 0; r < c->world; r++)
    if (r != c->rank && c->rv.send_fd(r, tag, myfd, &err)) return fail(B200MPI_ERR_SYS, err);
  for (int r = 0; r < c->world; r++) {
    if (r == c->rank) continue;
    int fd = -1;
    if (c->rv.recv_fd(r, tag, c->timeout_ms, &fd, &err)) return fail(B200MPI_ERR_SYS, err);
    CUresult cr = d.cuMemImportFromShareableHandle_(&W.h[r], (void*)(uintptr_t)fd, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR);
    close(fd);
    if (cr != CUDA_SUCCESS) return fail(B200MPI_ERR_PEER, "import peer window: " + cu_err(cr));
  }
  if (c->rv.barrier(c->timeout_ms, &err)) return fail(B200MPI_ERR_SYS, err);  // everyone imported -> fds may close
  close(myfd);

  CUmemAccessDesc acc;
  acc.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  acc.location.id = c->device;
  acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
  for (int r = 0; r < c->world; r++) {
    if (own && r == c->rank) { W.ptr[r] = own->ptr; continue; }   // already mapped by b200mpi_mem_alloc
    CUdeviceptr va = 0;
    CU_TRY(d.cuMemAddressReserve_(&va, W.mapped, gran, 0, 0));
    CU_TRY(d.cuMemMap_(va, W.mapped, 0, W.h[r], 0));
    CU_TRY(d.cuMemSetAccess_(va, W.mapped, &acc, 1));
    W.ptr[r] = reinterpret_cast<char*>(va);
  }
  if (!own) CUDA_TRY(cudaMemset(W.ptr[c->rank], 0, W.mapped));
  CUDA_TRY(cudaDeviceSynchronize());

  // NVLS: rank 0 creates the multicast object, everyone adds its device and binds its memory.
  if (own) {   // adopted allocations: every rank must bring the same size, and all must still want multicast
    struct { size_t mapped; int mc; } me{W.mapped, want_mc ? 1 : 0}, all[kMaxRanks];
    if (c->rv.allgather(&me, all, sizeof(me), c->timeout_ms, &err)) return fail(B200MPI_ERR_SYS, err);
    for (int r = 0; r < c->world; r++) {
      if (all[r].mapped != W.mapped) return fail(B200MPI_ERR_INVALID, "window_adopt: ranks registered allocations of different sizes");
      if (!all[r].mc) want_mc = false;
    }
  }
  int mc_ok = want_mc ? 1 : 0;
  if (want_mc) {
    int mcfd = -1;
    if (c->rank == 0) {
      CUresult cr = d.cuMulticastCreate_(&W.mch, &mprop);
      if (cr == CUDA_SUCCESS) cr = d.cuMemExportToShareableHandle_(&mcfd, W.mch, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR, 0);
      if (cr != CUDA_SUCCESS) { mc_ok = 0; mcfd = -1; }
    }
    // rank 0 tells everyone whether creation worked before any fd is expected
    int flag0 = mc_ok;
    std::vector<int> flags(c->world);
    if (c->rv.allgather(&flag0, flags.data(), sizeof(int), c->timeout_ms, &err)) return fail(B200MPI_ERR_SYS, err);
    if (!flags[0]) mc_ok = 0;
    if (mc_ok) {
      if (c->rank == 0) {
        for (int r = 1; r < c->world; r++)
          if (c->rv.send_fd(r, tag + 1, mcfd, &err)) return fail(B200MPI_ERR_SYS, err);
      } else {
        int fd = -1;
        if (c->rv.recv_fd(0, tag + 1, c->timeout_ms, &fd, &err)) return fail(B200MPI_ERR_SYS, err);
        CUresult cr = d.cuMemImportFromShareableHandle_(&W.mch, (void*)(uintptr_t)fd, CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR);
        close(fd);
        if (cr != CUDA_SUCCESS) mc_ok = 0;
      }
      if (mc_ok && d.cuMulticastAddDevice_(W.mch, c->device) != CUDA_SUCCESS) mc_ok = 0;
    }
    int mine = mc_ok;
    if (c->rv.allgather(&mine, flags.data(), sizeof(int), c->timeout_ms, &err)) return fail(B200MPI_ERR_SYS, err);
    if (c->rank == 0 && mcfd >= 0) close(mcfd);
    for (int r = 0; r < c->world; r++) if (!flags[r]) mc_ok = 0;
    if (mc_ok) {  // all devices added: bind + map
      CUresult cr = d.cuMulticastBindMem_(W.mch, 0, W.h[c->rank], 0, W.mapped, 0);
      CUdeviceptr va = 0;
      if (cr == CUDA_SUCCESS) cr = d.cuMemAddressReserve_(&va, W.mapped, gran, 0, 0);
      if (cr == CUDA_SUCCESS) cr = d.cuMemMap_(va, W.mapped, 0, W.mch, 0);
      if (cr == CUDA_SUCCESS) cr = d.cuMemSetAccess_(va, W.mapped, &acc, 1);
      if (cr == CUDA_SUCCESS) W.mc = reinterpret_cast<char*>(va);
      else mc_ok = 0;
    }
    mine = mc_ok;
    if (c->rv.allgather(&mine, flags.data(), sizeof(int), c->timeout_ms, &err)) return fail(B200MPI_ERR_SYS, err);
    for (int r = 0; r < c->world; r++) if (!flags[r]) mc_ok = 0;
    if (!mc_ok) W.mc = nullptr;  // (leaks the half-built object; harmless, freed at exit)
  }
  W.live = true;
  return 0;
}

static int window_alloc(b200mpi_comm* c, size_t bytes, int* out) {
  if (bytes == 0) return fail(B200MPI_ERR_INVALID, "window_alloc: zero bytes");
  int id = -1;
  for (size_t i = 0; i < c->wins.size(); i++) if (!c->wins[i].live) { id = (int)i; break; }
  if (id < 0) { c->wins.emplace_back(); id = (int)c->wins.size() - 1; }
  Window W;
  int rc;
  if (c->local) rc = window_alloc_local(c, W, bytes);
  else if (c->vmm) rc = window_alloc_vmm(c, W, bytes, c->multicast);
  else rc = window_alloc_ipc(c, W, bytes);
  if (rc) return rc;
  c->wins[id] = W;
  *out = id;
  return 0;
}

static void window_release(b200mpi_comm* c, Window& W) {
  if (!W.live) return;
  Driver& d = driver();
  if (c->local) {
    for (int r = 0; r < c->world; r++) if (W.ptr[r]) cudaFree(W.ptr[r]);
  } else if (W.vmm) {
    if (W.mc) {
      d.cuMemUnmap_((CUdeviceptr)W.mc, W.mapped);
      d.cuMemAddressFree_((CUdeviceptr)W.mc, W.mapped);
      d.cuMulticastUnbind_(W.mch, c->device, 0, W.mapped);
    }
    if (W.mch) d.cuMemRelease_(W.mch);
    for (int r = 0; r < c->world; r++) {
      if (W.adopted && r == c->rank) continue;   // belongs to b200mpi_mem_alloc / b200mpi_mem_free
      if (W.ptr[r]) { d.cuMemUnmap_((CUdeviceptr)W.ptr[r], W.mapped); d.cuMemAddressFree_((CUdeviceptr)W.ptr[r], W.mapped); }
      if (W.h[r]) d.cuMemRelease_(W.h[r]);
    }
  } else {
    for (int r = 0; r < c->world; r++) {
      if (!W.ptr[r]) continue;
      if (r == c->rank) cudaFree(W.ptr[r]);
      else cudaIpcCloseMemHandle(W.ptr[r]);
    }
  }
  W = Window();
}

// --------------------------------------------------------------- set-up ----
static int comm_finish_init(b200mpi_comm* c, size_t staging_bytes) {
  c->timeout_ms = env_int("B200MPI_TIMEOUT_MS", 30000);
  // Crossovers by world size (not yet measured on H100; benchmarks/allreduce_sweep.py + autotune.py re-derive them):
  //  world 2 : push one-shot wins to 1 MiB, then P2P two-shot; NVLS never pays (1.5 S vs 1.0 S link bytes)
  //  world 8 : one-shot to 64 KiB, NVLS above (S(1+1/N) vs 2S(N-1)/N link bytes per direction)
  if (c->world <= 2) { c->oneshot_max = (size_t)1 << 20; c->nvls_min = (size_t)-1; }
  else if (c->world <= 4) { c->oneshot_max = (size_t)256 << 10; c->nvls_min = (size_t)1 << 20; }
  else { c->oneshot_max = (size_t)64 << 10; c->nvls_min = 0; }
  c->oneshot_max = env_size("B200MPI_ONESHOT_MAX_BYTES", c->oneshot_max);
  c->nvls_min = env_size("B200MPI_NVLS_MIN_BYTES", c->nvls_min);
  c->max_blocks = std::min(env_int("B200MPI_MAX_BLOCKS", c->max_blocks), kMaxBlocks);
  c->nvls_blocks = std::min(env_int("B200MPI_NVLS_BLOCKS", c->nvls_blocks), kMaxBlocks);
  c->pipe_min = env_size("B200MPI_PIPE_MIN_BYTES", c->pipe_min);
  c->pipe_lanes_nvls = std::max(1, std::min(env_int("B200MPI_PIPE_LANES_NVLS", c->pipe_lanes_nvls), kPipeLanes));
  c->pipe_lanes_p2p = std::max(1, std::min(env_int("B200MPI_PIPE_LANES_P2P", c->pipe_lanes_p2p), kPipeLanes));
  c->pipe_lanes_wide = std::max(1, std::min(env_int("B200MPI_PIPE_LANES_WIDE", c->pipe_lanes_wide), kPipeLanes));
  c->pipe_depth = std::max(2, std::min(env_int("B200MPI_PIPE_DEPTH", c->pipe_depth), 8));
  c->pipe_p2p = env_int("B200MPI_PIPE_P2P", c->pipe_p2p);
  c->pipe_chunk = std::max((size_t)16 << 10, env_size("B200MPI_PIPE_CHUNK_BYTES", c->pipe_chunk));
  if (env_int("B200MPI_PIPE_DEBUG", 0) && !c->local) {
    const size_t n = (size_t)3 * kPipeLanes * kPipeDbgChunks * 3;
    CUDA_TRY(cudaMalloc((void**)&c->pipe_dbg, n * sizeof(unsigned long long)));
    CUDA_TRY(cudaMemset(c->pipe_dbg, 0, n * sizeof(unsigned long long)));
  }
  c->reg_min = env_size("B200MPI_REG_MIN_BYTES", c->reg_min);
  c->pipe_pref_min = env_size("B200MPI_PIPE_PREF_MIN_BYTES", c->pipe_pref_min);
  c->rs_reg_min = env_size("B200MPI_RS_REG_MIN_BYTES", c->rs_reg_min);
  c->reg_mode = env_int("B200MPI_REG", c->reg_mode);
  // 16 MiB one-shot region + 144 MiB for the pipelined kernels (44 lanes x 3 slots x 1 MiB = 132 MiB, plus slack)
  if (staging_bytes == 0) staging_bytes = env_size("B200MPI_STAGING_BYTES", c->local ? (size_t)64 << 20 : (size_t)160 << 20);
  // one-shot region: 2 parities x kOneshotBlocks CTAs x kMaxRanks slots x cap
  c->oneshot_cap_vecs = 2048;  // 32 KiB per slot -> 1 MiB max one-shot payload
  c->oneshot_region = (size_t)2 * kOneshotBlocks * kMaxRanks * c->oneshot_cap_vecs * 16;
  if (staging_bytes < c->oneshot_region + ((size_t)4 << 20)) staging_bytes = c->oneshot_region + ((size_t)4 << 20);
  c->stage_bytes = staging_bytes;
  c->twoshot_off = c->oneshot_region;
  c->twoshot_bytes = (staging_bytes - c->oneshot_region) / 4096 * 4096;
  c->oneshot_max = std::min(c->oneshot_max, (size_t)kOneshotBlocks * c->oneshot_cap_vecs * 16);

  CUDA_TRY(cudaHostAlloc((void**)&c->err_host, sizeof(int), cudaHostAllocMapped));
  *c->err_host = 0;
  CUDA_TRY(cudaHostGetDevicePointer((void**)&c->err_dev, c->err_host, 0));
  const int nlocal = c->local ? c->world : 1;
  for (int i = 0; i < nlocal; i++) {
    const int r = c->local ? i : c->rank;
    CUDA_TRY(cudaMalloc((void**)&c->epoch[r], kEpochWordsTotal * sizeof(uint32_t)));
    CUDA_TRY(cudaMemset(c->epoch[r], 0, kEpochWordsTotal * sizeof(uint32_t)));
  }
  if (c->local) CUDA_TRY(cudaMalloc((void**)&c->emu_ring, sizeof(KArgs) * kMaxRanks * b200mpi_comm::kEmuRing));
  int rc = window_alloc(c, kSigWordsTotal * sizeof(uint32_t), &c->sig_win);
  if (rc) return rc;
  rc = window_alloc(c, c->stage_bytes, &c->stage_win);
  if (rc) return rc;
  if (!c->local && c->world > 1 && env_int("B200MPI_P2P", 0)) {  // experimental point-to-point mailboxes (p2p.cu)
    rc = window_alloc(c, kP2PWindowBytes, &c->p2p_win);
    if (rc) return rc;
    CUDA_TRY(cudaMemset(c->wins[c->p2p_win].ptr[c->rank] + kP2PDataBytes, 0, kP2PFlagBytes));
    CUDA_TRY(cudaMalloc((void**)&c->p2p_cnt, 2 * kMaxRanks * sizeof(uint32_t)));
    CUDA_TRY(cudaMemset(c->p2p_cnt, 0, 2 * kMaxRanks * sizeof(uint32_t)));
  }
  CUDA_TRY(cudaDeviceSynchronize());
  if (!c->local) {
    std::string err;
    if (c->rv.barrier(c->timeout_ms, &err)) return fail(B200MPI_ERR_SYS, err);
  }
  return 0;
}

static int select_algo(b200mpi_comm* c, size_t bytes, int dtype, int op, bool symmetric) {
  (void)symmetric;
  if (bytes <= c->oneshot_max) return B200MPI_ALGO_ONESHOT;
  const bool nvls_ok = c->multicast && (op == B200MPI_SUM || dtype != B200MPI_F32);
  if (nvls_ok && bytes >= c->nvls_min) return B200MPI_ALGO_NVLS;
  return B200MPI_ALGO_TWOSHOT;
}

static int blocks_for(b200mpi_comm* c, size_t vecs_per_rank, int per_thread, int cap) {
  size_t b = (vecs_per_rank + (size_t)kThreads * per_thread - 1) / ((size_t)kThreads * per_thread);
  if (b < 1) b = 1;
  if (b > (size_t)cap) b = cap;
  return (int)b;
}

// pointer argument helper: real mode -> the pointer itself; emulated -> ptrs[r]
static const char* in_ptr(b200mpi_comm* c, const void* p, int r) {
  return c->local ? reinterpret_cast<const char* const*>(p)[r] : reinterpret_cast<const char*>(p);
}
static char* out_ptr(b200mpi_comm* c, void* p, int r) {
  return c->local ? reinterpret_cast<char* const*>(p)[r] : reinterpret_cast<char*>(p);
}
static std::vector<int> my_ranks(b200mpi_comm* c) {
  std::vector<int> v;
  if (c->local) for (int r = 0; r < c->world; r++) v.push_back(r);
  else v.push_back(c->rank);
  return v;
}

// ------------------------------------------------ lazy user-buffer registration ----
// Arbitrary device pointers (torch's caching-allocator blocks under the NCCL-ABI shim) become peer-addressable through
// cudaIpc: the allocation that contains the pointer is found with cuMemGetAddressRange, identified by its
// CU_POINTER_ATTRIBUTE_BUFFER_ID (a freed-and-reused address gets a new id), exported once, and opened once per peer.
// Whether a call can go zero-copy must be decided IDENTICALLY on every rank, so every eligible call (size >= reg_min:
// the same test everywhere) trades one 168-byte record per rank through the shm rendezvous (two host barriers, a few
// microseconds against >= 8 MiB of payload); if any rank cannot export (VMM/expandable segments, cudaMallocAsync pools,
// unaligned tensors) all ranks take the staged path together. In a CUDA-graph capture the exchange happens once at
// capture time and the mapped pointers are baked into the graph, like NCCL's graph registration.
struct LocalSeg { unsigned long long id; CUdeviceptr base; size_t size; cudaIpcMemHandle_t h; bool ok; };
static std::mutex g_seg_mu;
static std::map<unsigned long long, LocalSeg> g_segs;   // process-wide: by allocation id

static bool local_seg(const void* p, size_t bytes, LocalSeg* out, size_t* off) {
  Driver& d = driver();
  if (!d.cuMemGetAddressRange_ || !d.cuPointerGetAttribute_ || !p) return false;
  CUdeviceptr base = 0;
  size_t size = 0;
  unsigned long long id = 0;
  if (d.cuMemGetAddressRange_(&base, &size, (CUdeviceptr)p) != CUDA_SUCCESS) return false;
  if (d.cuPointerGetAttribute_(&id, CU_POINTER_ATTRIBUTE_BUFFER_ID, (CUdeviceptr)p) != CUDA_SUCCESS) return false;
  if ((CUdeviceptr)p + bytes > base + size) return false;
  std::lock_guard<std::mutex> l(g_seg_mu);
  auto it = g_segs.find(id);
  if (it == g_segs.end()) {
    LocalSeg sgm;
    memset(&sgm, 0, sizeof(sgm));
    sgm.id = id; sgm.base = base; sgm.size = size;
    sgm.ok = cudaIpcGetMemHandle(&sgm.h, (void*)base) == cudaSuccess;
    if (!sgm.ok) cudaGetLastError();
    if (g_segs.size() > 4096) g_segs.clear();   // ids of freed allocations never come back; keep the table bounded
    it = g_segs.emplace(id, sgm).first;
  }
  *out = it->second;
  *off = (size_t)((CUdeviceptr)p - base);
  return it->second.ok;
}

struct RegRec {   // one per rank per eligible call; must stay <= kRvScratch (256) bytes
  unsigned long long id[2];
  unsigned long long off[2];
  cudaIpcMemHandle_t h[2];
  int ok;          // both buffers exportable through cudaIpc
  int win;         // adopted (ncclCommRegister'ed) window that contains BOTH buffers, or -1
  unsigned long long woff[2];   // their offsets inside it
};
static_assert(sizeof(RegRec) <= kRvScratch, "RegRec must fit the rendezvous scratch slot");

static int adopted_window_of(b200mpi_comm* c, const void* p, size_t bytes, size_t* off) {
  for (size_t i = 0; i < c->wins.size(); i++) {
    const Window& W = c->wins[i];
    if (!W.live || !W.adopted) continue;
    const char* b = W.ptr[c->rank];
    if ((const char*)p >= b && (const char*)p + bytes <= b + W.mapped) { *off = (size_t)((const char*)p - b); return (int)i; }
  }
  return -1;
}

// Collective (host). On REG_IPC wins[k].p[r] = rank r's buffer k mapped in this process; on REG_SYM both buffers of
// every rank sit at the same offsets of the same adopted window (*sym_win, sym_off[2]).
enum { REG_NONE = 0, REG_IPC = 1, REG_SYM = 2 };
static int reg_exchange(b200mpi_comm* c, const void* in, void* out, size_t in_bytes, size_t out_bytes, bool want_ipc, Win* win_in,
                        Win* win_out, int* sym_win = nullptr, size_t* sym_off = nullptr) {
  RegRec mine;
  memset(&mine, 0, sizeof(mine));
  LocalSeg sg[2];
  size_t off[2] = {0, 0};
  const void* ptr[2] = {in, out};
  const size_t nb[2] = {in_bytes, out_bytes};
  mine.win = -1;
  if (c->n_adopted > 0 && sym_win) {
    size_t o0 = 0, o1 = 0;
    const int w0 = adopted_window_of(c, in, in_bytes, &o0), w1 = adopted_window_of(c, out, out_bytes, &o1);
    if (w0 >= 0 && w0 == w1 && o0 % 16 == 0 && o1 % 16 == 0) { mine.win = w0; mine.woff[0] = o0; mine.woff[1] = o1; }
  }
  mine.ok = want_ipc ? 1 : 0;
  for (int k = 0; k < 2 && mine.ok; k++) {
    if (!aligned16(ptr[k]) || !local_seg(ptr[k], nb[k], &sg[k], &off[k])) { mine.ok = 0; break; }
    mine.id[k] = sg[k].id; mine.off[k] = off[k]; mine.h[k] = sg[k].h;
  }
  std::vector<RegRec> all(c->world);
  std::string err;
  if (c->rv.allgather(&mine, all.data(), sizeof(RegRec), c->timeout_ms, &err)) return REG_NONE;
  bool sym = mine.win >= 0;
  for (auto& r : all) sym = sym && r.win == mine.win && r.woff[0] == mine.woff[0] && r.woff[1] == mine.woff[1];
  if (sym) {
    *sym_win = mine.win; sym_off[0] = mine.woff[0]; sym_off[1] = mine.woff[1];
    c->reg_hits++;
    return REG_SYM;
  }
  for (auto& r : all) if (!r.ok) { c->reg_refused += want_ipc ? 1 : 0; return REG_NONE; }
  Win* wins[2] = {win_in, win_out};
  bool ok = true;
  for (int k = 0; k < 2 && ok; k++) {
    memset(wins[k], 0, sizeof(Win));
    for (int r = 0; r < c->world && ok; r++) {
      if (r == c->rank) { wins[k]->p[r] = (char*)const_cast<void*>(ptr[k]); continue; }
      auto key = std::make_pair(r, all[r].id[k]);
      auto it = c->peer_maps.find(key);
      if (it == c->peer_maps.end()) {
        void* q = nullptr;
        if (cudaIpcOpenMemHandle(&q, all[r].h[k], cudaIpcMemLazyEnablePeerAccess) != cudaSuccess) { cudaGetLastError(); ok = false; break; }
        it = c->peer_maps.emplace(key, (char*)q).first;
        c->reg_opens++;
      }
      wins[k]->p[r] = it->second + all[r].off[k];
    }
  }
  // a failed open on one rank must send everybody to the staged path: second (tiny) agreement round
  int good = ok ? 1 : 0;
  std::vector<int> goods(c->world);
  if (c->rv.allgather(&good, goods.data(), sizeof(int), c->timeout_ms, &err)) return REG_NONE;
  for (int g : goods) if (!g) { c->reg_refused++; return REG_NONE; }
  c->reg_hits++;
  return REG_IPC;
}
static bool reg_wanted(b200mpi_comm* c, size_t bytes, bool p2p_path) {
  if (c->local || c->world < 2 || c->reg_mode == 0 || bytes < c->reg_min) return false;
  return c->reg_mode >= 2 || p2p_path;
}

// Pipelined staged collectives (k_pipe): `nbytes` = per-rank payload; `wide` ops keep `world` regions per staging slot.
static bool pipe_wanted(b200mpi_comm* c, size_t full_bytes) {
  return full_bytes >= c->pipe_min && !(c->flags & B200MPI_FLAG_NO_PIPE) && c->world > 1;
}
// without NVLS the pipelined kernel has to win against the zero-copy registered path (which it does not) and against the
// barrier-based staged kernel (unmeasured since the copy fix): opt-in until the sweep says otherwise
static bool pipe_p2p_ok(b200mpi_comm* c) { return c->pipe_p2p || c->local; }
// Geometry of one pipelined launch (pure arithmetic, checked exhaustively on the host by csrc/tests/comm_host_test.cu):
// L lanes of three CTAs, D staging slots per lane, chunks of `cv` vectors (x `regions` for the wide ops).
struct PipePlan { int lanes; int depth; size_t chunk_vecs; size_t regions; bool fits; };
static PipePlan pipe_plan(const b200mpi_comm* c, int kind, int mode, size_t nbytes, bool wide) {
  int L = wide ? c->pipe_lanes_wide : (mode == MODE_NVLS ? c->pipe_lanes_nvls : c->pipe_lanes_p2p);
  if (kind == PIPE_BROADCAST && mode == MODE_NVLS) L = kPipeLanes;   // one pushing rank: give it every lane
  if (c->local) L = std::max(1, std::min(L, emu_max_blocks(const_cast<b200mpi_comm*>(c)) / 3));
  const int D = c->pipe_depth;
  const size_t nvec = (nbytes + 15) / 16;
  const size_t regions = wide ? (size_t)c->world : 1;
  // chunk: a slot (regions x chunk) of at most pipe_chunk bytes, L*D slots must fit the staging region, and every lane
  // should get >= 2 chunks when the message allows it
  size_t cv = std::min(c->pipe_chunk / 16, c->twoshot_bytes / 16 / ((size_t)L * D)) / regions;
  cv = std::min(cv, std::max((size_t)1024 / regions, nvec / ((size_t)L * 2)));
  cv = std::max((size_t)c->world, cv / c->world * c->world);
  return PipePlan{L, D, cv, regions, (size_t)L * D * cv * regions * 16 <= c->twoshot_bytes};
}

template <typename Fill>
static int pipe_op(b200mpi_comm* c, const char* name, int kind, int mode, int dtype, size_t nbytes, bool wide,
                   cudaStream_t stream, int algo, Fill&& fill) {
  if (mode == MODE_NVLS && !(c->multicast && c->wins[c->stage_win].mc)) mode = MODE_P2P;
  const PipePlan plan = pipe_plan(c, kind, mode, nbytes, wide);
  if (!plan.fits) return fail(B200MPI_ERR_INVALID, std::string(name) + ": staging window too small");
  const int L = plan.lanes, D = plan.depth;
  const size_t nvec = (nbytes + 15) / 16, cv = plan.chunk_vecs;
  const auto ranks = my_ranks(c);
  std::vector<KArgs> args(c->local ? c->world : 1);
  for (size_t k = 0; k < ranks.size(); k++) {
    KArgs& a = args[k];
    memset(&a, 0, sizeof(a));
    a.c = dev_comm(c, ranks[k]);
    a.buf = win_region(c, c->stage_win, c->twoshot_off);
    a.nbytes = nbytes; a.nvec = nvec; a.per = cv; a.scale = 1.0f;
    a.lanes = L; a.depth = D;
    a.dbg = c->pipe_dbg;
    fill(a, ranks[k]);
  }
  return run(c, stream, 3 * L, name, nbytes, algo, args,
             [&](const Launch& l, const KArgs& a) { return launch_pipe(l, a, kind, dtype, mode); });
}

static int do_allreduce(b200mpi_comm* c, bool sym, int win, size_t off, const void* in, void* out, size_t count,
                        int dtype, int op, float scale, int algo, cudaStream_t stream) {
  if (count == 0) return 0;
  if (dtype < 0 || dtype > 2 || op < 0 || op > 2) return fail(B200MPI_ERR_INVALID, "allreduce: bad dtype/op");
  const size_t nbytes = count * esize(dtype);
  if (sym) {
    if (win < 0 || win >= (int)c->wins.size() || !c->wins[win].live) return fail(B200MPI_ERR_INVALID, "allreduce_sym: bad window");
    if (off % 16 || nbytes % 16 || off + nbytes > c->wins[win].bytes)
      return fail(B200MPI_ERR_INVALID, "allreduce_sym: region must be 16-byte aligned/sized and inside the window");
  }
  if (algo == B200MPI_ALGO_AUTO) algo = select_algo(c, nbytes, dtype, op, sym);
  if (algo == B200MPI_ALGO_NVLS && !(c->multicast && (op == B200MPI_SUM || dtype != B200MPI_F32))) algo = B200MPI_ALGO_TWOSHOT;
  if (algo == B200MPI_ALGO_ONESHOT && nbytes > (size_t)kOneshotBlocks * c->oneshot_cap_vecs * 16) algo = B200MPI_ALGO_TWOSHOT;
  const auto ranks = my_ranks(c);
  std::vector<KArgs> args(c->local ? c->world : 1);

  if (algo == B200MPI_ALGO_ONESHOT) {
    const size_t nvec = (nbytes + 15) / 16;
    int blocks = blocks_for(c, nvec, 1, kOneshotBlocks);
    if (c->local) blocks = std::min(blocks, emu_max_blocks(c));
    if ((nvec + blocks - 1) / blocks > c->oneshot_cap_vecs) algo = B200MPI_ALGO_TWOSHOT;  // does not fit the per-CTA slots
  }
  if (algo == B200MPI_ALGO_ONESHOT) {
    const size_t nvec = (nbytes + 15) / 16;
    int blocks = blocks_for(c, nvec, 1, kOneshotBlocks);
    if (c->local) blocks = std::min(blocks, emu_max_blocks(c));
    for (size_t k = 0; k < ranks.size(); k++) {
      const int r = ranks[k];
      KArgs& a = args[k];
      memset(&a, 0, sizeof(a));
      a.c = dev_comm(c, r);
      a.buf = win_region(c, c->stage_win, 0);
      a.in = sym ? c->wins[win].ptr[r] + off : in_ptr(c, in, r);
      a.out = sym ? c->wins[win].ptr[r] + off : out_ptr(c, out, r);
      a.nbytes = nbytes; a.nvec = nvec; a.per = c->oneshot_cap_vecs;
      a.scale = scale; a.op = op;
      a.in_aligned = aligned16(a.in); a.out_aligned = aligned16(a.out);
    }
    return run(c, stream, blocks, "allreduce", nbytes, algo, args,
               [&](const Launch& l, const KArgs& a) { return launch_allreduce_oneshot(l, a, dtype); });
  }

  const int mode = algo == B200MPI_ALGO_NVLS ? MODE_NVLS : MODE_P2P;
  const int cap = mode == MODE_NVLS ? c->nvls_blocks : c->max_blocks;
  if (sym) {
    const size_t nvec = nbytes / 16;
    const size_t per = (nvec + c->world - 1) / c->world;
    const int blocks = blocks_for(c, per, mode == MODE_NVLS ? 4 : 2, cap);
    for (size_t k = 0; k < ranks.size(); k++) {
      KArgs& a = args[k];
      memset(&a, 0, sizeof(a));
      a.c = dev_comm(c, ranks[k]);
      a.buf = win_region(c, win, off);
      a.nbytes = nbytes; a.nvec = nvec; a.per = per; a.scale = scale; a.op = op;
    }
    return run(c, stream, blocks, "allreduce", nbytes, algo, args,
               [&](const Launch& l, const KArgs& a) { return launch_allreduce_twoshot(l, a, dtype, mode, false); });
  }
  // large, P2P path: register the user buffers (cudaIpc) and run the zero-copy two-shot straight on them
  const bool ipc_ok = reg_wanted(c, nbytes, mode == MODE_P2P || nbytes < c->pipe_pref_min);
  if (nbytes % 16 == 0 && !c->local && nbytes >= c->reg_min && (ipc_ok || c->n_adopted > 0)) {
    Win win_in, win_out;
    int sw = -1;
    size_t so[2] = {0, 0};
    const int kind = reg_exchange(c, in, out, nbytes, nbytes, ipc_ok, &win_in, &win_out, &sw, so);
    if (kind == REG_SYM && so[0] == so[1])   // registered (ncclMemAlloc + ncclCommRegister) and in place: zero-copy NVLS on the window
      return do_allreduce(c, true, sw, so[0], nullptr, nullptr, count, dtype, op, scale, B200MPI_ALGO_AUTO, stream);
    if (kind == REG_IPC) {
      const size_t nvec = nbytes / 16;
      const size_t per = (nvec + c->world - 1) / c->world;
      const int blocks = blocks_for(c, per, 2, c->max_blocks);
      KArgs& a = args[0];
      memset(&a, 0, sizeof(a));
      a.c = dev_comm(c, c->rank);
      a.buf = win_in;
      if (in != out) a.param = win_out;
      a.nbytes = nbytes; a.nvec = nvec; a.per = per; a.scale = scale; a.op = op;
      return run(c, stream, blocks, "allreduce_reg", nbytes, B200MPI_ALGO_TWOSHOT, args,
                 [&](const Launch& l, const KArgs& a) { return launch_allreduce_twoshot(l, a, dtype, MODE_P2P, false); });
    }
  }
  // staged, large: ONE pipelined kernel (copy-in / reduce / copy-out CTAs chained through flags per lane)
  if (pipe_wanted(c, nbytes) && (mode == MODE_NVLS || pipe_p2p_ok(c)))
    return pipe_op(c, "allreduce_pipe", PIPE_ALLREDUCE, mode, dtype, nbytes, false, stream, algo, [&](KArgs& a, int r) {
      a.in = in_ptr(c, in, r);
      a.out = out_ptr(c, out, r);
      a.scale = scale; a.op = op;
      a.in_aligned = aligned16(a.in); a.out_aligned = aligned16(a.out);
    });
  // staged: chunk through the two-shot staging region
  const size_t chunk_max = c->twoshot_bytes / 16 * 16;
  for (size_t done = 0; done < nbytes; done += chunk_max) {
    const size_t nb = std::min(chunk_max, nbytes - done);
    const size_t nvec = (nb + 15) / 16;
    const size_t per = (nvec + c->world - 1) / c->world;
    const int blocks = blocks_for(c, per, mode == MODE_NVLS ? 4 : 2, cap);
    for (size_t k = 0; k < ranks.size(); k++) {
      const int r = ranks[k];
      KArgs& a = args[k];
      memset(&a, 0, sizeof(a));
      a.c = dev_comm(c, r);
      a.buf = win_region(c, c->stage_win, c->twoshot_off);
      a.in = in_ptr(c, in, r) + done;
      a.out = out_ptr(c, out, r) + done;
      a.nbytes = nb; a.nvec = nvec; a.per = per; a.scale = scale; a.op = op;
      a.in_aligned = aligned16(a.in); a.out_aligned = aligned16(a.out);
    }
    int rc = run(c, stream, blocks, "allreduce", nb, algo, args,
                 [&](const Launch& l, const KArgs& a) { return launch_allreduce_twoshot(l, a, dtype, mode, true); });
    if (rc) return rc;
  }
  return 0;
}

// generic staged op over a per-rank payload of `nbytes`, chunked so that
// `slots` staging slots of the chunk fit the two-shot staging region.
template <typename Fill, typename L>
static int staged_op(b200mpi_comm* c, const char* name, size_t nbytes, int slots, cudaStream_t stream, Fill&& fill, L&& launcher) {
  if (nbytes == 0) return 0;
  const size_t chunk_max = (c->twoshot_bytes / slots) / 4096 * 4096;
  const auto ranks = my_ranks(c);
  std::vector<KArgs> args(c->local ? c->world : 1);
  for (size_t done = 0; done < nbytes; done += chunk_max) {
    const size_t nb = std::min(chunk_max, nbytes - done);
    const size_t nvec = (nb + 15) / 16;
    const int blocks = blocks_for(c, nvec, 2, c->max_blocks);
    for (size_t k = 0; k < ranks.size(); k++) {
      KArgs& a = args[k];
      memset(&a, 0, sizeof(a));
      a.c = dev_comm(c, ranks[k]);
      a.buf = win_region(c, c->stage_win, c->twoshot_off);
      a.nbytes = nb; a.nvec = nvec; a.per = nvec; a.scale = 1.0f;
      fill(a, ranks[k], done, nb);
    }
    int rc = run(c, stream, blocks, name, nb, 0, args, launcher);
    if (rc) return rc;
  }
  return 0;
}

// ---- zero-copy collectives on a symmetric window region (k_*_sym) ------------------------------------------------
static int sym_check(b200mpi_comm* c, int win, size_t off, size_t nbytes, const char* what) {
  if (win < 0 || win >= (int)c->wins.size() || !c->wins[win].live) return fail(B200MPI_ERR_INVALID, std::string(what) + ": bad window");
  if (off % 16 || nbytes % 16 || off + nbytes > c->wins[win].bytes)
    return fail(B200MPI_ERR_INVALID, std::string(what) + ": region must be 16-byte aligned/sized and inside the window");
  return 0;
}
template <typename Fill, typename L>
static int sym_op(b200mpi_comm* c, const char* name, int win, size_t off, size_t nbytes, size_t per_vecs, int mode, int per_thread,
                  cudaStream_t stream, Fill&& fill, L&& launcher) {
  const auto ranks = my_ranks(c);
  std::vector<KArgs> args(c->local ? c->world : 1);
  const size_t nvec = nbytes / 16;
  const int blocks = blocks_for(c, per_vecs, per_thread, mode == MODE_NVLS ? c->nvls_blocks * 2 : c->max_blocks);
  for (size_t k = 0; k < ranks.size(); k++) {
    KArgs& a = args[k];
    memset(&a, 0, sizeof(a));
    a.c = dev_comm(c, ranks[k]);
    a.buf = win_region(c, win, off);
    a.nbytes = nbytes; a.nvec = nvec; a.per = per_vecs; a.scale = 1.0f;
    fill(a, ranks[k]);
  }
  return run(c, stream, blocks, name, nbytes, mode == MODE_NVLS ? B200MPI_ALGO_NVLS : B200MPI_ALGO_TWOSHOT, args, launcher);
}

// ---- exportable allocations (the shim's ncclMemAlloc) and windows built around them (ncclCommRegister) ----------------
struct MemAlloc { CUmemGenericAllocationHandle h; size_t mapped; int device; };
static std::mutex g_mem_mu;
static std::map<char*, MemAlloc> g_mem;   // by base pointer

static int mem_alloc(size_t bytes, void** out) {
  Driver& d = driver();
  if (!d.ok) return fail(B200MPI_ERR_UNSUPPORTED, "mem_alloc: CUDA VMM driver entry points unavailable");
  int dev = 0;
  CUDA_TRY(cudaGetDevice(&dev));
  CUmemAllocationProp prop;
  memset(&prop, 0, sizeof(prop));
  prop.type = CU_MEM_ALLOCATION_TYPE_PINNED;
  prop.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  prop.location.id = dev;
  prop.requestedHandleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
  size_t gran = 0;
  CU_TRY(d.cuMemGetAllocationGranularity_(&gran, &prop, CU_MEM_ALLOC_GRANULARITY_RECOMMENDED));
  CUmulticastObjectProp mprop;   // round to the multicast granularity of a full box so the allocation can be bound later
  memset(&mprop, 0, sizeof(mprop));
  mprop.numDevices = 2;
  mprop.handleTypes = CU_MEM_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR;
  mprop.size = round_up(bytes, gran);
  size_t mg = 0;
  if (d.cuMulticastGetGranularity_(&mg, &mprop, CU_MULTICAST_GRANULARITY_MINIMUM) == CUDA_SUCCESS && mg > gran) gran = mg;
  MemAlloc m;
  m.mapped = round_up(bytes ? bytes : 1, gran);
  m.device = dev;
  CU_TRY(d.cuMemCreate_(&m.h, m.mapped, &prop, 0));
  CUdeviceptr va = 0;
  CUresult r = d.cuMemAddressReserve_(&va, m.mapped, gran, 0, 0);
  if (r == CUDA_SUCCESS) r = d.cuMemMap_(va, m.mapped, 0, m.h, 0);
  CUmemAccessDesc acc;
  acc.location.type = CU_MEM_LOCATION_TYPE_DEVICE;
  acc.location.id = dev;
  acc.flags = CU_MEM_ACCESS_FLAGS_PROT_READWRITE;
  if (r == CUDA_SUCCESS) r = d.cuMemSetAccess_(va, m.mapped, &acc, 1);
  if (r != CUDA_SUCCESS) { d.cuMemRelease_(m.h); return fail(B200MPI_ERR_CUDA, "mem_alloc: " + cu_err(r)); }
  std::lock_guard<std::mutex> l(g_mem_mu);
  g_mem[(char*)va] = m;
  *out = (void*)va;
  return 0;
}
static int mem_free(void* p) {
  MemAlloc m;
  {
    std::lock_guard<std::mutex> l(g_mem_mu);
    auto it = g_mem.find((char*)p);
    if (it == g_mem.end()) return fail(B200MPI_ERR_INVALID, "mem_free: not a b200mpi_mem_alloc pointer");
    m = it->second;
    g_mem.erase(it);
  }
  Driver& d = driver();
  cudaDeviceSynchronize();
  d.cuMemUnmap_((CUdeviceptr)p, m.mapped);
  d.cuMemAddressFree_((CUdeviceptr)p, m.mapped);
  d.cuMemRelease_(m.h);
  return 0;
}

}  // namespace b200mpi

// =============================================================== C ABI ====
extern "C" {

const char* b200mpi_last_error(void) { return g_err.c_str(); }
const char* b200mpi_version(void) { return B200MPI_VERSION; }

int b200mpi_comm_init(b200mpi_comm_t* out, int rank, int world, int device, const char* job_id,
                      size_t staging_bytes, unsigned flags) {
  if (!out || world < 1 || world > kMaxRanks || rank < 0 || rank >= world) return fail(B200MPI_ERR_INVALID, "comm_init: bad rank/world (max 8 ranks per box)");
  CUDA_TRY(cudaSetDevice(device));
  CUDA_TRY(cudaFree(0));
  auto* c = new b200mpi_comm;
  c->rank = rank; c->world = world; c->device = device; c->flags = flags;
  std::string err;
  // rendezvous / setup timeout: B200MPI_INIT_TIMEOUT_MS, else the collective timeout, else 30 s
  const int timeout = env_int("B200MPI_INIT_TIMEOUT_MS", env_int("B200MPI_TIMEOUT_MS", 30000));
  if (c->rv.attach(job_id ? job_id : "default", rank, world, device, timeout, &err)) { delete c; return fail(B200MPI_ERR_SYS, err); }
  // capability consensus: VMM fd export + multicast need every rank to agree
  Driver& d = driver();
  int caps[2] = {0, 0};
  if (d.ok && !(flags & B200MPI_FLAG_FORCE_IPC) && !env_int("B200MPI_FORCE_IPC", 0)) {
    int v = 0;
    if (d.cuDeviceGetAttribute_(&v, CU_DEVICE_ATTRIBUTE_HANDLE_TYPE_POSIX_FILE_DESCRIPTOR_SUPPORTED, device) == CUDA_SUCCESS && v) caps[0] = 1;
    v = 0;
    if (caps[0] && !(flags & B200MPI_FLAG_NO_MULTICAST) && !env_int("B200MPI_NO_MULTICAST", 0) &&
        d.cuDeviceGetAttribute_(&v, CU_DEVICE_ATTRIBUTE_MULTICAST_SUPPORTED, device) == CUDA_SUCCESS && v) caps[1] = 1;
  }
  struct Cap { int vmm, mc, dev; } mine{caps[0], caps[1], device};
  std::vector<Cap> all(world);
  if (c->rv.allgather(&mine, all.data(), sizeof(Cap), timeout, &err)) { delete c; return fail(B200MPI_ERR_SYS, err); }
  bool vmm = true, mc = world > 1;
  std::set<int> devs;
  for (auto& x : all) { vmm = vmm && x.vmm; mc = mc && x.mc; devs.insert(x.dev); }
  if ((int)devs.size() != world) mc = false;  // ranks sharing a device: NVLS needs distinct devices
  c->vmm = vmm;
  c->multicast = vmm && mc;
  for (auto& x : all) {
    if (x.dev != device) {
      int can = 0;
      cudaDeviceCanAccessPeer(&can, device, x.dev);
      if (!can) { delete c; return fail(B200MPI_ERR_PEER, "no P2P access to device " + std::to_string(x.dev)); }
    }
  }
  int rc = comm_finish_init(c, staging_bytes);
  if (rc) { std::string keep = g_err; b200mpi_comm_destroy(c); g_err = keep; return rc; }
  // multicast may have been demoted during window creation: agree on the final state
  int have = (c->wins[c->stage_win].mc && c->wins[c->sig_win].mc) ? 1 : 0;
  std::vector<int> haves(world);
  if (c->rv.allgather(&have, haves.data(), sizeof(int), timeout, &err)) return fail(B200MPI_ERR_SYS, err);
  for (int h : haves) if (!h) c->multicast = false;
  if (getenv("B200MPI_DEBUG") && rank == 0)
    fprintf(stderr, "[b200mpi] comm up: world=%d vmm=%d multicast(NVLS)=%d staging=%zu MiB\n", world, (int)c->vmm, (int)c->multicast, c->stage_bytes >> 20);
  *out = c;
  return 0;
}

int b200mpi_comm_init_local(b200mpi_comm_t* out, int world, int device, size_t staging_bytes, unsigned flags) {
  if (!out || world < 1 || world > kMaxRanks) return fail(B200MPI_ERR_INVALID, "comm_init_local: bad world");
  CUDA_TRY(cudaSetDevice(device));
  CUDA_TRY(cudaFree(0));
  auto* c = new b200mpi_comm;
  c->rank = 0; c->world = world; c->device = device; c->flags = flags; c->local = true;
  int rc = comm_finish_init(c, staging_bytes);
  if (rc) { std::string keep = g_err; b200mpi_comm_destroy(c); g_err = keep; return rc; }
  *out = c;
  return 0;
}

int b200mpi_comm_destroy(b200mpi_comm_t c) {
  if (!c) return 0;
  cudaSetDevice(c->device);
  cudaDeviceSynchronize();
  if (!c->local && c->rv.header()) { std::string err; c->rv.barrier(2000, &err); }
  for (auto& kv : c->peer_maps) cudaIpcCloseMemHandle(kv.second);
  c->peer_maps.clear();
  for (auto& W : c->wins) window_release(c, W);
  for (int r = 0; r < kMaxRanks; r++) if (c->epoch[r]) cudaFree(c->epoch[r]);
  if (c->emu_ring) cudaFree(c->emu_ring);
  if (c->p2p_cnt) cudaFree(c->p2p_cnt);
  if (c->pipe_dbg) cudaFree(c->pipe_dbg);
  if (c->err_host) cudaFreeHost(c->err_host);
  c->rv.detach(c->rank == 0);
  delete c;
  return 0;
}

int b200mpi_comm_rank(b200mpi_comm_t c) { return c->rank; }
int b200mpi_comm_world(b200mpi_comm_t c) { return c->world; }
int b200mpi_comm_is_local(b200mpi_comm_t c) { return c->local ? 1 : 0; }
int b200mpi_comm_has_multicast(b200mpi_comm_t c) { return c->multicast ? 1 : 0; }
uint64_t b200mpi_comm_launch_count(b200mpi_comm_t c) { return c->launches.load(); }
int b200mpi_comm_check_error(b200mpi_comm_t c) {
  int e = *(volatile int*)c->err_host;
  if (e) { *c->err_host = 0; return fail(B200MPI_ERR_TIMEOUT, "device-side wait timed out waiting for rank " + std::to_string(e - 1)); }
  return 0;
}
int b200mpi_comm_host_barrier(b200mpi_comm_t c) {
  if (c->local) return 0;
  std::string err;
  if (c->rv.barrier(c->timeout_ms, &err)) return fail(B200MPI_ERR_SYS, err);
  return 0;
}
int b200mpi_comm_host_allgather(b200mpi_comm_t c, const void* in, void* out, size_t bytes) {
  if (c->local) { for (int r = 0; r < c->world; r++) memcpy((char*)out + r * bytes, in, bytes); return 0; }
  std::string err;
  if (c->rv.allgather(in, out, bytes, c->timeout_ms, &err)) return fail(B200MPI_ERR_SYS, err);
  return 0;
}

int b200mpi_window_alloc(b200mpi_comm_t c, size_t bytes, int* win) { return window_alloc(c, bytes, win); }
int b200mpi_window_free(b200mpi_comm_t c, int win) {
  if (win < 0 || win >= (int)c->wins.size() || !c->wins[win].live) return fail(B200MPI_ERR_INVALID, "window_free: bad window");
  cudaDeviceSynchronize();
  if (!c->local) { std::string err; if (c->rv.barrier(c->timeout_ms, &err)) return fail(B200MPI_ERR_SYS, err); }
  if (c->wins[win].adopted && c->n_adopted > 0) c->n_adopted--;
  window_release(c, c->wins[win]);
  return 0;
}
void* b200mpi_window_ptr(b200mpi_comm_t c, int win, int rank) {
  if (win < 0 || win >= (int)c->wins.size() || !c->wins[win].live) return nullptr;
  if (rank < 0) rank = c->rank;
  if (rank >= c->world) return nullptr;
  return c->wins[win].ptr[rank];
}
void* b200mpi_window_mc_ptr(b200mpi_comm_t c, int win) {
  if (win < 0 || win >= (int)c->wins.size() || !c->wins[win].live) return nullptr;
  return c->wins[win].mc;
}
size_t b200mpi_window_size(b200mpi_comm_t c, int win) {
  if (win < 0 || win >= (int)c->wins.size() || !c->wins[win].live) return 0;
  return c->wins[win].bytes;
}

int b200mpi_mem_alloc(size_t bytes, void** ptr) { return mem_alloc(bytes, ptr); }
int b200mpi_mem_free(void* ptr) { return mem_free(ptr); }
int b200mpi_mem_lookup(const void* p, void** base, size_t* size) {
  std::lock_guard<std::mutex> l(g_mem_mu);
  auto it = g_mem.upper_bound((char*)const_cast<void*>(p));
  if (it == g_mem.begin()) return 0;
  --it;
  if ((const char*)p >= it->first + it->second.mapped) return 0;
  if (base) *base = it->first;
  if (size) *size = it->second.mapped;
  return 1;
}
int b200mpi_window_adopt(b200mpi_comm_t c, void* base, int* win) {
  if (c->local || !c->vmm) return fail(B200MPI_ERR_UNSUPPORTED, "window_adopt: needs a multi-process communicator with VMM fd export");
  MemAlloc m;
  {
    std::lock_guard<std::mutex> l(g_mem_mu);
    auto it = g_mem.find((char*)base);
    if (it == g_mem.end()) return fail(B200MPI_ERR_INVALID, "window_adopt: not the base of a b200mpi_mem_alloc allocation");
    m = it->second;
  }
  if (m.device != c->device) return fail(B200MPI_ERR_INVALID, "window_adopt: allocation lives on another device");
  int id = -1;
  for (size_t i = 0; i < c->wins.size(); i++) if (!c->wins[i].live) { id = (int)i; break; }
  if (id < 0) { c->wins.emplace_back(); id = (int)c->wins.size() - 1; }
  Window W;
  OwnAlloc own{m.h, (char*)base, m.mapped};
  int rc = window_alloc_vmm(c, W, m.mapped, c->multicast, &own);
  if (rc) return rc;
  c->wins[id] = W;
  c->n_adopted++;
  *win = id;
  return 0;
}

int b200mpi_allreduce_sym(b200mpi_comm_t c, int win, size_t offset, size_t count, b200mpi_dtype_t dtype,
                          b200mpi_op_t op, float scale, b200mpi_algo_t algo, void* stream) {
  return do_allreduce(c, true, win, offset, nullptr, nullptr, count, dtype, op, scale, algo, (cudaStream_t)stream);
}
int b200mpi_allreduce(b200mpi_comm_t c, const void* in, void* out, size_t count, b200mpi_dtype_t dtype,
                      b200mpi_op_t op, float scale, b200mpi_algo_t algo, void* stream) {
  return do_allreduce(c, false, -1, 0, in, out, count, dtype, op, scale, algo, (cudaStream_t)stream);
}

size_t b200mpi_slice_elems(size_t count, int world, b200mpi_dtype_t dtype) {
  const size_t n = dtype == B200MPI_F32 ? 4 : 8;
  const size_t nvec = (count + n - 1) / n;
  return (nvec + world - 1) / world * n;
}

int b200mpi_allreduce_sgd_sym(b200mpi_comm_t c, int gwin, size_t goff, int pwin, size_t poff, int lwin, size_t loff,
                              void* momentum, size_t count, b200mpi_dtype_t gdtype, float scale, float lr, float mu,
                              float wd, int nesterov, int first_step, b200mpi_algo_t algo, void* stream) {
  if (count == 0) return 0;
  const size_t n = gdtype == B200MPI_F32 ? 4 : 8;
  auto okwin = [&](int w) { return w >= 0 && w < (int)c->wins.size() && c->wins[w].live; };
  if (!okwin(gwin) || !okwin(pwin) || (lwin >= 0 && !okwin(lwin))) return fail(B200MPI_ERR_INVALID, "allreduce_sgd: bad window");
  if (count % n || goff % 16 || poff % 16 || (lwin >= 0 && loff % 16)) return fail(B200MPI_ERR_INVALID, "allreduce_sgd: count must be a multiple of the 16-byte vector and offsets 16-byte aligned");
  if (goff + count * esize(gdtype) > c->wins[gwin].bytes || poff + count * 4 > c->wins[pwin].bytes) return fail(B200MPI_ERR_INVALID, "allreduce_sgd: region outside window");
  int mode = MODE_P2P;
  if (algo == B200MPI_ALGO_NVLS || (algo == B200MPI_ALGO_AUTO && c->multicast && count * esize(gdtype) >= c->nvls_min && count * esize(gdtype) > c->oneshot_max)) mode = MODE_NVLS;
  if (mode == MODE_NVLS && !(c->multicast && c->wins[gwin].mc && c->wins[pwin].mc)) mode = MODE_P2P;
  const size_t nvec = count / n, per = (nvec + c->world - 1) / c->world;
  const int blocks = blocks_for(c, per, mode == MODE_NVLS ? 4 : 2, mode == MODE_NVLS ? c->nvls_blocks : c->max_blocks);
  const auto ranks = my_ranks(c);
  std::vector<KArgs> args(c->local ? c->world : 1);
  for (size_t k = 0; k < ranks.size(); k++) {
    const int r = ranks[k];
    KArgs& a = args[k];
    memset(&a, 0, sizeof(a));
    a.c = dev_comm(c, r);
    a.buf = win_region(c, gwin, goff);
    a.param = win_region(c, pwin, poff);
    if (lwin >= 0) a.lowp = win_region(c, lwin, loff);
    a.mom = reinterpret_cast<float*>(c->local ? reinterpret_cast<void* const*>(momentum)[r] : momentum);
    a.nbytes = count * esize(gdtype); a.nvec = nvec; a.per = per;
    a.scale = scale; a.lr = lr; a.mu = mu; a.wd = wd; a.nesterov = nesterov; a.first_step = first_step;
    a.hyper = c->hyper;
  }
  return run(c, (cudaStream_t)stream, blocks, "allreduce_sgd", count * esize(gdtype), mode == MODE_NVLS ? B200MPI_ALGO_NVLS : B200MPI_ALGO_TWOSHOT, args,
             [&](const Launch& l, const KArgs& a) { return launch_allreduce_sgd(l, a, gdtype, mode); });
}

int b200mpi_set_hyper_ptr(b200mpi_comm_t c, const float* p) { c->hyper = p; return 0; }

int b200mpi_broadcast_bytes(b200mpi_comm_t c, void* buf, size_t bytes, int root, void* stream) {
  if (root < 0 || root >= c->world) return fail(B200MPI_ERR_INVALID, "broadcast: bad root");
  const int mode = c->multicast ? MODE_NVLS : MODE_P2P;
  const bool bc_ipc = reg_wanted(c, bytes, mode == MODE_P2P || c->world == 2);
  if (bytes % 16 == 0 && !c->local && bytes >= c->reg_min && (bc_ipc || c->n_adopted > 0)) {   // zero-copy: root stores into the peers' buffers
    Win w, w2;
    int sw = -1;
    size_t so[2] = {0, 0};
    const int kind = reg_exchange(c, buf, buf, bytes, bytes, bc_ipc, &w, &w2, &sw, so);
    if (kind == REG_SYM) return b200mpi_broadcast_sym(c, sw, so[0], bytes, root, stream);
    if (kind == REG_IPC) {
      std::vector<KArgs> args(1);
      KArgs& a = args[0];
      memset(&a, 0, sizeof(a));
      a.c = dev_comm(c, c->rank);
      a.buf = w;
      a.nbytes = bytes; a.nvec = bytes / 16; a.per = bytes / 16; a.scale = 1.0f; a.root = root;
      return run(c, (cudaStream_t)stream, blocks_for(c, bytes / 16, 4, c->max_blocks), "broadcast_reg", bytes, B200MPI_ALGO_TWOSHOT, args,
                 [&](const Launch& l, const KArgs& a) { return launch_broadcast_sym(l, a, MODE_P2P); });
    }
  }
  if (pipe_wanted(c, bytes) && (mode == MODE_NVLS || pipe_p2p_ok(c)))
    return pipe_op(c, "broadcast_pipe", PIPE_BROADCAST, mode, DT_F32, bytes, false, (cudaStream_t)stream, mode == MODE_NVLS ? B200MPI_ALGO_NVLS : B200MPI_ALGO_TWOSHOT,
                   [&](KArgs& a, int r) {
                     a.root = root;
                     a.in = out_ptr(c, buf, r); a.out = out_ptr(c, buf, r);
                     a.in_aligned = a.out_aligned = aligned16(a.in);
                   });
  return staged_op(c, "broadcast", bytes, 1, (cudaStream_t)stream,
                   [&](KArgs& a, int r, size_t done, size_t) {
                     a.root = root;
                     a.in = out_ptr(c, buf, r) + done; a.out = out_ptr(c, buf, r) + done;
                     a.in_aligned = a.out_aligned = aligned16(a.in);
                   },
                   [&](const Launch& l, const KArgs& a) { return launch_broadcast(l, a, mode); });
}
int b200mpi_broadcast(b200mpi_comm_t c, void* buf, size_t count, b200mpi_dtype_t dtype, int root, void* stream) {
  return b200mpi_broadcast_bytes(c, buf, count * esize(dtype), root, stream);
}

int b200mpi_allgather(b200mpi_comm_t c, const void* in, void* out, size_t count, b200mpi_dtype_t dtype, void* stream) {
  const size_t total = count * esize(dtype);
  if (total % 16 == 0 && reg_wanted(c, total * c->world, true)) {   // zero-copy: every rank stores its block into every output
    Win win_in, win_out;
    if (reg_exchange(c, in, out, total, total * c->world, true, &win_in, &win_out) == REG_IPC) {
      std::vector<KArgs> args(1);
      KArgs& a = args[0];
      memset(&a, 0, sizeof(a));
      a.c = dev_comm(c, c->rank);
      a.buf = win_out;
      a.in = (const char*)in;
      a.nbytes = total * c->world; a.nvec = total / 16 * c->world; a.per = total / 16; a.scale = 1.0f;
      return run(c, (cudaStream_t)stream, blocks_for(c, total / 16, 4, c->max_blocks), "allgather_reg", total, B200MPI_ALGO_TWOSHOT, args,
                 [&](const Launch& l, const KArgs& a) { return launch_allgather_sym(l, a, MODE_P2P); });
    }
  }
  if (pipe_wanted(c, total * c->world) && (c->multicast || pipe_p2p_ok(c))) {
    const int mode = c->multicast ? MODE_NVLS : MODE_P2P;
    return pipe_op(c, "allgather_pipe", PIPE_ALLGATHER, mode, DT_F32, total, true, (cudaStream_t)stream, mode == MODE_NVLS ? B200MPI_ALGO_NVLS : B200MPI_ALGO_TWOSHOT,
                   [&](KArgs& a, int r) {
                     a.in = in_ptr(c, in, r); a.out = out_ptr(c, out, r);
                     a.in_aligned = aligned16(a.in);
                     a.out_aligned = aligned16(a.out) && (total % 16 == 0);
                     a.ustride = total;
                   });
  }
  // chunks of the per-rank payload land at out + r*total + done
  return staged_op(c, "allgather", total, c->world, (cudaStream_t)stream,
                   [&](KArgs& a, int r, size_t done, size_t nb) {
                     a.in = in_ptr(c, in, r) + done;
                     a.out = out_ptr(c, out, r) + done;
                     a.in_aligned = aligned16(a.in);
                     a.out_aligned = aligned16(a.out) && (total % 16 == 0);
                     a.ustride = total;
                     (void)nb;
                   },
                   [&](const Launch& l, const KArgs& a) {
                     return launch_allgather(l, a);
                   });
}

// Adasum allreduce (adasum.cu): one launch, slice-parallel tree over peer memory. UNSUPPORTED (the caller falls back to the
// gather + local tree) when the world is not a power of two or the tensor does not fit the staging layout
// [dot board][A: world*per vectors][W: the same as fp32].
size_t b200mpi_adasum_max_bytes(b200mpi_comm_t c, b200mpi_dtype_t dtype) {
  if (!c || dtype < 0 || dtype > 2 || c->twoshot_bytes <= kAdaDotBytes + 4096) return 0;
  const size_t expand = dtype == B200MPI_F32 ? 1 : 2;                     // fp32 work copy per byte of T
  const size_t room = c->twoshot_bytes - kAdaDotBytes - 4096;             // slack for the round-up to world * per vectors
  return room / (1 + expand) / 256 * 256;
}
int b200mpi_adasum(b200mpi_comm_t c, const void* in, void* out, size_t count, b200mpi_dtype_t dtype, void* stream) {
  if (count == 0) return 0;
  if (dtype < 0 || dtype > 2) return fail(B200MPI_ERR_UNSUPPORTED, "adasum: f32 / bf16 / f16 only");
  if (c->world < 2 || (c->world & (c->world - 1))) return fail(B200MPI_ERR_UNSUPPORTED, "adasum kernel: the world must be a power of two >= 2");
  const size_t nbytes = count * esize(dtype);
  if (nbytes > b200mpi_adasum_max_bytes(c, dtype)) return fail(B200MPI_ERR_UNSUPPORTED, "adasum kernel: tensor larger than the staging layout");
  const size_t nvec = (nbytes + 15) / 16;
  const size_t per = (nvec + c->world - 1) / c->world;
  int blocks = blocks_for(c, per, 1, std::min(c->max_blocks, kAdaMaxBlocks));
  if (c->local) blocks = std::min(blocks, emu_max_blocks(c));
  const auto ranks = my_ranks(c);
  std::vector<KArgs> args(c->local ? c->world : 1);
  for (size_t k = 0; k < ranks.size(); k++) {
    const int r = ranks[k];
    KArgs& a = args[k];
    memset(&a, 0, sizeof(a));
    a.c = dev_comm(c, r);
    a.buf = win_region(c, c->stage_win, c->twoshot_off);
    a.in = in_ptr(c, in, r);
    a.out = out_ptr(c, out, r);
    a.nbytes = nbytes; a.nvec = nvec; a.per = per; a.scale = 1.0f;
    a.in_aligned = aligned16(a.in); a.out_aligned = aligned16(a.out);
  }
  return run(c, (cudaStream_t)stream, blocks, "adasum", nbytes, B200MPI_ALGO_TWOSHOT, args,
             [&](const Launch& l, const KArgs& a) { return launch_adasum(l, a, dtype); });
}

int b200mpi_reduce_scatter(b200mpi_comm_t c, const void* in, void* out, size_t count, b200mpi_dtype_t dtype,
                           b200mpi_op_t op, float scale, void* stream) {
  const size_t total = count * esize(dtype);
  if (dtype < 0 || dtype > 2 || op < 0 || op > 2) return fail(B200MPI_ERR_INVALID, "reduce_scatter: bad dtype/op");
  const bool rs_nvls = c->multicast && (op == B200MPI_SUM || dtype != B200MPI_F32);
  // zero-copy: pull the owned block from every input. Without NVLS always; with NVLS from rs_reg_min bytes of input up: the P2P
  // pull runs at the link's read rate with no staging copy of the N x larger input; below that size the per-call host
  // agreement of the registered path would cost more than the kernel gains
  if (total % 16 == 0 && reg_wanted(c, total * c->world, !rs_nvls || total * c->world >= c->rs_reg_min)) {
    Win win_in, win_out;
    if (reg_exchange(c, in, out, total * c->world, total, true, &win_in, &win_out) == REG_IPC) {
      std::vector<KArgs> args(1);
      KArgs& a = args[0];
      memset(&a, 0, sizeof(a));
      a.c = dev_comm(c, c->rank);
      a.buf = win_in;
      a.out = (char*)out;
      a.nbytes = total * c->world; a.nvec = total / 16 * c->world; a.per = total / 16; a.scale = scale; a.op = op;
      return run(c, (cudaStream_t)stream, blocks_for(c, total / 16, 2, c->max_blocks), "reduce_scatter_reg", total, B200MPI_ALGO_TWOSHOT, args,
                 [&](const Launch& l, const KArgs& a) { return launch_reduce_scatter_sym(l, a, dtype, MODE_P2P); });
    }
  }
  if (pipe_wanted(c, total * c->world) && (rs_nvls || pipe_p2p_ok(c))) {
    const int mode = rs_nvls ? MODE_NVLS : MODE_P2P;
    return pipe_op(c, "reduce_scatter_pipe", PIPE_REDUCE_SCATTER, mode, dtype, total, true, (cudaStream_t)stream, mode == MODE_NVLS ? B200MPI_ALGO_NVLS : B200MPI_ALGO_TWOSHOT,
                   [&](KArgs& a, int r) {
                     a.in = in_ptr(c, in, r); a.out = out_ptr(c, out, r);
                     a.in_aligned = aligned16(a.in) && (total % 16 == 0); a.out_aligned = aligned16(a.out);
                     a.op = op; a.scale = scale; a.ustride = total;
                   });
  }
  return staged_op(c, "reduce_scatter", total, c->world, (cudaStream_t)stream,
                   [&](KArgs& a, int r, size_t done, size_t) {
                     a.in = in_ptr(c, in, r) + done; a.out = out_ptr(c, out, r) + done;
                     a.in_aligned = aligned16(a.in) && (total % 16 == 0); a.out_aligned = aligned16(a.out);
                     a.op = op; a.scale = scale; a.ustride = total;
                   },
                   [&](const Launch& l, const KArgs& a) { return launch_reduce_scatter(l, a, dtype); });
}

int b200mpi_reduce(b200mpi_comm_t c, const void* in, void* out, size_t count, b200mpi_dtype_t dtype, b200mpi_op_t op,
                   float scale, int root, void* stream) {
  if (root < 0 || root >= c->world) return fail(B200MPI_ERR_INVALID, "reduce: bad root");
  return staged_op(c, "reduce", count * esize(dtype), 1, (cudaStream_t)stream,
                   [&](KArgs& a, int r, size_t done, size_t) {
                     a.in = in_ptr(c, in, r) + done;
                     a.out = (c->local || out) ? out_ptr(c, out, r) + done : nullptr;
                     a.in_aligned = aligned16(a.in); a.out_aligned = aligned16(a.out);
                     a.op = op; a.scale = scale; a.root = root;
                   },
                   [&](const Launch& l, const KArgs& a) { return launch_reduce(l, a, dtype); });
}

int b200mpi_allgather_sym(b200mpi_comm_t c, int win, size_t offset, size_t slice_bytes, void* stream) {
  if (slice_bytes == 0) return 0;
  int rc = sym_check(c, win, offset, slice_bytes * c->world, "allgather_sym");
  if (rc) return rc;
  const int mode = (c->multicast && c->wins[win].mc) ? MODE_NVLS : MODE_P2P;
  return sym_op(c, "allgather_sym", win, offset, slice_bytes * c->world, slice_bytes / 16, mode, 4, (cudaStream_t)stream,
                [&](KArgs&, int) {}, [&](const Launch& l, const KArgs& a) { return launch_allgather_sym(l, a, mode); });
}

int b200mpi_reduce_scatter_sym(b200mpi_comm_t c, int win, size_t offset, size_t slice_count, b200mpi_dtype_t dtype,
                               b200mpi_op_t op, float scale, void* out, void* stream) {
  if (slice_count == 0) return 0;
  if (dtype < 0 || dtype > 2 || op < 0 || op > 2) return fail(B200MPI_ERR_INVALID, "reduce_scatter_sym: bad dtype/op");
  const size_t slice_bytes = slice_count * esize(dtype);
  int rc = sym_check(c, win, offset, slice_bytes * c->world, "reduce_scatter_sym");
  if (rc) return rc;
  if (!c->local && out && !aligned16(out)) return fail(B200MPI_ERR_INVALID, "reduce_scatter_sym: output must be 16-byte aligned");
  const int mode = (c->multicast && c->wins[win].mc && (op == B200MPI_SUM || dtype != B200MPI_F32)) ? MODE_NVLS : MODE_P2P;
  return sym_op(c, "reduce_scatter_sym", win, offset, slice_bytes * c->world, slice_bytes / 16, mode, mode == MODE_NVLS ? 4 : 2,
                (cudaStream_t)stream,
                [&](KArgs& a, int r) { a.op = op; a.scale = scale; a.out = out ? out_ptr(c, out, r) : nullptr; },
                [&](const Launch& l, const KArgs& a) { return launch_reduce_scatter_sym(l, a, dtype, mode); });
}

int b200mpi_broadcast_sym(b200mpi_comm_t c, int win, size_t offset, size_t bytes, int root, void* stream) {
  if (bytes == 0) return 0;
  if (root < 0 || root >= c->world) return fail(B200MPI_ERR_INVALID, "broadcast_sym: bad root");
  int rc = sym_check(c, win, offset, bytes, "broadcast_sym");
  if (rc) return rc;
  const int mode = (c->multicast && c->wins[win].mc) ? MODE_NVLS : MODE_P2P;
  return sym_op(c, "broadcast_sym", win, offset, bytes, bytes / 16, mode, 4, (cudaStream_t)stream,
                [&](KArgs& a, int) { a.root = root; }, [&](const Launch& l, const KArgs& a) { return launch_broadcast_sym(l, a, mode); });
}

int b200mpi_alltoall(b200mpi_comm_t c, const void* in, void* out, size_t count, b200mpi_dtype_t dtype, void* stream) {
  const size_t total = count * esize(dtype);
  return staged_op(c, "alltoall", total, c->world, (cudaStream_t)stream,
                   [&](KArgs& a, int r, size_t done, size_t) {
                     a.in = in_ptr(c, in, r) + done; a.out = out_ptr(c, out, r) + done;
                     a.in_aligned = aligned16(a.in) && (total % 16 == 0);
                     a.out_aligned = aligned16(a.out) && (total % 16 == 0);
                     a.ustride = total;
                   },
                   [&](const Launch& l, const KArgs& a) { return launch_alltoall(l, a); });
}

int b200mpi_barrier(b200mpi_comm_t c, void* stream) {
  const auto ranks = my_ranks(c);
  std::vector<KArgs> args(c->local ? c->world : 1);
  for (size_t k = 0; k < ranks.size(); k++) { memset(&args[k], 0, sizeof(KArgs)); args[k].c = dev_comm(c, ranks[k]); }
  return run(c, (cudaStream_t)stream, 1, "barrier", 0, 0, args, [&](const Launch& l, const KArgs& a) { return launch_barrier(l, a); });
}

int b200mpi_scale_cast(const void* in, b200mpi_dtype_t idt, void* out, b200mpi_dtype_t odt, size_t count, float scale, void* stream) {
  cudaError_t e = launch_scale_cast((cudaStream_t)stream, in, idt, out, odt, count, scale);
  if (e != cudaSuccess) return fail(B200MPI_ERR_CUDA, std::string("scale_cast: ") + cudaGetErrorString(e));
  return 0;
}

int b200mpi_set_tuning(b200mpi_comm_t c, size_t oneshot_max, size_t nvls_min, int max_blocks, int timeout_ms) {
  if (oneshot_max != (size_t)-1) c->oneshot_max = std::min(oneshot_max, (size_t)kOneshotBlocks * c->oneshot_cap_vecs * 16);
  if (nvls_min != (size_t)-1) c->nvls_min = nvls_min;
  if (max_blocks > 0) { c->max_blocks = std::min(max_blocks, kMaxBlocks); c->nvls_blocks = std::min(max_blocks, kMaxBlocks); }  // explicit tuning applies to both paths
  if (timeout_ms > 0) c->timeout_ms = timeout_ms;
  return 0;
}
int b200mpi_get_tuning(b200mpi_comm_t c, size_t* oneshot_max, size_t* nvls_min, int* max_blocks, int* timeout_ms) {
  if (oneshot_max) *oneshot_max = c->oneshot_max;
  if (nvls_min) *nvls_min = c->nvls_min;
  if (max_blocks) *max_blocks = c->max_blocks;
  if (timeout_ms) *timeout_ms = c->timeout_ms;
  return 0;
}
int b200mpi_set_pipe(b200mpi_comm_t c, size_t min_bytes, int lanes_nvls, int lanes_p2p, int depth, size_t chunk_bytes) {
  if (min_bytes != (size_t)-1) c->pipe_min = min_bytes;
  if (lanes_nvls > 0) c->pipe_lanes_nvls = std::min(lanes_nvls, kPipeLanes);
  if (lanes_p2p > 0) { c->pipe_lanes_p2p = std::min(lanes_p2p, kPipeLanes); c->pipe_p2p = 1; }
  if (lanes_nvls > 0 && lanes_p2p > 0) c->pipe_lanes_wide = std::min(std::max(lanes_nvls, lanes_p2p), kPipeLanes);
  if (depth > 0) c->pipe_depth = std::max(2, std::min(depth, 8));
  if (chunk_bytes > 0) c->pipe_chunk = std::max((size_t)16 << 10, chunk_bytes);
  return 0;
}
// Timeline of the last pipelined launch (needs B200MPI_PIPE_DEBUG=1 at creation): out[role][lane][chunk][3] in ns
// relative to the earliest stamp; returns the number of u64 written (0 when disabled).
size_t b200mpi_pipe_timeline(b200mpi_comm_t c, unsigned long long* out, size_t cap) {
  const size_t n = (size_t)3 * kPipeLanes * kPipeDbgChunks * 3;
  if (!c->pipe_dbg || cap < n) return 0;
  cudaDeviceSynchronize();
  cudaMemcpy(out, c->pipe_dbg, n * sizeof(unsigned long long), cudaMemcpyDeviceToHost);
  cudaMemset(c->pipe_dbg, 0, n * sizeof(unsigned long long));
  return n;
}
int b200mpi_set_reg(b200mpi_comm_t c, int mode, size_t min_bytes) {
  if (mode >= 0) c->reg_mode = mode;
  if (min_bytes != (size_t)-1) c->reg_min = min_bytes;
  return 0;
}
int b200mpi_reg_stats(b200mpi_comm_t c, uint64_t* zero_copy_calls, uint64_t* handles_opened, uint64_t* refused) {
  if (zero_copy_calls) *zero_copy_calls = c->reg_hits;
  if (handles_opened) *handles_opened = c->reg_opens;
  if (refused) *refused = c->reg_refused;
  return 0;
}
int b200mpi_select_algo(b200mpi_comm_t c, size_t bytes, b200mpi_dtype_t dtype, b200mpi_op_t op, int symmetric) {
  return select_algo(c, bytes, dtype, op, symmetric != 0);
}

int b200mpi_comm_has_p2p(b200mpi_comm_t c) { return c->p2p_win >= 0 ? 1 : 0; }

// Plans one batch: per-stream chunk offsets for operations that share a (direction, peer) stream, totals for the commit
// kernel. Split from the launch so the host test can check it without a device.
static int p2p_plan(int rank, int world, const b200mpi_p2p_op_t* ops, int nops, P2PArgs* a, P2PCommit* add) {
  if (nops < 1 || nops > kMaxP2POps) return fail(B200MPI_ERR_INVALID, "p2p_batch: between 1 and 64 operations per batch");
  memset(add, 0, sizeof(*add));
  a->nops = nops;
  for (int i = 0; i < nops; i++) {
    const b200mpi_p2p_op_t& o = ops[i];
    if (o.peer < 0 || o.peer >= world) return fail(B200MPI_ERR_INVALID, "p2p_batch: peer out of range");
    if (o.peer == rank) return fail(B200MPI_ERR_UNSUPPORTED, "p2p_batch: send/recv to self (copy locally instead)");
    const void* buf = o.is_send ? o.send : o.recv;
    if (o.bytes && !buf) return fail(B200MPI_ERR_INVALID, "p2p_batch: null buffer");
    const size_t chunks = (o.bytes + kP2PChunk - 1) / kP2PChunk;
    if (chunks > 0x3fffffffu) return fail(B200MPI_ERR_INVALID, "p2p_batch: message too large");
    uint32_t& total = add->n[(o.is_send ? 0 : kMaxRanks) + o.peer];
    P2POp& d = a->ops[i];
    d.user = reinterpret_cast<const char*>(buf);
    d.bytes = o.bytes;
    d.peer = o.peer;
    d.is_send = o.is_send ? 1 : 0;
    d.seq_off = total;
    total += (uint32_t)chunks;
  }
  return 0;
}

int b200mpi_p2p_batch(b200mpi_comm_t c, const b200mpi_p2p_op_t* ops, int nops, void* stream) {
  if (c->local) return fail(B200MPI_ERR_UNSUPPORTED, "p2p_batch: not available on emulated communicators");
  if (c->p2p_win < 0) return fail(B200MPI_ERR_UNSUPPORTED, "point-to-point is experimental: set B200MPI_P2P=1 for every rank before the communicator is created");
  P2PArgs a;
  P2PCommit add;
  int rc = p2p_plan(c->rank, c->world, ops, nops, &a, &add);
  if (rc) return rc;
  a.c = dev_comm(c, c->rank);
  a.box = win_region(c, c->p2p_win, 0);
  a.cnt = c->p2p_cnt;
  cudaError_t e = launch_p2p_batch((cudaStream_t)stream, a, add);
  if (e != cudaSuccess) return fail(B200MPI_ERR_CUDA, std::string("p2p_batch launch: ") + cudaGetErrorString(e));
  c->launches.fetch_add(1, std::memory_order_relaxed);
  size_t bytes = 0;
  for (int i = 0; i < nops; i++) bytes += ops[i].bytes;
  {
    OpStat* st = nullptr;
    for (auto& x : c->stats) if (x.op == kP2PName && x.algo == 0) { st = &x; break; }
    if (!st) { c->stats.push_back(OpStat{kP2PName, 0, 0, 0}); st = &c->stats.back(); }
    st->calls++;
    st->bytes += bytes;
  }
  return 0;
}
int b200mpi_send(b200mpi_comm_t c, const void* buf, size_t bytes, int peer, void* stream) {
  b200mpi_p2p_op_t o{buf, nullptr, bytes, peer, 1};
  return b200mpi_p2p_batch(c, &o, 1, stream);
}
int b200mpi_recv(b200mpi_comm_t c, void* buf, size_t bytes, int peer, void* stream) {
  b200mpi_p2p_op_t o{nullptr, buf, bytes, peer, 0};
  return b200mpi_p2p_batch(c, &o, 1, stream);
}

int b200mpi_comm_stats_json(b200mpi_comm_t c, char* buf, size_t cap) {
  // {"rank":r,"world":w,"launches":n,"ops":[{"op":"allreduce","algo":"nvls","calls":k,"bytes":b},...]}; returns the length
  // needed (excluding NUL), like snprintf. Kernels replayed from a CUDA graph are not host launches and are not counted
  // here (DataParallelTrainer adds replays x per-capture counts on top).
  static const char* algos[] = {"auto", "oneshot", "twoshot", "nvls"};
  std::string o = "{\"rank\": " + std::to_string(c->rank) + ", \"world\": " + std::to_string(c->world) +
                  ", \"launches\": " + std::to_string((unsigned long long)c->launches.load()) + ", \"ops\": [";
  bool first = true;
  for (auto& x : c->stats) {
    if (!first) o += ", ";
    first = false;
    o += std::string("{\"op\": \"") + x.op + "\", \"algo\": \"" + algos[x.algo & 3] + "\", \"calls\": " +
         std::to_string((unsigned long long)x.calls) + ", \"bytes\": " + std::to_string((unsigned long long)x.bytes) + "}";
  }
  o += "]}";
  if (buf && cap) {
    size_t n = o.size() < cap - 1 ? o.size() : cap - 1;
    memcpy(buf, o.data(), n);
    buf[n] = 0;
  }
  return (int)o.size();
}

int b200mpi_trace_enable(b200mpi_comm_t c, int on) { c->trace_on = on != 0; return 0; }
int b200mpi_trace_dump(b200mpi_comm_t c, const char* path) {
  FILE* f = fopen(path, "a");
  if (!f) return fail(B200MPI_ERR_SYS, std::string("trace_dump: cannot open ") + path);
  static const char* algos[] = {"auto", "oneshot", "twoshot", "nvls"};
  for (auto& t : c->trace)
    fprintf(f, "{\"rank\": %d, \"op\": \"%s\", \"bytes\": %zu, \"algo\": \"%s\", \"blocks\": %d, \"t_ns\": %llu}\n", c->rank, t.op,
            t.bytes, algos[t.algo & 3], t.blocks, (unsigned long long)t.t_ns);
  fclose(f);
  c->trace.clear();
  return 0;
}

}  // extern "C"
