// Host-only checks of the runtime's launch planning (no GPU needed: nothing here calls into CUDA). The translation unit
// includes comm.cc so that its file-static helpers are visible; kernel launchers resolve from libb200mpi.so.
// Built and run by `make test_comm_host` and tests/test_native_cpu.py.
#include "../runtime/comm.cc"

#include <cstdio>
#include <cstring>

static int g_failed = 0;
#define EXPECT(cond)                                                        \
  do {                                                                      \
    if (!(cond)) { printf("FAILED %s:%d: %s\n", __FILE__, __LINE__, #cond); g_failed++; } \
  } while (0)

int main() {
  b200mpi_comm* c = new b200mpi_comm;
  c->rank = 3;
  c->world = 8;
  c->multicast = true;
  c->oneshot_max = 64 << 10;
  c->nvls_min = 0;

  // ---- algorithm selection: measured crossovers (tuning.json) are thresholds on the message size
  EXPECT(select_algo(c, 1024, B200MPI_F32, B200MPI_SUM, true) == B200MPI_ALGO_ONESHOT);
  EXPECT(select_algo(c, 64 << 10, B200MPI_F32, B200MPI_SUM, true) == B200MPI_ALGO_ONESHOT);
  EXPECT(select_algo(c, (64 << 10) + 16, B200MPI_F32, B200MPI_SUM, true) == B200MPI_ALGO_NVLS);
  EXPECT(select_algo(c, 1 << 30, B200MPI_BF16, B200MPI_SUM, false) == B200MPI_ALGO_NVLS);
  EXPECT(select_algo(c, 1 << 20, B200MPI_F32, B200MPI_MAX, true) == B200MPI_ALGO_TWOSHOT);   // no f32 min/max in the switch
  EXPECT(select_algo(c, 1 << 20, B200MPI_BF16, B200MPI_MAX, true) == B200MPI_ALGO_NVLS);
  c->multicast = false;
  EXPECT(select_algo(c, 1 << 20, B200MPI_F32, B200MPI_SUM, true) == B200MPI_ALGO_TWOSHOT);
  c->multicast = true;
  c->nvls_min = (size_t)-1;   // world <= 2 default: NVLS never wins
  EXPECT(select_algo(c, 1 << 30, B200MPI_F32, B200MPI_SUM, true) == B200MPI_ALGO_TWOSHOT);

  // ---- grid sizing: ceil(vectors / (threads x vectors-per-thread)) clamped to [1, cap]
  EXPECT(blocks_for(c, 0, 1, 32) == 1);
  EXPECT(blocks_for(c, 1, 4, 16) == 1);
  EXPECT(blocks_for(c, (size_t)kThreads * 4, 4, 16) == 1);
  EXPECT(blocks_for(c, (size_t)kThreads * 4 + 1, 4, 16) == 2);
  EXPECT(blocks_for(c, (size_t)1 << 30, 2, 64) == 64);
  EXPECT(emu_max_blocks(c) == 132 / 8);
  EXPECT(esize(B200MPI_F32) == 4 && esize(B200MPI_BF16) == 2 && esize(B200MPI_F16) == 2);

  // ---- per-(op, algorithm) counters -> JSON
  EXPECT(b200mpi_comm_stats_json(c, nullptr, 0) > 0);
  c->stats.push_back(OpStat{"allreduce", B200MPI_ALGO_NVLS, 2, 4096});
  c->stats.push_back(OpStat{"allreduce_sgd", B200MPI_ALGO_TWOSHOT, 9, 123456789012ull});
  c->launches = 11;
  const int n = b200mpi_comm_stats_json(c, nullptr, 0);
  char* buf = new char[n + 1];
  EXPECT(b200mpi_comm_stats_json(c, buf, n + 1) == n && (int)strlen(buf) == n);
  EXPECT(strstr(buf, "\"rank\": 3") && strstr(buf, "\"launches\": 11"));
  EXPECT(strstr(buf, "{\"op\": \"allreduce\", \"algo\": \"nvls\", \"calls\": 2, \"bytes\": 4096}"));
  EXPECT(strstr(buf, "{\"op\": \"allreduce_sgd\", \"algo\": \"twoshot\", \"calls\": 9, \"bytes\": 123456789012}"));
  char tiny[10];
  EXPECT(b200mpi_comm_stats_json(c, tiny, sizeof(tiny)) == n && strlen(tiny) == sizeof(tiny) - 1);   // truncates, NUL-terminated

  // ---- argument validation happens before anything touches the device
  EXPECT(b200mpi_slice_elems(1000, 8, B200MPI_F32) > 0);
  EXPECT(b200mpi_bn_supported(12544, 256) == 1 && b200mpi_bn_supported(12544, 12) == 0 && b200mpi_bn_supported(0, 64) == 0);
  EXPECT(b200mpi_bn_workspace_floats(64) == (size_t)4 * 64 + (size_t)296 * 2 * 64 + 4);

  // ---- point-to-point batch planning: chunk offsets per (direction, peer) stream, totals for the commit kernel
  {
    char bufs[8];
    b200mpi_p2p_op_t ops[5] = {
        {bufs, nullptr, (size_t)3 << 20, 1, 1},          // send 3 MiB to 1  -> 3 chunks, offset 0
        {nullptr, bufs, 100, 1, 0},                       // recv 100 B from 1 -> 1 chunk, offset 0 (other direction)
        {bufs, nullptr, ((size_t)1 << 20) + 1, 1, 1},     // send 1 MiB + 1 to 1 -> 2 chunks, offset 3
        {bufs, nullptr, 0, 2, 1},                          // empty message -> 0 chunks
        {nullptr, bufs, (size_t)1 << 20, 1, 0},           // recv 1 MiB from 1 -> 1 chunk, offset 1
    };
    P2PArgs a;
    P2PCommit add;
    EXPECT(p2p_plan(0, 4, ops, 5, &a, &add) == 0);
    EXPECT(a.nops == 5 && a.ops[0].seq_off == 0 && a.ops[1].seq_off == 0 && a.ops[2].seq_off == 3 && a.ops[4].seq_off == 1);
    EXPECT(a.ops[0].is_send == 1 && a.ops[1].is_send == 0 && a.ops[2].bytes == ((size_t)1 << 20) + 1);
    EXPECT(add.n[1] == 5 && add.n[kMaxRanks + 1] == 2 && add.n[2] == 0 && add.n[kMaxRanks + 2] == 0);
    EXPECT(p2p_plan(1, 4, ops, 5, &a, &add) == B200MPI_ERR_UNSUPPORTED);   // peer == self
    EXPECT(p2p_plan(0, 2, ops + 3, 1, &a, &add) == B200MPI_ERR_INVALID);   // peer 2 outside a 2-rank world
    EXPECT(p2p_plan(0, 4, ops, 0, &a, &add) == B200MPI_ERR_INVALID);
    // mailbox geometry: flags sit after the data, one 128-byte line each, READY and ACK disjoint
    char* base = reinterpret_cast<char*>(0x10000000);
    EXPECT(reinterpret_cast<char*>(p2p_flag(base, P2P_READY, 0)) == base + kP2PDataBytes);
    EXPECT(p2p_flag(base, P2P_READY, 1) - p2p_flag(base, P2P_READY, 0) == 2 * kP2PFlagStride);
    EXPECT(reinterpret_cast<char*>(p2p_flag(base, P2P_ACK, kMaxRanks - 1) + kP2PFlagStride + 1) <= base + kP2PWindowBytes);
    EXPECT(p2p_flag(base, P2P_ACK, 0) == p2p_flag(base, P2P_READY, kMaxRanks - 1) + 2 * kP2PFlagStride);
    b200mpi_comm* nc = new b200mpi_comm;     // no mailbox window: the API refuses instead of touching memory
    EXPECT(b200mpi_comm_has_p2p(nc) == 0 && b200mpi_p2p_batch(nc, ops, 1, nullptr) == B200MPI_ERR_UNSUPPORTED);
  }

  // ---- pipelined launches (k_pipe): every (world, op, mode, size) plan fits the staging region, the grid fits the GPU with
  //      one CTA per SM, chunks are whole multiples of the world (the reduce phase splits a chunk into per-rank slices),
  //      a broadcast with NVLS takes every lane, and the defaults of a real communicator (160 MiB staging) hold 44 x 3 x 1 MiB
  {
    b200mpi_comm* pc = new b200mpi_comm;
    pc->twoshot_bytes = (size_t)144 << 20;      // 160 MiB staging minus the 16 MiB one-shot region (comm_finish_init)
    size_t checked = 0;
    for (int world : {2, 3, 4, 8}) {
      pc->world = world;
      for (int kind : {PIPE_ALLREDUCE, PIPE_ALLGATHER, PIPE_REDUCE_SCATTER, PIPE_BROADCAST}) {
        const bool wide = kind == PIPE_ALLGATHER || kind == PIPE_REDUCE_SCATTER;
        for (int mode : {MODE_P2P, MODE_NVLS}) {
          for (size_t bytes = 1; bytes <= ((size_t)4 << 30); bytes = bytes * 3 + 5) {
            const PipePlan p = pipe_plan(pc, kind, mode, bytes, wide);
            EXPECT(p.fits);
            EXPECT(p.lanes >= 1 && p.lanes <= kPipeLanes && 3 * p.lanes <= 132);          // co-resident: one CTA per SM
            EXPECT(p.depth >= 2 && p.chunk_vecs >= (size_t)world && p.chunk_vecs % world == 0);
            EXPECT(p.chunk_vecs * p.regions * 16 <= pc->pipe_chunk + 16 * (size_t)world * p.regions);   // a slot is ~ pipe_chunk at most
            EXPECT((size_t)p.lanes * p.depth * p.chunk_vecs * p.regions * 16 <= pc->twoshot_bytes);
            if (kind == PIPE_BROADCAST && mode == MODE_NVLS) EXPECT(p.lanes == kPipeLanes);
            checked++;
          }
        }
      }
    }
    EXPECT(checked > 500);
    pc->world = 8;
    const PipePlan big = pipe_plan(pc, PIPE_BROADCAST, MODE_NVLS, (size_t)1 << 30, false);
    EXPECT(big.lanes == 44 && big.depth == 3 && big.chunk_vecs == ((size_t)1 << 20) / 16);   // 44 x 3 x 1 MiB fit the region
    pc->twoshot_bytes = (size_t)8 << 20;        // a small user-chosen staging region shrinks the chunks instead of failing
    const PipePlan small = pipe_plan(pc, PIPE_ALLREDUCE, MODE_NVLS, (size_t)1 << 30, false);
    EXPECT(small.fits && small.chunk_vecs * 16 * small.lanes * small.depth <= pc->twoshot_bytes);
    pc->local = true;                           // emulated communicators: the whole grid must fit one GPU next to `world` copies
    pc->twoshot_bytes = (size_t)48 << 20;
    const PipePlan emu = pipe_plan(pc, PIPE_BROADCAST, MODE_P2P, (size_t)1 << 24, false);
    EXPECT(emu.fits && 3 * emu.lanes * pc->world <= 132);
  }

  printf(g_failed ? "comm_host_test: %d check(s) FAILED\n" : "comm_host_test: all checks passed\n", g_failed);
  return g_failed ? 1 : 0;
}
