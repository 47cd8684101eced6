// Host model of the wgmma GEMM + BN-statistics kernel (csrc/kernels/gemm_bnstats.cu).
//
// The kernel's roles (one TMA producer, two consumer warpgroups) run here as threads of one "CTA", with the hardware
// pieces replaced by small host emulations — mbarriers (arrival count + transaction bytes + phase parity), TMA loads and
// stores (tile copies in the 128-byte-swizzled shared-memory layout, zero fill / clipping at the matrix edge), and
// wgmma.mma_async (fp32 accumulation of K=16 slices into the warpgroup's 64-row register fragment; complete on issue).
// Everything that is arithmetic rather than hardware — ring/phase bookkeeping, the persistent tile walk, the swizzled
// staging layout, column ownership, the partial-row addressing — is the SAME code as in the kernel
// (csrc/kernels/gemm_bnstats_logic.h); the role loops are transcribed statement by statement from the kernel.
// A grid of such CTAs runs over a problem and the result is compared with a plain triple loop: Y, and the per-column
// sum / sum of squares merged over the partial rows. A protocol error shows up as a deadlock (watchdog) or wrong data.
//
// What this cannot tell: whether the PTX wrappers mean what the model assumes (descriptor bits are cross-checked with
// CuTe in gmma_desc_test.cu). `make test_gemm_model`; run by tests/test_native_cpu.py.
#include <atomic>
#include <chrono>
#include <cmath>
#include <condition_variable>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <thread>
#include <vector>

#include "../kernels/gemm_bnstats_logic.h"

using namespace b200mpi::gemm;

static std::atomic<int> g_deadlocks{0};

// ------------------------------------------------------------------ bf16 ----
static inline uint16_t f2bf(float f) {  // round to nearest even, like __floats2bfloat162_rn
  uint32_t u;
  memcpy(&u, &f, 4);
  u += 0x7fffu + ((u >> 16) & 1u);
  return (uint16_t)(u >> 16);
}
static inline float bf2f(uint16_t h) {
  uint32_t u = (uint32_t)h << 16;
  float f;
  memcpy(&f, &u, 4);
  return f;
}

// -------------------------------------------------------------- mbarrier ----
struct MBar {
  std::mutex mu;
  std::condition_variable cv;
  int init = 1, pending = 1;
  long long tx = 0;
  uint32_t phase = 0;
  void reset(int count) { init = pending = count; tx = 0; phase = 0; }
  void maybe_flip() {
    if (pending == 0 && tx == 0) { phase ^= 1u; pending = init; cv.notify_all(); }
  }
  void arrive() { std::lock_guard<std::mutex> l(mu); pending--; maybe_flip(); }
  void arrive_expect_tx(long long bytes) { std::lock_guard<std::mutex> l(mu); tx += bytes; pending--; maybe_flip(); }
  void complete_tx(long long bytes) { std::lock_guard<std::mutex> l(mu); tx -= bytes; maybe_flip(); }
  // mbarrier.try_wait.parity P: true once the phase with parity P has completed, i.e. the current phase differs from P
  void wait(uint32_t parity) {
    std::unique_lock<std::mutex> l(mu);
    if (!cv.wait_for(l, std::chrono::seconds(20), [&] { return phase != parity; })) g_deadlocks++;
  }
};

struct NamedBarrier {  // bar.sync id, n
  std::mutex mu;
  std::condition_variable cv;
  int n, waiting = 0;
  uint64_t gen = 0;
  explicit NamedBarrier(int n_) : n(n_) {}
  void sync() {
    std::unique_lock<std::mutex> l(mu);
    const uint64_t g = gen;
    if (++waiting == n) { waiting = 0; gen++; cv.notify_all(); return; }
    if (!cv.wait_for(l, std::chrono::seconds(20), [&] { return gen != g; })) g_deadlocks++;
  }
};

struct Problem {
  int M, N, K, BN;
  std::vector<uint16_t> X, W, Y;   // row-major bf16: X [M,K], W [N,K], Y [M,N]
  std::vector<float> partials;     // [parts][2N]
};

// ------------------------------------------------------------------- CTA ----
constexpr int kConsumerWarps = 8;                    // empty-barrier arrivals per stage: one per consumer warp

struct CTA {
  Problem& p;
  const int cta, grid, num_n;
  const int BN;
  std::vector<uint8_t> sA, sB, sOut;                 // kStages x tile, kStages x tile, BN/64 boxes
  std::vector<float> sums;                           // [BN][2]: warpgroup 1's column sums
  MBar full[kStages], empty[kStages];
  NamedBarrier cons{2};                              // bar.sync 1, 256: the two consumer warpgroups (one thread each)
  std::mutex store_mu;                               // the TMA store "bulk group": finished when it returns

  CTA(Problem& p_, int cta_, int grid_, int num_n_)
      : p(p_), cta(cta_), grid(grid_), num_n(num_n_), BN(p_.BN), sA((size_t)kStages * BM * 128), sB((size_t)kStages * p_.BN * 128),
        sOut((size_t)(p_.BN / 64) * kBoxBytes), sums((size_t)2 * p_.BN, 0.f) {
    for (int s = 0; s < kStages; s++) { full[s].reset(1); empty[s].reset(kConsumerWarps); }
  }

  // cp.async.bulk.tensor.2d load with SWIZZLE_128B: box of `rows` x 64 elements at (row0, k0), zero fill outside the matrix
  void tma_load(uint8_t* dst, const std::vector<uint16_t>& src, int nrows_total, int row0, int k0, int rows, MBar& bar) {
    for (int r = 0; r < rows; r++)
      for (int k = 0; k < BK; k++) {
        uint16_t v = 0;
        if (row0 + r < nrows_total && k0 + k < p.K) v = src[(size_t)(row0 + r) * p.K + k0 + k];
        memcpy(dst + operand_elem_byte(r, k), &v, 2);
      }
    bar.complete_tx((long long)rows * 128);
  }
  // cp.async.bulk.tensor.2d store of one [128 x 64] box, clipped at the matrix edge
  void tma_store(const uint8_t* box, int col0, int row0) {
    for (int r = 0; r < BM; r++)
      for (int j = 0; j < 64; j++) {
        if (row0 + r >= p.M || col0 + j >= p.N) continue;
        uint16_t v;
        memcpy(&v, box + operand_elem_byte(r, j), 2);   // a 64-column box has the operand-tile layout
        p.Y[(size_t)(row0 + r) * p.N + col0 + j] = v;
      }
  }
  // wgmma m64nBNk16: D[64 x BN] (+)= A[64 x 16] . B[BN x 16]^T, A = rows [64 wg, 64 wg + 64) of the swizzled stage
  void wgmma(float* d, const uint8_t* a, const uint8_t* b, int wg, int kslice, bool accumulate) {
    for (int m = 0; m < 64; m++)
      for (int n = 0; n < BN; n++) {
        float acc = accumulate ? d[(size_t)m * BN + n] : 0.f;
        for (int k = 0; k < MMA_K; k++) {
          uint16_t av, bv;
          memcpy(&av, a + operand_elem_byte(wg * 64 + m, kslice * MMA_K + k), 2);
          memcpy(&bv, b + operand_elem_byte(n, kslice * MMA_K + k), 2);
          acc += bf2f(av) * bf2f(bv);
        }
        d[(size_t)m * BN + n] = acc;
      }
  }
  void release(int s) { for (int w = 0; w < kConsumerWarps / 2; w++) empty[s].arrive(); }   // lane 0 of each warp

  void producer() {  // warp 8, lane 0
    const TileWalk walk(cta, grid, num_n, p.M);
    const int num_k = p.K / BK, n0 = walk.n_blk * BN;
    Ring st;
    for (int m_blk = walk.m_first; m_blk < walk.num_m; m_blk += walk.m_step)
      for (int kb = 0; kb < num_k; kb++) {
        empty[st.s].wait(st.ph ^ 1u);
        full[st.s].arrive_expect_tx((long long)BM * 128 + (long long)BN * 128);
        tma_load(sA.data() + (size_t)st.s * BM * 128, p.X, p.M, m_blk * BM, kb * BK, BM, full[st.s]);
        tma_load(sB.data() + (size_t)st.s * BN * 128, p.W, p.N, n0, kb * BK, BN, full[st.s]);
        st.advance(kStages);
      }
  }
  // one consumer warpgroup; its 128 threads are executed one after the other between barriers
  void consumer(int wg) {
    const TileWalk walk(cta, grid, num_n, p.M);
    const int num_k = p.K / BK, n0 = walk.n_blk * BN;
    std::vector<float> d((size_t)64 * BN);               // the warpgroup's accumulator fragments
    std::vector<float> s1(BN, 0.f), s2(BN, 0.f);         // registers of the column owners t < BN
    Ring st;
    for (int m_blk = walk.m_first; m_blk < walk.num_m; m_blk += walk.m_step) {
      int prev = 0;
      for (int kb = 0; kb < num_k; kb++) {
        full[st.s].wait(st.ph);
        for (int k = 0; k < BK / MMA_K; k++)
          wgmma(d.data(), sA.data() + (size_t)st.s * BM * 128, sB.data() + (size_t)st.s * BN * 128, wg, k, (kb | k) != 0);
        if (kb > 0) release(prev);                         // wgmma.wait_group 1: the previous k-block is done
        prev = st.s;
        st.advance(kStages);
      }
      release(prev);                                       // wgmma.wait_group 0
      // (ct == 0: cp.async.bulk.wait_group.read 0 — the modelled store is synchronous)
      cons.sync();
      for (int w = 0; w < 4; w++)
        for (int lane = 0; lane < 32; lane++) {
          const int frag_row = wg * 64 + w * 16 + (lane >> 2);
          for (int j = 0; j < BN / 8; j++) {
            const int col = 8 * j + 2 * (lane & 3);
            for (int i = 0; i < 2; i++) {
              const int row = frag_row + 8 * i;
              const uint16_t pair[2] = {f2bf(d[(size_t)(row - wg * 64) * BN + col]), f2bf(d[(size_t)(row - wg * 64) * BN + col + 1])};
              memcpy(sOut.data() + stage_elem_byte(col, row), pair, 4);
            }
          }
        }
      cons.sync();
      if (wg == 0) {                                       // ct == 0 lives in warpgroup 0
        std::lock_guard<std::mutex> l(store_mu);
        for (int b = 0; b < BN / 64; b++) tma_store(sOut.data() + (size_t)b * kBoxBytes, n0 + b * 64, m_blk * BM);
      }
      for (int t = 0; t < BN; t++)                         // col_owner
        for (int r = wg * 64; r < wg * 64 + 64; r++) {
          uint16_t h;
          memcpy(&h, sOut.data() + stage_elem_byte(t, r), 2);
          const float f = bf2f(h);
          s1[t] += f;
          s2[t] = std::fma(f, f, s2[t]);
        }
    }
    if (wg == 1)
      for (int t = 0; t < BN; t++) { sums[2 * t] = s1[t]; sums[2 * t + 1] = s2[t]; }
    cons.sync();
    if (wg == 0 && walk.m_first < walk.num_m)
      for (int t = 0; t < BN; t++) {
        p.partials[partial_index(walk.m_first, p.N, n0 + t)] = s1[t] + sums[2 * t];
        p.partials[partial_index(walk.m_first, p.N, n0 + t) + 1] = s2[t] + sums[2 * t + 1];
      }
  }
  void run() {
    std::vector<std::thread> th;
    th.emplace_back([&] { producer(); });
    for (int wg = 0; wg < 2; wg++) th.emplace_back([&, wg] { consumer(wg); });
    for (auto& t : th) t.join();
  }
};

static int run_case(int M, int N, int K, int sms) {
  Problem p;
  p.M = M; p.N = N; p.K = K; p.BN = N % 128 == 0 ? 128 : 64;
  p.X.resize((size_t)M * K); p.W.resize((size_t)N * K); p.Y.assign((size_t)M * N, 0xffff);
  uint32_t x = 12345u + (uint32_t)M * 7u + (uint32_t)N * 13u + (uint32_t)K;
  auto rnd = [&] { x = x * 1664525u + 1013904223u; return ((int)(x >> 20) % 2001 - 1000) / 1000.0f; };
  for (auto& v : p.X) v = f2bf(rnd());
  for (auto& v : p.W) v = f2bf(rnd() * 0.25f);
  // launch geometry exactly as launch<BN>() in gemm_bnstats.cu
  const int num_n = N / p.BN, num_m = (M + BM - 1) / BM;
  int groups = sms / num_n;
  if (groups < 1) return 1;
  if (groups > num_m) groups = num_m;
  p.partials.assign((size_t)groups * 2 * N, 0.f);
  const int grid = groups * num_n;
  {
    std::vector<std::thread> ctas;
    std::vector<CTA*> objs;
    for (int c = 0; c < grid; c++) objs.push_back(new CTA(p, c, grid, num_n));
    for (int c = 0; c < grid; c++) ctas.emplace_back([&, c] { objs[c]->run(); });
    for (auto& t : ctas) t.join();
    for (auto* o : objs) delete o;
  }
  // reference
  int bad = 0;
  std::vector<double> rs1(N, 0.0), rs2(N, 0.0);
  for (int m = 0; m < M; m++)
    for (int n = 0; n < N; n++) {
      float acc = 0.f;
      for (int k = 0; k < K; k++) acc += bf2f(p.X[(size_t)m * K + k]) * bf2f(p.W[(size_t)n * K + k]);
      const uint16_t want = f2bf(acc);
      const uint16_t got = p.Y[(size_t)m * N + n];
      if (std::fabs(bf2f(want) - bf2f(got)) > 1e-2f * std::fabs(bf2f(want)) + 1e-3f) bad++;   // summation order differs
      rs1[n] += bf2f(got);
      rs2[n] += (double)bf2f(got) * bf2f(got);
    }
  for (int n = 0; n < N; n++) {
    double s1 = 0, s2 = 0;
    for (int g = 0; g < groups; g++) { s1 += p.partials[(size_t)g * 2 * N + 2 * n]; s2 += p.partials[(size_t)g * 2 * N + 2 * n + 1]; }
    if (std::fabs(s1 - rs1[n]) > 1e-3 * (std::fabs(rs1[n]) + 1.0) || std::fabs(s2 - rs2[n]) > 1e-3 * (rs2[n] + 1.0)) bad++;
  }
  printf("M=%-5d N=%-4d K=%-4d BN=%-3d grid=%-3d groups=%-3d : %s\n", M, N, K, p.BN, grid, groups, bad ? "MISMATCH" : "ok");
  return bad;
}

int main() {
  int bad = 0;
  // (M, N, K, SMs): single tile, ragged M, several k-blocks (ring wraps), several tiles per CTA (accumulator ring wraps),
  // both BN variants, more column blocks than one, fewer tiles than SMs
  bad += run_case(128, 64, 64, 4);
  bad += run_case(100, 64, 128, 4);
  bad += run_case(1000, 128, 320, 3);      // 8 row blocks over 3 CTAs, 5 k-blocks: stage ring wraps mid-tile
  bad += run_case(2048, 256, 64, 4);       // 2 column blocks x 2 groups, 8 tiles per CTA, one k-block per tile
  bad += run_case(700, 192, 192, 6);       // BN = 64, 3 column blocks
  bad += run_case(384, 128, 576, 16);      // 9 k-blocks per tile, more SMs than tiles
  bad += g_deadlocks.load();
  printf(bad ? "gemm_pipeline_model: FAILED (%d)\n" : "gemm_pipeline_model: all cases match the reference GEMM and column sums\n", bad);
  return bad ? 1 : 0;
}
