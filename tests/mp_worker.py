"""Multi-process (one rank per GPU) correctness worker for the b200mpi runtime.
Launched by tests/test_multigpu.py or directly:
  python tests/mp_launch.py -n 2 tests/mp_worker.py
Exits non-zero on any mismatch."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from collective_oracle import assert_bits, exact_inputs, expected  # noqa: E402
from mpi_operator_b200.launch.env import rank_info_from_env  # noqa: E402
from mpi_operator_b200.runtime.comm import Communicator  # noqa: E402


def main():
    info = rank_info_from_env()
    ndev = torch.cuda.device_count()
    dev = info.local_rank % ndev
    torch.cuda.set_device(dev)
    comm = Communicator.create(info.rank, info.world_size, dev, info.job_id)
    comm.set_tuning(timeout_ms=10000)
    W, R = comm.world, comm.rank
    if R == 0:
        print(f"[mp_worker] world={W} multicast={comm.has_multicast} tuning={comm.get_tuning()}", flush=True)
    fails = 0

    def gen(seed, n, dtype, r):
        g = torch.Generator(device="cuda").manual_seed(seed * 131 + r)
        return torch.randn(n, device="cuda", generator=g).to(dtype)

    # Exact-sum inputs (tests/collective_oracle.py): every rank generates every rank's values, and each result has exactly
    # one correct value. NVLS bf16 / f16 averages round twice (the switch returns the sum rounded to T, the kernel scales
    # and rounds again): at power-of-two worlds that equals the P2P result, at other worlds it may differ by one ulp of T,
    # so the oracle follows the algorithm that ran, read from the communicator's counters.
    def exact(seed, n, dtype):
        return exact_inputs(W, n, dtype, seed=seed, device="cuda")

    def calls():
        return {(o["op"], o["algo"]): o["calls"] for o in comm.stats(native_only=True)["ops"]}

    def nvls_ran(before):
        return any(algo == "nvls" and v > before.get((op, algo), 0) for (op, algo), v in calls().items())

    def same_bits(name, got, want):
        try:
            assert_bits(got, want, name)
        except AssertionError as e:
            print(f"[rank {R}] {e}", flush=True)
            return False
        return True

    algos = ["oneshot", "twoshot"] + (["nvls"] if comm.has_multicast else [])
    for dtype in (torch.float32, torch.bfloat16, torch.float16):
        for n in (1, 1000, 65536 + 8, 3 * 1024 * 1024 + 40):
            xs = exact(n, n, dtype)
            for algo in algos:
                if algo == "oneshot" and n * xs[0].element_size() > (1 << 20):
                    continue
                out = torch.empty_like(xs[R])
                before = calls()
                comm.allreduce(xs[R].clone(), out, op="avg", algo=algo)
                torch.cuda.synchronize()
                comm.check_error()
                fails += int(not same_bits(f"allreduce {dtype} n={n} {algo}", out, expected(xs, "avg", nvls=nvls_ran(before))))
    # symmetric window, in place, all algos
    n = 8 * 1024 * 1024
    win = comm.alloc_window(n * 4)
    for dtype in (torch.float32, torch.bfloat16):
        cnt = n if dtype == torch.float32 else 2 * n
        v = win.tensor(dtype, numel=cnt)
        for algo in algos[1:]:
            xs = exact(7, cnt, dtype)
            v.copy_(xs[R])
            torch.cuda.synchronize()
            comm.allreduce_window(win, 0, cnt, dtype, op="sum", algo=algo)
            torch.cuda.synchronize()
            comm.check_error()
            fails += int(not same_bits(f"allreduce_window {dtype} {algo}", v, expected(xs, "sum")))
    # fused SGD (both modes)
    cnt = 4 * 1024 * 1024
    gwin, pwin = comm.alloc_window(cnt * 4), comm.alloc_window(cnt * 4)
    p0 = gen(11, cnt, torch.float32, 0)
    pv, gv = pwin.tensor(torch.float32, numel=cnt), gwin.tensor(torch.float32, numel=cnt)
    for algo in algos[1:]:
        pv.copy_(p0)
        mom = torch.zeros(comm.slice_elems(cnt, torch.float32), device="cuda")
        ref = p0.clone()
        buf = None
        for step in range(2):
            gs = [gen(20 + step, cnt, torch.float32, r) for r in range(W)]
            gv.copy_(gs[R])
            torch.cuda.synchronize()
            comm.host_barrier()
            comm.allreduce_sgd_window(gwin, 0, pwin, 0, mom, cnt, torch.float32, lr=0.05, momentum_coef=0.9,
                                      weight_decay=1e-4, first_step=(step == 0), algo=algo)
            torch.cuda.synchronize()
            comm.check_error()
            g = torch.stack(gs).mean(0) + 1e-4 * ref
            buf = g.clone() if buf is None else 0.9 * buf + g
            ref = ref - 0.05 * buf
            err = (pv - ref).abs().max().item()
            if not err <= 1e-5:
                print(f"[rank {R}] fused sgd {algo} step {step}: max err {err}", flush=True)
                fails += 1
    # broadcast / allgather / reduce_scatter / alltoall / barrier
    x = gen(3, 100003, torch.float32, R)
    want = gen(3, 100003, torch.float32, W - 1)
    comm.broadcast(x, root=W - 1)
    torch.cuda.synchronize()
    fails += int(not torch.equal(x, want))
    x = gen(4, 50001 * 2, torch.bfloat16, R)
    out = torch.empty(W * x.numel(), device="cuda", dtype=torch.bfloat16)
    comm.allgather(x, out)
    torch.cuda.synchronize()
    fails += int(not torch.equal(out, torch.cat([gen(4, 50001 * 2, torch.bfloat16, r) for r in range(W)])))
    xs = [gen(5, W * 4096, torch.float32, r) for r in range(W)]
    out = torch.empty(4096, device="cuda")
    comm.reduce_scatter(xs[R], out)
    torch.cuda.synchronize()
    fails += int(not torch.allclose(out, torch.stack(xs).sum(0)[R * 4096:(R + 1) * 4096], atol=1e-4))
    out = torch.empty(W * 4096, device="cuda")
    comm.alltoall(xs[R], out)
    torch.cuda.synchronize()
    fails += int(not torch.equal(out, torch.cat([xs[s][R * 4096:(R + 1) * 4096] for s in range(W)])))
    comm.barrier()
    torch.cuda.synchronize()
    comm.check_error()

    # ---- user-pointer paths on REAL peers: pipelined kernels (NVLS where bound), cudaIpc-registered zero-copy kernels ----
    def check(name, ok):
        nonlocal fails
        if not ok:
            print(f"[rank {R}] {name} FAILED", flush=True)
            fails += 1

    for label, pipe_min, reg_mode in (("pipe", 0, 0), ("reg", 1 << 62, 2), ("auto", 8 << 20, 1)):
        comm.set_pipe(min_bytes=pipe_min, chunk_bytes=256 << 10)
        comm.set_reg(reg_mode, 0 if reg_mode == 2 else (8 << 20))
        for it, n in enumerate((1 << 20, 3 * (1 << 20) + 8, 12 * (1 << 20))):
            for dtype in (torch.float32, torch.bfloat16):
                xs = exact(40 + it, n, dtype)
                out = torch.empty_like(xs[R])
                b0 = calls()
                comm.allreduce(xs[R].clone(), out, op="avg")               # out of place
                torch.cuda.synchronize()
                want_out = expected(xs, "avg", nvls=nvls_ran(b0))
                inp = xs[R].clone()
                b0 = calls()
                comm.allreduce(inp, inp, op="avg")                         # in place
                torch.cuda.synchronize()
                want_inp = expected(xs, "avg", nvls=nvls_ran(b0))
                comm.check_error()
                check(f"{label} allreduce {dtype} n={n}", same_bits(f"{label} allreduce {dtype} n={n}", out, want_out)
                      and same_bits(f"{label} allreduce in place {dtype} n={n}", inp, want_inp))
                del xs
            x = gen(50 + it, n, torch.float32, R)
            ag = torch.empty(W * n, device="cuda")
            comm.allgather(x, ag)
            rs_in = exact(60 + it, W * n, torch.float32)
            full = rs_in[R].clone()
            rs = torch.empty(n, device="cuda")
            comm.reduce_scatter(full, rs)
            b = gen(70 + it, n, torch.float32, R)
            comm.broadcast(b, root=it % W)
            torch.cuda.synchronize()
            comm.check_error()
            check(f"{label} allgather n={n}", torch.equal(ag, torch.cat([gen(50 + it, n, torch.float32, r) for r in range(W)])))
            check(f"{label} reduce_scatter n={n}", same_bits(f"{label} reduce_scatter n={n}", rs, expected(rs_in, "sum")[R * n:(R + 1) * n]))
            del rs_in
            check(f"{label} broadcast n={n}", torch.equal(b, gen(70 + it, n, torch.float32, it % W)))
    if R == 0:
        print(f"[mp_worker] stats={[(o['op'], o['algo'], o['calls']) for o in comm.stats(native_only=True)['ops']]} reg={comm.reg_stats()}", flush=True)
    comm.set_pipe(min_bytes=8 << 20, chunk_bytes=1 << 20)
    comm.set_reg(1, 8 << 20)

    # ---- Adasum (K6) on device tensors: orthogonal gradients add, parallel gradients average ----
    from mpi_operator_b200.hvd.adasum import adasum_allreduce_
    e = torch.zeros(W * 1000, device="cuda")
    e[R * 1000:(R + 1) * 1000] = 1.0
    adasum_allreduce_(comm, e)
    p_ = torch.full((4096,), 2.0, device="cuda")
    adasum_allreduce_(comm, p_)
    torch.cuda.synchronize()
    check("adasum orthogonal", torch.allclose(e, torch.ones_like(e)))
    check("adasum parallel", torch.allclose(p_, torch.full_like(p_, 2.0)))
    # the one-kernel form on real peers, bit for bit: tests/adasum_mp_worker.py (test_zzz_adasum_gpu.py::test_adasum_on_real_peers)

    # ---- zero-copy window forms on real peers ----
    per = 1 << 18
    w2 = comm.alloc_window(W * per * 4)
    v = w2.tensor(torch.float32, numel=W * per)
    v.fill_(-1.0)
    v[R * per:(R + 1) * per].copy_(gen(80, per, torch.float32, R))
    torch.cuda.synchronize()
    comm.allgather_window(w2, 0, per * 4)
    torch.cuda.synchronize()
    check("allgather_window", torch.equal(v, torch.cat([gen(80, per, torch.float32, r) for r in range(W)])))
    rs_in = exact(81, W * per, torch.bfloat16)
    v.view(torch.bfloat16)[:W * per].copy_(rs_in[R])
    torch.cuda.synchronize()
    b0 = calls()
    comm.reduce_scatter_window(w2, 0, per, torch.bfloat16, op="avg")
    torch.cuda.synchronize()
    rs_want = expected(rs_in, "avg", nvls=nvls_ran(b0))[R * per:(R + 1) * per]
    check("reduce_scatter_window", same_bits("reduce_scatter_window", v.view(torch.bfloat16)[R * per:(R + 1) * per], rs_want))
    v.fill_(float(R))
    torch.cuda.synchronize()
    comm.broadcast_window(w2, 0, W * per * 4, root=W - 1)
    torch.cuda.synchronize()
    comm.check_error()
    check("broadcast_window", torch.equal(v, torch.full_like(v, float(W - 1))))

    # ---- stress (SURVEY.md section 5.2): STRESS_ITERS back-to-back allreduces of random sizes 4 B .. 8 MiB on integer-valued data
    # (fp32 sums are exact in any order, so every result must be bit-exact), random algorithm per call incl. NVLS, the
    # pipelined kernel and the fused allreduce+SGD kernel, check_error() every 100 calls ----
    iters = int(os.environ.get("B200MPI_STRESS_ITERS", "10000"))
    g = torch.Generator().manual_seed(1234)          # same sequence on every rank
    big = 2 * 1024 * 1024                              # elements (8 MiB fp32)
    base = [(gen(90, big, torch.float32, r) * 4).round() for r in range(W)]
    total = torch.stack(base).sum(0)
    swin = comm.alloc_window(big * 4)
    sv = swin.tensor(torch.float32, numel=big)
    pwin2 = comm.alloc_window(big * 4)
    spv = pwin2.tensor(torch.float32, numel=big)
    smom = torch.zeros(comm.slice_elems(big, torch.float32), device="cuda")
    kinds = ["oneshot", "twoshot", "auto", "pipe", "window"] + (["nvls"] if comm.has_multicast else []) + ["sgd"]
    bad = 0
    for i in range(iters):
        # log-uniform size, in elements; window / sgd kinds need 16-byte multiples
        n = int(2 ** (torch.rand((), generator=g).item() * 21)) if i % 50 else big
        n = max(1, min(big, n))
        kind = kinds[int(torch.randint(0, len(kinds), (), generator=g))]
        if kind == "oneshot" and n * 4 > (1 << 20):
            kind = "twoshot"
        if kind in ("window", "nvls", "sgd"):
            n = max(8, n // 8 * 8)
            sv[:n].copy_(base[R][:n])
            if kind == "sgd":     # p = 0 - lr * (scale * sum) with lr = scale = 1, no momentum: parameters = -sum, exact
                spv[:n].zero_()
                comm.allreduce_sgd_window(swin, 0, pwin2, 0, smom, n, torch.float32, lr=1.0, momentum_coef=0.0, first_step=True,
                                          scale=1.0)
                ok = torch.equal(spv[:n], -total[:n])
            else:
                comm.allreduce_window(swin, 0, n, torch.float32, op="sum", algo="nvls" if kind == "nvls" else "auto")
                ok = torch.equal(sv[:n], total[:n])
        else:
            x = base[R][:n].clone()
            if kind == "pipe":
                comm.set_pipe(min_bytes=0, chunk_bytes=64 << 10)
                comm.allreduce(x, x, algo="twoshot")
                comm.set_pipe(min_bytes=8 << 20, chunk_bytes=1 << 20)
            else:
                comm.allreduce(x, x, algo=kind)
            ok = torch.equal(x, total[:n])
        if not ok:
            bad += 1
            if bad <= 3:
                print(f"[rank {R}] stress iteration {i}: kind={kind} n={n} mismatch", flush=True)
        if i % 100 == 99:
            torch.cuda.synchronize()
            comm.check_error()
    torch.cuda.synchronize()
    comm.check_error()
    check(f"stress ({iters} iterations, {bad} mismatches)", bad == 0)
    comm.host_barrier()
    print(f"[rank {R}] mp_worker done, failures={fails}", flush=True)
    comm.destroy()
    sys.exit(1 if fails else 0)


if __name__ == "__main__":
    main()
