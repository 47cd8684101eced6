"""Multi-process (one rank per GPU) worker of tests/test_fused_optimizer_exact_gpu.py::test_nvls_steps_on_real_peers.

Runs the fused SGD (fp32 / bf16 / f16 gradients), grouped SGD and LARS steps with ``algo="nvls"`` (multimem.ld_reduce and
multimem.st) on real peers, three steps each, on exact-sum inputs (tests/collective_oracle.py), so that the switch's order
of adds does not matter. Each step is checked against tests/optimizer_oracle.py from the kernel's own previous state: the
parameters and bf16 shadow of every rank, this rank's momentum shard, and for LARS the trust ratios (inside the oracle's
interval, bitwise equal on every rank) and the update given them. Exits 3 without multicast, non-zero on any mismatch."""
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from collective_oracle import exact_inputs  # noqa: E402
from mpi_operator_b200.launch.env import rank_info_from_env  # noqa: E402
from mpi_operator_b200.runtime.comm import Communicator  # noqa: E402
from optimizer_oracle import (F32, expand_groups, lars_norm_interval, lars_step, owner_sum, sgd_step,  # noqa: E402
                              vec_elems)

NO_MULTICAST = 3
NAN = float("nan")


def bits_equal(got, want):
    """Bitwise equality; float32 NaNs match any NaN."""
    got, want = np.asarray(got), np.asarray(want)
    if got.dtype == np.float32:
        return bool(np.all((got.view(np.int32) == want.view(np.int32)) | (np.isnan(got) & np.isnan(want))))
    return bool(np.array_equal(got, want))


def main():
    info = rank_info_from_env()
    dev = info.local_rank % torch.cuda.device_count()
    torch.cuda.set_device(dev)
    comm = Communicator.create(info.rank, info.world_size, dev, info.job_id)
    comm.set_tuning(timeout_ms=10000)
    W, R = comm.world, comm.rank
    if not comm.has_multicast:
        print(f"[rank {R}] no multicast: NVLS steps not run", flush=True)
        comm.destroy()
        sys.exit(NO_MULTICAST)
    fails = []

    def check(ok, what):
        if not ok:
            fails.append(what)
            print(f"[rank {R}] MISMATCH {what}", flush=True)

    cases = [("sgd", torch.float32), ("sgd", torch.bfloat16), ("sgd", torch.float16), ("grouped", torch.float32),
             ("lars", torch.float32)]
    for ci, (kind, dtype) in enumerate(cases):
        N = vec_elems(dtype)
        n = 1013 * N
        esz = torch.empty((), dtype=dtype).element_size()
        gwin, pwin, lwin = comm.alloc_window(n * esz), comm.alloc_window(n * 4), comm.alloc_window(n * 2)
        gv, pv, lv = gwin.tensor(dtype, numel=n), pwin.tensor(torch.float32, numel=n), lwin.tensor(torch.bfloat16, numel=n)
        per = comm.slice_elems(n, dtype)
        live = max(0, min(per, n - R * per))
        mom = torch.full((per,), NAN, device="cuda")
        rng = np.random.default_rng(ci)                     # the same values on every rank
        pv.copy_(torch.from_numpy((rng.standard_normal(n) * 0.5).astype(F32)))
        gmap_np = (np.arange(n // 4) % 256).astype(np.uint8)
        gmap, ghyper = torch.from_numpy(gmap_np).cuda(), torch.zeros(256, 3, device="cuda")
        P = 3
        pmap_np = np.repeat(np.arange(P + 1), [1, 700, 300, n // 4 - 1001]).astype(np.int32)
        pmap = torch.from_numpy(pmap_np).to(torch.uint16).cuda()
        ptab_np = np.array([[0, 1], [1, 1], [0, 0]], dtype=np.uint8)
        ptab = torch.from_numpy(ptab_np).cuda()
        board = comm.alloc_window(P * W * 8 + 16)
        scratch = torch.zeros(comm.lars_scratch_bytes(n, P), dtype=torch.uint8, device="cuda")
        trust_t = torch.zeros(P, device="cuda")
        s = F32(1.0 / W)
        for step in range(3):
            what = f"world {W} {kind} {str(dtype)[6:]} step {step}"
            xs = exact_inputs(W, n, dtype, seed=1000 * ci + step)
            gs = [x.float().numpy() for x in xs]
            gv.copy_(xs[R])
            tab = np.stack([rng.uniform(0, 0.5, 256), rng.uniform(0, 0.99, 256), rng.uniform(0, 1e-2, 256)], 1).astype(F32)
            tab[::7, 0] = 0
            ghyper.copy_(torch.from_numpy(tab))
            p = pv.cpu().numpy()
            m = np.full(n, NAN, F32)
            m[R * per:R * per + live] = mom[:live].cpu().numpy()
            comm.host_barrier()
            first = step == 0
            common = dict(lowp_win=lwin, lowp_off=0, algo="nvls", first_step=first)
            if kind == "lars":
                comm.allreduce_lars_window(gwin, 0, pwin, 0, mom, n, torch.float32, group_hyper=ghyper, param_map=pmap,
                                           param_table=ptab, board_win=board, board_off=0, scratch=scratch,
                                           trust_coefficient=0.02, trust_out=trust_t, **common)
            elif kind == "grouped":
                comm.allreduce_sgd_window(gwin, 0, pwin, 0, mom, n, dtype, lr=9.0, group_map=gmap, group_hyper=ghyper,
                                          **common)
            else:
                comm.allreduce_sgd_window(gwin, 0, pwin, 0, mom, n, dtype, lr=0.1, momentum_coef=0.9, weight_decay=1e-4,
                                          **common)
            torch.cuda.synchronize()
            comm.check_error()
            S = owner_sum(gs, W, dtype, nvls=True)
            if kind == "lars":
                trust = trust_t.cpu().numpy()
                rows = torch.empty(W * P, device="cuda")
                comm.allgather(trust_t, rows)
                torch.cuda.synchronize()
                check(bits_equal(rows.view(W, P).cpu().numpy(), np.tile(trust, (W, 1))), f"{what}: trust differs between ranks")
                key = np.repeat(pmap_np, 4)
                gsc = (S * s).astype(F32)
                for q in range(P):
                    sel = key == q
                    lo, hi = (1.0, 1.0) if not ptab_np[q, 1] else \
                        lars_norm_interval(gsc[sel], p[sel], W, F32(0.02), tab[ptab_np[q, 0], 2])
                    check(lo <= float(trust[q]) <= hi, f"{what}: trust {q} = {trust[q]!r} not in [{lo!r}, {hi!r}]")
                grp = np.append(ptab_np[:, 0], 0)[key]
                t = np.append(trust, F32(1.0))[key]
                want = lars_step(p, m, S, s, t, tab[grp, 0], tab[grp, 1], tab[grp, 2], False, first)
            elif kind == "grouped":
                want = sgd_step(p, m, S, s, *expand_groups(tab, gmap_np, n), False, first)
            else:
                want = sgd_step(p, m, S, s, F32(0.1), F32(0.9), F32(1e-4), False, first)
            check(bits_equal(pv.cpu().numpy(), want[0]), f"{what}: parameters")
            check(bits_equal(lv.cpu().view(torch.int16).numpy(), want[2].view(np.int16)), f"{what}: bf16 shadow")
            check(bits_equal(mom[:live].cpu().numpy(), want[1][R * per:R * per + live]), f"{what}: momentum shard")
        comm.host_barrier()
        for w in (gwin, pwin, lwin, board):
            w.free()
    comm.host_barrier()
    print(f"[rank {R}] optimizer_mp_worker done, world {W}, failures={len(fails)}", flush=True)
    comm.destroy()
    sys.exit(1 if fails else 0)


if __name__ == "__main__":
    main()
