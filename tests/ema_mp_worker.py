"""Multi-process (one rank per GPU) weight-average worker, launched by tests/test_ema_gpu.py::test_ema_trainer_on_real_peers.

Every rank trains the same small BN CNN with ``ema_decay`` on its own part of the batch, on real peers: SGD and LARS, with the
two-shot and the NVLS (multicast) fused kernels. After each fused launch it applies the exact oracle of tests/ema_oracle.py to
the parameters that launch pushed into its parameter window. Then it checks four things:
- ``ema_weights()`` (one allgather per bucket) holds exactly that average;
- it is bit-identical on every rank;
- ``state_dict()["ema"]`` holds the same values;
- a second trainer that loads the checkpoint reproduces them.
A CUDA-graph run checks that k counts the capture warm-up and that the averages agree across ranks. Exits non-zero on any
mismatch."""
import os
import sys

import torch
import torch.nn as nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from ema_oracle import ema_step  # noqa: E402
from mpi_operator_b200.launch.env import rank_info_from_env  # noqa: E402
from mpi_operator_b200.parallel.data_parallel import DataParallelTrainer  # noqa: E402
from mpi_operator_b200.runtime.comm import Communicator  # noqa: E402

D = 0.99


def small_model():
    torch.manual_seed(0)
    return nn.Sequential(nn.Conv2d(3, 8, 3, padding=1, bias=False), nn.BatchNorm2d(8), nn.ReLU(),
                         nn.Conv2d(8, 16, 3, padding=1), nn.ReLU(), nn.AdaptiveAvgPool2d(1), nn.Flatten(),
                         nn.Linear(16, 10))


def data(rank, n):
    g = torch.Generator().manual_seed(100 + rank)
    return [(torch.randn(4, 3, 16, 16, generator=g).pin_memory(), torch.randint(0, 10, (4,), generator=g).pin_memory())
            for _ in range(n)]


def make(comm, lars, algo, graph):
    model = small_model()
    pg = [{"params": [p for p in model.parameters() if p.dim() == 1], "weight_decay": 0.0, "lars": False}] if lars else None
    return DataParallelTrainer(model, nn.CrossEntropyLoss(), comm, lr=0.05, momentum=0.9, weight_decay=1e-4,
                               autocast_dtype=None, cuda_graph=graph, bucket_bytes=4096, algo=algo, ema_decay=D, lars=lars,
                               param_groups=pg)


def follow(tr):
    """Wrap the fused calls: after each launch, fold the parameters it pushed into a host copy of the average."""
    comm, st = tr.comm, tr.state
    log = {"e": st.flat_param.cpu().numpy().copy(), "launches": 0}

    def wrap(orig):
        def call(grad_win, grad_off, param_win, param_off, momentum, count, *a, **kw):
            orig(grad_win, grad_off, param_win, param_off, momentum, count, *a, **kw)
            torch.cuda.synchronize()
            sl = slice(param_off // 4, param_off // 4 + count)
            log["e"][sl] = ema_step(log["e"][sl], st.flat_param[sl].cpu().numpy(), D, int(kw["ema_sched"][1]))
            log["launches"] += 1
        return call
    comm.allreduce_sgd_window = wrap(Communicator.allreduce_sgd_window.__get__(comm))
    comm.allreduce_lars_window = wrap(Communicator.allreduce_lars_window.__get__(comm))
    return log


def unfollow(comm):
    del comm.allreduce_sgd_window, comm.allreduce_lars_window


def all_ranks(comm, t):
    out = torch.empty(comm.world * t.numel(), dtype=t.dtype, device=t.device)
    comm.allgather(t.contiguous(), out)
    torch.cuda.synchronize()
    return out.view(comm.world, -1)


def main():
    info = rank_info_from_env()
    dev = info.local_rank % torch.cuda.device_count()
    torch.cuda.set_device(dev)
    comm = Communicator.create(info.rank, info.world_size, dev, info.job_id)
    comm.set_tuning(timeout_ms=10000)
    W, R = comm.world, comm.rank
    fails = []

    def check(ok, what):
        if not ok:
            fails.append(what)
            print(f"[rank {R}] MISMATCH {what}", flush=True)

    batches = data(R, 4)
    for lars in (False, True):
        for algo in ("twoshot", "nvls"):
            what = f"world {W} lars={lars} algo={algo}"
            tr = make(comm, lars, algo, graph=False)
            log = follow(tr)
            for x, y in batches:
                tr.step(x, y)
            torch.cuda.synchronize()
            comm.check_error()
            check(tr.ema_updates == len(batches), f"{what}: k = {tr.ema_updates}")
            check(log["launches"] >= len(tr.state.buckets) * len(batches), f"{what}: {log['launches']} launches")
            with tr.ema_weights():
                inside = tr.state.flat_param.clone()
            want = torch.from_numpy(log["e"]).cuda()
            check(torch.equal(inside.view(torch.int32), want.view(torch.int32)), f"{what}: ema_weights() vs oracle")
            rows = all_ranks(comm, inside.view(torch.int32))
            check(bool((rows == rows[0]).all()), f"{what}: ema_weights() differs between ranks")
            sd = tr.state_dict()
            names = {p: n for n, p in tr.model.named_parameters()}
            for p in tr.state.params:
                s = tr.state.param_slot[p][1]
                ref = want[s:s + p.numel()].as_strided(p.size(), p.stride()).cpu().contiguous()
                check(torch.equal(sd["ema"][names[p]].view(torch.int32), ref.view(torch.int32)),
                      f"{what}: state_dict ema {names[p]}")
            tr2 = make(comm, lars, algo, graph=False)
            tr2.load_state_dict(sd)
            sd2 = tr2.state_dict()
            check(sd2["ema_updates"] == sd["ema_updates"], f"{what}: reloaded k")
            for n, v in sd["ema"].items():
                check(torch.equal(sd2["ema"][n], v), f"{what}: reloaded ema {n}")
            unfollow(comm)
            del tr, tr2
    # CUDA graph: k counts the three warm-up steps of the capture; the average is the same on every rank
    tr = make(comm, False, None, graph=True)
    for x, y in batches:
        tr.step(x, y)
    torch.cuda.synchronize()
    comm.check_error()
    check(tr.ema_updates == len(batches) + 3, f"world {W} graph: k = {tr.ema_updates}")
    with tr.ema_weights():
        rows = all_ranks(comm, tr.state.flat_param.clone().view(torch.int32))
    check(bool((rows == rows[0]).all()), f"world {W} graph: ema_weights() differs between ranks")
    comm.host_barrier()
    print(f"[rank {R}] ema_mp_worker done, world {W}, multicast={getattr(comm, 'has_multicast', None)}, "
          f"failures={len(fails)}", flush=True)
    comm.destroy()
    sys.exit(1 if fails else 0)


if __name__ == "__main__":
    main()
