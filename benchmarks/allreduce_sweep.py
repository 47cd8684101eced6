"""Allreduce bandwidth sweep (BASELINE.json config #5): algbw / busbw vs message
size for every b200mpi algorithm and for stock NCCL (torch.distributed), device
timed with CUDA events, max over ranks.  Run one process per GPU, e.g.
  python tests/mp_launch.py -n 8 benchmarks/allreduce_sweep.py --out profiles/allreduce_sweep_n8.json
busbw = algbw * 2(N-1)/N, reported against the H100 NVLink data-sheet rate
(mpi_operator_b200.utils.roofline.LINK_GBS, 450 GB/s per direction)."""
import argparse
import json
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mpi_operator_b200.launch.env import rank_info_from_env  # noqa: E402
from mpi_operator_b200.runtime.comm import Communicator  # noqa: E402
from mpi_operator_b200.utils.roofline import LINK_GBS  # noqa: E402


def time_op(fn, iters, warmup, comm, flush=None, inner=1):
    """Median/best device time of one call. `inner` back-to-back calls are captured
    in a CUDA graph and replayed, so the number is device time, not Python/launch
    overhead (all b200mpi kernels keep their epochs on the device and are capturable)."""
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        for _ in range(warmup):
            fn()
    torch.cuda.current_stream().wait_stream(side)
    torch.cuda.synchronize()
    comm.host_barrier()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, capture_error_mode="thread_local"):
        for _ in range(inner):
            fn()
    torch.cuda.synchronize()
    comm.host_barrier()
    g.replay()
    torch.cuda.synchronize()
    comm.host_barrier()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    for a, b in ev:
        if flush is not None:
            flush.add_(1.0)  # rewrite a >L2 buffer between timed iterations
        a.record()
        g.replay()
        b.record()
    torch.cuda.synchronize()
    ts = sorted(a.elapsed_time(b) / inner for a, b in ev)
    return ts[len(ts) // 2], ts[0]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--min", type=int, default=1024)
    ap.add_argument("--max", type=int, default=1 << 30)
    ap.add_argument("--dtype", default="float32,bfloat16")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out", default="")
    ap.add_argument("--no-nccl", action="store_true")
    ap.add_argument("--flush-l2", action="store_true")
    ap.add_argument("--tune-blocks", default="", help="comma list of CTA counts to try for twoshot/nvls at sizes >= 16 MiB")
    a = ap.parse_args()
    info = rank_info_from_env()
    dev = info.local_rank % torch.cuda.device_count()
    torch.cuda.set_device(dev)
    comm = Communicator.create(info.rank, info.world_size, dev, info.job_id)
    W, R = comm.world, comm.rank
    use_nccl = not a.no_nccl and W > 1
    if use_nccl:
        dist.init_process_group("nccl", rank=R, world_size=W, device_id=torch.device("cuda", dev))
    flush = torch.zeros(160 << 20, device="cuda", dtype=torch.float32) if a.flush_l2 else None
    win = comm.alloc_window(a.max)
    rows = []
    default_blocks = comm.get_tuning()["max_blocks"]
    factor = 2.0 * (W - 1) / W if W > 1 else 1.0
    for dname in a.dtype.split(","):
        dtype = getattr(torch, dname)
        esz = torch.empty((), dtype=dtype).element_size()
        size = a.min
        while size <= a.max:
            n = size // esz
            v = win.tensor(dtype, numel=n)
            v.fill_(1.0)
            t = torch.ones(n, device="cuda", dtype=dtype)
            algos = {}
            if size <= (1 << 20):
                algos["oneshot"] = lambda: comm.allreduce(t, t, op="avg", algo="oneshot")
            if size >= 16 * W:
                algos["twoshot"] = lambda: comm.allreduce_window(win, 0, n, dtype, op="avg", algo="twoshot")
                if comm.has_multicast:
                    algos["nvls"] = lambda: comm.allreduce_window(win, 0, n, dtype, op="avg", algo="nvls")
                def user(pipe, reg):
                    def run():  # user pointers: chunked staged kernel / pipelined kernel / cudaIpc-registered zero-copy two-shot
                        comm.set_pipe(min_bytes=0 if pipe else (1 << 62))
                        comm.set_reg(2 if reg else 0, 0)
                        comm.allreduce(t, t, op="avg", algo="auto" if size > (1 << 20) else "twoshot")
                    return run
                algos["staged"] = user(False, False)
                if size >= (256 << 10):
                    algos["pipe"] = user(True, False)
                    algos["reg"] = user(False, True)
            if use_nccl:
                algos["nccl"] = lambda: dist.all_reduce(t, op=dist.ReduceOp.AVG)
            if a.tune_blocks and size >= (16 << 20):
                for nb in [int(x) for x in a.tune_blocks.split(",")]:
                    def mk(algo, nb=nb):
                        def run():
                            comm.set_tuning(max_blocks=nb)
                            comm.allreduce_window(win, 0, n, dtype, op="avg", algo=algo)
                        return run
                    algos[f"twoshot@{nb}"] = mk("twoshot")
                    if comm.has_multicast:
                        algos[f"nvls@{nb}"] = mk("nvls")
            comm.set_tuning(max_blocks=default_blocks)
            iters = a.iters if size <= (64 << 20) else max(5, a.iters // 4)
            for name, fn in algos.items():
                inner = 20 if size <= (1 << 20) else (4 if size <= (32 << 20) else 1)
                med, best = time_op(fn, iters, a.warmup, comm, flush, inner)
                tt = torch.tensor([med, best], device="cuda", dtype=torch.float64)
                got = comm.host_allgather(tt.cpu().numpy().tobytes())
                import numpy as np
                arr = np.frombuffer(b"".join(got), dtype=np.float64).reshape(W, 2)
                med_max, best_max = float(arr[:, 0].max()), float(arr[:, 1].max())
                algbw = size / (med_max * 1e-3) / 1e9
                rows.append({"dtype": dname, "bytes": size, "algo": name, "ms_median_max_over_ranks": med_max,
                             "ms_best_max_over_ranks": best_max, "algbw_gbs": algbw, "busbw_gbs": algbw * factor,
                             "busbw_frac_of_link": algbw * factor / LINK_GBS})
                if R == 0:
                    print(f"{dname:9s} {size:>11d} B {name:15s} {med_max * 1e3:10.1f} us  algbw {algbw:8.2f} GB/s  busbw {algbw * factor:8.2f} GB/s", flush=True)
            size *= 4 if size < (1 << 20) else 2
    if R == 0 and a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump({"world": W, "multicast": comm.has_multicast, "tuning": comm.get_tuning(), "rows": rows}, f, indent=1)
    comm.host_barrier()
    if use_nccl:
        dist.destroy_process_group()
    comm.destroy()


if __name__ == "__main__":
    main()
