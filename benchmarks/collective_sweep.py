"""Collective sweep THROUGH torch.distributed on plain ``torch.empty`` tensors (BASELINE.json config #5).

The same script is run twice by the same launcher:

  python tests/mp_launch.py -n 8 benchmarks/collective_sweep.py --tag nccl --out gpurun_out/sweep_nccl_n8.json
  LD_PRELOAD=mpi_operator_b200/lib/libb200mpi_nccl.so \
  python tests/mp_launch.py -n 8 benchmarks/collective_sweep.py --tag shim --out gpurun_out/sweep_shim_n8.json

so the second run measures exactly what an unmodified training script gets when the node agent injects the runtime:
``ncclAllReduce`` & co. on unregistered user pointers resolving to b200mpi kernels. ``benchmarks/roofline_tables.py``
merges the two files into the vs-NCCL tables under profiles/.

Timing: CUDA events around CUDA-graph replays of ``inner`` back-to-back calls (device time, no Python in the number),
median over ``iters``, max over ranks. busbw: allreduce 2(N-1)/N, allgather / reduce_scatter (N-1)/N of the FULL
buffer, broadcast 1 (reference call sites: SURVEY.md section 2.5 K3-K5, K7)."""
import argparse
import json
import os
import sys

import torch
import torch.distributed as dist

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mpi_operator_b200.utils.roofline import LINK_GBS  # noqa: E402


def timed(fn, iters, warmup, inner):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    dist.barrier()
    g = None
    try:
        side = torch.cuda.Stream()
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=side, capture_error_mode="thread_local"):
                for _ in range(inner):
                    fn()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
    except Exception as e:  # pragma: no cover - capture refused: time eagerly
        if dist.get_rank() == 0:
            print(f"[sweep] graph capture failed ({type(e).__name__}: {e}); timing eager launches", file=sys.stderr)
        g = None
        torch.cuda.synchronize()
    run = g.replay if g is not None else (lambda: [fn() for _ in range(inner)])
    run()
    torch.cuda.synchronize()
    dist.barrier()
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(iters)]
    for a, b in ev:
        a.record()
        run()
        b.record()
    torch.cuda.synchronize()
    ts = sorted(a.elapsed_time(b) / inner for a, b in ev)
    return ts[len(ts) // 2], ts[0], g is not None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--tag", default="nccl")
    ap.add_argument("--ops", default="allreduce,allgather,reduce_scatter,broadcast")
    ap.add_argument("--dtype", default="float32,bfloat16")
    ap.add_argument("--min", type=int, default=1024)
    ap.add_argument("--max", type=int, default=1 << 30)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    dev = int(os.environ.get("LOCAL_RANK", rank)) % torch.cuda.device_count()
    torch.cuda.set_device(dev)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", dev))
    rows = []
    for dname in a.dtype.split(","):
        dtype = getattr(torch, dname)
        esz = torch.empty((), dtype=dtype).element_size()
        for op in a.ops.split(","):
            size = a.min
            while size <= a.max:
                # `size` = bytes of the FULL buffer (allgather output / reduce_scatter input / allreduce / broadcast payload)
                n = max(world, size // esz // world * world)
                full = torch.empty(n, device="cuda", dtype=dtype).fill_(1.0)
                part = torch.empty(n // world, device="cuda", dtype=dtype).fill_(1.0)
                if op == "allreduce":
                    fn, factor = (lambda: dist.all_reduce(full, op=dist.ReduceOp.AVG)), 2.0 * (world - 1) / world
                elif op == "allgather":
                    fn, factor = (lambda: dist.all_gather_into_tensor(full, part)), (world - 1) / world
                elif op == "reduce_scatter":
                    fn, factor = (lambda: dist.reduce_scatter_tensor(part, full)), (world - 1) / world
                else:
                    fn, factor = (lambda: dist.broadcast(full, src=0)), 1.0
                inner = 20 if size <= (1 << 20) else (4 if size <= (32 << 20) else 1)
                iters = a.iters if size <= (64 << 20) else max(4, a.iters // 2)
                med, best, graphed = timed(fn, iters, a.warmup, inner)
                t = torch.tensor([med, best], device="cuda", dtype=torch.float64)
                dist.all_reduce(t, op=dist.ReduceOp.MAX)
                med, best = float(t[0]), float(t[1])
                nbytes = n * esz
                algbw = nbytes / (med * 1e-3) / 1e9
                rows.append({"impl": a.tag, "op": op, "dtype": dname, "bytes": nbytes, "us_median_max_over_ranks": med * 1e3,
                             "us_best_max_over_ranks": best * 1e3, "algbw_gbs": algbw, "busbw_gbs": algbw * factor,
                             "busbw_frac_of_link": algbw * factor / LINK_GBS, "graph_replay": graphed})
                if rank == 0:
                    print(f"{a.tag:5s} {op:14s} {dname:9s} {nbytes:>11d} B {med * 1e3:10.1f} us  busbw {algbw * factor:8.2f} GB/s", flush=True)
                del full, part
                size *= 4 if size < (1 << 20) else 2
    calls = fwd = None
    if "b200mpi" in os.environ.get("LD_PRELOAD", ""):
        import ctypes
        lib = ctypes.CDLL(os.environ["LD_PRELOAD"].split(":")[0])
        lib.b200mpi_shim_calls.restype = lib.b200mpi_shim_forwarded.restype = ctypes.c_uint64
        calls, fwd = int(lib.b200mpi_shim_calls()), int(lib.b200mpi_shim_forwarded())
    if rank == 0 and a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump({"impl": a.tag, "world": world, "shim_calls": calls, "shim_forwarded": fwd,
                       "torch": torch.__version__, "nccl": ".".join(map(str, torch.cuda.nccl.version())), "rows": rows}, f, indent=1)
    dist.barrier()
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
