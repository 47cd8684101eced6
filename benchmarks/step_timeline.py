"""Step timeline of the flagship trainer without nsys: a few eager (non-graph) steps under torch.profiler (CUPTI kernel
records: name, stream, start, duration) on every rank; rank 0 reports, per step, the wall span on the device, how long
each stream was busy, and the EXPOSED time of the comm stream and of the H2D copies (intervals where they run while the
compute stream is idle) - the part of the step that does not scale. Launch like bench.py:

  python -m torch.distributed.run --nproc-per-node 8 --master-addr 127.0.0.1 --master-port 29555 benchmarks/step_timeline.py --out profiles/step_timeline_n8.md

Numbers under the profiler are for attribution only (eager launches, CUPTI overhead), never throughput claims."""
import argparse
import json
import os
import sys

import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from mpi_operator_b200.launch.env import rank_info_from_env  # noqa: E402
from mpi_operator_b200.models import build_model  # noqa: E402
from mpi_operator_b200.parallel.data_parallel import DataParallelTrainer  # noqa: E402
from mpi_operator_b200.runtime.comm import Communicator  # noqa: E402


def union_len(iv):
    iv = sorted(iv)
    tot, cur_s, cur_e = 0.0, None, None
    for s, e in iv:
        if cur_e is None or s > cur_e:
            if cur_e is not None:
                tot += cur_e - cur_s
            cur_s, cur_e = s, e
        else:
            cur_e = max(cur_e, e)
    if cur_e is not None:
        tot += cur_e - cur_s
    return tot


def subtract(iv, mask):
    """total length of `iv` not covered by `mask` (both lists of (s, e))."""
    mask = sorted(mask)
    out = 0.0
    for s, e in iv:
        cur = s
        for ms, me in mask:
            if me <= cur:
                continue
            if ms >= e:
                break
            if ms > cur:
                out += ms - cur
            cur = max(cur, me)
            if cur >= e:
                break
        if cur < e:
            out += e - cur
    return out


KERNEL_CLASSES = ("bn_fwd", "bn_reduce", "bn_finalize", "bn_elemt", "autograd_add", "cublas_dgrad", "cublas_wgrad", "cudnn",
                  "wgmma_gemm", "weight_copy", "memset", "other")


def kernel_class(name: str, op: str, dims) -> str:
    """Device-time class of one kernel record. `op` / `dims` are the innermost CPU op that launched it and that op's input
    shapes (record_shapes): they tell autograd's gradient add from other elementwise kernels, and a 1x1 dgrad GEMM
    (dy [M,Cout] @ w [Cout,Cin]: inner dimension = a channel count) from its wgrad (dy^T @ x: inner dimension = M). That
    split assumes M > 2048, the widest ResNet channel count: true at batch 64, not for the 7x7 stage below batch 42.
    weight_copy: 2-D copies, i.e. the per-step transposed 1x1 weights the wgmma dgrad reads."""
    if "k_gemm_bnstats" in name or "k_gemm_dgrad" in name:
        return "wgmma_gemm"
    if "k_bn_bwd_reduce" in name:
        return "bn_reduce"
    if "finalize" in name and "k_bn_" in name:
        return "bn_finalize"
    if "k_bn_bwd_elemt" in name:
        return "bn_elemt"
    if "k_bn_fwd" in name:
        return "bn_fwd"
    if op in ("aten::copy_", "aten::clone", "aten::contiguous") and dims and len(dims[0] or ()) == 2:
        return "weight_copy"
    if op in ("aten::add", "aten::add_") and "elementwise" in name:
        return "autograd_add"
    if op in ("aten::mm", "aten::addmm", "aten::matmul"):
        try:
            inner = int(dims[0][1])
        except (TypeError, ValueError, IndexError):
            inner = 0
        return "cublas_wgrad" if inner > 2048 else "cublas_dgrad"   # every ResNet channel count is <= 2048 < M
    if op.startswith("aten::cudnn") or op.startswith("aten::convolution") or "cudnn" in name:
        return "cudnn"
    return "other"


def class_breakdown(trace: dict, steps: int) -> dict:
    """Device time (us) and kernel count per step for every KERNEL_CLASSES entry."""
    ops, corr_ext = {}, {}
    for e in trace["traceEvents"]:
        a = e.get("args") or {}
        if e.get("cat") == "cpu_op" and "External id" in a:
            ops[a["External id"]] = (e.get("name", ""), a.get("Input Dims"))
        elif e.get("cat") == "cuda_runtime" and "correlation" in a and "External id" in a:
            corr_ext[a["correlation"]] = a["External id"]
    out = {c: {"us": 0.0, "kernels": 0} for c in KERNEL_CLASSES}
    for e in trace["traceEvents"]:
        if e.get("cat") not in ("kernel", "gpu_memset") or "dur" not in e:
            continue
        a = e.get("args") or {}
        ext = a.get("External id", corr_ext.get(a.get("correlation")))
        op, dims = ops.get(ext, ("", None))
        c = "memset" if e["cat"] == "gpu_memset" else kernel_class(e["name"], op, dims)
        out[c]["us"] += e["dur"] / steps
        out[c]["kernels"] += 1 / steps
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--model", default="resnet101")
    ap.add_argument("--batch-size", type=int, default=64)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    info = rank_info_from_env()
    rank, world = info.rank, info.world_size
    dev = info.local_rank % torch.cuda.device_count()
    torch.cuda.set_device(dev)
    torch.backends.cudnn.benchmark = True
    comm = Communicator.create(rank, world, dev, info.job_id + "-timeline")
    tr = DataParallelTrainer(build_model(a.model), nn.CrossEntropyLoss(), comm, lr=0.01 * world, momentum=0.9, cuda_graph=False)
    B = a.batch_size
    xs = [torch.randn(B, 3, 224, 224).pin_memory() for _ in range(2)]
    ys = [torch.randint(0, 1000, (B,)).pin_memory() for _ in range(2)]
    for i in range(6):
        tr.step(xs[i % 2], ys[i % 2])
    torch.cuda.synchronize()
    comm.host_barrier()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA, ProfilerActivity.CPU], record_shapes=True) as prof:
        for i in range(a.steps):
            tr.step(xs[i % 2], ys[i % 2])
        torch.cuda.synchronize()
    comm.host_barrier()
    path = f"/tmp/b200mpi_timeline_{os.getpid()}.json"
    prof.export_chrome_trace(path)
    trace = json.load(open(path))
    os.unlink(path)
    ev = [e for e in trace["traceEvents"] if e.get("cat") in ("kernel", "gpu_memcpy", "gpu_memset") and "dur" in e]
    comm_k = [e for e in ev if "k_allreduce" in e["name"] or "b200mpi::k_" in e["name"]]
    comm_streams = {e["args"].get("stream") for e in comm_k}
    h2d = [e for e in ev if e.get("cat") == "gpu_memcpy" and "HtoD" in e["name"]]
    comp = [e for e in ev if e not in comm_k and e not in h2d and e["args"].get("stream") not in comm_streams]
    iv = lambda es: [(e["ts"], e["ts"] + e["dur"]) for e in es]  # noqa: E731
    span = (max(e["ts"] + e["dur"] for e in ev) - min(e["ts"] for e in ev)) / a.steps
    rep = {
        "rank": rank, "world": world, "steps": a.steps, "span_us_per_step": span,
        "compute_busy_us": union_len(iv(comp)) / a.steps,
        "comm_busy_us": union_len(iv(comm_k)) / a.steps,
        "comm_exposed_us": subtract(iv(comm_k), iv(comp)) / a.steps,
        "h2d_busy_us": union_len(iv(h2d)) / a.steps,
        "h2d_exposed_us": subtract(iv(h2d), iv(comp)) / a.steps,
        "comm_kernels_per_step": len(comm_k) / a.steps,
        "h2d_stream_is_compute_stream": bool({e["args"].get("stream") for e in h2d} & {e["args"].get("stream") for e in comp}),
    }
    # the last comm kernel of each step (the tail bucket): how much of it runs after the last compute kernel
    tails = []
    ordered = sorted(comm_k, key=lambda e: e["ts"])
    per = max(1, len(ordered) // a.steps)
    for s in range(a.steps):
        chunk = ordered[s * per:(s + 1) * per]
        if not chunk:
            continue
        last = chunk[-1]
        before = [e for e in comp if e["ts"] < last["ts"] + last["dur"]]
        last_comp_end = max((e["ts"] + e["dur"] for e in before), default=last["ts"])
        tails.append({"name": last["name"][:60], "dur_us": last["dur"], "exposed_us": max(0.0, last["ts"] + last["dur"] - max(last_comp_end, last["ts"]))})
    rep["tail_bucket"] = tails
    rep["classes"] = class_breakdown(trace, a.steps)
    import struct
    blob = json.dumps(rep).encode()
    if world > 1:
        sizes = comm.host_allgather(struct.pack("q", len(blob)))
    if rank == 0:
        lines = [f"# Step timeline, {a.model} bs {B}/GPU, {world} GPU(s), eager launches under torch.profiler (attribution only)", "",
                 "| per step (rank 0) | us |", "|---|---|"]
        for k in ("span_us_per_step", "compute_busy_us", "comm_busy_us", "comm_exposed_us", "h2d_busy_us", "h2d_exposed_us"):
            lines.append(f"| {k} | {rep[k]:.0f} |")
        lines += ["", f"comm kernels per step: {rep['comm_kernels_per_step']:.0f}; H2D on the compute stream: {rep['h2d_stream_is_compute_stream']}", "",
                  "tail bucket (last comm kernel of each step): " + json.dumps(tails), "",
                  "| kernel class | device us / step | kernels / step |", "|---|---|---|"]
        for c, v in rep["classes"].items():
            lines.append(f"| {c} | {v['us']:.0f} | {v['kernels']:.0f} |")
        lines.append("")
        text = "\n".join(lines)
        print(text)
        print("JSON " + json.dumps(rep))
        if a.out:
            os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
            with open(a.out, "w") as f:
                f.write(text + "\n")
    comm.host_barrier() if world > 1 else None
    comm.destroy()


if __name__ == "__main__":
    main()
