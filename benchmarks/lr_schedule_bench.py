"""Cost of the device-side learning-rate schedule (``DataParallelTrainer(lr_schedule=...)``) on one GPU.

Kernel alone: ``k_lr_schedule`` for two parameter groups (ResNet recipes keep BatchNorm and biases in a group of their own)
with a polynomial schedule, `--launches` launches between two CUDA events, repeated `--reps` times; the median time per
launch is reported for launches issued back to back from Python (which measures the host's enqueue rate more than the
kernel) and for the same launches replayed as one CUDA graph (as in the trainer's captured step).

Step A/B: ResNet-101, batch `--batch`, world 1, bf16 autocast, CUDA graph, the trainer's defaults (bench.py's flagship
configuration). Two trainers are built in one process, one with an MLPerf-style schedule (polynomial decay with warm-up)
and one without; their steps alternate, each step timed with CUDA events on the compute stream after the L2 is flushed (a
256 MiB buffer is rewritten). The median per arm over `--steps` steps after `--warmup` is reported.

The card's name, power limit and maximum SM clock are read with a read-only nvidia-smi query in the same process.

    python benchmarks/lr_schedule_bench.py --out profiles/lr_schedule_bench.json
"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn as nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mpi_operator_b200.models import build_model  # noqa: E402
from mpi_operator_b200.parallel.data_parallel import DataParallelTrainer  # noqa: E402
from mpi_operator_b200.parallel.lr_schedule import LRSchedule  # noqa: E402
from mpi_operator_b200.runtime.comm import Communicator  # noqa: E402


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (s.strip() for s in q.split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def _median(v):
    return sorted(v)[len(v) // 2]


def kernel_alone(comm, launches: int, reps: int) -> dict:
    """Per launch: back to back from Python (bound by the host's enqueue rate) and as nodes of one CUDA graph, as the
    trainer's captured step runs it."""
    sch = LRSchedule.polynomial(total_steps=1 << 40, power=2, warmup_steps=1000)
    table = torch.tensor(sch.table(), dtype=torch.float64, device="cuda")
    step = torch.zeros(1, dtype=torch.int64, device="cuda")
    base = torch.tensor([6.4, 6.4], dtype=torch.float64, device="cuda")
    hyper = torch.tensor([0.0, 0.9, 5e-5], device="cuda")
    group_hyper = torch.tensor([[0.0, 0.9, 5e-5], [0.0, 0.9, 0.0]], device="cuda")

    def launch(n, s):
        for _ in range(n):
            comm.lr_schedule(table, sch.form, 0, step, base, hyper, group_hyper, stream=s)
    s = torch.cuda.current_stream()
    launch(100, s)
    g = torch.cuda.CUDAGraph()
    cs = torch.cuda.Stream()
    cs.wait_stream(s)
    with torch.cuda.stream(cs):
        with torch.cuda.graph(g):
            launch(launches, torch.cuda.current_stream())
    torch.cuda.synchronize()
    res = {"launches_per_rep": launches, "reps": reps}
    for arm, run in (("eager", lambda: launch(launches, s)), ("graph", g.replay)):
        per = []
        for _ in range(reps):
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(s)
            run()
            b.record(s)
            b.synchronize()
            per.append(a.elapsed_time(b) * 1e3 / launches)
        res[arm] = {"us_per_launch_median": _median(per), "us_per_launch_min": min(per), "us_per_launch_max": max(per)}
    return res


def step_ab(batch: int, steps: int, warmup: int) -> dict:
    torch.backends.cudnn.benchmark = True
    sched = LRSchedule.polynomial(total_steps=10 ** 6, power=2, warmup_steps=100)
    trainers, comms = {}, {}
    for arm in ("off", "on"):   # a communicator each: the fused kernels read the {lr, mu, wd} table set on it
        torch.manual_seed(0)
        comms[arm] = comm = Communicator.create(0, 1, 0, f"lrs-bench-{arm}-{os.getpid()}")
        trainers[arm] = DataParallelTrainer(build_model("resnet101"), nn.CrossEntropyLoss(), comm, lr=0.1, momentum=0.9,
                                            weight_decay=5e-5, lr_schedule=sched if arm == "on" else None)
    x = torch.randn(batch, 3, 224, 224).pin_memory()
    y = torch.randint(0, 1000, (batch,)).pin_memory()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    times = {"off": [], "on": []}
    for i in range(warmup + steps):
        for arm in (("off", "on") if i % 2 == 0 else ("on", "off")):
            tr = trainers[arm]
            tr.prefetch(x, y)
            torch.cuda.synchronize()
            flush.fill_(i & 0xFF)
            s = torch.cuda.current_stream()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record(s)
            tr.step()
            b.record(s)
            b.synchronize()
            if i >= warmup:
                times[arm].append(a.elapsed_time(b))
    out = {arm: {"ms_median": _median(v), "ms_min": min(v), "ms_max": max(v), "images_per_sec_at_median": batch / _median(v) * 1e3,
                 "launches_per_step": trainers[arm].launches_per_step} for arm, v in times.items()}
    out["on"]["lr_schedule_step"] = trainers["on"].lr_schedule_step
    out["on"]["lr_after"] = trainers["on"].current_lrs()
    out["delta_ms_median"] = out["on"]["ms_median"] - out["off"]["ms_median"]
    for c in comms.values():
        c.check_error()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--launches", type=int, default=2000)
    ap.add_argument("--reps", type=int, default=21)
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("lr_schedule_bench: needs a CUDA device")
    torch.cuda.set_device(0)
    comm = Communicator.create(0, 1, 0, f"lrs-bench-{os.getpid()}")
    res = {"card": card(), "kernel": kernel_alone(comm, args.launches, args.reps),
           "step_ab": step_ab(args.batch, args.steps, args.warmup),
           "config": {"model": "resnet101", "batch": args.batch, "world": 1, "steps": args.steps, "warmup": args.warmup}}
    comm.check_error()
    print(json.dumps(res, indent=1))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)
    comm.destroy()


if __name__ == "__main__":
    main()
