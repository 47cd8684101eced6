"""Cost of parameter groups in the fused allreduce+SGD step, on one GPU.

Kernel A/B: the buckets of ResNet-101's flat layout (FlatModelState with the bf16 shadow, as the single-GPU trainer builds
it) on a world-1 communicator. One rep launches every bucket's k_allreduce_sgd once, i.e. one step's worth of optimizer
work, ungrouped (hyper-parameters from one device triple) or grouped (group map + table: no weight decay on BatchNorm and
bias parameters). CUDA events around each rep, L2 flushed before it (a 256 MiB buffer is rewritten), the arms alternate rep
by rep; the median per arm is reported.

End to end: ResNet-101, batch 64, bf16 autocast, CUDA graph, images/sec over `--steps` steps after `--warmup`, L2 flushed
before every step as bench.py does. Arm "none": param_groups=None, weight_decay=5e-5 on every parameter. Arm "recipe":
the same trainer-level weight_decay=5e-5, with BatchNorm and bias parameters in a group with weight_decay 0. The arms
alternate, `--runs` runs each.

The card's name, power limit and maximum SM clock are read with a read-only nvidia-smi query in the same process.

    python benchmarks/param_groups_bench.py --out profiles/param_groups_bench.json
"""
import argparse
import gc
import json
import os
import subprocess
import sys
import time

import torch
import torch.nn as nn

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mpi_operator_b200.models import build_model  # noqa: E402
from mpi_operator_b200.parallel.data_parallel import DataParallelTrainer, FlatModelState  # noqa: E402
from mpi_operator_b200.runtime.comm import Communicator  # noqa: E402


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (s.strip() for s in q.split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def no_decay(model):
    """BatchNorm gamma/beta and biases: every 1-D parameter of a ResNet."""
    return [p for p in model.parameters() if p.requires_grad and p.dim() == 1]


def kernel_ab(comm, reps: int) -> dict:
    torch.manual_seed(0)
    model = build_model("resnet101").cuda()
    nd = {p: 1 for p in no_decay(model)}
    st = FlatModelState(model, comm, 32 << 20, bf16_params=True, group_of=nd)
    st.flat_grad.copy_(torch.randn(st.total, device="cuda") * 1e-3)
    hyper = torch.tensor([1e-4, 0.9, 5e-5], device="cuda")
    table = torch.tensor([[1e-4, 0.9, 5e-5], [1e-4, 0.9, 0.0]], device="cuda")
    comm.set_hyper(hyper)
    maps = [st.bucket_group_map(b) for b in st.buckets]
    stream = torch.cuda.current_stream()

    def step(grouped):
        for b, m in zip(st.buckets, maps):
            kw = dict(group_map=m, group_hyper=table) if grouped else {}
            comm.allreduce_sgd_window(st.grad_win, b.start * 4, st.param_win, b.start * 4, b.momentum, b.numel, torch.float32,
                                      lr=1e-4, momentum_coef=0.9, weight_decay=5e-5, lowp_win=st.lowp_win,
                                      lowp_off=b.start * 2, stream=stream, **kw)

    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    for _ in range(5):
        step(False)
        step(True)
    torch.cuda.synchronize()
    times = {False: [], True: []}
    for _ in range(reps):
        for grouped in (False, True):
            flush.zero_()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            step(grouped)
            b.record()
            torch.cuda.synchronize()
            times[grouped].append(a.elapsed_time(b) * 1e3)
    comm.check_error()
    med = {k: sorted(v)[len(v) // 2] for k, v in times.items()}
    out = {"buckets": len(st.buckets), "params": sum(p.numel() for p in st.params), "map_bytes": st.group_map.numel(),
           "reps": reps, "ungrouped_us_median": round(med[False], 1), "grouped_us_median": round(med[True], 1),
           "ungrouped_us_p10_p90": [round(sorted(times[False])[reps // 10], 1), round(sorted(times[False])[reps * 9 // 10], 1)],
           "grouped_us_p10_p90": [round(sorted(times[True])[reps // 10], 1), round(sorted(times[True])[reps * 9 // 10], 1)],
           "overhead_pct": round(100.0 * (med[True] / med[False] - 1.0), 2)}
    comm.set_hyper(None)
    return out


def end_to_end(comm, arm: str, batch: int, steps: int, warmup: int) -> float:
    torch.manual_seed(1234)
    model = build_model("resnet101")
    groups = [{"params": no_decay(model), "weight_decay": 0.0}] if arm == "recipe" else None
    tr = DataParallelTrainer(model, nn.CrossEntropyLoss(), comm, lr=0.01, momentum=0.9, weight_decay=5e-5, cuda_graph=True,
                             autocast_dtype=torch.bfloat16, param_groups=groups)
    xs = [torch.randn(batch, 3, 224, 224).pin_memory() for _ in range(2)]
    ys = [torch.randint(0, 1000, (batch,)).pin_memory() for _ in range(2)]
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    for i in range(warmup):
        tr.step(xs[i % 2], ys[i % 2])
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(steps):
        flush.zero_()
        loss = tr.step(xs[i % 2], ys[i % 2])
    e1.record()
    torch.cuda.synchronize()
    comm.check_error()
    if float(loss) != float(loss):
        raise RuntimeError(f"arm {arm}: loss is NaN")
    ips = batch * steps / (e0.elapsed_time(e1) / 1e3)
    del tr, model, loss
    gc.collect()
    torch.cuda.empty_cache()
    return ips


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=300)
    ap.add_argument("--batch", type=int, default=64)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--runs", type=int, default=3)
    ap.add_argument("--skip-e2e", action="store_true")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("param_groups_bench needs a CUDA GPU")
    torch.cuda.set_device(0)
    torch.backends.cudnn.benchmark = True
    res = {"card": card(), "torch": torch.__version__}
    comm = Communicator.create(0, 1, 0, f"pgbench-{os.getpid()}")
    res["kernel"] = kernel_ab(comm, args.reps)
    print(json.dumps({"kernel": res["kernel"], "card": res["card"]}), flush=True)
    if not args.skip_e2e:
        runs = []
        for r in range(args.runs):
            for arm in ("none", "recipe"):
                t = time.time()
                ips = end_to_end(comm, arm, args.batch, args.steps, args.warmup)
                runs.append({"arm": arm, "run": r, "images_per_sec": round(ips, 1), "wall_s": round(time.time() - t, 1)})
                print(json.dumps(runs[-1]), flush=True)
        res["e2e"] = {"model": "resnet101", "batch": args.batch, "steps": args.steps, "warmup": args.warmup, "runs": runs}
    res["card_after"] = card()
    comm.destroy()
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
