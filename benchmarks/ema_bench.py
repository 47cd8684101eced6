"""Cost of the weight average (``ema_decay``) in the fused allreduce+optimizer step, on one GPU.

Kernel A/B: the buckets of ResNet-101's flat layout (FlatModelState with the bf16 shadow, as the single-GPU trainer builds
it) on a world-1 communicator, with BatchNorm and bias parameters in a group of their own. One rep launches one step's
worth of optimizer work, every bucket once: grouped k_allreduce_sgd without and with the average (arms "sgd" / "sgd_ema"),
and the LARS pair without and with it (arms "lars" / "lars_ema"). CUDA events around each rep, L2 flushed before it (a
256 MiB buffer is rewritten), the four arms alternate rep by rep; the median per arm is reported, next to the extra HBM bytes
the average moves by construction (the EMA slice read and written once: 2 x the fp32 parameter bytes at world 1).

End to end: ResNet-101, bf16 autocast, CUDA graph, images/sec over `--steps` steps after `--warmup`, L2 flushed before every
step as bench.py does, at each `--batch`. Arm "off": ema_decay=None; arm "ema": ema_decay=0.9999. The arms alternate,
`--runs` runs each, every run in a process of its own.

The card's name, power limit and maximum SM clock are read with a read-only nvidia-smi query in the same process.

    python benchmarks/ema_bench.py --out profiles/ema_bench.json
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

ARMS = ("sgd", "sgd_ema", "lars", "lars_ema")


def card() -> dict:
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    name, power, clock = (s.strip() for s in q.split(","))
    return {"name": name, "power_limit": power, "max_sm_clock": clock}


def _median(v):
    return sorted(v)[len(v) // 2]


def kernel_ab(comm, reps: int) -> dict:
    torch.manual_seed(0)
    model = build_model("resnet101").cuda()
    group_of = {p: 1 for p in model.parameters() if p.dim() == 1}
    lars_of = {p: p.dim() != 1 for p in model.parameters()}
    st = FlatModelState(model, comm, 32 << 20, bf16_params=True, group_of=group_of, lars_of=lars_of)
    st.flat_grad.copy_(torch.randn(st.total, device="cuda") * 1e-3)
    table = torch.tensor([[1e-4, 0.9, 5e-5], [1e-4, 0.9, 0.0]], device="cuda")
    P = max(len(b.params) for b in st.buckets)
    board = comm.alloc_window(P * comm.world * 8 + 16)
    scratch = torch.zeros(max(comm.lars_scratch_bytes(b.numel, len(b.params)) for b in st.buckets), dtype=torch.uint8,
                          device="cuda")
    gmaps = [st.bucket_group_map(b) for b in st.buckets]
    pmaps = [st.bucket_param_map(b) for b in st.buckets]
    emas = [torch.zeros_like(b.momentum) for b in st.buckets]
    sched = torch.tensor([0.9999, 1000.0], dtype=torch.float64, device="cuda")
    stream = torch.cuda.current_stream()

    def step(arm):
        for b, gm, pm, e in zip(st.buckets, gmaps, pmaps, emas):
            common = (st.grad_win, b.start * 4, st.param_win, b.start * 4, b.momentum, b.numel, torch.float32)
            ekw = {"ema": e, "ema_sched": sched} if arm.endswith("_ema") else {}
            if arm.startswith("lars"):
                comm.allreduce_lars_window(*common, group_hyper=table, param_map=pm, param_table=b.param_table,
                                           board_win=board, board_off=0, scratch=scratch, trust_coefficient=0.001,
                                           lowp_win=st.lowp_win, lowp_off=b.start * 2, stream=stream, trust_out=b.trust,
                                           **ekw)
            else:
                comm.allreduce_sgd_window(*common, lr=1e-4, momentum_coef=0.9, weight_decay=5e-5, lowp_win=st.lowp_win,
                                          lowp_off=b.start * 2, stream=stream, group_map=gm, group_hyper=table, **ekw)

    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    for _ in range(5):
        for arm in ARMS:
            step(arm)
    torch.cuda.synchronize()
    times = {arm: [] for arm in ARMS}
    for _ in range(reps):
        for arm in ARMS:
            flush.zero_()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            step(arm)
            b.record()
            torch.cuda.synchronize()
            times[arm].append(a.elapsed_time(b) * 1e3)
    comm.check_error()
    med = {k: _median(v) for k, v in times.items()}
    out = {"buckets": len(st.buckets), "params": sum(p.numel() for p in st.params), "reps": reps,
           "extra_hbm_bytes_by_construction": 2 * st.total * 4 // comm.world}
    for arm in ARMS:
        s = sorted(times[arm])
        out[f"{arm}_us_median"] = round(med[arm], 1)
        out[f"{arm}_us_p10_p90"] = [round(s[reps // 10], 1), round(s[reps * 9 // 10], 1)]
    out["sgd_ema_overhead_pct"] = round(100.0 * (med["sgd_ema"] / med["sgd"] - 1.0), 2)
    out["lars_ema_overhead_pct"] = round(100.0 * (med["lars_ema"] / med["lars"] - 1.0), 2)
    board.free()
    return out


def end_to_end(comm, arm: str, batch: int, steps: int, warmup: int) -> float:
    torch.manual_seed(1234)
    model = build_model("resnet101")
    tr = DataParallelTrainer(model, nn.CrossEntropyLoss(), comm, lr=0.01, momentum=0.9, weight_decay=5e-5, cuda_graph=True,
                             autocast_dtype=torch.bfloat16, ema_decay=0.9999 if arm == "ema" else None)
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


def end_to_end_in_subprocess(arm: str, batch: int, steps: int, warmup: int) -> float:
    """One end-to-end run in a fresh process: every run starts from an empty device (windows and graph pools included)."""
    out = subprocess.run([sys.executable, os.path.abspath(__file__), "--one", arm, "--batch", str(batch), "--steps", str(steps),
                          "--warmup", str(warmup)], capture_output=True, text=True, check=True).stdout
    return json.loads(out.strip().splitlines()[-1])["images_per_sec"]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--one", choices=["off", "ema"], help="run one end-to-end arm at the first --batch and print its rate")
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--batch", type=int, nargs="+", default=[64, 256])
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--runs", type=int, default=2)
    ap.add_argument("--skip-e2e", action="store_true")
    ap.add_argument("--out", default="")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("ema_bench needs a CUDA GPU")
    torch.cuda.set_device(0)
    torch.backends.cudnn.benchmark = True
    comm = Communicator.create(0, 1, 0, f"emabench-{os.getpid()}")
    if args.one:
        print(json.dumps({"images_per_sec": end_to_end(comm, args.one, args.batch[0], args.steps, args.warmup)}))
        comm.destroy()
        return
    res = {"card": card(), "torch": torch.__version__}
    res["kernel"] = kernel_ab(comm, args.reps)
    print(json.dumps({"kernel": res["kernel"], "card": res["card"]}), flush=True)
    if not args.skip_e2e:
        runs = []
        for batch in args.batch:
            for r in range(args.runs):
                for arm in ("off", "ema"):
                    t = time.time()
                    ips = end_to_end_in_subprocess(arm, batch, args.steps, args.warmup)
                    runs.append({"arm": arm, "batch": batch, "run": r, "images_per_sec": round(ips, 1),
                                 "wall_s": round(time.time() - t, 1)})
                    print(json.dumps(runs[-1]), flush=True)
        res["e2e"] = {"model": "resnet101", "steps": args.steps, "warmup": args.warmup, "runs": runs}
    res["card_after"] = card()
    comm.destroy()
    print(json.dumps(res))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
