"""ResNet-101 eval-mode throughput (images/sec), bf16 autocast, channels-last, at batch 64 and 256. Four arms, alternated
round by round within one run:

  (a) graph     DataParallelTrainer.evaluate() with cuda_graph=True: one CUDA-graph replay per call, fused eval kernels
  (b) eager     the same evaluate() with the graph off: fused eval kernels, one Python dispatch per kernel
  (c) unfused   evaluate() with B200MPI_FUSED_BN=0 and no graph (cuDNN convolutions, ATen batch norm, add, ReLU), in a
                subprocess because the switch is read at import
  (d) torchvision  torchvision's resnet101 forward in eval mode under autocast, channels-last, no trainer

Each call is timed with CUDA events around one evaluate() (forward, loss, top-1/top-5 and the device-to-host read of the
result) on device-resident inputs, with L2 flushed before it (a 256 MiB buffer is rewritten); the median over `--iters`
calls gives images/sec. The card's name and power limit are recorded next to the numbers.

    python benchmarks/eval_bench.py --out profiles/eval_bench.json
"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn as nn

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card() -> dict:
    info = {"name": torch.cuda.get_device_name(0), "power_limit_w": None}
    try:
        out = subprocess.run(["nvidia-smi", "--id=0", "--query-gpu=power.limit", "--format=csv,noheader,nounits"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        info["power_limit_w"] = float(out.splitlines()[0])
    except Exception:
        pass
    return info


def time_calls(fn, iters: int, flush: torch.Tensor) -> float:
    """Median milliseconds of one fn() call, L2 flushed before each."""
    for _ in range(3):
        fn()
    ts = []
    for _ in range(iters):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    ts.sort()
    return ts[len(ts) // 2]


class Arms:
    """The in-process arms, built once per batch size."""

    def __init__(self, batch: int, graph: bool):
        from mpi_operator_b200.models import build_model
        from mpi_operator_b200.parallel.data_parallel import DataParallelTrainer
        from mpi_operator_b200.runtime.comm import Communicator
        torch.manual_seed(0)
        self.comm = Communicator.create(0, 1, 0, f"eval-bench-{os.getpid()}-{batch}-{int(graph)}")
        self.trainer = DataParallelTrainer(build_model("resnet101"), nn.CrossEntropyLoss(), self.comm, lr=0.1, momentum=0.9,
                                           cuda_graph=graph)
        self.x = torch.randn(batch, 3, 224, 224, device="cuda")
        self.y = torch.randint(0, 1000, (batch,), device="cuda")

    def evaluate(self):
        return self.trainer.evaluate(self.x, self.y)


def torchvision_arm(batch: int):
    import torchvision
    model = torchvision.models.resnet101().cuda().eval().to(memory_format=torch.channels_last)
    x = torch.randn(batch, 3, 224, 224, device="cuda").contiguous(memory_format=torch.channels_last)

    @torch.no_grad()
    def run():
        with torch.autocast("cuda", dtype=torch.bfloat16):
            out = model(x)
        return out.float().topk(5, dim=1).indices.tolist()
    return run


def child(batch: int, iters: int) -> None:
    """Arm (c): this process was started with B200MPI_FUSED_BN=0."""
    from mpi_operator_b200.ops import fused_bn
    assert not fused_bn._ENABLED
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    arm = Arms(batch, graph=False)
    ms = time_calls(arm.evaluate, iters, flush)
    print(json.dumps({"ms": ms}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", default="64,256")
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default="")
    ap.add_argument("--child", type=int, default=0, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("eval_bench.py needs a CUDA device")
    if a.child:
        child(a.child, a.iters)
        return
    torch.cuda.set_device(0)
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    result = {"card": card(), "model": "resnet101", "dtype": "bf16 autocast", "layout": "channels_last", "iters": a.iters,
              "l2": "256 MiB buffer rewritten before every call", "batches": {}}
    for batch in [int(b) for b in a.batches.split(",")]:
        graph, eager = Arms(batch, graph=True), Arms(batch, graph=False)
        tv = torchvision_arm(batch)
        torch.cuda.synchronize()
        before = torch.cuda.memory_reserved()
        graph.evaluate()                      # captures the eval graph for this shape
        torch.cuda.synchronize()
        extra = torch.cuda.memory_reserved() - before
        ms = {"graph": [], "eager": [], "unfused": [], "torchvision": []}
        for _ in range(a.rounds):
            ms["graph"].append(time_calls(graph.evaluate, a.iters, flush))
            ms["eager"].append(time_calls(eager.evaluate, a.iters, flush))
            r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", str(batch), "--iters", str(a.iters)],
                               env={**os.environ, "B200MPI_FUSED_BN": "0"}, capture_output=True, text=True, timeout=1200)
            if r.returncode != 0:
                raise RuntimeError(r.stdout[-2000:] + r.stderr[-2000:])
            ms["unfused"].append(json.loads(r.stdout.strip().splitlines()[-1])["ms"])
            ms["torchvision"].append(time_calls(tv, a.iters, flush))
        row = {arm: {"ms": [round(t, 3) for t in v], "images_per_sec": [round(batch / t * 1e3, 1) for t in v]}
               for arm, v in ms.items()}
        row["eval_graph_memory_reserved_mib"] = round(extra / 2 ** 20, 1)
        result["batches"][batch] = row
        print(json.dumps({"batch": batch, **row}), flush=True)
        graph.comm.destroy()
        eager.comm.destroy()
        del graph, eager, tv
        torch.cuda.empty_cache()
    print(json.dumps(result), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
