"""profiles/roofline_<op>.md from the collective_sweep JSONs of a session (stock NCCL vs the injected shim, same script) and,
for allreduce, the native sweep (window / NVLS / pipelined / registered rows).
Usage: python benchmarks/roofline_per_op.py profiles/r2 --out profiles"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mpi_operator_b200.utils.roofline import LINK_GBS  # noqa: E402


def load(path):
    try:
        return json.load(open(path))
    except (OSError, ValueError):
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("root")
    ap.add_argument("--out", default="profiles")
    a = ap.parse_args()
    per_op = {}
    for n in (8, 4, 2):
        nc, sh = load(f"{a.root}/n{n}/sweep_nccl_n{n}.json"), load(f"{a.root}/n{n}/sweep_shim_n{n}.json")
        if not nc or not sh:
            continue
        rows = {}
        for d in (nc, sh):
            for r in d["rows"]:
                rows.setdefault((r["op"], r["dtype"], r["bytes"]), {})[r["impl"]] = r
        for (op, dt, b), v in rows.items():
            per_op.setdefault(op, {}).setdefault(n, {}).setdefault(dt, {})[b] = v
    for op, by_n in per_op.items():
        out = [f"# {op}: bus bandwidth vs message size, injected shim (`LD_PRELOAD=libb200mpi_nccl.so`) vs stock NCCL 2.28.9", "",
               "Same script (`benchmarks/collective_sweep.py`: torch.distributed on plain `torch.empty` tensors), same launcher, same box;",
               "CUDA events around CUDA-graph replays, median, max over ranks. busbw = algbw x " +
               {"allreduce": "2(N-1)/N", "allgather": "(N-1)/N", "reduce_scatter": "(N-1)/N", "broadcast": "1"}[op] +
               f"; the roofline is {LINK_GBS:.0f} GB/s per direction per GPU (H100 SXM data sheet, NVLink 4).", ""]
        for n in sorted(by_n, reverse=True):
            out += [f"## {n} GPUs", ""]
            for dt in sorted(by_n[n]):
                out += [f"### {dt}", "", f"| bytes | shim us | shim busbw GB/s | busbw / {LINK_GBS:.0f} | NCCL us | NCCL busbw GB/s | shim / NCCL |", "|---|---|---|---|---|---|---|"]
                worst = None
                for b in sorted(by_n[n][dt]):
                    v = by_n[n][dt][b]
                    s, c = v.get("shim"), v.get("nccl")
                    if not s or not c:
                        continue
                    ratio = c["us_median_max_over_ranks"] / s["us_median_max_over_ranks"]
                    worst = ratio if worst is None else min(worst, ratio)
                    out.append(f"| {b} | {s['us_median_max_over_ranks']:.1f} | {s['busbw_gbs']:.1f} | {s['busbw_gbs'] / LINK_GBS:.3f} | "
                               f"{c['us_median_max_over_ranks']:.1f} | {c['busbw_gbs']:.1f} | {ratio:.2f}x |")
                out += ["", f"worst ratio: {worst:.2f}x" if worst else "", ""]
        if op == "allreduce":
            for n in (8, 4):
                nat = load(f"{a.root}/n{n}/allreduce_sweep_n{n}_f32.json")
                if not nat:
                    continue
                by = {}
                for r in nat["rows"]:
                    by.setdefault(r["bytes"], {})[r["algo"]] = r
                cols = ["oneshot", "twoshot", "nvls", "staged", "pipe", "reg", "nccl"]
                out += [f"## native API, fp32, {n} GPUs: every algorithm (busbw GB/s; window = zero-copy symmetric window, user pointers = staged / pipe / reg)", "",
                        "| bytes | " + " | ".join({"oneshot": "one-shot", "twoshot": "two-shot P2P (window)", "nvls": "NVLS (window)", "staged": "staged two-shot (user ptr)",
                                                    "pipe": "pipelined NVLS (user ptr)", "reg": "cudaIpc-registered two-shot (user ptr)", "nccl": "NCCL"}[c] for c in cols) + " |",
                        "|---|" + "---|" * len(cols)]
                for b in sorted(by):
                    out.append(f"| {b} | " + " | ".join(f"{by[b][c]['busbw_gbs']:.0f}" if c in by[b] else "-" for c in cols) + " |")
                out.append("")
        path = os.path.join(a.out, f"roofline_{op.replace('_', '')}.md")
        with open(path, "w") as f:
            f.write("\n".join(out) + "\n")
        print("wrote", path)


if __name__ == "__main__":
    main()
