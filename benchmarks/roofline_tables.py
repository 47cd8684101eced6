"""Merge ``collective_sweep.py`` outputs (stock NCCL run + injected-shim run of the SAME script) into markdown tables:
one table per (op, dtype) with time, bus bandwidth, fraction of the H100 NVLink data-sheet rate (LINK_GBS, 450 GB/s per direction) and the ratio
to NCCL.  Usage: python benchmarks/roofline_tables.py nccl.json shim.json [--out profiles/roofline_x.md]"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mpi_operator_b200.utils.roofline import LINK_GBS  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("files", nargs="+")
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    data = {}
    meta = []
    for f in a.files:
        d = json.load(open(f))
        meta.append(f"{d['impl']}: world {d['world']}, torch {d.get('torch')}, NCCL {d.get('nccl')}, "
                    f"shim_calls={d.get('shim_calls')}, forwarded={d.get('shim_forwarded')} ({f})")
        world = d["world"]
        for r in d["rows"]:
            data.setdefault((r["op"], r["dtype"]), {}).setdefault(r["bytes"], {})[r["impl"]] = r
    out = [f"# torch.distributed collectives on plain `torch.empty` tensors, {world} x H100 (NVSwitch)", ""]
    out += ["Same script (`benchmarks/collective_sweep.py`), same launcher; `shim` = `LD_PRELOAD=libb200mpi_nccl.so` (b200mpi kernels",
            "behind the NCCL C ABI, unregistered user pointers), `nccl` = no injection. CUDA events around CUDA-graph replays,",
            "median, max over ranks. busbw factors: allreduce 2(N-1)/N, allgather / reduce_scatter (N-1)/N, broadcast 1.", ""]
    out += [f"* {m}" for m in meta] + [""]
    for (op, dt), sizes in sorted(data.items()):
        out += [f"## {op}, {dt}", "", f"| bytes | shim us | shim busbw GB/s | busbw / {LINK_GBS:.0f} | NCCL us | NCCL busbw GB/s | speed-up vs NCCL |", "|---|---|---|---|---|---|---|"]
        worst = None
        for b in sorted(sizes):
            s, n = sizes[b].get("shim"), sizes[b].get("nccl")
            f = lambda r, k, fmt: (fmt % r[k]) if r else "-"  # noqa: E731
            ratio = (n["us_median_max_over_ranks"] / s["us_median_max_over_ranks"]) if s and n else None
            if ratio is not None and (worst is None or ratio < worst[0]):
                worst = (ratio, b)
            out.append(f"| {b} | {f(s, 'us_median_max_over_ranks', '%.1f')} | {f(s, 'busbw_gbs', '%.1f')} | {('%.3f' % (s['busbw_gbs'] / LINK_GBS)) if s else '-'} | "
                       f"{f(n, 'us_median_max_over_ranks', '%.1f')} | {f(n, 'busbw_gbs', '%.1f')} | {('%.2fx' % ratio) if ratio else '-'} |")
        if worst:
            out += ["", f"worst ratio vs NCCL: {worst[0]:.2f}x at {worst[1]} bytes", ""]
    text = "\n".join(out)
    if a.out:
        with open(a.out, "w") as f:
            f.write(text + "\n")
    print(text)


if __name__ == "__main__":
    main()
