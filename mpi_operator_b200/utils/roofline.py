"""Roofline report for the collective sweeps: achieved bus bandwidth per message size and algorithm against the
NVLink data-sheet rate of the H100 SXM (450 GB/s per direction per GPU, NVLink 4), next to stock NCCL on the same box.
Writes markdown.

    python -m mpi_operator_b200.utils.roofline profiles/allreduce_sweep_n8_f32.json [more.json] > profiles/roofline_allreduce.md
"""
from __future__ import annotations

import json
import sys

LINK_GBS = 450.0   # H100 SXM data sheet: NVLink 4, 18 links, 450 GB/s per direction per GPU (every sweep's denominator)


def report(path: str) -> str:
    d = json.load(open(path))
    rows = d["rows"]
    W = d["world"]
    by = {}
    for r in rows:
        by.setdefault((r["dtype"], r["bytes"]), {})[r["algo"]] = r
    out = [f"## {W} GPUs — `{path.split('/')[-1]}` (NVLS multicast: {d.get('multicast')})", "",
           f"| dtype | bytes | best b200mpi algo | us | algbw GB/s | busbw GB/s | busbw / {LINK_GBS:.0f} | NCCL us | NCCL busbw | speed-up |",
           "|---|---|---|---|---|---|---|---|---|---|"]
    for (dt, b), algos in sorted(by.items()):
        ours = {k: v for k, v in algos.items() if k != "nccl"}
        if not ours:
            continue
        k = min(ours, key=lambda k: ours[k]["ms_median_max_over_ranks"])
        o = ours[k]
        n = algos.get("nccl")
        nccl_us = f"{n['ms_median_max_over_ranks'] * 1e3:.1f}" if n else "-"
        nccl_bw = f"{n['busbw_gbs']:.1f}" if n else "-"
        sp = f"{n['ms_median_max_over_ranks'] / o['ms_median_max_over_ranks']:.2f}x" if n else "-"
        out.append(f"| {dt} | {b} | {k} | {o['ms_median_max_over_ranks'] * 1e3:.1f} | {o['algbw_gbs']:.1f} | {o['busbw_gbs']:.1f} | "
                   f"{o['busbw_gbs'] / LINK_GBS:.2f} | {nccl_us} | {nccl_bw} | {sp} |")
    return "\n".join(out)


def main(argv=None) -> int:
    argv = argv or sys.argv[1:]
    print("# Allreduce roofline (device time from CUDA-graph replays, median, max over ranks)\n")
    print(f"busbw = algbw x 2(N-1)/N. Denominator: {LINK_GBS:.0f} GB/s per direction per GPU (H100 SXM data sheet, NVLink 4). An NVLS "
          "allreduce moves S(1+1/N) bytes per direction instead of 2S(N-1)/N, so its bus bandwidth can exceed the link rate.\n")
    for p in argv:
        print(report(p))
        print()
    return 0


if __name__ == "__main__":
    sys.exit(main())
