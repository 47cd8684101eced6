"""Micro-benchmark of the fused BN(+add)+ReLU kernels on ResNet-101 layer shapes vs the ATen
path (F.batch_norm + add + relu under the same bf16 channels-last inputs). CUDA events, L2
flushed between iterations, achieved bytes/s against MEASURED_PEAKS.json hbm_gbs."""
import json
import os
import sys

import torch
import torch.nn as nn
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import mpi_operator_b200.ops.fused_bn as ops  # noqa: E402

SHAPES = [(64, 64, 112, 112, False), (64, 64, 56, 56, False), (64, 256, 56, 56, True), (64, 128, 28, 28, False),
          (64, 512, 28, 28, True), (64, 256, 14, 14, False), (64, 1024, 14, 14, True), (64, 512, 7, 7, False), (64, 2048, 7, 7, True)]


def timeit(fn, flush, iters=10):
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


def main():
    peak = 3350.0   # H100 SXM data sheet (HBM3); MEASURED_PEAKS.json overrides with a measured figure
    try:
        peak = json.load(open(os.path.join(os.path.dirname(__file__), "..", "MEASURED_PEAKS.json")))["hbm_gbs"]
    except Exception:
        pass
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    rows = []
    sel = os.environ.get("BN_SHAPES")
    shapes = [SHAPES[int(i)] for i in sel.split(",")] if sel else SHAPES
    for n, c, h, w, res in shapes:
        bn = nn.BatchNorm2d(c).cuda()
        x = torch.randn(n, c, h, w, device="cuda").to(torch.bfloat16).contiguous(memory_format=torch.channels_last).requires_grad_(True)
        r = torch.randn_like(x).requires_grad_(True) if res else None
        dz = torch.randn_like(x)
        T = x.numel() * 2

        def fwd_bwd():
            z = ops.bn_act(bn, x, residual=r, relu=True)
            z.backward(dz)
            x.grad = None
            if r is not None:
                r.grad = None
        out = {}
        for fused in (True, False):
            ops._ENABLED = fused
            out[fused] = timeit(fwd_bwd, flush)
        ops._ENABLED = True
        # minimal traffic of the fused design: fwd stats T + apply (2T [+T res]) ; bwd reduce 2T + elemt (3T [+T dres]) ; masks ~T/8
        min_bytes = T * (8 + (2 if res else 0)) + T / 8
        rows.append({"shape": [n, c, h, w], "residual": res, "fused_ms": out[True], "aten_ms": out[False], "speedup": out[False] / out[True],
                     "fused_gbs_on_min_traffic": min_bytes / out[True] / 1e6, "frac_of_measured_hbm": min_bytes / out[True] / 1e6 / peak})
        print(f"{(n, c, h, w)} res={res}: fused {out[True]*1e3:7.1f} us  aten {out[False]*1e3:7.1f} us  x{out[False]/out[True]:.2f}  "
              f"{min_bytes/out[True]/1e6:7.0f} GB/s ({100*min_bytes/out[True]/1e6/peak:.0f}% of HBM peak)", flush=True)
    if len(sys.argv) > 1:
        json.dump({"hbm_gbs_measured": peak, "rows": rows}, open(sys.argv[1], "w"), indent=1)


if __name__ == "__main__":
    main()
