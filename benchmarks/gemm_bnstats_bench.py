"""Micro-benchmark of the wgmma 1x1-convolution GEMM with BatchNorm statistics in its epilogue (csrc/kernels/gemm_bnstats.cu)
on the 1x1 layers of ResNet-101 at batch 64, against what the default path does for the same work: cuBLAS/cuDNN GEMM (torch.matmul
on the same [M,K] x [N,K]^T bf16 operands) followed by the BN statistics pass of bn_act.cu's forward (re-reads Y from HBM).

CUDA events, L2 flushed between iterations (a 256 MiB buffer is rewritten), median of `--iters`. Roofline: the op is memory
bound for these shapes (K <= 2048: >= 1 byte moved per ~K flops), so each row reports achieved bytes/s — X + W + Y once — against
`hbm_gbs`, plus TFLOP/s against `bf16_tflops`: the H100 SXM data-sheet figures (3.35 TB/s, 989 dense bf16 TFLOP/s) unless
MEASURED_PEAKS.json supplies measured ones. Numerics are checked in tests/test_zz_gemm_bnstats_gpu.py.

    python benchmarks/gemm_bnstats_bench.py --out profiles/gemm_bnstats_bench.json
"""
import argparse
import json
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from mpi_operator_b200.ops import gemm_bnstats  # noqa: E402

# (M = 64 * H * W, K = Cin, N = Cout) of the stride-1 1x1 convolutions of ResNet-101's four stages
SHAPES = [(64 * 56 * 56, 64, 64), (64 * 56 * 56, 64, 256), (64 * 56 * 56, 256, 64), (64 * 28 * 28, 256, 128), (64 * 28 * 28, 128, 512),
          (64 * 28 * 28, 512, 128), (64 * 14 * 14, 512, 256), (64 * 14 * 14, 256, 1024), (64 * 14 * 14, 1024, 256),
          (64 * 7 * 7, 1024, 512), (64 * 7 * 7, 512, 2048), (64 * 7 * 7, 2048, 512)]


def timeit(fn, flush, iters):
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
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default="")
    a = ap.parse_args()
    peaks = {"hbm_gbs": 3350.0, "bf16_tflops": 989.0}
    try:
        peaks.update(json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "MEASURED_PEAKS.json"))))
    except Exception:
        pass
    dev = torch.device("cuda")
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    rows = []
    for m, k, n in SHAPES:
        if not gemm_bnstats.supported(m, n, k):
            rows.append({"M": m, "K": k, "N": n, "skipped": "unsupported shape"})
            continue
        x = torch.randn(m, k, device=dev, dtype=torch.bfloat16)
        w = torch.randn(n, k, device=dev, dtype=torch.bfloat16) * (k ** -0.5)

        def ours():
            return gemm_bnstats.gemm_bnstats_raw(x, w)

        def library():
            y = x @ w.t()
            yf = y.float()
            return y, yf.sum(0), (yf * yf).sum(0)      # stand-in for the separate statistics pass (reads Y again)

        def library_gemm_only():
            return x @ w.t()
        t_ours, t_lib, t_gemm = timeit(ours, flush, a.iters), timeit(library, flush, a.iters), timeit(library_gemm_only, flush, a.iters)
        nbytes = 2 * (m * k + n * k + m * n)
        flops = 2.0 * m * n * k
        rows.append({"M": m, "K": k, "N": n, "ours_us": round(1e3 * t_ours, 1), "cublas_gemm_us": round(1e3 * t_gemm, 1),
                     "cublas_gemm_plus_stats_us": round(1e3 * t_lib, 1), "speedup_vs_gemm_plus_stats": round(t_lib / t_ours, 2),
                     "ours_gbs": round(nbytes / t_ours / 1e6, 1), "ours_frac_hbm": round(nbytes / t_ours / 1e6 / peaks["hbm_gbs"], 3),
                     "ours_tflops": round(flops / t_ours / 1e9, 1), "ours_frac_bf16_peak": round(flops / t_ours / 1e9 / peaks["bf16_tflops"], 3)})
        print(json.dumps(rows[-1]), flush=True)
    out = {"peaks": {k_: peaks[k_] for k_ in ("hbm_gbs", "bf16_tflops")}, "l2": "256 MiB buffer rewritten between iterations",
           "iters": a.iters, "rows": rows}
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
