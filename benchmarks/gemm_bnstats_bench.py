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


# conv1 data gradients of ResNet-101's residual blocks without downsample, with the residual gradient added in the epilogue:
# (M, K = planes, N = 4 * planes, blocks per step)
DGRAD_SHAPES = [(64 * 56 * 56, 64, 256, 2), (64 * 28 * 28, 128, 512, 3), (64 * 14 * 14, 256, 1024, 22), (64 * 7 * 7, 512, 2048, 2)]


def dgrad_bytes_removed(m: int, n: int) -> int:
    """HBM bytes per block that the residual epilogue removes. Before: bn3's backward writes dres = mask ⊙ dv (T), the
    library dgrad writes its output (T), autograd's add reads both and writes the sum (3T). After: the kernel reads dv (T)
    and the mask (T/16) and writes the sum (T). T = one bf16 [M, N] tensor."""
    t = 2 * m * n
    return 5 * t - (2 * t + t // 16)


def eval_bytes(m: int, k: int, n: int, fused: bool) -> int:
    """HBM bytes of an eval-mode 1x1 conv + BN + residual + ReLU. Fused: X, W, R read, Y written once. Library GEMM + the eval
    kernel: the GEMM writes Y, the eval kernel reads it back with R and writes the output: two more [M, N] passes."""
    x, w, t = 2 * m * k, 2 * n * k, 2 * m * n
    return x + w + 2 * t + (0 if fused else 2 * t)


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
            return gemm_bnstats.gemm_bnstats_shifted(x, w)

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
    dgrad_rows, removed = [], 0
    for m, k, n, blocks in DGRAD_SHAPES:
        dy = torch.randn(m, k, device=dev, dtype=torch.bfloat16)
        w2d = torch.randn(k, n, device=dev, dtype=torch.bfloat16) * (k ** -0.5)     # conv1 weight [Cout = planes, Cin]
        dv = torch.randn(m, n, device=dev, dtype=torch.bfloat16)
        mask = torch.randint(0, 256, (m * n // 8,), dtype=torch.uint8, device=dev)
        dres = torch.randn(m, n, device=dev, dtype=torch.bfloat16)

        def ours_dgrad():      # includes the per-step transposed copy of the weight
            return gemm_bnstats.dgrad_residual(dy, w2d.t().contiguous(), dv, mask)

        def library_dgrad():   # cuBLAS dgrad + autograd's add of the residual gradient bn3's backward wrote
            return (dy @ w2d) + dres
        t_ours, t_lib = timeit(ours_dgrad, flush, a.iters), timeit(library_dgrad, flush, a.iters)
        removed += blocks * dgrad_bytes_removed(m, n)
        nbytes = 2 * (m * k + k * n + 2 * m * n) + m * n // 8
        dgrad_rows.append({"M": m, "K": k, "N": n, "blocks": blocks, "ours_us": round(1e3 * t_ours, 1),
                           "cublas_dgrad_plus_add_us": round(1e3 * t_lib, 1), "speedup": round(t_lib / t_ours, 2),
                           "ours_gbs": round(nbytes / t_ours / 1e6, 1), "step_bytes_removed": blocks * dgrad_bytes_removed(m, n)})
        print(json.dumps(dgrad_rows[-1]), flush=True)
    print(json.dumps({"dgrad_residual_bytes_removed_per_step": removed}), flush=True)
    # eval epilogue: conv + BatchNorm (running statistics) + residual + ReLU in the GEMM, against cuBLAS + the one-pass eval kernel
    from mpi_operator_b200.runtime import _lib
    eval_rows = []
    for m, k, n in SHAPES:
        x = torch.randn(m, k, device=dev, dtype=torch.bfloat16)
        w = torch.randn(n, k, device=dev, dtype=torch.bfloat16) * (k ** -0.5)
        r = torch.randn(m, n, device=dev, dtype=torch.bfloat16)
        bn = torch.nn.BatchNorm2d(n).to(dev).eval()
        z = torch.empty(m, n, device=dev, dtype=torch.bfloat16)

        def ours_eval():
            return gemm_bnstats.gemm_bn_eval(x, w, bn, r, True)

        def library_eval():
            y = x @ w.t()
            rc = _lib.lib().b200mpi_bn_act_eval(y.data_ptr(), r.data_ptr(), z.data_ptr(), bn.weight.data_ptr(), bn.bias.data_ptr(),
                                                bn.running_mean.data_ptr(), bn.running_var.data_ptr(), m, n, bn.eps, 1,
                                                torch.cuda.current_stream().cuda_stream)
            assert rc == 0, rc
            return z
        t_ours, t_lib = timeit(ours_eval, flush, a.iters), timeit(library_eval, flush, a.iters)
        b_ours, b_lib = eval_bytes(m, k, n, True), eval_bytes(m, k, n, False)
        eval_rows.append({"M": m, "K": k, "N": n, "ours_us": round(1e3 * t_ours, 1), "cublas_plus_eval_kernel_us": round(1e3 * t_lib, 1),
                          "speedup": round(t_lib / t_ours, 2), "ours_bytes": b_ours, "library_bytes": b_lib,
                          "ours_gbs": round(b_ours / t_ours / 1e6, 1), "ours_frac_hbm": round(b_ours / t_ours / 1e6 / peaks["hbm_gbs"], 3)})
        print(json.dumps(eval_rows[-1]), flush=True)
    out = {"peaks": {k_: peaks[k_] for k_ in ("hbm_gbs", "bf16_tflops")}, "l2": "256 MiB buffer rewritten between iterations",
           "iters": a.iters, "rows": rows, "dgrad_rows": dgrad_rows, "dgrad_residual_bytes_removed_per_step": removed,
           "eval_rows": eval_rows, "card": torch.cuda.get_device_name(0)}
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
