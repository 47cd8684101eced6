"""Python front-end of the wgmma 1x1-convolution GEMM with fused BatchNorm statistics
(csrc/kernels/gemm_bnstats.cu -> lib/libb200mpi_gemm.so).

    y, partials, parts = gemm_bnstats_raw(x, weight)       # partial rows of plain sums
    y, partials, parts = gemm_bnstats_shifted(x, weight)   # the kernel's own rows, as BatchNorm merges them
    y = gemm_bn_eval(x, weight, bn, residual, relu)        # eval mode: BatchNorm with running statistics in the epilogue

``x``: channels-last bf16 activations viewed as [M = N*H*W, Cin]; ``weight``: the convolution weight [Cout, Cin]
(``conv.weight.view(Cout, Cin)``) in bf16. Both return the bf16 output [M, Cout] and ``parts`` rows of per-channel sums of
that output (fp32), i.e. what BatchNorm's statistics pass would compute by re-reading ``y`` from HBM. Partial row p covers
the 128-row tiles p, p + parts, ... of ``y``.

The kernel shifts row p by a value of its own column, ``y[128 p]``: it holds ``sum (y - y[128 p])`` and
``sum (y - y[128 p])^2``, which keep the variance when |mean| >> std. ``b200mpi_bn_act_fwd_prestats`` merges those rows
(ops/fused_bn.py). ``gemm_bnstats_raw`` converts them to plain ``sum y`` and ``sum y^2`` in float64, for callers that
want the sums themselves.

The kernel is compiled for sm_90a (H100); ops/fused_bn.py calls it for eligible 1x1 convolutions. The reference ships no
kernels (SURVEY.md §2.2)."""
from __future__ import annotations

import ctypes as C
from pathlib import Path
from typing import Tuple

import torch

LIB_PATH = Path(__file__).resolve().parent.parent / "lib" / "libb200mpi_gemm.so"
_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        if not LIB_PATH.exists():
            raise RuntimeError(f"{LIB_PATH} is missing; run `make` (or __graft_entry__.build())")
        L = C.CDLL(str(LIB_PATH))
        L.b200mpi_gemm_bnstats_supported.argtypes = [C.c_longlong, C.c_int, C.c_int]
        L.b200mpi_gemm_bnstats_partial_floats.argtypes = [C.c_int]
        L.b200mpi_gemm_bnstats_partial_floats.restype = C.c_size_t
        L.b200mpi_gemm_bnstats_walk_rows.argtypes = [C.c_int, C.c_int, C.c_longlong]
        L.b200mpi_gemm_bnstats_walk_rows.restype = C.c_longlong
        L.b200mpi_gemm_bnstats.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int), C.c_longlong,
                                           C.c_int, C.c_int, C.c_void_p]
        L.b200mpi_gemm_dgrad_res_supported.argtypes = [C.c_longlong, C.c_int, C.c_int]
        L.b200mpi_gemm_bn_eval_supported.argtypes = [C.c_longlong, C.c_int, C.c_int]
        L.b200mpi_gemm_bn_eval.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                           C.c_void_p, C.c_float, C.c_int, C.c_longlong, C.c_int, C.c_int, C.c_void_p]
        L.b200mpi_gemm_dgrad_res.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p,
                                             C.c_void_p, C.c_void_p, C.POINTER(C.c_int), C.c_longlong, C.c_int, C.c_int, C.c_void_p]
        _lib = L
    return _lib


def supported(m: int, n: int, k: int) -> bool:
    return bool(lib().b200mpi_gemm_bnstats_supported(m, n, k))


def gemm_bnstats_shifted(x: torch.Tensor, weight: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor, int]:
    """Runs the kernel; returns (y [M,N] bf16, partials [parts, N, 2] fp32, parts). Row p holds {sum (y - y[128 p]),
    sum (y - y[128 p])^2} over the rows of the tiles p, p + parts, ... (csrc/kernels/gemm_bnstats_logic.h)."""
    if x.dtype != torch.bfloat16 or weight.dtype != torch.bfloat16 or not x.is_cuda:
        raise ValueError("gemm_bnstats needs CUDA bf16 tensors")
    if x.dim() != 2 or weight.dim() != 2 or x.shape[1] != weight.shape[1] or not x.is_contiguous() or not weight.is_contiguous():
        raise ValueError("expected contiguous x [M,K] and weight [N,K]")
    m, k = x.shape
    n = weight.shape[0]
    if not supported(m, n, k):
        raise ValueError(f"unsupported shape M={m} N={n} K={k} (N, K multiples of 64)")
    y = torch.empty(m, n, dtype=torch.bfloat16, device=x.device)
    # the kernel writes every one of the `parts` rows it reports: no memset needed
    partials = torch.empty(int(lib().b200mpi_gemm_bnstats_partial_floats(n)), dtype=torch.float32, device=x.device)
    parts = C.c_int(0)
    rc = lib().b200mpi_gemm_bnstats(x.data_ptr(), weight.data_ptr(), y.data_ptr(), partials.data_ptr(), C.byref(parts), m, n, k,
                                    torch.cuda.current_stream(x.device).cuda_stream)
    if rc != 0:
        raise RuntimeError(f"b200mpi_gemm_bnstats failed ({rc})")
    return y, partials[:parts.value * 2 * n].view(parts.value, n, 2), parts.value


def walk_rows(m: int, parts: int) -> list:
    """Rows of y that each partial row covers: the 128-row tiles p, p + parts, ..., the last tile holding the rest of M
    (the kernel's own rule, walk_rows in csrc/kernels/gemm_bnstats_logic.h)."""
    return [int(lib().b200mpi_gemm_bnstats_walk_rows(p, parts, m)) for p in range(parts)]


def gemm_bnstats_raw(x: torch.Tensor, weight: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor, int]:
    """Runs the kernel; returns (y [M,N] bf16, partials [parts, N, 2] fp32, parts) with row p = {sum y, sum y^2} over the
    rows that partial row covers. The kernel's shifted rows are moved to plain sums in float64, then rounded to fp32."""
    y, partials, parts = gemm_bnstats_shifted(x, weight)
    k = y[0:(parts - 1) * 128 + 1:128].double()                                   # each row's shift y[128 p]
    n = torch.tensor(walk_rows(x.shape[0], parts), dtype=torch.float64, device=y.device)[:, None]
    a1, a2 = partials[..., 0].double(), partials[..., 1].double()
    partials.copy_(torch.stack([a1 + n * k, a2 + k * (2 * a1 + n * k)], -1))
    return y, partials, parts


def dgrad_res_supported(m: int, n: int, k: int) -> bool:
    return bool(lib().b200mpi_gemm_dgrad_res_supported(m, n, k))


def dgrad_residual(dy: torch.Tensor, wt: torch.Tensor, r: torch.Tensor, mask: torch.Tensor, below=None):
    """``dy [M,K] @ wt[N,K]^T + mask ⊙ r`` in one kernel (fp32 sum, one bf16 rounding): the input gradient of a 1x1
    convolution plus the residual gradient of the same tensor. ``wt`` is the weight transposed to [Cin, Cout], ``r`` a
    contiguous bf16 [M,N] tensor and ``mask`` its ReLU mask, one bit per element ([M, N/8] uint8, bit c%8 of byte c/8).

    Without ``below`` returns dx [M,N]. With ``below = (xb, maskb, mean_b)`` — the saved input [M,N] bf16, ReLU mask and
    saved mean [N] fp32 of the BatchNorm that produced the convolution's input — returns (dx, partials [parts, N, 2],
    parts): that BN's backward reduction (sum g, sum g * (xb - mean_b), g = maskb ⊙ dx) for bn_act_bwd_prestats."""
    if not (dy.is_cuda and dy.dtype == wt.dtype == r.dtype == torch.bfloat16 and mask.dtype == torch.uint8):
        raise ValueError("dgrad_residual needs CUDA bf16 dy, wt, r and a uint8 mask")
    m, k = dy.shape
    n = wt.shape[0]
    if (wt.shape[1] != k or r.shape != (m, n) or mask.numel() != m * n // 8 or not dy.is_contiguous() or not wt.is_contiguous()
            or not r.is_contiguous() or not mask.is_contiguous()):
        raise ValueError("expected contiguous dy [M,K], wt [N,K], r [M,N] and mask [M*N/8]")
    if not dgrad_res_supported(m, n, k):
        raise ValueError(f"unsupported shape M={m} N={n} K={k} (N multiple of 128, K of 64)")
    dx = torch.empty(m, n, dtype=torch.bfloat16, device=dy.device)
    xb = maskb = mean_b = partials = None
    if below is not None:
        xb, maskb, mean_b = below
        if not (xb.dtype == torch.bfloat16 and xb.numel() == m * n and xb.is_contiguous() and maskb.dtype == torch.uint8
                and maskb.numel() == m * n // 8 and maskb.is_contiguous() and mean_b.dtype == torch.float32 and mean_b.numel() == n):
            raise ValueError("below = (xb [M,N] bf16, maskb [M*N/8] uint8, mean_b [N] fp32), contiguous")
        partials = torch.empty(int(lib().b200mpi_gemm_bnstats_partial_floats(n)), dtype=torch.float32, device=dy.device)
    parts = C.c_int(0)
    p = lambda t: t.data_ptr() if t is not None else None  # noqa: E731
    rc = lib().b200mpi_gemm_dgrad_res(dy.data_ptr(), wt.data_ptr(), dx.data_ptr(), r.data_ptr(), mask.data_ptr(), p(xb), p(maskb),
                                      p(mean_b), p(partials), C.byref(parts), m, n, k, torch.cuda.current_stream(dy.device).cuda_stream)
    if rc != 0:
        raise RuntimeError(f"b200mpi_gemm_dgrad_res failed ({rc})")
    if below is None:
        return dx
    return dx, partials[:parts.value * 2 * n].view(parts.value, n, 2), parts.value


def bn_eval_supported(m: int, n: int, k: int) -> bool:
    return bool(lib().b200mpi_gemm_bn_eval_supported(m, n, k))


def gemm_bn_eval(x: torch.Tensor, weight: torch.Tensor, bn: torch.nn.BatchNorm2d, residual: torch.Tensor = None,
                 relu: bool = True) -> torch.Tensor:
    """``relu?(bn(x @ weight^T) [+ residual])`` with ``bn`` in eval mode, in one kernel: the epilogue applies
    ``a = gamma * rsqrt(running_var + eps)``, ``b = beta - running_mean * a`` per column to the fp32 accumulator, adds the
    residual and rounds to bf16 once. ``x`` [M,K], ``weight`` [N,K] and ``residual`` [M,N] are contiguous CUDA bf16; the
    module's parameters and running statistics are fp32 and only read. Returns y [M,N] bf16."""
    if not (x.is_cuda and x.dtype == weight.dtype == torch.bfloat16):
        raise ValueError("gemm_bn_eval needs CUDA bf16 x and weight")
    if x.dim() != 2 or weight.dim() != 2 or x.shape[1] != weight.shape[1] or not x.is_contiguous() or not weight.is_contiguous():
        raise ValueError("expected contiguous x [M,K] and weight [N,K]")
    m, k = x.shape
    n = weight.shape[0]
    if residual is not None and not (residual.dtype == torch.bfloat16 and residual.shape == (m, n) and residual.is_contiguous()):
        raise ValueError("residual: contiguous bf16 [M,N]")
    stats = [t for t in (bn.weight, bn.bias, bn.running_mean, bn.running_var) if t is not None]
    if (bn.running_mean is None or bn.running_var is None
            or any(t.dtype != torch.float32 or t.numel() != n or not t.is_contiguous() or t.device != x.device for t in stats)):
        raise ValueError("bn: fp32 contiguous parameters and running statistics of N channels on x's device")
    if not bn_eval_supported(m, n, k):
        raise ValueError(f"unsupported shape M={m} N={n} K={k} (M >= 128, N and K multiples of 64)")
    y = torch.empty(m, n, dtype=torch.bfloat16, device=x.device)
    p = lambda t: t.data_ptr() if t is not None else None  # noqa: E731
    rc = lib().b200mpi_gemm_bn_eval(x.data_ptr(), weight.data_ptr(), y.data_ptr(), p(residual), p(bn.weight), p(bn.bias),
                                    bn.running_mean.data_ptr(), bn.running_var.data_ptr(), float(bn.eps), int(relu), m, n, k,
                                    torch.cuda.current_stream(x.device).cuda_stream)
    if rc != 0:
        raise RuntimeError(f"b200mpi_gemm_bn_eval failed ({rc})")
    return y
