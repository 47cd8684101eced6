"""Python front-end of the wgmma 1x1-convolution GEMM with fused BatchNorm statistics
(csrc/kernels/gemm_bnstats.cu -> lib/libb200mpi_gemm.so).

    y, s1, s2 = conv1x1_with_stats(x, weight)

``x``: channels-last bf16 activations viewed as [M = N*H*W, Cin]; ``weight``: the convolution weight [Cout, Cin]
(``conv.weight.view(Cout, Cin)``) in bf16. Returns the bf16 output [M, Cout] and the per-channel sum / sum of squares
of that output (fp32), i.e. what BatchNorm's statistics pass would compute by re-reading ``y`` from HBM.

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
        L.b200mpi_gemm_bnstats.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.POINTER(C.c_int), C.c_longlong,
                                           C.c_int, C.c_int, C.c_void_p]
        _lib = L
    return _lib


def supported(m: int, n: int, k: int) -> bool:
    return bool(lib().b200mpi_gemm_bnstats_supported(m, n, k))


def gemm_bnstats_raw(x: torch.Tensor, weight: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor, int]:
    """Runs the kernel; returns (y [M,N] bf16, partials [parts, N, 2] fp32, parts)."""
    if x.dtype != torch.bfloat16 or weight.dtype != torch.bfloat16 or not x.is_cuda:
        raise ValueError("gemm_bnstats needs CUDA bf16 tensors")
    if x.dim() != 2 or weight.dim() != 2 or x.shape[1] != weight.shape[1] or not x.is_contiguous() or not weight.is_contiguous():
        raise ValueError("expected contiguous x [M,K] and weight [N,K]")
    m, k = x.shape
    n = weight.shape[0]
    if not supported(m, n, k):
        raise ValueError(f"unsupported shape M={m} N={n} K={k} (N, K multiples of 64)")
    y = torch.empty(m, n, dtype=torch.bfloat16, device=x.device)
    partials = torch.zeros(int(lib().b200mpi_gemm_bnstats_partial_floats(n)), dtype=torch.float32, device=x.device)
    parts = C.c_int(0)
    rc = lib().b200mpi_gemm_bnstats(x.data_ptr(), weight.data_ptr(), y.data_ptr(), partials.data_ptr(), C.byref(parts), m, n, k,
                                    torch.cuda.current_stream(x.device).cuda_stream)
    if rc != 0:
        raise RuntimeError(f"b200mpi_gemm_bnstats failed ({rc})")
    return y, partials[:parts.value * 2 * n].view(parts.value, n, 2), parts.value


def conv1x1_with_stats(x: torch.Tensor, weight: torch.Tensor) -> Tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    y, partials, _ = gemm_bnstats_raw(x, weight)
    tot = partials.sum(0)
    return y, tot[:, 0].contiguous(), tot[:, 1].contiguous()
