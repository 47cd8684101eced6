"""Fused BatchNorm(+residual)+ReLU autograd op over csrc/kernels/bn_act.cu.

``bn_act(bn_module, x, residual=None, relu=True)`` computes
``relu(batch_norm(x) [+ residual])`` with the module's parameters and running
statistics. The fused kernels run when x is a CUDA bf16 channels-last tensor in
training mode with a supported channel count; anything else (CPU, eval, fp32)
takes the plain PyTorch path, so models stay runnable everywhere and
``state_dict`` layout is untouched.
"""
from __future__ import annotations

import os

import torch
import torch.nn.functional as F


def _lib():
    from ..runtime import _lib as L
    return L.lib()


_ENABLED = os.environ.get("B200MPI_FUSED_BN", "1") != "0"


def fused_bn_available(x: torch.Tensor, bn: torch.nn.BatchNorm2d) -> bool:
    if not (_ENABLED and x.is_cuda and x.dtype == torch.bfloat16 and x.dim() == 4 and bn.training and bn.affine
            and bn.track_running_stats and bn.momentum is not None):
        return False
    n, c, h, w = x.shape
    return bool(_lib().b200mpi_bn_supported(n * h * w, c)) and x.is_contiguous(memory_format=torch.channels_last)


_WS_CACHE = {}
_LAUNCHES = 0   # kernels of this module launched so far (each fused call = 3: stats/reduce, finalize, apply/elemt)


def launch_count() -> int:
    return _LAUNCHES


# ``num_batches_tracked`` bookkeeping: one 1-element add kernel per BN layer per step (104 launches for ResNet-101). Inside
# ``defer_counters()`` the fused ops only collect the counters; the caller bumps them all with one multi-tensor add.
_DEFERRED_COUNTERS = None


class defer_counters:
    """``with defer_counters() as pending: out = model(x)`` then ``torch._foreach_add_(pending, 1)``."""

    def __enter__(self):
        global _DEFERRED_COUNTERS
        self._prev = _DEFERRED_COUNTERS
        _DEFERRED_COUNTERS = []
        return _DEFERRED_COUNTERS

    def __exit__(self, *exc):
        global _DEFERRED_COUNTERS
        _DEFERRED_COUNTERS = self._prev
        return False


def _count_batch(bn: torch.nn.BatchNorm2d) -> None:
    if bn.num_batches_tracked is None:
        return
    if _DEFERRED_COUNTERS is not None:
        _DEFERRED_COUNTERS.append(bn.num_batches_tracked)
    else:
        bn.num_batches_tracked.add_(1)


def _ws(bn: torch.nn.BatchNorm2d, device) -> torch.Tensor:
    """Scratch for per-CTA partial sums + per-channel coefficients. BN kernels of one stream run
    back to back, so one buffer per (device, stream) is shared by every layer (sized for the widest)."""
    key = (device.index, torch.cuda.current_stream(device).cuda_stream)
    need = int(_lib().b200mpi_bn_workspace_floats(bn.num_features))
    ws = _WS_CACHE.get(key)
    if ws is None or ws.numel() < need:
        ws = torch.zeros(max(need, int(_lib().b200mpi_bn_workspace_floats(2048))), dtype=torch.float32, device=device)
        _WS_CACHE[key] = ws
    return ws


def _ptr(t):
    return t.data_ptr() if t is not None else None


def _never():
    return False


class _BNAct(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, residual, weight, bias, running_mean, running_var, ws, eps, momentum, relu, direct):
        n, c, h, w = x.shape
        m = n * h * w
        y = torch.empty_like(x, memory_format=torch.channels_last)
        mask = torch.empty(m * c // 8, dtype=torch.uint8, device=x.device) if relu else None
        save_mean = torch.empty(c, dtype=torch.float32, device=x.device)
        save_invstd = torch.empty(c, dtype=torch.float32, device=x.device)
        stream = torch.cuda.current_stream(x.device).cuda_stream
        rc = _lib().b200mpi_bn_act_fwd(x.data_ptr(), _ptr(residual), y.data_ptr(), _ptr(mask), weight.data_ptr(), bias.data_ptr(),
                                       running_mean.data_ptr(), running_var.data_ptr(), save_mean.data_ptr(), save_invstd.data_ptr(),
                                       ws.data_ptr(), m, c, eps, momentum, int(relu), stream)
        if rc != 0:
            raise RuntimeError(f"b200mpi_bn_act_fwd failed ({rc})")
        global _LAUNCHES
        _LAUNCHES += 3
        ctx.save_for_backward(x, mask, weight, save_mean, save_invstd, ws)
        ctx.relu, ctx.has_res = relu, residual is not None
        ctx.direct, ctx.wb = direct, (weight, bias)
        return y

    @staticmethod
    def backward(ctx, dz):
        x, mask, weight, save_mean, save_invstd, ws = ctx.saved_tensors
        n, c, h, w = x.shape
        m = n * h * w
        if dz.dtype != torch.bfloat16 or not dz.is_contiguous(memory_format=torch.channels_last):
            dz = dz.to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
        dx = torch.empty_like(x, memory_format=torch.channels_last)
        dres = torch.empty_like(x, memory_format=torch.channels_last) if ctx.has_res else None
        direct = (ctx.direct is not None and ctx.wb[0].grad is not None and ctx.wb[1].grad is not None
                  and not getattr(ctx.direct, "accumulating", _never)())  # no_sync(): grads must add up, not overwrite
        if direct:
            # the trainer owns pre-zeroed flat gradient views: write dgamma/dbeta straight into them and
            # skip autograd's AccumulateGrad add kernels (2 tiny launches per BN layer per step)
            dw, db = ctx.wb[0].grad, ctx.wb[1].grad
        else:
            dw = torch.empty(c, dtype=torch.float32, device=x.device)
            db = torch.empty(c, dtype=torch.float32, device=x.device)
        stream = torch.cuda.current_stream(x.device).cuda_stream
        rc = _lib().b200mpi_bn_act_bwd(dz.data_ptr(), x.data_ptr(), _ptr(mask), dx.data_ptr(), _ptr(dres), weight.data_ptr(),
                                       save_mean.data_ptr(), save_invstd.data_ptr(), dw.data_ptr(), db.data_ptr(), ws.data_ptr(),
                                       m, c, int(ctx.relu), stream)
        if rc != 0:
            raise RuntimeError(f"b200mpi_bn_act_bwd failed ({rc})")
        global _LAUNCHES
        _LAUNCHES += 3
        if direct:
            ctx.direct(ctx.wb[0])
            ctx.direct(ctx.wb[1])
            return dx, dres, None, None, None, None, None, None, None, None, None
        return dx, dres, dw, db, None, None, None, None, None, None, None


def bn_act(bn: torch.nn.BatchNorm2d, x: torch.Tensor, residual: torch.Tensor = None, relu: bool = True) -> torch.Tensor:
    if fused_bn_available(x, bn) and (residual is None or (residual.dtype == torch.bfloat16 and residual.shape == x.shape)):
        if residual is not None and not residual.is_contiguous(memory_format=torch.channels_last):
            residual = residual.contiguous(memory_format=torch.channels_last)
        _count_batch(bn)
        return _BNAct.apply(x, residual, bn.weight, bn.bias, bn.running_mean, bn.running_var, _ws(bn, x.device), bn.eps,
                            bn.momentum, relu, getattr(bn, "_b200_grad_ready", None))
    out = bn(x)
    if residual is not None:
        out = out + residual
    return F.relu(out) if relu else out


# --------------------------------------------------------------------------------------------------------------
# 1x1 convolution + BatchNorm(+residual)+ReLU with the BN statistics taken in the GEMM epilogue
# (csrc/kernels/gemm_bnstats.cu: TMA + wgmma). On by default (numerics: tests/test_zz_gemm_bnstats_gpu.py);
# B200MPI_FUSED_CONV1X1=0 keeps cuDNN for the 1x1 convolutions.
# Forward = 3 launches (GEMM+stats, finalize, apply) instead of conv + 3; backward = the fused BN backward kernels + two
# library GEMMs (dgrad, wgrad).
_CONV1X1 = os.environ.get("B200MPI_FUSED_CONV1X1", "1") == "1"


def _conv1x1_eligible(conv: torch.nn.Conv2d, bn: torch.nn.BatchNorm2d, x: torch.Tensor) -> bool:
    if not (conv.kernel_size == (1, 1) and conv.stride == (1, 1) and conv.padding == (0, 0) and conv.dilation == (1, 1)
            and conv.groups == 1 and conv.bias is None and x.is_cuda and x.dim() == 4 and x.dtype == torch.bfloat16
            and x.is_contiguous(memory_format=torch.channels_last) and bn.training and bn.affine and bn.track_running_stats
            and bn.momentum is not None and _ENABLED):
        return False
    from . import gemm_bnstats
    n, c, h, w = x.shape
    return (gemm_bnstats.supported(n * h * w, conv.out_channels, c)
            and bool(_lib().b200mpi_bn_supported(n * h * w, conv.out_channels)))


class _Conv1x1BNAct(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, residual, w2d, weight, bias, running_mean, running_var, ws, eps, momentum, relu, direct):
        from . import gemm_bnstats
        n, cin, h, w = x.shape
        cout = w2d.shape[0]
        m = n * h * w
        x2d = x.permute(0, 2, 3, 1).reshape(m, cin)      # a view: channels-last memory is [M, Cin] row-major
        yconv, partials, parts = gemm_bnstats.gemm_bnstats_raw(x2d, w2d)
        z = torch.empty((n, cout, h, w), dtype=torch.bfloat16, device=x.device, memory_format=torch.channels_last)
        mask = torch.empty(m * cout // 8, dtype=torch.uint8, device=x.device) if relu else None
        save_mean = torch.empty(cout, dtype=torch.float32, device=x.device)
        save_invstd = torch.empty(cout, dtype=torch.float32, device=x.device)
        stream = torch.cuda.current_stream(x.device).cuda_stream
        rc = _lib().b200mpi_bn_act_fwd_prestats(yconv.data_ptr(), _ptr(residual), z.data_ptr(), _ptr(mask), weight.data_ptr(),
                                                bias.data_ptr(), running_mean.data_ptr(), running_var.data_ptr(),
                                                save_mean.data_ptr(), save_invstd.data_ptr(), ws.data_ptr(), partials.data_ptr(),
                                                parts, m, cout, eps, momentum, int(relu), stream)
        if rc != 0:
            raise RuntimeError(f"b200mpi_bn_act_fwd_prestats failed ({rc})")
        global _LAUNCHES
        _LAUNCHES += 3   # GEMM+stats, finalize, apply
        ctx.save_for_backward(x2d, w2d, yconv, mask, weight, save_mean, save_invstd, ws)
        ctx.relu, ctx.has_res, ctx.shape = relu, residual is not None, (n, cin, cout, h, w)
        ctx.direct, ctx.wb = direct, (weight, bias)
        return z

    @staticmethod
    def backward(ctx, dz):
        x2d, w2d, yconv, mask, weight, save_mean, save_invstd, ws = ctx.saved_tensors
        n, cin, cout, h, w = ctx.shape
        m = n * h * w
        if dz.dtype != torch.bfloat16 or not dz.is_contiguous(memory_format=torch.channels_last):
            dz = dz.to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
        dy = torch.empty(m, cout, dtype=torch.bfloat16, device=dz.device)          # gradient w.r.t. the convolution output
        dres = torch.empty_like(dz, memory_format=torch.channels_last) if ctx.has_res else None
        direct = (ctx.direct is not None and ctx.wb[0].grad is not None and ctx.wb[1].grad is not None
                  and not getattr(ctx.direct, "accumulating", _never)())
        if direct:
            dw, db = ctx.wb[0].grad, ctx.wb[1].grad
        else:
            dw = torch.empty(cout, dtype=torch.float32, device=dz.device)
            db = torch.empty(cout, dtype=torch.float32, device=dz.device)
        stream = torch.cuda.current_stream(dz.device).cuda_stream
        rc = _lib().b200mpi_bn_act_bwd(dz.data_ptr(), yconv.data_ptr(), _ptr(mask), dy.data_ptr(), _ptr(dres), weight.data_ptr(),
                                       save_mean.data_ptr(), save_invstd.data_ptr(), dw.data_ptr(), db.data_ptr(), ws.data_ptr(),
                                       m, cout, int(ctx.relu), stream)
        if rc != 0:
            raise RuntimeError(f"b200mpi_bn_act_bwd failed ({rc})")
        global _LAUNCHES
        _LAUNCHES += 3
        dx = (dy @ w2d).view(n, h, w, cin).permute(0, 3, 1, 2) if ctx.needs_input_grad[0] else None   # dgrad: [M,Cout] x [Cout,Cin]
        dw2d = dy.t() @ x2d if ctx.needs_input_grad[2] else None                                          # wgrad: [Cout,M] x [M,Cin]
        if direct:
            ctx.direct(ctx.wb[0])
            ctx.direct(ctx.wb[1])
            return dx, dres, dw2d, None, None, None, None, None, None, None, None, None
        return dx, dres, dw2d, dw, db, None, None, None, None, None, None, None


def conv_bn_act(conv: torch.nn.Conv2d, bn: torch.nn.BatchNorm2d, x: torch.Tensor, residual: torch.Tensor = None,
                relu: bool = True) -> torch.Tensor:
    """``relu(bn(conv(x)) [+ residual])``. With B200MPI_FUSED_CONV1X1=1 an eligible 1x1 stride-1 convolution runs on the
    wgmma GEMM whose epilogue already produces the BatchNorm statistics; everything else is ``bn_act(bn, conv(x), ...)``."""
    if (_CONV1X1 and _conv1x1_eligible(conv, bn, x)
            and (residual is None or (residual.dtype == torch.bfloat16 and residual.shape[0] == x.shape[0]
                                      and residual.shape[1] == conv.out_channels and residual.shape[2:] == x.shape[2:]))):
        if residual is not None and not residual.is_contiguous(memory_format=torch.channels_last):
            residual = residual.contiguous(memory_format=torch.channels_last)
        _count_batch(bn)
        w2d = conv.weight.to(torch.bfloat16).reshape(conv.out_channels, conv.in_channels)
        return _Conv1x1BNAct.apply(x, residual, w2d, bn.weight, bn.bias, bn.running_mean, bn.running_var, _ws(bn, x.device), bn.eps,
                                   bn.momentum, relu, getattr(bn, "_b200_grad_ready", None))
    return bn_act(bn, conv(x), residual=residual, relu=relu)
