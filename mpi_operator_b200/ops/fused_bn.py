"""Fused BatchNorm(+residual)+ReLU autograd op over csrc/kernels/bn_act.cu.

``bn_act(bn_module, x, residual=None, relu=True)`` computes
``relu(batch_norm(x) [+ residual])`` with the module's parameters and running
statistics. The fused kernels run when x is a CUDA bf16 channels-last tensor with
a supported channel count, in training mode, or in eval mode when the module uses
its running statistics and no autograd graph is recorded (one kernel per layer,
``b200mpi_bn_act_eval``); anything else (CPU, fp32, eval with autograd) takes the
plain PyTorch path, so models stay runnable everywhere and ``state_dict`` layout
is untouched.
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
    # one value per channel: training-mode batch norm is undefined, and nn.BatchNorm2d's error should reach the caller
    if n * h * w < 2:
        return False
    # the kernels move 16-byte vectors: a view at an odd storage offset takes the PyTorch path
    return (bool(_lib().b200mpi_bn_supported(n * h * w, c)) and x.is_contiguous(memory_format=torch.channels_last)
            and x.data_ptr() % 16 == 0)


def _eval_bn_ready(bn: torch.nn.BatchNorm2d, *inputs) -> bool:
    """Eval mode with running statistics (PyTorch would use batch statistics otherwise) and nothing for autograd to record:
    BatchNorm is a fixed per-channel affine map, which the eval kernels apply."""
    if not (_ENABLED and not bn.training and bn.track_running_stats and bn.running_mean is not None
            and bn.running_var is not None):
        return False
    params = (bn.weight, bn.bias)
    if torch.is_grad_enabled() and any(t is not None and t.requires_grad for t in inputs + params):
        return False
    return all(t is None or (t.is_cuda and t.dtype == torch.float32 and t.is_contiguous())
               for t in params + (bn.running_mean, bn.running_var))


def _eval_input_ok(x: torch.Tensor, bn: torch.nn.BatchNorm2d) -> bool:
    if not (x.is_cuda and x.dtype == torch.bfloat16 and x.dim() == 4 and x.shape[1] == bn.num_features
            and x.is_contiguous(memory_format=torch.channels_last) and x.data_ptr() % 16 == 0):
        return False
    n, c, h, w = x.shape
    return n * h * w >= 1 and bool(_lib().b200mpi_bn_supported(n * h * w, c))


def _bn_eval(bn: torch.nn.BatchNorm2d, x: torch.Tensor, residual, relu: bool) -> torch.Tensor:
    n, c, h, w = x.shape
    y = torch.empty_like(x, memory_format=torch.channels_last)
    rc = _lib().b200mpi_bn_act_eval(x.data_ptr(), _ptr(residual), y.data_ptr(), _ptr(bn.weight), _ptr(bn.bias),
                                    bn.running_mean.data_ptr(), bn.running_var.data_ptr(), n * h * w, c, bn.eps, int(relu),
                                    torch.cuda.current_stream(x.device).cuda_stream)
    if rc != 0:
        raise RuntimeError(f"b200mpi_bn_act_eval failed ({rc})")
    global _LAUNCHES
    _LAUNCHES += 1
    return y


def _residual_cl(residual: torch.Tensor):
    if residual is not None and not residual.is_contiguous(memory_format=torch.channels_last):
        residual = residual.contiguous(memory_format=torch.channels_last)
    return residual


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
        if dz.data_ptr() % 16:
            dz = dz.clone(memory_format=torch.channels_last)
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
    if (_eval_bn_ready(bn, x, residual) and _eval_input_ok(x, bn)
            and (residual is None or (residual.dtype == torch.bfloat16 and residual.shape == x.shape))):
        residual = _residual_cl(residual)
        if residual is None or residual.data_ptr() % 16 == 0:
            return _bn_eval(bn, x, residual, relu)
    if fused_bn_available(x, bn) and (residual is None or (residual.dtype == torch.bfloat16 and residual.shape == x.shape)):
        residual = _residual_cl(residual)
        if residual is None or residual.data_ptr() % 16 == 0:
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
# library GEMMs (dgrad, wgrad), except for the residual hand-over below.
_CONV1X1 = os.environ.get("B200MPI_FUSED_CONV1X1", "1") == "1"
# In a residual block without downsample the block input x feeds both conv1 and the residual add, so autograd sums its two
# gradients with an add kernel (read two tensors, write one) after bn3's backward has written mask3 ⊙ dv (dv = gradient of
# the block output) as a tensor of its own. Through a ResidualLink, bn3's backward hands (dv, mask3) to conv1's node
# instead, whose dgrad then runs on the wgmma kernel with mask3 ⊙ dv added in its epilogue: ~3 tensor passes less per block.
# When x is itself the output of a fused conv+BN+ReLU (the previous block's bn3), the same epilogue also takes that BN's
# backward reduction over the gradient it writes; the previous block's backward then skips its reduce pass (one tensor pass
# less), provided the gradient it receives is that very tensor, unmodified.
# B200MPI_FUSED_CONV1X1_BWD=0 keeps the autograd add and the reduce pass (A/B runs).
_CONV1X1_BWD = os.environ.get("B200MPI_FUSED_CONV1X1_BWD", "1") == "1"


class ResidualLink:
    """Joins the conv3 node of a residual block (the one that adds the residual x) to the conv1 node that reads the same x.
    conv1's fused forward arms it; conv3's backward fills ``dv`` / ``mask``; conv1's backward consumes them."""
    __slots__ = ("armed", "dv", "mask")

    def __init__(self):
        self.armed, self.dv, self.mask = False, None, None


class _HandedPartials:
    """BN-backward partial rows taken by a later dgrad epilogue, and the identity of the gradient tensor they describe
    (storage, version counter, shape, strides): the BN's backward may use them only for that exact tensor."""
    __slots__ = ("partials", "parts", "key")

    def __init__(self):
        self.partials, self.parts, self.key = None, 0, None


def _grad_key(t: torch.Tensor):
    return (t.data_ptr(), t._version, tuple(t.shape), t.stride(), t.dtype)


def _conv1x1_geometry(conv: torch.nn.Conv2d, x: torch.Tensor) -> bool:
    return (conv.kernel_size == (1, 1) and conv.stride == (1, 1) and conv.padding == (0, 0) and conv.dilation == (1, 1)
            and conv.groups == 1 and conv.bias is None and x.is_cuda and x.dim() == 4 and x.dtype == torch.bfloat16
            and x.is_contiguous(memory_format=torch.channels_last))


def _conv1x1_eligible(conv: torch.nn.Conv2d, bn: torch.nn.BatchNorm2d, x: torch.Tensor) -> bool:
    if not (_conv1x1_geometry(conv, x) and bn.training and bn.affine and bn.track_running_stats
            and bn.momentum is not None and _ENABLED):
        return False
    from . import gemm_bnstats
    n, c, h, w = x.shape
    return (gemm_bnstats.supported(n * h * w, conv.out_channels, c)
            and bool(_lib().b200mpi_bn_supported(n * h * w, conv.out_channels)))


class _Conv1x1BNAct(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, residual, w2d, weight, bias, running_mean, running_var, ws, eps, momentum, relu, direct, link):
        from . import gemm_bnstats
        n, cin, h, w = x.shape
        cout = w2d.shape[0]
        m = n * h * w
        x2d = x.permute(0, 2, 3, 1).reshape(m, cin)      # a view: channels-last memory is [M, Cin] row-major
        yconv, partials, parts = gemm_bnstats.gemm_bnstats_shifted(x2d, w2d)
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
        ctx.direct, ctx.wb, ctx.link = direct, (weight, bias), link
        # what the next fused 1x1 node needs to take this BN's backward reduction in its dgrad epilogue
        ctx.handed = _HandedPartials() if residual is not None and relu and _CONV1X1_BWD else None
        if ctx.handed is not None:
            z._b200_bn_below = (yconv, mask, save_mean, ctx.handed)
        below = getattr(x, "_b200_bn_below", None) if link is not None and residual is None else None
        ctx.below = below if below is not None and below[0].shape == (m, cin) else None
        return z

    @staticmethod
    def backward(ctx, dz):
        x2d, w2d, yconv, mask, weight, save_mean, save_invstd, ws = ctx.saved_tensors
        n, cin, cout, h, w = ctx.shape
        m = n * h * w
        # this BN's reduction, if the next block's dgrad took it over exactly the gradient that arrives here
        pre = None
        if ctx.handed is not None and ctx.handed.partials is not None:
            if ctx.handed.key == _grad_key(dz):
                pre = (ctx.handed.partials, ctx.handed.parts)
            ctx.handed.partials = None
        if dz.dtype != torch.bfloat16 or not dz.is_contiguous(memory_format=torch.channels_last):
            dz = dz.to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
        if dz.data_ptr() % 16:
            dz = dz.clone(memory_format=torch.channels_last)
        dy = torch.empty(m, cout, dtype=torch.bfloat16, device=dz.device)          # gradient w.r.t. the convolution output
        accumulating = ctx.direct is not None and getattr(ctx.direct, "accumulating", _never)()
        # residual side of a link: the residual gradient mask ⊙ dz goes to conv1's dgrad epilogue, not to autograd
        hand_over = (ctx.link is not None and ctx.has_res and ctx.relu and ctx.needs_input_grad[1] and not accumulating
                     and dz.data_ptr() % 16 == 0)
        dres = torch.empty_like(dz, memory_format=torch.channels_last) if ctx.has_res and not hand_over else None
        direct = (ctx.direct is not None and ctx.wb[0].grad is not None and ctx.wb[1].grad is not None and not accumulating)
        if direct:
            dw, db = ctx.wb[0].grad, ctx.wb[1].grad
        else:
            dw = torch.empty(cout, dtype=torch.float32, device=dz.device)
            db = torch.empty(cout, dtype=torch.float32, device=dz.device)
        stream = torch.cuda.current_stream(dz.device).cuda_stream
        global _LAUNCHES
        if pre is not None:
            rc = _lib().b200mpi_bn_act_bwd_prestats(dz.data_ptr(), yconv.data_ptr(), _ptr(mask), dy.data_ptr(), _ptr(dres),
                                                    weight.data_ptr(), save_mean.data_ptr(), save_invstd.data_ptr(), dw.data_ptr(),
                                                    db.data_ptr(), ws.data_ptr(), pre[0].data_ptr(), pre[1], m, cout, int(ctx.relu),
                                                    stream)
            _LAUNCHES += 2
        else:
            rc = _lib().b200mpi_bn_act_bwd(dz.data_ptr(), yconv.data_ptr(), _ptr(mask), dy.data_ptr(), _ptr(dres), weight.data_ptr(),
                                           save_mean.data_ptr(), save_invstd.data_ptr(), dw.data_ptr(), db.data_ptr(), ws.data_ptr(),
                                           m, cout, int(ctx.relu), stream)
            _LAUNCHES += 3
        if rc != 0:
            raise RuntimeError(f"b200mpi_bn_act_bwd{'_prestats' if pre is not None else ''} failed ({rc})")
        if hand_over:
            ctx.link.dv, ctx.link.mask = dz, mask
        # input side of a link: the residual gradient of x, if the block's conv3 node handed it over
        dv, mask_v = (ctx.link.dv, ctx.link.mask) if ctx.link is not None and not ctx.has_res else (None, None)
        if dv is not None:
            ctx.link.dv = ctx.link.mask = None
        dx = None
        if ctx.needs_input_grad[0] and dv is not None:
            from . import gemm_bnstats
            # W^T [Cin, Cout] is the K-major B operand of the kernel: a per-step copy of the (small) 1x1 weight
            wt, dv2d = w2d.t().contiguous(), dv.permute(0, 2, 3, 1).reshape(m, cin)
            if ctx.below is not None:
                yb, mb, meanb, handed = ctx.below
                dx, partials, parts = gemm_bnstats.dgrad_residual(dy, wt, dv2d, mask_v, below=(yb, mb, meanb))
                dx = dx.view(n, h, w, cin).permute(0, 3, 1, 2)
                handed.partials, handed.parts, handed.key = partials, parts, _grad_key(dx)
            else:
                dx = gemm_bnstats.dgrad_residual(dy, wt, dv2d, mask_v).view(n, h, w, cin).permute(0, 3, 1, 2)
            _LAUNCHES += 1
        elif ctx.needs_input_grad[0]:
            dx = (dy @ w2d).view(n, h, w, cin).permute(0, 3, 1, 2)                    # dgrad: [M,Cout] x [Cout,Cin]
        dw2d = dy.t() @ x2d if ctx.needs_input_grad[2] else None                      # wgrad: [Cout,M] x [M,Cin]
        if direct:
            ctx.direct(ctx.wb[0])
            ctx.direct(ctx.wb[1])
            return dx, dres, dw2d, None, None, None, None, None, None, None, None, None, None
        return dx, dres, dw2d, dw, db, None, None, None, None, None, None, None, None


def conv_bn_act(conv: torch.nn.Conv2d, bn: torch.nn.BatchNorm2d, x: torch.Tensor, residual: torch.Tensor = None,
                relu: bool = True, link: ResidualLink = None) -> torch.Tensor:
    """``relu(bn(conv(x)) [+ residual])``. With B200MPI_FUSED_CONV1X1=1 an eligible 1x1 stride-1 convolution runs on the
    wgmma GEMM whose epilogue already produces the BatchNorm statistics; everything else is ``bn_act(bn, conv(x), ...)``.
    In eval mode without autograd (``_eval_bn_ready``) the same GEMM applies the BatchNorm with its running statistics, the
    residual and the ReLU in its epilogue instead: one kernel for the whole layer (M >= 128).

    ``link``: one ResidualLink per residual block whose residual is the input of its first 1x1 convolution, passed to both
    that call (``residual=None``: the link is armed if the fused dgrad can take the hand-over) and the call that adds the
    residual (it hands the residual gradient over only to an armed link)."""
    if (_CONV1X1 and _conv1x1_eligible(conv, bn, x)
            and (residual is None or (residual.dtype == torch.bfloat16 and residual.shape[0] == x.shape[0]
                                      and residual.shape[1] == conv.out_channels and residual.shape[2:] == x.shape[2:]))):
        residual = _residual_cl(residual)
        _count_batch(bn)
        w2d = conv.weight.to(torch.bfloat16).reshape(conv.out_channels, conv.in_channels)
        if link is not None and residual is None:
            from . import gemm_bnstats
            n, cin, h, w = x.shape
            link.armed = _CONV1X1_BWD and gemm_bnstats.dgrad_res_supported(n * h * w, cin, conv.out_channels)
        if link is not None and not link.armed:
            link = None
        return _Conv1x1BNAct.apply(x, residual, w2d, bn.weight, bn.bias, bn.running_mean, bn.running_var, _ws(bn, x.device), bn.eps,
                                   bn.momentum, relu, getattr(bn, "_b200_grad_ready", None), link)
    if _CONV1X1 and _conv1x1_geometry(conv, x) and _eval_bn_ready(bn, x, residual, conv.weight):
        from . import gemm_bnstats
        n, cin, h, w = x.shape
        cout = conv.out_channels
        if (gemm_bnstats.bn_eval_supported(n * h * w, cout, cin) and bn.num_features == cout and x.data_ptr() % 16 == 0
                and (residual is None or (residual.dtype == torch.bfloat16 and residual.shape == (n, cout, h, w)))):
            residual = _residual_cl(residual)
            res2d = residual.permute(0, 2, 3, 1).reshape(n * h * w, cout) if residual is not None else None
            if res2d is None or res2d.data_ptr() % 16 == 0:
                w2d = conv.weight.to(torch.bfloat16).reshape(cout, cin)
                y = gemm_bnstats.gemm_bn_eval(x.permute(0, 2, 3, 1).reshape(n * h * w, cin), w2d, bn, res2d, relu)
                global _LAUNCHES
                _LAUNCHES += 1
                return y.view(n, h, w, cout).permute(0, 3, 1, 2)
    return bn_act(bn, conv(x), residual=residual, relu=relu)
