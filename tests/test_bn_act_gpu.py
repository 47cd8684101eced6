"""Fused BN(+residual)+ReLU kernels (csrc/kernels/bn_act.cu) vs a plain PyTorch fp32 reference."""
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _ref(x, res, bn, relu):
    y = F.batch_norm(x.float(), None, None, bn.weight, bn.bias, True, 0.0, bn.eps)
    if res is not None:
        y = y + res.float()
    return F.relu(y) if relu else y


@pytest.mark.parametrize("shape", [(4, 64, 9, 7), (8, 256, 14, 14), (3, 2048, 7, 7), (2, 8, 5, 5), (16, 128, 28, 28), (1, 512, 1, 3)])
@pytest.mark.parametrize("relu,use_res", [(True, False), (True, True), (False, False)])
def test_bn_act_forward_backward_matches_fp32_reference(shape, relu, use_res):
    from mpi_operator_b200.ops.fused_bn import bn_act, fused_bn_available
    torch.manual_seed(sum(shape))
    n, c, h, w = shape
    bn = nn.BatchNorm2d(c).cuda()
    with torch.no_grad():
        bn.weight.uniform_(0.5, 1.5)
        bn.bias.uniform_(-0.5, 0.5)
    x = (torch.randn(shape, device="cuda") * 2 + 3).to(torch.bfloat16).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    res = (torch.randn(shape, device="cuda").to(torch.bfloat16).contiguous(memory_format=torch.channels_last).requires_grad_(True)
           if use_res else None)
    assert fused_bn_available(x, bn)
    z = bn_act(bn, x, residual=res, relu=relu)
    assert z.dtype == torch.bfloat16 and z.is_contiguous(memory_format=torch.channels_last)
    dz = torch.randn(shape, device="cuda").to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    z.backward(dz)
    # reference in fp32 on the same bf16-rounded inputs
    bn_ref = nn.BatchNorm2d(c).cuda()
    bn_ref.load_state_dict({k: v for k, v in bn.state_dict().items() if k in ("weight", "bias")}, strict=False)
    xr = x.detach().float().requires_grad_(True)
    rr = res.detach().float().requires_grad_(True) if use_res else None
    zr = _ref(xr, rr, bn_ref, relu)
    zr.backward(dz.float())
    tol = dict(rtol=2e-2, atol=3e-2)
    torch.testing.assert_close(z.float(), zr, **tol)
    torch.testing.assert_close(x.grad.float(), xr.grad, rtol=3e-2, atol=3e-2)
    if use_res:
        torch.testing.assert_close(res.grad.float(), rr.grad, **tol)
    m = n * h * w
    scale = max(1.0, m ** 0.5)
    torch.testing.assert_close(bn.weight.grad, bn_ref.weight.grad, rtol=2e-2, atol=2e-2 * scale)
    torch.testing.assert_close(bn.bias.grad, bn_ref.bias.grad, rtol=2e-2, atol=2e-2 * scale)
    # running statistics follow nn.BatchNorm2d (momentum 0.1, unbiased variance)
    mean = x.detach().float().mean((0, 2, 3))
    var = x.detach().float().var((0, 2, 3), unbiased=m > 1)
    torch.testing.assert_close(bn.running_mean, 0.1 * mean, rtol=1e-3, atol=1e-3)
    torch.testing.assert_close(bn.running_var, 0.9 + 0.1 * var, rtol=2e-3, atol=2e-3)
    assert int(bn.num_batches_tracked) == 1


def test_bn_act_statistics_robust_to_large_mean():
    """|mean| >> std: the shifted accumulation must not lose the variance."""
    from mpi_operator_b200.ops.fused_bn import bn_act
    bn = nn.BatchNorm2d(64).cuda()
    x = (torch.randn(32, 64, 16, 16, device="cuda") * 0.5 + 200.0).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    z = bn_act(bn, x, relu=False)
    xf = x.float()
    want = (xf - xf.mean((0, 2, 3), keepdim=True)) / torch.sqrt(xf.var((0, 2, 3), unbiased=False, keepdim=True) + bn.eps)
    torch.testing.assert_close(z.float(), want, rtol=3e-2, atol=3e-2)


def test_bn_act_repeated_calls_and_cuda_graph():
    """The op can be called repeatedly and replayed inside a CUDA graph. Every CTA writes its own partial row and a fixed
    merge order adds them up, so repeated results are bitwise equal."""
    from mpi_operator_b200.ops.fused_bn import bn_act
    bn = nn.BatchNorm2d(256).cuda()
    x = torch.randn(8, 256, 14, 14, device="cuda").to(torch.bfloat16).contiguous(memory_format=torch.channels_last).requires_grad_(True)
    outs, grads = [], []
    for _ in range(3):
        x.grad = None
        z = bn_act(bn, x)
        z.float().sum().backward()
        outs.append(z.detach().clone())
        grads.append(x.grad.clone())
    assert torch.equal(outs[0], outs[1]) and torch.equal(outs[1], outs[2])
    assert torch.equal(grads[0], grads[1]) and torch.equal(grads[1], grads[2])
    g = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        static = torch.empty_like(outs[0])
        with torch.cuda.graph(g):
            static.copy_(bn_act(bn, x.detach()))
    g.replay()
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(static, outs[0])


def test_resnet_block_fused_matches_unfused(monkeypatch):
    from mpi_operator_b200.models.resnet import Bottleneck
    import mpi_operator_b200.ops.fused_bn as ops
    torch.manual_seed(0)
    blk = Bottleneck(256, 64).cuda().to(memory_format=torch.channels_last)
    x = torch.randn(8, 256, 14, 14, device="cuda").contiguous(memory_format=torch.channels_last)
    outs = {}
    for fused in (True, False):
        monkeypatch.setattr(ops, "_ENABLED", fused)
        b = Bottleneck(256, 64).cuda().to(memory_format=torch.channels_last)
        b.load_state_dict(blk.state_dict())
        with torch.autocast("cuda", dtype=torch.bfloat16):
            y = b(x)
        y.float().pow(2).mean().backward()
        outs[fused] = (y.detach().float(), b.conv1.weight.grad.clone(), b.bn3.weight.grad.clone())
    torch.testing.assert_close(outs[True][0], outs[False][0], rtol=5e-2, atol=5e-2)
    torch.testing.assert_close(outs[True][1], outs[False][1], rtol=1e-1, atol=2e-3)
    torch.testing.assert_close(outs[True][2], outs[False][2], rtol=1e-1, atol=2e-2)
