"""The fused 1x1 conv + BN + ReLU layer on the wgmma GEMM with fused BN statistics (csrc/kernels/gemm_bnstats.cu) against
a plain PyTorch reference. The kernel itself is checked bit for bit against float64 in test_zz_gemm_exact_gpu.py.

Each case runs in a subprocess so that a trap in
the kernel (every wait is bounded and traps) cannot poison the CUDA context of the test session; the file sorts last for the
same reason. B200MPI_SKIP_GEMM_TESTS=1 skips the file."""
import os
import subprocess
import sys

import pytest

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(os.environ.get("B200MPI_SKIP_GEMM_TESTS") == "1", reason="B200MPI_SKIP_GEMM_TESTS=1")]

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

LAYER_CASE = r"""
import os, sys, copy, torch, torch.nn as nn
os.environ["B200MPI_FUSED_CONV1X1"] = "1"
sys.path.insert(0, {repo!r})
from mpi_operator_b200.ops import fused_bn
assert fused_bn._CONV1X1
torch.manual_seed(0)
N, CIN, COUT, H = {n}, {cin}, {cout}, {h}
conv = nn.Conv2d(CIN, COUT, 1, bias=False).cuda().to(memory_format=torch.channels_last)
bn = nn.BatchNorm2d(COUT).cuda()
conv_r, bn_r = copy.deepcopy(conv), copy.deepcopy(bn)
x = torch.randn(N, CIN, H, H, device="cuda").to(torch.bfloat16).contiguous(memory_format=torch.channels_last).requires_grad_()
res = torch.randn(N, COUT, H, H, device="cuda").to(torch.bfloat16).contiguous(memory_format=torch.channels_last).requires_grad_()
xr, rr = x.detach().clone().requires_grad_(), res.detach().clone().requires_grad_()
with torch.autocast("cuda", dtype=torch.bfloat16):
    z = fused_bn.conv_bn_act(conv, bn, x, residual=res if {use_res} else None)
    assert type(z.grad_fn).__name__.startswith("_Conv1x1BNAct"), type(z.grad_fn).__name__
    # reference: fp32 batch norm on the bf16 convolution output, same rounding points as the fused path
    yc = conv_r(xr)
    zr = torch.relu(nn.functional.batch_norm(yc.float(), None, None, bn_r.weight, bn_r.bias, True, 0.1, bn_r.eps)
                    + (rr.float() if {use_res} else 0)).to(torch.bfloat16)
g = torch.randn_like(z)
z.backward(g); zr.backward(g)
def close(a, b, what, tol=3e-2):
    d = (a.float() - b.float()).abs().max().item(); s = b.float().abs().max().item()
    assert d <= tol * s + tol, (what, d, s)
close(z, zr, "out"); close(x.grad, xr.grad, "dx"); close(conv.weight.grad, conv_r.weight.grad, "dW", 5e-2)
close(bn.weight.grad, bn_r.weight.grad, "dgamma", 5e-2); close(bn.bias.grad, bn_r.bias.grad, "dbeta", 5e-2)
if {use_res}: close(res.grad, rr.grad, "dres")
print("OK")
"""


@pytest.mark.parametrize("n,cin,cout,h,use_res", [(8, 64, 256, 14, True), (8, 256, 64, 14, False), (4, 512, 2048, 7, True)])
def test_conv1x1_bn_act_layer_matches_reference(n, cin, cout, h, use_res):
    src = LAYER_CASE.format(repo=REPO, n=n, cin=cin, cout=cout, h=h, use_res=use_res)
    r = subprocess.run([sys.executable, "-c", src], capture_output=True, text=True, timeout=180)
    assert r.returncode == 0 and "OK" in r.stdout, r.stdout[-1500:] + r.stderr[-3000:]
