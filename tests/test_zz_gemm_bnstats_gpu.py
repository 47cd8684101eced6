"""wgmma GEMM + fused BN statistics (csrc/kernels/gemm_bnstats.cu) against a plain PyTorch fp32 reference.

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

CASE = r"""
import sys, torch
sys.path.insert(0, {repo!r})
from mpi_operator_b200.ops.gemm_bnstats import gemm_bnstats_raw
M, N, K = {m}, {n}, {k}
torch.manual_seed(0)
x = (torch.randn(M, K, device="cuda") * 0.5).to(torch.bfloat16)
w = (torch.randn(N, K, device="cuda") * 0.1).to(torch.bfloat16)
y, partials, parts = gemm_bnstats_raw(x, w)
torch.cuda.synchronize()
ref = x.float() @ w.float().t()
err = (y.float() - ref).abs().max().item()
tol = 2e-2 * ref.abs().max().item() + 1e-2
assert err <= tol, ("gemm", err, tol)
yb = y.float()
s1, s2 = partials.sum(0)[:, 0], partials.sum(0)[:, 1]
e1 = (s1 - yb.sum(0)).abs().max().item()
e2 = (s2 - (yb * yb).sum(0)).abs().max().item()
assert e1 <= 1e-3 * yb.abs().sum(0).max().item() + 1e-2, ("sum", e1)
assert e2 <= 1e-3 * (yb * yb).sum(0).max().item() + 1e-2, ("sumsq", e2)
print("OK", M, N, K, "parts", parts, "max err", err)
"""


@pytest.mark.parametrize("m,n,k", [(128, 64, 64), (256, 128, 64), (1000, 128, 256), (4096, 256, 64), (12544, 512, 128),
                                   (200704, 256, 64), (50176, 2048, 512)])
def test_gemm_bnstats_matches_fp32_reference(m, n, k):
    r = subprocess.run([sys.executable, "-c", CASE.format(repo=REPO, m=m, n=n, k=k)], capture_output=True, text=True, timeout=180)
    assert r.returncode == 0 and "OK" in r.stdout, r.stdout[-1500:] + r.stderr[-3000:]


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
