"""The residual hand-over of ops/fused_bn.py to the wgmma dgrad with the residual-gradient epilogue
(csrc/kernels/gemm_bnstats.cu, b200mpi_gemm_dgrad_res) in whole bottleneck blocks: fused vs B200MPI_FUSED_CONV1X1_BWD off
vs fp32, plus the cases that must keep autograd's add (downsample, accumulation) or sum extra gradients (a second consumer). The
kernel itself is checked bit for bit against float64 in test_zz_gemm_exact_gpu.py.

Each case runs in a subprocess, like test_zz_gemm_bnstats_gpu.py, so that a trap in the kernel cannot poison the CUDA context
of the test session. B200MPI_SKIP_GEMM_TESTS=1 skips the file."""
import os
import subprocess
import sys

import pytest

pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(os.environ.get("B200MPI_SKIP_GEMM_TESTS") == "1", reason="B200MPI_SKIP_GEMM_TESTS=1")]

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _run(src):
    r = subprocess.run([sys.executable, "-c", src], capture_output=True, text=True, timeout=300)
    assert r.returncode == 0 and "OK" in r.stdout, r.stdout[-1500:] + r.stderr[-3000:]


BLOCK_CASE = r"""
import copy, sys, torch, torch.nn as nn
sys.path.insert(0, {repo!r})
from mpi_operator_b200.ops import fused_bn, gemm_bnstats
from mpi_operator_b200.models.resnet import Bottleneck, _Downsample
assert fused_bn._CONV1X1
calls = [0]
_orig = gemm_bnstats.dgrad_residual
def counting(*a, **kw):
    calls[0] += 1
    return _orig(*a, **kw)
gemm_bnstats.dgrad_residual = counting
L = fused_bn._lib()
pre_calls = [0]
_orig_pre = L.b200mpi_bn_act_bwd_prestats
def counting_pre(*a):
    pre_calls[0] += 1
    return _orig_pre(*a)
L.b200mpi_bn_act_bwd_prestats = counting_pre

class Accumulating:          # a trainer's grad-ready hook inside no_sync(): gradients must add up
    def __call__(self, p): pass
    def accumulating(self): return True

torch.manual_seed(0)
blocks = [Bottleneck(256, 64, downsample=_Downsample(256, 256, 1) if {downsample} else None)] + [Bottleneck(256, 64) for _ in range({nblocks} - 1)]
net = nn.Sequential(*blocks).cuda().to(memory_format=torch.channels_last)
for m in net.modules():       # non-trivial BN parameters (bn3 is not zero-initialised here)
    if isinstance(m, nn.BatchNorm2d):
        nn.init.uniform_(m.weight, 0.5, 1.5); nn.init.uniform_(m.bias, -0.2, 0.2)
    if {accumulate} and isinstance(m, nn.BatchNorm2d):
        m._b200_grad_ready = Accumulating()
x0 = torch.randn(8, 256, 14, 14, device="cuda").to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
g = torch.randn(8, 256, 14, 14, device="cuda").to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
g2 = torch.randn_like(g)

def run(model, fused_bwd, dtype):
    fused_bn._CONV1X1_BWD = fused_bwd
    x = x0.to(dtype).detach().requires_grad_()
    with torch.autocast("cuda", dtype=torch.bfloat16, enabled=dtype == torch.bfloat16):
        h = model[0](x)
        out = model[1:](h) if len(model) > 1 else h
        loss = (out.float() * g.float()).sum()
        if {extra_consumer}:   # the output of block 0 also feeds the loss directly
            loss = loss + (h.float() * g2.float()).sum()
    loss.backward()
    return [x.grad] + [p.grad for p in model.parameters()]

net_off, net_ref = copy.deepcopy(net), copy.deepcopy(net).float()
got = run(net, True, torch.bfloat16)
n_fused, n_pre = calls[0], pre_calls[0]
off = run(net_off, False, torch.bfloat16)
assert calls[0] == n_fused and pre_calls[0] == n_pre, "the switch did not turn the fused backward off"
ref = run(net_ref, True, torch.float32)    # fp32 tensors: plain PyTorch everywhere
expect = 0 if {accumulate} else {nblocks} - (1 if {downsample} else 0)
assert n_fused == expect, ("fused dgrads", n_fused, expect)
# a block's bn3 skips its reduce pass when the next block's dgrad took the partials of exactly the gradient it receives
expect_pre = 0 if {accumulate} else {nblocks} - 1 - (1 if {extra_consumer} else 0)
assert n_pre == expect_pre, ("bn backward from handed-over partials", n_pre, expect_pre)
names = ["x"] + [n for n, _ in net.named_parameters()]
def dist(a, b):
    return (a.float() - b.float()).abs().max().item()
for name, a, b, r in zip(names, got, off, ref):
    s = r.float().abs().max().item()
    assert dist(a, b) <= 3e-2 * s + 1e-3, ("fused vs off", name, dist(a, b), s)
    # against fp32 the fused path (one rounding of dY.W + residual) is no worse than autograd's add (two roundings)
    assert dist(a, r) <= 1.25 * dist(b, r) + 1e-2 * s + 1e-3, ("fused vs fp32", name, dist(a, r), dist(b, r), s)
print("OK fused dgrads", n_fused, "prestats", n_pre)
"""


@pytest.mark.parametrize("nblocks,downsample,extra_consumer,accumulate", [
    (1, False, False, False),      # one bottleneck
    (3, False, False, False),      # a 3-block stack: hand-over in every block
    (3, True, False, False),       # first block has a downsample: no hand-over there
    (3, False, True, False),       # block 0's output has a second consumer: its bn3 must reduce the summed gradient
    (3, False, False, True),       # gradient accumulation keeps autograd's add
])
def test_bottleneck_residual_handover_matches_reference(nblocks, downsample, extra_consumer, accumulate):
    _run(BLOCK_CASE.format(repo=REPO, nblocks=nblocks, downsample=downsample, extra_consumer=extra_consumer, accumulate=accumulate))
