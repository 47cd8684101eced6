"""Eval-mode BatchNorm on the fused kernels: the one-pass kernel ``b200mpi_bn_act_eval``, the wgmma 1x1-GEMM eval epilogue
``b200mpi_gemm_bn_eval``, their dispatch from ``bn_act`` / ``conv_bn_act``, whole ResNets in eval mode, and
``DataParallelTrainer.evaluate()`` under a CUDA graph.

References are float64 computations on the same bf16 operands, and the oracle of tests/bn_oracle.py: rsqrtf is not
correctly rounded, so per channel one of the fp32 values within 2 ulps of the correctly rounded rsqrt must reproduce the
kernel's whole column bit for bit. BatchNorm layers get random gamma / beta and running
statistics (mean ~ N(0, 1), var ~ U(0.1, 4)): ResNet zero-initialises bn3.weight, which would hide every error on the residual
branch. Each case runs in a subprocess, so that a trap in a kernel cannot poison the CUDA context of the test session."""
import os
import subprocess
import sys

import pytest

pytestmark = pytest.mark.gpu

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

PRELUDE = r"""
import os, sys, copy, ctypes, numpy as np, torch, torch.nn as nn
sys.path.insert(0, {repo!r})
sys.path.insert(0, os.path.join({repo!r}, "tests"))
import bn_oracle as O
from mpi_operator_b200.ops import fused_bn, gemm_bnstats
torch.manual_seed(0)
dev = torch.device("cuda")

def randomize_bn(bn):
    with torch.no_grad():
        c = bn.num_features
        if bn.weight is not None:
            bn.weight.copy_(torch.rand(c) + 0.5)
            bn.bias.copy_(torch.randn(c) * 0.5)
        if bn.running_mean is not None:
            bn.running_mean.copy_(torch.randn(c))
            bn.running_var.copy_(torch.rand(c) * 3.9 + 0.1)

def coef64(bn):
    a = bn.running_var.double().add(bn.eps).rsqrt()
    if bn.weight is not None:
        a = a * bn.weight.double()
    b = -bn.running_mean.double() * a
    if bn.bias is not None:
        b = b + bn.bias.double()
    return a, b

def coef_mag64(bn):
    # what the rounding errors of a, b scale with: |beta| + |running_mean * a|
    a, _ = coef64(bn)
    m = (bn.running_mean.double() * a).abs()
    return m + bn.bias.double().abs() if bn.bias is not None else m

def exact_columns(y, x, r, bn, relu, what):
    # rows [0, 2048) and the last 256: the eval kernels have no reduction, every row is computed alike
    M = x.shape[0]
    idx = torch.tensor(sorted(set(range(min(M, 2048))) | set(range(max(0, M - 256), M))), device=x.device)
    found = O.eval_match(O._bits(y[idx]), O.to_np(x[idx]), None if r is None else O.to_np(r[idx]), O.to_np(bn.weight),
                         O.to_np(bn.bias), O.to_np(bn.running_mean), O.to_np(bn.running_var), bn.eps, relu)
    bad = np.nonzero(np.abs(found) > 2)[0]
    assert bad.size == 0, (what, "no rsqrtf candidate reproduces channels", bad[:8].tolist())

def ulp(ref):
    # one bf16 ulp at |ref| (8 significant bits)
    e = torch.floor(torch.log2(ref.abs().clamp_min(1e-30)))
    return torch.exp2(e - 7)
"""


def _run(body, env=None, timeout=900, **fmt):
    code = PRELUDE.format(repo=REPO) + body.format(**fmt)
    r = subprocess.run([sys.executable, "-c", code], env={**os.environ, **(env or {})}, capture_output=True, text=True,
                       timeout=timeout)
    assert r.returncode == 0 and "OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
    return r.stdout


# ------------------------------------------------------------------------------------------------------- eval kernel --
KERNEL_CASE = r"""
C = {c}
bn = nn.BatchNorm2d(C).cuda().eval()
randomize_bn(bn)
# a training-mode call first, so that the BN workspace exists and can be checked for writes
xt = torch.randn(64, C, 2, 2, device=dev).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
bn.train(); fused_bn.bn_act(bn, xt); bn.eval()
torch.cuda.synchronize()
bufs = [t.clone() for t in (bn.running_mean, bn.running_var, bn.num_batches_tracked)]
ws = {{k: v.clone() for k, v in fused_bn._WS_CACHE.items()}}
a64, b64 = coef64(bn)
for M in (1, 7, 1000, 200704):
    x = (torch.randn(M, C, 1, 1, device=dev) * 2 + 0.5).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    r = torch.randn(M, C, 1, 1, device=dev).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    for use_res in (False, True):
        for relu in (False, True):
            n0 = fused_bn.launch_count()
            with torch.no_grad():
                z = fused_bn.bn_act(bn, x, residual=r if use_res else None, relu=relu)
            assert fused_bn.launch_count() == n0 + 1, "the eval kernel did not run"
            torch.cuda.synchronize()
            for lo in range(0, M, 1 << 16):
                hi = min(M, lo + (1 << 16))
                xs = x.reshape(M, C)[lo:hi].double()
                t = a64 * xs + b64
                mag = (a64 * xs).abs() + coef_mag64(bn)
                if use_res:
                    rs = r.reshape(M, C)[lo:hi].double()
                    t = t + rs
                    mag = mag + rs.abs()
                ref = t.clamp_min(0) if relu else t
                got = z.reshape(M, C)[lo:hi].double()
                # one bf16 ulp, plus fp32 rounding of a, b and the sum where ref is near a cancellation
                tol = ulp(ref) + 1e-6 * mag
                err = (got - ref).abs()
                assert bool((err <= tol).all()), ("value", C, M, use_res, relu, float((err - tol).max()))
                if relu:
                    assert bool((got >= 0).all())
                    neg = t < -1e-6 * mag
                    assert bool((got[neg] == 0).all()), ("zeros", C, M, use_res)
            exact_columns(z.reshape(M, C), x.reshape(M, C), r.reshape(M, C) if use_res else None, bn, relu,
                          ("kernel", C, M, use_res, relu))
for a, b in zip(bufs, (bn.running_mean, bn.running_var, bn.num_batches_tracked)):
    assert torch.equal(a, b), "running statistics changed"
assert all(torch.equal(ws[k], fused_bn._WS_CACHE[k]) for k in ws) and set(ws) == set(fused_bn._WS_CACHE), "workspace changed"
print("OK")
"""


@pytest.mark.parametrize("c", [8, 16, 32, 64, 128, 256, 512, 1024, 2048])
def test_bn_eval_kernel_matches_fp64(c):
    _run(KERNEL_CASE, c=c)


# --------------------------------------------------------------------------------------------- GEMM eval epilogue --
# (M, K = Cin, N = Cout) of ResNet-101's stride-1 1x1 convolutions at batch 64, a ragged M and a single row tile; then
# tile width 64 with several column blocks, 3 and 5 k-blocks, one CTA per column block (N = 8384: 131 blocks of 64) and
# fewer row tiles than m-groups (M = 129, 255)
GEMM_SHAPES = [(64 * 56 * 56, 64, 64), (64 * 56 * 56, 64, 256), (64 * 56 * 56, 256, 64), (64 * 28 * 28, 256, 128),
               (64 * 28 * 28, 128, 512), (64 * 28 * 28, 512, 128), (64 * 14 * 14, 512, 256), (64 * 14 * 14, 256, 1024),
               (64 * 14 * 14, 1024, 256), (64 * 7 * 7, 1024, 512), (64 * 7 * 7, 512, 2048), (64 * 7 * 7, 2048, 512),
               (1000, 256, 128), (1000, 64, 64), (128, 512, 2048),
               (129, 192, 192), (255, 320, 320), (1000, 128, 8384), (256, 2048, 192), (1000, 4096, 256)]

GEMM_CASE = r"""
M, K, N = {m}, {k}, {n}
L = gemm_bnstats.lib()
assert L.b200mpi_gemm_bn_eval_supported(M, N, K) == 1
bn = nn.BatchNorm2d(N).cuda().eval()
randomize_bn(bn)
a64, b64 = coef64(bn)
x = torch.randn(M, K, device=dev).to(torch.bfloat16)
w = (torch.randn(N, K, device=dev) * K ** -0.5).to(torch.bfloat16)
r = torch.randn(M, N, device=dev).to(torch.bfloat16)
acc = x.double() @ w.double().t()
mag = a64.abs() * (x.double().abs() @ w.double().abs().t())
stream = torch.cuda.current_stream().cuda_stream
for use_res in (False, True):
    for relu in (False, True):
        # Y has 128 guard rows past M, NaN-filled: the kernel must not write them
        yfull = torch.full((M + 128, N), float("nan"), device=dev, dtype=torch.bfloat16)
        rc = L.b200mpi_gemm_bn_eval(x.data_ptr(), w.data_ptr(), yfull.data_ptr(), r.data_ptr() if use_res else None,
                                    bn.weight.data_ptr(), bn.bias.data_ptr(), bn.running_mean.data_ptr(), bn.running_var.data_ptr(),
                                    bn.eps, int(relu), M, N, K, stream)
        assert rc == 0, rc
        torch.cuda.synchronize()
        assert bool(yfull[M:].isnan().all()), "rows past M written"
        t = a64 * acc + b64 + (r.double() if use_res else 0)
        ref = t.clamp_min(0) if relu else t
        got = yfull[:M].double()
        tol = ulp(ref) + 1e-5 * mag + 1e-6 * (coef_mag64(bn) + (r.double().abs() if use_res else 0))
        err = (got - ref).abs()
        assert bool((err <= tol).all()), ("value", use_res, relu, float((err - tol).max()), int((err > tol).sum()))
        # the Python wrapper gives the same bits
        y2 = gemm_bnstats.gemm_bn_eval(x, w, bn, r if use_res else None, relu)
        assert torch.equal(y2, yfull[:M])
# argument checks: misaligned pointers and unsupported shapes are refused
assert L.b200mpi_gemm_bn_eval(x.data_ptr() + 2, w.data_ptr(), yfull.data_ptr(), None, None, None, bn.running_mean.data_ptr(),
                              bn.running_var.data_ptr(), bn.eps, 1, M, N, K, stream) != 0
assert L.b200mpi_gemm_bn_eval_supported(127, N, K) == 0 and L.b200mpi_gemm_bn_eval_supported(M, N + 8, K) == 0
print("OK")
"""


@pytest.mark.parametrize("m,k,n", GEMM_SHAPES)
def test_gemm_bn_eval_epilogue_matches_fp64(m, k, n):
    _run(GEMM_CASE, m=m, k=k, n=n)


# The epilogue on gemm_oracle's family E: the fp32 accumulator is exact, so a * acc + b (+ r) is checked bit for bit with the
# candidate rsqrtf; tile widths 128 and 64 (N = 192), and a full ResNet-101 layer.
GEMM_EXACT_CASE = r"""
import gemm_oracle as G
M, K, N = {m}, {k}, {n}
op = G.family_e(M, N, K, x_full=True, seed=M + N, device="cuda")
acc, mag = G.ref_chunk(op, 0, M)
G.check_exact_precondition(op, 0, M, mag)
acc32 = acc.float()
assert torch.equal(acc32.double(), acc)
bn = nn.BatchNorm2d(N).cuda().eval()
randomize_bn(bn)
with torch.no_grad():
    bn.running_mean.mul_(acc.abs().mean())              # the conv output's scale: b matters against a * acc
    bn.running_var.mul_(acc.var(0).mean())
r = torch.randn(M, N, device=dev).to(torch.bfloat16)
for use_res in (False, True):
    for relu in (False, True):
        y = gemm_bnstats.gemm_bn_eval(op.x, op.w, bn, r if use_res else None, relu)
        exact_columns(y, acc32, r if use_res else None, bn, relu, ("gemm", M, K, N, use_res, relu))
print("OK")
"""


@pytest.mark.parametrize("m,k,n", [(1000, 64, 128), (1000, 64, 192), (64 * 7 * 7, 512, 2048)])
def test_gemm_bn_eval_epilogue_exact_on_exact_accumulators(m, k, n):
    _run(GEMM_EXACT_CASE, m=m, k=k, n=n)


# ------------------------------------------------------------------------------------------------------- dispatch --
DISPATCH_CASE = r"""
from mpi_operator_b200.models import resnet
calls = {{"gemm": 0, "kernel": 0}}
_gemm, _kernel = gemm_bnstats.gemm_bn_eval, fused_bn._bn_eval
def gemm_hook(*a, **k):
    calls["gemm"] += 1
    return _gemm(*a, **k)
def kernel_hook(*a, **k):
    calls["kernel"] += 1
    return _kernel(*a, **k)
gemm_bnstats.gemm_bn_eval, fused_bn._bn_eval = gemm_hook, kernel_hook

model = resnet.resnet50().cuda().to(memory_format=torch.channels_last)
for m in model.modules():
    if isinstance(m, nn.BatchNorm2d):
        randomize_bn(m)
model.eval()
x = torch.randn(2, 3, 64, 64, device=dev).contiguous(memory_format=torch.channels_last)
bufs = [b.clone() for b in model.buffers()]
with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
    n0 = fused_bn.launch_count()
    out = model(x)
n_bn = sum(isinstance(m, nn.BatchNorm2d) for m in model.modules())
# 2x3x64x64: 16x16 after the stem. The stride-1 1x1 conv_bn_act layers with M = N*H*W >= 128 take the GEMM: layer1's 3 blocks
# x 2 (M = 512), layer2's conv1 of block 1 (16x16) and all its conv3 and later conv1 (8x8: M = 128), 8, and layer3's first
# conv1 (8x8): 15. Every other BatchNorm (stem, 3x3 outputs, downsample, M < 128) runs the eval kernel.
assert calls == {{"gemm": 15, "kernel": n_bn - 15}}, calls
assert fused_bn.launch_count() - n0 == n_bn
assert all(torch.equal(a, b) for a, b in zip(bufs, model.buffers()))

def reset():
    calls["gemm"] = calls["kernel"] = 0

# fall-backs: bitwise equal to the plain PyTorch composition, and no eval kernel runs
bn = nn.BatchNorm2d(64).cuda()
randomize_bn(bn)
bn.eval()
xb = torch.randn(4, 64, 8, 8, device=dev).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
rb = torch.randn(4, 64, 8, 8, device=dev).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
def plain(bn, x, r, relu=True):
    out = bn(x)
    if r is not None:
        out = out + r
    return torch.relu(out) if relu else out
conv = nn.Conv2d(64, 64, 1, bias=False).cuda().to(memory_format=torch.channels_last)
def check(name, fn, want_fn):
    reset()
    got = fn()
    assert calls == {{"gemm": 0, "kernel": 0}}, (name, calls)
    want = want_fn()
    assert torch.equal(got, want), name
# autograd: grad mode on and the BN parameters require grad
check("autograd bn_act", lambda: fused_bn.bn_act(bn, xb, rb).detach(), lambda: plain(bn, xb, rb).detach())
xg = xb.detach().clone().requires_grad_()
check("autograd input", lambda: fused_bn.bn_act(bn, xg, rb).detach(), lambda: plain(bn, xg, rb).detach())
with torch.autocast("cuda", dtype=torch.bfloat16):
    check("autograd conv_bn_act", lambda: fused_bn.conv_bn_act(conv, bn, xb, rb).detach(),
          lambda: plain(bn, conv(xb), rb).detach())
with torch.no_grad():
    # fp32 input, non-channels-last input
    xf = xb.float()
    check("fp32", lambda: fused_bn.bn_act(bn, xf, None), lambda: plain(bn, xf, None))
    xc = xb.contiguous()
    check("contiguous", lambda: fused_bn.bn_act(bn, xc, None), lambda: plain(bn, xc, None))
    # track_running_stats=False: PyTorch uses batch statistics in eval mode
    bnb = nn.BatchNorm2d(64, track_running_stats=False).cuda().eval()
    check("no running stats", lambda: fused_bn.bn_act(bnb, xb, rb), lambda: plain(bnb, xb, rb))
    with torch.autocast("cuda", dtype=torch.bfloat16):
        check("no running stats conv", lambda: fused_bn.conv_bn_act(conv, bnb, xb, None), lambda: plain(bnb, conv(xb), None))
    # and the eval path itself runs for the same module once nothing stands in its way
    reset()
    fused_bn.bn_act(bn, xb, rb)
    assert calls == {{"gemm": 0, "kernel": 1}}, calls
print("OK")
"""


def test_eval_dispatch_and_fallbacks():
    _run(DISPATCH_CASE)


SWITCH_OFF_CASE = r"""
assert not fused_bn._ENABLED
bn = nn.BatchNorm2d(64).cuda().eval()
randomize_bn(bn)
conv = nn.Conv2d(64, 64, 1, bias=False).cuda().to(memory_format=torch.channels_last)
xb = torch.randn(4, 64, 8, 8, device=dev).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
def boom(*a, **k):
    raise AssertionError("eval kernel ran with B200MPI_FUSED_BN=0")
gemm_bnstats.gemm_bn_eval = fused_bn._bn_eval = boom
with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
    got = fused_bn.conv_bn_act(conv, bn, xb, xb)
    want = torch.relu(bn(conv(xb)) + xb)
assert torch.equal(got, want)
print("OK")
"""


def test_eval_kernels_off_with_fused_bn_switch():
    _run(SWITCH_OFF_CASE, env={"B200MPI_FUSED_BN": "0"})


# ----------------------------------------------------------------------------------------------------- whole model --
MODEL_CASE = r"""
from mpi_operator_b200.models import resnet
torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False
model = getattr(resnet, {name!r})().cuda()
for m in model.modules():
    if isinstance(m, nn.BatchNorm2d):
        randomize_bn(m)
model.eval()
x = torch.randn({batch}, 3, 224, 224, device=dev)
with torch.no_grad():
    ref = model(x).double()                                  # fp32, NCHW: the generic PyTorch path
    ml = model.to(memory_format=torch.channels_last)
    xl = x.contiguous(memory_format=torch.channels_last)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        n0 = fused_bn.launch_count()
        fused = ml(xl).double()
        assert fused_bn.launch_count() > n0
        fused_bn._ENABLED = False                            # the bf16 eval path without the eval kernels
        parent = ml(xl).double()
        fused_bn._ENABLED = True
def rel(a):
    return float((a - ref).norm() / ref.norm())
e_f, e_p = rel(fused), rel(parent)
top = ref.argmax(1)
agree_f = float((fused.argmax(1) == top).double().mean())
agree_p = float((parent.argmax(1) == top).double().mean())
print("errors", e_f, e_p, "top-1 agreement", agree_f, agree_p)
assert e_f <= 1.1 * e_p, (e_f, e_p)
assert agree_f >= min(0.99, agree_p), (agree_f, agree_p)
print("OK")
"""


@pytest.mark.parametrize("name", ["resnet50", "resnet101"])
@pytest.mark.parametrize("batch", [64, 1])
def test_resnet_eval_fused_is_as_accurate_as_the_bf16_path(name, batch):
    _run(MODEL_CASE, name=name, batch=batch)


# ------------------------------------------------------------------------------------------------------- trainer --
TRAINER_CASE = r"""
from mpi_operator_b200.models import resnet
from mpi_operator_b200.parallel.data_parallel import DataParallelTrainer
from mpi_operator_b200.runtime.comm import Communicator
comm = Communicator.create(0, 1, 0, f"t-bn-eval-{{os.getpid()}}")
model = resnet.ResNet(resnet.Bottleneck, [1, 1, 1, 1], num_classes=10)
for m in model.modules():
    if isinstance(m, nn.BatchNorm2d):
        randomize_bn(m)
g = torch.Generator().manual_seed(1)
batches = [(torch.randn(8, 3, 64, 64, generator=g), torch.randint(0, 10, (8,), generator=g)) for _ in range(4)]
ex, ey = torch.randn(8, 3, 64, 64, generator=g), torch.randint(0, 10, (8,), generator=g)
rx, ry = ex[:5].clone(), ey[:5].clone()                     # a ragged last batch
tr = DataParallelTrainer(model, nn.CrossEntropyLoss(), comm, lr=0.05, momentum=0.9, weight_decay=1e-4, cuda_graph=True)

def eager_eval(x, y):
    tr.use_graph = False
    try:
        return tr.evaluate(x, y)
    finally:
        tr.use_graph = True

def training_state():
    # everything a training step reads or carries over: master parameters and bf16 shadow, momentum, BN running statistics
    # and counters, the BN workspace, the training graph's static inputs
    torch.cuda.synchronize()
    st = tr.state
    out = [st.flat_param, st.flat_grad] + ([st.flat_lowp] if st.flat_lowp is not None else [])
    out += [b.momentum for b in st.buckets] + list(tr.model.buffers()) + list(fused_bn._WS_CACHE.values())
    out += [tr._static_x, tr._static_y]
    return [t.clone() for t in out]

first = None
for i, (x, y) in enumerate(batches):
    tr.step(x.pin_memory(), y.pin_memory())
    if i in (0, 2):
        before = training_state()
        mem = torch.cuda.memory_reserved()
        r = tr.evaluate(ex, ey)
        rr = tr.evaluate(rx, ry)
        if i == 0:
            print("eval graphs memory_reserved delta MiB", (torch.cuda.memory_reserved() - mem) / 2**20)
            first = r
        after = training_state()
        assert len(before) == len(after) and all(torch.equal(p, q) for p, q in zip(before, after)), "evaluate() changed training state"
        # graph replay == eager fused evaluate(), bit for bit
        assert r == eager_eval(ex, ey), (r, eager_eval(ex, ey))
        assert rr == eager_eval(rx, ry) and rr["examples"] == 5
assert len(tr._eval_graphs) == 2
# after further steps the same graphs see the new weights and running statistics
r = tr.evaluate(ex, ey)
assert r == eager_eval(ex, ey) and r != first, (r, first)
# a third shape runs eagerly
r3 = tr.evaluate(ex[:3], ey[:3])
assert len(tr._eval_graphs) == 2 and r3 == eager_eval(ex[:3], ey[:3])
assert tr.model.training
comm.destroy()
print("OK")
"""


def test_trainer_evaluate_under_cuda_graph():
    _run(TRAINER_CASE)
