"""BatchNorm statistics of the fused kernels against float64, at the shapes ResNet-101 runs at batch 64.

The reference is float64 PyTorch on the same bf16-rounded inputs the kernels read. fp32 outputs (save_mean, save_invstd,
running stats, dgamma, dbeta) are compared directly, bf16 outputs elementwise. The bn_act.cu cases are also held bit for bit
to the oracle of tests/bn_oracle.py (the float64 bounds say the algorithm is accurate, the oracle that it is the one the
kernels implement), and each of ResNet-101's layers has at least one output that is an exact bf16 tie. Covered:
  * bn_act.cu through its C entry points (forward + backward, with and without residual and ReLU) at ResNet-101's (M, C)
    pairs, at every supported channel count, and with the reduce grid forced to its 296-row cap and to a single CTA;
  * the fused 1x1 path (conv_bn_act -> gemm_bnstats_shifted -> b200mpi_bn_act_fwd_prestats) on conv outputs with
    |mean| / std from 1 to 1000 and on a constant channel;
  * the backward from the partial rows a dgrad epilogue hands over (b200mpi_bn_act_bwd_prestats);
  * bitwise determinism (eager, CUDA-graph replay, fused path), the fall-back for unsupported C, and M = 1.

Cases that launch the wgmma GEMM, or that set B200MPI_BN_REDUCE_CHUNK (read once per process), run in a subprocess, so a
trap in a kernel cannot poison the CUDA context of the test session; the file sorts after the other BN tests for the same
reason. B200MPI_SKIP_GEMM_TESTS=1 skips the GEMM cases."""
import os
import subprocess
import sys

import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HERE = os.path.dirname(os.path.abspath(__file__))
skip_gemm = pytest.mark.skipif(os.environ.get("B200MPI_SKIP_GEMM_TESTS") == "1", reason="B200MPI_SKIP_GEMM_TESTS=1")

EPS, MOMENTUM = 1e-5, 0.1
from bn_oracle import MAX_PARTS, REDUCE_CHUNK, THREADS, plan_rows  # noqa: E402
import bn_oracle  # noqa: E402

ULP_REL = 2.0 ** -7                        # one bf16 ulp, relative: the rounding of every bf16 output

# (M = N*H*W, C) of ResNet-101's BatchNorm layers at batch 64 (224x224 input)
RESNET101 = [(802816, 64), (200704, 64), (200704, 128), (200704, 256), (50176, 128), (50176, 512), (12544, 256),
             (12544, 1024), (3136, 512), (3136, 2048)]


# ------------------------------------------------------------------------------------------------ helpers ----
def _lib():
    from mpi_operator_b200.runtime import _lib as L
    return L.lib()


def _p(t):
    return t.data_ptr() if t is not None else None


def _stream():
    return torch.cuda.current_stream().cuda_stream


def new_workspace(c):
    """NaN-filled, so that the partial rows a kernel wrote can be counted afterwards."""
    return torch.full((int(_lib().b200mpi_bn_workspace_floats(c)),), float("nan"), device="cuda")


def rows_written(ws, c):
    part = ws[4 * c: 4 * c + MAX_PARTS * 2 * c].view(MAX_PARTS, 2 * c)
    done = ~torch.isnan(part).any(1)
    n = int(done.sum())
    assert bool(done[:n].all()), "partial rows are not a prefix of the workspace"
    return n


def bn_fwd(x, res, gamma, beta, rm, rv, relu, ws):
    m, c = x.shape
    y = torch.empty_like(x)
    mask = torch.empty(m * c // 8, dtype=torch.uint8, device=x.device) if relu else None
    mean = torch.empty(c, device=x.device)
    invstd = torch.empty(c, device=x.device)
    rc = _lib().b200mpi_bn_act_fwd(x.data_ptr(), _p(res), y.data_ptr(), _p(mask), gamma.data_ptr(), beta.data_ptr(), rm.data_ptr(),
                                   rv.data_ptr(), mean.data_ptr(), invstd.data_ptr(), ws.data_ptr(), m, c, EPS, MOMENTUM, int(relu),
                                   _stream())
    assert rc == 0, rc
    return y, mask, mean, invstd


def bn_bwd(dz, x, mask, gamma, mean, invstd, relu, with_res, ws, pre=None):
    """b200mpi_bn_act_bwd, or b200mpi_bn_act_bwd_prestats with pre = (partials, parts)."""
    m, c = x.shape
    dx = torch.empty_like(x)
    dres = torch.empty_like(x) if with_res else None
    dgamma = torch.empty(c, device=x.device)
    dbeta = torch.empty(c, device=x.device)
    args = (dz.data_ptr(), x.data_ptr(), _p(mask), dx.data_ptr(), _p(dres), gamma.data_ptr(), mean.data_ptr(), invstd.data_ptr(),
            dgamma.data_ptr(), dbeta.data_ptr(), ws.data_ptr())
    if pre is None:
        rc = _lib().b200mpi_bn_act_bwd(*args, m, c, int(relu), _stream())
    else:
        rc = _lib().b200mpi_bn_act_bwd_prestats(*args, pre[0].data_ptr(), pre[1], m, c, int(relu), _stream())
    assert rc == 0, rc
    return dx, dres, dgamma, dbeta


def mask_bits(mask, m, c):
    """[M*C/8] uint8, bit c%8 of byte (m*C + c)/8 -> [M, C] bool"""
    shifts = torch.arange(8, device=mask.device, dtype=torch.int32)
    return ((mask.view(m, c // 8).unsqueeze(-1).int() >> shifts) & 1).reshape(m, c).bool()


def ref_stats(x):
    xd = x.double()
    mu = xd.mean(0)
    var = xd.var(0, unbiased=False)
    return xd, mu, var, (var + EPS).rsqrt()


def ref_running(rm0, rv0, mu, var, m, calls):
    rm, rv = rm0.double(), rv0.double()
    for _ in range(calls):
        rm = (1 - MOMENTUM) * rm + MOMENTUM * mu
        rv = (1 - MOMENTUM) * rv + MOMENTUM * var * (m / (m - 1))
    return rm, rv


def assert_elementwise(got, ref, what):
    # about one bf16 ulp of each element, plus 1e-4 of the tensor's largest magnitude for values near zero
    err = (got.double() - ref).abs()
    bound = ULP_REL * ref.abs() + 1e-4 * ref.abs().max()
    worst = (err / bound.clamp_min(1e-300)).max().item()
    assert worst <= 1.0, f"{what}: worst error / bound = {worst:.3g}"


def assert_stats(mean, invstd, mu, var, inv_ref, what):
    sigma = var.sqrt()
    # the mean to 1e-4 of a standard deviation, plus the fp32 resolution of a mean far from zero
    mean_ratio = ((mean.double() - mu).abs() / (1e-4 * sigma + 1e-6 * mu.abs()).clamp_min(1e-300)).max().item()
    # invstd to a relative 1e-4: every normalised value inherits this error
    inv_err = ((invstd.double() - inv_ref).abs() / inv_ref).max().item()
    assert mean_ratio <= 1.0 and inv_err <= 1e-4, f"{what}: mean error / bound = {mean_ratio:.3g}, invstd rel. error = {inv_err:.3g}"


def assert_running(rm, rv, want_rm, want_rv, what):
    # the fp32 update of an accurate mean / variance: a relative 1e-5
    e_m = ((rm.double() - want_rm).abs() / want_rm.abs()).max().item()
    e_v = ((rv.double() - want_rv).abs() / want_rv.abs()).max().item()
    assert e_m <= 1e-5 and e_v <= 1e-5, f"{what}: running_mean rel. error {e_m:.3g}, running_var rel. error {e_v:.3g}"


def ref_bwd(dz, xd, bits, gamma, mu, inv, relu):
    g = dz.double() * bits if relu else dz.double()
    xhat = (xd - mu) * inv
    dbeta, dgamma = g.sum(0), (g * xhat).sum(0)
    m = xd.shape[0]
    dx = gamma.double() * inv * (g - dbeta / m - xhat * (dgamma / m))
    # per-channel scale of the summed terms, for the dgamma / dbeta bounds
    return g, dx, dgamma, dbeta, (g * xhat).abs().sum(0), g.abs().sum(0)


def assert_param_grads(dgamma, dbeta, ref_dgamma, ref_dbeta, abs_gx, abs_g, what, rel=1e-4):
    # fp32 sums over M terms: within `rel` of the sum of the terms' magnitudes, per channel
    eg = ((dgamma.double() - ref_dgamma).abs() / (rel * abs_gx).clamp_min(1e-300)).max().item()
    eb = ((dbeta.double() - ref_dbeta).abs() / (rel * abs_g).clamp_min(1e-300)).max().item()
    assert eg <= 1.0 and eb <= 1.0, f"{what}: dgamma error / bound = {eg:.3g}, dbeta error / bound = {eb:.3g}"


def make_bn_inputs(m, c, use_res, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    # per-channel means of either sign with |mean| / std up to 8, so that relative running-stat bounds are meaningful
    mu = (torch.rand(c, device="cuda", generator=g) * 3 + 1) * torch.where(torch.rand(c, device="cuda", generator=g) < 0.5, -1.0, 1.0)
    sd = torch.rand(c, device="cuda", generator=g) * 1.5 + 0.5
    x = (torch.randn(m, c, device="cuda", generator=g) * sd + mu).to(torch.bfloat16)
    res = torch.randn(m, c, device="cuda", generator=g).to(torch.bfloat16) if use_res else None
    gamma = torch.rand(c, device="cuda", generator=g) + 0.5
    beta = torch.rand(c, device="cuda", generator=g) - 0.5
    dz = torch.randn(m, c, device="cuda", generator=g).to(torch.bfloat16)
    return x, res, gamma, beta, dz


# ------------------------------------------------------------------------------------------- bn_act.cu ----
def check_bn_act(m, c, relu, use_res, chunk=REDUCE_CHUNK, calls=3):
    """Forward `calls` times and backward twice on the same inputs; everything against float64 and bit for bit against
    the oracle (tests/bn_oracle.py), and every repeat bitwise equal to the first. Returns the partial-row counts of the
    forward and backward reduce grids and the bf16 ties among y and dx."""
    x, res, gamma, beta, dz = make_bn_inputs(m, c, use_res, seed=m + c)
    rm = torch.zeros(c, device="cuda")
    rv = torch.ones(c, device="cuda")
    rm0, rv0 = rm.clone(), rv.clone()
    xd, mu, var, inv = ref_stats(x)
    tag = f"M={m} C={c} relu={relu} res={use_res}"

    ws = new_workspace(c)
    first = bn_fwd(x, res, gamma, beta, rm, rv, relu, ws)
    fwd_rows = rows_written(ws, c)
    assert fwd_rows == plan_rows(m, c, 2 * c, chunk), (tag, fwd_rows)
    assert_running(rm, rv, *ref_running(rm0, rv0, mu, var, m, 1), tag + " after 1 call")
    y, mask, mean, invstd = first
    fin, y_ties = bn_oracle.check_forward(x, res, y, mask, mean, invstd, ws, gamma, beta, rm0, rv0, rm, rv, EPS, MOMENTUM, relu,
                                          chunk=chunk, what=tag)
    want_rm, want_rv = fin["rm"], fin["rv"]
    for _ in range(calls - 1):
        again = bn_fwd(x, res, gamma, beta, rm, rv, relu, ws)
        for a, b in zip(first, again):
            assert a is None or torch.equal(a, b), tag + ": forward not deterministic"
        fin = bn_oracle.fwd_finalize(bn_oracle.merge(bn_oracle.to_np(ws[4 * c:4 * c + fwd_rows * 2 * c]).reshape(fwd_rows, -1)),
                                     bn_oracle.to_np(x[0]), m, None, None, want_rm, want_rv, EPS, MOMENTUM, invstd=fin["invstd"])
        want_rm, want_rv = fin["rm"], fin["rv"]
    bn_oracle.assert_bits(rm, want_rm, tag + " running_mean after every call")
    bn_oracle.assert_bits(rv, want_rv, tag + " running_var after every call")
    assert_running(rm, rv, *ref_running(rm0, rv0, mu, var, m, calls), tag + f" after {calls} calls")

    assert_stats(mean, invstd, mu, var, inv, tag)
    z = (xd - mu) * inv * gamma.double() + beta.double()
    if use_res:
        z = z + res.double()
    if relu:
        z = z.clamp_min(0)
        bits = mask_bits(mask, m, c)
        assert torch.equal(bits, y > 0), tag + ": ReLU mask differs from z > 0"
    assert_elementwise(y, z, tag + " z")
    del z

    ws.fill_(float("nan"))
    grads = bn_bwd(dz, x, mask, gamma, mean, invstd, relu, use_res, ws)
    bwd_rows = rows_written(ws, c)
    assert bwd_rows == plan_rows(m, c, 4 * c, chunk), (tag, bwd_rows)
    for a, b in zip(grads, bn_bwd(dz, x, mask, gamma, mean, invstd, relu, use_res, ws)):
        assert a is None or torch.equal(a, b), tag + ": backward not deterministic"
    dx, dres, dgamma, dbeta = grads
    dx_ties = bn_oracle.check_backward(dz, x, mask, dx, dres, dgamma, dbeta, ws, gamma, mean, invstd, relu, chunk=chunk, what=tag)
    g, ref_dx, ref_dgamma, ref_dbeta, abs_gx, abs_g = ref_bwd(dz, xd, bits if relu else None, gamma, mu, inv, relu)
    assert_param_grads(dgamma, dbeta, ref_dgamma, ref_dbeta, abs_gx, abs_g, tag)
    assert_elementwise(dx, ref_dx, tag + " dx")
    if use_res:
        assert_elementwise(dres, g, tag + " dres")
    print(f"{tag}: bf16 ties among y {y_ties}, among dx {dx_ties}")
    return fwd_rows, bwd_rows, y_ties, dx_ties


@pytest.mark.parametrize("relu,use_res", [(True, True), (True, False), (False, True), (False, False)])
@pytest.mark.parametrize("m,c", RESNET101)
def test_bn_act_resnet101_shapes_match_fp64(m, c, relu, use_res):
    fwd_rows, bwd_rows, y_ties, dx_ties = check_bn_act(m, c, relu, use_res)
    # the oracle has decided round-to-nearest-even ties at every one of these shapes
    assert y_ties + dx_ties > 0
    # every layer merges >= 97 partial rows in at least one direction: the merge's 4-way unrolled loop runs
    assert max(fwd_rows, bwd_rows) >= 97
    if (m, c) == (802816, 64):
        assert fwd_rows == bwd_rows == MAX_PARTS


@pytest.mark.parametrize("c", [8, 16, 32, 64, 128, 256, 512, 1024, 2048])
def test_bn_act_every_channel_count_matches_fp64(c):
    m = 12345   # not a multiple of 4 row passes (8192 / C rows) for any C
    assert m % (4 * THREADS // (c // 8)) != 0
    check_bn_act(m, c, relu=True, use_res=True, calls=1)


@pytest.mark.parametrize("c", [24, 96, 4096])
def test_bn_act_unsupported_channels_fall_back_to_pytorch(c):
    from mpi_operator_b200.ops.fused_bn import bn_act, fused_bn_available
    torch.manual_seed(c)
    bn = nn.BatchNorm2d(c).cuda()
    with torch.no_grad():
        bn.weight.uniform_(0.5, 1.5)
        bn.bias.uniform_(-0.5, 0.5)
    ref = nn.BatchNorm2d(c).cuda()
    ref.load_state_dict(bn.state_dict())
    x = torch.randn(2, c, 5, 7, device="cuda").to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    res = torch.randn(2, c, 5, 7, device="cuda").to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    assert not _lib().b200mpi_bn_supported(70, c)
    assert not fused_bn_available(x, bn)
    z = bn_act(bn, x, residual=res, relu=True)
    want = F.relu(ref(x) + res)
    assert torch.equal(z, want)
    assert torch.equal(bn.running_mean, ref.running_mean) and torch.equal(bn.running_var, ref.running_var)


def test_bn_act_single_value_per_channel_raises_like_pytorch():
    from mpi_operator_b200.ops.fused_bn import bn_act, fused_bn_available
    bn = nn.BatchNorm2d(64).cuda()
    x = torch.randn(1, 64, 1, 1, device="cuda").to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    assert not fused_bn_available(x, bn)
    with pytest.raises(ValueError, match="more than 1 value per channel"):
        bn_act(bn, x)
    x2 = torch.randn(2, 64, 1, 1, device="cuda").to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    assert fused_bn_available(x2, bn)


def _run(expr, env=None, timeout=900):
    code = f"import sys; sys.path[:0] = [{REPO!r}, {HERE!r}]; import test_zz_bn_stats_gpu as T; {expr}; print('OK')"
    r = subprocess.run([sys.executable, "-c", code], env={**os.environ, **(env or {})}, capture_output=True, text=True, timeout=timeout)
    assert r.returncode == 0 and "OK" in r.stdout, r.stdout[-3000:] + r.stderr[-3000:]
    return r.stdout


def test_bn_act_reduce_grid_at_its_cap_for_a_small_layer():
    # a 1-byte chunk leaves the CTA count to the row rule and the cap: 37888 rows at C = 64 give exactly 296 CTAs
    assert plan_rows(37888, 64, 2 * 64, chunk=1) == plan_rows(37888, 64, 4 * 64, chunk=1) == MAX_PARTS
    _run("assert T.check_bn_act(37888, 64, True, True, chunk=1)[:2] == (T.MAX_PARTS, T.MAX_PARTS)",
         env={"B200MPI_BN_REDUCE_CHUNK": "1"})


def test_bn_act_reduce_grid_of_one_cta():
    # one CTA over all of M: ~6,300 serial fp32 adds per thread at M = 200704, C = 64
    _run("assert T.check_bn_act(200704, 64, True, False, chunk=10**15, calls=1)[:2] == (1, 1)",
         env={"B200MPI_BN_REDUCE_CHUNK": str(10 ** 15)})


def test_bn_act_bitwise_deterministic_and_graph_replay_matches_eager():
    m, c = 50176, 256
    x, res, gamma, beta, dz = make_bn_inputs(m, c, True, seed=1)
    rm0 = torch.randn(c, device="cuda")
    rv0 = torch.rand(c, device="cuda") + 0.5
    ws = new_workspace(c)

    def step(rm, rv):
        y, mask, mean, invstd = bn_fwd(x, res, gamma, beta, rm, rv, True, ws)
        return (y, mask, mean, invstd, rm, rv) + bn_bwd(dz, x, mask, gamma, mean, invstd, True, True, ws)

    eager = [step(rm0.clone(), rv0.clone()) for _ in range(2)]
    for a, b in zip(*eager):
        assert torch.equal(a, b)
    rm, rv = rm0.clone(), rv0.clone()
    graph = torch.cuda.CUDAGraph()
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        with torch.cuda.graph(graph):
            captured = step(rm, rv)
    for _ in range(2):
        rm.copy_(rm0)
        rv.copy_(rv0)
        graph.replay()
        torch.cuda.synchronize()
        for a, b in zip(eager[0], captured):
            assert torch.equal(a, b)


# ------------------------------------------------------------------------- fused 1x1 convolution path ----
RATIOS = (1.0, 10.0, 100.0, 1000.0)   # |mean| / std of the convolution output channels, c % 4 -> RATIOS[c % 4]
CONST = 3.140625                       # a full 8-bit bf16 mantissa: its sums of squares are inexact in fp32


def check_conv1x1(m, cout, nhw, cin=64):
    """conv_bn_act on a 1x1 convolution whose output channels have |mean| / std = RATIOS[c % 4], plus one constant channel
    (the last). Input channel 0 is 1.0, so weight column 0 sets each output channel's mean; the other columns have unit
    norm and feed zero-mean noise, the channel's std."""
    from mpi_operator_b200.ops import fused_bn, gemm_bnstats
    n, h, w = nhw
    assert n * h * w == m
    gen = torch.Generator(device="cuda").manual_seed(m + cout)
    x = torch.randn(m, cin, device="cuda", generator=gen)
    x[:, 0] = 1.0
    x = x.to(torch.bfloat16)
    noise = torch.randn(cout, cin - 1, device="cuda", generator=gen)
    chan = torch.arange(cout, device="cuda")
    target = torch.tensor(RATIOS, device="cuda")[chan % 4]
    sign = torch.where(chan % 8 < 4, 1.0, -1.0)
    wgt = torch.cat([(target * sign)[:, None], noise / noise.norm(dim=1, keepdim=True)], 1)
    wgt[-1] = 0.0
    wgt[-1, 0] = CONST
    wgt = wgt.to(torch.bfloat16)

    conv = nn.Conv2d(cin, cout, 1, bias=False).cuda()
    bn = nn.BatchNorm2d(cout).cuda()
    with torch.no_grad():
        conv.weight.copy_(wgt.float().view(cout, cin, 1, 1))
        bn.weight.uniform_(0.5, 1.5, generator=gen)
        bn.bias.uniform_(0.25, 0.75, generator=gen)   # > 0: the constant channel's output is beta itself
    x4 = x.view(n, h, w, cin).permute(0, 3, 1, 2)
    assert x4.is_contiguous(memory_format=torch.channels_last)

    # partial rows of the GEMM: one per m-group, as many groups as SMs (up to the kernel's partial-row capacity) allow
    _, _, parts = gemm_bnstats.gemm_bnstats_shifted(x, wgt)
    cap = int(gemm_bnstats.lib().b200mpi_gemm_bnstats_partial_floats(cout)) // (2 * cout)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    num_n = cout // (128 if cout % 128 == 0 else 64)
    assert parts == min(min(sms, cap) // num_n, (m + 127) // 128), parts

    z = fused_bn.conv_bn_act(conv, bn, x4, relu=True)
    assert type(z.grad_fn).__name__.startswith("_Conv1x1BNAct"), type(z.grad_fn).__name__
    saved = z.grad_fn.saved_tensors
    yconv, mask, mean, invstd = saved[2], saved[3], saved[5], saved[6]
    z2 = z.permute(0, 2, 3, 1).reshape(m, cout)

    yd, mu, var, inv = ref_stats(yconv)
    sigma = var.sqrt()
    achieved = (mu.abs() / sigma)[:-1]
    assert bool(((achieved >= 0.5 * target[:-1]) & (achieved <= 2 * target[:-1])).all()), achieved

    report, failed = [], False
    mean_ratio = (mean.double() - mu).abs() / (1e-4 * sigma + 1e-6 * mu.abs()).clamp_min(1e-300)
    inv_err = (invstd.double() - inv).abs() / inv
    for k, r in enumerate(RATIOS):
        sel = (chan % 4 == k) & (chan < cout - 1)
        mr, ie = mean_ratio[sel].max().item(), inv_err[sel].max().item()
        failed |= mr > 1.0 or ie > 1e-4
        report.append(f"|mean|/std={r:g}: mean error / bound {mr:.3g}, invstd rel. error {ie:.3g}")
    # the constant channel: variance exactly 0, so invstd = rsqrt(eps) (rsqrtf: a few fp32 ulps)
    ie = inv_err[-1].item()
    failed |= ie > 1e-6 or mean_ratio[-1].item() > 1.0
    report.append(f"constant channel: invstd {invstd[-1].item():.7g} (want {inv[-1].item():.7g}), rel. error {ie:.3g}")
    tag = f"M={m} Cout={cout}"
    print(tag, "; ".join(report))
    assert not failed, tag + ": " + "; ".join(report)

    beta = bn.bias.detach().double()
    assert bool(((z2[:, -1].double() - beta[-1]).abs() <= ULP_REL * beta[-1]).all()), "constant channel: z != beta"
    zr = ((yd - mu) * inv * bn.weight.detach().double() + beta).clamp_min(0)
    assert torch.equal(mask_bits(mask, m, cout), z2 > 0), tag + ": ReLU mask differs from z > 0"
    assert_elementwise(z2, zr, tag + " z")
    assert_running(bn.running_mean, bn.running_var,
                   *ref_running(torch.zeros(cout, device="cuda"), torch.ones(cout, device="cuda"), mu, var, m, 1), tag)


@skip_gemm
@pytest.mark.parametrize("cout", [64, 128, 256, 2048])
@pytest.mark.parametrize("m,nhw", [(200704, (64, 56, 56)), (3136, (64, 7, 7)), (1000, (10, 10, 10))])
def test_conv1x1_bn_statistics_large_mean_and_constant_channel(m, nhw, cout):
    _run(f"T.check_conv1x1({m}, {cout}, {nhw})")


def check_gemm_partials(m, n, k):
    """Partial rows of the GEMM against float64, row by row: the kernel's shifted rows (gemm_bnstats_shifted) and their
    conversion to plain sums (gemm_bnstats_raw). The output columns have |mean| / std of about 10."""
    from mpi_operator_b200.ops import gemm_bnstats
    gen = torch.Generator(device="cuda").manual_seed(m + n + k)
    x = torch.randn(m, k, device="cuda", generator=gen)
    x[:, 0] = 1.0
    x = x.to(torch.bfloat16)
    w = torch.randn(n, k, device="cuda", generator=gen) / k ** 0.5
    w[:, 0] = 10.0
    w = w.to(torch.bfloat16)
    y, shifted, parts = gemm_bnstats.gemm_bnstats_shifted(x, w)
    shifted = shifted.clone()
    y2, plain, parts2 = gemm_bnstats.gemm_bnstats_raw(x, w)
    assert parts2 == parts and torch.equal(y, y2)
    yd = y.double()
    tile_of_row = (torch.arange(m, device="cuda") // 128) % parts
    covered = torch.bincount(tile_of_row, minlength=parts).tolist()
    assert covered == gemm_bnstats.walk_rows(m, parts), (covered, gemm_bnstats.walk_rows(m, parts))

    def per_row(v):
        return torch.zeros(parts, n, dtype=torch.float64, device="cuda").index_add_(0, tile_of_row, v)

    dev = yd - yd[tile_of_row * 128]
    # fp32 sums of a few thousand terms per thread: within 1e-5 of the sum of the terms' magnitudes
    for got, want, scale, what in ((shifted[..., 0], per_row(dev), per_row(dev.abs()), "shifted sum"),
                                   (shifted[..., 1], per_row(dev * dev), per_row(dev * dev), "shifted sum of squares"),
                                   (plain[..., 0], per_row(yd), per_row(yd.abs()), "sum"),
                                   (plain[..., 1], per_row(yd * yd), per_row(yd * yd), "sum of squares")):
        worst = ((got.double() - want).abs() / (1e-5 * scale).clamp_min(1e-300)).max().item()
        assert worst <= 1.0, f"M={m} N={n} K={k} {what}: worst error / bound = {worst:.3g}"


@skip_gemm
@pytest.mark.parametrize("m,n,k", [(128, 64, 64), (1000, 128, 256), (3136, 2048, 512), (200704, 64, 64), (200704, 256, 64)])
def test_gemm_partial_rows_match_fp64(m, n, k):
    _run(f"T.check_gemm_partials({m}, {n}, {k})")


def check_bwd_prestats(m, n, k):
    """The dgrad of a 1x1 convolution (dX = dY . Wt^T + mask ⊙ R) takes the backward partials of the BatchNorm below it;
    b200mpi_bn_act_bwd_prestats on those rows and b200mpi_bn_act_bwd on the same gradient must both match float64 and
    agree with each other to fp32 summation."""
    from mpi_operator_b200.ops import gemm_bnstats
    gen = torch.Generator(device="cuda").manual_seed(m + n)
    # the BatchNorm below (a bottleneck's bn3: residual + ReLU)
    xb, resb, gamma, beta, _ = make_bn_inputs(m, n, True, seed=m + n + 1)
    ws = new_workspace(n)
    _, maskb, meanb, invb = bn_fwd(xb, resb, gamma, beta, torch.zeros(n, device="cuda"), torch.ones(n, device="cuda"), True, ws)
    # the dgrad operands
    dy = torch.randn(m, k, device="cuda", generator=gen).to(torch.bfloat16)
    wt = (torch.randn(n, k, device="cuda", generator=gen) / k ** 0.5).to(torch.bfloat16)
    r = torch.randn(m, n, device="cuda", generator=gen).to(torch.bfloat16)
    mask = torch.randint(0, 256, (m * n // 8,), device="cuda", generator=gen, dtype=torch.int32).to(torch.uint8)
    dz, partials, parts = gemm_bnstats.dgrad_residual(dy, wt, r, mask, below=(xb, maskb, meanb))
    torch.cuda.synchronize()

    xd, _, _, _ = ref_stats(xb)
    bits = mask_bits(maskb, m, n)
    g, ref_dx, ref_dgamma, ref_dbeta, abs_gx, abs_g = ref_bwd(dz, xd, bits, gamma, meanb.double(), invb.double(), True)
    pre = bn_bwd(dz, xb, maskb, gamma, meanb, invb, True, True, ws, pre=(partials.reshape(-1), parts))
    again = bn_bwd(dz, xb, maskb, gamma, meanb, invb, True, True, ws, pre=(partials.reshape(-1), parts))
    for a, b in zip(pre, again):
        assert torch.equal(a, b), "prestats backward not deterministic"
    red = bn_bwd(dz, xb, maskb, gamma, meanb, invb, True, True, ws)
    for name, out in (("prestats", pre), ("reduce", red)):
        dx, dres, dgamma, dbeta = out
        tag = f"M={m} N={n} K={k} {name}"
        assert_param_grads(dgamma, dbeta, ref_dgamma, ref_dbeta, abs_gx, abs_g, tag)
        assert_elementwise(dx, ref_dx, tag + " dx")
        assert torch.equal(dres, (g.to(torch.bfloat16))), tag + " dres"
    # the two paths differ only in fp32 summation order
    assert_param_grads(pre[2], pre[3], red[2].double(), red[3].double(), abs_gx, abs_g, f"M={m} prestats vs reduce", rel=1e-5)
    err = (pre[0].double() - red[0].double()).abs()
    assert bool((err <= ULP_REL * red[0].double().abs() + 1e-5 * red[0].double().abs().max()).all()), "dx: prestats vs reduce"


@skip_gemm
@pytest.mark.parametrize("m,n,k", [(200704, 256, 64), (50176, 512, 128), (12544, 1024, 256), (3136, 2048, 512), (1000, 256, 64)])
def test_bn_backward_from_dgrad_partials_matches_fp64(m, n, k):
    _run(f"T.check_bwd_prestats({m}, {n}, {k})")


def check_conv1x1_determinism():
    """Two forward + backward runs of the fused 1x1 path (GEMM statistics, prestats finalize, residual, ReLU) from the same
    state give bitwise-equal outputs, statistics, running stats and gradients."""
    import copy
    from mpi_operator_b200.ops import fused_bn
    torch.manual_seed(0)
    conv = nn.Conv2d(256, 512, 1, bias=False).cuda().to(memory_format=torch.channels_last)
    bn = nn.BatchNorm2d(512).cuda()
    x = (torch.randn(64, 256, 28, 28, device="cuda") + 1).to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    res = torch.randn(64, 512, 28, 28, device="cuda").to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    dz = torch.randn(64, 512, 28, 28, device="cuda").to(torch.bfloat16).contiguous(memory_format=torch.channels_last)
    runs = []
    for _ in range(2):
        c, b = copy.deepcopy(conv), copy.deepcopy(bn)
        xi, ri = x.clone().requires_grad_(), res.clone().requires_grad_()
        z = fused_bn.conv_bn_act(c, b, xi, residual=ri, relu=True)
        assert type(z.grad_fn).__name__.startswith("_Conv1x1BNAct")
        saved = z.grad_fn.saved_tensors
        out = [z.detach(), saved[3], saved[5], saved[6], b.running_mean, b.running_var]
        z.backward(dz)
        runs.append(out + [xi.grad, ri.grad, c.weight.grad, b.weight.grad, b.bias.grad])
    for i, (a, b) in enumerate(zip(*runs)):
        assert torch.equal(a, b), f"output {i} differs between runs"


@skip_gemm
def test_conv1x1_bn_act_bitwise_deterministic():
    _run("T.check_conv1x1_determinism()")
