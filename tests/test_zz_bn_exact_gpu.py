"""The fused BatchNorm kernels (csrc/kernels/bn_act.cu) bit for bit against the oracle of tests/bn_oracle.py.

Each case compares stage by stage, so that a failure names one kernel: the partial rows in the workspace, the finalize
(save_invstd within 2 ulps of the correctly rounded rsqrt, everything else bitwise), then y and the mask, then the backward's
partial rows, coef rows, dgamma / dbeta, dx and dres. Outputs carry poisoned guard bytes past their end. Covered: every
channel count at M in {1, 2, 3, rpp - 1, rpp * 64 +- 1, 12345} with and without ReLU and residual; constant channels
(variance 0, and z exactly 0 for the mask's test); null optional pointers; synthetic partial rows into both prestats entry
points (the WALK merge, the clamp of a negative variance, 1 to 296 rows); the autograd glue of ``bn_act`` (dgamma / dbeta
written into ``.grad`` or accumulated); NaN and Inf through the fused ReLU; misaligned activations. ResNet-101's shapes and
the forced reduce grids run through the same oracle in test_zz_bn_stats_gpu.py; the eval kernels in
test_zz_bn_eval_gpu.py."""
import numpy as np
import pytest
import torch
import torch.nn as nn
import torch.nn.functional as F

import bn_oracle as O

pytestmark = pytest.mark.gpu

EPS, MOMENTUM = 1e-5, 0.1
GUARD = 64                  # poisoned elements past every output
POISON16, POISON8 = 0x7FC1, 0xA5
ERR_INVALID = -1


def _lib():
    from mpi_operator_b200.runtime import _lib as L
    return L.lib()


def _p(t):
    return t.data_ptr() if t is not None else None


def _stream():
    return torch.cuda.current_stream().cuda_stream


def guarded(n, dtype):
    """(buffer, its first n elements): the GUARD elements past them hold a poison pattern."""
    buf = torch.empty(n + GUARD * 16, dtype=dtype, device="cuda")
    if dtype == torch.uint8:
        buf.fill_(POISON8)
    else:
        buf.view(torch.int16).fill_(POISON16)
    return buf, buf[:n]


def assert_guard(buf, n, what):
    tail = buf[n:]
    ok = bool((tail == POISON8).all()) if buf.dtype == torch.uint8 else bool((tail.view(torch.int16) == POISON16).all())
    assert ok, f"{what}: written past its end"


def workspace(c):
    return torch.full((int(_lib().b200mpi_bn_workspace_floats(c)),), float("nan"), device="cuda")


def inputs(m, c, seed, loc=2.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = (torch.randn(m, c, device="cuda", generator=g) * (torch.rand(c, device="cuda", generator=g) + 0.5) + loc).to(torch.bfloat16)
    res = torch.randn(m, c, device="cuda", generator=g).to(torch.bfloat16)
    dz = torch.randn(m, c, device="cuda", generator=g).to(torch.bfloat16)
    gamma = torch.rand(c, device="cuda", generator=g) + 0.5
    beta = torch.rand(c, device="cuda", generator=g) - 0.5
    rm = torch.randn(c, device="cuda", generator=g)
    rv = torch.rand(c, device="cuda", generator=g) + 0.5
    return x, res, dz, gamma, beta, rm, rv


def run_and_check(x, res, dz, gamma, beta, rm0, rv0, relu, what, nulls=False):
    """b200mpi_bn_act_fwd + b200mpi_bn_act_bwd on guarded outputs, both against the oracle. ``nulls``: no weight, bias,
    running statistics, dgamma or dbeta."""
    m, c = x.shape
    L = _lib()
    ybuf, y = guarded(m * c, torch.bfloat16)
    mbuf, mask = guarded(m * c // 8, torch.uint8) if relu else (None, None)
    mean, invstd = torch.empty(c, device="cuda"), torch.empty(c, device="cuda")
    w, b = (None, None) if nulls else (gamma, beta)
    rm, rv = (None, None) if nulls else (rm0.clone(), rv0.clone())
    ws = workspace(c)
    rc = L.b200mpi_bn_act_fwd(x.data_ptr(), _p(res), y.data_ptr(), _p(mask), _p(w), _p(b), _p(rm), _p(rv), mean.data_ptr(),
                              invstd.data_ptr(), ws.data_ptr(), m, c, EPS, MOMENTUM, int(relu), _stream())
    assert rc == 0, rc
    torch.cuda.synchronize()
    assert_guard(ybuf, m * c, what + " y")
    if relu:
        assert_guard(mbuf, m * c // 8, what + " mask")
    y2 = y.view(m, c)
    fin, _ = O.check_forward(x, res, y2, mask, mean, invstd, ws, w, b, None if nulls else rm0, None if nulls else rv0, rm, rv,
                             EPS, MOMENTUM, relu, what=what)

    dxbuf, dx = guarded(m * c, torch.bfloat16)
    drbuf, dres = guarded(m * c, torch.bfloat16) if res is not None else (None, None)
    dgamma, dbeta = (None, None) if nulls else (torch.empty(c, device="cuda"), torch.empty(c, device="cuda"))
    ws.fill_(float("nan"))
    rc = L.b200mpi_bn_act_bwd(dz.data_ptr(), x.data_ptr(), _p(mask), dx.data_ptr(), _p(dres), _p(w), mean.data_ptr(),
                              invstd.data_ptr(), _p(dgamma), _p(dbeta), ws.data_ptr(), m, c, int(relu), _stream())
    assert rc == 0, rc
    torch.cuda.synchronize()
    assert_guard(dxbuf, m * c, what + " dx")
    if res is not None:
        assert_guard(drbuf, m * c, what + " dres")
    O.check_backward(dz, x, mask, dx.view(m, c), None if dres is None else dres.view(m, c), dgamma, dbeta, ws, w, mean, invstd,
                     relu, what=what)
    return y2, mask, fin


def edge_rows(c):
    rpp = O.rows_per_pass(c)
    blk = rpp * O.UNROLL * O.BLOCK_PASSES
    return sorted({m for m in (1, 2, 3, rpp - 1, blk - 1, blk + 1, 12345) if m >= 1})


@pytest.mark.parametrize("c", O.CHANNELS)
def test_every_channel_count_at_edge_row_counts(c):
    for m in edge_rows(c):
        x, res, dz, gamma, beta, rm, rv = inputs(m, c, seed=m * 7 + c)
        for relu in (True, False):
            for use_res in (True, False):
                run_and_check(x, res if use_res else None, dz, gamma, beta, rm, rv, relu, f"M={m} C={c} relu={relu} res={use_res}")


@pytest.mark.parametrize("c", [64, 2048])
def test_constant_channels_and_exact_zeros(c):
    """Channel 0 is a constant with a full significand (variance exactly 0); channel 1 is the constant 2 with beta = 0,
    so a * 2 is exact, b = -(a * 2) and z is exactly 0 in every row: the mask's `<= 0` decides, and y is +0."""
    m = 5000
    x, res, dz, gamma, beta, rm, rv = inputs(m, c, seed=c)
    x[:, 0] = 3.140625
    x[:, 1] = 2.0
    beta[1] = 0.0
    for use_res in (False, True):
        y, mask, fin = run_and_check(x, res if use_res else None, dz, gamma, beta, rm, rv, True, f"constant C={c} res={use_res}")
        assert fin["var"][0] == 0 and fin["var"][1] == 0
        if not use_res:
            bits = O.unpack_mask(mask.cpu().numpy(), m, c)
            assert not bits[:, 1].any() and bool((y[:, 1].view(torch.int16) == 0).all())


def test_null_optional_pointers():
    for m, c in ((1000, 64), (3, 8), (777, 2048)):
        x, res, dz, gamma, beta, rm, rv = inputs(m, c, seed=m)
        for relu, use_res in ((True, True), (False, False)):
            run_and_check(x, res if use_res else None, dz, gamma, beta, rm, rv, relu, f"nulls M={m} C={c}", nulls=True)


@pytest.mark.parametrize("parts", [1, 2, 31, 97, 129, 296])
def test_prestats_entry_points_on_synthetic_partial_rows(parts):
    """Partial rows as a GEMM epilogue (forward, shifted by x[128 p]) or a dgrad epilogue (backward) would hand them over,
    at the largest (parts - 1) * 128 < M. Some channels get a sum of squares so small that the variance comes out
    negative: the finalize clamps it to 0."""
    L = _lib()
    c = 128
    m = (parts - 1) * 128 + 1
    x, res, dz, gamma, beta, rm0, rv0 = inputs(m, c, seed=parts)
    g = torch.Generator(device="cuda").manual_seed(parts + 1)
    n = torch.tensor(O.rows_per_part(m, parts).numpy(), device="cuda", dtype=torch.float32)[:, None]
    s1 = torch.randn(parts, c, device="cuda", generator=g) * n.sqrt()
    s2 = (torch.rand(parts, c, device="cuda", generator=g) + 0.5) * n
    s2[:, :8] = 0.0
    s1[:, :8] = n * 8.0          # sums about x[128 p] of n * 8 with no spread: the variance is var(x[128 p]) - 64 < 0
    fpart = torch.stack([s1, s2], -1).reshape(parts, 2 * c).contiguous()
    for relu, use_res in ((True, True), (True, False), (False, False)):
        what = f"prestats parts={parts} relu={relu} res={use_res}"
        r = res if use_res else None
        ybuf, y = guarded(m * c, torch.bfloat16)
        mbuf, mask = guarded(m * c // 8, torch.uint8) if relu else (None, None)
        mean, invstd = torch.empty(c, device="cuda"), torch.empty(c, device="cuda")
        rm, rv = rm0.clone(), rv0.clone()
        ws = workspace(c)
        rc = L.b200mpi_bn_act_fwd_prestats(x.data_ptr(), _p(r), y.data_ptr(), _p(mask), gamma.data_ptr(), beta.data_ptr(),
                                           rm.data_ptr(), rv.data_ptr(), mean.data_ptr(), invstd.data_ptr(), ws.data_ptr(),
                                           fpart.data_ptr(), parts, m, c, EPS, MOMENTUM, int(relu), _stream())
        assert rc == 0, rc
        torch.cuda.synchronize()
        assert_guard(ybuf, m * c, what + " y")
        fin, _ = O.check_forward(x, r, y.view(m, c), mask, mean, invstd, ws, gamma, beta, rm0, rv0, rm, rv, EPS, MOMENTUM, relu,
                                 pre=(fpart, parts), what=what)
        assert (fin["var"][:8] == 0).all(), fin["var"][:8]
        assert np.isnan(O.to_np(ws[4 * c:])).all(), what + ": the prestats forward wrote partial rows"

        bpart = torch.randn(parts, 2 * c, device="cuda", generator=g) * n.sqrt()
        dxbuf, dx = guarded(m * c, torch.bfloat16)
        drbuf, dres = guarded(m * c, torch.bfloat16) if use_res else (None, None)
        dgamma, dbeta = torch.empty(c, device="cuda"), torch.empty(c, device="cuda")
        ws.fill_(float("nan"))
        rc = L.b200mpi_bn_act_bwd_prestats(dz.data_ptr(), x.data_ptr(), _p(mask), dx.data_ptr(), _p(dres), gamma.data_ptr(),
                                           mean.data_ptr(), invstd.data_ptr(), dgamma.data_ptr(), dbeta.data_ptr(), ws.data_ptr(),
                                           bpart.data_ptr(), parts, m, c, int(relu), _stream())
        assert rc == 0, rc
        torch.cuda.synchronize()
        assert_guard(dxbuf, m * c, what + " dx")
        if use_res:
            assert_guard(drbuf, m * c, what + " dres")
        O.check_backward(dz, x, mask, dx.view(m, c), None if dres is None else dres.view(m, c), dgamma, dbeta, ws, gamma,
                         mean, invstd, relu, pre=(bpart, parts), what=what)


# ----------------------------------------------------------------------------------------------- autograd glue --
def _module(c, seed):
    torch.manual_seed(seed)
    bn = nn.BatchNorm2d(c).cuda()
    with torch.no_grad():
        bn.weight.uniform_(0.5, 1.5)
        bn.bias.uniform_(-0.5, 0.5)
    return bn


def _cl(t):
    return t.to(torch.bfloat16).contiguous(memory_format=torch.channels_last)


def _param_grads_oracle(z, dz, relu):
    """dgamma, dbeta of the oracle for the backward of the fused node that produced z, from what it saved."""
    x, mask, weight, save_mean, save_invstd, _ = z.grad_fn.saved_tensors
    n, c, h, w = x.shape
    m = n * h * w
    xn = O.to_np(x.permute(0, 2, 3, 1).reshape(m, c))
    dzn = O.to_np(dz.permute(0, 2, 3, 1).reshape(m, c))
    mk = O.unpack_mask(mask.cpu().numpy(), m, c) if relu else None
    grid, rows = O.plan(m, c, O.MAX_PARTS, 4 * c, O.REDUCE_CHUNK)
    tot = O.merge(O.bwd_partials(dzn, xn, mk, O.to_np(save_mean), grid, rows))
    co = O.bwd_finalize(tot, m, O.to_np(weight), O.to_np(save_mean), O.to_np(save_invstd))
    return co["dgamma"], co["dbeta"]


@pytest.mark.parametrize("direct", [False, True])
def test_autograd_parameter_gradients_match_the_oracle(direct):
    """dgamma / dbeta reach .grad through AccumulateGrad, or (the trainer's flat gradient) written in place; under
    no_sync the second micro-batch accumulates: the fp32 sum of both."""
    from mpi_operator_b200.ops.fused_bn import bn_act
    c = 256
    bn = _module(c, 0)
    accumulating = [False]
    if direct:
        ready = lambda p: None                      # noqa: E731
        ready.accumulating = lambda: accumulating[0]
        bn._b200_grad_ready = ready
        bn.weight.grad = torch.zeros_like(bn.weight)
        bn.bias.grad = torch.zeros_like(bn.bias)
    want = None
    for step in range(2):
        accumulating[0] = step == 1
        x = _cl(torch.randn(8, c, 14, 14, device="cuda") * 2 + 1).requires_grad_()
        res = _cl(torch.randn(8, c, 14, 14, device="cuda")).requires_grad_()
        dz = _cl(torch.randn(8, c, 14, 14, device="cuda"))
        z = bn_act(bn, x, residual=res, relu=True)
        assert type(z.grad_fn).__name__ == "_BNActBackward"
        dg, db = _param_grads_oracle(z, dz, True)
        z.backward(dz)
        want = (dg, db) if want is None else (want[0] + dg, want[1] + db)
        O.assert_bits(bn.weight.grad, want[0], f"step {step} weight.grad")
        O.assert_bits(bn.bias.grad, want[1], f"step {step} bias.grad")


# ---------------------------------------------------------------------------------------- non-finite values --
def test_relu_passes_nan_and_inf_like_pytorch():
    """A NaN input element poisons its channel's statistics; torch.relu keeps NaN (and threshold_backward passes its
    gradient), so the fused op must too. ±Inf in the residual: +Inf passes, -Inf becomes 0. The other channels equal a
    fused run on the clean inputs, bit for bit."""
    from mpi_operator_b200.ops.fused_bn import bn_act
    c, nan_c, inf_c = 64, 5, 9
    torch.manual_seed(1)
    x0 = _cl(torch.randn(4, c, 8, 8, device="cuda") + 1)
    r0 = _cl(torch.randn(4, c, 8, 8, device="cuda"))
    dz = _cl(torch.randn(4, c, 8, 8, device="cuda"))
    xb, rb = x0.clone(), r0.clone()
    xb[1, nan_c, 2, 3] = float("nan")
    rb[0, inf_c, 1, 1] = float("inf")
    rb[2, inf_c, 4, 4] = float("-inf")

    def fused(xv, rv):
        bn = _module(c, 2)
        xi, ri = xv.clone().requires_grad_(), rv.clone().requires_grad_()
        z = bn_act(bn, xi, residual=ri, relu=True)
        assert type(z.grad_fn).__name__ == "_BNActBackward"
        mask = z.grad_fn.saved_tensors[1]
        z.backward(dz)
        return [z.detach(), xi.grad, ri.grad, bn.weight.grad, bn.bias.grad, bn.running_mean, bn.running_var], mask

    got, mask = fused(xb, rb)
    clean, _ = fused(x0, r0)
    # PyTorch in fp32 on the same bf16 values (a bf16 composition rounds bn(x) before the add, which moves the sign of
    # values near 0 and with it their gradient)
    bn = _module(c, 2)
    xi, ri = xb.float().requires_grad_(), rb.float().requires_grad_()
    zr = F.relu(bn(xi) + ri)
    zr.backward(dz.float())
    ref = [zr.detach(), xi.grad, ri.grad, bn.weight.grad, bn.bias.grad, bn.running_mean, bn.running_var]
    names = ["z", "x.grad", "res.grad", "weight.grad", "bias.grad", "running_mean", "running_var"]
    for name, a, b in zip(names, got, ref):
        a, b = a.float(), b.float()
        assert torch.equal(torch.isnan(a), torch.isnan(b)), f"{name}: NaN positions differ"
        assert torch.equal(torch.isinf(a) & (a > 0), torch.isinf(b) & (b > 0)), f"{name}: +Inf positions differ"
        assert torch.equal(torch.isinf(a) & (a < 0), torch.isinf(b) & (b < 0)), f"{name}: -Inf positions differ"
        fin = torch.isfinite(b)
        atol = 3e-2 * (a.numel() // c) ** 0.5 if a.dim() == 1 else 3e-2    # parameter gradients: sums over N*H*W terms
        torch.testing.assert_close(a[fin], b[fin], rtol=3e-2, atol=atol, msg=name)
    assert bool(torch.isnan(got[0][:, nan_c]).all()) and bool(torch.isinf(got[0][0, inf_c, 1, 1]))
    # the mask is !(z <= 0) of the fused output (positive fp32 values never round to a bf16 zero), and where the PyTorch
    # composition is not finite the two agree: NaN and +Inf pass, -Inf does not
    z = got[0].permute(0, 2, 3, 1).reshape(-1, c)
    bits = torch.from_numpy(O.unpack_mask(mask.cpu().numpy(), z.shape[0], c)).cuda()
    assert torch.equal(bits, ~(z <= 0)), "mask differs from !(y <= 0)"
    zt = zr.detach().permute(0, 2, 3, 1).reshape(-1, c)
    odd = ~torch.isfinite(zt)
    assert bool(odd.any()) and torch.equal(bits[odd], ~(zt[odd] <= 0))
    other = [k for k in range(c) if k not in (nan_c, inf_c)]
    for name, a, b in zip(names, got, clean):
        sel = (slice(None), other) if a.dim() == 4 else other
        assert torch.equal(a[sel], b[sel]), f"{name}: a channel without NaN / Inf changed"


# -------------------------------------------------------------------------------------------------- alignment --
def test_misaligned_activations_fall_back_and_are_refused():
    from mpi_operator_b200.ops.fused_bn import bn_act, fused_bn_available
    n, c, h, w = 2, 64, 4, 4
    m = n * h * w
    torch.manual_seed(3)
    buf = torch.empty(1 + m * c, dtype=torch.bfloat16, device="cuda")
    x = buf[1:].view(n, h, w, c).permute(0, 3, 1, 2)
    x.copy_(torch.randn(n, c, h, w, device="cuda"))
    assert x.is_contiguous(memory_format=torch.channels_last) and x.data_ptr() % 16 == 2
    aligned = x.contiguous(memory_format=torch.channels_last).clone()
    rbuf = torch.empty(1 + m * c, dtype=torch.bfloat16, device="cuda")
    r = rbuf[1:].view(n, h, w, c).permute(0, 3, 1, 2)
    r.copy_(torch.randn(n, c, h, w, device="cuda"))
    bn, ref = _module(c, 4), _module(c, 4)
    assert fused_bn_available(x, bn) is False
    assert fused_bn_available(aligned, bn) is True
    for xi, ri in ((x, None), (aligned, r), (x, r)):
        got = bn_act(bn, xi, residual=ri, relu=True)
        want = F.relu(ref(xi) + ri) if ri is not None else F.relu(ref(xi))
        assert got.grad_fn is None or "BNAct" not in type(got.grad_fn).__name__
        assert torch.equal(got, want)
        assert torch.equal(bn.running_mean, ref.running_mean) and torch.equal(bn.running_var, ref.running_var)

    # the C entry points refuse such pointers instead of issuing misaligned vector loads
    L = _lib()
    ok = aligned.permute(0, 2, 3, 1).reshape(m, c)
    y, dx = torch.empty_like(ok), torch.empty_like(ok)
    mask = torch.empty(m * c // 8, dtype=torch.uint8, device="cuda")
    stats = [torch.empty(c, device="cuda") for _ in range(4)]
    ws = workspace(c)
    part = torch.zeros(1, 2 * c, device="cuda")
    p = lambda t: t.data_ptr()                      # noqa: E731
    s = _stream()
    for xp, rp in ((p(x), None), (p(ok), p(r)), (p(ok), p(ok) + 2)):
        assert L.b200mpi_bn_act_fwd(xp, rp, p(y), p(mask), None, None, None, None, p(stats[0]), p(stats[1]), p(ws), m, c, EPS,
                                    MOMENTUM, 1, s) == ERR_INVALID
        assert L.b200mpi_bn_act_fwd_prestats(xp, rp, p(y), p(mask), None, None, None, None, p(stats[0]), p(stats[1]), p(ws),
                                             p(part), 1, m, c, EPS, MOMENTUM, 1, s) == ERR_INVALID
    for dzp, xp, dxp, drp in ((p(x), p(ok), p(dx), None), (p(ok), p(x), p(dx), None), (p(ok), p(ok), p(dx) + 2, None),
                              (p(ok), p(ok), p(dx), p(y) + 2)):
        assert L.b200mpi_bn_act_bwd(dzp, xp, p(mask), dxp, drp, None, p(stats[0]), p(stats[1]), None, None, p(ws), m, c, 1,
                                    s) == ERR_INVALID
        assert L.b200mpi_bn_act_bwd_prestats(dzp, xp, p(mask), dxp, drp, None, p(stats[0]), p(stats[1]), None, None, p(ws),
                                             p(part), 1, m, c, 1, s) == ERR_INVALID
    torch.cuda.synchronize()
