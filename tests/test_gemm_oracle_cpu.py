"""The GEMM oracle of tests/gemm_oracle.py, checked on the CPU against emulations of the wgmma 1x1-convolution GEMM.

The emulation does what the kernel's contract allows: fp32 accumulation of 16-wide k-chunks in shuffled order (optionally
with alignment that truncates inside a chunk), the residual added in fp32, one round-to-nearest-even, and partial rows
summed in fp32 per 64-row warpgroup slice of each tile from the bf16 tile. The oracle must accept it and reject each
mutation a kernel could plausibly turn into."""
import pytest
import torch

import gemm_oracle as go

BM = go.BM


def _chunk_sum(p, trunc_align, g):
    """fp32 sum of one k-chunk of exact products p [M, N, 16] (float64), in a shuffled order, or exactly after truncating
    every product to the fp32 ulp of the chunk's largest one (tensor-core style alignment)."""
    if trunc_align:
        big = p.abs().amax(-1, keepdim=True)
        _, e = torch.frexp(big)
        ulp = torch.exp2((e - 24).double())
        q = torch.trunc(p / ulp) * ulp
        return q.sum(-1).float()
    acc = torch.zeros(p.shape[:2], dtype=torch.float32)
    for k in torch.randperm(p.shape[-1], generator=g).tolist():
        acc = acc + p[..., k].float()
    return acc


def emulate_y(op, *, seed=0, trunc_align=False, rounding="rne", round_before_res=False, drop_k16=None, mask=None):
    """The kernel's output for ``op`` (fp32 accumulator and bf16 result). ``mask`` overrides the residual mask the kernel
    reads (a bit-order bug)."""
    g = torch.Generator().manual_seed(seed)
    x, w = op.x.double(), op.w.double()
    K = x.shape[1]
    acc = torch.zeros(x.shape[0], w.shape[0], dtype=torch.float32)
    for c in torch.randperm(K // 16, generator=g).tolist():
        if c == drop_k16:
            continue
        p = x[:, None, 16 * c:16 * c + 16] * w[None, :, 16 * c:16 * c + 16]
        acc = acc + _chunk_sum(p, trunc_align, g)
    if op.r is not None:
        m = op.mask if mask is None else mask
        rr = torch.where(m, op.r.float(), torch.zeros(()))
        if round_before_res:
            acc = go.round_bf16(acc).float()
        acc = acc + rr
    return go.round_bf16(acc, rounding), acc


def emulate_stats(y, parts, *, past_m=False, shift_row=0):
    """Forward partial rows [parts, N, 2] fp32 of ``y`` [M, N] (bf16 or fp32): per tile, each 64-row half summed in fp32
    in order, then added to the running column sums. ``past_m`` also sums the zero rows TMA fills in past M."""
    M, N = y.shape
    num_m = -(-M // BM)
    v = y.float()
    if past_m:
        v = torch.cat([v, torch.zeros(num_m * BM - M, N)])
    out = torch.zeros(parts, N, 2)
    for p in range(parts):
        shift = v[p * BM + shift_row]
        s1 = torch.zeros(N)
        s2 = torch.zeros(N)
        for t in range(p, num_m, parts):
            for h in (0, 64):
                t1 = torch.zeros(N)
                t2 = torch.zeros(N)
                for r in range(t * BM + h, min(t * BM + h + 64, v.shape[0])):
                    f = v[r] - shift
                    t1 = t1 + f
                    t2 = (f.double() * f.double() + t2.double()).float()
                s1, s2 = s1 + t1, s2 + t2
        out[p, :, 0], out[p, :, 1] = s1, s2
    return out


def emulate_gst(dx, xb, maskb, mean, parts):
    """dgrad BN-backward partial rows of ``dx`` (bf16, or fp32 for the mutation): sum g, fma(g, xb - mean, s)."""
    M, N = dx.shape
    g = torch.where(maskb, dx.float(), torch.zeros(()))
    d = xb.float() - mean.float()
    out = torch.zeros(parts, N, 2)
    part = go.part_of_row(M, parts)
    for p in range(parts):
        s1 = torch.zeros(N)
        s2 = torch.zeros(N)
        for r in (part == p).nonzero().flatten().tolist():
            s1 = s1 + g[r]
            s2 = (g[r].double() * d[r].double() + s2.double()).float()
        out[p, :, 0], out[p, :, 1] = s1, s2
    return out


def _rejects(fn):
    try:
        fn()
    except AssertionError:
        return True
    return False


def _check_stats(y, got, parts, exact, unit=None):
    sh, mg, _ = go.stats_ref(y, parts)
    if exact:
        go.check_exact_sums(sh, mg, unit, "stats")
    go.check_rows(got, sh, mg, exact, "stats")


# --------------------------------------------------------------------------------------------------- families --
@pytest.mark.parametrize("K", [64, 256, 1024, 4096])
@pytest.mark.parametrize("x_full", [True, False])
def test_family_e_precondition_ties_and_full_significands(K, x_full):
    op = go.family_e(256, 64, K, x_full=x_full, residual=True, seed=K)
    want, ref, bound = go.expected_y(op, 0, 256)
    assert bound is None
    full = op.x if x_full else op.w
    assert float(go.full_significand(full).double().mean()) > 0.4, "the full operand must use all 8 significand bits"
    assert int((full.double().abs() > 128).sum()) > 0
    assert int(go.is_tie(ref).sum()) > 0, "family E must produce round-to-nearest-even ties"
    assert not torch.equal(go.round_bf16(ref), go.round_bf16(ref, "trunc")), "no output needs rounding"
    # the precondition is the exactness of the fp32 sum: it must hold at the extreme
    mag = go.ref_chunk(op, 0, 256)[1] / torch.exp2((op.ea[:, None] + op.eb[None, :]).double())
    assert float(mag.max()) <= 2 ** 23


def test_family_e_precondition_is_enforced():
    op = go.family_e(128, 64, 64, x_full=True, seed=1)
    op.x = (op.x.double() * 2 ** 9).to(torch.bfloat16)     # x * 2^9 breaks sum |terms| <= 2^23 units
    op.ea = op.ea.clone()
    with pytest.raises(AssertionError, match="precondition"):
        go.expected_y(op, 0, 128)


@pytest.mark.parametrize("M,N,K,residual", [(1000, 128, 256, False), (200704, 256, 64, False), (2 ** 24 + 37, 128, 64, False),
                                            (1000, 384, 192, True), (802816, 256, 64, True), (16897, 128, 2048, True)])
def test_family_s_plan_keeps_partial_rows_exact(M, N, K, residual):
    B, offset = go.stats_plan(M, N, K, residual)
    rows = int(go.rows_per_part(M, go.plan_parts(M, N)).max())
    if residual:
        assert rows * (offset + B + 4) * 6 < 2 ** 22
    else:
        assert rows * (2 * B + (8 if offset else 0)) ** 2 < 2 ** 24
    if M <= 1000:
        op = go.family_s(M, N, K, residual=residual, seed=3)
        nz = (op.w != 0).sum(1)
        assert bool((nz == B + (1 if offset else 0)).all())
        assert set(op.x.unique().tolist()) <= {-1.0, 0.0, 1.0}


def test_plan_parts_and_walk():
    assert go.plan_parts(128, 64) == 1 and go.plan_parts(129, 128) == 2 and go.plan_parts(16897, 128) == 132
    assert go.plan_parts(10 ** 6, 8384) == 1 and go.plan_parts(10 ** 6, 8448) == 2 and go.plan_parts(10 ** 6, 192) == 44
    assert go.plan_parts(10 ** 6, 2048, sms=114) == 7
    M, parts = 1000, 3
    rows = go.rows_per_part(M, parts)
    assert rows.tolist() == [384, 360, 256] and int(rows.sum()) == M


def test_mask_pack_roundtrip_and_bit_order():
    bits = torch.rand(16, 64) < 0.5
    assert torch.equal(go.unpack_mask(go.pack_mask(bits), 64), bits)
    one = torch.zeros(1, 16, dtype=torch.bool)
    one[0, 10] = True                                      # column 10: bit 2 of byte 1
    assert go.pack_mask(one).tolist() == [[0, 4]]


def test_rounding_helpers():
    v = torch.tensor([257.0, 259.0, 261.0, 263.0, -257.0, 1.0 + 2 ** -8, 3.0 * 2 ** -130], dtype=torch.float64)
    assert go.round_bf16(v).double().tolist() == v.to(torch.bfloat16).double().tolist()
    assert go.round_bf16(v, "trunc").double().tolist()[:4] == [256.0, 258.0, 260.0, 262.0]
    assert go.is_tie(v).tolist() == [True, True, True, True, True, True, False]   # odd 9-bit integers are ties
    h = go.half_ulp_bf16(torch.tensor([1.0, 1.5, 255.0, 256.0, 0.0], dtype=torch.float64))
    assert h.tolist() == [2 ** -8, 2 ** -8, 0.5, 1.0, 0.0]


# ----------------------------------------------------------------------------------------------- forward Y --
FAMILIES = [("E", dict(x_full=True)), ("E", dict(x_full=False)), ("S", {}), ("R", {})]


def _make(fam, kw, M, N, K, residual=False, seed=0):
    if fam == "E":
        return go.family_e(M, N, K, residual=residual, seed=seed, **kw)
    if fam == "S":
        return go.family_s(M, N, K, residual=residual, seed=seed, scale=not residual)
    return go.family_r(M, N, K, residual=residual, seed=seed)


@pytest.mark.parametrize("fam,kw", FAMILIES)
@pytest.mark.parametrize("K", [64, 320])
def test_oracle_accepts_fp32_accumulation_in_any_order(fam, kw, K):
    op = _make(fam, kw, 200, 64, K)
    for seed in range(3):
        y, _ = emulate_y(op, seed=seed)
        go.check_y(y, op, f"order {seed}")
    y, _ = emulate_y(op, seed=5, trunc_align=True)
    go.check_y(y, op, "truncating alignment")


@pytest.mark.parametrize("fam,kw", FAMILIES)
def test_oracle_rejects_truncation_dropped_slice(fam, kw):
    op = _make(fam, kw, 200, 64, 256, seed=1)
    if fam != "S":      # family S outputs are exact in bf16 without an offset column: nothing to round
        y, _ = emulate_y(op, rounding="trunc")
        assert _rejects(lambda: go.check_y(y, op, "trunc")), "truncation instead of RNE was accepted"
    y, _ = emulate_y(op, drop_k16=3)
    assert _rejects(lambda: go.check_y(y, op, "drop")), "a dropped k16 slice was accepted"


def test_oracle_rejects_truncation_on_offset_family_s():
    op = go.family_s(1000, 128, 256, seed=2)
    assert go.stats_plan(1000, 128, 256)[1] == go.OFFSET
    y, _ = emulate_y(op, rounding="trunc")
    assert _rejects(lambda: go.check_y(y, op, "trunc"))


# ------------------------------------------------------------------------------------------- residual epilogue --
@pytest.mark.parametrize("fam,kw", FAMILIES)
def test_residual_epilogue(fam, kw):
    op = _make(fam, kw, 200, 128, 192, residual=True, seed=4)
    y, _ = emulate_y(op, seed=1)
    go.check_y(y, op, "dgrad")
    y, _ = emulate_y(op, seed=1, trunc_align=True)
    go.check_y(y, op, "dgrad, truncating alignment")
    # masked-out residual replaced by NaN / Inf: the reference with that operand is the same value
    poisoned = op.r.clone()
    poisoned[~op.mask] = float("nan")
    go.check_y(y, op, "poisoned r", r=poisoned)
    y, _ = emulate_y(op, round_before_res=True)
    assert _rejects(lambda: go.check_y(y, op, "double rounding")), "rounding before the residual add was accepted"
    packed = go.pack_mask(op.mask)
    rev = packed.view(-1, 1).bitwise_and(1 << torch.arange(8)).ne(0).flip(1).reshape(200, 128)
    y, _ = emulate_y(op, mask=rev)
    assert _rejects(lambda: go.check_y(y, op, "bit order")), "a reversed mask bit order was accepted"


# ----------------------------------------------------------------------------------------------- statistics --
@pytest.mark.parametrize("M", [200, 383, 1000])
def test_stats_exact_on_family_s_and_mutations_rejected(M):
    N, K = 64, 128
    op = go.family_s(M, N, K, seed=M)
    parts = go.plan_parts(M, N, sms=3)       # a few partial rows so that each walks several tiles
    y, acc = emulate_y(op)
    go.check_y(y, op, "y")
    unit = torch.exp2(op.eb.double())[:, None] * torch.tensor([1.0, 1.0]).double()
    unit[:, 1] = unit[:, 0] ** 2
    _check_stats(y, emulate_stats(y, parts), parts, True, unit)
    if M % BM:
        assert _rejects(lambda: _check_stats(y, emulate_stats(y, parts, past_m=True), parts, True, unit)), "rows past M"
    assert _rejects(lambda: _check_stats(y, emulate_stats(acc, parts), parts, True, unit)), "stats from unrounded Y"
    assert _rejects(lambda: _check_stats(y, emulate_stats(y, parts, shift_row=1), parts, True, unit)), "shift from row 1"


@pytest.mark.parametrize("fam,kw", [("E", dict(x_full=True)), ("R", {})])
def test_stats_within_bound_on_inexact_families(fam, kw):
    M, N = 1000, 64
    op = _make(fam, kw, M, N, 256, seed=9)
    parts = go.plan_parts(M, N)
    y, acc = emulate_y(op)
    _check_stats(y, emulate_stats(y, parts), parts, False)
    assert _rejects(lambda: _check_stats(y, emulate_stats(acc, parts), parts, False)), "stats from unrounded Y"


# ------------------------------------------------------------------------------------------------ GST partials --
@pytest.mark.parametrize("M", [200, 1000])
def test_gst_exact_on_family_s_and_fp32_dx_rejected(M):
    N, K = 128, 192
    op = go.family_s(M, N, K, residual=True, scale=False, seed=M)
    assert go.stats_plan(M, N, K, True)[1] == go.OFFSET
    xb, maskb, mean = go.below_operands(M, N, fam="S", seed=M)
    parts = go.plan_parts(M, N)
    dx, acc = emulate_y(op)
    go.check_y(dx, op, "dx")
    rows, mg = go.gst_ref(dx, xb, maskb, mean, parts)
    assert float(mg[..., 1].max()) < 2 ** 22
    go.check_exact_sums(rows, mg, torch.tensor([1.0, 0.25], dtype=torch.float64), "gst")
    go.check_rows(emulate_gst(dx, xb, maskb, mean, parts), rows, mg, True, "gst")
    assert _rejects(lambda: go.check_rows(emulate_gst(acc, xb, maskb, mean, parts), rows, mg, True, "gst")), "GST from fp32 dX"


def test_gst_within_bound_on_family_r():
    M, N = 1000, 128
    op = go.family_r(M, N, 256, residual=True, seed=11)
    xb, maskb, mean = go.below_operands(M, N, fam="R", seed=11)
    parts = go.plan_parts(M, N)
    dx, _ = emulate_y(op)
    rows, mg = go.gst_ref(dx, xb, maskb, mean, parts)
    go.check_rows(emulate_gst(dx, xb, maskb, mean, parts), rows, mg, False, "gst")


def test_guarded_buffers():
    buf, v = go.guarded(5, 8, torch.bfloat16, "cpu")
    assert v.shape == (5, 8) and bool(buf[5:].isnan().all()) and buf.shape[0] == 5 + go.GUARD_ROWS
    mb, _ = go.guarded(5, 8, torch.uint8, "cpu")
    assert bool((mb[5:] == 0xFF).all())
    go.set_guard(mb, 5, poison=False)
    assert bool((mb[5:] == 0).all())
