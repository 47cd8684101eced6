"""The exact-sum oracle of tests/collective_oracle.py, checked on the CPU against emulations of the kernels' reduction.

The correct emulation (fp32 accumulation in any rank order, scale after the sum, one rounding when packing) must pass at
every world size; the wrong ones a kernel could plausibly turn into must be rejected where they differ in principle."""
import pytest
import torch

from collective_oracle import Guarded, assert_bits, effective_scale, exact_inputs, exact_sum, expected

N = 1 << 16
LOWP = [torch.bfloat16, torch.float16]


def _emulate(xs, op, scale=None, order=None, round_each_add=False, round_before_scale=False, scale_twice=False, drop=None):
    """The per-element reduction of one output vector, as a kernel would compute it."""
    dtype, W = xs[0].dtype, len(xs)
    s32 = effective_scale(op, W, scale)
    order = list(range(W)) if order is None else list(order)
    if drop is not None:
        order.remove(drop)
    acc = xs[order[0]].float()
    for k in order[1:]:
        acc = acc + xs[k].float()
        if round_each_add:
            acc = acc.to(dtype).float()
    if float(s32) != 1.0:
        if round_before_scale:
            acc = acc.to(dtype).float()
        acc = acc * s32
        if scale_twice:
            acc = acc * s32
    return acc.to(dtype)


def _differs(got, want):
    try:
        assert_bits(got, want)
    except AssertionError:
        return True
    return False


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("world", range(1, 9))
@pytest.mark.parametrize("op,scale", [("sum", None), ("avg", None), ("sum", 0.1), ("max", None), ("min", None)])
def test_oracle_accepts_fp32_accumulation_in_any_rank_order(dtype, world, op, scale):
    xs = exact_inputs(world, N, dtype, seed=world)
    want = expected(xs, op, scale)
    g = torch.Generator().manual_seed(7 * world)
    for _ in range(3):
        order = torch.randperm(world, generator=g).tolist()
        if op in ("max", "min"):
            f = torch.fmax if op == "max" else torch.fmin
            got = xs[order[0]].float()
            for k in order[1:]:
                got = f(got, xs[k].float())
            got = (got * effective_scale(op, world, scale)).to(dtype)
        else:
            got = _emulate(xs, op, scale, order=order)
        assert_bits(got, want, f"order {order}")


@pytest.mark.parametrize("dtype", LOWP)
@pytest.mark.parametrize("world", range(3, 9))
def test_oracle_rejects_rounding_after_every_add(dtype, world):
    xs = exact_inputs(world, N, dtype, seed=world)
    assert _differs(_emulate(xs, "sum", round_each_add=True), expected(xs, "sum"))


@pytest.mark.parametrize("dtype", LOWP)
@pytest.mark.parametrize("world", [3, 5, 6, 7])
def test_oracle_rejects_rounding_before_the_average(dtype, world):
    xs = exact_inputs(world, N, dtype, seed=world)
    assert _differs(_emulate(xs, "avg", round_before_scale=True), expected(xs, "avg"))


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("world", range(2, 9))
def test_oracle_rejects_a_dropped_rank(dtype, world):
    xs = exact_inputs(world, N, dtype, seed=world)
    for drop in (0, world - 1):
        assert _differs(_emulate(xs, "sum", drop=drop), expected(xs, "sum"))


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float16])
@pytest.mark.parametrize("world", range(1, 9))
@pytest.mark.parametrize("op,scale", [("avg", None), ("sum", 0.1)])
def test_oracle_rejects_the_scale_applied_twice(dtype, world, op, scale):
    if op == "avg" and world == 1:
        pytest.skip("avg at world 1 has scale 1, which the kernels skip")
    xs = exact_inputs(world, N, dtype, seed=world)
    assert _differs(_emulate(xs, op, scale, scale_twice=True), expected(xs, op, scale))


def test_nvls_oracle_rounds_twice_only_where_the_scale_is_inexact():
    """NVLS bf16 avg: the switch returns the sum rounded to bf16 and the kernel scales and rounds again. With a power-of-two
    world the scale is exact and both contracts agree; at world 3 they differ in some elements."""
    for world, same in ((2, True), (4, True), (8, True), (3, False)):
        xs = exact_inputs(world, N, torch.bfloat16, seed=world)
        assert _differs(expected(xs, "avg", nvls=True), expected(xs, "avg")) != same, world


def test_exact_inputs_satisfy_the_precondition_and_bad_ones_are_refused():
    for dtype in (torch.float32, torch.bfloat16, torch.float16):
        xs = exact_inputs(8, N, dtype, seed=3)
        assert all(bool((x != 0).all()) for x in xs)
        exact_sum(xs)
    wide = [torch.tensor([1.0, 2.0 ** 30]), torch.tensor([2.0 ** -30, 1.0])]   # 61 significant bits: fp32 cannot hold it
    with pytest.raises(AssertionError):
        exact_sum(wide)


def test_assert_bits_tells_signed_zeros_apart_and_matches_any_nan():
    assert_bits(torch.tensor([float("nan"), 1.0]), torch.tensor([-float("nan"), 1.0]))
    with pytest.raises(AssertionError):
        assert_bits(torch.tensor([0.0]), torch.tensor([-0.0]))
    with pytest.raises(AssertionError):
        assert_bits(torch.tensor([float("nan")]), torch.tensor([1.0]))


def test_max_min_ignore_a_nan_unless_every_rank_has_one():
    nan, inf = float("nan"), float("inf")
    xs = [torch.tensor([nan, nan, 1.0, -inf]), torch.tensor([2.0, nan, nan, 3.0])]
    assert_bits(expected(xs, "max"), torch.tensor([2.0, nan, 1.0, 3.0]))
    assert_bits(expected(xs, "min"), torch.tensor([2.0, nan, 1.0, -inf]))


def test_guarded_views_are_offset_and_record_their_sentinels():
    for dtype in (torch.float32, torch.bfloat16):
        for off in (0, 1, 3):
            g = Guarded(10, dtype, off, device="cpu").seal()
            assert g.view.numel() == 10 and g.view.data_ptr() - g.buf.data_ptr() == 64 + off * g.view.element_size()
            g.view.fill_(1.0)
            assert g.guards_intact() and not g.unchanged()
            g.buf[g.hi] ^= 1
            assert not g.guards_intact()
