"""The Adasum oracle (tests/adasum_oracle.py) checked on the CPU, and the torch tree (hvd/adasum.py) held to it bit for bit.

The oracle's coefficients must equal an exact rational computation, its outputs must stay within its bound of the float64
tree, and its tie guard must fire on a constructed tie. ``adasum_pair`` / ``adasum_tree`` must equal it bit for bit at
worlds 2 to 8, must be exactly scale equivariant, and must average identical tensors whatever their scale (a clamp on the
norm once summed tensors of norm below 1e-15 instead of combining them, and fp32 norms overflowed past 2^64)."""
import math
from fractions import Fraction

import numpy as np
import pytest
import torch

from adasum_oracle import TieError, coefficient, expected, kernel_depth, kernel_geometry, torch_depth, tree64, tree64_bound
from collective_oracle import assert_bits
from mpi_operator_b200.hvd.adasum import adasum_pair, adasum_tree

DTYPES = [torch.float32, torch.bfloat16, torch.float16]
LOOSEST = {torch.float32: 2.0 ** -12, torch.bfloat16: 2.0 ** -6, torch.float16: 2.0 ** -9}   # median of bound / |tree64|


def gaussians(world, n, dtype, seed):
    """Correlated gradients (a shared direction plus rank noise) with different norms per rank."""
    g = torch.Generator().manual_seed(seed)
    base = torch.randn(n, generator=g)
    return [((0.5 * base + torch.randn(n, generator=g)) * (1.0 + 0.25 * r)).to(dtype) for r in range(world)]


def spread(world, n, dtype, seed, span=40):
    """Per-rank norms spread over 2^±span (f16: 2^±6, to stay in range)."""
    g = torch.Generator().manual_seed(seed)
    span = 6 if dtype == torch.float16 else span
    xs = gaussians(world, n, torch.float32, seed)
    ks = torch.randint(-span, span + 1, (world,), generator=g)
    return [(x * 2.0 ** int(k)).to(dtype) for x, k in zip(xs, ks)]


def torch_result(xs, dtype):
    return adasum_tree(list(xs)).to(dtype)


def fp32_of(q: Fraction) -> float:
    """``q`` rounded once to fp32, to nearest even."""
    c = np.float32(float(q))
    cands = [c, np.nextafter(c, np.float32(-np.inf)), np.nextafter(c, np.float32(np.inf))]
    best = min(abs(Fraction(float(v)) - q) for v in cands)
    near = [v for v in cands if abs(Fraction(float(v)) - q) == best]
    if len(near) > 1:
        near = [v for v in near if not (v.view(np.int32) & 1)]
    return float(near[0])


# ------------------------------------------------------------------------------------------------ the oracle --
@pytest.mark.parametrize("world", [2, 4, 8])
@pytest.mark.parametrize("seed", range(4))
def test_coefficients_equal_exact_rationals(world, seed):
    """Every coefficient the oracle uses is the exact rational ``1 - d / (2 n)`` of its level's fp32 inputs, rounded once."""
    xs = gaussians(world, 5 + 7 * seed, torch.float32, seed) if seed % 2 else spread(world, 33, torch.float32, seed)
    info = {}
    expected(xs, torch.float32, info=info)
    level, k = [x.numpy().astype(np.float32) for x in xs], 0
    while len(level) > 1:
        nxt = []
        for i in range(0, len(level), 2):
            x, y = level[i], level[i + 1]
            fx, fy = [Fraction(float(v)) for v in x], [Fraction(float(v)) for v in y]
            d, na, nb = (sum(p * q for p, q in zip(a, b)) for a, b in ((fx, fy), (fx, fx), (fy, fy)))
            ca, cb = fp32_of(1 - d / (2 * na)), fp32_of(1 - d / (2 * nb))
            assert info["coefs"][k] == (ca, cb), (world, seed, k)
            nxt.append(np.float32(ca) * x + np.float32(cb) * y)
            k += 1
        level = nxt


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("world", [2, 3, 4, 8])
def test_oracle_within_bound_of_float64_tree(dtype, world):
    for seed, xs in enumerate((gaussians(world, 3000, dtype, 1), spread(world, 2000, dtype, 2))):
        want, ref, bound = expected(xs, dtype).double(), tree64(xs), tree64_bound(xs, dtype)
        assert bool(torch.isfinite(bound).all()), "the bound must not be vacuous on well-conditioned inputs"
        assert bool(((want - ref).abs() <= bound).all()), (seed, float(((want - ref).abs() / bound).max()))
        assert float((bound / ref.abs()).median()) < LOOSEST[dtype], "the bound must be tight enough to catch a wrong contract"


def test_float64_tree_bound_catches_a_wrong_contract():
    """A tree with the ``2`` dropped from the coefficients, or summing instead of combining, falls outside the bound."""
    xs = gaussians(4, 3000, torch.float32, 5)
    ref, bound = tree64(xs), tree64_bound(xs, torch.float32)
    ones = [x.double() for x in xs]
    plain_sum = sum(ones)
    assert bool(((plain_sum - ref).abs() > bound).any())

    def no_two(a, b):
        d = float(a @ b)
        return (1 - d / float(a @ a)) * a + (1 - d / float(b @ b)) * b
    wrong = no_two(no_two(ones[0], ones[1]), no_two(ones[2], ones[3]))
    assert bool(((wrong - ref).abs() > bound).any())


def test_tie_guard_fires_on_a_constructed_tie():
    """``1 - d / (2 n)`` exactly on the fp32 midpoint between 0.75 and 0.75 + 2^-24, and just beside it."""
    x = torch.tensor([1.0, 0.0])
    t = 0.5 - 2.0 ** -24                                   # c = 1 - t / 2 = 0.75 + 2^-25: a midpoint
    with pytest.raises(TieError, match="midpoint"):
        expected([x, torch.tensor([t, 0.0])], torch.float32)
    # 2^-40 beside the midpoint: exact sums decide it, but an order-dependent error of 2^-36 in `d` does not
    d = 0.5 - 2.0 ** -24 - 2.0 ** -39                     # c = 0.75 + 2^-25 + 2^-40
    assert coefficient(d, 1.0, 0.0, 0.0) == np.float32(0.75 + 2.0 ** -24)
    with pytest.raises(TieError, match="midpoint"):
        coefficient(d, 1.0, 2.0 ** -36, 0.0)
    with pytest.raises(TieError, match="midpoint"):
        coefficient(d, 1.0, 0.0, 2.0 ** -36)               # an error in the norm moves it as much
    # far from a midpoint the guard is quiet and the coefficient is the fp32 rounding
    assert coefficient(0.25, 1.0, 1e-12, 1e-12) == np.float32(0.875)


def test_kernel_geometry_and_depth():
    nvec, per, blocks = kernel_geometry(1 << 20, torch.float32, 8)
    assert (nvec, per, blocks) == (1 << 18, 1 << 15, 16)
    assert kernel_geometry(1, torch.bfloat16, 2) == (1, 1, 1)
    assert kernel_geometry(1 << 24, torch.float32, 2, emulated=False)[2] == 64
    assert kernel_geometry(1 << 24, torch.float32, 2, max_blocks=3)[2] == 3
    assert kernel_depth(1 << 15, 16, 8, torch.float32) == 4 * 4 + 5 + 16 + 4 + 5


# -------------------------------------------------------------------------------------- the torch tree path --
@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("world", [2, 3, 4, 5, 6, 8])
def test_torch_tree_matches_oracle_bitwise(dtype, world):
    for n in (1, 7, 1000, 4099):
        for fam, xs in (("gauss", gaussians(world, n, dtype, n)), ("spread", spread(world, n, dtype, n + 1))):
            assert_bits(torch_result(xs, dtype), expected(xs, dtype, depth=torch_depth(n), what=f"{fam} seed {n}"),
                        f"torch tree {fam} world {world} n {n}")
    a, b = gaussians(2, 513, dtype, 3)
    assert_bits(adasum_pair(a, b).to(dtype), expected([a, b], dtype), "adasum_pair")


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("k", [-100, -60, 40, 60])
def test_scale_equivariance_is_exact(dtype, k):
    """``adasum(2^k x) == 2^k adasum(x)`` bit for bit while every value the tree forms stays normal."""
    for world in (2, 4, 8):
        g = torch.Generator().manual_seed(world)
        xs = [(torch.sign(torch.randn(999, generator=g)) * (1 + torch.rand(999, generator=g))
               * torch.exp2(torch.randint(-4, 5, (999,), generator=g).float())).to(dtype) for _ in range(world)]
        info = {}
        want = expected(xs, dtype, info=info)
        assert info["min_abs"] * 2.0 ** k >= 2.0 ** -126 and info["max_abs"] * 2.0 ** k < 2.0 ** 127, \
            f"precondition: a value of the tree leaves the normal range at 2^{k} (world {world})"
        scaled = [(x.float() * 2.0 ** k).to(dtype) for x in xs]
        assert_bits(expected(scaled, dtype), (want.float() * 2.0 ** k).to(dtype), f"oracle 2^{k}")
        assert_bits(torch_result(scaled, dtype), (torch_result(xs, dtype).float() * 2.0 ** k).to(dtype), f"torch 2^{k}")


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("value", [1e-17, 2.0 ** -80, 2.0 ** 70], ids=["1e-17", "2^-80", "2^70"])
@pytest.mark.parametrize("world", [2, 4, 8])
def test_identical_tensors_average_at_any_scale(dtype, value, world):
    x = torch.full((4096,), value).to(dtype)
    xs = [x.clone() for _ in range(world)]
    assert_bits(expected(xs, dtype), x, "oracle")
    assert_bits(torch_result(xs, dtype), x, "adasum_tree")
    assert_bits(adasum_pair(x, x).to(dtype), x, "adasum_pair")


def test_nonfinite_inputs_follow_ieee():
    """NaN / Inf in one rank: NaN coefficients (``n > 0`` is false for a NaN norm, so that side keeps 1) and NaN outputs."""
    for bad in (math.nan, math.inf, -math.inf):
        xs = gaussians(4, 100, torch.float32, 9)
        xs[1][17] = bad
        want = expected(xs, torch.float32)
        assert bool(torch.isnan(want).all())
        assert_bits(torch_result(xs, torch.float32), want, f"torch tree with {bad}")
