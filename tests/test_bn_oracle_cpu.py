"""The BatchNorm oracle (tests/bn_oracle.py) on the CPU: its plan follows plan()'s rules, its sums are as accurate as fp32
summation allows against float64 and exact rationals (so it is not merely a transcription of the kernel), and it tells
apart the kernel mistakes the GPU tests are meant to catch."""
from fractions import Fraction

import numpy as np
import pytest

import bn_oracle as O

F32 = np.float32
U = 2.0 ** -24


def gamma(n):
    return n * U / (1 - n * U)


def bf16_data(shape, seed, loc=0.0, scale=1.0):
    rng = np.random.default_rng(seed)
    x = (rng.standard_normal(shape) * scale + loc).astype(F32)
    return O.bf16_value(O.bf16(x))


@pytest.mark.parametrize("c", O.CHANNELS)
def test_plan_follows_the_rules_at_every_channel_count(c):
    rpp = O.rows_per_pass(c)
    assert O.supported(1, c) and rpp * (c // 8) == O.THREADS
    for m in (1, 2, 3, max(1, rpp - 1), rpp * 64 - 1, rpp * 64 + 1, 12345, 200704, 802816):
        for cap, bpr, chunk in ((O.MAX_PARTS, 2 * c, O.REDUCE_CHUNK), (O.MAX_PARTS, 4 * c, O.REDUCE_CHUNK),
                                (O.ELEM_CAP, 6 * c, O.ELEM_CHUNK), (O.MAX_PARTS, 2 * c, 1), (O.MAX_PARTS, 2 * c, 10 ** 15)):
            g, rows = O.plan(m, c, cap, bpr, chunk)
            assert rows % rpp == 0 and 1 <= g <= cap
            assert (g - 1) * rows < m <= g * rows          # every CTA has rows, and they cover M
            want = max(1, min(-(-m // (4 * rpp)), -(-(m * bpr) // chunk), cap))
            assert g <= want                               # rounding rows up to whole passes only removes CTAs
            assert rows - rpp < -(-m // want)              # ... by less than one pass per CTA
    assert not O.supported(0, c)


def test_plan_known_grids():
    assert [O.supported(1, c) for c in (24, 96, 4096)] == [False] * 3
    assert O.plan_rows(802816, 64, 128) == O.plan_rows(802816, 64, 256) == O.MAX_PARTS
    assert O.plan_rows(37888, 64, 128, chunk=1) == O.MAX_PARTS
    assert O.plan_rows(200704, 64, 128, chunk=10 ** 15) == 1
    assert O.plan(1, 2048, O.MAX_PARTS, 4096, O.REDUCE_CHUNK) == (1, 1)


def fsum_rows(x, grid, rows, f):
    """float64 per-CTA sums of f(row) and of |f(row)|."""
    M = x.shape[0]
    out, mag = np.zeros((grid, x.shape[1])), np.zeros((grid, x.shape[1]))
    for g in range(grid):
        v = f(x[g * rows:min(M, (g + 1) * rows)].astype(np.float64))
        out[g], mag[g] = v.sum(0), np.abs(v).sum(0)
    return out, mag


@pytest.mark.parametrize("m,c", [(5000, 64), (777, 8), (4099, 2048), (20000, 256)])
def test_partial_rows_within_fp32_summation_bound_of_float64(m, c):
    x = bf16_data((m, c), m + c, loc=3.0, scale=2.0)
    dz = bf16_data((m, c), m + c + 1)
    mask = np.random.default_rng(m).random((m, c)) < 0.5
    mu = x.astype(np.float64).mean(0).astype(F32)
    for chunk in (O.REDUCE_CHUNK, 1):
        grid, rows = O.plan(m, c, O.MAX_PARTS, 2 * c, chunk)
        P = O.fwd_partials(x, grid, rows).reshape(grid, c, 2)
        K = x[0].astype(np.float64)
        n = rows // O.rows_per_pass(c) + O.rows_per_pass(c) + 1
        for s, f in ((0, lambda v: v - K), (1, lambda v: (v - K) ** 2)):
            ref, mag = fsum_rows(x, grid, rows, f)
            assert (np.abs(P[..., s] - ref) <= gamma(n) * mag).all()
        tot = O.merge(P.reshape(grid, 2 * c))
        ref = P.reshape(grid, 2 * c).astype(np.float64).sum(0)
        assert (np.abs(tot - ref) <= gamma(grid + 8) * np.abs(P.reshape(grid, 2 * c)).astype(np.float64).sum(0)).all()

        grid, rows = O.plan(m, c, O.MAX_PARTS, 4 * c, chunk)
        B = O.bwd_partials(dz, x, mask, mu, grid, rows).reshape(grid, c, 2)
        g64 = np.where(mask, dz, 0).astype(np.float64)
        both = np.concatenate([g64, g64 * (x.astype(np.float64) - mu.astype(np.float64))], 1)
        ref, mag = fsum_rows(both, grid, rows, lambda v: v)
        n = rows + O.rows_per_pass(c) + 1
        assert (np.abs(B[..., 0] - ref[:, :c]) <= gamma(n) * mag[:, :c] + 1e-30).all()
        # g * (x - mu) has two roundings per term (the subtraction and the fma)
        assert (np.abs(B[..., 1] - ref[:, c:]) <= gamma(n + 1) * mag[:, c:] + 1e-30).all()


def test_small_integer_data_is_summed_exactly():
    """Integers below 2^24 in every partial sum: any order gives the exact rational, which the oracle must reproduce."""
    m, c = 3001, 32
    rng = np.random.default_rng(5)
    x = rng.integers(-20, 21, (m, c)).astype(F32)
    grid, rows = O.plan(m, c, O.MAX_PARTS, 2 * c, 1)
    tot = O.merge(O.fwd_partials(x, grid, rows))
    d = [[Fraction(int(v)) - Fraction(int(x[0, j])) for v in x[:, j]] for j in range(c)]
    assert [float(t) for t in tot[0::2]] == [float(sum(col)) for col in d]
    assert [float(t) for t in tot[1::2]] == [float(sum(v * v for v in col)) for col in d]
    out = O.fwd_finalize(tot, x[0], m, None, None, np.zeros(c, F32), np.ones(c, F32), 1e-5, 0.1)
    mean = x.astype(np.float64).mean(0)
    var = x.astype(np.float64).var(0)
    K = x[0].astype(np.float64)
    # mean = K + S1 * (1/M): three roundings, of the quotient, the product and the sum
    assert (np.abs(out["mean"] - mean) <= 3 * U * (np.abs(K) + np.abs(mean - K))).all()
    # var = fma(-d, d, S2 * (1/M)): the roundings of 1/M, d, S2/M and the fma, on the scale of S2/M and d^2
    assert (np.abs(out["var"] - var) <= 6 * U * (var + 2 * (mean - K) ** 2)).all()
    assert (O.ulps(out["rsqrt_rn"], (1 / np.sqrt(np.float64(out["var"]) + np.float64(F32(1e-5))))) <= 1).all()


def test_walk_merge_recentres_gemm_rows_exactly():
    """Synthetic GEMM partial rows of small integers: the WALK merge gives the sums about x[0] exactly."""
    m, c = 1000, 16
    rng = np.random.default_rng(9)
    x = rng.integers(-8, 9, (m, c)).astype(F32)
    parts = 5
    part = (np.arange(m) // 128) % parts
    P = np.zeros((parts, c, 2), F32)
    for p in range(parts):
        d = x[part == p] - x[p * 128]
        P[p, :, 0], P[p, :, 1] = d.sum(0), (d * d).sum(0)
    tot = O.merge(P.reshape(parts, 2 * c), walk=O.walk_rows(x, parts))
    d = x.astype(np.float64) - x[0]
    assert np.array_equal(tot[0::2], d.sum(0)) and np.array_equal(tot[1::2], (d * d).sum(0))


def test_fma_and_rounding_helpers():
    a = np.array([1 + 2 ** -23, 3.0, np.nan, 2.0 ** 100], F32)
    b = np.array([1 - 2 ** -23, 1 / 3, 1.0, 2.0 ** 100], F32)
    c = np.array([-1.0, -1.0, 0.0, 0.0], F32)
    r = O.fma(a, b, c)
    assert r[0] == F32(-(2.0 ** -46)) and np.isnan(r[2]) and np.isinf(r[3])
    assert r[1] == F32(float(Fraction(3) * Fraction(float(F32(1 / 3))) - 1))
    z = np.array([1 + 2 ** -8, 1 + 3 * 2 ** -8, -0.0, np.nan], F32)     # two ties (to even: down, up), -0, NaN
    assert list(O.bf16(z)[:3]) == [0x3F80, 0x3F82, 0x8000] and O.ties(z) == 2
    y, mask, _ = O.apply(z[None, :], None, np.ones(4, F32), np.zeros(4, F32), relu=True)
    assert list(mask[0]) == [True, True, False, True] and y[0, 2] == 0 and np.isnan(O.bf16_value(y[0, 3]))
    bits = np.random.default_rng(1).random((3, 64)) < 0.5
    assert np.array_equal(O.unpack_mask(O.pack_mask(bits), 3, 64), bits)


# ------------------------------------------------------------------------------------ the kernel's mistakes --
def test_dropped_block_passes_changes_the_partial_rows():
    m, c = 16384, 64
    x = bf16_data((m, c), 1, loc=5.0, scale=1.0)
    grid, rows = O.plan(m, c, O.MAX_PARTS, 2 * c, 10 ** 15)
    assert grid == 1 and rows // O.rows_per_pass(c) > 4 * O.BLOCK_PASSES
    good, bad = O.fwd_partials(x, grid, rows), O.fwd_partials(x, grid, rows, block_passes=1 << 30)
    assert not np.array_equal(good, bad)


def test_reassociated_merge_changes_the_totals():
    P = np.random.default_rng(2).standard_normal((296, 128)).astype(F32)
    assert not np.array_equal(O.merge(P), O.merge(P, order="serial"))
    # fewer than 97 rows never reach the 4-way loop: the orders agree
    assert np.array_equal(O.merge(P[:96]), O.merge(P[:96], order="serial"))


def test_biased_running_variance_and_running_mean_form_change_the_bits():
    m, c = 200704, 64
    rng = np.random.default_rng(3)
    tot = np.stack([rng.standard_normal(c) * 100, rng.random(c) * m * 4 + m], 1).astype(F32).reshape(-1)
    rm, rv = rng.standard_normal(c).astype(F32), (rng.random(c) + 0.5).astype(F32)
    x0 = bf16_data(c, 4)
    good = O.fwd_finalize(tot, x0, m, None, None, rm, rv, 1e-5, 0.1)
    bad = O.fwd_finalize(tot, x0, m, None, None, rm, rv, 1e-5, 0.1, unbiased=False)
    assert not np.array_equal(good["rv"], bad["rv"])
    assert np.allclose(good["rv"], bad["rv"], rtol=1e-5)              # a relative 5e-6: inside the old tolerance
    alt = rm + F32(0.1) * (good["mean"] - rm)
    assert not np.array_equal(good["rm"], alt)


def test_mask_and_rounding_mistakes_change_the_outputs():
    # z exactly 0: a power-of-two constant times a, minus the same product
    x = np.full((4, 8), 0.5, F32)
    a = bf16_data(8, 5) + F32(2)
    _, b = O.eval_coef(a, None, np.full(8, 0.5, F32), np.ones(8, F32))
    y, mask, z = O.apply(x, None, a, b, relu=True)
    assert (z == 0).all() and not mask.any()
    assert O.apply(x, None, a, b, relu=True, mask_ge=True)[1].all()
    # truncation instead of round-to-nearest-even
    z = np.random.default_rng(6).standard_normal(1000).astype(F32)
    trunc = (z.view(np.uint32) >> 16).astype(np.uint16)
    assert not np.array_equal(O.bf16(z), trunc)


def test_backward_contraction_mistakes_change_the_outputs():
    m, c = 4099, 64      # not a power of two: 1/M is inexact
    x = bf16_data((m, c), 7, loc=2.0)
    dz = bf16_data((m, c), 8)
    mask = np.random.default_rng(9).random((m, c)) < 0.5
    mu = x.astype(np.float64).mean(0).astype(F32)
    inv = (1 / x.astype(np.float64).std(0)).astype(F32)
    grid, rows = O.plan(m, c, O.MAX_PARTS, 4 * c, O.REDUCE_CHUNK)
    tot = O.merge(O.bwd_partials(dz, x, mask, mu, grid, rows))
    co = O.bwd_finalize(tot, m, None, mu, inv)
    alt_c3 = co["dgamma"] * (F32(1) / F32(m) * inv)
    assert not np.array_equal(co["c3"], alt_c3)
    _, _, dx32 = O.elemt(dz, x, mask, co, False)
    g = np.where(mask, dz, F32(0))
    alt = co["a"] * (g - co["gm"] - (x * co["c3"] - co["mu"] * co["c3"]))
    # before the bf16 rounding: the difference is a few fp32 ulps, which reaches the bf16 output only near a rounding boundary
    assert not np.array_equal(dx32, alt)
