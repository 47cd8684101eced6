"""The weight-average oracle (tests/ema_oracle.py) is exact, and it tells apart the plausible ways a kernel could get the
update wrong: an unfused multiply-add, c_k in fp32, k off by one, the pre-update parameters, no warm-up."""
from fractions import Fraction

import numpy as np
import pytest

from ema_oracle import _round_exact, ema_coef, ema_step, fma32


def _inputs(n=4096, seed=0):
    rng = np.random.default_rng(seed)
    e = rng.standard_normal(n).astype(np.float32)
    p = (e + rng.standard_normal(n).astype(np.float32) * np.float32(1e-3)).astype(np.float32)
    scale = np.float32(2.0) ** rng.integers(-60, 61, n).astype(np.float32)
    e, p = (e * scale).astype(np.float32), (p * scale).astype(np.float32)
    e[:8] = [0, -0.0, 1e-45, -1e-45, 3e-39, 2.0 ** 60, -(2.0 ** -60), 1.0]    # zeros, subnormals, 2^±60
    p[:8] = [0, 1e-45, -1e-45, 0, -3e-39, 2.0 ** 60 + 2.0 ** 37, 2.0 ** -60, 1.0 + 2.0 ** -23]
    return e, p


def _fma_fraction(a, b, c):
    """fp32 fma by exact rational arithmetic on every element: the independent emulation the oracle must match."""
    out = np.empty_like(c)
    for i in range(c.size):
        x = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
        out[i] = _round_exact(x, np.float32(float(x)))
    return out


def _exact(e, p, d, k):
    c = np.full_like(e, np.float32(1.0 - min(float(np.float32(d)), (1.0 + k) / (10.0 + k))))
    return _fma_fraction(c, p - e, e)


def _bits(x):
    return np.asarray(x, dtype=np.float32).view(np.uint32)


@pytest.mark.parametrize("d", [0.5, 0.999, 0.9999])
@pytest.mark.parametrize("k", [1, 2, 7, 1000, 10 ** 6])
def test_oracle_equals_rational_fma(d, k):
    e, p = _inputs(2048, seed=k)
    assert np.array_equal(_bits(ema_step(e, p, d, k)), _bits(_exact(e, p, d, k)))


def test_fma_rounds_boundary_cases_exactly():
    u = 2.0 ** -23
    # float64 sums exactly on an fp32 midpoint whose exact value lies just below (t < 0) or just above (t > 0) it: the
    # naive rounding of the float64 sum, ties to even, is wrong in both; and two exact ties (t == 0), ties to even
    a = np.array([1 + u, -(1 + u), 1, 1], dtype=np.float32)
    b = np.array([2.0 ** -24 * (1 - u), 2.0 ** -24 * (1 - u), 2.0 ** -24, 2.0 ** -24], dtype=np.float32)
    c = np.array([1 + u, 1 + 3 * u, 1, 1 + u], dtype=np.float32)
    want = np.array([1 + u, 1 + 3 * u, 1, 1 + 2 * u], dtype=np.float32)
    prod = a.astype(np.float64) * b.astype(np.float64)
    s64 = prod + c.astype(np.float64)
    t = (prod - (s64 - (s64 - prod))) + (c.astype(np.float64) - (s64 - prod))
    assert list(np.sign(t)) == [-1, 1, 0, 0]                     # the branches the inputs are meant to reach
    naive = s64.astype(np.float32)
    assert not np.array_equal(_bits(naive[:2]), _bits(want[:2]))
    assert np.array_equal(_bits(fma32(a, b, c)), _bits(want))
    assert np.array_equal(_bits(_fma_fraction(a, b, c)), _bits(want))


def test_schedule():
    assert ema_coef(0.9999, 1) == np.float32(1 - 2 / 11)
    assert ema_coef(0.5, 1) == np.float32(1 - 2 / 11)            # the warm-up term is the smaller one at first
    assert ema_coef(0.5, 8) == np.float32(0.5)                   # from k = 8 on, d = 0.5 is
    assert ema_coef(0.999, 10 ** 7) == np.float32(1.0 - float(np.float32(0.999)))
    ks = [ema_coef(0.9999, k) for k in range(1, 200)]
    assert all(a >= b for a, b in zip(ks, ks[1:]))                # the warm-up only ever lowers the coefficient


def _mutations(e, p_old, p, d, k):
    c = ema_coef(d, k)
    diff = p - e
    c32 = np.float32(1) - np.minimum(np.float32(d), (np.float32(1) + np.float32(k)) / (np.float32(10) + np.float32(k)))
    return {
        "unfused multiply then add": (c * diff).astype(np.float32) + e,
        "c_k in fp32": fma32(np.full_like(e, c32), diff, e),
        "k + 1": ema_step(e, p, d, k + 1),
        "k - 1": ema_step(e, p, d, k - 1) if k > 1 else ema_step(e, p, d, k + 2),
        "pre-update parameters": ema_step(e, p_old, d, k),
        "no warm-up": fma32(np.full_like(e, np.float32(1.0 - float(np.float32(d)))), diff, e),
    }


@pytest.mark.parametrize("d,k", [(0.999, 9), (0.9999, 12), (0.9999, 37)])   # k where c_k in fp32 differs
def test_oracle_rejects_each_mutation(d, k):
    e, p_old = _inputs(4096, seed=3)
    p = (p_old - np.float32(1e-2) * p_old).astype(np.float32)
    want = ema_step(e, p, d, k)
    for name, got in _mutations(e, p_old, p, d, k).items():
        assert not np.array_equal(_bits(got), _bits(want)), name
