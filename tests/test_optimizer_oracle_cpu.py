"""tests/optimizer_oracle.py on the CPU: the owner-order sum against a plain loop, every operation against exact rationals,
the exactness precondition, and a list of plausible kernel mistakes that the oracle must tell apart from the contract."""
from fractions import Fraction

import numpy as np
import pytest
import torch

from optimizer_oracle import (bf16_bits, fma, fmul, lars_norm_interval, lars_step, lars_trust, owner_sum, sgd_step,
                              slice_vecs, vec_elems)

F32 = np.float32


def _rng(seed):
    return np.random.default_rng(seed)


def _q(x):
    return Fraction(float(x))


def _rn32(x: Fraction) -> np.float32:
    """Round a rational to the nearest fp32, ties to even (finite, no overflow)."""
    near = F32(float(x))
    best = None
    for c in (np.nextafter(near, F32(-np.inf)), near, np.nextafter(near, F32(np.inf))):
        dist = abs(_q(c) - x)
        if best is None or dist < best[0] or (dist == best[0] and int(c.view(np.uint32)) & 1 == 0):
            best = (dist, c)
    return F32(best[1])


def _same(got, want):
    """Bitwise, except that a rational has no signed zero: a zero matches either zero (IEEE's signs come from numpy)."""
    return got == 0 if want == 0 else got.view(np.int32) == want.view(np.int32)


# ------------------------------------------------------------------------------------------------------ owner_sum --
@pytest.mark.parametrize("world", range(1, 9))
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16], ids=["f32", "bf16"])
@pytest.mark.parametrize("nvec", [1, 3, 1013])
def test_owner_sum_is_the_owner_order_loop(world, dtype, nvec):
    N = vec_elems(dtype)
    n = nvec * N
    rng = _rng(world * 100 + nvec)
    grads = [(rng.standard_normal(n) * 10.0 ** rng.integers(-3, 4, n)).astype(F32) for _ in range(world)]
    per = slice_vecs(n, world, dtype)
    want = np.empty(n, F32)
    for e in range(n):
        owner = (e // N) // per                        # empty slices (owner > last used rank) simply own nothing
        acc = grads[owner][e]
        for k in range(1, world):
            acc = F32(acc + grads[(owner + k) % world][e])
        want[e] = acc
    got = owner_sum(grads, world, dtype)
    assert np.array_equal(got.view(np.int32), want.view(np.int32))


def test_owner_sum_nvls_needs_exact_sums():
    g = [np.array([1.0, 2.0 ** 30, 0, 0], F32), np.array([2.0 ** -30, -(2.0 ** 30), 0, 0], F32)]
    with pytest.raises(AssertionError, match="precondition"):
        owner_sum(g, 2, torch.float32, nvls=True)
    g = [np.array([1.0, 0.5, 0, 0, 0, 0, 0, 0], F32), np.array([2.0 ** -8, 0.25, 0, 0, 0, 0, 0, 0], F32)]
    got = owner_sum(g, 2, torch.bfloat16, nvls=True)            # 1 + 2^-8 is a bf16 tie: back to 1
    assert got[0] == 1.0 and got[1] == 0.75


# ---------------------------------------------------------------------------------------------- exact rationals --
def _sgd_fraction(p, m, S, scale, lr, mu, wd, nesterov, first, trust=None):
    d = _rn32(_q(S) * _q(scale) + _q(_rn32(_q(wd) * _q(p))))
    if trust is not None:
        d = _rn32(_q(trust) * _q(d))
    mn = d if first else _rn32(_q(mu) * _q(m) + _q(d))
    upd = _rn32(_q(mu) * _q(mn) + _q(d)) if nesterov else mn
    return _rn32(-_q(lr) * _q(upd) + _q(p)), mn


@pytest.mark.parametrize("nesterov", [False, True])
@pytest.mark.parametrize("first", [False, True])
def test_sgd_step_against_fractions(nesterov, first):
    rng = _rng(int(nesterov) * 2 + int(first))
    n = 400
    p = (rng.standard_normal(n) * 2.0 ** rng.integers(-20, 20, n)).astype(F32)
    m = (rng.standard_normal(n) * 2.0 ** rng.integers(-20, 20, n)).astype(F32)
    S = (rng.standard_normal(n) * 2.0 ** rng.integers(-20, 20, n)).astype(F32)
    p[:4] = [1e-45, -3e-39, 0.0, -0.0]                          # subnormal and signed-zero parameters
    S[:4] = [2e-45, 1e-40, -0.0, 0.0]
    lr, mu, wd = rng.uniform(0, 1, n).astype(F32), rng.uniform(0, 1, n).astype(F32), rng.uniform(0, 1e-2, n).astype(F32)
    trust = rng.uniform(0, 2, n).astype(F32)
    for t in (None, trust):
        pn, mn, sh = sgd_step(p, m, S, F32(0.125 / 3), lr, mu, wd, nesterov, first, trust=t)
        for i in range(n):
            wp, wm = _sgd_fraction(p[i], m[i], S[i], F32(0.125 / 3), lr[i], mu[i], wd[i], nesterov, first,
                                   None if t is None else t[i])
            assert _same(pn[i], wp) and _same(mn[i], wm), i
        assert np.array_equal(sh, bf16_bits(pn))


def test_fma_rounds_constructed_midpoints_once():
    """a*b lands exactly half an ulp from c's grid, the float64 sum is a midpoint, and only the exact value decides."""
    cases = []
    for k in range(1, 60):
        a = F32(1 + 2.0 ** -12)
        b = F32(1 + 2.0 ** -12 + k * 2.0 ** -23)
        c = F32(-(1 + 2.0 ** -11))
        cases.append((a, b, c))
        cases.append((F32(1 + 2.0 ** -23), F32(1 + 2.0 ** -23 * k), F32(1.0)))
    a, b, c = (np.array(v, F32) for v in zip(*cases))
    got = fma(a, b, c)
    for i in range(len(cases)):
        assert got[i].view(np.int32) == _rn32(_q(a[i]) * _q(b[i]) + _q(c[i])).view(np.int32), i
    naive = (a * b + c).astype(F32)                                # two roundings
    assert not np.array_equal(naive, got)


def test_fma_and_shadow_non_finite_and_ties():
    assert np.isnan(fma(np.nan, 1, 1)) and fma(np.inf, 2, 1) == np.inf and np.isnan(fma(np.inf, 0, 1))
    assert fma(F32(3e38), F32(2), F32(0)) == np.inf
    ties = np.array([1 + 2.0 ** -8, 1 + 3 * 2.0 ** -8, -(1 + 2.0 ** -8), 3 * 2.0 ** -134, 5 * 2.0 ** -134], F32)
    assert list(bf16_bits(ties)) == [0x3F80, 0x3F82, 0xBF80, 0x0002, 0x0002]      # normal and subnormal ties to even
    assert bf16_bits(F32(np.inf)) == 0x7F80 and bf16_bits(F32(3.4028235e38)) == 0x7F80


# -------------------------------------------------------------------------------------------------------- LARS --
def _trust_fraction(sg, sp, eta, wd):
    gn, wn = F32(np.sqrt(F32(sg))), F32(np.sqrt(F32(sp)))
    if not (wn > 0 and gn > 0):
        return F32(1)
    den = _rn32(_q(_rn32(_q(wd) * _q(wn) + _q(gn))) + _q(F32(1e-8)))
    return _rn32(_q(_rn32(_q(eta) * _q(wn))) / _q(den))


def test_lars_trust_against_fractions():
    rng = _rng(5)
    n = 300
    sg = (rng.uniform(0, 4, n) * 2.0 ** rng.integers(-60, 60, n)).astype(F32)
    sp = (rng.uniform(0, 4, n) * 2.0 ** rng.integers(-60, 60, n)).astype(F32)
    sg[:3], sp[3:6] = 0, 0
    eta, wd = F32(0.001), rng.uniform(0, 1e-2, n).astype(F32)
    got = lars_trust(sg, sp, eta, wd)
    for i in range(n):
        assert got[i].view(np.int32) == _trust_fraction(sg[i], sp[i], eta, wd[i]).view(np.int32), i
    assert (got[:6] == 1).all()
    assert lars_trust(F32(np.nan), F32(1), eta, F32(0)) == 1 and lars_trust(F32(np.inf), F32(1), eta, F32(0)) == 0


def _exact_grads(rng, n, world):
    """gs on a 2^-8 grid with small integer multiples, w on a 2^-8 grid: every order of the sums of squares is exact."""
    gs = (rng.integers(-24, 25, n) * 2.0 ** -8 / world).astype(F32)
    w = (rng.integers(-31, 32, n) * 2.0 ** -8).astype(F32)
    return gs, w


@pytest.mark.parametrize("world", [1, 2, 4, 8])
def test_lars_exact_family_is_order_free(world):
    rng = _rng(world)
    gs, w = _exact_grads(rng, 4 * 3001, world)
    lo, hi = lars_norm_interval(gs, w, world, F32(0.5), F32(1e-3), exact=True)
    assert lo == hi
    for _ in range(3):                                            # any order of fp32 adds gives the same sums
        perm = rng.permutation(gs.size)
        sg = np.cumsum(gs[perm] * gs[perm], dtype=F32)[-1]       # squares are exact; sequential and pairwise orders
        sp = np.add.reduce(w[perm] * w[perm], dtype=F32)
        assert float(lars_trust(sg, sp, F32(0.5), F32(1e-3))) == lo


def test_lars_exactness_precondition_fires():
    gs = np.array([1.0, 2.0 ** -13, 2.0 ** -13, 0.5], F32)        # 1 + 2^-26 + 2^-26: order-dependent in fp32
    w = np.ones(4, F32)
    with pytest.raises(AssertionError, match="precondition"):
        lars_norm_interval(gs, w, 1, F32(0.5), F32(0), exact=True)
    lo, hi = lars_norm_interval(gs, w, 1, F32(0.5), F32(0))
    assert lo < hi


def test_lars_interval_contains_every_order():
    rng = _rng(9)
    gs = (rng.standard_normal(5000) * 1e-2).astype(F32)
    w = rng.standard_normal(5000).astype(F32)
    lo, hi = lars_norm_interval(gs, w, 8, F32(0.02), F32(1e-4))
    assert 0 < lo < hi and (hi - lo) / lo < 1e-3
    for _ in range(4):
        perm = rng.permutation(gs.size)
        sg = np.add.reduce(gs[perm].astype(F32) ** 2, dtype=F32)
        sp = np.add.reduce(w[perm].astype(F32) ** 2, dtype=F32)
        assert lo <= float(lars_trust(sg, sp, F32(0.02), F32(1e-4))) <= hi


# ------------------------------------------------------------------------------------------- mistakes rejected --
def _case(seed=11, n=4096, world=4):
    rng = _rng(seed)
    grads = [(rng.standard_normal(n) * 2.0 ** rng.integers(-8, 8, n)).astype(F32) for _ in range(world)]
    p = (rng.standard_normal(n) * 2.0 ** rng.integers(-4, 4, n)).astype(F32)
    m = (rng.standard_normal(n) * 1e-2).astype(F32)
    return grads, p, m


SC, LR, MU, WD = F32(0.25 / 3), F32(0.1), F32(0.9), F32(1e-2)


def _differs(a, b):
    return not np.array_equal(np.asarray(a).view(np.int32 if np.asarray(a).dtype == F32 else np.int16),
                              np.asarray(b).view(np.int32 if np.asarray(b).dtype == F32 else np.int16))


def _oracle(grads, p, m, nesterov=False, world=4):
    S = owner_sum(grads, world, torch.float32)
    return S, sgd_step(p, m, S, SC, LR, MU, WD, nesterov, False)


def test_rejects_other_contraction():
    grads, p, m = _case()
    S, (pn, mn, _) = _oracle(grads, p, m)
    d = fma(WD, p, fmul(S, SC))
    assert _differs(fma(MU, m, d), mn)


def test_rejects_two_roundings():
    grads, p, m = _case()
    S, (pn, mn, _) = _oracle(grads, p, m)
    d = np.add(fmul(S, SC), fmul(WD, p), dtype=F32)
    assert _differs(fma(MU, m, d), mn)


def test_rejects_sum_from_rank_zero():
    grads, p, m = _case()
    S, (pn, _, _) = _oracle(grads, p, m)
    S0 = grads[0].copy()
    for g in grads[1:]:
        S0 = S0 + g
    assert _differs(S0, S) and _differs(sgd_step(p, m, S0, SC, LR, MU, WD, False, False)[0], pn)


def test_rejects_scale_per_rank():
    grads, p, m = _case()
    S, (pn, _, _) = _oracle(grads, p, m)
    Ss = owner_sum([fmul(g, SC) for g in grads], 4, torch.float32)
    got = fma(-LR, fma(MU, m, np.add(Ss, fmul(WD, p), dtype=F32)), p)
    assert _differs(got, pn)


def test_rejects_nesterov_with_old_momentum():
    grads, p, m = _case()
    S, (pn, mn, _) = _oracle(grads, p, m, nesterov=True)
    d = fma(S, SC, fmul(WD, p))
    assert _differs(fma(-LR, fma(MU, m, d), p), pn)


def test_rejects_truncated_shadow():
    grads, p, m = _case()
    _, (pn, _, sh) = _oracle(grads, p, m)
    trunc = (pn.view(np.uint32) >> 16).astype(np.uint16)
    assert _differs(trunc, sh)


def _lars_case(seed=3):
    rng = _rng(seed)
    sg = (rng.uniform(0.5, 4, 2000) * 2.0 ** rng.integers(-20, 0, 2000)).astype(F32)
    sp = rng.uniform(1, 400, 2000).astype(F32)
    return sg, sp, F32(0.02), F32(0.05)


def test_rejects_unfused_trust_denominator():
    sg, sp, eta, wd = _lars_case()
    gn, wn = np.sqrt(sg), np.sqrt(sp)
    den = np.add(np.add(fmul(wd, wn), gn, dtype=F32), F32(1e-8), dtype=F32)
    assert _differs(np.divide(fmul(eta, wn), den, dtype=F32), lars_trust(sg, sp, eta, wd))


def test_rejects_eps_before_the_fma():
    sg, sp, eta, wd = _lars_case()
    gn, wn = np.sqrt(sg), np.sqrt(sp)
    den = fma(wd, wn, np.add(gn, F32(1e-8), dtype=F32))
    assert _differs(np.divide(fmul(eta, wn), den, dtype=F32), lars_trust(sg, sp, eta, wd))


def test_rejects_trust_on_the_gradient_only():
    grads, p, m = _case()
    S = owner_sum(grads, 4, torch.float32)
    t = F32(0.37)
    pn, mn, _ = lars_step(p, m, S, SC, t, LR, MU, WD, False, False)
    d = fma(fmul(t, fmul(S, SC)), F32(1), fmul(WD, p))
    assert _differs(fma(MU, m, d), mn)
