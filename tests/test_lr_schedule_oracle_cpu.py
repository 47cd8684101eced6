"""The learning-rate schedule oracle (tests/lr_schedule_oracle.py) against hand-worked values, and proof that it tells
apart six plausible implementation mistakes on the step counts of its own grid."""
from fractions import Fraction

import numpy as np
import pytest

import lr_schedule_oracle as O

# the schedules every mutant is tried on, and the GPU tests use
SPECS = [
    {"form": "constant", "warmup_steps": 0},
    {"form": "constant", "warmup_steps": 7},
    {"form": "piecewise", "warmup_steps": 0, "boundaries": [3, 10, 1000], "multipliers": [1.0, 0.1, 0.01, 0.001]},
    {"form": "piecewise", "warmup_steps": 5, "boundaries": [3, 10, 1000], "multipliers": [1.0, 0.1, 0.01, 0.001]},
    {"form": "exponential", "warmup_steps": 0, "decay_steps": 3, "factor": 0.94, "floor": 0.0},
    {"form": "exponential", "warmup_steps": 10, "decay_steps": 3, "factor": 0.94, "floor": 0.3},
    {"form": "polynomial", "warmup_steps": 0, "total_steps": 97, "power": 2, "end": 0.0},
    {"form": "polynomial", "warmup_steps": 13, "total_steps": 97, "power": 3, "end": 0.0001},
]
BASES = [0.1, 1.7, 12.8, 3e-4]


def _differs(fn, specs=SPECS):
    """Does ``fn(spec, k)`` give another rate than the oracle anywhere on the grids, with the fixed bases or the ones that
    straddle an fp32 midpoint?"""
    for spec in specs:
        for k in O.k_grid(spec):
            for base in BASES + O.edge_bases(O.multiplier(spec, k)):
                want = O.rate(spec, base, k)
                with np.errstate(over="ignore"):
                    got = np.float32(float(base) * float(fn(spec, k)))
                if got.view(np.int32) != want.view(np.int32):
                    return True
    return False


def test_hand_worked_values():
    pw = {"form": "piecewise", "warmup_steps": 0, "boundaries": [3, 10], "multipliers": [1.0, 0.5, 0.25]}
    assert [O.multiplier(pw, k) for k in (0, 3, 4, 10, 11)] == [1.0, 1.0, 0.5, 0.5, 0.25]
    ex = {"form": "exponential", "warmup_steps": 0, "decay_steps": 2, "factor": 0.5, "floor": 0.2}
    assert [O.multiplier(ex, k) for k in (0, 1, 2, 3, 4, 6)] == [1.0, 1.0, 0.5, 0.5, 0.25, 0.2]
    po = {"form": "polynomial", "warmup_steps": 2, "total_steps": 6, "power": 2, "end": 0.0}
    assert [O.multiplier(po, k) for k in (0, 1, 2, 4, 5, 6, 9)] == [0.0, 0.5, 1.0, 0.25, 0.0625, 0.0, 0.0]
    # each operation is rounded once: 1/3 then 1 - 1/3 then its square, not (2/3)^2 exactly
    po3 = {"form": "polynomial", "warmup_steps": 0, "total_steps": 3, "power": 2, "end": 0.0}
    x = float(Fraction(1) - Fraction(1 / 3))
    assert O.multiplier(po3, 1) == float(Fraction(x) * Fraction(x))
    assert O.rate(pw, 0.1, 4) == np.float32(0.05)


def test_operations_are_correctly_rounded():
    rng = np.random.default_rng(0)
    for a, b in rng.uniform(-2, 2, (200, 2)):
        assert O.add(a, b) == a + b and O.mul(a, b) == a * b and O.div(a, b) == a / b and O.sub(a, b) == a - b
    assert O.pow_int(0.94, 0) == 1.0 and O.pow_int(0.0, 5) == 0.0


def test_grid_hits_the_edges():
    assert O.k_grid(SPECS[3])[:7] == [0, 1, 2, 3, 4, 5, 6]
    g = O.k_grid(SPECS[6])
    assert {96, 97, 98, (1 << 31) + 5, 1 << 40} <= set(g)


def test_rejects_warmup_counted_from_one():
    def mutant(spec, k):
        W = spec.get("warmup_steps", 0)
        if k < W:
            return (k + 1) / W
        return O.multiplier(spec, k)
    assert _differs(mutant)


def test_rejects_less_than_instead_of_less_equal_at_a_boundary():
    def mutant(spec, k):
        if spec["form"] != "piecewise" or k < spec.get("warmup_steps", 0):
            return O.multiplier(spec, k)
        return spec["multipliers"][len([b for b in spec["boundaries"] if b <= k])]
    assert _differs(mutant)


def test_rejects_non_staircase_decay():
    def mutant(spec, k):
        if spec["form"] != "exponential" or k < spec.get("warmup_steps", 0):
            return O.multiplier(spec, k)
        return max(spec["factor"] ** (k / spec["decay_steps"]), spec["floor"])
    assert _differs(mutant)


def test_rejects_floor_applied_before_the_warmup():
    def mutant(spec, k):
        m = O.multiplier(spec, k)
        return max(m, spec.get("floor", 0.0)) if spec["form"] == "exponential" else m
    assert _differs(mutant)


def test_rejects_multiplier_in_fp32():
    def mutant(spec, k):
        f = np.float32
        W = spec.get("warmup_steps", 0)
        if k < W:
            return f(k) / f(W)
        if spec["form"] == "polynomial":
            T, end = spec["total_steps"], f(spec["end"])
            if k >= T:
                return end
            t = f(k - W) / f(T - W)
            return end + (f(1) - end) * (f(1) - t) ** spec["power"]
        if spec["form"] == "exponential":
            return max(f(spec["factor"]) ** (k // spec["decay_steps"]), f(spec["floor"]))
        return O.multiplier(spec, k)
    with np.errstate(all="ignore"):
        assert _differs(mutant)


def test_rejects_pow_by_left_to_right_multiplication():
    def pow_ltr(x, n):
        r = 1.0
        for _ in range(n):
            r, prev = r * x, r     # one correctly rounded float64 multiply
            if r == prev:          # a fixed point (0, or the least subnormal that x < 1 rounds back to itself)
                break
        return r

    def mutant(spec, k):
        if spec["form"] == "exponential" and k >= spec.get("warmup_steps", 0):
            return max(pow_ltr(spec["factor"], k // spec["decay_steps"]), spec["floor"])
        if spec["form"] == "polynomial" and spec.get("warmup_steps", 0) <= k < spec["total_steps"]:
            W, T, end = spec.get("warmup_steps", 0), spec["total_steps"], spec["end"]
            t = O.div(float(k - W), float(T - W))
            return O.add(end, O.mul(O.sub(1.0, end), pow_ltr(O.sub(1.0, t), spec["power"])))
        return O.multiplier(spec, k)
    assert _differs(mutant)


@pytest.mark.parametrize("spec", SPECS, ids=[f"{s['form']}-W{s['warmup_steps']}" for s in SPECS])
def test_oracle_is_not_its_own_mutant(spec):
    assert not _differs(O.multiplier, [spec])
