"""Exact oracle of the learning-rate schedule contract (mpi_operator_b200/parallel/lr_schedule.py, csrc/kernels/lr_schedule.cu).

Written from the contract, not from either implementation: every float64 operation is computed exactly in rationals and
rounded to the nearest float64 once (``float(Fraction)`` is correctly rounded), and the rate is that float64 product
rounded to fp32 once. A schedule is the plain dictionary of ``LRSchedule.to_dict()``::

    {"form": "constant" | "piecewise" | "exponential" | "polynomial", "warmup_steps": W, ...form keys}

``k_grid`` lists the step counts where an implementation is most likely to be off by one or to lose bits.
"""
from fractions import Fraction

import numpy as np


def _round64(q: Fraction) -> float:
    try:
        return float(q)
    except OverflowError:
        return float("inf") if q > 0 else float("-inf")


def add(a: float, b: float) -> float:
    return _round64(Fraction(a) + Fraction(b))


def sub(a: float, b: float) -> float:
    return _round64(Fraction(a) - Fraction(b))


def mul(a: float, b: float) -> float:
    if np.isinf(a) or np.isinf(b):
        return a * b
    return _round64(Fraction(a) * Fraction(b))


def div(a: float, b: float) -> float:
    return _round64(Fraction(a) / Fraction(b))


def pow_int(x: float, n: int) -> float:
    """Right-to-left binary exponentiation, each multiply rounded to float64."""
    r, b = 1.0, float(x)
    while n > 0:
        if n % 2 == 1:
            r = mul(r, b)
        b = mul(b, b)
        n //= 2
    return r


def multiplier(spec: dict, k: int) -> float:
    W = int(spec.get("warmup_steps", 0))
    if k < W:
        return div(float(k), float(W))
    form = spec["form"]
    if form == "constant":
        return 1.0
    if form == "piecewise":
        i = len([b for b in spec["boundaries"] if b < k])     # value 0 while k <= boundaries[0]
        return float(spec["multipliers"][i])
    if form == "exponential":
        p = pow_int(float(spec["factor"]), k // int(spec["decay_steps"]))
        return max(p, float(spec.get("floor", 0.0)))
    if form == "polynomial":
        T, end = int(spec["total_steps"]), float(spec.get("end", 0.0))
        if k >= T:
            return end
        t = div(float(k - W), float(T - W))
        return add(end, mul(sub(1.0, end), pow_int(sub(1.0, t), int(spec.get("power", 2)))))
    raise ValueError(f"unknown form {form!r}")


def rate(spec: dict, base: float, k: int) -> np.float32:
    """``fp32_rn(base * m(k))``."""
    with np.errstate(over="ignore"):
        return np.float32(mul(float(base), multiplier(spec, k)))


def _step(x: float, j: int) -> float:
    """``x`` moved by ``j`` float64 ulps."""
    for _ in range(abs(j)):
        x = float(np.nextafter(x, np.inf if j > 0 else -np.inf))
    return x


def edge_bases(m: float, reach: int = 2) -> list:
    """Base rates whose products with ``m`` straddle fp32 rounding midpoints, ``-reach .. reach`` float64 ulps around
    ``midpoint / m``: their fp32 rates show a change in the last bits of the float64 multiplier. Empty unless ``m`` is
    finite and > 0."""
    if not (np.isfinite(m) and m > 0):
        return []
    out = []
    for v in (np.float32(1.5), np.float32(0.1), np.float32(3e-4)):
        b = div(float(v) + float(np.spacing(v)) / 2, m)      # the midpoint is exact in float64
        out += [_step(b, j) for j in range(-reach, reach + 1)]
    return out


def k_grid(spec: dict) -> list:
    """0, 1, W - 1, W, W + 1, every boundary / decay multiple / T and its neighbours, 2^31 + 5 and 2^40 (ascending, >= 0).
    Decay multiples are taken up to 70 periods and around the two large k."""
    W = int(spec.get("warmup_steps", 0))
    ks = {0, 1, W - 1, W, W + 1, (1 << 31) + 5, 1 << 40}
    marks = []
    if spec["form"] == "piecewise":
        marks = list(spec["boundaries"])
    elif spec["form"] == "exponential":
        d = int(spec["decay_steps"])
        marks = [d * j for j in range(1, 71)] + [(1 << 31) + 5 - ((1 << 31) + 5) % d, (1 << 40) - (1 << 40) % d]
    elif spec["form"] == "polynomial":
        T = int(spec["total_steps"])
        marks = [T] + [W + (T - W) * j // 7 for j in range(1, 7)]
    for b in marks:
        ks.update((b - 1, b, b + 1))
    return sorted(k for k in ks if k >= 0)
