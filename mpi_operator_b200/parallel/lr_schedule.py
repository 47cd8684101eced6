"""Learning-rate schedules that the trainer evaluates on the device, inside its captured step.

An ``LRSchedule`` is a multiplier ``m(k)`` of the step count ``k`` (the synchronising steps completed before the current
one: 0 for the first update, as tf's ``global_step``). Group g's rate for the step is ``fp32_rn(base_g * m(k))`` with
``base_g`` the group's learning rate as a Python float.

``warmup_steps=W`` gives ``m = k / W`` for ``k < W`` (a ramp from 0 to the base rate, tf_cnn_benchmarks'
``--num_learning_rate_warmup_epochs``); for ``k >= W``:

* ``constant()``: 1;
* ``piecewise(boundaries, multipliers)``: ``multipliers[i]`` with ``i`` the number of boundaries ``b < k``
  (``tf.train.piecewise_constant``);
* ``exponential(decay_steps, factor, floor)``: ``max(factor ** (k // decay_steps), floor)`` (staircase
  ``tf.train.exponential_decay`` with tf_cnn_benchmarks' ``--minimum_learning_rate``);
* ``polynomial(total_steps, power, end)``: ``end + (1 - end) * (1 - (k - W) / (T - W)) ** power`` for ``k < T``, ``end``
  after (MLPerf ResNet's LARS decay).

Every operation is one IEEE float64 add, multiply or divide in the order written, with no contraction; integer powers are
right-to-left binary exponentiation. Python floats follow the same rules, so ``multiplier`` here and the kernel
(csrc/kernels/lr_schedule.cu) give the same bits. Cosine and arbitrary callables are left out on purpose: the host's and
CUDA's ``cos`` / ``pow`` are not bit-identical.
"""
from __future__ import annotations

import math
import operator
from typing import List, Sequence

import numpy as np

MAX_BOUNDARIES = 64          # the kernel keeps the table in one float64 array of at most 2 * 64 + 2 entries
MAX_POWER = 64
_INT_LIMIT = 1 << 53         # step counts and boundaries are exact in float64 below it

CONSTANT, PIECEWISE, EXPONENTIAL, POLYNOMIAL = 0, 1, 2, 3
_FORMS = {CONSTANT: "constant", PIECEWISE: "piecewise", EXPONENTIAL: "exponential", POLYNOMIAL: "polynomial"}


def _int(name: str, v, lo: int = 0) -> int:
    if isinstance(v, bool):
        raise ValueError(f"{name} must be an int, got {v!r}")
    try:
        i = operator.index(v)
    except TypeError:
        raise ValueError(f"{name} must be an int, got {v!r}") from None
    if not lo <= i < _INT_LIMIT:
        raise ValueError(f"{name} must be an int in [{lo}, 2**53), got {i}")
    return i


def _real(name: str, v) -> float:
    if isinstance(v, bool):
        raise ValueError(f"{name} must be a number, got {v!r}")
    try:
        f = float(v)
    except (TypeError, ValueError):
        raise ValueError(f"{name} must be a number, got {v!r}") from None
    if not (math.isfinite(f) and f >= 0.0):
        raise ValueError(f"{name} must be finite and >= 0, got {v!r}")
    return f


def pow_int(x: float, n: int) -> float:
    """``x ** n`` by right-to-left binary exponentiation, one float64 multiply per step (the kernel's order)."""
    r, b = 1.0, x
    while n:
        if n & 1:
            r *= b
        b *= b
        n >>= 1
    return r


class LRSchedule:
    """A learning-rate multiplier ``m(k)``; build one with ``constant``, ``piecewise``, ``exponential`` or ``polynomial``."""

    def __init__(self, form: int, warmup_steps: int = 0, boundaries: Sequence[int] = (), multipliers: Sequence[float] = (),
                 decay_steps: int = 1, factor: float = 1.0, floor: float = 0.0, total_steps: int = 1, power: int = 1,
                 end: float = 0.0):
        if form not in _FORMS:
            raise ValueError(f"unknown schedule form {form!r}")
        self.form = form
        self.warmup_steps = _int("warmup_steps", warmup_steps)
        self.boundaries: List[int] = []
        self.multipliers: List[float] = []
        self.decay_steps, self.factor, self.floor = 1, 1.0, 0.0
        self.total_steps, self.power, self.end = 1, 1, 0.0
        if form == PIECEWISE:
            bs = [_int(f"boundaries[{i}]", b) for i, b in enumerate(boundaries)]
            if len(bs) > MAX_BOUNDARIES:
                raise ValueError(f"{len(bs)} boundaries: at most {MAX_BOUNDARIES}")
            if any(b1 <= b0 for b0, b1 in zip(bs, bs[1:])):
                raise ValueError(f"boundaries must be strictly increasing, got {bs}")
            ms = [_real(f"multipliers[{i}]", m) for i, m in enumerate(multipliers)]
            if len(ms) != len(bs) + 1:
                raise ValueError(f"piecewise needs len(boundaries) + 1 = {len(bs) + 1} multipliers, got {len(ms)}")
            self.boundaries, self.multipliers = bs, ms
        elif form == EXPONENTIAL:
            self.decay_steps = _int("decay_steps", decay_steps, lo=1)
            self.factor = _real("factor", factor)
            self.floor = _real("floor", floor)
        elif form == POLYNOMIAL:
            self.total_steps = _int("total_steps", total_steps, lo=1)
            if self.total_steps <= self.warmup_steps:
                raise ValueError(f"total_steps ({self.total_steps}) must be > warmup_steps ({self.warmup_steps})")
            if isinstance(power, bool) or not isinstance(power, (int, np.integer)) or not 1 <= int(power) <= MAX_POWER:
                raise ValueError(f"power must be an int in [1, {MAX_POWER}], got {power!r}")
            self.power = int(power)
            self.end = _real("end", end)

    # ------------------------------------------------------------ constructors --
    @classmethod
    def constant(cls, warmup_steps: int = 0) -> "LRSchedule":
        return cls(CONSTANT, warmup_steps)

    @classmethod
    def piecewise(cls, boundaries: Sequence[int], multipliers: Sequence[float], warmup_steps: int = 0) -> "LRSchedule":
        return cls(PIECEWISE, warmup_steps, boundaries=boundaries, multipliers=multipliers)

    @classmethod
    def exponential(cls, decay_steps: int, factor: float, floor: float = 0.0, warmup_steps: int = 0) -> "LRSchedule":
        return cls(EXPONENTIAL, warmup_steps, decay_steps=decay_steps, factor=factor, floor=floor)

    @classmethod
    def polynomial(cls, total_steps: int, power: int = 2, end: float = 0.0, warmup_steps: int = 0) -> "LRSchedule":
        return cls(POLYNOMIAL, warmup_steps, total_steps=total_steps, power=power, end=end)

    # -------------------------------------------------------------- evaluation --
    def multiplier(self, k: int) -> float:
        """``m(k)`` in float64, the bits the kernel computes."""
        if isinstance(k, bool) or not isinstance(k, (int, np.integer)) or not 0 <= int(k) < (1 << 63):
            raise ValueError(f"k must be an int in [0, 2**63), got {k!r}")
        k, W = int(k), self.warmup_steps
        if k < W:
            return k / W                   # int / int: the correctly rounded quotient, as the kernel's float64 divide
        if self.form == PIECEWISE:
            return self.multipliers[sum(1 for b in self.boundaries if b < k)]
        if self.form == EXPONENTIAL:
            p = pow_int(self.factor, k // self.decay_steps)
            return p if p > self.floor else self.floor
        if self.form == POLYNOMIAL:
            if k >= self.total_steps:
                return self.end
            t = (k - W) / (self.total_steps - W)
            return self.end + (1.0 - self.end) * pow_int(1.0 - t, self.power)
        return 1.0

    def rate(self, base: float, k: int) -> float:
        """The learning rate of a group with base rate ``base`` at step ``k``: ``fp32_rn(base * m(k))`` as a Python float."""
        with np.errstate(over="ignore"):
            return float(np.float32(float(base) * self.multiplier(k)))

    def table(self) -> List[float]:
        """The float64 device table the kernel decodes, given its form and ``len(boundaries)``: ``[W, ...]`` followed by
        the boundaries then the multipliers (piecewise), ``decay_steps, factor, floor`` (exponential) or ``total_steps,
        power, end`` (polynomial)."""
        head = [float(self.warmup_steps)]
        if self.form == PIECEWISE:
            return head + [float(b) for b in self.boundaries] + list(self.multipliers)
        if self.form == EXPONENTIAL:
            return head + [float(self.decay_steps), self.factor, self.floor]
        if self.form == POLYNOMIAL:
            return head + [float(self.total_steps), float(self.power), self.end]
        return head

    # ------------------------------------------------------------- checkpoints --
    def to_dict(self) -> dict:
        d = {"form": _FORMS[self.form], "warmup_steps": self.warmup_steps}
        if self.form == PIECEWISE:
            d.update(boundaries=list(self.boundaries), multipliers=list(self.multipliers))
        elif self.form == EXPONENTIAL:
            d.update(decay_steps=self.decay_steps, factor=self.factor, floor=self.floor)
        elif self.form == POLYNOMIAL:
            d.update(total_steps=self.total_steps, power=self.power, end=self.end)
        return d

    @classmethod
    def from_dict(cls, d: dict) -> "LRSchedule":
        forms = {v: k for k, v in _FORMS.items()}
        if not isinstance(d, dict) or d.get("form") not in forms:
            raise ValueError(f"not an LRSchedule dictionary: {d!r}")
        kw = {k: v for k, v in d.items() if k != "form"}
        return cls(forms[d["form"]], **kw)

    def __eq__(self, other) -> bool:
        return isinstance(other, LRSchedule) and self.to_dict() == other.to_dict()

    def __repr__(self) -> str:
        d = self.to_dict()
        form = d.pop("form")
        return f"LRSchedule.{form}({', '.join(f'{k}={v!r}' for k, v in d.items())})"
