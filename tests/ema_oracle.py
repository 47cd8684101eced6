"""Exact host oracle of the fused SGD / LARS steps' weight average (``ema_coef`` / ``ema_update`` in
csrc/kernels/device.cuh): given the average ``e``, the updated fp32 parameters ``p`` the kernel pushed, the decay ``d`` and the
update count ``k``, it returns the bits the kernel must store:

    c_k = fp32(1 - min(d, (1 + k) / (10 + k)))      float64 arithmetic, d the fp32 decay widened, one rounding to fp32
    e'  = fmaf(c_k, fp32(p - e), e)                 the product and the sum rounded once, to fp32

The fused multiply-add is computed exactly: the float64 product of two fp32 values is exact, TwoSum gives the float64 sum
and its error, and the few elements whose float64 sum sits on an fp32 rounding boundary are rounded from the exact rational
value (``fractions.Fraction``)."""
from fractions import Fraction

import numpy as np


def ema_coef(d: float, k: int) -> np.float32:
    """c_k of the k-th update (k >= 1) with decay ``d`` (rounded to fp32 first, as the trainer stores it)."""
    d64 = float(np.float32(d))
    k64 = float(k)
    return np.float32(1.0 - min(d64, (1.0 + k64) / (10.0 + k64)))


def _round_exact(x: Fraction, near: np.float32) -> np.float32:
    """Round the rational ``x`` to the nearest fp32 (ties to even); ``near`` is within one fp32 step of the answer."""
    cands = [np.nextafter(near, np.float32(-np.inf)), near, np.nextafter(near, np.float32(np.inf))]
    best = None
    for c in cands:
        if not np.isfinite(c):
            continue
        dist = abs(Fraction(float(c)) - x)
        if best is None or dist < best[0] or (dist == best[0] and (int(c.view(np.uint32)) & 1) == 0):
            best = (dist, c)
    return np.float32(best[1])


def fma32(a: np.ndarray, b: np.ndarray, c: np.ndarray) -> np.ndarray:
    """fp32 a * b + c with one rounding, element-wise (fp32 inputs, finite, no fp32 overflow)."""
    a, b, c = (np.asarray(v, dtype=np.float32) for v in (a, b, c))
    a, b, c = np.broadcast_arrays(a, b, c)
    prod = a.astype(np.float64) * b.astype(np.float64)          # exact: 24 + 24 significant bits
    cc = c.astype(np.float64)
    s = prod + cc
    bb = s - prod                                                # TwoSum: s + t == prod + c exactly
    t = (prod - (s - bb)) + (cc - bb)
    out = s.astype(np.float32)
    # RN32(s) == RN32(s + t) unless s is an fp32 midpoint (a midpoint strictly between s and s + t would be closer to the
    # exact value than s is) and t != 0; those elements are rounded from the exact value (with t == 0, s is exact and the
    # cast above already rounded a tie to even)
    lo = out.astype(np.float64)
    other = np.where(lo <= s, np.nextafter(out, np.float32(np.inf)), np.nextafter(out, np.float32(-np.inf))).astype(np.float64)
    mid = ((lo + other) * 0.5 == s) & (t != 0)
    for i in zip(*np.nonzero(mid)):
        x = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
        out[i] = _round_exact(x, out[i])
    return out


def ema_step(e, p, d: float, k: int) -> np.ndarray:
    """e' of the k-th update from the average ``e`` and the updated parameters ``p`` (fp32 arrays)."""
    e = np.asarray(e, dtype=np.float32)
    p = np.asarray(p, dtype=np.float32)
    diff = p - e                                                 # IEEE fp32 subtraction, one rounding
    return fma32(np.full_like(e, ema_coef(d, k)), diff, e)
