"""Float64 oracle for Adasum: the one-kernel allreduce (csrc/kernels/adasum.cu) and the torch tree (hvd/adasum.py).

Both follow one arithmetic contract for f32 / bf16 / f16 inputs:

* values are widened to fp32 (exact); the pair sums ``d = a.b``, ``na = a.a``, ``nb = b.b`` add fp64 products, which are
  exact for fp32 factors, in fp64;
* ``c = fp32(1.0 - d / (2.0 * n))`` when ``n > 0`` (in fp64), else ``1.0``;
* ``z = fp32(fp32(ca * a) + fp32(cb * b))``, element by element; intermediate levels stay fp32;
* the tree pairs (0, 1), (2, 3), ... and then their results in the same way (an odd last entry moves up unchanged: the torch
  tree at worlds that are not powers of two); the root is rounded once, to nearest even, into T.

Only the order of the fp64 additions is left to the implementation (the kernel's is set by its grid, the torch path's by
torch). ``expected`` computes every sum exactly (``math.fsum``, one rounding) and bounds what any order of ``depth`` nested
additions can do to it: ``|sum - S| <= gamma(depth) * sum|terms|`` with ``gamma(k) = k u / (1 - k u)``, ``u = 2^-53``. With
the roundings of the division and the subtraction added, each fp64 coefficient lies in an interval; the **tie guard**
asserts that no fp32 rounding midpoint lies in it. When it holds, every coefficient - and so every bit of the output - has
exactly one correct value, whatever the order; when it fails, the test fails and says where, instead of passing by luck.
Non-finite sums are order independent (IEEE: NaN if any term is NaN or both infinities occur, else the infinity), so NaN /
Inf inputs have one correct output too.

``tree64`` is the plain mathematical tree in float64, an independent check of the contract itself; ``tree64_bound`` bounds
``|expected - tree64|`` element by element by propagating first-order error bounds through the tree.
"""
from __future__ import annotations

import math
from fractions import Fraction
from typing import Optional, Sequence

import numpy as np
import torch

U64 = 2.0 ** -53
THREADS = 512                       # CTA size of the kernel
MAX_BLOCKS = 64                     # kAdaMaxBlocks
EMU_SMS = 132                       # the emulated communicator keeps world * CTAs <= 132 (all co-resident)
VEC_ELEMS = {torch.float32: 4, torch.bfloat16: 8, torch.float16: 8}    # elements per 16-byte vector
UNIT = {torch.float32: 2.0 ** -24, torch.bfloat16: 2.0 ** -8, torch.float16: 2.0 ** -11}
TINY = {torch.float32: 2.0 ** -149, torch.bfloat16: 2.0 ** -133, torch.float16: 2.0 ** -24}   # smallest subnormal


class TieError(AssertionError):
    """The oracle's precondition failed: an fp64 coefficient may round to either of two fp32 values."""


def gamma(k: int) -> float:
    return k * U64 / (1.0 - k * U64)


def kernel_geometry(numel: int, dtype, world: int, max_blocks: int = 64, emulated: bool = True):
    """``(nvec, per, blocks)`` as b200mpi_adasum plans them: 16-byte vectors, ``per`` vectors per rank slice, and the CTA
    count ``min(ceil(per / 512), max_blocks, 64)`` (emulated: also ``<= 132 // world``)."""
    nvec = -(-numel * torch.empty((), dtype=dtype).element_size() // 16)
    per = -(-nvec // world)
    blocks = max(1, min(-(-per // THREADS), min(max_blocks, MAX_BLOCKS)))
    if emulated:
        blocks = min(blocks, max(1, EMU_SMS // world))
    return nvec, per, blocks


def kernel_depth(per: int, blocks: int, world: int, dtype) -> int:
    """Most fp64 additions any product passes through in the kernel: the per-thread chain (``VN`` products per vector,
    ``ceil(per / (512 blocks))`` vectors), the warp butterfly (5), the 16 warps, the board (``ceil(world blocks / 32)`` per
    lane) and its butterfly (5)."""
    iters = max(1, -(-per // (THREADS * blocks)))
    return iters * VEC_ELEMS[dtype] + 5 + THREADS // 32 + -(-world * blocks // 32) + 5


def torch_depth(numel: int) -> int:
    """Any order of summing ``numel`` terms nests at most ``numel - 1`` additions (fused multiply-adds included)."""
    return max(1, numel)


# ------------------------------------------------------------------------------------------------ the contract --
def _f32(t) -> np.ndarray:
    if isinstance(t, np.ndarray):
        return t.astype(np.float32, copy=False).ravel()
    return t.detach().reshape(-1).float().cpu().numpy()


def _sum(p: np.ndarray):
    """(fp64 sum rounded once, sum of |terms|) of fp64 products; IEEE results when a term is not finite."""
    if np.isfinite(p).all():
        a = float(np.abs(p).sum()) * (1.0 + 1e-9)       # an upper bound: numpy's own sum error is far below 1e-9
        return math.fsum(memoryview(np.ascontiguousarray(p))), a
    with np.errstate(all="ignore"):
        return float(np.sum(p)), math.inf


def coefficient(d: float, n: float, ed: float, en: float, what: str = "") -> np.float32:
    """``fp32(1 - d / (2 n))`` (1 when ``n > 0`` is false) after checking the tie guard: ``d`` and ``n`` are the fp64 sums
    rounded once, ``ed`` / ``en`` bound how far an implementation's sums may be from them."""
    if not n > 0:
        return np.float32(1.0)
    with np.errstate(all="ignore"):
        c64 = 1.0 - d / (2.0 * n)
    c32 = np.float32(c64)
    if not (math.isfinite(d) and math.isfinite(n) and math.isfinite(ed) and math.isfinite(en)):
        if math.isfinite(c64):
            raise TieError(f"{what}: finite coefficient {c64!r} from non-finite sums")
        return c32
    D, N, ED, EN = Fraction(d), Fraction(n), Fraction(ed), Fraction(en)
    if N - EN <= 0:
        raise TieError(f"{what}: |n| = {n!r} is within its error bound {en!r}")
    qs = [(D + s * ED) / (2 * m) for s in (-1, 1) for m in (N - EN, N + EN)]
    u = Fraction(1, 2 ** 53)
    qlo, qhi = min(qs), max(qs)
    qlo, qhi = qlo - u * abs(qlo), qhi + u * abs(qhi)              # rounding of the division
    lo, hi = 1 - qhi, 1 - qlo
    lo, hi = lo - u * abs(lo), hi + u * abs(hi)                    # rounding of the subtraction
    c = Fraction(float(c32))
    below = Fraction(float(np.nextafter(c32, np.float32(-np.inf))))
    above = Fraction(float(np.nextafter(c32, np.float32(np.inf))))
    if not ((c + below) / 2 < lo and hi < (c + above) / 2):
        raise TieError(f"{what}: coefficient {c64!r} in [{float(lo)!r}, {float(hi)!r}] may round to either side of an "
                       f"fp32 midpoint (fp32 {float(c32)!r})")
    return c32


def pair(x: np.ndarray, y: np.ndarray, depth: int, what: str = "", info: Optional[dict] = None) -> np.ndarray:
    """One Adasum combine under the contract (fp32 numpy in, fp32 numpy out)."""
    x64, y64 = x.astype(np.float64), y.astype(np.float64)
    with np.errstate(all="ignore"):
        (d, ad), (na, an), (nb, bn) = _sum(x64 * y64), _sum(x64 * x64), _sum(y64 * y64)
    g = gamma(depth + 1)                                            # + 1: the oracle's own rounding of the exact sum
    ca = coefficient(d, na, g * ad, g * an, f"{what} ca")
    cb = coefficient(d, nb, g * ad, g * bn, f"{what} cb")
    with np.errstate(all="ignore"):
        px, py = ca * x, cb * y
        z = px + py
    if info is not None:
        info.setdefault("coefs", []).append((float(ca), float(cb)))
        for v in (px, py, z):
            _track(info, v)
    return z


def _track(info: dict, v: np.ndarray) -> None:
    a = np.abs(v[np.isfinite(v) & (v != 0)])
    if a.size:
        info["min_abs"] = min(info.get("min_abs", math.inf), float(a.min()))
        info["max_abs"] = max(info.get("max_abs", 0.0), float(a.max()))


def expected(xs: Sequence, dtype=None, depth: Optional[int] = None, what: str = "",
             info: Optional[dict] = None) -> torch.Tensor:
    """The one correct Adasum of ``xs`` (one tensor per rank) in ``dtype`` (default: the inputs'), on the CPU.

    ``depth`` is the implementation's nesting of fp64 additions (``kernel_depth`` / ``torch_depth``; default: any order).
    Raises ``TieError`` when the answer is not unique. ``info``, when given, receives the coefficients level by level and the
    smallest / largest nonzero finite magnitude of every fp32 value the tree forms (inputs included)."""
    dtype = dtype or xs[0].dtype
    level = [_f32(x) for x in xs]
    depth = torch_depth(level[0].size) if depth is None else depth
    if info is not None:
        for v in level:
            _track(info, v)
    lv = 0
    while len(level) > 1:
        nxt = [pair(level[i], level[i + 1], depth, f"{what} level {lv} pair {i // 2}", info)
               for i in range(0, len(level) - 1, 2)]
        if len(level) % 2:
            nxt.append(level[-1])
        level, lv = nxt, lv + 1
    return torch.from_numpy(level[0].copy()).to(dtype)


# ------------------------------------------------------------------------------------- the mathematical tree --
def tree64(xs: Sequence) -> torch.Tensor:
    """The Adasum tree in float64 throughout (no fp32 rounding anywhere), on the CPU."""
    return torch.from_numpy(_tree64(xs)[0])


def tree64_bound(xs: Sequence, dtype=None) -> torch.Tensor:
    """Per-element bound on ``|expected(xs, dtype) - tree64(xs)|`` (first-order error propagation with a factor 2 of
    slack); infinite where a level's norms are too small for the first-order terms to mean anything."""
    dtype = dtype or xs[0].dtype
    z, e = _tree64(xs)
    return torch.from_numpy(2.0 * (e + UNIT[dtype] * np.abs(z)) + TINY[dtype])


def _tree64(xs: Sequence):
    u32, tiny32 = 2.0 ** -24, 2.0 ** -149
    level = [(_f32(x).astype(np.float64), np.zeros(_f32(x).size)) for x in xs]
    while len(level) > 1:
        nxt = []
        for i in range(0, len(level) - 1, 2):
            (x, ex), (y, ey) = level[i], level[i + 1]
            d, na, nb = float(x @ y), float(x @ x), float(y @ y)
            nx, ny, Ex, Ey = math.sqrt(na), math.sqrt(nb), float(np.linalg.norm(ex)), float(np.linalg.norm(ey))
            dd = Ex * ny + nx * Ey + Ex * Ey + 1e-15 * nx * ny

            def coef(n, nn, E):
                if n == 0:
                    return 1.0, (0.0 if E == 0 else math.inf)
                dn = 2 * nn * E + E * E + 1e-15 * n
                if dn >= n / 2:
                    return 1.0 - d / (2 * n), math.inf
                c = 1.0 - d / (2 * n)
                dc = dd / (2 * (n - dn)) + abs(d) * dn / (2 * n * (n - dn))
                return c, dc + u32 * (abs(c) + dc)                       # + the coefficient's rounding to fp32

            (ca, dca), (cb, dcb) = coef(na, nx, Ex), coef(nb, ny, Ey)
            z = ca * x + cb * y
            px, py = (abs(ca) + dca) * (np.abs(x) + ex), (abs(cb) + dcb) * (np.abs(y) + ey)
            with np.errstate(invalid="ignore"):
                e = abs(ca) * ex + abs(cb) * ey + dca * (np.abs(x) + ex) + dcb * (np.abs(y) + ey) \
                    + u32 * (px + py) + u32 * (px + py) + 3 * tiny32          # two products and the add, each rounded
            nxt.append((z, np.nan_to_num(e, nan=math.inf)))
        if len(level) % 2:
            nxt.append(level[-1])
        level = nxt
    return level[0]
