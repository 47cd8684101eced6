"""Exact-sum oracle for the reducing collectives.

Inputs are ``±2^u`` with ``u`` uniform in [-6, 3], rounded to the tested dtype (fp32 inputs are rounded to bf16 first), never
zero. With at most 8 ranks the exact sum of such values needs at most 23 significant bits, so an fp32 sum is exact whatever
the order of the adds, and every reduction path has exactly one correct output:

* sum / avg / user scale: ``S64.float().to(T)`` when the scale is 1, else ``(S64.float() * s32).to(T)`` with
  ``s32 = fp32(scale / world)``. This is the kernel's contract: fp32 accumulation, the scale applied once after the sum
  (skipped when it is exactly 1), one round-to-nearest-even when the result is packed to T.
* max / min: ``fmaxf`` / ``fminf`` across the ranks (a NaN is ignored unless every rank has NaN there), which is exact.

``assert_bits`` compares bit patterns, so -0 and +0 differ; NaNs only have to sit at the same places (their payload is not
part of the contract). ``expected`` asserts the exactness precondition itself, so a test that feeds it inputs whose fp32 sum
depends on the order fails loudly instead of passing by luck.
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import torch

INT_VIEW = {torch.float32: torch.int32, torch.bfloat16: torch.int16, torch.float16: torch.int16}
GUARD_BYTES = 64   # sentinel bytes on each side of a guarded view (a multiple of 16: the view's alignment is its offset's)


def exact_inputs(world: int, n: int, dtype, seed: int = 0, device: str = "cpu") -> List[torch.Tensor]:
    """``world`` tensors of ``n`` values ``±2^u`` whose fp32 sum is exact in any rank order (the same values for the same
    seed on every process that generates them on the same kind of device)."""
    g = torch.Generator(device=device).manual_seed(seed)
    mag = torch.exp2(torch.empty(world, n, dtype=torch.float64, device=device).uniform_(-6.0, 3.0, generator=g))
    sgn = torch.where(torch.rand(world, n, generator=g, device=device) < 0.5, -1.0, 1.0).double()
    x = (mag * sgn).to(torch.bfloat16 if dtype == torch.float32 else dtype).to(dtype)
    assert bool((x != 0).all()), "exact-sum inputs must not contain zeros"
    return list(x.unbind(0))


def effective_scale(op: str, world: int, scale: Optional[float] = None) -> torch.Tensor:
    """The fp32 scale a kernel receives: ``scale / world`` for avg, computed in double and passed as a C float."""
    s = 1.0 if scale is None else float(scale)
    if op in ("avg", "average"):
        s /= world
    return torch.tensor(s, dtype=torch.float32)


def exact_sum(xs: Sequence[torch.Tensor]) -> torch.Tensor:
    """The float64 sum of the ranks' inputs, after checking that an fp32 sum in rank order gives the same value."""
    st = torch.stack([x.detach().double() for x in xs])
    s64 = st.sum(0)
    s32 = torch.zeros(st.shape[1:], dtype=torch.float32, device=st.device)
    for row in st:
        s32 = s32 + row.float()
    torch.testing.assert_close(s32.double(), s64, rtol=0, atol=0, equal_nan=True,
                               msg="oracle precondition: the fp32 sum of these inputs is not exact")
    return s64


def expected(xs: Sequence[torch.Tensor], op: str, scale: Optional[float] = None, nvls: bool = False) -> torch.Tensor:
    """The one correct output of reducing ``xs`` (one tensor per rank) with ``op``, on their device and of their dtype.

    ``nvls=True`` gives the NVLS contract for bf16 / f16 sums: ``multimem.ld_reduce ... acc::f32`` returns the sum already
    rounded to T and the scale is applied to that value and rounded again."""
    dtype = xs[0].dtype
    world = len(xs)
    s32 = effective_scale(op, world, scale)
    if op in ("max", "min"):
        f = torch.fmax if op == "max" else torch.fmin
        r = xs[0].detach().float()
        for x in xs[1:]:
            r = f(r, x.detach().float())
    else:
        r = exact_sum(xs).float()
        if nvls and dtype != torch.float32:
            r = r.to(dtype).float()
    if float(s32) != 1.0:
        r = r * s32.to(r.device)
    return r.to(dtype)


def bits(t: torch.Tensor) -> torch.Tensor:
    return t.detach().contiguous().view(INT_VIEW[t.dtype])


def assert_bits(got: torch.Tensor, want: torch.Tensor, what: str = "") -> None:
    """Bitwise equality, except that a NaN matches any NaN (compared on ``got``'s device)."""
    got = got.detach()
    want = want.detach().to(got.device)
    assert got.dtype == want.dtype and got.shape == want.shape, f"{what}: {got.dtype}{tuple(got.shape)} vs {want.dtype}{tuple(want.shape)}"
    gn, wn = torch.isnan(got), torch.isnan(want)
    bad = (gn != wn) | (~gn & ~wn & (bits(got) != bits(want)))
    if bool(bad.any()):
        idx = bad.nonzero().flatten().cpu()
        i = int(idx[0])
        raise AssertionError(f"{what}: {idx.numel()} of {got.numel()} elements differ; first at {i}: "
                             f"got {got[i].item()!r} want {want[i].item()!r}")


def assert_ranks_agree(outs: Sequence[torch.Tensor], what: str = "") -> None:
    """Every rank holds the same bits (NaN payloads included)."""
    b0 = bits(outs[0])
    for r, o in enumerate(outs[1:], 1):
        assert torch.equal(bits(o).to(b0.device), b0), f"{what}: rank {r} differs from rank 0"


class Guarded:
    """A CUDA view of ``numel`` elements at an element offset ``offset`` into a byte buffer with ``GUARD_BYTES`` of random
    sentinel bytes on each side. ``unchanged()`` / ``guards_intact()`` compare against the bytes recorded by ``seal()``."""

    def __init__(self, numel: int, dtype, offset: int, seed: int = 0, device: str = "cuda"):
        esz = torch.empty((), dtype=dtype).element_size()
        self.lo = GUARD_BYTES + offset * esz
        self.hi = self.lo + numel * esz
        g = torch.Generator(device=device).manual_seed(seed)
        self.buf = torch.randint(0, 256, (self.hi + GUARD_BYTES,), dtype=torch.uint8, generator=g, device=device)
        self.view = self.buf[self.lo:self.hi].view(dtype)
        self.snap = None

    def seal(self) -> "Guarded":
        self.snap = self.buf.clone()
        return self

    def guards_intact(self) -> bool:
        return torch.equal(self.buf[:self.lo], self.snap[:self.lo]) and torch.equal(self.buf[self.hi:], self.snap[self.hi:])

    def unchanged(self) -> bool:
        return torch.equal(self.buf, self.snap)
