"""Exact operands and a float64 reference for the wgmma 1x1-convolution GEMM (csrc/kernels/gemm_bnstats.cu).

The kernel's contract, for the training forward ``b200mpi_gemm_bnstats`` and the dgrad ``b200mpi_gemm_dgrad_res``:

* ``Y = rne_bf16(fp32 sum_k x[m,k] w[n,k] (+ mask[m,n] * r[m,n]))``: exact bf16 x bf16 products, accumulated in fp32 in
  an order the tensor cores choose, the residual added in fp32, one round-to-nearest-even to bf16. A masked-out ``r`` is
  never read into the result (NaN / Inf there change nothing).
* Partial row ``p`` of ``parts = min(min(SMs, 132) // num_n, num_m)`` covers the 128-row tiles ``p, p + parts, ...`` of its
  column block. The forward holds ``sum (y - y[128 p])`` and ``sum (y - y[128 p])^2`` over those rows of the bf16 ``Y``;
  the dgrad with ``Xb`` holds ``sum g`` and ``sum g * (xb - mean_b)``, ``g = maskB * bf16(dX)``. Rows past M add nothing.

Three operand families make that checkable:

* **E** (exact dense): ``x = i * 2^a_m``, ``w = j * 2^b_n``, ``r = l * 2^(a_m + b_n)`` with integer ``i, j, l``. One operand
  has full 8-bit significands (128 <= |i| <= 255), the other a per-row / per-column range chosen from K so that
  ``sum_k |i j| + |l| <= 2^23``. Every partial sum is then an integer multiple of ``2^(a_m + b_n)`` below ``2^24`` of them,
  so fp32 accumulation is exact in any order and chunking, even with alignment that truncates: ``Y`` has one correct bf16
  value. Many outputs have more than 8 significant bits, and some are exact round-to-nearest-even ties.
* **S** (exact statistics): ``x in {-1, 0, 1}``, each row of ``w`` has exactly B entries ``±2^c_n``, the rest 0. ``y`` is an
  integer multiple of ``2^c_n`` in ``[-B, B] 2^c_n``, and B is chosen so that every shifted sum and sum of squares of a
  partial row stays below ``2^24`` units: the partial rows have one correct fp32 value. Where the rows of a partial row allow
  it, an offset column (``x = 1``, ``w = 1024``) moves ``y`` to where bf16 rounds, so that statistics taken from the fp32
  accumulator instead of the bf16 tile differ in their bits. For the dgrad partials ``dY``, ``Wt``, ``R`` and ``Xb`` are
  small integers and ``mean_b`` is in Z/4.
* **R** (random): bf16 ``N(0, 1)`` activations, ``N(0, 1/K)`` weights. ``|Y - ref| <= ulp(ref) / 2 + 2^-20 (sum_k |x w| +
  |mask r|)``: one rounding plus fp32 accumulation error, tight enough to see a dropped k-slice or truncating rounding.

Every generator and reference asserts its own precondition, so a test that feeds it operands whose fp32 sums depend on the
order fails loudly instead of passing by luck. Everything runs on the CPU or the GPU; references are computed in row chunks
so that a large M never allocates ``M x N`` float64.
"""
from __future__ import annotations

import math
from dataclasses import dataclass
from typing import Optional

import torch

BM = 128                  # rows per tile and per partial-row shift stride
MAX_PARTS = 132           # partial rows: at most one per SM, and at most 132
GUARD_ROWS = 128          # rows past M of every guard-banded allocation
SLACK = 2.0 ** -20        # family R: fp32 accumulation error allowed per unit of sum |terms|
STATS_REL = 1e-5          # fp32 partial rows of inexact data: error per unit of sum |terms|
CHUNK_ELEMS = 1 << 24     # float64 elements per reference chunk


# ------------------------------------------------------------------------------------------------- bf16 helpers --
def bf16_bits(t: torch.Tensor) -> torch.Tensor:
    return t.contiguous().view(torch.int16)


def round_bf16(t: torch.Tensor, mode: str = "rne") -> torch.Tensor:
    """fp32 (or fp32-exact float64) values rounded to bf16 by bit arithmetic: ``rne`` or ``trunc`` (toward zero)."""
    f = t.float()
    if t.dtype == torch.float64:
        assert torch.equal(f.double(), t), "round_bf16: float64 input is not exact in fp32"
    u = f.view(torch.int32).long() & 0xFFFFFFFF
    if mode == "rne":
        u = u + 0x7FFF + ((u >> 16) & 1)
    elif mode != "trunc":
        raise ValueError(mode)
    hi = ((u >> 16) & 0xFFFF).to(torch.int32)
    hi = torch.where(hi >= 0x8000, hi - 0x10000, hi).to(torch.int16)
    return hi.view(torch.bfloat16)


def half_ulp_bf16(ref: torch.Tensor) -> torch.Tensor:
    """Half a bf16 ulp at |ref| (8 significant bits), 0 at 0."""
    _, e = torch.frexp(ref.double())            # ref = m 2^e, 0.5 <= |m| < 1: ulp = 2^(e - 8)
    return torch.where(ref == 0, torch.zeros_like(ref, dtype=torch.float64), torch.exp2((e - 9).double()))


def is_tie(ref: torch.Tensor) -> torch.Tensor:
    """fp32-exact values that lie exactly halfway between two bf16 values."""
    u = ref.float().view(torch.int32).long() & 0xFFFF
    return (u == 0x8000) & torch.isfinite(ref)


def full_significand(t: torch.Tensor) -> torch.Tensor:
    """bf16 values whose significand uses all 8 bits (the lowest one set)."""
    return ((bf16_bits(t).long() & 1) == 1) & (t != 0)


# -------------------------------------------------------------------------------------------------------- masks --
def pack_mask(bits: torch.Tensor) -> torch.Tensor:
    """bool [M, N] -> uint8 [M, N/8]: bit c % 8 of byte c / 8."""
    M, N = bits.shape
    w = (1 << torch.arange(8, device=bits.device, dtype=torch.int32))
    return (bits.view(M, N // 8, 8).int() * w).sum(-1).to(torch.uint8)


def unpack_mask(packed: torch.Tensor, N: int) -> torch.Tensor:
    """uint8 [M, N/8] (or flat) -> bool [M, N]."""
    p = packed.reshape(-1, N // 8)
    sh = torch.arange(8, device=p.device, dtype=torch.int32)
    return ((p.int()[..., None] >> sh) & 1).reshape(p.shape[0], N).bool()


# ------------------------------------------------------------------------------------------------- tile walk --
def tile_width(N: int) -> int:
    return 128 if N % 128 == 0 else 64


def plan_parts(M: int, N: int, sms: int = MAX_PARTS) -> int:
    """Partial rows the kernel writes: ``min(min(SMs, 132) // num_n, num_m)`` (one CTA per column block and m-group)."""
    num_n = N // tile_width(N)
    num_m = -(-M // BM)
    return min(min(sms, MAX_PARTS) // num_n, num_m)


def part_of_row(M: int, parts: int, device="cpu", lo: int = 0, hi: int = None) -> torch.Tensor:
    """Partial row index of rows [lo, hi) of Y: row m is in tile m // 128, which partial row (m // 128) % parts walks."""
    return (torch.arange(lo, M if hi is None else hi, device=device) // BM) % parts


def rows_per_part(M: int, parts: int) -> torch.Tensor:
    return torch.bincount(part_of_row(M, parts), minlength=parts)


# -------------------------------------------------------------------------------------------- guarded memory --
def guarded(rows: int, cols: int, dtype, device, poison: bool = True):
    """A [rows + GUARD_ROWS, cols] buffer whose first ``rows`` rows are the operand; the guard rows hold NaN (0xFF for
    uint8) when ``poison``, else zeros. Returns (buffer, view of the first rows)."""
    buf = torch.empty(rows + GUARD_ROWS, cols, dtype=dtype, device=device)
    set_guard(buf, rows, poison)
    return buf, buf[:rows]


def set_guard(buf: torch.Tensor, rows: int, poison: bool) -> None:
    if buf.dtype == torch.uint8:
        buf[rows:] = 0xFF if poison else 0
    else:
        buf[rows:] = float("nan") if poison else 0.0


# ------------------------------------------------------------------------------------------------- operands --
@dataclass
class Operands:
    """x [M,K], w [N,K] bf16 (for the dgrad: dY and Wt); optional r [M,N] bf16 and its mask (bool [M,N]). Families E / S
    have per-row and per-column exponents ``ea`` [M], ``eb`` [N]: every term of output (m, n) is an integer multiple of
    ``2^(ea[m] + eb[n])``."""
    fam: str
    x: torch.Tensor
    w: torch.Tensor
    ea: Optional[torch.Tensor] = None
    eb: Optional[torch.Tensor] = None
    r: Optional[torch.Tensor] = None
    mask: Optional[torch.Tensor] = None


def _gen(device, seed):
    return torch.Generator(device=device).manual_seed(seed)


def _randint(lo, hi, shape, g, device, dtype=torch.int32):
    return torch.randint(lo, hi + 1, shape, generator=g, device=device, dtype=dtype)


def family_e(M: int, N: int, K: int, *, x_full: bool, residual: bool = False, seed: int = 0, device="cpu") -> Operands:
    g = _gen(device, seed)
    ea = _randint(-6, 6, (M,), g, device)
    eb = _randint(-6, 6, (N,), g, device)
    lmax = 255 if residual else 0
    other_max = (2 ** 23 - lmax) // (K * 255)
    assert other_max >= 1, f"family E: K = {K} is too deep for 8-bit significands"
    full_rows, narrow_rows = (M, N) if x_full else (N, M)
    # 8-bit integers 128..255 with random signs: half of them odd, i.e. with all 8 significand bits in use
    full = _randint(128, 255, (full_rows, K), g, device) * (_randint(0, 1, (full_rows, K), g, device) * 2 - 1)
    # per-row range of the narrow operand: 2^u for u uniform in [0, log2(other_max)], so that some outputs are small
    # enough to round with ties and some use the whole 2^23 budget
    top = int(math.log2(other_max))
    rng = torch.exp2(_randint(0, top, (narrow_rows, 1), g, device).double()).long().clamp_max(other_max)
    narrow = torch.floor(torch.rand(narrow_rows, K, generator=g, device=device) * (2 * rng + 1)).int() - rng
    i, j = (full, narrow) if x_full else (narrow, full)
    x = (i.double() * torch.exp2(ea.double())[:, None]).to(torch.bfloat16)
    w = (j.double() * torch.exp2(eb.double())[:, None]).to(torch.bfloat16)
    op = Operands("E", x, w, ea, eb)
    if residual:
        l = _randint(-255, 255, (M, N), g, device)
        op.r = (l.double() * torch.exp2(ea.double()[:, None] + eb.double()[None, :])).to(torch.bfloat16)
        op.mask = torch.rand(M, N, generator=g, device=device) < 0.5
    return op


OFFSET = 1024       # family S: the offset column's weight, where bf16 has an ulp of 4 or 8


def stats_plan(M: int, N: int, K: int, residual: bool = False):
    """Family S: (B, offset) for a shape. Without ``offset`` ``y in [-B, B]`` is exact in bf16; with it ``y = offset +
    [-B, B]`` rounds (|error| <= 4), so statistics or GST partials taken from the fp32 accumulator instead of the bf16 tile
    differ from the oracle's bits. Both keep every partial sum below 2^24 units: ``rows * (2B + 8)^2 < 2^24`` for the
    forward, ``rows * (offset + B + 4) * 6 < 2^22`` for the dgrad's ``sum |g| |xb - mean|``."""
    rows = int(rows_per_part(M, plan_parts(M, N)).max())
    if residual:
        ok = lambda b, c: rows * (c + b + 4) * 6 < 2 ** 22             # noqa: E731
    else:
        ok = lambda b, c: rows * (2 * b + (8 if c else 0)) ** 2 < 2 ** 24  # noqa: E731
    for c in (OFFSET, 0):
        b = min(64, K - (1 if c else 0))
        while b > 0 and not ok(b, c):
            b -= 1
        if b >= (8 if c else 1):
            return b, c
    raise AssertionError(f"family S: no B fits M={M} N={N} K={K}")


def family_s(M: int, N: int, K: int, *, residual: bool = False, scale: bool = True, seed: int = 0, device="cpu") -> Operands:
    g = _gen(device, seed)
    B, offset = stats_plan(M, N, K, residual)
    x = _randint(-1, 1, (M, K), g, device, torch.int8)
    # exactly B nonzero ±1 entries per row of w, at random columns (not the offset column K - 1)
    kk = K - 1 if offset else K
    cols = torch.rand(N, kk, generator=g, device=device).argsort(1)[:, :B]
    j = torch.zeros(N, K, dtype=torch.int32, device=device)
    j.scatter_(1, cols, _randint(0, 1, (N, B), g, device) * 2 - 1)
    if offset:
        x[:, K - 1] = 1
        j[:, K - 1] = offset
    eb = _randint(-3, 3, (N,), g, device) if scale else torch.zeros(N, dtype=torch.int64, device=device)
    ea = torch.zeros(M, dtype=torch.int64, device=device)
    op = Operands("S", x.to(torch.bfloat16), (j.double() * torch.exp2(eb.double())[:, None]).to(torch.bfloat16), ea, eb)
    if residual:
        op.r = (_randint(-4, 4, (M, N), g, device).double() * torch.exp2(eb.double())[None, :]).to(torch.bfloat16)
        op.mask = torch.rand(M, N, generator=g, device=device) < 0.5
    return op


def family_r(M: int, N: int, K: int, *, residual: bool = False, seed: int = 0, device="cpu") -> Operands:
    g = _gen(device, seed)
    x = torch.randn(M, K, generator=g, device=device).to(torch.bfloat16)
    w = (torch.randn(N, K, generator=g, device=device) * K ** -0.5).to(torch.bfloat16)
    op = Operands("R", x, w)
    if residual:
        op.r = torch.randn(M, N, generator=g, device=device).to(torch.bfloat16)
        op.mask = torch.rand(M, N, generator=g, device=device) < 0.5
    return op


def below_operands(M: int, N: int, *, fam: str, seed: int = 0, device="cpu"):
    """Xb [M,N] bf16, maskB bool [M,N] and mean_b [N] fp32 of the BatchNorm below a dgrad: small integers and Z/4 means
    (exact) for families E / S, N(0, 1) and N(0, 0.1) for R."""
    g = _gen(device, seed + 7)
    if fam == "R":
        xb = torch.randn(M, N, generator=g, device=device).to(torch.bfloat16)
        mean = (torch.randn(N, generator=g, device=device) * 0.1).float()
    else:
        xb = _randint(-4, 4, (M, N), g, device).to(torch.bfloat16)
        mean = (_randint(-8, 8, (N,), g, device).double() / 4).float()
    maskb = torch.rand(M, N, generator=g, device=device) < 0.5
    return xb, maskb, mean


# ------------------------------------------------------------------------------------------------ references --
def row_chunks(M: int, N: int):
    step = max(1, CHUNK_ELEMS // max(N, 1))
    for lo in range(0, M, step):
        yield lo, min(M, lo + step)


def ref_chunk(op: Operands, lo: int, hi: int, r: Optional[torch.Tensor] = None, mask: Optional[torch.Tensor] = None):
    """(exact float64 value, float64 sum of |terms|) of rows [lo, hi) of the output. ``r`` / ``mask`` override the
    operand's residual (the kernel's residual operand may differ from the generated one only where the mask is 0)."""
    r = op.r if r is None else r
    mask = op.mask if mask is None else mask
    x = op.x[lo:hi].double()
    w = op.w.double()
    ref = x @ w.t()
    mag = x.abs() @ w.abs().t()
    if r is not None:
        rr = torch.where(mask[lo:hi], r[lo:hi].double(), torch.zeros((), dtype=torch.float64, device=x.device))
        ref = ref + rr
        mag = mag + rr.abs()
    return ref, mag


def check_exact_precondition(op: Operands, lo: int, hi: int, mag: torch.Tensor) -> None:
    """Families E / S: every term of each output is an integer multiple of 2^unit and their magnitudes sum to at most
    2^23 units, so any fp32 order and chunking sums them exactly."""
    unit = torch.exp2((op.ea[lo:hi, None] + op.eb[None, :]).double())
    q = mag / unit
    assert bool((q <= 2 ** 23).all()), f"oracle precondition: sum |terms| reaches {float(q.max())} units (> 2^23)"
    xs = op.x[lo:hi].double() / torch.exp2(op.ea[lo:hi].double())[:, None]
    assert bool((xs == xs.round()).all()), "oracle precondition: x is not an integer multiple of 2^a"


def expected_y(op: Operands, lo: int, hi: int, r=None, mask=None):
    """Rows [lo, hi) of the one correct output (families E / S; asserts the precondition) as bf16, or for family R the
    float64 value and the allowed error. Returns (want_bf16 or None, ref64, bound or None)."""
    ref, mag = ref_chunk(op, lo, hi, r, mask)
    if op.fam in ("E", "S"):
        check_exact_precondition(op, lo, hi, mag)
        return round_bf16(ref), ref, None
    return None, ref, half_ulp_bf16(ref) + SLACK * mag


def check_y(got: torch.Tensor, op: Operands, what: str, r=None, mask=None) -> float:
    """Compares the kernel's output [M,N] with the oracle: bit for bit on E / S, within the bound on R. Returns the
    largest err / bound (0 for exact families)."""
    M, N = got.shape
    worst = 0.0
    for lo, hi in row_chunks(M, N):
        want, ref, bound = expected_y(op, lo, hi, r, mask)
        g = got[lo:hi]
        if want is not None:
            assert_bits(g, want, f"{what} rows {lo}..{hi}")
        else:
            err = (g.double() - ref).abs()
            ratio = err / bound
            bad = ~(err <= bound)
            if bool(bad.any()):
                idx = bad.nonzero()[0].tolist()
                raise AssertionError(f"{what}: {int(bad.sum())} elements outside the family-R bound; first at "
                                     f"({lo + idx[0]}, {idx[1]}): got {float(g[idx[0], idx[1]])} ref "
                                     f"{float(ref[idx[0], idx[1]])} bound {float(bound[idx[0], idx[1]])}")
            worst = max(worst, float(ratio.nan_to_num(0.0).max()))
    return worst


def assert_bits(got: torch.Tensor, want: torch.Tensor, what: str = "") -> None:
    """Bitwise equality of two tensors of one dtype."""
    assert got.dtype == want.dtype and got.shape == want.shape, f"{what}: {got.dtype}{tuple(got.shape)} vs {want.dtype}{tuple(want.shape)}"
    iv = {torch.bfloat16: torch.int16, torch.float32: torch.int32, torch.float64: torch.int64}[got.dtype]
    bad = got.contiguous().view(iv) != want.to(got.device).contiguous().view(iv)
    if bool(bad.any()):
        idx = bad.nonzero()[0].tolist()
        raise AssertionError(f"{what}: {int(bad.sum())} of {got.numel()} elements differ; first at {tuple(idx)}: "
                             f"got {float(got[tuple(idx)])} want {float(want[tuple(idx)])}")


# ------------------------------------------------------------------------------------------- partial rows --
def _scatter_parts(vals: torch.Tensor, part: torch.Tensor, parts: int) -> torch.Tensor:
    out = torch.zeros(parts, vals.shape[1], dtype=torch.float64, device=vals.device)
    return out.index_add_(0, part, vals)


def stats_ref(y: torch.Tensor, parts: int):
    """Float64 forward partial rows of the kernel's own bf16 ``Y`` [M,N]: returns (shifted [parts,N,2], magnitudes
    [parts,N,2] = sum |y - K|, sum (y - K)^2, plain [parts,N,2] = sum y, sum y^2) with K = Y[128 p]."""
    M, N = y.shape
    shift = y[0:(parts - 1) * BM + 1:BM].double()                       # [parts, N]
    sh = torch.zeros(parts, N, 2, dtype=torch.float64, device=y.device)
    mg = torch.zeros_like(sh)
    pl = torch.zeros_like(sh)
    for lo, hi in row_chunks(M, N):
        part = part_of_row(M, parts, y.device, lo, hi)
        v = y[lo:hi].double()
        d = v - shift[part]
        sh[..., 0] += _scatter_parts(d, part, parts)
        sh[..., 1] += _scatter_parts(d * d, part, parts)
        mg[..., 0] += _scatter_parts(d.abs(), part, parts)
        pl[..., 0] += _scatter_parts(v, part, parts)
        pl[..., 1] += _scatter_parts(v * v, part, parts)
    mg[..., 1] = sh[..., 1]
    return sh, mg, pl


def gst_ref(dx: torch.Tensor, xb: torch.Tensor, maskb: torch.Tensor, mean: torch.Tensor, parts: int):
    """Float64 BN-backward partial rows of the kernel's own bf16 ``dX``: (rows [parts,N,2] = sum g, sum g (xb - mean),
    magnitudes [parts,N,2]) with g = maskB * dX."""
    M, N = dx.shape
    rows = torch.zeros(parts, N, 2, dtype=torch.float64, device=dx.device)
    mg = torch.zeros_like(rows)
    mu = mean.double()[None, :]
    for lo, hi in row_chunks(M, N):
        part = part_of_row(M, parts, dx.device, lo, hi)
        gv = torch.where(maskb[lo:hi], dx[lo:hi].double(), torch.zeros((), dtype=torch.float64, device=dx.device))
        t = gv * (xb[lo:hi].double() - mu)
        rows[..., 0] += _scatter_parts(gv, part, parts)
        rows[..., 1] += _scatter_parts(t, part, parts)
        mg[..., 0] += _scatter_parts(gv.abs(), part, parts)
        mg[..., 1] += _scatter_parts(t.abs(), part, parts)
    return rows, mg


def check_exact_sums(rows: torch.Tensor, mag: torch.Tensor, unit: torch.Tensor, what: str, limit: float = 2.0 ** 24) -> None:
    """Precondition of a bit-exact partial row: every term is a multiple of ``unit`` (per column, [N] or [N,2]) and
    their magnitudes sum to less than ``limit`` units."""
    q = mag / unit
    assert bool((q < limit).all()), f"{what}: oracle precondition: sum |terms| reaches {float(q.max())} units"
    assert bool(((rows / unit) == (rows / unit).round()).all()), f"{what}: oracle precondition: sums not in units"


def check_rows(got: torch.Tensor, rows: torch.Tensor, mag: torch.Tensor, exact: bool, what: str) -> float:
    """Partial rows [parts,N,2] fp32 against float64: bit for bit (``exact``) or within STATS_REL * sum |terms|. Returns
    the largest err / bound."""
    if exact:
        assert_bits(got.float(), rows.float(), what)
        return 0.0
    err = (got.double() - rows).abs()
    bound = STATS_REL * mag + 1e-30
    bad = ~(err <= bound)
    if bool(bad.any()):
        idx = tuple(bad.nonzero()[0].tolist())
        raise AssertionError(f"{what}: {int(bad.sum())} partial sums outside {STATS_REL} * sum |terms|; first at {idx}: "
                             f"got {float(got[idx])} want {float(rows[idx])} bound {float(bound[idx])}")
    return float((err / bound).max())
