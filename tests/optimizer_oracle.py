"""Exact host oracle of the fused allreduce+SGD and allreduce+LARS steps (``k_allreduce_sgd`` in
csrc/kernels/collectives.cu, ``k_allreduce_lars_norms`` / ``k_lars_update`` in csrc/kernels/lars.cu).

The kernels' contract, every operation an IEEE fp32 operation rounded to nearest even:

    S  = fp32 sum of the ranks' gradients (widened to fp32) in the slice owner's order: owner, owner+1, ... (mod world)
         (NVLS: the switch adds in an unknown order, so inputs must have an exact sum; bf16 / f16 sums come back rounded
         to T)
    d  = fmaf(S, scale, fmul(wd, p))                  LARS: d = fmul(t, fmaf(S, scale, fmul(wd, p)))
    m' = first_step ? d : fmaf(mu, m, d)
    p' = fmaf(-lr, nesterov ? fmaf(mu, m', d) : m', p)
    shadow = bf16 round-to-nearest-even of p'

and LARS's trust ratio of a parameter, from gs = fp32(S * scale) over its elements:

    sg, sp = fp32 sums of fmaf(gs, gs, .) / fmaf(w, w, .)     order: per rank slice along the grid, then ranks 0..W-1
    gn = sqrtf(sg), wn = sqrtf(sp)
    t  = (wn > 0 && gn > 0) ? fdiv(fmul(eta, wn), fadd(fmaf(wd, wn, gn), 1e-8f)) : 1

The order of the norm sums within a slice depends on the grid, so the host states them exactly only when every order
gives the same bits (``lars_norm_interval`` asserts that precondition), and otherwise bounds the trust ratio; the update
is then exact *given* the kernel's trust (``lars_step``).

Arrays are numpy float32; hyper-parameters are fp32 values (what the C ABI receives), scalars or per-element arrays."""
import math
from typing import Optional, Sequence

import numpy as np
import torch

from collective_oracle import exact_sum
from ema_oracle import fma32

F32 = np.float32
LARS_EPS = F32(1e-8)
U32 = 2.0 ** -24            # unit roundoff of fp32


def vec_elems(dtype) -> int:
    """Elements per 16-byte vector of the gradient dtype: 4 for fp32, 8 for bf16 / f16."""
    return 4 if dtype == torch.float32 else 8


def slice_vecs(count: int, world: int, dtype) -> int:
    """Vectors per rank slice (``b200mpi_slice_elems(count) / N``)."""
    nvec = -(-count // vec_elems(dtype))
    return -(-nvec // world)


def fma(a, b, c) -> np.ndarray:
    """fp32 fmaf, element-wise, for any inputs: exact (``ema_oracle.fma32``) where the operands and the result are finite,
    otherwise the float64 value rounded to fp32 (NaN / Inf propagate as in IEEE, overflow goes to Inf)."""
    shape = np.broadcast_shapes(*(np.shape(v) for v in (a, b, c)))
    a, b, c = np.broadcast_arrays(*(np.atleast_1d(np.asarray(v, dtype=F32)) for v in (a, b, c)))
    with np.errstate(all="ignore"):
        wide = (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(F32)
    ok = np.isfinite(a) & np.isfinite(b) & np.isfinite(c) & np.isfinite(wide)
    out = wide.copy()
    if ok.any():
        out[ok] = fma32(a[ok], b[ok], c[ok])
    return out.reshape(shape)


def fmul(a, b) -> np.ndarray:
    with np.errstate(all="ignore"):
        return np.multiply(np.asarray(a, dtype=F32), np.asarray(b, dtype=F32), dtype=F32)


def bf16_bits(x) -> np.ndarray:
    """bf16 round-to-nearest-even of fp32 values, as uint16 bit patterns (NaN stays NaN)."""
    x = np.asarray(x, dtype=F32)
    u = np.atleast_1d(x).view(np.uint32).astype(np.uint64)
    r = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)
    nan = np.isnan(np.atleast_1d(x))
    r[nan] = ((u[nan] >> 16) | 0x40).astype(np.uint16)
    return r.reshape(x.shape)


def round_to(x, dtype) -> np.ndarray:
    """fp32 values rounded to the gradient dtype and widened back."""
    x = np.asarray(x, dtype=F32)
    if dtype == torch.float32:
        return x
    if dtype == torch.float16:
        with np.errstate(all="ignore"):
            return x.astype(np.float16).astype(F32)
    return (bf16_bits(x).astype(np.uint32) << 16).view(F32)


def owner_sum(grads: Sequence[np.ndarray], world: int, dtype, nvls: bool = False) -> np.ndarray:
    """S: the ranks' gradients (widened to fp32, one array per rank) summed in fp32 in the slice owner's order."""
    g = np.stack([np.asarray(x, dtype=F32) for x in grads])
    assert g.shape[0] == world
    count = g.shape[1]
    if nvls:
        s = exact_sum([torch.from_numpy(x.astype(np.float64)) for x in g]).numpy().astype(F32)
        return round_to(s, dtype)
    N = vec_elems(dtype)
    per = slice_vecs(count, world, dtype) * N
    out = np.empty(count, dtype=F32)
    for r in range(world):
        lo, hi = min(r * per, count), min((r + 1) * per, count)
        if lo == hi:
            continue
        acc = g[r, lo:hi].copy()
        for k in range(1, world):
            with np.errstate(all="ignore"):
                acc = acc + g[(r + k) % world, lo:hi]
        out[lo:hi] = acc
    return out


def expand_groups(table, gmap, count: int):
    """Per-element {lr, mu, wd} fp32 arrays from a [G, 3] table and one group per 4-element vector."""
    table = np.asarray(table, dtype=F32)
    rows = table[np.repeat(np.asarray(gmap, dtype=np.int64), 4)[:count]]
    return rows[:, 0], rows[:, 1], rows[:, 2]


def sgd_step(p, m, S, scale, lr, mu, wd, nesterov: bool, first: bool, trust=None):
    """(p', m', bf16 shadow bits) of one fused step; ``trust`` (per element) makes it the LARS update."""
    p = np.asarray(p, dtype=F32)
    S = np.asarray(S, dtype=F32)
    d = fma(S, F32(scale), fmul(wd, p))
    if trust is not None:
        d = fmul(trust, d)
    mn = d if first else fma(mu, np.asarray(m, dtype=F32), d)
    upd = fma(mu, mn, d) if nesterov else mn
    pn = fma(-np.asarray(lr, dtype=F32), upd, p)
    return pn, mn, bf16_bits(pn)


def lars_step(p, m, S, scale, trust, lr, mu, wd, nesterov: bool, first: bool):
    """The LARS update given a per-element trust ratio (the kernel's own ``trust_out`` expanded over its parameter)."""
    return sgd_step(p, m, S, scale, lr, mu, wd, nesterov, first, trust=np.asarray(trust, dtype=F32))


def lars_trust(sg, sp, eta, wd) -> np.ndarray:
    """t from the fp32 sums of squares, exactly (np.sqrt on float32 is correctly rounded, as the non-fast-math sqrtf)."""
    sg, sp = np.asarray(sg, dtype=F32), np.asarray(sp, dtype=F32)
    with np.errstate(all="ignore"):
        gn, wn = np.sqrt(sg), np.sqrt(sp)
        den = np.add(fma(wd, wn, gn), LARS_EPS, dtype=F32)
        t = np.divide(fmul(eta, wn), den, dtype=F32)
    return np.where((wn > 0) & (gn > 0), t, F32(1.0)).astype(F32)


def _exact_sum_of_squares(x: np.ndarray) -> Optional[np.float32]:
    """The fp32 sum of x*x if every order of fmaf(x, x, .) gives it exactly, else None: every square is a multiple of
    2^e (e from the smallest nonzero square) and the sum of the squares is below 2^(24+e), and 2^e is an fp32 number."""
    x = np.asarray(x, dtype=np.float64)
    nz = x[x != 0]
    if nz.size == 0:
        return F32(0.0)
    sq = nz * nz                                     # exact: fp32 values have 24 significant bits
    mant, ex = np.frexp(sq)
    mi = (mant * 2.0 ** 53).astype(np.int64)         # sq == mi * 2^(ex - 53) exactly
    low = np.log2((mi & -mi).astype(np.float64)).astype(np.int64) + ex - 53
    e = int(low.min())                               # the largest 2^e that divides every square
    if e < -149:
        return None
    total = math.fsum(sq)
    if total >= 2.0 ** (24 + e) or total >= float(np.finfo(F32).max):
        return None
    return F32(total)


def lars_norm_interval(gs, w, world: int, eta, wd, exact: bool = False):
    """Trust of one LARS parameter from its scaled gradient ``gs = fp32(S*scale)`` and weights ``w`` (fp32 arrays).

    If every order of the norm sums gives the same fp32 sums, returns ``(t, t)`` with the one correct trust; with
    ``exact=True`` that precondition is asserted. Otherwise returns float64 bounds ``(lo, hi)``: each sum of squares is
    within gamma_n of its exact value (n = elements + world), and sqrt, fmul, fmaf, fadd and fdiv each add one rounding."""
    gs, w = np.asarray(gs, dtype=F32), np.asarray(w, dtype=F32)
    if not np.isfinite(gs).all():
        # sg is NaN (t = 1) or +Inf (t = 0 for any finite wn > 0): the value of a finite weight norm does not matter
        assert np.isfinite(w).all()
        sg = F32(np.nan) if np.isnan(gs).any() else F32(np.inf)
        sp = F32(math.fsum(np.asarray(w, dtype=np.float64) ** 2))
        t = lars_trust(sg, sp, eta, wd)
        return float(t), float(t)
    sg, sp = _exact_sum_of_squares(gs), _exact_sum_of_squares(w)
    if sg is not None and sp is not None:
        t = lars_trust(sg, sp, eta, wd)
        return float(t), float(t)
    assert not exact, "oracle precondition: these norm sums depend on the order of the adds"
    assert float(wd) >= 0
    n = gs.size + world
    gam = n * U32 / (1 - n * U32)
    qg = math.fsum(np.asarray(gs, dtype=np.float64) ** 2)
    qp = math.fsum(np.asarray(w, dtype=np.float64) ** 2)
    assert qg > 0 and qp > 0 and qg * (1 + gam) < float(np.finfo(F32).max), "interval: norms must be positive and finite"
    assert qg * (1 - gam) > 2.0 ** -126 and qp * (1 - gam) > 2.0 ** -126, "interval: sums must stay normal"
    lo_u, hi_u = 1 - U32, 1 + U32
    slack = 1 + 2.0 ** -50                           # the float64 arithmetic of the bounds themselves
    wn = (math.sqrt(qp * (1 - gam)) * lo_u / slack, math.sqrt(qp * (1 + gam)) * hi_u * slack)
    gn = (math.sqrt(qg * (1 - gam)) * lo_u / slack, math.sqrt(qg * (1 + gam)) * hi_u * slack)
    eta, wd = float(F32(eta)), float(F32(wd))
    num = (eta * wn[0] * lo_u / slack, eta * wn[1] * hi_u * slack)
    den = ((((wd * wn[0] + gn[0]) * lo_u) + float(LARS_EPS)) * lo_u / slack,
           (((wd * wn[1] + gn[1]) * hi_u) + float(LARS_EPS)) * hi_u * slack)
    return num[0] / den[1] * lo_u / slack, num[1] / den[0] * hi_u * slack
