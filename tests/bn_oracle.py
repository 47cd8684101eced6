"""Exact host oracle of the fused BatchNorm kernels (csrc/kernels/bn_act.cu) and of the wgmma GEMM's eval epilogue.

Given the C ABI's inputs it returns every output bit for bit: the partial rows and ``coef`` rows of the workspace,
``save_mean``, the running statistics, ``y``, the ReLU mask, ``dx``, ``dres``, dgamma and dbeta. Every operation below is an
IEEE fp32 operation rounded to nearest even; ``fma`` is one rounding (``ema_oracle.fma32``), and the expressions nvcc
contracts under its default ``-fmad=true`` are written the way the sm_90a SASS of the Makefile's build computes them.

Plan (``plan()``): ``tpr = C/8`` threads per row, ``rpp = 256/tpr`` rows per pass. A reduce grid has at most 296 CTAs of
``rows`` rows each (a multiple of rpp); thread (r, cg) of CTA g walks rows ``g*rows + r + k*rpp`` in order of k.

Forward statistics (``k_bn_fwd_stats``), per thread and channel, with the shift ``K = x[0, c]``:

    d = x - K;   t1 += d;   t2 = fma(d, d, t2)          over blocks of 64 consecutive k (kBlockPasses = 16 passes of 4)
    s1 += t1;    s2 += t2                               after each block, t1 = t2 = 0 again

Backward reduce (``k_bn_bwd_reduce``), no blocks: ``g = mask ? dz : 0;  s1 += g;  s2 = fma(g, x - save_mean, s2)``.
Both then store ``0 + red[0] + red[1] + ... + red[rpp-1]`` (the rpp row slots in order) as the CTA's partial row
``{s1, s2}`` per channel.

Merge (``merge_partials``): slot b (0..31) adds rows b, b+32, b+64, b+96 into a0..a3 while b + 96 < parts (b += 128),
then its remaining rows b, b+32, ... into a0; ``acc = (a0 + a1) + (a2 + a3)``; the xor-8 and xor-16 shuffles give warp w
``(acc[4w] + acc[4w+1]) + (acc[4w+2] + acc[4w+3])``; the total is ``0 + warp0 + ... + warp7``. The prestats forward (WALK)
first moves GEMM partial row p (shift ``x[128 p, c]``, n rows, gemm_oracle's ``part_of_row``) onto the shift ``k0 = x[0, c]``
with ``d = x[128 p, c] - k0``: ``s1' = fma(n, d, s1)``, ``s2' = fma(d, fma(n, d, 2 s1), s2)``.

Forward finalize (``k_bn_fwd_finalize``), S1 / S2 the merged sums:

    inv_m = 1 / fp32(M);   d = S1 * inv_m;   mean = K + d
    var = fma(-d, d, S2 * inv_m), negative -> 0;   invstd = rsqrtf(var + eps)                (MUFU.RSQ: see below)
    running_mean' = fma(momentum, mean, (1 - momentum) * running_mean)
    running_var'  = fma(momentum, var * (fp32(M) / fp32(M - 1)), (1 - momentum) * running_var)    (M = 1: var itself)
    a = weight * invstd;   b = fma(-mean, a, bias)                                    (coef rows 0, 1)

Apply (``k_bn_fwd_apply``): ``z = fma(a, x, b) [+ res]``; with ReLU the mask bit is ``!(z <= 0)`` and ``y = z <= 0 ? 0 : z``
(NaN passes with mask 1, as ``torch.relu`` and ``threshold_backward`` do); ``y`` is z rounded to bf16, nearest even.

Backward finalize (``k_bn_bwd_finalize``): ``S2' = S2 * invstd``; dbeta = S1, dgamma = S2'; coef = {a = weight * invstd,
gm = S1 * inv_m, c3 = (S2' * inv_m) * invstd, mu = save_mean}. Elementwise (``k_bn_bwd_elemt``), two FADD, one FFMA and
one FMUL in the SASS:

    dres = bf16(g);   dx = bf16(a * fma(-(x - mu), c3, g - gm))

Eval (``k_bn_eval_apply`` and the GEMM epilogue): ``a = weight * rsqrtf(running_var + eps)``, ``b = fma(-running_mean, a,
bias)``, then the apply above without a mask.

``rsqrtf`` compiles to MUFU.RSQ, which is not correctly rounded (2 ulp in the CUDA guide) and cannot be reproduced here.
Training: the kernel's ``save_invstd`` is checked within 2 ulps of the correctly rounded ``rsqrt(var + eps)`` of the
oracle's exact ``var`` and then fed downstream, so everything after it stays bit for bit. Eval: ``a`` is never stored, so
``eval_candidates`` gives the fp32 values within 2 ulps and a column must match for one of them.

Arrays are numpy: activations float32 [M, C] holding bf16 values, masks bool [M, C], parameters float32 [C]."""
from __future__ import annotations

import numpy as np

from ema_oracle import fma32
from gemm_oracle import BM, rows_per_part
from optimizer_oracle import bf16_bits, fma as fma_any

F32 = np.float32
THREADS, UNROLL, BLOCK_PASSES = 256, 4, 16    # bn_act.cu: kThreadsBN, kUnroll, kBlockPasses
MAX_PARTS, ELEM_CAP = 296, 1184               # reduce-grid cap (kMaxParts), elementwise-grid cap
REDUCE_CHUNK = ELEM_CHUNK = 64 << 10          # defaults of B200MPI_BN_REDUCE_CHUNK / B200MPI_BN_ELEM_CHUNK
CHANNELS = (8, 16, 32, 64, 128, 256, 512, 1024, 2048)
ROW_CHUNK = 1 << 20                           # elements per elementwise chunk


def supported(M: int, C: int) -> bool:
    return C % 8 == 0 and C >= 8 and C // 8 <= THREADS and THREADS % (C // 8) == 0 and M >= 1


def rows_per_pass(C: int) -> int:
    return THREADS // (C // 8)


def plan(M: int, C: int, cap: int, bytes_per_row: int, chunk: int):
    """(grid, rows per CTA) of ``plan()``: >= ``chunk`` bytes and >= kUnroll passes per CTA, at most ``cap`` CTAs, rows per
    CTA rounded up to whole passes."""
    rpp = rows_per_pass(C)
    g = max(1, min(-(-M // (rpp * UNROLL)), -(-(M * bytes_per_row) // chunk), cap))
    rows = -(-M // g)
    rows = -(-rows // rpp) * rpp
    return -(-M // rows), rows


def plan_rows(M: int, C: int, bytes_per_row: int, chunk: int = REDUCE_CHUNK) -> int:
    """Partial rows a reduce-type kernel writes: forward statistics read 2C bytes per row, the backward reduce 4C."""
    return plan(M, C, MAX_PARTS, bytes_per_row, chunk)[0]


# ------------------------------------------------------------------------------------------------- arithmetic --
def fma(a, b, c) -> np.ndarray:
    """fp32 fmaf: exact for finite operands; NaN / Inf as IEEE."""
    a, b, c = (np.asarray(v, dtype=F32) for v in (a, b, c))
    if np.isfinite(a).all() and np.isfinite(b).all() and np.isfinite(c).all():
        with np.errstate(over="ignore"):
            if np.isfinite(a.astype(np.float64) * b + c).all():
                return fma32(a, b, c)
    return fma_any(a, b, c)


def rsqrt_rn(v) -> np.ndarray:
    """rsqrt of fp32 values, correctly rounded to fp32 (the float64 value is within 2^-52 of exact)."""
    with np.errstate(divide="ignore", invalid="ignore"):
        return (1.0 / np.sqrt(np.asarray(v, dtype=F32).astype(np.float64))).astype(F32)


def ulps(a, b) -> np.ndarray:
    """fp32 ulp distance of finite values of one sign."""
    ia = np.asarray(a, dtype=F32).view(np.int32).astype(np.int64)
    ib = np.asarray(b, dtype=F32).view(np.int32).astype(np.int64)
    return np.abs(ia - ib)


def near(v, k: int) -> np.ndarray:
    """The fp32 value k steps (ulps) above v (below for k < 0), for positive finite v."""
    return (np.asarray(v, dtype=F32).view(np.int32) + np.int32(k)).view(F32)


def bf16(z) -> np.ndarray:
    """fp32 values rounded to bf16 (nearest even), as uint16 bit patterns."""
    return bf16_bits(z)


def bf16_value(bits) -> np.ndarray:
    return (np.asarray(bits, dtype=np.uint16).astype(np.uint32) << 16).view(F32)


def ties(z) -> int:
    """How many fp32 values lie exactly halfway between two bf16 values (round-to-nearest-even decides them)."""
    z = np.asarray(z, dtype=F32)
    return int(((z.view(np.uint32) & 0xFFFF) == 0x8000).sum())


def pack_mask(bits) -> np.ndarray:
    """bool [M, C] -> the kernel's mask bytes [M*C/8]: bit c % 8 of byte (m*C + c) / 8."""
    return np.packbits(np.asarray(bits, dtype=bool).reshape(-1, 8), axis=1, bitorder="little").reshape(-1)


def unpack_mask(packed, M: int, C: int) -> np.ndarray:
    return np.unpackbits(np.asarray(packed, dtype=np.uint8).reshape(-1, 1), axis=1, bitorder="little").reshape(M, C).astype(bool)


# ---------------------------------------------------------------------------------------------- partial rows --
def _thread_rows(M: int, C: int, grid: int, rows: int):
    """Yields (valid [grid, rpp], row index [grid, rpp]) for k = 0, 1, ...: the row thread (g, r) reads at step k."""
    rpp = rows_per_pass(C)
    base = np.arange(grid)[:, None] * rows + np.arange(rpp)[None, :]
    for k in range(rows // rpp):
        m = base + k * rpp
        yield k, m < M, np.minimum(m, M - 1)


def _block_reduce(s: np.ndarray) -> np.ndarray:
    """[grid, rpp, C] per-thread sums -> [grid, C]: 0 + red[0] + red[1] + ... in row-slot order."""
    acc = np.zeros((s.shape[0], s.shape[2]), dtype=F32)
    for q in range(s.shape[1]):
        acc = acc + s[:, q, :]
    return acc


def _interleave(s1: np.ndarray, s2: np.ndarray) -> np.ndarray:
    return np.stack([s1, s2], axis=-1).reshape(s1.shape[0], -1)


def fwd_partials(x, grid: int, rows: int, block_passes: int = BLOCK_PASSES) -> np.ndarray:
    """Partial rows [grid, 2C] of ``k_bn_fwd_stats``: {sum (x - K), sum (x - K)^2} per channel, K = x[0, c]."""
    x = np.asarray(x, dtype=F32)
    M, C = x.shape
    rpp = rows_per_pass(C)
    K = x[0]
    z = np.zeros((grid, rpp, C), dtype=F32)
    s1, s2, t1, t2 = z.copy(), z.copy(), z.copy(), z.copy()
    per_block = UNROLL * block_passes
    with np.errstate(invalid="ignore", over="ignore"):
        for k, valid, m in _thread_rows(M, C, grid, rows):
            if k % per_block == 0 and k:
                s1, s2, t1, t2 = s1 + t1, s2 + t2, z.copy(), z.copy()
            v = valid[..., None]
            d = x[m] - K
            t1 = np.where(v, t1 + d, t1)
            t2 = np.where(v, fma(d, d, t2), t2)
        s1, s2 = s1 + t1, s2 + t2
        return _interleave(_block_reduce(s1), _block_reduce(s2))


def bwd_partials(dz, x, mask, save_mean, grid: int, rows: int) -> np.ndarray:
    """Partial rows [grid, 2C] of ``k_bn_bwd_reduce``: {sum g, sum g (x - save_mean)}, g = mask ? dz : 0."""
    dz, x = np.asarray(dz, dtype=F32), np.asarray(x, dtype=F32)
    M, C = x.shape
    rpp = rows_per_pass(C)
    mu = np.asarray(save_mean, dtype=F32)
    s1 = np.zeros((grid, rpp, C), dtype=F32)
    s2 = s1.copy()
    with np.errstate(invalid="ignore", over="ignore"):
        for _, valid, m in _thread_rows(M, C, grid, rows):
            v = valid[..., None]
            g = dz[m] if mask is None else np.where(mask[m], dz[m], F32(0))
            s1 = np.where(v, s1 + g, s1)
            s2 = np.where(v, fma(g, x[m] - mu, s2), s2)
        return _interleave(_block_reduce(s1), _block_reduce(s2))


def walk_rows(x, parts: int):
    """WALK merge inputs of the prestats forward: for GEMM partial row p, (d_p = x[128 p, c] - x[0, c], n_p) as [parts, C]
    fp32 and [parts] fp32."""
    x = np.asarray(x, dtype=F32)
    M = x.shape[0]
    d = x[np.arange(parts) * BM] - x[0]
    n = rows_per_part(M, parts).numpy().astype(F32)
    return d, n


def merge(P, walk=None, order: str = "pairs") -> np.ndarray:
    """``merge_partials`` over partial rows P [parts, nout] -> [nout]. ``walk`` = walk_rows(x, parts) for the prestats
    forward. ``order="serial"`` is a kernel mistake for the oracle's own tests: ((a0 + a1) + a2) + a3."""
    P = np.asarray(P, dtype=F32)
    parts, nout = P.shape
    with np.errstate(invalid="ignore", over="ignore"):
        if walk is not None:
            d, n = walk
            s1 = P[:, 0::2]
            rows = np.empty_like(P)
            rows[:, 0::2] = fma(n[:, None], d, s1)
            rows[:, 1::2] = fma(d, fma(n[:, None], d, F32(2) * s1), P[:, 1::2])
            P = rows
        acc = np.zeros((32, nout), dtype=F32)
        for slot in range(32):
            a = [np.zeros(nout, dtype=F32) for _ in range(4)]
            b = slot
            while b + 96 < parts:
                for i in range(4):
                    a[i] = a[i] + P[b + 32 * i]
                b += 128
            while b < parts:
                a[0] = a[0] + P[b]
                b += 32
            acc[slot] = ((a[0] + a[1]) + a[2]) + a[3] if order == "serial" else (a[0] + a[1]) + (a[2] + a[3])
        tot = np.zeros(nout, dtype=F32)
        for w in range(8):
            tot = tot + ((acc[4 * w] + acc[4 * w + 1]) + (acc[4 * w + 2] + acc[4 * w + 3]))
    return tot


# ------------------------------------------------------------------------------------------------- finalize --
def fwd_finalize(tot, x0, M: int, weight, bias, running_mean, running_var, eps, momentum, invstd=None,
                 unbiased: bool = True) -> dict:
    """``k_bn_fwd_finalize`` from the merged sums ``tot`` [2C] and the shift row ``x0 = x[0]``. ``invstd`` is the kernel's
    save_invstd (None: the correctly rounded value). Returns var, rsqrt_rn (correctly rounded rsqrt(var + eps)), mean,
    invstd, a, b and, if running_mean is given, rm / rv. ``unbiased=False`` is a kernel mistake for the oracle's tests."""
    tot = np.asarray(tot, dtype=F32)
    S1, S2 = tot[0::2], tot[1::2]
    with np.errstate(invalid="ignore", over="ignore"):
        inv_m = F32(1) / F32(M)
        d = S1 * inv_m
        mean = np.asarray(x0, dtype=F32) + d
        var = fma(-d, d, S2 * inv_m)
        var = np.where(var < 0, F32(0), var).astype(F32)
        ref = rsqrt_rn(var + F32(eps))
        inv = ref if invstd is None else np.asarray(invstd, dtype=F32)
        out = dict(mean=mean, var=var, rsqrt_rn=ref, invstd=inv)
        mom = F32(momentum)
        keep = F32(1) - mom
        if running_mean is not None:
            out["rm"] = fma(mom, mean, keep * np.asarray(running_mean, dtype=F32))
            uv = var * (F32(M) / F32(M - 1)) if M > 1 and unbiased else var
            out["rv"] = fma(mom, uv, keep * np.asarray(running_var, dtype=F32))
        a = inv if weight is None else np.asarray(weight, dtype=F32) * inv
        out["a"] = a
        out["b"] = fma(-mean, a, F32(0) if bias is None else np.asarray(bias, dtype=F32))
    return out


def bwd_finalize(tot, M: int, weight, save_mean, save_invstd) -> dict:
    """``k_bn_bwd_finalize``: dbeta, dgamma and the coef rows a, gm, c3, mu."""
    tot = np.asarray(tot, dtype=F32)
    inv = np.asarray(save_invstd, dtype=F32)
    with np.errstate(invalid="ignore", over="ignore"):
        inv_m = F32(1) / F32(M)
        S1, S2 = tot[0::2], tot[1::2] * inv
        return dict(dbeta=S1, dgamma=S2, a=inv if weight is None else np.asarray(weight, dtype=F32) * inv,
                    gm=S1 * inv_m, c3=(S2 * inv_m) * inv, mu=np.asarray(save_mean, dtype=F32))


# ------------------------------------------------------------------------------------------------ elementwise --
def _chunks(M: int, C: int):
    step = max(1, ROW_CHUNK // C)
    for lo in range(0, M, step):
        yield lo, min(M, lo + step)


def apply(x, res, a, b, relu: bool, mask_ge: bool = False):
    """``k_bn_fwd_apply`` / ``k_bn_eval_apply``: (y as bf16 bits [M, C], mask bool [M, C] or None, z fp32 [M, C]).
    ``mask_ge`` is a kernel mistake for the oracle's tests: the pre-fix ``z >= 0`` test for the mask."""
    x = np.asarray(x, dtype=F32)
    M, C = x.shape
    z = np.empty((M, C), dtype=F32)
    with np.errstate(invalid="ignore", over="ignore"):
        for lo, hi in _chunks(M, C):
            t = fma(a, x[lo:hi], b)
            if res is not None:
                t = t + np.asarray(res[lo:hi], dtype=F32)
            z[lo:hi] = t
    if not relu:
        return bf16(z), None, z
    keep = ~(z <= 0)
    return bf16(np.where(keep, z, F32(0))), z >= 0 if mask_ge else keep, z


def elemt(dz, x, mask, co: dict, with_res: bool):
    """``k_bn_bwd_elemt``: (dx bits, dres bits or None, the fp32 dx before rounding)."""
    dz, x = np.asarray(dz, dtype=F32), np.asarray(x, dtype=F32)
    M, C = x.shape
    out = np.empty((M, C), dtype=F32)
    g = dz if mask is None else np.where(mask, dz, F32(0))
    with np.errstate(invalid="ignore", over="ignore"):
        for lo, hi in _chunks(M, C):
            t = x[lo:hi] - co["mu"]
            out[lo:hi] = co["a"] * fma(-t, co["c3"], g[lo:hi] - co["gm"])
    return bf16(out), bf16(g) if with_res else None, out


def eval_coef(weight, bias, running_mean, rsq):
    """(a, b) of the eval kernels for a given fp32 ``rsq = rsqrtf(running_var + eps)``."""
    rsq = np.asarray(rsq, dtype=F32)
    with np.errstate(invalid="ignore", over="ignore"):
        a = rsq if weight is None else np.asarray(weight, dtype=F32) * rsq
        return a, fma(-np.asarray(running_mean, dtype=F32), a, F32(0) if bias is None else np.asarray(bias, dtype=F32))


def eval_candidates(running_var, eps, spread: int = 2):
    """[2 spread + 1, C] fp32 candidates for rsqrtf(running_var + eps): the correctly rounded value and its neighbours."""
    ref = rsqrt_rn(np.asarray(running_var, dtype=F32) + F32(eps))
    return np.stack([near(ref, k) for k in range(-spread, spread + 1)])


def eval_match(y_bits, x, res, weight, bias, running_mean, running_var, eps, relu: bool) -> np.ndarray:
    """Per channel, the offset (in ulps from the correctly rounded rsqrt) of the first candidate whose whole column
    reproduces the kernel's bf16 output ``y_bits`` [M, C], or a large value where none does."""
    cands = eval_candidates(running_var, eps)
    C = cands.shape[1]
    found = np.full(C, 99)
    y_bits = np.asarray(y_bits, dtype=np.uint16)
    for i, rsq in enumerate(cands):
        a, b = eval_coef(weight, bias, running_mean, rsq)
        want, _, _ = apply(x, res, a, b, relu)
        ok = (want == y_bits).all(0) & (found == 99)
        found[ok] = i - (len(cands) // 2)
    return found


# ---------------------------------------------------------------------------------- against the kernels' outputs --
def to_np(t) -> np.ndarray:
    """A CUDA / CPU tensor (bf16 or fp32) as numpy float32 (bf16 widens exactly)."""
    return t.detach().float().cpu().numpy()


def _bits(a) -> np.ndarray:
    import torch
    if isinstance(a, torch.Tensor):
        a = a.detach().cpu()
        if a.dtype == torch.bfloat16:
            return a.contiguous().view(torch.int16).numpy().view(np.uint16)
        if a.dtype == torch.uint8:
            return a.numpy()
        return a.float().contiguous().numpy().view(np.uint32)
    a = np.asarray(a)
    return a if a.dtype in (np.uint16, np.uint8) else a.astype(F32).view(np.uint32)


def assert_bits(got, want, what: str) -> None:
    """Bitwise equality; ``want`` is a numpy fp32 array, bf16 bits (uint16) or mask bytes (uint8)."""
    g, w = _bits(got).reshape(-1), _bits(want).reshape(-1)
    assert g.shape == w.shape, f"{what}: {g.shape} vs {w.shape}"
    bad = np.nonzero(g != w)[0]
    if bad.size:
        i = int(bad[0])
        raise AssertionError(f"{what}: {bad.size} of {g.size} differ; first at flat index {i}: got {g[i]:#x} want {w[i]:#x}")


def _opt(t):
    return None if t is None else to_np(t)


SAMPLE_ELEMS = 1 << 22     # elementwise outputs compared per call: every row up to this, a row sample beyond it


def sample_rows(M: int, C: int) -> np.ndarray:
    """Rows whose elementwise outputs are compared: all of them for small tensors; else the first and last 2048 and an
    evenly strided sample in between (every row is computed by the same code, so a sample across all CTAs of the
    elementwise grid sees a wrong formula as surely as every row does; the reductions are always compared in full)."""
    if M * C <= SAMPLE_ELEMS:
        return np.arange(M)
    stride = -(-M * C // (SAMPLE_ELEMS // 2))
    return np.unique(np.concatenate([np.arange(2048), np.arange(M - 2048, M), np.arange(0, M, stride)]))


def check_forward(x, res, y, mask, save_mean, save_invstd, ws, weight, bias, rm0, rv0, rm, rv, eps, momentum, relu,
                  chunk: int = REDUCE_CHUNK, pre=None, what: str = ""):
    """One forward call of bn_act.cu against the oracle, stage by stage: partial rows (``b200mpi_bn_act_fwd``; rows past
    the grid must still be NaN) or the WALK merge of ``pre = (partials [parts, 2C], parts)`` (the prestats forward), then
    save_invstd within 2 ulps, save_mean, running statistics and coef rows bitwise, then y and the mask bitwise (on the
    rows of ``sample_rows``).
    ``x`` / ``res`` / ``y`` are [M, C] views. Returns (the oracle's finalize dict, bf16 ties among the outputs)."""
    M, C = x.shape
    xn = to_np(x)
    wsn = to_np(ws)
    if pre is None:
        grid, rows = plan(M, C, MAX_PARTS, 2 * C, chunk)
        part = wsn[4 * C:4 * C + MAX_PARTS * 2 * C].reshape(MAX_PARTS, 2 * C)
        assert np.isnan(part[grid:]).all(), f"{what}: partial rows past the grid of {grid} written"
        P = fwd_partials(xn, grid, rows)
        assert_bits(part[:grid], P, f"{what} forward partial rows")
        tot = merge(P)
    else:
        P, parts = pre
        tot = merge(to_np(P).reshape(parts, 2 * C), walk=walk_rows(xn, parts))
    inv = to_np(save_invstd)
    fin = fwd_finalize(tot, xn[0], M, _opt(weight), _opt(bias), _opt(rm0), _opt(rv0), eps, momentum, invstd=inv)
    u = ulps(inv, fin["rsqrt_rn"])
    assert (u <= 2).all(), f"{what}: save_invstd {int(u.max())} ulps from the correctly rounded rsqrt"
    assert_bits(save_mean, fin["mean"], f"{what} save_mean")
    if rm is not None:
        assert_bits(rm, fin["rm"], f"{what} running_mean")
        assert_bits(rv, fin["rv"], f"{what} running_var")
    assert_bits(wsn[:C], fin["a"], f"{what} coef a")
    assert_bits(wsn[C:2 * C], fin["b"], f"{what} coef b")
    rows = sample_rows(M, C)
    yb, mk, z = apply(xn[rows], None if res is None else to_np(res)[rows], fin["a"], fin["b"], relu)
    assert_bits(_bits(y).reshape(M, C)[rows], yb, f"{what} y")
    if relu:
        assert_bits(_bits(mask).reshape(M, C // 8)[rows], pack_mask(mk), f"{what} mask")
    return fin, ties(z)


def check_backward(dz, x, mask, dx, dres, dgamma, dbeta, ws, weight, save_mean, save_invstd, relu,
                   chunk: int = REDUCE_CHUNK, pre=None, what: str = "") -> int:
    """One backward call against the oracle: partial rows (or ``pre = (partials, parts)``), the four coef rows, dgamma /
    dbeta, dx and dres (on the rows of ``sample_rows``), all bitwise. Returns the number of bf16 ties among dx."""
    M, C = x.shape
    xn, dzn = to_np(x), to_np(dz)
    wsn = to_np(ws)
    mk = unpack_mask(mask.cpu().numpy(), M, C) if relu else None
    mu, inv = to_np(save_mean), to_np(save_invstd)
    if pre is None:
        grid, rows = plan(M, C, MAX_PARTS, 4 * C, chunk)
        part = wsn[4 * C:4 * C + MAX_PARTS * 2 * C].reshape(MAX_PARTS, 2 * C)
        assert np.isnan(part[grid:]).all(), f"{what}: backward partial rows past the grid of {grid} written"
        P = bwd_partials(dzn, xn, mk, mu, grid, rows)
        assert_bits(part[:grid], P, f"{what} backward partial rows")
    else:
        P = to_np(pre[0]).reshape(pre[1], 2 * C)
    co = bwd_finalize(merge(P), M, _opt(weight), mu, inv)
    for i, k in enumerate(("a", "gm", "c3", "mu")):
        assert_bits(wsn[i * C:(i + 1) * C], co[k], f"{what} backward coef {k}")
    if dgamma is not None:
        assert_bits(dgamma, co["dgamma"], f"{what} dgamma")
    if dbeta is not None:
        assert_bits(dbeta, co["dbeta"], f"{what} dbeta")
    rows = sample_rows(M, C)
    dxb, dresb, dx32 = elemt(dzn[rows], xn[rows], None if mk is None else mk[rows], co, dres is not None)
    assert_bits(_bits(dx).reshape(M, C)[rows], dxb, f"{what} dx")
    if dres is not None:
        assert_bits(_bits(dres).reshape(M, C)[rows], dresb, f"{what} dres")
    return ties(dx32)
